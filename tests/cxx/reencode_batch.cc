// C++ caller in the shape of "xc-enc --reencode" (frontend/xc-enc.cc:262-327) for several chunks at once, written against
// the host mirror: every chunk's prediction stream is parsed by its own Decoder (labels kept), every chunk gets an Encoder
// built from its deserialized Decoder, and the chunks are walked frame position by frame position -- Encoder::reencode's
// options 2 and 4 (update_residues) of all chunks at a position go through one alfalfa_gpu::update_residues_batch,
// options 1 and 3 stay single calls.  Afterwards the error path: the same Encoder twice in one batch must throw.
// usage: reencode_batch OUT_PREFIX WIDTH HEIGHT KF_Q_WEIGHT EXTRA_FRAME_CHUNK (TARGETS.yuv PRED.ivf STATE.bin)...
// OUT_PREFIX.<chunk>.ivf gets each chunk's emitted frames (32-byte DKIF header, 12-byte frame headers).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <string>
#include <vector>

#include "../../alfalfa_b200/host/alfalfa_gpu.hh"

using namespace alfalfa_gpu;

static std::vector<uint8_t> slurp(const char* path) {
  std::vector<uint8_t> b;
  FILE* f = fopen(path, "rb");
  if (!f) throw std::runtime_error(std::string("cannot open ") + path);
  uint8_t buf[65536];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) b.insert(b.end(), buf, buf + n);
  fclose(f);
  return b;
}
static uint32_t le32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (uint32_t(p[3]) << 24); }

static void write_ivf(const std::string& path, int w, int h, const std::vector<std::vector<uint8_t>>& out) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) throw std::runtime_error("cannot write output");
  uint8_t hdr[32] = {'D', 'K', 'I', 'F', 0, 0, 32, 0, 'V', 'P', '8', '0'};
  hdr[12] = w & 255, hdr[13] = w >> 8, hdr[14] = h & 255, hdr[15] = h >> 8;
  hdr[16] = 1, hdr[20] = 1;
  hdr[24] = out.size() & 255, hdr[25] = (out.size() >> 8) & 255;
  fwrite(hdr, 1, 32, f);
  for (size_t i = 0; i < out.size(); i++) {
    uint8_t fh[12] = {0};
    const uint32_t n = (uint32_t)out[i].size();
    fh[0] = n & 255, fh[1] = (n >> 8) & 255, fh[2] = (n >> 16) & 255, fh[3] = n >> 24;
    fh[4] = i & 255, fh[5] = (i >> 8) & 255;
    fwrite(fh, 1, 12, f);
    fwrite(out[i].data(), 1, out[i].size(), f);
  }
  fclose(f);
}

struct ChunkInput {
  std::vector<uint8_t> targets;
  std::vector<ParsedFrame> prediction_frames;
  std::vector<SourceFrame> original_rasters;
  std::vector<std::vector<uint8_t>> out;
};

int main(int argc, char** argv) {
  try {
    if (argc < 9 || (argc - 6) % 3 != 0) {
      fprintf(stderr, "usage: reencode_batch OUT_PREFIX W H KF_Q_WEIGHT EXTRA_FRAME_CHUNK (TARGETS.yuv PRED.ivf STATE.bin)...\n");
      return 2;
    }
    const int w = atoi(argv[2]), h = atoi(argv[3]);
    const double kf_q_weight = atof(argv[4]);
    const bool extra_frame_chunk = atoi(argv[5]) != 0;
    const size_t n_chunks = (argc - 6) / 3;
    const size_t cw = (w + 1) / 2, ch = (h + 1) / 2, frame_bytes = size_t(w) * h + 2 * cw * ch;

    Context ctx(0, w, h);
    std::vector<ChunkInput> chunks(n_chunks);
    std::vector<Encoder> encoders;
    for (size_t c = 0; c < n_chunks; c++) {
      ChunkInput& k = chunks[c];
      k.targets = slurp(argv[6 + 3 * c]);
      const std::vector<uint8_t> ivf = slurp(argv[7 + 3 * c]), state = slurp(argv[8 + 3 * c]);
      if (ivf.size() < 32 || memcmp(ivf.data(), "DKIF", 4) != 0) throw std::runtime_error("not an IVF file");
      Decoder pred_decoder(ctx, w, h);
      for (size_t off = 32; off + 12 <= ivf.size();) {
        const uint32_t n = le32(&ivf[off]);
        off += 12;
        if (off + n > ivf.size()) throw std::runtime_error("truncated IVF");
        ParsedFrame frame = pred_decoder.parse_frame(Chunk{&ivf[off], n}, true);
        pred_decoder.decode_frame(frame);
        k.prediction_frames.push_back(frame);
        off += n;
      }
      if (k.targets.size() < frame_bytes * k.prediction_frames.size()) throw std::runtime_error("target input too short");
      for (size_t i = 0; i < k.prediction_frames.size(); i++) {
        const uint8_t* p = k.targets.data() + i * frame_bytes;
        k.original_rasters.push_back(SourceFrame{p, p + size_t(w) * h, p + size_t(w) * h + cw * ch, size_t(w), cw});
      }
      encoders.emplace_back(Decoder::deserialize(ctx, state, w, h));
    }

    // Encoder::reencode (reencode.cc:315-381) position by position over all chunks
    auto qi_of = [](const ParsedFrame& f) {
      const int q = f.y_ac_qi();
      if (q < 0) throw LogicError("reencode: prediction frames must be parsed with keep_labels");
      return q;
    };
    size_t longest = 0;
    for (const ChunkInput& k : chunks) longest = std::max(longest, k.prediction_frames.size());
    for (size_t i = extra_frame_chunk ? 1 : 0; i < longest; i++) {
      std::vector<ReencodeJob> batch;
      std::vector<size_t> of;
      for (size_t c = 0; c < n_chunks; c++) {
        ChunkInput& k = chunks[c];
        const std::vector<ParsedFrame>& pf = k.prediction_frames;
        if (i >= pf.size()) continue;
        const bool first = i == (extra_frame_chunk ? 1u : 0u), last = i == pf.size() - 1;
        if (first && pf[i].key_frame()) {  // option 1
          int qi = qi_of(pf[i]);
          if (i + 1 < pf.size() && !pf[i + 1].key_frame()) qi = (int)lrint(kf_q_weight * qi_of(pf[i]) + (1 - kf_q_weight) * qi_of(pf[i + 1]));
          k.out.push_back(encoders[c].reencode_as_interframe(k.original_rasters[i], pf[i], (uint8_t)qi));
        } else if (first && extra_frame_chunk) {  // option 2
          if (!pf[0].key_frame()) throw std::runtime_error("extra-frame chunks must start with a keyframe.");
          const int qi = (int)lrint(kf_q_weight * qi_of(pf[0]) + (1 - kf_q_weight) * qi_of(pf[i]));
          batch.push_back(ReencodeJob{&encoders[c], k.original_rasters[i], &pf[i], qi, last});
          of.push_back(c);
        } else if (pf[i].key_frame()) {  // option 3
          k.out.push_back(encoders[c].write_frame(pf[i]));
        } else {  // option 4
          batch.push_back(ReencodeJob{&encoders[c], k.original_rasters[i], &pf[i], -1, last});
          of.push_back(c);
        }
      }
      const std::vector<std::vector<uint8_t>> frames = update_residues_batch(batch);
      for (size_t j = 0; j < frames.size(); j++) chunks[of[j]].out.push_back(frames[j]);
    }
    for (size_t c = 0; c < n_chunks; c++) write_ivf(std::string(argv[1]) + "." + std::to_string(c) + ".ivf", w, h, chunks[c].out);

    // the same Encoder twice: the whole call is refused and nothing moves
    const uint32_t before = encoders[0].minihash();
    const ChunkInput& k = chunks[0];
    const size_t i = k.prediction_frames.size() - 1;
    bool thrown = false;
    try {
      update_residues_batch({ReencodeJob{&encoders[0], k.original_rasters[i], &k.prediction_frames[i], -1, false},
                             ReencodeJob{&encoders[0], k.original_rasters[i], &k.prediction_frames[i], -1, false}});
    } catch (const LogicError&) {
      thrown = true;
    }
    if (!thrown || encoders[0].minihash() != before) throw std::runtime_error("the same Encoder twice was not refused");
    printf("ok %zu\n", n_chunks);
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "exception: %s\n", e.what());
    return 1;
  }
}
