// engine.h -- device-side job description shared by kernels.cu (device code) and
// engine.cu (host orchestration).  Internal to the library; the public surface is
// include/vp8gpu.h.
#pragma once
#include <stdint.h>

#include "../../include/vp8gpu.h"

// Kernel launches go through one macro: in the product build it is the ordinary <<< >>> launch; the test-only
// SIMT-emulated build (tests/simt: the same sources compiled with g++, kernels run as fibers on the CPU to check
// their logic where there is no GPU; never part of libvp8gpu.so) turns it into a call of the emulator.
#ifdef VP8GPU_SIMT_EMUL
#define VP8_LAUNCH(kern, grid, block, smem, stream) ::simt::make_launch((grid), (block), (smem), [](auto... a_) { kern(a_...); })
#else
#define VP8_LAUNCH(kern, grid, block, smem, stream) kern<<<(grid), (block), (smem), (stream)>>>
#endif

namespace vp8 {

// Geometry of every raster of a context.  Planes live in one allocation:
//   Y at 0 (y_pitch x H), U at u_off, V at v_off (c_pitch x H/2 each).
// Pitches are multiples of 32 / 16 bytes so rows can be moved as 16-byte / 8-byte vectors.
struct Geom {
  int mb_cols, mb_rows;
  int W, H;              // MB-aligned luma size (16*mb_cols, 16*mb_rows), VP8Raster dims
  int y_pitch, c_pitch;  // bytes
  uint32_t u_off, v_off; // byte offsets of the chroma planes
  uint32_t frame_bytes;
  // Wavefront hand-over areas behind the pixels of every raster (zeroed once when the raster is allocated):
  // rows of one frame pass their edges to the row below as 8-byte { data, epoch } words -- the flag travels
  // in the same store as the data, so neither side needs a fence (kernels.cu "hand-over messages").
  //   loop filter: [mb_rows][mb_cols + 1][32] words, intra prediction: [mb_rows][mb_cols][8] words
  uint32_t msg_lf_off, msg_intra_off;
  uint32_t alloc_bytes;  // pixels + both areas
};

// One frame's decode job as the kernels see it (an array of these lives in HBM).
struct DevJob {
  const vp8gpu_mb* mbs;
  const vp8gpu_token* tokens;
  const vp8gpu_split_mvs* split;
  uint8_t* out;
  const uint8_t* ref[3];   // last, golden, altref (ref_frame - 1)
  const void* ref_tmap[3]; // per reference: its three TMA tensor maps (Y, U, V; 128 bytes each) in HBM
  int* intra_progress;     // [mb_rows] wavefront counters, zeroed before launch
  int* lf_progress;        // [mb_rows]
  vp8gpu_quant quant[4];
  uint8_t key_frame, sharpness, lf_enabled;
  uint8_t lf_force;        // != 0: every macroblock is filtered at this level instead of its record's
                           // (the encoder's loop-filter search, encoder.cc:460-508)
  uint32_t n_intra;        // intra-coded macroblocks in the frame
  uint32_t n_inter;
  uint32_t pad2;
};

// One frame's ENCODE job (device pointers): one wavefront pass that takes the reference encoder's
// decisions macroblock by macroblock (encoder/encode_intra.cc, encode_inter.cc), transforms, quantises,
// emits tokens + macroblock records and reconstructs exactly what a decoder will reconstruct.
struct EncTables;
struct TrellisTables;
struct EncJob {
  const uint8_t* src;      // source raster (same layout as every other raster)
  const uint8_t* ref;      // last reconstructed + loop-filtered frame; nullptr for key frames
  uint8_t* out;            // reconstruction (before the loop filter, which runs afterwards in place)
  vp8gpu_mb* mbs;          // [cols * rows] records written by the device
  vp8gpu_token* tokens;    // token pool
  uint32_t* tok_counter;   // tokens used so far (atomic)
  uint32_t tok_cap;
  int* progress;           // [rows] wavefront counters (zeroed)
  const EncTables* tab;    // rate tables (enc_costs.h)
  vp8gpu_quant q;
  uint32_t rate_mult, dist_mult;  // Encoder::update_rd_multipliers (encoder.cc:179-194)
  uint16_t cols, rows;     // macroblocks coded by this pass: the whole frame, or the 1/16 sample of
  uint8_t sub;             //   Encoder::estimate_size (size_estimation.cc:36-99): macroblock (c, r) of the pass is
                           //   source macroblock (sub * c, sub * r); sub = 1 or 4
  uint8_t key_frame, lf_level;
  uint8_t sad_per_bit;     // sad_per_bit16lut[y_ac_qi] (encode_inter.cc:160-170)
  uint8_t realtime;        // REALTIME_QUALITY: no B_PRED in inter frames, motion search on every 4th column and row
  uint8_t mv_costs_zero;   // the reference fills its motion-vector cost tables (Costs::fill_mv_component_costs,
                           //   fill_mv_sad_costs) at the start of the first FULL inter-frame pass (encode_inter.cc:601-602);
                           //   the size estimates that precede it price every vector at 0
  uint8_t mv_sad_zero;     // the same for the diamond search's vector cost alone (Costs::fill_mv_sad_costs): Encoder::
                           //   reencode_as_interframe fills the component costs but not these (reencode.cc:85)
  uint8_t pad[1];
  // second pass of a two-pass key frame (k_enc_rd<true>, trellis quantisation encoder.cc:220-408)
  const TrellisTables* trellis;  // token costs of the default probabilities, value costs
  const uint8_t* y2_prev;        // [cols * rows] what the FIRST pass left in the frame object: bit 0 = Y2Block::has_nonzero()
                                 //   (the flag a B_PRED macroblock of the second pass keeps: its Y2 block is not touched,
                                 //   encode_intra.cc:181-184), bit 1 = the macroblock was B_PRED (its Y blocks' type)
};

// Encoder::update_residues on the device (reencode.cuh): keep a coded frame's modes and vectors, recompute its
// residues against the current references so that it decodes close to `target`.
struct ReencJob {
  const uint8_t* target;   // the raster to approximate (update_residues' original_raster)
  uint8_t* recon;          // in: every inter macroblock predicted / reconstructed by k_inter; out: + the intra ones
  const vp8gpu_mb* mbs_in; // the coded frame's records (modes, vectors, references); may alias mbs_out
  vp8gpu_mb* mbs_out;      // the same records with the new tok_off / tok_cnt
  vp8gpu_token* tokens;    // token pool
  uint32_t* tok_counter;   // tokens used so far (atomic)
  uint32_t tok_cap;
  int* progress;           // [rows] wavefront counters (zeroed)
  vp8gpu_quant q;          // Quantizer( quant_indices ): one for the whole frame (reencode.cc:283)
  uint16_t cols, rows;
};

// One frame's token-decode job (tokens.cu): DCT partitions -> token stream + tok_off / tok_cnt.
struct TokJob {
  vp8gpu_mb* mbs;             // in: y_mode, VP8GPU_MB_SKIP; out: tok_off, tok_cnt, flag cleared
  vp8gpu_token* tokens;       // out
  const uint8_t* bits;        // the frame's DCT partitions, back to back
  const uint8_t* coef_probs;  // 1056 bytes: the frame's coefficient probabilities
  uint32_t* result;           // [0] tokens written, [1] non-zero if the pool was too small
  uint16_t* above;            // mb_cols words of scratch (unused since the lock-step decoder keeps its contexts in shared memory)
  const uint32_t* mbinfo;     // lock-step variant: 2 bits per macroblock (flags & 3), 16 macroblocks per word
  uint32_t part_off[8], part_len[8];
  uint32_t nparts;            // 1, 2, 4 or 8
  uint32_t tok_cap;
};

// Kernel launchers (kernels.cu, tokens.cu).  `stream` is a cudaStream_t passed as void* so this header
// stays free of CUDA includes.  Return 0 or a cudaError_t value.
int launch_inter(const DevJob* jobs, int njobs, const Geom& g, void* stream);
int launch_enc_rd_trellis(const EncJob* job, int rows, const Geom& g, int* ticket, void* stream);
// re-encoding: njobs frames of the context in one launch (each job its own target, records, tokens and counters)
int launch_reenc_inter(const ReencJob* jobs, int njobs, int n_mbs, const Geom& g, void* stream);
int launch_reenc_intra(const ReencJob* jobs, int njobs, int rows, const Geom& g, int* ticket, void* stream);
// `epoch`: a value no earlier launch on this context has used (Engine::next_epoch); it marks the hand-over
// messages of this launch.  epoch == 0 selects the round-1 kernels (progress counters + acquire / release).
int launch_intra(const DevJob* jobs, int njobs, const Geom& g, int* ticket, uint32_t epoch, void* stream);
int launch_loopfilter(const DevJob* jobs, int njobs, const Geom& g, int* ticket, uint32_t epoch, void* stream);
// token jobs sit at the start of equally spaced ring slots: slot (first + i) % nslots for block i
int launch_tokens(const uint8_t* ring, size_t stride, int first, int count, int nslots, const Geom& g, void* stream);
int launch_fetch_header(void* dst, const void* src_host_devptr, size_t bytes, void* stream);  // bytes % 16 == 0
int launch_ssim(const uint8_t* a, const uint8_t* b, const Geom& g, float* d_windows, void* stream);
int launch_enc_rd(const EncJob* jobs, int njobs, int rows, const Geom& g, int* ticket, void* stream);

}  // namespace vp8
