// capi.cc -- the extern "C" surface declared in include/vp8gpu.h, on top of Engine (device
// side) and parser (CPU entropy front end).  Also holds the Decoder object (state + three
// reference rasters, explicit state passing as in decoder/decoder.hh:244-300) and the
// GOP-parallel whole-stream helper.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/resource.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <chrono>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/vp8gpu.h"
#include "engine.hpp"
#include "hostpool.h"
#include "parser.h"
#include "serializer.h"

using vp8::Engine;
using vp8::HostJob;
using vp8::ParsedFrame;
using vp8::State;

struct vp8gpu_parsed;
struct vp8gpu_ctx {
  Engine* engine = nullptr;
  std::string create_error;
  std::atomic<int> next_lane{0};
  // pinned parsed-frame buffers are expensive to create (cudaHostAlloc serialises on the driver):
  // decoders borrow them from this pool and hand them back when they are destroyed
  std::mutex pool_mu;
  std::vector<vp8gpu_parsed*> pinned_pool;
  // wall-clock accounting of the last vp8gpu_decode_ivf call (seconds, summed over threads)
  double stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // device-side token decoding: option, a one-slot ring for vp8gpu_parse_frame_device, and the
  // rings / streams of vp8gpu_decode_ivf's workers (kept between calls: cudaMalloc / cudaHostAlloc
  // of hundreds of MB are slow)
  std::atomic<int> device_tokens{1};
  std::mutex scratch_mu;
  vp8::TokenRing* scratch_ring = nullptr;
  std::vector<struct ivf_worker_kit*> kit_pool;
  // Optional limit (off by default, see vp8gpu_decode_ivf) on the frames whose DCT partitions may be on the
  // device at the same time: counting semaphore, released by a host function the token stream runs after the
  // kernel.
  std::mutex tok_mu;
  std::condition_variable tok_cv;
  int tok_permits = 0, tok_capacity = 0;
};
struct TokRelease {
  vp8gpu_ctx* ctx;
  int n;
};
static void CUDART_CB tok_release_cb(void* p) {
  TokRelease* r = static_cast<TokRelease*>(p);
  {
    std::lock_guard<std::mutex> lk(r->ctx->tok_mu);
    r->ctx->tok_permits += r->n;
  }
  r->ctx->tok_cv.notify_all();
  delete r;
}
struct vp8gpu_state {
  State s;
  vp8gpu_state(int w, int h) : s(w, h) {}
  explicit vp8gpu_state(const State& o) : s(o) {}
};
struct vp8gpu_parsed {
  ParsedFrame f;
  uint32_t n_intra = 0, n_filtered = 0;
  cudaEvent_t consumed = nullptr;  // set for pinned instances owned by a decoder
  bool busy = false;
  explicit vp8gpu_parsed(const vp8::Allocator& a) : f(a) {}
};
// what one vp8gpu_decode_ivf worker needs for device-side token decoding
constexpr int kTokSlots = 96;  // frames a worker may have between "first partition parsed" and "pixels done"
constexpr int kTokChunk = 32;  // frames per k_tokens launch: one lane each (at most a third of the slots)
constexpr int kTokStreams = 4; // k_tokens launches of one worker that may overlap
struct ivf_worker_kit {
  vp8::TokenRing* ring = nullptr;
  // uploads never queue behind a running k_tokens: they have their own stream, and consecutive
  // launches rotate over kTokStreams streams that only wait for their own upload
  cudaStream_t copy_stream = nullptr;
  cudaStream_t kstream[kTokStreams] = {};
  int next_kstream = 0;
  vp8gpu_parsed* parsed[kTokSlots] = {};
  cudaEvent_t staged[kTokSlots] = {}, ready[kTokSlots] = {}, finished[kTokSlots] = {};
  bool busy[kTokSlots] = {};
};
struct vp8gpu_resident_batch {
  Engine::Resident* r = nullptr;
};

namespace {

// events a host thread waits on: block instead of spinning -- vp8gpu_decode_ivf runs more host threads
// than there are CPUs, and a spinning waiter takes the core the dispatcher needs
constexpr unsigned kWaitableEvent = cudaEventDisableTiming | cudaEventBlockingSync;

void* pinned_alloc(size_t n) {
  void* p = nullptr;
  return cudaHostAlloc(&p, n, cudaHostAllocDefault) == cudaSuccess ? p : nullptr;
}
void pinned_free(void* p) { cudaFreeHost(p); }
const vp8::Allocator kPinned = {&pinned_alloc, &pinned_free};

// partition capacity of a token ring for streams whose largest frame has n bytes (some slack, so
// that a pooled ring fits the next stream too)
size_t ring_bytes_for(size_t n) { return n + n / 4 + 4096; }

void count_mbs(vp8gpu_parsed* p) {
  const vp8gpu_frame_desc& d = p->f.desc;
  const size_t n = (size_t)d.mb_cols * d.mb_rows;
  const vp8gpu_mb* m = p->f.mbs.data();
  uint32_t ni = 0, nf = 0;
  for (size_t i = 0; i < n; i++) {
    ni += m[i].ref_frame == VP8GPU_REF_CURRENT;
    nf += m[i].lf_level != 0;
  }
  p->n_intra = ni;
  p->n_filtered = nf;
}

}  // namespace

// =============================================================================================
// context and frames
// =============================================================================================
extern "C" {

// internal hooks for encoder.cu
Engine* vp8gpu_ctx_engine(vp8gpu_ctx* ctx) { return ctx->engine; }
int vp8gpu_ctx_next_lane(vp8gpu_ctx* ctx) { return ctx->next_lane.fetch_add(1) % vp8::kMaxLanes; }
// internal (encoder.cu): the flat frame behind a vp8gpu_parsed handle
const vp8::ParsedFrame* vp8gpu_parsed_frame(const vp8gpu_parsed* p) { return p ? &p->f : nullptr; }

int vp8gpu_ctx_create(int device, int width, int height, int max_frames, vp8gpu_ctx** out) {
  if (!out) return VP8GPU_ERR_LOGIC;
  *out = nullptr;
  // Many streams carry long-running k_tokens launches next to the short pixel launches; with the
  // default 8 hardware queues, work of unrelated streams would line up behind them.  Only has an
  // effect if the CUDA context does not exist yet; never overrides the user's choice.
  setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
  vp8gpu_ctx* c = new vp8gpu_ctx();
  const int rc = Engine::create(device, width, height, max_frames, &c->engine, &c->create_error);
  if (rc != VP8GPU_OK) {
    delete c;
    return rc;
  }
  *out = c;
  return VP8GPU_OK;
}
extern "C" void vp8gpu_encoder_pool_purge(Engine* e);
void vp8gpu_ctx_destroy(vp8gpu_ctx* ctx) {
  if (!ctx) return;
  for (vp8gpu_parsed* p : ctx->pinned_pool) vp8gpu_parsed_destroy(p);
  ctx->engine->sync_all();
  if (ctx->scratch_ring) ctx->engine->token_ring_free(ctx->scratch_ring);
  for (ivf_worker_kit* k : ctx->kit_pool) {
    ctx->engine->token_ring_free(k->ring);
    if (k->copy_stream) cudaStreamDestroy(k->copy_stream);
    for (cudaStream_t st : k->kstream)
      if (st) cudaStreamDestroy(st);
    for (int i = 0; i < kTokSlots; i++) {
      if (k->parsed[i]) vp8gpu_parsed_destroy(k->parsed[i]);
      if (k->staged[i]) cudaEventDestroy(k->staged[i]);
      if (k->ready[i]) cudaEventDestroy(k->ready[i]);
    }
    delete k;
  }
  vp8gpu_encoder_pool_purge(ctx->engine);  // buffer sets of destroyed Encoders of this context (encoder.cu)
  delete ctx->engine;
  delete ctx;
}
const char* vp8gpu_last_error(const vp8gpu_ctx* ctx) { return ctx && ctx->engine ? ctx->engine->last_error() : ""; }

int vp8gpu_frame_alloc(vp8gpu_ctx* ctx, vp8gpu_frame_id* out) { return ctx->engine->frame_alloc(out); }
int vp8gpu_frame_retain(vp8gpu_ctx* ctx, vp8gpu_frame_id id) { return ctx->engine->frame_retain(id); }
int vp8gpu_frame_release(vp8gpu_ctx* ctx, vp8gpu_frame_id id) { return ctx->engine->frame_release(id); }
int vp8gpu_frame_upload(vp8gpu_ctx* ctx, vp8gpu_frame_id id, const uint8_t* y, size_t ys, const uint8_t* u,
                        const uint8_t* v, size_t cs) {
  return ctx->engine->frame_upload(id, y, ys, u, v, cs);
}
int vp8gpu_frame_download(vp8gpu_ctx* ctx, vp8gpu_frame_id id, uint8_t* y, size_t ys, uint8_t* u, uint8_t* v,
                          size_t cs) {
  return ctx->engine->frame_download(id, y, ys, u, v, cs);
}
int vp8gpu_frame_download_display(vp8gpu_ctx* ctx, vp8gpu_frame_id id, uint8_t* dst, size_t dst_size) {
  return ctx->engine->frame_download_display(id, 0, dst, dst_size, true);
}
int vp8gpu_frame_download_display_async(vp8gpu_ctx* ctx, vp8gpu_frame_id id, uint8_t* dst, size_t dst_size) {
  return ctx->engine->frame_download_display(id, 0, dst, dst_size, false);
}
int vp8gpu_frame_hash(vp8gpu_ctx* ctx, vp8gpu_frame_id id, uint64_t* out) { return ctx->engine->frame_hash(id, 0, out); }
int vp8gpu_frame_ssim(vp8gpu_ctx* ctx, vp8gpu_frame_id a, vp8gpu_frame_id b, double* out) {
  if (!ctx || !out) return VP8GPU_ERR_LOGIC;
  return ctx->engine->frames_ssim(a, b, 0, out);
}
size_t vp8gpu_frame_bytes(const vp8gpu_ctx* ctx) { return ctx->engine->geom().frame_bytes; }
int vp8gpu_frame_export(vp8gpu_ctx* ctx, vp8gpu_frame_id id, void* dst, size_t bytes) {
  return ctx->engine->frame_copy_raw(id, dst, bytes, false);
}
int vp8gpu_frame_import(vp8gpu_ctx* ctx, vp8gpu_frame_id id, const void* src, size_t bytes) {
  return ctx->engine->frame_copy_raw(id, const_cast<void*>(src), bytes, true);
}
int vp8gpu_ctx_sync(vp8gpu_ctx* ctx) { return ctx->engine->sync_all(); }
int vp8gpu_host_alloc(void** out, size_t bytes) {
  return cudaHostAlloc(out, bytes, cudaHostAllocDefault) == cudaSuccess ? VP8GPU_OK : VP8GPU_ERR_NOMEM;
}
void vp8gpu_host_free(void* p) {
  if (p) cudaFreeHost(p);
}
uint64_t vp8gpu_launch_count(const vp8gpu_ctx* ctx) { return ctx->engine->launches(); }
int vp8gpu_frames_in_use(const vp8gpu_ctx* ctx) { return ctx->engine->frames_in_use(); }
int vp8gpu_serialize_frame_ex(const vp8gpu_encode_header* hdr, const vp8gpu_encode_features* ft, const vp8gpu_mb* mbs,
                              const vp8gpu_token* tokens, const vp8gpu_split_mvs* split, uint8_t* out, size_t cap,
                              size_t* size) {
  if (!hdr || !mbs || !size) return VP8GPU_ERR_LOGIC;
  vp8::EncodeHeader h;
  h.key_frame = hdr->key_frame;
  h.show_frame = hdr->show_frame;
  h.width = hdr->width;
  h.height = hdr->height;
  h.y_ac_qi = hdr->y_ac_qi;
  h.loop_filter_level = hdr->loop_filter_level;
  h.sharpness = hdr->sharpness;
  h.optimize_token_probs = hdr->optimize_token_probs;
  vp8::EncodeFeatures x;
  if (ft) {
    x.log2_partitions = ft->log2_partitions;
    x.segmentation_enabled = ft->segmentation_enabled;
    x.update_mb_segmentation_map = ft->update_mb_segmentation_map;
    x.update_segment_feature_data = ft->update_segment_feature_data;
    x.segment_feature_absolute = ft->segment_feature_absolute;
    for (int i = 0; i < 4; i++) {
      x.segment_quant[i] = ft->segment_quant[i];
      x.segment_lf[i] = ft->segment_lf[i];
      x.ref_lf_delta[i] = ft->ref_lf_delta[i];
      x.mode_lf_delta[i] = ft->mode_lf_delta[i];
    }
    for (int i = 0; i < 3; i++) x.segment_tree_probs[i] = ft->segment_tree_probs[i];
    x.lf_delta_enabled = ft->lf_delta_enabled;
    x.lf_delta_update = ft->lf_delta_update;
    x.y_dc_delta = ft->y_dc_delta;
    x.y2_dc_delta = ft->y2_dc_delta;
    x.y2_ac_delta = ft->y2_ac_delta;
    x.uv_dc_delta = ft->uv_dc_delta;
    x.uv_ac_delta = ft->uv_ac_delta;
    x.refresh_golden = ft->refresh_golden;
    x.refresh_alternate = ft->refresh_alternate;
    x.refresh_last = ft->refresh_last;
    x.refresh_entropy_probs = ft->refresh_entropy_probs;
    x.copy_to_golden = ft->copy_to_golden;
    x.copy_to_alternate = ft->copy_to_alternate;
    x.sign_bias_golden = ft->sign_bias_golden;
    x.sign_bias_alternate = ft->sign_bias_alternate;
    x.saved_coef_probs = ft->saved_coef_probs;
  }
  const std::vector<uint8_t> bytes = vp8::serialize_frame(h, mbs, tokens, split, ft ? &x : nullptr);
  if (bytes.empty()) return VP8GPU_ERR_UNSUPPORTED;
  *size = bytes.size();
  if (!out || cap < bytes.size()) return VP8GPU_ERR_NOMEM;
  memcpy(out, bytes.data(), bytes.size());
  return VP8GPU_OK;
}
int vp8gpu_serialize_frame(const vp8gpu_encode_header* hdr, const vp8gpu_mb* mbs, const vp8gpu_token* tokens,
                           const vp8gpu_split_mvs* split, uint8_t* out, size_t cap, size_t* size) {
  return vp8gpu_serialize_frame_ex(hdr, nullptr, mbs, tokens, split, out, cap, size);
}
void vp8gpu_decode_ivf_stats(const vp8gpu_ctx* ctx, double out[8]) { memcpy(out, ctx->stats, sizeof(ctx->stats)); }

// =============================================================================================
// the seam
// =============================================================================================
static HostJob to_host_job(const vp8gpu_job& j) {
  HostJob h;
  h.desc = j.desc;
  h.mbs = j.mbs;
  h.tokens = j.tokens;
  h.split = j.split;
  memcpy(h.refs, j.refs, sizeof(h.refs));
  h.out = j.out;
  return h;
}

int vp8gpu_decode_batch(vp8gpu_ctx* ctx, int lane, const vp8gpu_job* jobs, int n) {
  if (!ctx || !jobs || n < 0) return VP8GPU_ERR_LOGIC;
  std::vector<HostJob> hj;
  hj.reserve(n);
  for (int i = 0; i < n; i++) {
    if (!jobs[i].desc || !jobs[i].mbs) return ctx->engine->fail(VP8GPU_ERR_LOGIC, "decode_batch: null records");
    if (jobs[i].desc->mb_cols != ctx->engine->geom().mb_cols || jobs[i].desc->mb_rows != ctx->engine->geom().mb_rows)
      return ctx->engine->fail(VP8GPU_ERR_LOGIC, "decode_batch: frame size does not match the context");
    hj.push_back(to_host_job(jobs[i]));
  }
  const int rc = ctx->engine->submit(lane, hj.data(), n, nullptr);
  if (rc != VP8GPU_OK) return rc;
  // the caller's arrays may be pageable or pinned; make "consumed before return" unconditional
  cudaError_t e = cudaStreamSynchronize(ctx->engine->stream(lane));
  return e == cudaSuccess ? VP8GPU_OK : ctx->engine->cuda_fail(e, "decode_batch sync");
}

int vp8gpu_decode_parsed(vp8gpu_ctx* ctx, int lane, const vp8gpu_frame_desc* desc, const vp8gpu_mb* mbs,
                         const vp8gpu_token* tokens, const vp8gpu_split_mvs* split, const vp8gpu_frame_id refs[3],
                         vp8gpu_frame_id out) {
  vp8gpu_job j;
  j.desc = desc;
  j.mbs = mbs;
  j.tokens = tokens;
  j.split = split;
  for (int i = 0; i < 3; i++) j.refs[i] = refs ? refs[i] : -1;
  j.out = out;
  return vp8gpu_decode_batch(ctx, lane, &j, 1);
}

int vp8gpu_batch_upload(vp8gpu_ctx* ctx, const vp8gpu_job* jobs, int n, vp8gpu_resident_batch** out) {
  std::vector<HostJob> hj;
  for (int i = 0; i < n; i++) hj.push_back(to_host_job(jobs[i]));
  vp8gpu_resident_batch* b = new vp8gpu_resident_batch();
  const int rc = ctx->engine->resident_upload(hj.data(), n, &b->r);
  if (rc != VP8GPU_OK) {
    delete b;
    return rc;
  }
  *out = b;
  return VP8GPU_OK;
}
int vp8gpu_batch_run(vp8gpu_ctx* ctx, int lane, vp8gpu_resident_batch* b, float* kernel_ms) {
  return ctx->engine->resident_run(lane, b->r, kernel_ms);
}
int vp8gpu_batches_run(vp8gpu_ctx* ctx, int lane, vp8gpu_resident_batch* const* batches, int n, float* total_ms) {
  std::vector<Engine::Resident*> rs;
  for (int i = 0; i < n; i++) rs.push_back(batches[i]->r);
  return ctx->engine->resident_run_many(lane, rs.data(), n, total_ms);
}
int vp8gpu_batch_run_timed(vp8gpu_ctx* ctx, int lane, vp8gpu_resident_batch* b, float kernel_ms[3]) {
  return ctx->engine->resident_run_timed(lane, b->r, kernel_ms);
}
void vp8gpu_batch_free(vp8gpu_ctx* ctx, vp8gpu_resident_batch* b) {
  if (!b) return;
  ctx->engine->resident_free(b->r);
  delete b;
}

// =============================================================================================
// CPU front end
// =============================================================================================
int vp8gpu_state_create(int width, int height, vp8gpu_state** out) {
  if (!out || width <= 0 || height <= 0) return VP8GPU_ERR_LOGIC;
  *out = new vp8gpu_state(width, height);
  return VP8GPU_OK;
}
int vp8gpu_state_clone(const vp8gpu_state* s, vp8gpu_state** out) {
  if (!s || !out) return VP8GPU_ERR_LOGIC;
  *out = new vp8gpu_state(s->s);
  return VP8GPU_OK;
}
void vp8gpu_state_destroy(vp8gpu_state* s) { delete s; }
int vp8gpu_state_equal(const vp8gpu_state* a, const vp8gpu_state* b) { return a && b && a->s == b->s; }
uint64_t vp8gpu_state_hash(const vp8gpu_state* s) { return s->s.hash(); }
size_t vp8gpu_state_serialize(const vp8gpu_state* s, uint8_t* out, size_t cap) {
  if (!s) return 0;
  const std::vector<uint8_t> b = s->s.serialize();
  if (out && cap >= b.size()) memcpy(out, b.data(), b.size());
  return b.size();
}
int vp8gpu_state_deserialize(const uint8_t* data, size_t len, vp8gpu_state** out) {
  if (!data || !out) return VP8GPU_ERR_LOGIC;
  State st(16, 16);
  if (!State::deserialize(data, len, st)) return VP8GPU_ERR_INVALID;
  *out = new vp8gpu_state(st);
  return VP8GPU_OK;
}

int vp8gpu_parsed_create(vp8gpu_parsed** out) {
  if (!out) return VP8GPU_ERR_LOGIC;
  *out = new vp8gpu_parsed(vp8::kMallocAllocator);
  return VP8GPU_OK;
}
void vp8gpu_parsed_destroy(vp8gpu_parsed* p) {
  if (!p) return;
  if (p->consumed) cudaEventDestroy(p->consumed);
  delete p;
}
const vp8gpu_frame_desc* vp8gpu_parsed_desc(const vp8gpu_parsed* p) { return &p->f.desc; }
const vp8gpu_mb* vp8gpu_parsed_mbs(const vp8gpu_parsed* p) { return p->f.mbs.data(); }
const vp8gpu_token* vp8gpu_parsed_tokens(const vp8gpu_parsed* p) { return p->f.tokens.data(); }
const vp8gpu_split_mvs* vp8gpu_parsed_split(const vp8gpu_parsed* p) { return p->f.split.data(); }

int vp8gpu_parse_frame(vp8gpu_state* state, const uint8_t* data, size_t len, vp8gpu_parsed* out) {
  if (!state || !data || !out) return VP8GPU_ERR_LOGIC;
  const int rc = vp8::parse_frame(state->s, data, len, out->f);
  if (rc == VP8GPU_OK) count_mbs(out);
  return rc;
}

int vp8gpu_parsed_y_ac_qi(const vp8gpu_parsed* p) {
  if (!p || p->f.verbatim.header_tape.empty()) return -1;
  return p->f.verbatim.y_ac_qi;
}
int vp8gpu_parsed_keep_labels(vp8gpu_parsed* p, int on) {
  if (!p) return VP8GPU_ERR_LOGIC;
  p->f.keep_verbatim = on != 0;
  return VP8GPU_OK;
}
int vp8gpu_parsed_serialize(const vp8gpu_parsed* p, uint8_t* out, size_t cap, size_t* size) {
  if (!p || !size) return VP8GPU_ERR_LOGIC;
  if (!p->f.keep_verbatim || p->f.verbatim.header_tape.empty()) return VP8GPU_ERR_LOGIC;
  const std::vector<uint8_t> bytes = vp8::serialize_parsed(p->f);
  if (bytes.empty()) return VP8GPU_ERR_UNSUPPORTED;
  *size = bytes.size();
  if (!out || cap < bytes.size()) return VP8GPU_ERR_NOMEM;
  memcpy(out, bytes.data(), bytes.size());
  return VP8GPU_OK;
}

int vp8gpu_ctx_set_option(vp8gpu_ctx* ctx, int option, int value) {
  if (!ctx) return VP8GPU_ERR_LOGIC;
  if (option == VP8GPU_OPT_DEVICE_TOKENS) {
    ctx->device_tokens = value != 0;
    return VP8GPU_OK;
  }
  return ctx->engine->fail(VP8GPU_ERR_LOGIC, "unknown context option");
}

int vp8gpu_parse_frame_device(vp8gpu_ctx* ctx, vp8gpu_state* state, const uint8_t* data, size_t len,
                              vp8gpu_parsed* out) {
  if (!ctx || !state || !data || !out) return VP8GPU_ERR_LOGIC;
  Engine* e = ctx->engine;
  cudaSetDevice(e->device());
  int rc = vp8::parse_frame(state->s, data, len, out->f, true);
  if (rc != VP8GPU_OK) return rc;
  std::lock_guard<std::mutex> lk(ctx->scratch_mu);
  if (ctx->scratch_ring && ctx->scratch_ring->bits_cap < out->f.tw.bits_len) {
    e->sync_all();
    e->token_ring_free(ctx->scratch_ring);
    ctx->scratch_ring = nullptr;
  }
  if (!ctx->scratch_ring) {
    rc = e->token_ring_create(1, len * 2 + 4096, &ctx->scratch_ring);
    if (rc != VP8GPU_OK) return rc;
  }
  vp8::TokenRing* r = ctx->scratch_ring;
  rc = e->ensure_lane(0);
  if (rc != VP8GPU_OK) return rc;
  cudaStream_t s = e->stream(0);
  rc = e->token_ring_stage(r, 0, out->f, s);
  if (rc == VP8GPU_OK) rc = e->token_ring_clear_result(r, 0, s);
  if (rc == VP8GPU_OK) rc = e->token_ring_launch(r, 0, 1, s);
  uint32_t result[2] = {0, 0};
  if (rc == VP8GPU_OK) rc = e->token_ring_result(r, 0, s, result);
  if (rc != VP8GPU_OK) return rc;
  if (result[1] || result[0] > r->tok_cap) return e->fail(VP8GPU_ERR_NOMEM, "device token pool overflow");
  const vp8gpu_frame_desc& d = out->f.desc;
  const size_t n_mbs = (size_t)d.mb_cols * d.mb_rows;
  if (!out->f.tokens.reserve(result[0] + 1, 0)) return VP8GPU_ERR_NOMEM;
  if (cudaMemcpyAsync(out->f.mbs.data(), r->dev_slot(0) + r->mbs_off, n_mbs * sizeof(vp8gpu_mb), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
      (result[0] && cudaMemcpyAsync(out->f.tokens.data(), r->dev_slot(0) + r->tok_off, (size_t)result[0] * sizeof(vp8gpu_token),
                                    cudaMemcpyDeviceToHost, s) != cudaSuccess) ||
      cudaStreamSynchronize(s) != cudaSuccess)
    return e->fail(VP8GPU_ERR_CUDA, "parse_frame_device: copy back failed");
  out->f.desc.n_tokens = result[0];
  out->f.tw.deferred = false;
  out->f.tw.bits = nullptr;
  count_mbs(out);
  return VP8GPU_OK;
}

}  // extern "C"

// =============================================================================================
// Decoder
// =============================================================================================
struct vp8gpu_decoder {
  vp8gpu_ctx* ctx = nullptr;
  int lane = 0;
  vp8gpu_state state;
  int refs[3] = {-1, -1, -1};  // last, golden, alternative; each holds one reference count
  // ring of pinned parsed-frame buffers so the host can parse frame N+1 while the DMA engine
  // is still reading frame N's records
  vp8gpu_parsed* ring[vp8::kStagingDepth] = {};
  int ring_next = 0;
  // optional device-side token decoding (vp8gpu_decoder_set_device_tokens)
  bool device_tokens = false;
  vp8::TokenRing* tok_ring = nullptr;
  cudaEvent_t tok_finished[vp8::kStagingDepth] = {};
  bool tok_busy[vp8::kStagingDepth] = {};
  int tok_next = 0;
  vp8gpu_decoder(vp8gpu_ctx* c, int w, int h) : ctx(c), state(w, h) {}
  vp8gpu_decoder(vp8gpu_ctx* c, const State& s) : ctx(c), state(s) {}
};

namespace {

void set_ref(Engine* e, int* slot, int id) {
  // RasterHandle assignment: retain the new raster, release the old one
  if (*slot == id) return;
  e->frame_retain(id);
  if (*slot >= 0) e->frame_release(*slot);
  *slot = id;
}

vp8gpu_parsed* next_ring_slot(vp8gpu_decoder* d) {
  vp8gpu_parsed*& p = d->ring[d->ring_next];
  d->ring_next = (d->ring_next + 1) % vp8::kStagingDepth;
  if (!p) {
    {
      std::lock_guard<std::mutex> lk(d->ctx->pool_mu);
      if (!d->ctx->pinned_pool.empty()) {
        p = d->ctx->pinned_pool.back();
        d->ctx->pinned_pool.pop_back();
      }
    }
    if (!p) {
      p = new vp8gpu_parsed(kPinned);
      cudaEventCreateWithFlags(&p->consumed, kWaitableEvent);
      // size the token buffer generously up front: growing pinned memory means a new cudaHostAlloc
      const vp8::Geom& g = d->ctx->engine->geom();
      const size_t n_mbs = (size_t)g.mb_cols * g.mb_rows;
      p->f.mbs.reserve(n_mbs, 0);
      p->f.tokens.reserve(n_mbs * 32 + 1024, 0);
      p->f.split.reserve(256, 0);
    }
  }
  if (p->busy) {
    cudaEventSynchronize(p->consumed);
    p->busy = false;
  }
  return p;
}

// Frame::copy_to (frame.cc:272-307): the decoder's references after frame `out` (decoded from desc)
void copy_to_references(vp8gpu_decoder* d, const vp8gpu_frame_desc& desc, int out) {
  Engine* e = d->ctx->engine;
  if (desc.key_frame) {
    set_ref(e, &d->refs[0], out);
    set_ref(e, &d->refs[1], out);
    set_ref(e, &d->refs[2], out);
  } else {
    if (desc.copy_to_alternate == 1) set_ref(e, &d->refs[2], d->refs[0]);
    else if (desc.copy_to_alternate == 2) set_ref(e, &d->refs[2], d->refs[1]);
    if (desc.copy_to_golden == 1) set_ref(e, &d->refs[1], d->refs[0]);
    else if (desc.copy_to_golden == 2) set_ref(e, &d->refs[1], d->refs[2]);
    if (desc.refresh_golden) set_ref(e, &d->refs[1], out);
    if (desc.refresh_alternate) set_ref(e, &d->refs[2], out);
    if (desc.refresh_last) set_ref(e, &d->refs[0], out);
  }
}

// Decoder::decode_frame (decoder.cc:101-118): decode + loopfilter into a fresh raster, then
// Frame::copy_to (frame.cc:272-307) on the references.
int decode_parsed_impl(vp8gpu_decoder* d, vp8gpu_parsed* p, bool pinned_ring, int* shown, int* out_id,
                       int tok_slot = -1) {
  Engine* e = d->ctx->engine;
  const vp8gpu_frame_desc& desc = p->f.desc;
  int out = -1;
  int rc = e->frame_alloc(&out);
  if (rc != VP8GPU_OK) return rc;
  HostJob j;
  j.desc = &desc;
  j.mbs = p->f.mbs.data();
  j.tokens = p->f.tokens.data();
  j.split = p->f.split.data();
  memcpy(j.refs, d->refs, sizeof(j.refs));
  j.out = out;
  j.n_intra = (int)p->n_intra;
  j.n_filtered = (int)p->n_filtered;
  if (tok_slot >= 0) {  // records and tokens are already in the ring, produced on this lane's stream
    j.ring = d->tok_ring;
    j.ring_slot = tok_slot;
    j.finished = &d->tok_finished[tok_slot];
  }
  rc = e->submit(d->lane, &j, 1, pinned_ring ? p->consumed : nullptr);
  if (rc != VP8GPU_OK) {
    e->frame_release(out);
    return rc;
  }
  if (pinned_ring) p->busy = true;
  else cudaStreamSynchronize(e->stream(d->lane));  // caller-owned (possibly pageable) records
  copy_to_references(d, desc, out);
  if (shown) *shown = desc.show_frame;
  if (out_id) *out_id = out;  // the allocation's reference goes to the caller
  else e->frame_release(out);
  return VP8GPU_OK;
}

}  // namespace

extern "C" {

int vp8gpu_decoder_create(vp8gpu_ctx* ctx, vp8gpu_decoder** out) {
  if (!ctx || !out) return VP8GPU_ERR_LOGIC;
  Engine* e = ctx->engine;
  vp8gpu_decoder* d = new vp8gpu_decoder(ctx, e->width(), e->height());
  d->lane = ctx->next_lane.fetch_add(1) % vp8::kMaxLanes;
  int id = -1;
  int rc = e->frame_alloc(&id);
  if (rc == VP8GPU_OK) rc = e->frame_clear(id, d->lane);
  if (rc != VP8GPU_OK) {
    if (id >= 0) e->frame_release(id);
    delete d;
    return rc;
  }
  // References( MutableRasterHandle ): last, golden and alternative share one raster (decoder.cc:165-169)
  d->refs[0] = d->refs[1] = d->refs[2] = id;
  e->frame_retain(id);
  e->frame_retain(id);
  *out = d;
  return VP8GPU_OK;
}

int vp8gpu_decoder_create_from(vp8gpu_ctx* ctx, const vp8gpu_state* state, const vp8gpu_frame_id refs[3],
                               vp8gpu_decoder** out) {
  if (!ctx || !state || !refs || !out) return VP8GPU_ERR_LOGIC;
  Engine* e = ctx->engine;
  if (state->s.width != e->width() || state->s.height != e->height())
    return e->fail(VP8GPU_ERR_LOGIC, "decoder_create_from: state size does not match the context");
  for (int i = 0; i < 3; i++)
    if (e->frame_retain(refs[i]) != VP8GPU_OK) {
      for (int k = 0; k < i; k++) e->frame_release(refs[k]);
      return VP8GPU_ERR_LOGIC;
    }
  vp8gpu_decoder* d = new vp8gpu_decoder(ctx, state->s);
  d->lane = ctx->next_lane.fetch_add(1) % vp8::kMaxLanes;
  memcpy(d->refs, refs, sizeof(d->refs));
  *out = d;
  return VP8GPU_OK;
}

// Decoder::serialize (decoder.cc:54-69) in the reference's tag-length-value format: DECODER { DECODER_STATE {...}
// REFERENCES { display size, REF_LAST { planes } } }.  Like the reference, only the LAST reference is stored
// (decoder.cc:177-197) and a deserialised Decoder has golden = alternative = last (decoder.cc:171-175).
int vp8gpu_decoder_serialize(vp8gpu_decoder* d, uint8_t* out, size_t cap, size_t* size) {
  if (!d || !size) return VP8GPU_ERR_LOGIC;
  Engine* e = d->ctx->engine;
  const vp8::Geom& g = e->geom();
  const std::vector<uint8_t> st = d->state.s.serialize();
  const size_t raster = (size_t)g.W * g.H + 2 * (size_t)(g.W / 2) * (g.H / 2);
  const size_t refs_body = 4 + 5 + raster;
  const size_t total = 5 + st.size() + 5 + refs_body;
  *size = total;
  if (!out || cap < total) return VP8GPU_ERR_NOMEM;
  auto u32 = [](uint8_t* p, size_t v) { p[0] = v & 0xFF, p[1] = (v >> 8) & 0xFF, p[2] = (v >> 16) & 0xFF, p[3] = (v >> 24) & 0xFF; };
  uint8_t* p = out;
  *p++ = 11;  // EncoderSerDesTag::DECODER
  u32(p, st.size() + 5 + refs_body);
  p += 4;
  memcpy(p, st.data(), st.size());
  p += st.size();
  *p++ = 7;  // REFERENCES
  u32(p, refs_body);
  p += 4;
  p[0] = e->width() & 0xFF, p[1] = e->width() >> 8, p[2] = e->height() & 0xFF, p[3] = e->height() >> 8;
  p += 4;
  *p++ = 8;  // REF_LAST
  u32(p, raster);
  p += 4;
  cudaSetDevice(e->device());
  return e->frame_download(d->refs[0], p, g.W, p + (size_t)g.W * g.H, p + (size_t)g.W * g.H + (size_t)(g.W / 2) * (g.H / 2), g.W / 2);
}

// Decoder::deserialize (decoder.cc:71-81)
int vp8gpu_decoder_deserialize(vp8gpu_ctx* ctx, const uint8_t* data, size_t len, vp8gpu_decoder** out) {
  if (!ctx || !data || !out) return VP8GPU_ERR_LOGIC;
  Engine* e = ctx->engine;
  auto u32 = [](const uint8_t* p) { return (size_t)p[0] | ((size_t)p[1] << 8) | ((size_t)p[2] << 16) | ((size_t)p[3] << 24); };
  if (len < 5 || data[0] != 11 || u32(data + 1) != len - 5) return e->fail(VP8GPU_ERR_INVALID, "not a serialised Decoder");
  vp8gpu_state st(e->width(), e->height());
  size_t used = 0;
  if (!State::deserialize(data + 5, len - 5, st.s, &used)) return e->fail(VP8GPU_ERR_INVALID, "bad DECODER_STATE record");
  if (st.s.width != e->width() || st.s.height != e->height())
    return e->fail(VP8GPU_ERR_UNSUPPORTED, "serialised Decoder has another frame size than the context");
  const uint8_t* p = data + 5 + used;
  const size_t left = len - 5 - used;
  const vp8::Geom& g = e->geom();
  const size_t raster = (size_t)g.W * g.H + 2 * (size_t)(g.W / 2) * (g.H / 2);
  if (left < 9 || p[0] != 7) return e->fail(VP8GPU_ERR_INVALID, "bad REFERENCES record");
  const int rw = p[5] | (p[6] << 8), rh = p[7] | (p[8] << 8);
  if (rw != e->width() || rh != e->height()) return e->fail(VP8GPU_ERR_INVALID, "REFERENCES size mismatch");
  vp8gpu_frame_id id = -1;
  cudaSetDevice(e->device());
  int rc = e->frame_alloc(&id);
  if (rc != VP8GPU_OK) return rc;
  if (left >= 9 + 5 + raster && p[9] == 8 && u32(p + 10) == raster) {
    const uint8_t* y = p + 14;
    rc = e->frame_upload(id, y, g.W, y + (size_t)g.W * g.H, y + (size_t)g.W * g.H + (size_t)(g.W / 2) * (g.H / 2), g.W / 2);
  } else if (left != 9) {
    rc = e->fail(VP8GPU_ERR_INVALID, "bad REF_LAST record");
  }  // no REF_LAST record: EncoderStateDeserializer::get_ref returns a fresh raster (enc_state_serializer.hh:168-190)
  if (rc == VP8GPU_OK) {
    const vp8gpu_frame_id three[3] = {id, id, id};
    rc = vp8gpu_decoder_create_from(ctx, &st, three, out);
  }
  e->frame_release(id);
  return rc;
}

int vp8gpu_decoder_clone(const vp8gpu_decoder* src, vp8gpu_decoder** out) {
  if (!src || !out) return VP8GPU_ERR_LOGIC;
  const vp8gpu_state tmp(src->state.s);
  return vp8gpu_decoder_create_from(src->ctx, &tmp, src->refs, out);
}

void vp8gpu_decoder_destroy(vp8gpu_decoder* d) {
  if (!d) return;
  Engine* e = d->ctx->engine;
  for (auto& p : d->ring)
    if (p && p->busy) {
      cudaEventSynchronize(p->consumed);
      p->busy = false;
    }
  for (int i = 0; i < 3; i++)
    if (d->refs[i] >= 0) e->frame_release(d->refs[i]);
  {
    std::lock_guard<std::mutex> lk(d->ctx->pool_mu);
    for (auto& p : d->ring)
      if (p) d->ctx->pinned_pool.push_back(p);
  }
  if (d->tok_ring) {
    e->sync_lane(d->lane);
    e->token_ring_free(d->tok_ring);
  }
  delete d;
}

int vp8gpu_decoder_set_device_tokens(vp8gpu_decoder* d, int on) {
  if (!d) return VP8GPU_ERR_LOGIC;
  d->device_tokens = on != 0;
  return VP8GPU_OK;
}

int vp8gpu_decoder_decode(vp8gpu_decoder* d, const uint8_t* data, size_t len, int* shown, vp8gpu_frame_id* out) {
  if (!d || !data) return VP8GPU_ERR_LOGIC;
  Engine* e = d->ctx->engine;
  cudaSetDevice(e->device());
  vp8gpu_parsed* p = next_ring_slot(d);
  if (!d->device_tokens) {
    const int rc = vp8::parse_frame(d->state.s, data, len, p->f);
    if (rc != VP8GPU_OK) return e->fail(rc, "parse_frame failed");
    count_mbs(p);
    return decode_parsed_impl(d, p, true, shown, out);
  }
  // host: first partition; device: DCT partitions, then the pixel kernels, all on this lane
  int rc = e->ensure_lane(d->lane);
  if (rc != VP8GPU_OK) return rc;
  if (d->tok_ring && d->tok_ring->bits_cap < len) {
    e->sync_lane(d->lane);
    e->token_ring_free(d->tok_ring);
    d->tok_ring = nullptr;
    for (bool& b : d->tok_busy) b = false;
  }
  if (!d->tok_ring) {
    rc = e->token_ring_create(vp8::kStagingDepth, len * 2 + 65536, &d->tok_ring);
    if (rc != VP8GPU_OK) return rc;
  }
  const int slot = d->tok_next;
  d->tok_next = (d->tok_next + 1) % vp8::kStagingDepth;
  if (d->tok_busy[slot]) {
    if (d->tok_finished[slot]) cudaEventSynchronize(d->tok_finished[slot]);
    d->tok_busy[slot] = false;
    // the frame that used this slot is done: k_tokens reports a token pool that was too small instead of
    // writing out of bounds (the capacity rule of Engine::token_ring_layout makes that impossible, so a set
    // flag is an internal error -- but it must not pass silently)
    uint32_t res[2] = {0, 0};
    if (cudaMemcpy(res, d->tok_ring->dev_slot(slot) + d->tok_ring->result_off, sizeof(res), cudaMemcpyDeviceToHost) != cudaSuccess)
      return e->fail(VP8GPU_ERR_CUDA, "token result read failed");
    if (res[1]) return e->fail(VP8GPU_ERR_LOGIC, "device token pool overflow in an earlier frame of this decoder");
  }
  rc = vp8::parse_frame(d->state.s, data, len, p->f, true);
  if (rc != VP8GPU_OK) return e->fail(rc, "parse_frame failed");
  count_mbs(p);
  cudaStream_t s = e->stream(d->lane);
  rc = e->token_ring_stage(d->tok_ring, slot, p->f, s);
  if (rc == VP8GPU_OK) rc = e->token_ring_launch(d->tok_ring, slot, 1, s);
  if (rc != VP8GPU_OK) return rc;
  p->f.tw.bits = nullptr;  // staged: the caller's buffer is no longer needed
  rc = decode_parsed_impl(d, p, true, shown, out, slot);
  if (rc == VP8GPU_OK) d->tok_busy[slot] = true;
  return rc;
}

}  // extern "C"

namespace {

// vp8gpu_decoders_decode_written with records: the first partition is parsed like any other frame's (state, modes,
// vectors, resolved loop-filter levels), but the DCT partitions are not decoded again: their content is the token lists
// they were written from (tok_off / tok_cnt of the writer's records index enc_tokens; the order inside a macroblock's
// list does not matter to the kernels).  Saves the serial half of the parse, which is most of a frame's host time.
int parse_written(vp8gpu_decoder* d, vp8gpu_parsed* p, const uint8_t* data, size_t len, const vp8gpu_mb* enc_mbs,
                  const vp8gpu_token* enc_tokens, uint32_t n_tok) {
  Engine* e = d->ctx->engine;
  if (!enc_mbs) {  // the full parse
    const int rc = vp8::parse_frame(d->state.s, data, len, p->f);
    if (rc != VP8GPU_OK) return e->fail(rc, "parse_frame failed");
    count_mbs(p);
    return VP8GPU_OK;
  }
  if (n_tok && !enc_tokens) return VP8GPU_ERR_LOGIC;
  const int rc = vp8::parse_frame(d->state.s, data, len, p->f, true);
  if (rc != VP8GPU_OK) return e->fail(rc, "parse_frame failed");
  const size_t n = (size_t)p->f.desc.mb_cols * p->f.desc.mb_rows;
  if (!p->f.tokens.reserve((size_t)n_tok + 1, 0)) return e->fail(VP8GPU_ERR_NOMEM, "token buffer");
  if (n_tok) memcpy(p->f.tokens.data(), enc_tokens, (size_t)n_tok * sizeof(vp8gpu_token));
  vp8gpu_mb* m = p->f.mbs.data();
  for (size_t i = 0; i < n; i++) {
    const vp8gpu_mb& w = enc_mbs[i];
    // the frame must be the one written from these records: same decisions, a skipped macroblock has no tokens
    if (m[i].y_mode != w.y_mode || m[i].ref_frame != w.ref_frame || ((m[i].flags & VP8GPU_MB_SKIP) && w.tok_cnt) ||
        (size_t)w.tok_off + w.tok_cnt > n_tok)
      return e->fail(VP8GPU_ERR_LOGIC, "decode_known_tokens: the records do not belong to this frame");
    m[i].tok_off = w.tok_off;
    m[i].tok_cnt = w.tok_cnt;
    m[i].flags = static_cast<uint8_t>(m[i].flags & ~VP8GPU_MB_SKIP);
  }
  p->f.desc.n_tokens = n_tok;
  p->f.tw.deferred = false;
  count_mbs(p);
  return VP8GPU_OK;
}

}  // namespace

extern "C" {

// Internal (encoder.cu, Encoder::write_frame's "decode what was written", encoder.cc:153-158): frame i, just written by
// this library, decoded by decoder ds[i] -- vp8gpu_decoder_decode of every frame, but the n frames share one set of
// launches (one Engine::submit on `lane`; < 0: the first decoder's lane) and their first partitions are parsed on the
// host pool.  enc_mbs[i] / enc_tokens[i] / n_tok[i]: the records and token lists frame i was written from (see
// parse_written); enc_mbs[i] == nullptr: the full parse.  The decoders must be distinct.  rcs[i]: frame i's status (a
// refused frame leaves its decoder as it was); returns the first failure or VP8GPU_OK.
int vp8gpu_decoders_decode_written(vp8gpu_decoder* const* ds, int n, int lane, const uint8_t* const* data, const size_t* len,
                                   const vp8gpu_mb* const* enc_mbs, const vp8gpu_token* const* enc_tokens, const uint32_t* n_tok,
                                   int* rcs) {
  if (n <= 0) return n < 0 ? VP8GPU_ERR_LOGIC : VP8GPU_OK;
  Engine* e = ds[0]->ctx->engine;
  cudaSetDevice(e->device());
  std::vector<vp8gpu_parsed*> ps(n);
  for (int i = 0; i < n; i++) ps[i] = next_ring_slot(ds[i]);
  auto parse = [&](int i) { rcs[i] = parse_written(ds[i], ps[i], data[i], len[i], enc_mbs[i], enc_tokens[i], n_tok[i]); };
  {
    vp8::HostPool::Group grp;
    for (int i = 1; i < n; i++) grp.run([&parse, i] { parse(i); });
    parse(0);
    grp.wait();
  }
  std::vector<HostJob> jobs;
  std::vector<int> which;
  for (int i = 0; i < n; i++) {
    if (rcs[i] != VP8GPU_OK) continue;
    int out = -1;
    rcs[i] = e->frame_alloc(&out);
    if (rcs[i] != VP8GPU_OK) continue;
    HostJob j;
    j.desc = &ps[i]->f.desc;
    j.mbs = ps[i]->f.mbs.data();
    j.tokens = ps[i]->f.tokens.data();
    j.split = ps[i]->f.split.data();
    memcpy(j.refs, ds[i]->refs, sizeof(j.refs));
    j.out = out;
    j.n_intra = (int)ps[i]->n_intra;
    j.n_filtered = (int)ps[i]->n_filtered;
    j.consumed = ps[i]->consumed;
    jobs.push_back(j);
    which.push_back(i);
  }
  const int rc = e->submit(lane < 0 ? ds[0]->lane : lane, jobs.data(), (int)jobs.size(), nullptr);
  for (size_t k = 0; k < jobs.size(); k++) {
    const int i = which[k];
    if (rc == VP8GPU_OK) {
      ps[i]->busy = true;
      copy_to_references(ds[i], *jobs[k].desc, jobs[k].out);
    } else {
      rcs[i] = rc;
    }
    e->frame_release(jobs[k].out);
  }
  for (int i = 0; i < n; i++)
    if (rcs[i] != VP8GPU_OK) return rcs[i];
  return VP8GPU_OK;
}

int vp8gpu_decoder_decode_parsed(vp8gpu_decoder* d, const vp8gpu_parsed* parsed, int* shown, vp8gpu_frame_id* out) {
  if (!d || !parsed) return VP8GPU_ERR_LOGIC;
  cudaSetDevice(d->ctx->engine->device());
  return decode_parsed_impl(d, const_cast<vp8gpu_parsed*>(parsed), false, shown, out);
}

vp8gpu_state* vp8gpu_decoder_state(vp8gpu_decoder* d) { return &d->state; }
int vp8gpu_decoder_references(const vp8gpu_decoder* d, vp8gpu_frame_id refs[3]) {
  memcpy(refs, d->refs, sizeof(d->refs));
  return VP8GPU_OK;
}
int vp8gpu_decoder_lane(const vp8gpu_decoder* d) { return d->lane; }

int vp8gpu_decoder_hash(vp8gpu_decoder* d, uint64_t* out) {
  if (!d || !out) return VP8GPU_ERR_LOGIC;
  uint64_t h = d->state.s.hash();
  for (int i = 0; i < 3; i++) {
    uint64_t r = 0;
    const int rc = d->ctx->engine->frame_hash(d->refs[i], d->lane, &r);
    if (rc != VP8GPU_OK) return rc;
    h = (h ^ r) * 0x9E3779B97F4A7C15ull + (h >> 29) + i;  // order dependent: last, golden, alternative
  }
  *out = h;
  return VP8GPU_OK;
}

int vp8gpu_decoder_equal(vp8gpu_decoder* a, vp8gpu_decoder* b, int* equal) {
  if (!a || !b || !equal || a->ctx != b->ctx) return VP8GPU_ERR_LOGIC;
  *equal = 0;
  if (!(a->state.s == b->state.s)) return VP8GPU_OK;
  for (int i = 0; i < 3; i++) {
    int eq = 0;
    const int rc = a->ctx->engine->frames_equal(a->refs[i], b->refs[i], a->lane, &eq);
    if (rc != VP8GPU_OK) return rc;
    if (!eq) return VP8GPU_OK;
  }
  *equal = 1;
  return VP8GPU_OK;
}

// =============================================================================================
// whole-stream helper: FilePlayer semantics (player.cc:88-143) with GOP-level parallelism
// =============================================================================================
// DIAGNOSTIC ONLY (VP8GPU_PARSE_CACHE=1, tools/e2e_probe.py): the bench decodes replicas of a few GOPs, so the result
// of parsing a first partition can be remembered by content and replayed with a memcpy.  This answers "what would
// vp8gpu_decode_ivf do if the host front end cost nothing" (DESIGN.md section 7, first partitions on the device); it
// is never enabled by default and the numbers it produces are not decode throughput.
struct CachedFirstPartition {
  vp8gpu_frame_desc desc;
  std::vector<vp8gpu_mb> mbs;
  std::vector<vp8gpu_split_mvs> split;
  vp8::TokenWork tw;
  size_t bits_delta = 0;
};
std::mutex g_parse_cache_mu;
std::unordered_map<uint64_t, std::shared_ptr<CachedFirstPartition>> g_parse_cache;
uint64_t frame_key(const uint8_t* p, size_t n) {
  uint64_t h = 1469598103934665603ull ^ n;
  auto mix = [&](const uint8_t* q, size_t k) {
    for (size_t i = 0; i < k; i++) h = (h ^ q[i]) * 1099511628211ull;
  };
  mix(p, n < 64 ? n : 64);
  if (n > 64) mix(p + n - 64, 64);
  return h;
}
int parse_first_partition_cached(vp8::State& state, const uint8_t* data, size_t len, vp8::ParsedFrame& out) {
  const uint64_t key = frame_key(data, len);
  std::shared_ptr<CachedFirstPartition> c;
  {
    std::lock_guard<std::mutex> lk(g_parse_cache_mu);
    auto it = g_parse_cache.find(key);
    if (it != g_parse_cache.end()) c = it->second;
  }
  if (!c) {
    const int rc = vp8::parse_frame(state, data, len, out, true);
    if (rc != VP8GPU_OK) return rc;
    c = std::make_shared<CachedFirstPartition>();
    c->desc = out.desc;
    const size_t n = (size_t)out.desc.mb_cols * out.desc.mb_rows;
    c->mbs.assign(out.mbs.data(), out.mbs.data() + n);
    c->split.assign(out.split.data(), out.split.data() + out.desc.n_split);
    c->tw = out.tw;
    c->bits_delta = (size_t)(out.tw.bits - data);
    std::lock_guard<std::mutex> lk(g_parse_cache_mu);
    g_parse_cache[key] = c;
    return VP8GPU_OK;
  }
  out.desc = c->desc;
  if (!out.mbs.reserve(c->mbs.size(), 0) || !out.split.reserve(c->split.size() + 1, 0)) return VP8GPU_ERR_NOMEM;
  memcpy(out.mbs.data(), c->mbs.data(), c->mbs.size() * sizeof(vp8gpu_mb));
  if (!c->split.empty()) memcpy(out.split.data(), c->split.data(), c->split.size() * sizeof(vp8gpu_split_mvs));
  out.tw = c->tw;
  out.tw.bits = data + c->bits_delta;
  return VP8GPU_OK;
}

// Tuning knobs of vp8gpu_decode_ivf, read ONCE per call from the environment (diagnostics and the sweeps of
// tools/e2e_probe.py).  -1 = not set.
struct IvfKnobs {
  int tok_slots = -1;      // VP8GPU_TOK_SLOTS     frames a worker keeps between "first partition parsed" and "pixels done"
  int tok_chunk = -1;      // VP8GPU_TOK_CHUNK     frames per token-kernel launch
  int tok_inflight = -1;   // VP8GPU_TOK_INFLIGHT  cap on frames inside token kernels (0 = unlimited)
  int tok_arena = -1;      // VP8GPU_TOK_ARENA     token arena per worker, in largest frames (never below plan()'s floor)
  int dispatchers = -1;    // VP8GPU_DISPATCHERS   dispatcher threads
  int worker_nice = -1;    // VP8GPU_WORKER_NICE   niceness of the parsing workers (0 = leave alone)
  bool trace = false;      // VP8GPU_TRACE         per-batch device times and per-worker arena counters on stderr
  bool parse_cache = false;  // VP8GPU_PARSE_CACHE  diagnostic: replay remembered first partitions (see above)
  static int num(const char* name) {
    const char* v = getenv(name);
    return v ? atoi(v) : -1;
  }
  IvfKnobs()
      : tok_slots(num("VP8GPU_TOK_SLOTS")), tok_chunk(num("VP8GPU_TOK_CHUNK")), tok_inflight(num("VP8GPU_TOK_INFLIGHT")),
        tok_arena(num("VP8GPU_TOK_ARENA")), dispatchers(num("VP8GPU_DISPATCHERS")), worker_nice(num("VP8GPU_WORKER_NICE")),
        trace(getenv("VP8GPU_TRACE") != nullptr), parse_cache(getenv("VP8GPU_PARSE_CACHE") != nullptr) {}
};

// vp8gpu_decode_ivf as an object, one instance per call: parse_container() reads the IVF file into GOPs, plan() sizes
// the pipeline (workers, token-ring slots, dispatchers), run() starts one thread per worker -- worker_host parses whole
// frames, worker_device only first partitions and launches k_tokens for the rest -- and one per dispatcher, which
// batches whatever the workers have queued (at most one frame per worker: consecutive frames of a GOP depend on each
// other) onto the device.
class IvfDecode {
 public:
  IvfDecode(vp8gpu_ctx* ctx_, const uint8_t* ivf_, size_t len_, int threads_, uint8_t* dst_, size_t dst_size_)
      : ctx(ctx_), e(ctx_->engine), ivf(ivf_), len(len_), threads(threads_), dst(dst_), dst_size(dst_size_) {}
  int parse_container();
  void plan();
  int run(uint32_t* n_decoded, uint32_t* n_shown);

 private:
  struct Item {
    const uint8_t* p;
    uint32_t n;
    int64_t out_off;  // -1 = hidden
  };
  static constexpr int kSlots = 4;  // parsed frames a host-token worker may have in flight
  enum SlotState { kFree = 0, kQueued = 1 };
  struct Pending {
    vp8gpu_parsed* slot;
    int refs[3];
    int out;
    int64_t out_off;
    int* slot_state;
    int tid = 0;  // the worker that queued it
    // device-side tokens: the records live in ring slot `ring_slot` once `ready` has fired
    const vp8::TokenRing* ring = nullptr;
    int ring_slot = 0;
    cudaEvent_t ready = nullptr;
    cudaEvent_t* finished = nullptr;  // where submit() leaves the event that fires after the pixel kernels
  };

  vp8gpu_ctx* const ctx;
  Engine* const e;
  const IvfKnobs knobs;
  const uint8_t* const ivf;
  const size_t len;
  int threads;
  uint8_t* const dst;
  const size_t dst_size;
  // the container
  int w = 0, h = 0;
  std::vector<Item> items;
  std::vector<uint32_t> gop_start;
  uint32_t shown_total = 0, max_frame_bytes = 0;
  int n_gops = 0;
  // the plan
  int tok_slots = 0, tok_chunk = 1, n_disp = 1, worker_nice = 5;
  size_t arena_tokens = 0;  // per worker (device-side token decoding)
  bool device_tokens = false;
  // shared between workers and dispatchers
  std::mutex mu;
  // one condition variable per worker: a batch wakes exactly the workers whose slots it freed (a shared one
  // woke every worker for every batch: hundreds of thousands of futile wake-ups per second of decoding)
  std::vector<std::condition_variable> cv_worker, cv_disp;
  std::vector<std::deque<Pending>> queues;
  std::vector<int> running;  // workers each dispatcher still serves
  std::atomic<int> next_gop{0};
  std::atomic<int> first_error{VP8GPU_OK};
  std::mutex stats_mu;
  double st_parse = 0, st_wait_slot = 0, st_wait_dma = 0, st_submit = 0, st_download = 0, st_disp_idle = 0;
  double st_batches = 0, st_jobs = 0;

  void set_error(int rc) {
    int ok = VP8GPU_OK;
    first_error.compare_exchange_strong(ok, rc);
  }
  static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
  // Frame::copy_to (frame.cc:272-307) on the worker's three reference handles
  static void advance_refs(Engine* e, int refs[3], const vp8gpu_frame_desc& desc, int out) {
    if (desc.key_frame) {
      set_ref(e, &refs[0], out);
      set_ref(e, &refs[1], out);
      set_ref(e, &refs[2], out);
    } else {
      if (desc.copy_to_alternate == 1) set_ref(e, &refs[2], refs[0]);
      else if (desc.copy_to_alternate == 2) set_ref(e, &refs[2], refs[1]);
      if (desc.copy_to_golden == 1) set_ref(e, &refs[1], refs[0]);
      else if (desc.copy_to_golden == 2) set_ref(e, &refs[1], refs[2]);
      if (desc.refresh_golden) set_ref(e, &refs[1], out);
      if (desc.refresh_alternate) set_ref(e, &refs[2], out);
      if (desc.refresh_last) set_ref(e, &refs[0], out);
    }
  }
  void worker_host(int tid);
  ivf_worker_kit* acquire_kit();
  void worker_device(int tid);
  void dispatcher(int di);
};

// IVF container (util/ivf.cc:36-82) -> items (frames from the first key frame on) and GOP boundaries
int IvfDecode::parse_container() {
  if (len < 32 || memcmp(ivf, "DKIF", 4) != 0) return e->fail(VP8GPU_ERR_INVALID, "missing IVF file header");
  if ((ivf[4] | (ivf[5] << 8)) != 0) return e->fail(VP8GPU_ERR_UNSUPPORTED, "not an IVF version 0 file");
  if ((ivf[6] | (ivf[7] << 8)) != 32) return e->fail(VP8GPU_ERR_UNSUPPORTED, "unsupported IVF header length");
  if (memcmp(ivf + 8, "VP80", 4) != 0) return e->fail(VP8GPU_ERR_UNSUPPORTED, "not a VP8 file");
  w = ivf[12] | (ivf[13] << 8), h = ivf[14] | (ivf[15] << 8);
  if (w != e->width() || h != e->height()) return e->fail(VP8GPU_ERR_UNSUPPORTED, "IVF size does not match the context");
  const uint32_t count = ivf[24] | (ivf[25] << 8) | (ivf[26] << 16) | ((uint32_t)ivf[27] << 24);
  const size_t frame_bytes = (size_t)w * h + 2 * (size_t)((w + 1) / 2) * ((h + 1) / 2);
  size_t pos = 32, out_off = 0;
  for (uint32_t i = 0; i < count; i++) {
    if (pos + 12 > len) return e->fail(VP8GPU_ERR_INVALID, "IVF file truncated");
    const uint32_t n = ivf[pos] | (ivf[pos + 1] << 8) | (ivf[pos + 2] << 16) | ((uint32_t)ivf[pos + 3] << 24);
    if (pos + 12 + n > len) return e->fail(VP8GPU_ERR_INVALID, "IVF file truncated");
    const uint8_t* p = ivf + pos + 12;
    pos += 12 + n;
    const bool key = n > 0 && !(p[0] & 1);
    if (items.empty() && !key) continue;  // FilePlayer starts at the first key frame
    if (key) gop_start.push_back((uint32_t)items.size());
    const bool shown = n > 0 && ((p[0] >> 4) & 1);
    Item it = {p, n, shown ? (int64_t)out_off : -1};
    if (shown) {
      out_off += frame_bytes;
      shown_total++;
    }
    items.push_back(it);
  }
  if (dst && dst_size < out_off) return e->fail(VP8GPU_ERR_LOGIC, "decode_ivf: destination too small");
  gop_start.push_back((uint32_t)items.size());
  n_gops = (int)gop_start.size() - 1;
  for (const Item& it : items) max_frame_bytes = it.n > max_frame_bytes ? it.n : max_frame_bytes;
  return VP8GPU_OK;
}

// how many workers, token-ring slots per worker, frames per k_tokens launch, dispatchers
void IvfDecode::plan() {
  if (threads < 1) threads = 1;
  if (threads > 512) threads = 512;
  if (threads > n_gops) threads = n_gops > 0 ? n_gops : 1;
  // device-side token decoding needs rasters for the frames a worker keeps in flight
  if (ctx->device_tokens.load()) {
    tok_slots = e->frames_free() / threads - 4;
    // k_tokens needs tens of milliseconds per frame (one thread each), so a worker wants to run a
    // GOP or two ahead of the pixel kernels; bounded by a device-memory budget for the rings: half of the
    // device (40 GB of an 80 GB H100), the other half for the rasters of the workers' frames in flight.
    // Measured on an H100 (bench.py 1080p, 64 workers): a quarter of the device leaves fewer slots per worker
    // and costs a fifth of the whole-decode throughput.
    size_t free_mem = 0, total_mem = (size_t)80 << 30;
    if (cudaSetDevice(e->device()) != cudaSuccess || cudaMemGetInfo(&free_mem, &total_mem) != cudaSuccess) total_mem = (size_t)80 << 30;
    const size_t ring_budget = total_mem / 2;
    // The slots hold records and partitions; the tokens go to an arena per worker, where a frame takes what its own
    // partitions can produce (Engine::token_cap_for), so that a slot costs what a typical frame needs and not what
    // the largest one does.  The arena holds at least the largest chunk (half the slots) of the largest frames and
    // two frames more (a chunk never waits for its own space, and wrapping around wastes less than a frame), and at
    // most what slots of the largest frame's size would take.
    const size_t worst = e->token_cap_for(max_frame_bytes), worst_bytes = worst * sizeof(vp8gpu_token);
    const size_t stride = e->token_ring_layout(ring_bytes_for(max_frame_bytes), true).stride;
    const size_t per_worker = ring_budget / (size_t)threads;
    // s * stride + (s / 2 + 2) * worst_bytes <= per_worker
    int want = per_worker > 2 * worst_bytes ? (int)std::min<size_t>((per_worker - 2 * worst_bytes) / (stride + worst_bytes / 2), kTokSlots) : 0;
    if (knobs.tok_slots >= 0) want = knobs.tok_slots;
    if (want > kTokSlots) want = kTokSlots;
    if (tok_slots > want) tok_slots = want;
    if (tok_slots < 4) tok_slots = 0;  // pool too small: the host workers parse everything
    if (tok_slots > 0) {
      const size_t room = per_worker > (size_t)tok_slots * stride ? (per_worker - (size_t)tok_slots * stride) / sizeof(vp8gpu_token) : 0;
      arena_tokens = std::max(std::min(room, (size_t)tok_slots * worst), (size_t)(tok_slots / 2 + 2) * worst);
      // VP8GPU_TOK_ARENA=<n>: room for n largest frames, never less than the floor above, so that a small stream on a large device can run
      // the allocator in the regime of a memory-bound plan (many workers, large frames)
      if (knobs.tok_arena >= 0) arena_tokens = std::max((size_t)knobs.tok_arena * worst, (size_t)(tok_slots / 2 + 2) * worst);
    }
  }
  device_tokens = tok_slots > 0;
  if (!device_tokens) {
    // host-token path: a worker holds up to kSlots queued outputs plus its three references, and
    // Engine::frame_alloc fails rather than blocks, so the worker count is bounded by the raster pool
    const int fit = e->frames_free() / 8;
    if (threads > fit) threads = fit > 0 ? fit : 1;
  }
  if (device_tokens) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->device());
    // The token warps in flight are not limited by default (the pipeline is bound by frames in flight);
    // the knob stays for experiments: VP8GPU_TOK_INFLIGHT=<frames>, 0 = unlimited.
    int cap = 0;
    (void)sms;
    if (knobs.tok_inflight >= 0) cap = knobs.tok_inflight;
    std::lock_guard<std::mutex> lk(ctx->tok_mu);
    ctx->tok_capacity = cap;
    ctx->tok_permits = cap;  // every earlier call has returned: all permits are back
  }
  tok_chunk = tok_slots / 3 > kTokChunk ? kTokChunk : (tok_slots / 3 > 0 ? tok_slots / 3 : 1);
  if (knobs.tok_chunk >= 0) {
    const int c = knobs.tok_chunk;
    if (c >= 1 && c <= tok_slots / 2) tok_chunk = c;
  }
  n_disp = device_tokens ? (threads >= 32 ? 4 : (threads >= 8 ? 2 : 1)) : 1;
  if (knobs.dispatchers >= 0) {
    const int n = knobs.dispatchers;
    if (n >= 1 && n <= 16 && n <= threads) n_disp = n;
  }
  // The dispatchers feed the device and must not queue behind dozens of parsing workers for a CPU: the workers
  // run at a lower priority (per-thread nice on Linux; VP8GPU_WORKER_NICE overrides, 0 = leave alone).
  if (knobs.worker_nice >= 0) worker_nice = knobs.worker_nice;
  cv_worker = std::vector<std::condition_variable>(threads);
  cv_disp = std::vector<std::condition_variable>(n_disp);
  queues.assign(threads, {});
  running.assign(n_disp, 0);
  for (int t = 0; t < threads; t++) running[t % n_disp]++;
}

// Host workers only parse (CPU entropy front end) and keep the per-GOP codec state; a dispatcher gathers
// whatever they have produced -- at most one frame per worker, because consecutive frames of a GOP depend on
// each other -- into ONE batched decode per round, so the device sees a few large launches instead of three small
// ones per frame, and the wavefront kernels get rows of many frames to hide their latency with.
void IvfDecode::worker_host(int tid) {
  cudaSetDevice(e->device());
  double t_parse = 0, t_slot = 0, t_dma = 0;
  State state(w, h);
  int refs[3] = {-1, -1, -1};
  vp8gpu_parsed* slots[kSlots] = {};
  int slot_state[kSlots] = {};
  int next_slot = 0;
  int rc = VP8GPU_OK;
  for (;;) {
    const int g = next_gop.fetch_add(1);
    if (g >= n_gops || first_error.load() != VP8GPU_OK) break;
    for (uint32_t i = gop_start[g]; i < gop_start[g + 1] && rc == VP8GPU_OK; i++) {
      const int si = next_slot;
      next_slot = (next_slot + 1) % kSlots;
      if (!slots[si]) {
        {
          std::lock_guard<std::mutex> lk(ctx->pool_mu);
          if (!ctx->pinned_pool.empty()) {
            slots[si] = ctx->pinned_pool.back();
            ctx->pinned_pool.pop_back();
          }
        }
        if (!slots[si]) {
          slots[si] = new vp8gpu_parsed(kPinned);
          cudaEventCreateWithFlags(&slots[si]->consumed, kWaitableEvent);
          const size_t n_mbs = (size_t)e->geom().mb_cols * e->geom().mb_rows;
          slots[si]->f.mbs.reserve(n_mbs, 0);
          slots[si]->f.tokens.reserve(n_mbs * 32 + 1024, 0);
          slots[si]->f.split.reserve(256, 0);
        }
      }
      vp8gpu_parsed* p = slots[si];
      const double t0 = now();
      {  // the dispatcher must have picked the slot's previous frame up ...
        std::unique_lock<std::mutex> lk(mu);
        cv_worker[tid].wait(lk, [&] { return slot_state[si] == kFree; });
      }
      const double t1 = now();
      if (p->busy) {  // ... and the DMA engine must have read it
        cudaEventSynchronize(p->consumed);
        p->busy = false;
      }
      const double t2 = now();
      rc = vp8::parse_frame(state, items[i].p, items[i].n, p->f);
      if (rc != VP8GPU_OK) break;
      count_mbs(p);
      t_slot += t1 - t0;
      t_dma += t2 - t1;
      t_parse += now() - t2;
      const vp8gpu_frame_desc& desc = p->f.desc;
      Pending job;
      job.slot = p;
      job.slot_state = &slot_state[si];
      job.out_off = (dst && desc.show_frame) ? items[i].out_off : -1;
      rc = e->frame_alloc(&job.out);
      if (rc != VP8GPU_OK) break;
      for (int k = 0; k < 3; k++) {
        job.refs[k] = desc.key_frame ? -1 : refs[k];
        if (job.refs[k] >= 0) e->frame_retain(job.refs[k]);  // keeps the raster alive until submitted
      }
      advance_refs(e, refs, desc, job.out);  // Frame::copy_to
      {
        std::lock_guard<std::mutex> lk(mu);
        slot_state[si] = kQueued;
        job.tid = tid;
        queues[tid].push_back(job);
      }
      cv_disp[tid % n_disp].notify_one();
    }
    if (rc != VP8GPU_OK) {
      set_error(rc);
      break;
    }
  }
  {  // wait until everything this worker queued has been submitted, then retire
    std::unique_lock<std::mutex> lk(mu);
    cv_worker[tid].wait(lk, [&] {
      for (int k = 0; k < kSlots; k++)
        if (slot_state[k] != kFree) return false;  // the dispatcher still owns that slot
      return true;
    });
    running[tid % n_disp]--;
  }
  cv_disp[tid % n_disp].notify_one();
  {
    std::lock_guard<std::mutex> lk(stats_mu);
    st_parse += t_parse;
    st_wait_slot += t_slot;
    st_wait_dma += t_dma;
  }
  for (int k = 0; k < 3; k++)
    if (refs[k] >= 0) e->frame_release(refs[k]);
  for (auto* p : slots)
    if (p) {
      if (p->busy) {
        cudaEventSynchronize(p->consumed);
        p->busy = false;
      }
      std::lock_guard<std::mutex> lk(ctx->pool_mu);
      ctx->pinned_pool.push_back(p);
    }
}

// ---- workers with device-side token decoding: the host only walks the first partition; the DCT
//      partitions of up to tok_chunk frames go to the device in one k_tokens launch on the worker's
//      own stream, tok_slots frames may be in flight per worker, and the dispatcher picks a frame up
//      once its `ready` event has fired ----
ivf_worker_kit* IvfDecode::acquire_kit() {
  ivf_worker_kit* k = nullptr;
  {
    std::lock_guard<std::mutex> lk(ctx->pool_mu);
    for (size_t i = 0; i < ctx->kit_pool.size(); i++)
      if (ctx->kit_pool[i]->ring->bits_cap >= max_frame_bytes + 16 && ctx->kit_pool[i]->ring->nslots >= tok_slots &&
          ctx->kit_pool[i]->ring->arena_cap >= arena_tokens) {
        k = ctx->kit_pool[i];
        ctx->kit_pool.erase(ctx->kit_pool.begin() + i);
        break;
      }
  }
  if (k) return k;  // its overflow flags are clear: worker_device clears a flagged slot before pooling the kit
  k = new ivf_worker_kit();
  bool ok = e->token_ring_create(tok_slots, ring_bytes_for(max_frame_bytes), &k->ring, arena_tokens) == VP8GPU_OK &&
            cudaStreamCreateWithFlags(&k->copy_stream, cudaStreamNonBlocking) == cudaSuccess;
  for (cudaStream_t& st : k->kstream) ok = ok && cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess;
  if (!ok) {
    if (k->ring) e->token_ring_free(k->ring);
    if (k->copy_stream) cudaStreamDestroy(k->copy_stream);
    for (cudaStream_t st : k->kstream)
      if (st) cudaStreamDestroy(st);
    delete k;
    return nullptr;
  }
  const size_t n_mbs = (size_t)e->geom().mb_cols * e->geom().mb_rows;
  for (int i = 0; i < tok_slots; i++) {
    k->parsed[i] = new vp8gpu_parsed(kPinned);
    k->parsed[i]->f.mbs.reserve(n_mbs, 0);
    k->parsed[i]->f.split.reserve(256, 0);
    cudaEventCreateWithFlags(&k->staged[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&k->ready[i], cudaEventDisableTiming);
  }
  return k;
}

void IvfDecode::worker_device(int tid) {
  if (worker_nice > 0) setpriority(PRIO_PROCESS, (id_t)syscall(SYS_gettid), worker_nice);
  cudaSetDevice(e->device());
  double t_parse = 0, t_slot = 0, t_dma = 0;
  State state(w, h);
  int refs[3] = {-1, -1, -1};
  int slot_state[kTokSlots] = {};
  int next_slot = 0;
  int launches_done = 0;
  int rc = VP8GPU_OK;
  ivf_worker_kit* kit = acquire_kit();
  if (!kit) rc = e->fail(VP8GPU_ERR_NOMEM, "decode_ivf: token ring allocation failed");
  // The token arena is used as a ring in staging order, which is slot order: the space of the oldest frames comes
  // back first.  live: slots that hold arena space, oldest first; [start, start + len) their tokens.
  // The plan's size, not the kit's: a kit from an earlier call may hold a larger arena.
  // Counters (VP8GPU_TRACE): pieces taken, pieces placed back at offset 0, frames waited for to free space.
  std::deque<int> live;
  size_t head = 0, a_start[kTokSlots] = {};
  bool held[kTokSlots] = {};
  long n_takes = 0, n_wraps = 0, n_waits = 0;
  auto arena_take = [&](int si, size_t need, auto in_chunk, vp8gpu_token** out) {
    const size_t cap = arena_tokens;
    if (held[si]) {  // the slot's previous frame is done: its space is the oldest
      live.erase(std::find(live.begin(), live.end(), si));
      held[si] = false;
    }
    for (;;) {
      size_t at = SIZE_MAX;
      if (live.empty()) {
        at = need <= cap ? 0 : SIZE_MAX;
      } else {
        const size_t tail = a_start[live.front()];
        if (head > tail) {  // in use: [tail, head)
          if (cap - head >= need) at = head;
          else if (tail >= need) at = 0;
        } else if (tail - head >= need) {  // in use: [tail, end) and [0, head)
          at = head;
        }
      }
      if (at != SIZE_MAX) {
        n_takes++;
        if (at == 0 && head > 0) n_wraps++;
        a_start[si] = at;
        head = at + need;
        held[si] = true;
        live.push_back(si);
        *out = kit->ring->arena + at;
        return VP8GPU_OK;
      }
      // wait for the oldest frame's pixel kernels (plan() sizes the arena so that it is never one of this chunk)
      if (live.empty() || in_chunk(live.front())) return e->fail(VP8GPU_ERR_LOGIC, "decode_ivf: token arena too small");
      const int s = live.front();
      n_waits++;
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_worker[tid].wait(lk, [&] { return slot_state[s] == kFree; });
      }
      if (kit->busy[s]) {
        if (kit->finished[s]) cudaEventSynchronize(kit->finished[s]);
        kit->busy[s] = false;
      }
      live.pop_front();
      held[s] = false;
    }
  };
  while (rc == VP8GPU_OK) {
    const int g = next_gop.fetch_add(1);
    if (g >= n_gops || first_error.load() != VP8GPU_OK) break;
    uint32_t i = gop_start[g];
    while (i < gop_start[g + 1] && rc == VP8GPU_OK) {
      const uint32_t left = gop_start[g + 1] - i;
      // slow start: the first launches of a worker are small so that its pixel work can begin
      // after one k_tokens latency instead of after a whole chunk's parse time on top of it
      int want = tok_chunk;
      if (launches_done < 3 && (2 << launches_done) < want) want = 2 << launches_done;
      launches_done++;
      const int n = (int)left < want ? (int)left : want;
      const int first_slot = next_slot;
      int staged = 0, permits_taken = 0;
      for (int c = 0; c < n && rc == VP8GPU_OK; c++) {
        const int si = (first_slot + c) % tok_slots;
        const double t0 = now();
        {  // the dispatcher must have submitted the slot's previous frame ...
          std::unique_lock<std::mutex> lk(mu);
          cv_worker[tid].wait(lk, [&] { return slot_state[si] == kFree; });
        }
        const double t1 = now();
        if (kit->busy[si]) {  // ... and the pixel kernels must have read its records
          if (kit->finished[si]) cudaEventSynchronize(kit->finished[si]);
          kit->busy[si] = false;
        }
        const double t2 = now();
        vp8gpu_parsed* p = kit->parsed[si];
        rc = knobs.parse_cache ? parse_first_partition_cached(state, items[i + c].p, items[i + c].n, p->f)
                               : vp8::parse_frame(state, items[i + c].p, items[i + c].n, p->f, true);
        if (rc != VP8GPU_OK) break;
        count_mbs(p);
        vp8gpu_token* tokens = nullptr;
        rc = arena_take(si, e->token_cap_for(p->f.tw.bits_len), [&](int s) {  // staged in this chunk
          return (s - first_slot + tok_slots) % tok_slots < c;
        }, &tokens);
        if (rc != VP8GPU_OK) break;
        rc = e->token_ring_stage(kit->ring, si, p->f, kit->copy_stream, tokens);
        if (rc != VP8GPU_OK) break;
        staged++;
        t_slot += t1 - t0;
        t_dma += t2 - t1;
        t_parse += now() - t2;
      }
      if (rc != VP8GPU_OK) break;
      cudaStream_t ks = kit->kstream[kit->next_kstream];
      kit->next_kstream = (kit->next_kstream + 1) % kTokStreams;
      cudaEventRecord(kit->staged[first_slot], kit->copy_stream);
      cudaStreamWaitEvent(ks, kit->staged[first_slot], 0);
      if (ctx->tok_capacity > 0) {  // permits for the frames of this launch (returned by tok_release_cb when the kernel is done)
        std::unique_lock<std::mutex> lk(ctx->tok_mu);
        const int need = staged < ctx->tok_capacity ? staged : ctx->tok_capacity;
        ctx->tok_cv.wait(lk, [&] { return ctx->tok_permits >= need; });
        ctx->tok_permits -= need;
        permits_taken = need;
      }
      // the ring is used modulo tok_slots (<= its real size): a chunk that wraps needs two launches
      const int until_wrap = tok_slots - first_slot;
      rc = e->token_ring_launch(kit->ring, first_slot, staged < until_wrap ? staged : until_wrap, ks);
      if (rc == VP8GPU_OK && staged > until_wrap) rc = e->token_ring_launch(kit->ring, 0, staged - until_wrap, ks);
      if (rc == VP8GPU_OK)
        cudaEventRecord(kit->ready[first_slot], ks);  // one event per launch: its frames become ready together
      // the permits come back when the stream gets here (also after a failed launch); queued after the
      // `ready` events so that the host-function thread is not on the frames' critical path
      if (permits_taken && cudaLaunchHostFunc(ks, tok_release_cb, new TokRelease{ctx, permits_taken}) != cudaSuccess) {
        std::lock_guard<std::mutex> lk(ctx->tok_mu);
        ctx->tok_permits += permits_taken;
      }
      if (rc != VP8GPU_OK) break;
      for (int c = 0; c < staged && rc == VP8GPU_OK; c++) {
        const int si = (first_slot + c) % tok_slots;
        vp8gpu_parsed* p = kit->parsed[si];
        const vp8gpu_frame_desc& desc = p->f.desc;
        Pending job;
        job.slot = p;
        job.slot_state = &slot_state[si];
        job.out_off = (dst && desc.show_frame) ? items[i + c].out_off : -1;
        job.ring = kit->ring;
        job.ring_slot = si;
        job.ready = kit->ready[first_slot];
        job.finished = &kit->finished[si];
        rc = e->frame_alloc(&job.out);
        if (rc != VP8GPU_OK) break;
        for (int k = 0; k < 3; k++) {
          job.refs[k] = desc.key_frame ? -1 : refs[k];
          if (job.refs[k] >= 0) e->frame_retain(job.refs[k]);
        }
        advance_refs(e, refs, desc, job.out);  // Frame::copy_to
        kit->busy[si] = true;
        {
          std::lock_guard<std::mutex> lk(mu);
          slot_state[si] = kQueued;
          job.tid = tid;
        queues[tid].push_back(job);
        }
        cv_disp[tid % n_disp].notify_one();
      }
      next_slot = (first_slot + staged) % tok_slots;
      i += (uint32_t)staged;
    }
    if (rc != VP8GPU_OK) break;
  }
  if (rc != VP8GPU_OK) set_error(rc);
  {  // wait until everything this worker queued has been submitted, then retire
    std::unique_lock<std::mutex> lk(mu);
    cv_worker[tid].wait(lk, [&] {
      for (int k = 0; k < kTokSlots; k++)
        if (slot_state[k] != kFree) return false;
      return true;
    });
    running[tid % n_disp]--;
  }
  cv_disp[tid % n_disp].notify_one();
  {
    std::lock_guard<std::mutex> lk(stats_mu);
    st_parse += t_parse;
    st_wait_slot += t_slot;
    st_wait_dma += t_dma;
  }
  for (int k = 0; k < 3; k++)
    if (refs[k] >= 0) e->frame_release(refs[k]);
  if (kit) {
    for (int k = 0; k < kTokSlots; k++)
      if (kit->busy[k]) {
        if (kit->finished[k]) cudaEventSynchronize(kit->finished[k]);
        kit->busy[k] = false;
      }
    cudaStreamSynchronize(kit->copy_stream);
    for (cudaStream_t st : kit->kstream) cudaStreamSynchronize(st);
    // k_tokens reports a token pool that was too small instead of writing out of bounds; the capacity
    // rule (Engine::token_ring_layout) makes that impossible, so a set flag is an internal error.  The flag is
    // sticky: it covers every frame this call staged in the slot, not only the last one.  A kit goes back to the pool
    // with every flag clear (slots beyond tok_slots were not used by this call and are still clear).
    uint32_t res[kTokSlots][2];
    if (cudaMemcpy2D(res, 8, kit->ring->dev + kit->ring->result_off, kit->ring->stride, 8, (size_t)kit->ring->nslots,
                     cudaMemcpyDeviceToHost) == cudaSuccess) {
      bool cleared = false;
      for (int k = 0; k < kit->ring->nslots && k < tok_slots; k++)
        if (res[k][1]) {
          set_error(e->fail(VP8GPU_ERR_LOGIC, "device token pool overflow"));
          cleared = e->token_ring_clear_result(kit->ring, k, kit->copy_stream) == VP8GPU_OK || cleared;
        }
      if (cleared) cudaStreamSynchronize(kit->copy_stream);
    }
    if (knobs.trace)
      fprintf(stderr, "decode_ivf arena: worker %d takes %ld wraps %ld waits %ld cap %zu slots %d chunk %d\n", tid, n_takes, n_wraps,
              n_waits, arena_tokens, tok_slots, tok_chunk);
    std::lock_guard<std::mutex> lk(ctx->pool_mu);
    ctx->kit_pool.push_back(kit);
  }
}

// Dispatchers: dispatcher d serves the workers with tid % D == d on its own two lanes.  Queueing a
// frame costs a few dozen driver calls (stream ordering of its rasters, the launches, the download),
// which one thread cannot do for more than ~10k frames/s.
void IvfDecode::dispatcher(int di) {
  cudaSetDevice(e->device());
  std::vector<Pending> batch;
  std::vector<HostJob> hj;
  std::vector<int> dl_ids;
  std::vector<uint8_t*> dl_dst;
  int round = 0;
  double t_idle = 0, t_submit = 0, t_download = 0, n_batches = 0, n_jobs = 0;
  // VP8GPU_TRACE=1: device-side duration of every batch (diagnostic, printed to stderr)
  struct Trace {
    cudaEvent_t a, b;
    int lane, n;
    double host_t;
    cudaEvent_t mid[4] = {nullptr, nullptr, nullptr, nullptr};  // -, after k_inter, after k_intra, before k_inter
  };
  std::vector<Trace> trace;
  const bool tracing = knobs.trace;
  for (;;) {
    batch.clear();
    const double ti = now();
    {
      std::unique_lock<std::mutex> lk(mu);
      // a queue's front is eligible once its tokens are in HBM (device-side token decoding)
      // The answer is remembered: once the event of a chunk has fired, every frame of that chunk at the head of
      // the queue is marked (a query takes the driver's lock, and this runs for every queue on every poll --
      // hundreds of thousands of queries per second next to the workers' own CUDA calls).
      auto eligible = [&](std::deque<Pending>& q) {
        if (q.empty()) return false;
        Pending& f = q.front();
        if (!f.ready) return true;
        if (cudaEventQuery(f.ready) != cudaSuccess) return false;
        const cudaEvent_t fired = f.ready;
        for (Pending& p : q) {
          if (p.ready != fired) break;
          p.ready = nullptr;
        }
        return true;
      };
      auto ready = [&] {
        int n = 0;
        for (int t = di; t < threads; t += n_disp) n += eligible(queues[t]);
        return n;
      };
      auto queued = [&] {
        for (int t = di; t < threads; t += n_disp)
          if (!queues[t].empty()) return true;
        return false;
      };
      // nothing signals the condition variable when a CUDA event fires: poll while frames wait for one
      while (!(running[di] == 0 && !queued()) && ready() == 0) {
        if (queued()) cv_disp[di].wait_for(lk, std::chrono::microseconds(100));
        else cv_disp[di].wait(lk);
      }
      // Device time per batch is almost flat in the number of frames (the wavefront kernels
      // are latency bound), so give the other workers a moment to finish their current frame:
      // go once most of them have something queued, or after a short grace period.
      const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(1500);
      while (running[di] > 0 && ready() < (running[di] * 3 + 3) / 4) {
        if (device_tokens) {
          if (std::chrono::steady_clock::now() >= deadline) break;
          cv_disp[di].wait_for(lk, std::chrono::microseconds(100));
        } else if (cv_disp[di].wait_until(lk, deadline) == std::cv_status::timeout) {
          break;
        }
      }
      for (int t = di; t < threads; t += n_disp)
        if (eligible(queues[t])) {
          batch.push_back(queues[t].front());
          queues[t].pop_front();
        }
      if (batch.empty() && running[di] == 0 && !queued()) break;
    }
    if (batch.empty()) continue;
    const double ts = now();
    t_idle += ts - ti;
    n_batches += 1;
    n_jobs += batch.size();
    const int lane = 2 * di + (round++ & 1);
    hj.clear();
    for (const Pending& b : batch) {
      HostJob j;
      j.desc = &b.slot->f.desc;
      j.mbs = b.slot->f.mbs.data();
      j.tokens = b.slot->f.tokens.data();
      j.split = b.slot->f.split.data();
      memcpy(j.refs, b.refs, sizeof(j.refs));
      j.out = b.out;
      j.n_intra = (int)b.slot->n_intra;
      j.n_filtered = (int)b.slot->n_filtered;
      j.consumed = b.slot->consumed;  // fires as soon as the records are in HBM, before the kernels
      if (b.ring) {
        j.ring = b.ring;
        j.ring_slot = b.ring_slot;
        j.ready = nullptr;  // already fired (eligible() checked it)
        j.finished = b.finished;
        j.consumed = nullptr;
      }
      hj.push_back(j);
    }
    Trace tr{nullptr, nullptr, lane, (int)batch.size(), ts};
    if (tracing) {
      e->ensure_lane(lane);
      cudaEventCreate(&tr.a);
      cudaEventCreate(&tr.b);
      for (cudaEvent_t& m : tr.mid) cudaEventCreate(&m);
      cudaEventRecord(tr.a, e->stream(lane));
    }
    int rc = e->submit(lane, hj.data(), (int)hj.size(), nullptr, tracing ? tr.mid + 1 : nullptr);
    if (tracing) {
      cudaEventRecord(tr.b, e->stream(lane));
      trace.push_back(tr);
    }
    const double td = now();
    t_submit += td - ts;
    if (rc == VP8GPU_OK) {
      dl_ids.clear();
      dl_dst.clear();
      for (const Pending& b : batch) {
        if (!b.ring) b.slot->busy = true;
        if (b.out_off >= 0) {
          dl_ids.push_back(b.out);
          dl_dst.push_back(dst + b.out_off);
        }
      }
      if (!dl_ids.empty()) rc = e->frames_download_display(dl_ids.data(), dl_dst.data(), (int)dl_ids.size(), lane);
    }
    for (const Pending& b : batch) {
      for (int k = 0; k < 3; k++)
        if (b.refs[k] >= 0) e->frame_release(b.refs[k]);
      e->frame_release(b.out);
    }
    if (rc != VP8GPU_OK) set_error(rc);
    t_download += now() - td;
    {
      std::lock_guard<std::mutex> lk(mu);
      for (const Pending& b : batch) *b.slot_state = kFree;
    }
    for (const Pending& b : batch) cv_worker[b.tid].notify_one();
  }
  e->sync_lane(2 * di);
  e->sync_lane(2 * di + 1);
  if (tracing && !trace.empty()) {
    // per batch: device time from "stream reaches the batch" to "its kernels are done", and the
    // device-side gap to the previous batch of this dispatcher
    double sum_ms = 0, sum_gap = 0, first_host = trace.front().host_t, last_host = trace.back().host_t;
    double sum_intra = 0, sum_lf = 0, sum_inter = 0, sum_pre = 0, sum_turn = 0;
    float ms = 0;
    for (size_t i = 0; i < trace.size(); i++) {
      if (cudaEventElapsedTime(&ms, trace[i].mid[3], trace[i].mid[1]) == cudaSuccess) sum_inter += ms;
      if (cudaEventElapsedTime(&ms, trace[i].a, trace[i].mid[3]) == cudaSuccess) sum_pre += ms;
      if (cudaEventElapsedTime(&ms, trace[i].mid[1], trace[i].mid[2]) == cudaSuccess) sum_intra += ms;
      if (cudaEventElapsedTime(&ms, trace[i].mid[2], trace[i].b) == cudaSuccess) sum_lf += ms;
      cudaEventElapsedTime(&ms, trace[i].a, trace[i].b);
      sum_ms += ms;
      if (i) {
        cudaEventElapsedTime(&ms, trace[i - 1].b, trace[i].b);
        sum_gap += ms;
        // device-side turn-around: end of the previous batch -> first kernel of this one (negative: overlapped)
        if (cudaEventElapsedTime(&ms, trace[i - 1].b, trace[i].mid[3]) == cudaSuccess) sum_turn += ms;
      }
    }
    fprintf(stderr, "[trace] dispatcher %d: %zu batches, avg %.2f frames, device %.3f ms per batch, end-to-end period %.3f ms, "
            "host span %.1f ms; per batch: waits + upload %.3f ms, k_inter %.3f ms, k_intra %.3f ms, k_loopfilter %.3f ms, turn-around %.3f ms\n", di,
            trace.size(), n_jobs / n_batches, sum_ms / trace.size(), trace.size() > 1 ? sum_gap / (trace.size() - 1) : 0.0,
            (last_host - first_host) * 1e3, sum_pre / trace.size(), sum_inter / trace.size(), sum_intra / trace.size(),
            sum_lf / trace.size(), trace.size() > 1 ? sum_turn / (trace.size() - 1) : 0.0);
    for (Trace& t : trace) {
      cudaEventDestroy(t.a);
      cudaEventDestroy(t.b);
      for (cudaEvent_t m : t.mid)
        if (m) cudaEventDestroy(m);
    }
  }
  std::lock_guard<std::mutex> lk(stats_mu);
  st_disp_idle += t_idle;
  st_submit += t_submit;
  st_download += t_download;
  st_batches += n_batches;
  st_jobs += n_jobs;
}

int IvfDecode::run(uint32_t* n_decoded, uint32_t* n_shown) {
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; t++) {
    if (device_tokens) pool.emplace_back(&IvfDecode::worker_device, this, t);
    else pool.emplace_back(&IvfDecode::worker_host, this, t);
  }
  std::vector<std::thread> dispatchers;
  for (int d = 1; d < n_disp; d++) dispatchers.emplace_back(&IvfDecode::dispatcher, this, d);
  dispatcher(0);
  for (auto& t : dispatchers) t.join();
  for (auto& t : pool) t.join();
  ctx->stats[0] = st_parse;
  ctx->stats[1] = st_wait_slot;
  ctx->stats[2] = st_wait_dma;
  ctx->stats[3] = st_submit;
  ctx->stats[4] = st_download;
  ctx->stats[5] = st_disp_idle;
  ctx->stats[6] = st_batches;
  ctx->stats[7] = st_jobs;
  if (n_decoded) *n_decoded = (uint32_t)items.size();
  if (n_shown) *n_shown = shown_total;
  return first_error.load();
}

int vp8gpu_decode_ivf(vp8gpu_ctx* ctx, const uint8_t* ivf, size_t len, int threads, uint8_t* dst, size_t dst_size,
                      uint32_t* n_decoded, uint32_t* n_shown) {
  if (!ctx || !ivf) return VP8GPU_ERR_LOGIC;
  IvfDecode job(ctx, ivf, len, threads, dst, dst_size);
  const int rc = job.parse_container();
  if (rc != VP8GPU_OK) return rc;
  job.plan();
  return job.run(n_decoded, n_shown);
}

}  // extern "C"
