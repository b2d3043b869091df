// engine.cu -- see engine.hpp.
//
// Ownership model = the reference's RasterHandle (decoder/raster_handle.hh:95-123): device
// rasters are reference counted, immutable once a decode has been queued into them, and return
// to a per-context pool (not a process-global one, cf. raster_handle.cc:74-83).  Because work is
// asynchronous and several decoders run on different CUDA streams ("lanes"), every raster
// remembers which streams touched it (one event per stream slot); a stream that wants to read,
// or to recycle and overwrite, a raster first waits for the other streams' events.
#include "engine.hpp"

#include <cuda.h>  // CUtensorMap types only: the driver entry point is fetched through the runtime
#include <stdlib.h>
#include <string.h>

namespace vp8 {

int launch_compare(const uint8_t* a, const uint8_t* b, const Geom& g, int* d_flag, void* stream);
int launch_hash(const uint8_t* a, const Geom& g, unsigned long long* d_out, void* stream);

namespace {
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Tensor maps live in a per-device arena whose slots are handed out once and never reused or freed: a map
// is written (cudaMemcpy) before the first kernel that can see its address is launched and is immutable
// afterwards, so the TMA unit's descriptor cache can never hold a stale copy and k_inter needs no
// tensormap-proxy fence per use (measured: one `fence.proxy.tensormap::generic.acquire.sys` per window
// makes k_inter 9x slower).  384 bytes per raster.
std::mutex g_tmap_mu;
struct TmapChunk {
  uint8_t* base;
  size_t used, cap;
};
std::vector<TmapChunk> g_tmap_chunks[64];
uint8_t* tmap_arena_alloc(int device, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  if (device < 0 || device >= 64) return nullptr;
  auto& chunks = g_tmap_chunks[device];
  if (chunks.empty() || chunks.back().used + bytes > chunks.back().cap) {
    TmapChunk c{nullptr, 0, bytes > ((size_t)4 << 20) ? bytes : ((size_t)4 << 20)};
    if (cudaMalloc(&c.base, c.cap) != cudaSuccess) return nullptr;
    chunks.push_back(c);
  }
  uint8_t* p = chunks.back().base + chunks.back().used;
  chunks.back().used += align_up(bytes, 128);
  return p;
}
constexpr int kSyncHeaderInts = 64;  // [0] = intra ticket, [32] = loop-filter ticket (own cache lines)
}  // namespace

// workers and dispatchers of vp8gpu_decode_ivf report errors concurrently: the text has its own lock
std::string& Engine::thread_error() {
  thread_local std::string err;
  return err;
}
int Engine::fail(int code, const std::string& what) {
  std::lock_guard<std::mutex> lk(err_mu_);
  err_ = what;
  thread_error() = what;
  return code;
}
int Engine::cuda_fail(cudaError_t e, const char* what) {
  std::lock_guard<std::mutex> lk(err_mu_);
  err_ = std::string(what) + ": " + cudaGetErrorString(e);
  thread_error() = err_;
  return VP8GPU_ERR_CUDA;
}
#define CU(call)                                             \
  do {                                                       \
    cudaError_t e__ = (call);                                \
    if (e__ != cudaSuccess) return cuda_fail(e__, #call);    \
  } while (0)

int Engine::create(int device, int width, int height, int max_frames, Engine** out, std::string* err) {
  if (width <= 0 || height <= 0 || width > 16383 || height > 16383) {
    if (err) *err = "bad frame size";
    return VP8GPU_ERR_LOGIC;
  }
  // vp8gpu_decode_ivf keeps hundreds of streams busy (per worker: uploads, token kernels that run for tens of
  // milliseconds one after the other); with the default 8 hardware work queues the short pixel batches of the
  // dispatcher lanes queue behind them (false dependencies between streams that share a queue).  Ask for the
  // maximum; only effective if this is the process's first CUDA call, and never overrides the user's setting.
  setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || device < 0 || device >= ndev) {
    if (err) *err = std::string("no usable CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "bad index");
    return VP8GPU_ERR_CUDA;
  }
  e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    if (err) *err = cudaGetErrorString(e);
    return VP8GPU_ERR_CUDA;
  }
  Engine* en = new Engine();
  en->device_ = device;
  en->width_ = width;
  en->height_ = height;
  Geom& g = en->g_;
  g.mb_cols = (width + 15) / 16;
  g.mb_rows = (height + 15) / 16;
  g.W = 16 * g.mb_cols;
  g.H = 16 * g.mb_rows;
  g.y_pitch = (int)align_up(g.W, 32);
  g.c_pitch = g.y_pitch / 2;
  g.u_off = (uint32_t)((size_t)g.y_pitch * g.H);
  g.v_off = g.u_off + (uint32_t)((size_t)g.c_pitch * (g.H / 2));
  g.frame_bytes = g.v_off + (uint32_t)((size_t)g.c_pitch * (g.H / 2));
  if (const char* v = getenv("VP8GPU_WAVEFRONT"))
    en->ll_mask_ = !strcmp(v, "legacy") ? 0 : (!strcmp(v, "ll") ? 3 : (!strcmp(v, "lf-ll") ? 2 : (!strcmp(v, "intra-ll") ? 1 : en->ll_mask_)));
  // hand-over areas only for the kernels that use them (the loop filter's is two thirds of a raster)
  g.msg_lf_off = (uint32_t)align_up((size_t)g.frame_bytes + 64, 256);  // + 64: slack read by staged window rows
  g.msg_intra_off = g.msg_lf_off + ((en->ll_mask_ & 2) ? (uint32_t)((size_t)g.mb_rows * (g.mb_cols + 1) * 32 * 8) : 0u);
  g.alloc_bytes = g.msg_intra_off + ((en->ll_mask_ & 1) ? (uint32_t)((size_t)g.mb_rows * g.mb_cols * 8 * 8) : 0u);
  if (max_frames <= 0) max_frames = 64;
  en->tmaps_ = tmap_arena_alloc(device, (size_t)max_frames * 384);
  if (!en->tmaps_) {
    if (err) *err = "cudaMalloc(tensor map arena) failed";
    delete en;
    return VP8GPU_ERR_CUDA;
  }
  en->frames_.resize(max_frames);
  for (int i = max_frames - 1; i >= 0; i--) en->free_.push_back(i);
  *out = en;
  return VP8GPU_OK;
}

Engine::~Engine() {
  cudaSetDevice(device_);
  cudaDeviceSynchronize();
  for (auto& f : frames_) {
    if (f.dev) cudaFree(f.dev);
  }
  for (auto& ring : ring_)
    for (auto& ev : ring)
      if (ev) cudaEventDestroy(ev);
  for (int l = 0; l < kMaxLanes; l++)
    for (auto& s : staging_[l]) {
      if (s.dev) cudaFree(s.dev);
      if (s.host) cudaFreeHost(s.host);
      if (s.done) cudaEventDestroy(s.done);
    }
  for (auto& s : lanes_)
    if (s) cudaStreamDestroy(s);
  if (cmp_scratch_) cudaFree(cmp_scratch_);
  for (float* p : ssim_dev_)
    if (p) cudaFree(p);
  for (float* p : ssim_host_)
    if (p) cudaFreeHost(p);
  // tmaps_ belongs to the tensor-map arena: never reused, never freed
}

// One 2-D tensor map per plane of raster `id` (u8 elements, plane size W x H resp. W/2 x H/2, row pitch
// from Geom), box = 48 x 21 luma / 32 x 13 chroma: the source window of a six-tap prediction
// (prediction.cc:655-674) with its 2 + 3 pixel halo, plus up to 15 pixels of slack because a box has to
// start on a 16-byte boundary of the row.  Out-of-range pixels are zero-filled by the hardware, so
// k_inter only uses TMA for windows inside the plane.
int Engine::make_tensor_maps(int id) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CU(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) return fail(VP8GPU_ERR_CUDA, "cuTensorMapEncodeTiled not available");
    encode = reinterpret_cast<EncodeFn>(fn);
  }
  alignas(64) CUtensorMap maps[3];
  for (int p = 0; p < 3; p++) {
    uint8_t* base = frames_[id].dev + (p == 0 ? 0 : (p == 1 ? g_.u_off : g_.v_off));
    const cuuint64_t dims[2] = {(cuuint64_t)(p ? g_.W / 2 : g_.W), (cuuint64_t)(p ? g_.H / 2 : g_.H)};
    const cuuint64_t strides[1] = {(cuuint64_t)(p ? g_.c_pitch : g_.y_pitch)};
    const cuuint32_t box[2] = {p ? 32u : 48u, p ? 13u : 21u};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode(&maps[p], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(VP8GPU_ERR_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
  }
  static_assert(sizeof(CUtensorMap) == 128, "tensor map size");
  CU(cudaMemcpy(tmaps_ + (size_t)id * 384, maps, 384, cudaMemcpyHostToDevice));
  return VP8GPU_OK;
}

int Engine::ensure_lane(int lane) {
  if (lane < 0 || lane >= kMaxLanes) return fail(VP8GPU_ERR_LOGIC, "lane out of range");
  std::lock_guard<std::mutex> lk(mu_);
  CU(cudaSetDevice(device_));
  if (!lanes_[lane]) {
    // the lanes carry the latency-critical pixel batches: highest priority, so that their thread blocks are
    // placed ahead of the long-running token kernels' (lower number = higher priority)
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    CU(cudaStreamCreateWithPriority(&lanes_[lane], cudaStreamNonBlocking, prio_hi));
    CU(cudaStreamCreateWithFlags(&lanes_[kMaxLanes + lane], cudaStreamNonBlocking));
  }
  return VP8GPU_OK;
}

// ---------------------------------------------------------------------------------------------
// frame pool
// ---------------------------------------------------------------------------------------------
int Engine::frame_alloc(int* id) {
  std::lock_guard<std::mutex> lk(mu_);
  if (free_.empty()) return fail(VP8GPU_ERR_NOMEM, "device frame pool exhausted");
  const int i = free_.back();
  Frame& f = frames_[i];
  if (!f.dev) {
    CU(cudaSetDevice(device_));
    CU(cudaMalloc(&f.dev, g_.alloc_bytes));
    // the hand-over areas must never hold a value that a later launch could take for its epoch
    if (g_.alloc_bytes > g_.msg_lf_off) CU(cudaMemset(f.dev + g_.msg_lf_off, 0, g_.alloc_bytes - g_.msg_lf_off));
    if (int rc = make_tensor_maps(i)) return rc;
  }
  free_.pop_back();
  f.refcnt = 1;
  *id = i;
  return VP8GPU_OK;
}
int Engine::frame_retain(int id) {
  std::lock_guard<std::mutex> lk(mu_);
  if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "retain: bad frame id");
  frames_[id].refcnt++;
  return VP8GPU_OK;
}
int Engine::frame_release(int id) {
  std::lock_guard<std::mutex> lk(mu_);
  if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "release: bad frame id");
  if (--frames_[id].refcnt == 0) free_.push_back(id);  // `pending` keeps guarding the memory
  return VP8GPU_OK;
}

int Engine::frames_free() {
  std::lock_guard<std::mutex> lk(mu_);
  return (int)free_.size();
}

// Stream ordering of rasters.  A raster remembers the stream slot that last WROTE it (wslot, wev)
// and the slots that READ it since (pending, ev[slot]): a reader only waits for the writer, so that
// e.g. the download of a frame does not delay the next frame's motion compensation from it; a
// writer (a recycled raster) waits for everybody.  The events are not owned by the raster: they come
// from a small ring per stream slot, and one record serves every raster a batch touched.  A ring
// entry that has been re-recorded since only makes a later waiter wait for newer work of the same
// stream (conservative, and never cyclic: waits always point at work queued earlier).
// Caller holds mu_.
cudaEvent_t Engine::next_event(int slot) {
  cudaEvent_t& ev = ring_[slot][ring_next_[slot]];
  ring_next_[slot] = (ring_next_[slot] + 1) % kEventRing;
  if (!ev && cudaEventCreateWithFlags(&ev, cudaEventDisableTiming | cudaEventBlockingSync) != cudaSuccess) return nullptr;
  return ev;
}
int Engine::touch(Frame& f, int slot, bool write, cudaEvent_t shared) {
  cudaEvent_t ev = shared;
  if (!ev) {
    ev = next_event(slot);
    if (!ev) return fail(VP8GPU_ERR_CUDA, "event creation failed");
    CU(cudaEventRecord(ev, lanes_[slot]));
  }
  if (write) {
    f.wev = ev;
    f.wslot = slot;
    f.pending = 0;  // the preceding wait ordered this stream after every reader
  } else {
    f.ev[slot] = ev;
    f.pending |= 1ull << slot;
  }
  return VP8GPU_OK;
}
void Engine::collect_waits(const Frame& f, int slot, bool write, std::vector<cudaEvent_t>& out) const {
  auto add = [&out](cudaEvent_t ev) {
    for (cudaEvent_t o : out)
      if (o == ev) return;
    out.push_back(ev);
  };
  if (f.wslot >= 0 && f.wslot != slot) add(f.wev);
  if (!write) return;
  uint64_t m = f.pending & ~(1ull << slot);
  while (m) {
    const int t = __builtin_ctzll(m);
    m &= m - 1;
    add(f.ev[t]);
  }
}
int Engine::wait_for(Frame& f, int slot, cudaStream_t s, bool write) {
  std::vector<cudaEvent_t> w;
  collect_waits(f, slot, write, w);
  for (cudaEvent_t ev : w) CU(cudaStreamWaitEvent(s, ev, 0));
  return VP8GPU_OK;
}

int Engine::frame_clear(int id, int lane) {
  if (int rc = ensure_lane(lane)) return rc;
  std::lock_guard<std::mutex> lk(mu_);
  Frame& f = frames_[id];
  if (int rc = wait_for(f, lane, lanes_[lane])) return rc;
  CU(cudaMemsetAsync(f.dev, 0, g_.frame_bytes, lanes_[lane]));
  return touch(f, lane);
}

int Engine::frame_copy(int dst, int src, int lane) {
  if (int rc = ensure_lane(lane)) return rc;
  std::lock_guard<std::mutex> lk(mu_);
  for (int id : {dst, src})
    if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "frame_copy: bad frame id");
  cudaStream_t s = lanes_[lane];
  if (int rc = wait_for(frames_[dst], lane, s, true)) return rc;
  if (int rc = wait_for(frames_[src], lane, s, false)) return rc;
  CU(cudaMemcpyAsync(frames_[dst].dev, frames_[src].dev, g_.frame_bytes, cudaMemcpyDeviceToDevice, s));
  if (int rc = touch(frames_[src], lane, false)) return rc;
  return touch(frames_[dst], lane, true);
}

int Engine::frame_copy_raw(int id, void* buf, size_t bytes, bool into_frame) {
  if (int rc = ensure_lane(0)) return rc;
  if (!buf || bytes != g_.frame_bytes) return fail(VP8GPU_ERR_LOGIC, "frame_copy_raw: size must be vp8gpu_frame_bytes");
  cudaStream_t s = lanes_[0];
  {
    std::lock_guard<std::mutex> lk(mu_);
    if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "frame_copy_raw: bad frame id");
    Frame& f = frames_[id];
    if (int rc = wait_for(f, 0, s, into_frame)) return rc;
    if (into_frame) CU(cudaMemcpyAsync(f.dev, buf, bytes, cudaMemcpyDefault, s));
    else CU(cudaMemcpyAsync(buf, f.dev, bytes, cudaMemcpyDefault, s));
    if (int rc = touch(f, 0, into_frame)) return rc;
  }
  CU(cudaStreamSynchronize(s));
  return VP8GPU_OK;
}

int Engine::frame_upload(int id, const uint8_t* y, size_t ys, const uint8_t* u, const uint8_t* v, size_t cs) {
  if (int rc = ensure_lane(0)) return rc;
  std::lock_guard<std::mutex> lk(mu_);
  if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "upload: bad frame id");
  Frame& f = frames_[id];
  cudaStream_t s = lanes_[0];
  if (int rc = wait_for(f, 0, s)) return rc;
  CU(cudaMemcpy2DAsync(f.dev, g_.y_pitch, y, ys, g_.W, g_.H, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpy2DAsync(f.dev + g_.u_off, g_.c_pitch, u, cs, g_.W / 2, g_.H / 2, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpy2DAsync(f.dev + g_.v_off, g_.c_pitch, v, cs, g_.W / 2, g_.H / 2, cudaMemcpyHostToDevice, s));
  if (int rc = touch(f, 0)) return rc;
  CU(cudaStreamSynchronize(s));
  return VP8GPU_OK;
}

int Engine::frame_download(int id, uint8_t* y, size_t ys, uint8_t* u, uint8_t* v, size_t cs) {
  if (int rc = ensure_lane(0)) return rc;
  cudaStream_t s;
  {
    std::lock_guard<std::mutex> lk(mu_);
    if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "download: bad frame id");
    Frame& f = frames_[id];
    const int slot = kMaxLanes + 0;
    s = lanes_[slot];
    if (int rc = wait_for(f, slot, s, false)) return rc;
    CU(cudaMemcpy2DAsync(y, ys, f.dev, g_.y_pitch, g_.W, g_.H, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpy2DAsync(u, cs, f.dev + g_.u_off, g_.c_pitch, g_.W / 2, g_.H / 2, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpy2DAsync(v, cs, f.dev + g_.v_off, g_.c_pitch, g_.W / 2, g_.H / 2, cudaMemcpyDeviceToHost, s));
    if (int rc = touch(f, slot, false)) return rc;
  }
  CU(cudaStreamSynchronize(s));
  return VP8GPU_OK;
}

int Engine::frames_download_display(const int* ids, uint8_t* const* dsts, int n, int lane) {
  if (n <= 0) return VP8GPU_OK;
  if (int rc = ensure_lane(lane)) return rc;
  const int cw = (width_ + 1) / 2, ch = (height_ + 1) / 2;
  const int slot = kMaxLanes + lane;
  cudaStream_t s = lanes_[slot];
  std::vector<cudaEvent_t> waits;
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (int i = 0; i < n; i++) {
      if (ids[i] < 0 || ids[i] >= (int)frames_.size() || frames_[ids[i]].refcnt <= 0)
        return fail(VP8GPU_ERR_LOGIC, "download: bad frame id");
      collect_waits(frames_[ids[i]], slot, false, waits);
    }
  }
  for (cudaEvent_t ev : waits) CU(cudaStreamWaitEvent(s, ev, 0));
  // rows are contiguous when the pitch equals the display width (e.g. 1080p): plain copies
  const bool flat = g_.y_pitch == width_ && g_.c_pitch == cw;
  for (int i = 0; i < n; i++) {
    const uint8_t* src = frames_[ids[i]].dev;
    uint8_t* p = dsts[i];
    if (flat) {
      CU(cudaMemcpyAsync(p, src, (size_t)width_ * height_, cudaMemcpyDeviceToHost, s));
      p += (size_t)width_ * height_;
      CU(cudaMemcpyAsync(p, src + g_.u_off, (size_t)cw * ch, cudaMemcpyDeviceToHost, s));
      p += (size_t)cw * ch;
      CU(cudaMemcpyAsync(p, src + g_.v_off, (size_t)cw * ch, cudaMemcpyDeviceToHost, s));
    } else {
      CU(cudaMemcpy2DAsync(p, width_, src, g_.y_pitch, width_, height_, cudaMemcpyDeviceToHost, s));
      p += (size_t)width_ * height_;
      CU(cudaMemcpy2DAsync(p, cw, src + g_.u_off, g_.c_pitch, cw, ch, cudaMemcpyDeviceToHost, s));
      p += (size_t)cw * ch;
      CU(cudaMemcpy2DAsync(p, cw, src + g_.v_off, g_.c_pitch, cw, ch, cudaMemcpyDeviceToHost, s));
    }
  }
  std::lock_guard<std::mutex> lk(mu_);
  cudaEvent_t ev = next_event(slot);
  if (!ev) return fail(VP8GPU_ERR_CUDA, "event creation failed");
  CU(cudaEventRecord(ev, s));
  for (int i = 0; i < n; i++) touch(frames_[ids[i]], slot, false, ev);
  return VP8GPU_OK;
}

int Engine::frame_download_display(int id, int lane, uint8_t* dst, size_t dst_size, bool wait) {
  const int cw = (width_ + 1) / 2, ch = (height_ + 1) / 2;
  const size_t need = (size_t)width_ * height_ + 2 * (size_t)cw * ch;
  if (dst_size < need) return fail(VP8GPU_ERR_LOGIC, "download_display: destination too small");
  if (int rc = frames_download_display(&id, &dst, 1, lane)) return rc;
  if (wait) CU(cudaStreamSynchronize(lanes_[kMaxLanes + lane]));
  return VP8GPU_OK;
}

int Engine::frames_equal(int a, int b, int lane, int* equal) {
  if (int rc = ensure_lane(lane)) return rc;
  if (a == b) {
    *equal = 1;
    return VP8GPU_OK;
  }
  int* flag;
  cudaStream_t s = lanes_[lane];
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (int id : {a, b})
      if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "compare: bad frame id");
    if (!cmp_scratch_) CU(cudaMalloc(&cmp_scratch_, 1024));
    flag = reinterpret_cast<int*>(cmp_scratch_ + 640 + 4 * lane);  // one flag per lane; the hash slots end at 64 + 8 * 64
    if (int rc = wait_for(frames_[a], lane, s, false)) return rc;
    if (int rc = wait_for(frames_[b], lane, s, false)) return rc;
    CU(cudaMemsetAsync(flag, 0, sizeof(int), s));
    if (int e = launch_compare(frames_[a].dev, frames_[b].dev, g_, flag, s)) return cuda_fail((cudaError_t)e, "compare");
    launches_++;
    if (int rc = touch(frames_[a], lane, false)) return rc;
    if (int rc = touch(frames_[b], lane, false)) return rc;
  }
  int h = 0;
  CU(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  *equal = h == 0;
  return VP8GPU_OK;
}

int Engine::frames_ssim(int a, int b, int lane, double* out) {
  if (int rc = ensure_lane(lane)) return rc;
  cudaStream_t s = lanes_[lane];
  const int n = (g_.W / 4 - 1) * (g_.H / 4 - 1);
  if (n <= 0) {
    *out = 0.0;
    return VP8GPU_OK;
  }
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (int id : {a, b})
      if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "ssim: bad frame id");
    if (!ssim_dev_[lane]) {
      CU(cudaSetDevice(device_));
      CU(cudaMalloc(&ssim_dev_[lane], (size_t)n * sizeof(float)));
      CU(cudaHostAlloc(&ssim_host_[lane], (size_t)n * sizeof(float), cudaHostAllocDefault));
    }
    if (int rc = wait_for(frames_[a], lane, s, false)) return rc;
    if (int rc = wait_for(frames_[b], lane, s, false)) return rc;
    if (int e = launch_ssim(frames_[a].dev, frames_[b].dev, g_, ssim_dev_[lane], s)) return cuda_fail((cudaError_t)e, "ssim");
    launches_++;
    if (int rc = touch(frames_[a], lane, false)) return rc;
    if (int rc = touch(frames_[b], lane, false)) return rc;
  }
  CU(cudaMemcpyAsync(ssim_host_[lane], ssim_dev_[lane], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  // x264's pixel_ssim_wxh adds the per-window values into one float in raster order (util/ssim.cc via
  // oracle/ref_shim/ssim_stub.cc); the encoder's loop-filter search compares these sums with `>`, so the
  // sum is formed the same way, on the host
  float total = 0.0f;
  const float* v = ssim_host_[lane];
  for (int i = 0; i < n; i++) total += v[i];
  *out = total / n;
  return VP8GPU_OK;
}

int Engine::frame_hash(int id, int lane, uint64_t* out) {
  if (int rc = ensure_lane(lane)) return rc;
  unsigned long long* d;
  cudaStream_t s = lanes_[lane];
  {
    std::lock_guard<std::mutex> lk(mu_);
    if (id < 0 || id >= (int)frames_.size() || frames_[id].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "hash: bad frame id");
    if (!cmp_scratch_) CU(cudaMalloc(&cmp_scratch_, 1024));
    d = reinterpret_cast<unsigned long long*>(cmp_scratch_ + 64 + 8 * lane);
    if (int rc = wait_for(frames_[id], lane, s, false)) return rc;
    CU(cudaMemsetAsync(d, 0, sizeof(unsigned long long), s));
    if (int e = launch_hash(frames_[id].dev, g_, d, s)) return cuda_fail((cudaError_t)e, "hash");
    launches_++;
    if (int rc = touch(frames_[id], lane, false)) return rc;
  }
  unsigned long long h = 0;
  CU(cudaMemcpyAsync(&h, d, sizeof(h), cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  *out = h;
  return VP8GPU_OK;
}

// ---------------------------------------------------------------------------------------------
// job submission
// ---------------------------------------------------------------------------------------------
int Engine::count_jobs(const HostJob& j, uint32_t* n_intra, uint32_t* n_inter, uint32_t* n_filtered) const {
  const size_t n = (size_t)g_.mb_cols * g_.mb_rows;
  uint32_t ni = 0, nf = 0;
  if (j.n_intra >= 0 && j.n_filtered >= 0) {
    ni = (uint32_t)j.n_intra;
    nf = (uint32_t)j.n_filtered;
  } else {
    for (size_t i = 0; i < n; i++) {
      ni += j.mbs[i].ref_frame == VP8GPU_REF_CURRENT;
      nf += j.mbs[i].lf_level != 0;
    }
  }
  *n_intra = ni;
  *n_inter = (uint32_t)n - ni;
  *n_filtered = j.desc->loop_filter_level ? nf : 0;
  return VP8GPU_OK;
}

namespace {
struct Layout {
  size_t jobs_off, sync_off, sync_bytes, total;
  std::vector<size_t> mbs_off, tok_off, split_off;
};
Layout plan(const Geom& g, const HostJob* jobs, int n) {
  Layout L;
  L.jobs_off = 0;
  L.sync_off = align_up(sizeof(DevJob) * n, 256);
  L.sync_bytes = sizeof(int) * (kSyncHeaderInts + (size_t)n * 2 * g.mb_rows);
  size_t off = align_up(L.sync_off + L.sync_bytes, 256);
  const size_t n_mbs = (size_t)g.mb_cols * g.mb_rows;
  for (int i = 0; i < n; i++) {
    if (jobs[i].ring) {  // records already in HBM
      L.mbs_off.push_back(0);
      L.tok_off.push_back(0);
      L.split_off.push_back(0);
      continue;
    }
    L.mbs_off.push_back(off);
    off = align_up(off + n_mbs * sizeof(vp8gpu_mb), 256);
    L.tok_off.push_back(off);
    off = align_up(off + (size_t)jobs[i].desc->n_tokens * sizeof(vp8gpu_token) + 4, 256);
    L.split_off.push_back(off);
    off = align_up(off + (size_t)jobs[i].desc->n_split * sizeof(vp8gpu_split_mvs) + 4, 256);
  }
  L.total = off;
  return L;
}
}  // namespace

int Engine::build_and_launch(int lane, const DevJob* d_jobs, int* d_sync, int n, bool any_inter, bool any_intra,
                             bool any_lf, cudaEvent_t* between) {
  cudaStream_t s = lanes_[lane];
  if (between) CU(cudaEventRecord(between[2], s));  // the stream has passed its waits and the record upload
  if (any_inter) {
    if (int e = launch_inter(d_jobs, n, g_, s)) return cuda_fail((cudaError_t)e, "k_inter launch");
    launches_++;
  }
  if (between) CU(cudaEventRecord(between[0], s));
  if (any_intra) {
    if (int e = launch_intra(d_jobs, n, g_, d_sync + 0, next_epoch(1), s)) return cuda_fail((cudaError_t)e, "k_intra launch");
    launches_++;
  }
  if (between) CU(cudaEventRecord(between[1], s));
  if (any_lf) {
    if (int e = launch_loopfilter(d_jobs, n, g_, d_sync + 32, next_epoch(2), lf_band(), s)) return cuda_fail((cudaError_t)e, "k_loopfilter launch");
    launches_++;
  }
  return VP8GPU_OK;
}

// ------------------------------------------------------------------------------------------
// device-side token decoding (tokens.cu)
// ------------------------------------------------------------------------------------------
uint32_t Engine::token_cap_for(size_t bits) const {
  // Every non-zero token ends with a sign decoded at probability 128, which consumes >= 0.98 bit
  // of the partition, and past the end of the data every block ends at once (only zero bits
  // arrive): tokens <= 8.2 * bytes + lookahead.  Never more than 25 * 16 per macroblock.
  const size_t by_bytes = align_up(bits + 16, 256) * 9 + 1024, by_blocks = (size_t)g_.mb_cols * g_.mb_rows * 400;
  return (uint32_t)(by_bytes < by_blocks ? by_bytes : by_blocks);
}

TokenRing Engine::token_ring_layout(size_t max_frame_bytes, bool arena) const {
  const size_t n_mbs = (size_t)g_.mb_cols * g_.mb_rows;
  TokenRing r;
  r.bits_cap = (uint32_t)align_up(max_frame_bytes + 16, 256);
  r.split_cap = (uint32_t)n_mbs;
  r.tok_cap = token_cap_for(max_frame_bytes);
  static_assert(sizeof(TokJob) <= 256, "a slot's TokJob area");
  size_t off = 256;  // TokJob
  r.probs_off = off;
  off += 1280;
  r.info_off = off;  // 2 bits per macroblock for the lock-step token decoder, one word of slack
  off = align_up(off + 4 * ((n_mbs + 15) / 16 + 1), 256);
  r.bits_off = off;
  off = align_up(off + r.bits_cap, 256);
  r.host_stride = off;
  r.result_off = off;
  r.ready_off = off + 8;  // after the two result words
  off += 256;
  r.above_off = off;
  off = align_up(off + 2 * (size_t)g_.mb_cols, 256);
  r.mbs_off = off;
  off = align_up(off + n_mbs * sizeof(vp8gpu_mb), 256);
  r.split_off = off;
  off = align_up(off + (size_t)r.split_cap * sizeof(vp8gpu_split_mvs), 256);
  r.tok_off = off;
  if (!arena) off = align_up(off + (size_t)r.tok_cap * sizeof(vp8gpu_token), 256);
  r.stride = off;
  return r;
}

int Engine::token_ring_create(int nslots, size_t max_frame_bytes, TokenRing** out, size_t arena_tokens) {
  CU(cudaSetDevice(device_));
  TokenRing* r = new TokenRing(token_ring_layout(max_frame_bytes, arena_tokens > 0));
  r->nslots = nslots;
  r->slot_tokens.assign(nslots, nullptr);
  r->slot_epoch.assign(nslots, 0);
  r->arena_cap = arena_tokens;
  if (cudaMalloc(&r->dev, r->stride * nslots) != cudaSuccess ||
      (arena_tokens && cudaMalloc(&r->arena, arena_tokens * sizeof(vp8gpu_token)) != cudaSuccess) ||
      cudaHostAlloc(&r->host, r->host_stride * nslots, cudaHostAllocDefault) != cudaSuccess ||
      cudaHostAlloc(&r->ready_host, sizeof(uint32_t) * nslots, cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer(reinterpret_cast<void**>(&r->ready_host_dev), r->ready_host, 0) != cudaSuccess) {
    token_ring_free(r);
    return fail(VP8GPU_ERR_NOMEM, "token ring allocation failed");
  }
  // result words (tokens written, overflow flag) of slots that are never used must read as "fine"; ready words hold
  // no epoch (0 is never one)
  memset(r->ready_host, 0, sizeof(uint32_t) * nslots);
  CU(cudaMemset2D(r->dev + r->result_off, r->stride, 0, 12, (size_t)nslots));
  *out = r;
  return VP8GPU_OK;
}

void Engine::token_ring_free(TokenRing* r) {
  if (!r) return;
  cudaSetDevice(device_);
  if (r->dev) cudaFree(r->dev);
  if (r->arena) cudaFree(r->arena);
  if (r->host) cudaFreeHost(r->host);
  if (r->ready_host) cudaFreeHost(r->ready_host);
  delete r;
}

int Engine::token_ring_stage(TokenRing* r, int slot, const ParsedFrame& f, cudaStream_t s, vp8gpu_token* tokens,
                             unsigned long long* stamp) {
  const TokenWork& tw = f.tw;
  if (!tw.deferred) return fail(VP8GPU_ERR_LOGIC, "token_ring_stage: frame was not parsed with defer_tokens");
  if (tw.bits_len > r->bits_cap || f.desc.n_split > r->split_cap)
    return fail(VP8GPU_ERR_NOMEM, "token_ring_stage: frame larger than the ring was sized for");
  if ((r->arena != nullptr) != (tokens != nullptr)) return fail(VP8GPU_ERR_LOGIC, "token_ring_stage: token area");
  uint8_t* h = r->host_slot(slot);
  uint8_t* d = r->dev_slot(slot);
  TokJob* j = reinterpret_cast<TokJob*>(h);
  j->mbs = reinterpret_cast<vp8gpu_mb*>(d + r->mbs_off);
  j->tokens = tokens ? tokens : reinterpret_cast<vp8gpu_token*>(d + r->tok_off);
  r->slot_tokens[slot] = j->tokens;
  j->bits = d + r->bits_off;
  j->coef_probs = d + r->probs_off;
  j->result = reinterpret_cast<uint32_t*>(d + r->result_off);
  j->above = reinterpret_cast<uint16_t*>(d + r->above_off);
  j->mbinfo = reinterpret_cast<const uint32_t*>(d + r->info_off);
  memcpy(j->part_off, tw.part_off, sizeof(j->part_off));
  memcpy(j->part_len, tw.part_len, sizeof(j->part_len));
  j->nparts = tw.nparts;
  j->tok_cap = tokens ? token_cap_for(tw.bits_len) : r->tok_cap;
  j->ready = reinterpret_cast<uint32_t*>(d + r->ready_off);
  j->ready_host = r->ready_host_dev + slot;
  j->epoch = r->slot_epoch[slot] = fresh_epoch();
  j->stamp = stamp;
  memcpy(h + r->probs_off, tw.coef_probs, 1056);
  memcpy(h + r->bits_off, tw.bits, tw.bits_len);
  const size_t n_mbs = (size_t)g_.mb_cols * g_.mb_rows;
  {
    uint32_t* info = reinterpret_cast<uint32_t*>(h + r->info_off);
    const vp8gpu_mb* m = f.mbs.data();
    for (size_t w = 0; w < (n_mbs + 15) / 16; w++) {
      uint32_t v = 0;
      const size_t n = n_mbs - 16 * w < 16 ? n_mbs - 16 * w : 16;
      for (size_t k = 0; k < n; k++) v |= (uint32_t)(m[16 * w + k].flags & 3u) << (2 * k);
      info[w] = v;
    }
  }
  CU(cudaMemcpyAsync(d, h, r->bits_off + align_up(tw.bits_len, 16), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(d + r->mbs_off, f.mbs.data(), n_mbs * sizeof(vp8gpu_mb), cudaMemcpyHostToDevice, s));
  if (f.desc.n_split)
    CU(cudaMemcpyAsync(d + r->split_off, f.split.data(), (size_t)f.desc.n_split * sizeof(vp8gpu_split_mvs),
                       cudaMemcpyHostToDevice, s));
  return VP8GPU_OK;
}

int Engine::token_ring_launch(TokenRing* r, int first, int count, cudaStream_t s) {
  if (count <= 0) return VP8GPU_OK;
  if (int e = launch_tokens(r->dev, r->stride, first, count, r->nslots, g_, s)) return cuda_fail((cudaError_t)e, "k_tokens launch");
  launches_++;
  return VP8GPU_OK;
}

int Engine::token_ring_clear_result(TokenRing* r, int slot, cudaStream_t s) {
  CU(cudaMemsetAsync(r->dev_slot(slot) + r->result_off, 0, 8, s));
  return VP8GPU_OK;
}

int Engine::token_ring_result(TokenRing* r, int slot, cudaStream_t s, uint32_t result[2]) {
  CU(cudaMemcpyAsync(result, r->dev_slot(slot) + r->result_off, 8, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return VP8GPU_OK;
}

int Engine::submit(int lane, const HostJob* jobs, int n, cudaEvent_t consumed, cudaEvent_t* between) {
  if (n <= 0) return VP8GPU_OK;
  if (int rc = ensure_lane(lane)) return rc;
  CU(cudaSetDevice(device_));
  cudaStream_t s = lanes_[lane];
  const Layout L = plan(g_, jobs, n);
  Staging& st = staging_[lane][staging_next_[lane]];
  staging_next_[lane] = (staging_next_[lane] + 1) % kStagingDepth;
  if (st.in_flight) {
    CU(cudaEventSynchronize(st.done));
    st.in_flight = false;
  }
  if (!st.done) CU(cudaEventCreateWithFlags(&st.done, cudaEventDisableTiming | cudaEventBlockingSync));
  const size_t hdr_bytes = align_up(L.sync_off + L.sync_bytes, 256);
  if (st.host_cap < hdr_bytes) {
    if (st.host) CU(cudaFreeHost(st.host));
    st.host_cap = hdr_bytes * 2;
    CU(cudaHostAlloc(&st.host, st.host_cap, cudaHostAllocMapped));
    CU(cudaHostGetDevicePointer(reinterpret_cast<void**>(&st.host_dev), st.host, 0));
  }
  if (st.dev_cap < L.total) {
    if (st.dev) CU(cudaFree(st.dev));
    st.dev_cap = L.total + L.total / 2;
    CU(cudaMalloc(&st.dev, st.dev_cap));
  }
  // header: device-side job descriptors + zeroed tickets / progress counters
  memset(st.host, 0, hdr_bytes);
  DevJob* hj = reinterpret_cast<DevJob*>(st.host);
  int* d_sync = reinterpret_cast<int*>(st.dev + L.sync_off);
  bool any_inter = false, any_intra = false, any_lf = false;
  std::vector<cudaEvent_t> waits;
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (int i = 0; i < n; i++) {
      const HostJob& j = jobs[i];
      if (j.out < 0 || j.out >= (int)frames_.size() || frames_[j.out].refcnt <= 0)
        return fail(VP8GPU_ERR_LOGIC, "submit: bad output frame");
      DevJob& d = hj[i];
      if (j.ring) {
        const uint8_t* slot = j.ring->dev_slot(j.ring_slot);
        d.mbs = reinterpret_cast<const vp8gpu_mb*>(slot + j.ring->mbs_off);
        d.tokens = j.ring->slot_tokens[j.ring_slot];
        d.split = reinterpret_cast<const vp8gpu_split_mvs*>(slot + j.ring->split_off);
        d.ready = j.ring->dev_ready_word(j.ring_slot);
        d.ready_epoch = j.ring->slot_epoch[j.ring_slot];
      } else {
        d.mbs = reinterpret_cast<const vp8gpu_mb*>(st.dev + L.mbs_off[i]);
        d.tokens = reinterpret_cast<const vp8gpu_token*>(st.dev + L.tok_off[i]);
        d.split = reinterpret_cast<const vp8gpu_split_mvs*>(st.dev + L.split_off[i]);
      }
      d.out = frames_[j.out].dev;
      for (int r = 0; r < 3; r++) {
        d.ref[r] = nullptr;
        d.ref_tmap[r] = nullptr;
        if (!j.desc->key_frame) {
          if (j.refs[r] < 0 || j.refs[r] >= (int)frames_.size() || frames_[j.refs[r]].refcnt <= 0)
            return fail(VP8GPU_ERR_LOGIC, "submit: bad reference frame");
          d.ref[r] = frames_[j.refs[r]].dev;
          d.ref_tmap[r] = frame_tmaps(j.refs[r]);
        }
      }
      d.intra_progress = d_sync + kSyncHeaderInts + (size_t)(2 * i) * g_.mb_rows;
      d.lf_progress = d_sync + kSyncHeaderInts + (size_t)(2 * i + 1) * g_.mb_rows;
      memcpy(d.quant, j.desc->quant, sizeof(d.quant));
      d.key_frame = j.desc->key_frame;
      d.sharpness = j.desc->sharpness;
      uint32_t n_filtered;
      count_jobs(j, &d.n_intra, &d.n_inter, &n_filtered);
      d.lf_enabled = n_filtered != 0;
      any_inter |= d.n_inter != 0;
      any_intra |= d.n_intra != 0;
      any_lf |= d.lf_enabled != 0;
    }
    // stream ordering against other users of the rasters: most frames of a batch were last touched
    // by the same earlier batch, i.e. share one event
    for (int i = 0; i < n; i++) {
      collect_waits(frames_[jobs[i].out], lane, true, waits);
      if (!jobs[i].desc->key_frame)
        for (int r = 0; r < 3; r++) collect_waits(frames_[jobs[i].refs[r]], lane, false, waits);
    }
  }
  for (cudaEvent_t ev : waits) CU(cudaStreamWaitEvent(s, ev, 0));
  if (int ce = launch_fetch_header(st.dev, st.host_dev, hdr_bytes, s)) return cuda_fail((cudaError_t)ce, "header fetch");
  launches_++;
  const size_t n_mbs = (size_t)g_.mb_cols * g_.mb_rows;
  for (int i = 0; i < n; i++) {
    const HostJob& j = jobs[i];
    if (j.ring) continue;
    CU(cudaMemcpyAsync(st.dev + L.mbs_off[i], j.mbs, n_mbs * sizeof(vp8gpu_mb), cudaMemcpyHostToDevice, s));
    if (j.desc->n_tokens)
      CU(cudaMemcpyAsync(st.dev + L.tok_off[i], j.tokens, (size_t)j.desc->n_tokens * sizeof(vp8gpu_token),
                         cudaMemcpyHostToDevice, s));
    if (j.desc->n_split)
      CU(cudaMemcpyAsync(st.dev + L.split_off[i], j.split, (size_t)j.desc->n_split * sizeof(vp8gpu_split_mvs),
                         cudaMemcpyHostToDevice, s));
    if (j.consumed) CU(cudaEventRecord(j.consumed, s));
  }
  if (consumed) CU(cudaEventRecord(consumed, s));
  if (int rc = build_and_launch(lane, reinterpret_cast<const DevJob*>(st.dev), d_sync, n, any_inter, any_intra, any_lf, between))
    return rc;
  {
    std::lock_guard<std::mutex> lk(mu_);
    cudaEvent_t ev = next_event(lane);  // one record for every raster of the batch
    if (!ev) return fail(VP8GPU_ERR_CUDA, "event creation failed");
    CU(cudaEventRecord(ev, s));
    for (int i = 0; i < n; i++) {
      touch(frames_[jobs[i].out], lane, true, ev);
      if (!jobs[i].desc->key_frame)
        for (int r = 0; r < 3; r++) touch(frames_[jobs[i].refs[r]], lane, false, ev);
      if (jobs[i].finished) *jobs[i].finished = ev;
    }
  }
  CU(cudaEventRecord(st.done, s));
  st.in_flight = true;
  return VP8GPU_OK;
}

// ---------------------------------------------------------------------------------------------
// device-resident batches (bench / profiling): records stay in HBM, kernels can be re-run
// ---------------------------------------------------------------------------------------------
struct Engine::Resident {
  uint8_t* dev = nullptr;
  size_t sync_off = 0, sync_bytes = 0;
  int n = 0;
  bool any_inter = false, any_intra = false, any_lf = false;
  std::vector<int> outs, refs;
  cudaEvent_t t0 = nullptr, t1 = nullptr;
};

int Engine::resident_upload(const HostJob* jobs, int n, Resident** out) {
  if (n <= 0) return fail(VP8GPU_ERR_LOGIC, "empty batch");
  if (int rc = ensure_lane(0)) return rc;
  CU(cudaSetDevice(device_));
  const Layout L = plan(g_, jobs, n);
  Resident* r = new Resident();
  r->n = n;
  r->sync_off = L.sync_off;
  r->sync_bytes = L.sync_bytes;
  cudaError_t e = cudaMalloc(&r->dev, L.total);
  if (e != cudaSuccess) {
    delete r;
    return cuda_fail(e, "cudaMalloc(resident batch)");
  }
  std::vector<uint8_t> hdr(align_up(L.sync_off + L.sync_bytes, 256), 0);
  DevJob* hj = reinterpret_cast<DevJob*>(hdr.data());
  int* d_sync = reinterpret_cast<int*>(r->dev + L.sync_off);
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (int i = 0; i < n; i++) {
      const HostJob& j = jobs[i];
      DevJob& d = hj[i];
      d.mbs = reinterpret_cast<const vp8gpu_mb*>(r->dev + L.mbs_off[i]);
      d.tokens = reinterpret_cast<const vp8gpu_token*>(r->dev + L.tok_off[i]);
      d.split = reinterpret_cast<const vp8gpu_split_mvs*>(r->dev + L.split_off[i]);
      if (j.out < 0 || j.out >= (int)frames_.size() || frames_[j.out].refcnt <= 0) {
        cudaFree(r->dev);
        delete r;
        return fail(VP8GPU_ERR_LOGIC, "resident: bad output frame");
      }
      d.out = frames_[j.out].dev;
      r->outs.push_back(j.out);
      for (int k = 0; k < 3; k++) {
        d.ref[k] = nullptr;
        d.ref_tmap[k] = nullptr;
        if (!j.desc->key_frame) {
          if (j.refs[k] < 0 || j.refs[k] >= (int)frames_.size() || frames_[j.refs[k]].refcnt <= 0) {
            cudaFree(r->dev);
            delete r;
            return fail(VP8GPU_ERR_LOGIC, "resident: bad reference frame");
          }
          d.ref[k] = frames_[j.refs[k]].dev;
          d.ref_tmap[k] = frame_tmaps(j.refs[k]);
          r->refs.push_back(j.refs[k]);
        }
      }
      d.intra_progress = d_sync + kSyncHeaderInts + (size_t)(2 * i) * g_.mb_rows;
      d.lf_progress = d_sync + kSyncHeaderInts + (size_t)(2 * i + 1) * g_.mb_rows;
      memcpy(d.quant, j.desc->quant, sizeof(d.quant));
      d.key_frame = j.desc->key_frame;
      d.sharpness = j.desc->sharpness;
      uint32_t n_filtered;
      count_jobs(j, &d.n_intra, &d.n_inter, &n_filtered);
      d.lf_enabled = n_filtered != 0;
      r->any_inter |= d.n_inter != 0;
      r->any_intra |= d.n_intra != 0;
      r->any_lf |= d.lf_enabled != 0;
    }
  }
  const size_t n_mbs = (size_t)g_.mb_cols * g_.mb_rows;
  CU(cudaMemcpy(r->dev, hdr.data(), hdr.size(), cudaMemcpyHostToDevice));
  for (int i = 0; i < n; i++) {
    CU(cudaMemcpy(r->dev + L.mbs_off[i], jobs[i].mbs, n_mbs * sizeof(vp8gpu_mb), cudaMemcpyHostToDevice));
    if (jobs[i].desc->n_tokens)
      CU(cudaMemcpy(r->dev + L.tok_off[i], jobs[i].tokens, (size_t)jobs[i].desc->n_tokens * 4, cudaMemcpyHostToDevice));
    if (jobs[i].desc->n_split)
      CU(cudaMemcpy(r->dev + L.split_off[i], jobs[i].split, (size_t)jobs[i].desc->n_split * 64, cudaMemcpyHostToDevice));
  }
  CU(cudaEventCreate(&r->t0));
  CU(cudaEventCreate(&r->t1));
  *out = r;
  return VP8GPU_OK;
}

int Engine::resident_run(int lane, Resident* r, float* ms) {
  if (int rc = ensure_lane(lane)) return rc;
  CU(cudaSetDevice(device_));
  cudaStream_t s = lanes_[lane];
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (int id : r->outs) {
      if (int rc = wait_for(frames_[id], lane, s)) return rc;
    }
    for (int id : r->refs)
      if (int rc = wait_for(frames_[id], lane, s)) return rc;
  }
  CU(cudaMemsetAsync(r->dev + r->sync_off, 0, r->sync_bytes, s));
  if (ms) CU(cudaEventRecord(r->t0, s));
  if (int rc = build_and_launch(lane, reinterpret_cast<const DevJob*>(r->dev), reinterpret_cast<int*>(r->dev + r->sync_off),
                                r->n, r->any_inter, r->any_intra, r->any_lf))
    return rc;
  if (ms) CU(cudaEventRecord(r->t1, s));
  {
    std::lock_guard<std::mutex> lk(mu_);
    cudaEvent_t ev = next_event(lane);
    if (!ev) return fail(VP8GPU_ERR_CUDA, "event creation failed");
    CU(cudaEventRecord(ev, s));
    for (int id : r->refs) touch(frames_[id], lane, false, ev);
    for (int id : r->outs) touch(frames_[id], lane, true, ev);
  }
  if (ms) {
    CU(cudaEventSynchronize(r->t1));
    CU(cudaEventElapsedTime(ms, r->t0, r->t1));
  }
  return VP8GPU_OK;
}

int Engine::resident_run_many(int lane, Resident* const* rs, int n, float* total_ms) {
  if (n <= 0) return VP8GPU_OK;
  if (int rc = ensure_lane(lane)) return rc;
  cudaStream_t s = lanes_[lane];
  if (total_ms) CU(cudaEventRecord(rs[0]->t0, s));
  for (int i = 0; i < n; i++)
    if (int rc = resident_run(lane, rs[i], nullptr)) return rc;
  if (total_ms) {
    CU(cudaEventRecord(rs[0]->t1, s));
    CU(cudaEventSynchronize(rs[0]->t1));
    CU(cudaEventElapsedTime(total_ms, rs[0]->t0, rs[0]->t1));
  }
  return VP8GPU_OK;
}

int Engine::resident_run_timed(int lane, Resident* r, float ms[3]) {
  if (int rc = ensure_lane(lane)) return rc;
  CU(cudaSetDevice(device_));
  cudaStream_t s = lanes_[lane];
  cudaEvent_t mid[3];
  for (cudaEvent_t& m : mid) CU(cudaEventCreate(&m));
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (int id : r->outs)
      if (int rc = wait_for(frames_[id], lane, s)) return rc;
    for (int id : r->refs)
      if (int rc = wait_for(frames_[id], lane, s)) return rc;
  }
  CU(cudaMemsetAsync(r->dev + r->sync_off, 0, r->sync_bytes, s));
  CU(cudaEventRecord(r->t0, s));
  if (int rc = build_and_launch(lane, reinterpret_cast<const DevJob*>(r->dev), reinterpret_cast<int*>(r->dev + r->sync_off),
                                r->n, r->any_inter, r->any_intra, r->any_lf, mid))
    return rc;
  CU(cudaEventRecord(r->t1, s));
  {
    std::lock_guard<std::mutex> lk(mu_);
    cudaEvent_t ev = next_event(lane);
    if (!ev) return fail(VP8GPU_ERR_CUDA, "event creation failed");
    CU(cudaEventRecord(ev, s));
    for (int id : r->refs) touch(frames_[id], lane, false, ev);
    for (int id : r->outs) touch(frames_[id], lane, true, ev);
  }
  CU(cudaEventSynchronize(r->t1));
  CU(cudaEventElapsedTime(&ms[0], r->t0, mid[0]));
  CU(cudaEventElapsedTime(&ms[1], mid[0], mid[1]));
  CU(cudaEventElapsedTime(&ms[2], mid[1], r->t1));
  cudaEventDestroy(mid[0]);
  cudaEventDestroy(mid[1]);
  cudaEventDestroy(mid[2]);
  return VP8GPU_OK;
}

void Engine::resident_free(Resident* r) {
  if (!r) return;
  cudaSetDevice(device_);
  cudaDeviceSynchronize();
  if (r->dev) cudaFree(r->dev);
  if (r->t0) cudaEventDestroy(r->t0);
  if (r->t1) cudaEventDestroy(r->t1);
  delete r;
}

int Engine::acquire_frames(int lane, const int* ids, int n, uint32_t write_mask) {
  if (int rc = ensure_lane(lane)) return rc;
  std::lock_guard<std::mutex> lk(mu_);
  for (int i = 0; i < n; i++) {
    if (ids[i] < 0 || ids[i] >= (int)frames_.size() || frames_[ids[i]].refcnt <= 0) return fail(VP8GPU_ERR_LOGIC, "bad frame id");
    if (int rc = wait_for(frames_[ids[i]], lane, lanes_[lane], (write_mask >> i) & 1)) return rc;
  }
  return VP8GPU_OK;
}
int Engine::mark_frames(int lane, const int* ids, int n, uint32_t write_mask) {
  std::lock_guard<std::mutex> lk(mu_);
  for (int i = 0; i < n; i++)
    if (int rc = touch(frames_[ids[i]], lane, (write_mask >> i) & 1)) return rc;
  return VP8GPU_OK;
}

int Engine::sync_all() {
  CU(cudaSetDevice(device_));
  CU(cudaDeviceSynchronize());
  return VP8GPU_OK;
}
int Engine::sync_lane(int lane) {
  if (int rc = ensure_lane(lane)) return rc;
  CU(cudaStreamSynchronize(lanes_[lane]));
  CU(cudaStreamSynchronize(lanes_[kMaxLanes + lane]));
  return VP8GPU_OK;
}

}  // namespace vp8
