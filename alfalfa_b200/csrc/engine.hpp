// engine.hpp -- host orchestration of the device side: frame pool (RasterHandle semantics),
// per-lane CUDA streams, staging of parsed records, kernel launches.  Internal header.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "engine.h"
#include "parser.h"

namespace vp8 {

constexpr int kMaxLanes = 32;       // compute lanes; lane i's copy stream is slot kMaxLanes + i
constexpr int kStagingDepth = 3;    // device record buffers in flight per lane

// Device + pinned staging for frames whose DCT partitions are decoded on the device (tokens.cu):
// `nslots` slots of equal size in one allocation, so that consecutive slots can share one launch.
// Device slot: TokJob | probabilities | partitions | result words | mbs | split MVs | tokens.  A ring created with a
// token arena has no token part in its slots: the caller hands every staged frame a piece of the arena sized for that
// frame's partitions (token_cap_for), so the slots cost what a typical frame needs, not what the largest one does.
struct TokenRing {
  int nslots = 0;
  uint8_t* dev = nullptr;
  uint8_t* host = nullptr;       // pinned mirror of the first three parts of every slot
  size_t stride = 0, host_stride = 0;
  size_t probs_off = 0, info_off = 0, bits_off = 0, result_off = 0, above_off = 0, mbs_off = 0, split_off = 0, tok_off = 0;
  uint32_t bits_cap = 0, split_cap = 0, tok_cap = 0;  // tok_cap: tokens of a frame of bits_cap partition bytes
  vp8gpu_token* arena = nullptr;  // tokens of the slots when not in the slots themselves
  size_t arena_cap = 0;           // in tokens
  std::vector<vp8gpu_token*> slot_tokens;  // where the tokens of each slot's current frame go
  uint8_t* dev_slot(int i) const { return dev + (size_t)i * stride; }
  uint8_t* host_slot(int i) const { return host + (size_t)i * host_stride; }
};

// a decode job with host-side record arrays
struct HostJob {
  const vp8gpu_frame_desc* desc;
  const vp8gpu_mb* mbs;
  const vp8gpu_token* tokens;
  const vp8gpu_split_mvs* split;
  int refs[3];
  int out;
  int n_intra = -1;    // -1: count them here
  int n_filtered = -1;
  cudaEvent_t consumed = nullptr;  // recorded as soon as this job's host arrays have been copied
  // records already in HBM (token_ring_stage + token_ring_launch): nothing is copied, the stream
  // waits for `ready` instead; `finished` (optional) is recorded after the job's kernels
  const TokenRing* ring = nullptr;
  int ring_slot = 0;
  cudaEvent_t ready = nullptr;
  cudaEvent_t* finished = nullptr;  // out: an event (owned by the engine) that fires after the job's kernels
};

class Engine {
 public:
  static int create(int device, int width, int height, int max_frames, Engine** out, std::string* err);
  ~Engine();

  const Geom& geom() const { return g_; }
  int width() const { return width_; }
  int height() const { return height_; }
  int device() const { return device_; }

  // frame pool
  int frame_alloc(int* id);
  int frame_retain(int id);
  int frame_release(int id);
  int frames_free();  // rasters the pool can still hand out
  int frames_in_use() {
    std::lock_guard<std::mutex> lk(mu_);
    int n = 0;
    for (const Frame& f : frames_) n += f.refcnt > 0;
    return n;
  }
  // marks the hand-over messages of one wavefront launch; never 0, never repeats within 2^32 launches
  uint32_t next_epoch(int kernel_bit = 3) {
    if (!(ll_mask_ & kernel_bit)) return 0;
    uint32_t e = ++epoch_;
    if (e == 0) e = ++epoch_;
    return e;
  }
  int frame_upload(int id, const uint8_t* y, size_t ys, const uint8_t* u, const uint8_t* v, size_t cs);
  int frame_download(int id, uint8_t* y, size_t ys, uint8_t* u, uint8_t* v, size_t cs);
  int frame_download_display(int id, int lane, uint8_t* dst, size_t dst_size, bool wait);
  // asynchronous display-rectangle downloads of n rasters on lane's copy stream (one stream wait and
  // one event for the whole batch); every dst holds width*height*3/2-ish bytes like the call above
  int frames_download_display(const int* ids, uint8_t* const* dsts, int n, int lane);
  int frame_clear(int id, int lane);  // all-zero raster (initial References)
  int frame_copy(int dst, int src, int lane);  // VP8Raster::copy_from, asynchronous on the lane
  // whole raster <-> a host or device buffer of geom().frame_bytes bytes (synchronous)
  int frame_copy_raw(int id, void* buf, size_t bytes, bool into_frame);
  int frames_equal(int a, int b, int lane, int* equal);
  int frame_hash(int id, int lane, uint64_t* out);
  int frames_ssim(int a, int b, int lane, double* out);  // BaseRaster::quality: luma SSIM, synchronous

  // decode n frames in one set of launches on `lane`; host arrays must stay valid until the
  // returned event (*consumed, optional) has fired (pinned) or are consumed on return (pageable)
  // `between` (optional, diagnostics): three events: [0] after k_inter, [1] after k_intra, [2] before k_inter
  int submit(int lane, const HostJob* jobs, int n, cudaEvent_t consumed, cudaEvent_t* between = nullptr);

  // device-side token decoding
  // offsets and capacities only; arena: no token part in the slots
  TokenRing token_ring_layout(size_t max_frame_bytes, bool arena = false) const;
  // the most tokens k_tokens can write for partitions of `bits` bytes (the capacity rule of token_ring_layout)
  uint32_t token_cap_for(size_t bits) const;
  // arena_tokens > 0: the slots' tokens go to a separate arena of that many tokens (see TokenRing)
  int token_ring_create(int nslots, size_t max_frame_bytes, TokenRing** out, size_t arena_tokens = 0);
  void token_ring_free(TokenRing* r);
  // queue on `s` the upload of one frame parsed with defer_tokens (records + partitions); a ring with an arena
  // takes the frame's token area (`tokens`, token_cap_for(f.tw.bits_len) tokens) from the caller
  int token_ring_stage(TokenRing* r, int slot, const ParsedFrame& f, cudaStream_t s, vp8gpu_token* tokens = nullptr);
  // one k_tokens launch over `count` consecutive slots (wrapping around the ring)
  int token_ring_launch(TokenRing* r, int first, int count, cudaStream_t s);
  // queue on `s` the reset of a slot's result words; k_tokens only ever sets the overflow flag, so it stays set for
  // all the frames staged in the slot until this runs (token_ring_create starts every slot clear)
  int token_ring_clear_result(TokenRing* r, int slot, cudaStream_t s);
  // synchronous: tokens written / overflow flag of a slot whose kernel has been queued on `s`
  int token_ring_result(TokenRing* r, int slot, cudaStream_t s, uint32_t result[2]);

  // device-resident batches
  struct Resident;
  int resident_upload(const HostJob* jobs, int n, Resident** out);
  int resident_run(int lane, Resident* r, float* ms);
  int resident_run_many(int lane, Resident* const* rs, int n, float* total_ms);
  int resident_run_timed(int lane, Resident* r, float ms[3]);
  void resident_free(Resident* r);

  // for other device-side users of rasters (the encoder): raw pointer + stream-ordering hooks
  uint8_t* frame_dev(int id) { return frames_[id].dev; }
  // the raster's TMA tensor maps (Y, U, V; 128 bytes each) in device memory, for kernels that stage windows by TMA
  const void* frame_tmaps(int id) const { return tmaps_ ? tmaps_ + (size_t)id * 384 : nullptr; }
  // bit i of write_mask: ids[i] is written (waits for / excludes every other user); otherwise only read
  int acquire_frames(int lane, const int* ids, int n, uint32_t write_mask = ~0u);  // stream `lane` waits for other users
  int mark_frames(int lane, const int* ids, int n, uint32_t write_mask = ~0u);     // record that `lane` used them
  void count_launches(int n) { launches_ += n; }

  int ensure_lane(int lane);  // creates the lane's streams on first use
  int sync_all();
  int sync_lane(int lane);
  cudaStream_t stream(int lane) const { return lanes_[lane]; }
  uint64_t launches() const { return launches_.load(); }
  const char* last_error() const { return err_.c_str(); }
  int fail(int code, const std::string& what);
  int cuda_fail(cudaError_t e, const char* what);
  // the message of the calling thread's last fail / cuda_fail (of any Engine): work spread over host threads tells its
  // own failures apart from the other threads' (last_error is the context's, whichever thread wrote it last)
  static std::string& thread_error();

 private:
  Engine() = default;
  struct Frame {
    uint8_t* dev = nullptr;
    int refcnt = 0;
    uint64_t pending = 0;                  // stream slots that read it since the last write
    cudaEvent_t ev[2 * kMaxLanes] = {};    // per reading slot: the event recorded after the read (not owned)
    int wslot = -1;                        // slot of the last writer
    cudaEvent_t wev = nullptr;             // recorded after the write (not owned)
  };
  struct Staging {
    uint8_t* dev = nullptr;
    size_t dev_cap = 0;
    uint8_t* host = nullptr;  // pinned, device-mapped header: DevJob[n] + sync words
    uint8_t* host_dev = nullptr;  // the device's address of `host`
    size_t host_cap = 0;
    cudaEvent_t done = nullptr;
    bool in_flight = false;
  };
  static constexpr int kEventRing = 2048;  // must exceed the number of batches a raster outlives on any one stream slot: a re-recorded
                                            // entry makes a later waiter wait for NEWER work of that slot (false dependency, not an error)
  cudaEvent_t next_event(int slot);  // next event of the slot's ring (caller records it)
  // note that `slot` used the frame; `shared` = an event of that slot the caller has already recorded
  int touch(Frame& f, int slot, bool write = true, cudaEvent_t shared = nullptr);
  void collect_waits(const Frame& f, int slot, bool write, std::vector<cudaEvent_t>& out) const;
  int wait_for(Frame& f, int slot, cudaStream_t s, bool write = true);  // make stream s wait for other users
  int build_and_launch(int lane, const DevJob* d_jobs, int* d_sync, int n, bool any_inter, bool any_intra,
                       bool any_lf, cudaEvent_t* between = nullptr);
  int count_jobs(const HostJob& j, uint32_t* n_intra, uint32_t* n_inter, uint32_t* n_filtered) const;

  int device_ = 0, width_ = 0, height_ = 0;
  Geom g_{};
  std::mutex mu_;
  std::vector<Frame> frames_;
  std::vector<int> free_;
  cudaStream_t lanes_[2 * kMaxLanes] = {};
  cudaEvent_t ring_[2 * kMaxLanes][kEventRing] = {};
  int ring_next_[2 * kMaxLanes] = {};
  Staging staging_[kMaxLanes][kStagingDepth];
  int staging_next_[kMaxLanes] = {};
  uint8_t* cmp_scratch_ = nullptr;
  float* ssim_dev_[kMaxLanes] = {};   // per lane: one float per 8x8 SSIM window (frames_ssim)
  float* ssim_host_[kMaxLanes] = {};
  uint8_t* tmaps_ = nullptr;  // [max_frames][3] CUtensorMap, written when a raster's memory is first allocated
  int make_tensor_maps(int id);
  std::atomic<uint64_t> launches_{0};
  std::string err_;
  std::mutex err_mu_;
  std::atomic<uint32_t> epoch_{0};
  // which wavefront kernels use hand-over messages (bit 0 intra prediction, bit 1 loop filter); the others run
  // the round-1 kernels (progress counters).  VP8GPU_WAVEFRONT = legacy | ll | intra-ll | lf-ll for A/B runs.
  int ll_mask_ = 1;
};

}  // namespace vp8
