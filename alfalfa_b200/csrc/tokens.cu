// tokens.cu -- device-side coefficient-token decoder (the DCT partitions of a VP8 frame).
//
// Replaces, for throughput-oriented callers (vp8gpu_decode_ivf), the token half of the CPU front
// end: Frame::parse_tokens -> Macroblock::parse_tokens -> Block::parse_tokens (decoder/frame.cc:
// 122-137, macroblock.cc:468-502, tokens.cc:50-135) over BoolDecoder (bool_decoder.hh:82-107).
// The arithmetic code of one partition is inherently serial, and a macroblock row needs the
// "has non-zero" context of the row above, so ONE thread walks one frame in raster order; the
// parallelism is across frames: token partitions do not depend on pixels, so the host parses the
// first partitions of many frames (cheap: ~12 % of the bytes) and launches this kernel over all of
// them while the pixel kernels work on earlier frames.  One warp per frame: lane 0 decodes, the
// other lanes only help to stage the probability table.
//
// In:  vp8gpu_mb records written by the host with y_mode and VP8GPU_MB_SKIP (mb_skip_coeff) set,
//      the frame's coefficient probabilities (after the header's updates), the raw partitions.
// Out: the same token stream the CPU front end emits (csrc/parser.cc parse_block) and, per
//      record, tok_off / tok_cnt; VP8GPU_MB_SKIP is cleared, so the records end up byte-identical
//      to the ones the CPU path produces.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "engine.h"
#include "tokens_core.cuh"

namespace vp8 {
namespace {

constexpr int kMaxCols = 1024;  // 16383 px / 16

// The frame's records, tokens and result words are written (by this thread): publish its epoch.  The release at gpu
// scope orders those writes before the device word, which the pixel kernels acquire (kernels.cu acquire_job); the
// system-scope fence orders the device word before the host word, so that a host that has seen the host word
// launches pixel kernels that find the device word set.
__device__ __forceinline__ void publish_ready(const TokJob& J) {
#ifndef VP8GPU_SIMT_EMUL
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(J.ready), "r"(J.epoch) : "memory");
  asm volatile("fence.acq_rel.sys;" ::: "memory");
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(J.ready_host), "r"(J.epoch) : "memory");
  if (J.stamp) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    *J.stamp = t;
  }
#else
  __atomic_store_n(J.ready, J.epoch, __ATOMIC_RELEASE);
  __atomic_store_n(J.ready_host, J.epoch, __ATOMIC_RELEASE);
  if (J.stamp) *J.stamp = 1;
#endif
}
// jobs live at the start of equally spaced slots of a ring (engine.hpp TokenRing); one warp per frame,
// kTokWarps frames per CTA (measured: one-warp CTAs spread over the SMs best; VP8GPU_TOK_WARPS=8 packs them)
template <int kTokWarps>
__global__ void __launch_bounds__(32 * kTokWarps) k_tokens(const uint8_t* ring, size_t stride, int first, int count,
                                                          int nslots, Geom g) {
  __shared__ __align__(16) uint8_t probs_all[kTokWarps][tok::kProbBytes];
  __shared__ uint16_t above_all[kTokWarps][kMaxCols];
  const int warp = kTokWarps == 1 ? 0 : threadIdx.x >> 5, lane = threadIdx.x & 31;  // a constant table address for one warp
  const int job = blockIdx.x * kTokWarps + warp;
  if (job >= count) return;
  uint8_t* probs = probs_all[warp];
  uint16_t* above_nz = above_all[warp];
  const TokJob& J = *reinterpret_cast<const TokJob*>(ring + static_cast<size_t>((first + job) % nslots) * stride);
  for (int e = lane; e < tok::kProbEntries; e += 32) tok::expand_prob_entry(J.coef_probs, probs, e);
  for (int i = lane; i < g.mb_cols; i += 32) above_nz[i] = 0;
  __syncwarp();
  if (lane != 0) return;
  tok::decode_frame_tokens(J, g, probs, above_nz);
  publish_ready(J);
}

// lock-step variant: one LANE per frame, 32 frames per warp (tokens_core.cuh decode_frame_tokens_lockstep).
// Dynamic shared memory: the 32 frames' probability tables transposed ([1056][32] bytes: lanes at the same
// tree position read one 32-byte row), then the 32 rows of above-contexts, also transposed ([mb_cols][32]).
__global__ void __launch_bounds__(32) k_tokens_lockstep(const uint8_t* ring, size_t stride, int first, int count,
                                                         int nslots, Geom g) {
#ifdef VP8GPU_SIMT_EMUL
  uint8_t* const dyn = simt::dyn_smem();
#else
  extern __shared__ __align__(16) uint8_t dyn[];
#endif
  __shared__ tok::LockstepTables T;
  uint8_t* const P = dyn;
  uint16_t* const above = reinterpret_cast<uint16_t*>(dyn + 1056 * 32);
  const int lane = threadIdx.x;
  tok::fill_lockstep_tables(T, lane, 32);
  const int job = blockIdx.x * 32 + lane;
  const TokJob* J = job < count ? reinterpret_cast<const TokJob*>(ring + static_cast<size_t>((first + job) % nslots) * stride) : nullptr;
  if (J) {  // this frame's 1056 probabilities -> column `lane` (the table in HBM is 4-byte aligned, 264 words)
    const uint32_t* src = reinterpret_cast<const uint32_t*>(J->coef_probs);
    for (int w = 0; w < 264; w++) {
      const uint32_t v = __ldg(src + w);
      P[(4 * w + 0) * 32 + lane] = v & 0xFF;
      P[(4 * w + 1) * 32 + lane] = (v >> 8) & 0xFF;
      P[(4 * w + 2) * 32 + lane] = (v >> 16) & 0xFF;
      P[(4 * w + 3) * 32 + lane] = v >> 24;
    }
  }
  __syncwarp();
  if (!J) return;
  tok::decode_frame_tokens_lockstep<32>(*J, g, T, P + lane, above + lane);
  publish_ready(*J);
}

__global__ void k_stamp(unsigned long long* dst) {
#ifndef VP8GPU_SIMT_EMUL
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  *dst = t;
#else
  *dst = 0;
#endif
}

}  // namespace

int launch_stamp(unsigned long long* dst, void* stream) {
  VP8_LAUNCH(k_stamp, 1, 1, 0, static_cast<cudaStream_t>(stream))(dst);
  return (int)cudaGetLastError();
}

int launch_tokens(const uint8_t* ring, size_t stride, int first, int count, int nslots, const Geom& g, void* stream) {
  if (g.mb_cols > kMaxCols) return (int)cudaErrorInvalidValue;
  // Variant knob.  1 (default) = one warp per frame, lane 0 decodes: the shortest latency per decision, but a
  // whole warp instruction per decision.  32 = one LANE per frame (lock-step state machine, 32 x fewer issue
  // slots, a longer latency per frame, which the pipeline feels because it is bounded by frames in flight).
  // 8 = 8 frames per CTA.
  static const int warps = [] {
    const char* v = getenv("VP8GPU_TOK_WARPS");
    return v && atoi(v) == 8 ? 8 : (v && atoi(v) == 32 ? 32 : 1);
  }();
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (warps == 32) {
    const size_t smem = 1056 * 32 + (size_t)g.mb_cols * 32 * sizeof(uint16_t);
    static const cudaError_t attr = cudaFuncSetAttribute(k_tokens_lockstep, cudaFuncAttributeMaxDynamicSharedMemorySize, 1056 * 32 + kMaxCols * 64);
    if (attr != cudaSuccess) return (int)attr;
    VP8_LAUNCH(k_tokens_lockstep, (count + 31) / 32, 32, smem, s)(ring, stride, first, count, nslots, g);
  }
  else if (warps == 8) VP8_LAUNCH(k_tokens<8>, (count + 7) / 8, 256, 0, s)(ring, stride, first, count, nslots, g);
  else VP8_LAUNCH(k_tokens<1>, count, 32, 0, s)(ring, stride, first, count, nslots, g);
  return (int)cudaGetLastError();
}

}  // namespace vp8
