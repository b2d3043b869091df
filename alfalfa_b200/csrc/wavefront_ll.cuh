// wavefront_ll.cuh -- included by kernels.cu inside namespace vp8 { namespace { ... } }.
//
// Round-2 versions of the two wavefront kernels (Macroblock::reconstruct_intra, macroblock.cc:524-551, and
// Frame::loopfilter, frame.cc:139-182).  Arithmetic, lane roles and shared-memory layouts are those of
// k_intra / k_loopfilter above; what changes is how a row learns that the row above is far enough and how
// it gets that row's pixels:
//
//   round 1   producer: pixels -> HBM, __syncwarp, st.release.gpu of a progress counter (a fence that waits for
//             the pixel stores), consumer: ld.acquire.gpu polling of the counter, THEN the loads of the pixels
//             -- two dependent L2 round trips plus the fence on every macroblock step of every row
//             (profiles/r2_phase_profile.txt: publish + wait + edge loads = half of a step).
//   round 2   hand-over messages: the producer writes the few pixels the row below needs (loop filter: its
//             bottom 4 lines, 128 bytes per macroblock; intra prediction: its bottom line, 32 bytes) a second
//             time, as 8-byte words { 4 pixels, epoch } into an area behind the raster.  Data and flag are one
//             naturally aligned 64-bit store, so no fence orders anything; the consumer's lanes load their
//             own words (one round trip, issued a macroblock ahead) and retry while the flag is not this
//             launch's epoch.  Pixels in the frame are no longer read by any other warp of the same kernel,
//             and each pixel is written by exactly one warp (the loop filter's bottom 4 lines of a macroblock
//             row are written by the row below, which filters them last), so the kernels contain no fence, no
//             acquire / release and no atomics besides the row ticket.
//   Epochs: the areas are zeroed when a raster is allocated and every launch uses a number no earlier launch
//   used (Engine::next_epoch), so a stale word can never look valid.
//
// Forward progress is as before: rows take tickets in row order, so the row a warp waits for was claimed by
// a warp that is already running.

struct Msg {
  uint32_t d, f;
};
#ifndef VP8GPU_SIMT_EMUL
__device__ __forceinline__ Msg ld_msg(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  Msg m;
  m.d = (uint32_t)v;
  m.f = (uint32_t)(v >> 32);
  return m;
}
__device__ __forceinline__ void st_msg(unsigned long long* p, uint32_t d, uint32_t f) {
  const unsigned long long v = (unsigned long long)d | ((unsigned long long)f << 32);
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
#else
__device__ __forceinline__ Msg ld_msg(const unsigned long long* p) {
  simt::yield();  // tests/simt: a poll lets the other threads of the CTA run
  const unsigned long long v = *reinterpret_cast<const volatile unsigned long long*>(p);
  Msg m;
  m.d = (uint32_t)v;
  m.f = (uint32_t)(v >> 32);
  return m;
}
__device__ __forceinline__ void st_msg(unsigned long long* p, uint32_t d, uint32_t f) {
  *reinterpret_cast<volatile unsigned long long*>(p) = (unsigned long long)d | ((unsigned long long)f << 32);
}
#endif
// Every lane with `need` retries its word until it carries this launch's epoch; `m` is the copy that was
// requested earlier.  Returns the data word (0 for lanes without need).
__device__ __forceinline__ uint32_t wait_msg(const unsigned long long* p, Msg m, bool need, uint32_t epoch) {
  unsigned ns = 32;
  for (;;) {
    const bool ok = !need || m.f == epoch;
    const unsigned late = __ballot_sync(0xffffffffu, !ok);
    if (!late) break;
    // one lane watches its word (one 8-byte request per retry instead of up to 32); the words of a message
    // are written by one store instruction and arrive together, so when it turns valid the others are
    // reloaded once -- and every lane still validates its own flag before using its data
    const int watcher = __ffs(late) - 1;
    if ((threadIdx.x & 31) == watcher) {
      for (;;) {
        __nanosleep(ns);
        m = ld_msg(p);
        if (m.f == epoch) break;
        if (ns < 256) ns += ns;
      }
    }
    __syncwarp();
    if (!ok && (threadIdx.x & 31) != watcher) m = ld_msg(p);
  }
  return need ? m.d : 0u;
}

// The words of a macroblock record that the wavefront kernels use, requested one macroblock ahead and decoded
// when the macroblock's turn comes (a decoded MbFields would occupy 13 registers across the whole step).
struct MbRaw {
  uint32_t x, y, z, bz, bw;
};
__device__ __forceinline__ MbRaw load_mb_raw(const vp8gpu_mb* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  const uint4 a = __ldg(q);
  const uint2 b = __ldg(reinterpret_cast<const uint2*>(p) + 3);  // b_modes
  MbRaw r;
  r.x = a.x, r.y = a.y, r.z = a.z, r.bz = b.x, r.bw = b.y;
  return r;
}
__device__ __forceinline__ MbFields decode_mb(const MbRaw& r) {
  MbFields f;
  f.tok_off = r.x;
  f.tok_cnt = r.y & 0xFFFF;
  f.y_mode = (r.y >> 16) & 0xFF;
  f.uv_mode = r.y >> 24;
  f.ref = r.z & 0xFF;
  f.segment = (r.z >> 8) & 0xFF;
  f.lf_level = (r.z >> 16) & 0xFF;
  f.flags = r.z >> 24;
  f.mv_x = f.mv_y = 0;
  f.split_idx = 0;
  f.bm_lo = r.bz;
  f.bm_hi = r.bw;
  return f;
}

// ================================================================================================
// k_intra_ll
// ================================================================================================
// message of intra macroblock (col, row), 8 words: 0-3 the bottom luma line, 4-5 the bottom U line, 6-7 V
__global__ void __launch_bounds__(32 * WF_WARPS, 18) k_intra_ll(const DevJob* __restrict__ jobs, int njobs, Geom g, int* ticket,
                                                                 uint32_t epoch) {
  __shared__ __align__(16) uint8_t s_W[WF_WARPS][17 * WS];
  __shared__ __align__(16) uint8_t s_pixc[WF_WARPS][128];  // U 8x8, V 8x8
  __shared__ __align__(16) int16_t s_coef[WF_WARPS][COEF_I16];
  __shared__ uint8_t s_aboveC[WF_WARPS][2][12];  // [0] = above-left, [1..8] = above
  __shared__ uint8_t s_leftC[WF_WARPS][2][8];
  __shared__ uint16_t s_lut[WF_WARPS][128];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* const W = s_W[warp];
  uint8_t* const pixc = s_pixc[warp];
  int16_t* const coef = s_coef[warp];
  uint8_t (*const aboveC)[12] = s_aboveC[warp];
  uint8_t (*const leftC)[8] = s_leftC[warp];
  uint16_t* const lut = s_lut[warp];
  for (int i = lane; i < 128; i += 32) lut[i] = k_bpred_lut[i];
  int t = 0;
  if (lane == 0) t = atomicAdd(ticket, 1);
  t = __shfl_sync(0xffffffffu, t, 0);
  const int row = t / njobs, job = t - row * njobs;
  if (row >= g.mb_rows) return;
  const DevJob& J = jobs[job];
  if (J.n_intra == 0) return;
  acquire_job(J, lane);
  const int cols = g.mb_cols;
  const vp8gpu_mb* row_mbs = J.mbs + (size_t)row * cols;

  // which macroblocks of this row, and of the row above, are intra-coded: bit c of a mask spread one word per
  // lane.  Inter-coded neighbours were finished by k_inter before this kernel started: their pixels are read
  // from the frame; intra-coded neighbours in the row above arrive as messages.
  const int nwords = (cols + 31) >> 5;
  uint32_t my_word = 0, above_word = 0;
  for (int w = 0; w < nwords; w++) {
    const int c = w * 32 + lane;
    const bool intra = c < cols && (__ldg(reinterpret_cast<const uint32_t*>(row_mbs + c) + 2) & 0xFF) == VP8GPU_REF_CURRENT;
    const uint32_t bits = __ballot_sync(0xffffffffu, intra);
    if (lane == w) my_word = bits;
    bool above = false;
    if (row > 0) above = c < cols && (__ldg(reinterpret_cast<const uint32_t*>(row_mbs - cols + c) + 2) & 0xFF) == VP8GPU_REF_CURRENT;
    const uint32_t abits = __ballot_sync(0xffffffffu, above);
    if (lane == w) above_word = abits;
  }
  int col = next_marked(my_word, 0, nwords);

  uint8_t* const Y = J.out;
  uint8_t* const U = J.out + g.u_off;
  uint8_t* const V = J.out + g.v_off;
  unsigned long long* const msg_row = reinterpret_cast<unsigned long long*>(J.out + g.msg_intra_off) + (size_t)row * cols * 8;
  const unsigned long long* const msg_above = msg_row - (size_t)cols * 8;  // only dereferenced when row > 0
  const bool sends = row + 1 < g.mb_rows;

  MbRaw raw;
  raw.x = raw.y = raw.z = raw.bz = raw.bw = 0;
  if (col >= 0) raw = load_mb_raw(row_mbs + col);
  int prev = -2;  // the macroblock this warp reconstructed last: its right column is still in shared memory

  PROF_DECL;
  while (col >= 0) {
    PROF(7);
    const int next = next_marked(my_word, col + 1, nwords);
    const MbFields f = decode_mb(raw);
    if (next >= 0) raw = load_mb_raw(row_mbs + next);  // in flight during this macroblock
    const bool has_res = f.tok_cnt != 0;
    PROF(0);

    // ---- request the edges (prediction.cc:99-167): messages for intra-coded macroblocks of the row above,
    //      the frame for inter-coded ones and for an inter-coded left neighbour; everything is issued
    //      before the residual is built, so the round trip overlaps the inverse transforms ----
    bool ia_l = false, ia_c = false, ia_r = false;  // above-left, above, above-right macroblock intra-coded
    if (row > 0) {
#pragma unroll
      for (int d = -1; d <= 1; d++) {
        const int c = col + d;
        const uint32_t word = __shfl_sync(0xffffffffu, above_word, (c >> 5) & 31);
        const bool bit = c >= 0 && c < cols && ((word >> (c & 31)) & 1);
        if (d == -1) ia_l = bit;
        else if (d == 0) ia_c = bit;
        else ia_r = bit;
      }
    }
    // lanes 0-7: the 8 words of the macroblock above; lane 8: word 0 of above-right (4 pixels);
    // lanes 9-11: words 3, 5, 7 of above-left (their last byte is the corner pixel of Y, U, V)
    const unsigned long long* mp = msg_above;
    bool need = false;
    if (lane < 8) {
      need = ia_c;
      mp = msg_above + (size_t)col * 8 + lane;
    } else if (lane == 8) {
      need = ia_r;
      mp = msg_above + (size_t)(col + 1) * 8;
    } else if (lane < 12) {
      need = ia_l;
      mp = msg_above + (size_t)(col - 1) * 8 + (2 * (lane - 9) + 3);
    }
    Msg m;
    m.d = 0, m.f = 0;
    if (need) m = ld_msg(mp);

    const int outside_above = row == 0 ? 127 : 129;  // value of above[-1] when it is not a pixel
    // (a) luma above row incl. corner and above-right: lanes 0..20, x = -1 .. 19
    const int ax = (lane >= 17 && col == cols - 1) ? 15 : lane - 1;  // replicate at the right frame edge
    const bool va = lane < 21 && row > 0 && !(lane == 0 && col == 0);
    const bool a_msg = va && (ax < 0 ? ia_l : (ax < 16 ? ia_c : ia_r));
    int a = outside_above;
    if (va && !a_msg) a = (int)ldcg_u8(Y + (size_t)(16 * row - 1) * g.y_pitch + 16 * col + ax);
    // (c) chroma above rows incl. corner: lanes 0..17, x = -1 .. 7 of U then V
    const int cpl = lane >= 9, ck = lane - 9 * cpl;
    const bool vc = lane < 18 && row > 0 && !(ck == 0 && col == 0);
    const bool c_msg = vc && (ck == 0 ? ia_l : ia_c);
    int c = outside_above;
    if (vc && !c_msg) c = (int)ldcg_u8((cpl ? V : U) + (size_t)(8 * row - 1) * g.c_pitch + 8 * col + ck - 1);
    // (b) left columns: lanes 0..15 luma, 16..23 U, 24..31 V.  An intra-coded left neighbour is the macroblock
    //     this warp has just reconstructed (still in shared memory); an inter-coded one is in the frame.
    int b = 129;
    if (col > 0) {
      if (prev == col - 1) {
        b = lane < 16 ? W[(lane + 1) * WS + 31] : pixc[((lane >> 3) & 1) * 64 + (lane & 7) * 8 + 7];
      } else {
        const uint8_t* pb = lane < 16 ? Y + (size_t)(16 * row + lane) * g.y_pitch + 16 * col - 1
                                      : ((lane & 8) ? V : U) + (size_t)(8 * row + (lane & 7)) * g.c_pitch + 8 * col - 1;
        b = (int)ldcg_u8(pb);
      }
    }
    __syncwarp();  // the left column has been read out of W / pixc before anything below overwrites them

    // the residual only depends on this macroblock's tokens
    if (has_res) build_residuals(J, f, coef, lane);
    PROF(1);

    // ---- messages: wait, then hand every lane its pixel ----
    const uint32_t md = wait_msg(mp, m, need, epoch);
    PROF(2);
    {
      const int sl = ax < 0 ? 9 : (ax < 16 ? (ax >> 2) : 8);
      const int sb = ax < 0 ? 3 : (ax & 3);
      const uint32_t w = __shfl_sync(0xffffffffu, md, sl & 31);
      if (a_msg) a = (int)((w >> (8 * sb)) & 0xFF);
      const int cx = ck - 1;
      const int cl = cx < 0 ? 10 + cpl : 4 + 2 * cpl + ((cx >> 2) & 1);
      const int cb = cx < 0 ? 3 : (cx & 3);
      const uint32_t wc = __shfl_sync(0xffffffffu, md, cl & 31);
      if (c_msg) c = (int)((wc >> (8 * cb)) & 0xFF);
    }
    if (lane < 21) W[15 + lane] = (uint8_t)a;
    if (lane < 16) W[(lane + 1) * WS + 15] = (uint8_t)b;
    else leftC[(lane >> 3) & 1][lane & 7] = (uint8_t)b;
    if (lane < 18) aboveC[cpl][ck] = (uint8_t)c;
    __syncwarp();
    PROF(3);

    // ---- chroma 8x8 prediction (prediction.cc:435-449): one 4-pixel word per lane ----
    {
      const int plane = lane >> 4, y = (lane >> 1) & 7, x4 = (lane & 1) * 4;
      const uint8_t* A = aboveC[plane] + 1;
      const uint8_t* L = leftC[plane];
      uint32_t word;
      if (f.uv_mode == VP8GPU_DC_PRED) {
        int s = 0, n = 0;
        if (row > 0) { for (int k = 0; k < 8; k++) s += A[k]; n += 8; }
        if (col > 0) { for (int k = 0; k < 8; k++) s += L[k]; n += 8; }
        word = (uint32_t)(n == 16 ? (s + 8) >> 4 : (n == 8 ? (s + 4) >> 3 : 128)) * 0x01010101u;
      } else if (f.uv_mode == VP8GPU_V_PRED) {
        word = (uint32_t)A[x4] | ((uint32_t)A[x4 + 1] << 8) | ((uint32_t)A[x4 + 2] << 16) | ((uint32_t)A[x4 + 3] << 24);
      } else if (f.uv_mode == VP8GPU_H_PRED) {
        word = (uint32_t)L[y] * 0x01010101u;
      } else {
        const int base = L[y] - A[-1];
        word = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) word |= (uint32_t)vp8m::clamp255(base + A[x4 + k]) << (8 * k);
      }
      *reinterpret_cast<uint32_t*>(pixc + plane * 64 + y * 8 + x4) = word;
    }

    if (f.y_mode != VP8GPU_B_PRED) {
      // ---- luma 16x16 prediction (prediction.cc:451-467): 8 pixels (two words) per lane ----
      const int y = lane >> 1, x8 = (lane & 1) * 8;
      const uint8_t* A = W + 16;  // above[x]
      const int left = W[(y + 1) * WS + 15];
      uint32_t w0, w1;
      if (f.y_mode == VP8GPU_DC_PRED) {
        int s = 0, n = 0;
        if (row > 0) { for (int k = 0; k < 16; k++) s += A[k]; n += 16; }
        if (col > 0) { for (int k = 0; k < 16; k++) s += W[(k + 1) * WS + 15]; n += 16; }
        w0 = w1 = (uint32_t)(n == 32 ? (s + 16) >> 5 : (n == 16 ? (s + 8) >> 4 : 128)) * 0x01010101u;
      } else if (f.y_mode == VP8GPU_V_PRED) {
        w0 = *reinterpret_cast<const uint32_t*>(A + x8);
        w1 = *reinterpret_cast<const uint32_t*>(A + x8 + 4);
      } else if (f.y_mode == VP8GPU_H_PRED) {
        w0 = w1 = (uint32_t)left * 0x01010101u;
      } else {
        const int base = left - W[15];
        w0 = w1 = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
          w0 |= (uint32_t)vp8m::clamp255(base + A[x8 + k]) << (8 * k);
          w1 |= (uint32_t)vp8m::clamp255(base + A[x8 + 4 + k]) << (8 * k);
        }
      }
      __syncwarp();  // all lanes have read the left column / above row they need
      *reinterpret_cast<uint32_t*>(W + (y + 1) * WS + 16 + x8) = w0;
      *reinterpret_cast<uint32_t*>(W + (y + 1) * WS + 20 + x8) = w1;
      __syncwarp();
      if (has_res) add_residuals_intra(W, pixc, coef, lane, true);
    } else {
      // ---- B_PRED: 16 sub-blocks in raster order, each predicted from reconstructed
      //      neighbours, residual added before the next one starts (macroblock.cc:540-545) ----
      if (lane < 12) W[(4 + 4 * (lane >> 2)) * WS + 32 + (lane & 3)] = W[32 + (lane & 3)];  // above-right copies
      __syncwarp();
      if (has_res) add_residuals_intra(W, pixc, coef, lane, false);  // chroma only
      const uint64_t modes = ((uint64_t)f.bm_hi << 32) | f.bm_lo;
      const int x = lane & 3, y = (lane >> 2) & 3;
#pragma unroll
      for (int bi = 0; bi < 16; bi++) {  // fully unrolled: table entries and residuals load ahead of the chain
        const int bx = bi & 3, by = bi >> 2;
        const int mode = (int)((modes >> (4 * bi)) & 15);
        // edge entry i of this sub-block: i < 4 -> left[3 - i], i = 4 -> above[-1], i > 4 -> above[i - 5]
        const uint8_t* e0 = W + (4 * by) * WS + 15 + 4 * bx;  // = above[-1]
        if (lane < 16) {
          int v;
          if (mode == VP8GPU_B_DC_PRED) {
            int s4 = 4;
#pragma unroll
            for (int k = 0; k < 4; k++) s4 += e0[1 + k] + e0[(1 + k) * WS];
            v = s4 >> 3;
          } else if (mode == VP8GPU_B_TM_PRED) {
            v = vp8m::clamp255(e0[(1 + y) * WS] + e0[1 + x] - e0[0]);
          } else {
            const unsigned entry = lut[(mode - 2) * 16 + lane];
            const int ia = entry & 15, ib = (entry >> 4) & 15, ic = (entry >> 8) & 15;
            const int pa = e0[ia < 4 ? (4 - ia) * WS : ia - 4];
            const int pb = e0[ib < 4 ? (4 - ib) * WS : ib - 4];
            const int pc = e0[ic < 4 ? (4 - ic) * WS : ic - 4];
            v = (entry & 0x1000) ? ((pa + 2 * pb + pc + 2) >> 2) : ((pa + pb + 1) >> 1);
          }
          if (has_res) v = vp8m::clamp255(v + coef[bi * CS + lane]);
          W[(4 * by + y + 1) * WS + 16 + 4 * bx + x] = (uint8_t)v;
        }
        __syncwarp();
      }
    }
    __syncwarp();
    PROF(4);
    // ---- hand the bottom lines to the row below, then macroblock -> frame ----
    if (sends && lane < 8) {
      const uint32_t d = lane < 4 ? *reinterpret_cast<const uint32_t*>(W + 16 * WS + 16 + 4 * lane)
                                  : *reinterpret_cast<const uint32_t*>(pixc + ((lane - 4) >> 1) * 64 + 56 + 4 * (lane & 1));
      st_msg(msg_row + (size_t)col * 8 + lane, d, epoch);
    }
    if (lane < 16) {
      *reinterpret_cast<uint4*>(Y + (size_t)(16 * row + lane) * g.y_pitch + 16 * col) =
          *reinterpret_cast<const uint4*>(W + (lane + 1) * WS + 16);
    } else {
      const int plane = (lane - 16) >> 3, yy = lane & 7;
      *reinterpret_cast<uint2*>((plane ? V : U) + (size_t)(8 * row + yy) * g.c_pitch + 8 * col) =
          *reinterpret_cast<const uint2*>(pixc + plane * 64 + yy * 8);
    }
    PROF(5);
    PROF(6);
    PROF_COUNT();
    prev = col;
    col = next;
  }
  PROF_FLUSH(0);
}

// ================================================================================================
// k_loopfilter_ll
// ================================================================================================
// Every row walks ALL its macroblocks (one whose level is 0 passes through unfiltered): the step of macroblock c
// finalises region columns 0..15 = frame x in [16c - 4, 16c + 12).  Message A(row, c), c = 0 .. cols, 32 words:
// the bottom 4 lines of that span -- lanes 0-15: luma line j = lane >> 2, word w = lane & 3 (x = 16c - 4 + 4w);
// lanes 16-31: plane p, line j, word w of chroma (x = 8c - 4 + 4w); A(row, cols) carries the last 4 columns
// in its words w = 0.  The row below needs x in [16c, 16c + 16) for its macroblock c: words 1-3 of A(c) and
// word 0 of A(c + 1), i.e. one new message per step, requested one step ahead.
__global__ void __launch_bounds__(32 * WF_WARPS, 14) k_loopfilter_ll(const DevJob* __restrict__ jobs, int njobs, Geom g, int* ticket,
                                                                      uint32_t epoch) {
  constexpr int YS = 20, CSZ = 12;
  __shared__ __align__(16) uint8_t s_ry[WF_WARPS][20 * YS];
  __shared__ __align__(16) uint8_t s_rc[WF_WARPS][2][12 * CSZ];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* const ry = s_ry[warp];
  uint8_t (*const rc)[12 * CSZ] = s_rc[warp];
  int t = 0;
  if (lane == 0) t = atomicAdd(ticket, 1);
  t = __shfl_sync(0xffffffffu, t, 0);
  const int row = t / njobs, job = t - row * njobs;
  if (row >= g.mb_rows) return;
  const DevJob& J = jobs[job];
  if (!J.lf_enabled) return;
  acquire_job(J, lane);
  const int cols = g.mb_cols;
  const vp8gpu_mb* row_mbs = J.mbs + (size_t)row * cols;
  const bool last_row = row == g.mb_rows - 1;

  uint8_t* const Y = J.out;
  uint8_t* const U = J.out + g.u_off;
  uint8_t* const V = J.out + g.v_off;
  const int y_lo = row > 0 ? 0 : 4;           // first region row that exists in the frame
  const int y_hi = last_row ? 20 : 16;        // luma region rows this warp writes: the bottom 4 lines of a
  const int yc_hi = last_row ? 12 : 8;        // macroblock row are final only after the row below filtered them
  // message c of row r (this lane's word); derived from Y on use instead of being kept in registers
  auto msg_at = [&](int r, int c) {
    return reinterpret_cast<unsigned long long*>(Y + g.msg_lf_off) + ((size_t)r * (cols + 1) + c) * 32 + lane;
  };

  // this lane's word in a message / in the top 4 lines of the region
  const bool luma_w = lane < 16;
  const int mj = luma_w ? lane >> 2 : ((lane - 16) & 7) >> 1;  // line 0..3
  const int mw = luma_w ? lane & 3 : lane & 1;                // word within the line
  const int mp = luma_w ? 0 : (lane - 16) >> 3;               // chroma plane
  const int words = luma_w ? 4 : 2;
  const int line0 = luma_w ? 4 * mj : 16 + 8 * mp + 2 * mj;    // lane that holds word 0 of this line

  auto own_ptr = [&](int k, int c, const uint8_t*& gp, uint8_t*& sp) {
    const int w = lane + 32 * k;
    if (w < 64) {
      const int r = w >> 2, wx = w & 3;
      gp = Y + (size_t)(16 * row + r) * g.y_pitch + 16 * c + 4 * wx;
      sp = ry + (4 + r) * YS + 4 + 4 * wx;
    } else {
      const int cw = w - 64, plane = cw >> 4, k2 = cw & 15, r = k2 >> 1, wx = k2 & 1;
      gp = (plane ? V : U) + (size_t)(8 * row + r) * g.c_pitch + 8 * c + 4 * wx;
      sp = rc[plane] + (4 + r) * CSZ + 4 + 4 * wx;
    }
  };
  uint32_t own[3];
  auto prefetch_own = [&](int c) {
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const uint8_t* gp;
      uint8_t* sp;
      own_ptr(k, c, gp, sp);
      own[k] = __ldcg(reinterpret_cast<const uint32_t*>(gp));
    }
  };
  prefetch_own(0);
  uint32_t a0 = 0;
  Msg spec;
  spec.d = 0, spec.f = 0;
  if (row > 0) {
    a0 = wait_msg(msg_at(row - 1, 0), ld_msg(msg_at(row - 1, 0)), true, epoch);
    spec = ld_msg(msg_at(row - 1, 1));
  }

  PROF_DECL;
  for (int col = 0; col < cols; col++) {
    PROF(7);
    PROF(0);
    // ---- top 4 lines (final output of the row above): words 1.. of A(col), word 0 of A(col + 1) ----
    uint32_t top = 0;
    if (row > 0) {
      const uint32_t a1 = wait_msg(msg_at(row - 1, col + 1), spec, true, epoch);
      if (col + 2 <= cols) spec = ld_msg(msg_at(row - 1, col + 2));  // in flight while this macroblock is filtered
      const uint32_t t0 = __shfl_sync(0xffffffffu, a0, (line0 + ((mw + 1) & (words - 1))) & 31);
      const uint32_t t1 = __shfl_sync(0xffffffffu, a1, line0 & 31);
      top = mw == words - 1 ? t1 : t0;
      a0 = a1;
    }
    PROF(1);
    // ---- left 4 columns: slide them over from the previous macroblock ----
    uint32_t left0 = 0, left1 = 0;
    if (col > 0) {
      if (lane < 20) left0 = *reinterpret_cast<const uint32_t*>(ry + lane * YS + 16);
      if (lane < 24) left1 = *reinterpret_cast<const uint32_t*>(rc[lane / 12] + (lane % 12) * CSZ + 8);
    }
    __syncwarp();  // everybody has read the old region before it is overwritten
    if (col > 0) {
      if (lane < 20) *reinterpret_cast<uint32_t*>(ry + lane * YS) = left0;
      if (lane < 24) *reinterpret_cast<uint32_t*>(rc[lane / 12] + (lane % 12) * CSZ) = left1;
    }
    if (row > 0) {
      if (luma_w) *reinterpret_cast<uint32_t*>(ry + mj * YS + 4 + 4 * mw) = top;
      else *reinterpret_cast<uint32_t*>(rc[mp] + mj * CSZ + 4 + 4 * mw) = top;
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const uint8_t* gp;
      uint8_t* sp;
      own_ptr(k, col, gp, sp);
      *reinterpret_cast<uint32_t*>(sp) = own[k];
    }
    __syncwarp();
    PROF(2);
    if (col + 1 < cols) prefetch_own(col + 1);  // in flight while this macroblock is filtered

    // of the record the filter needs tok_cnt (word 1) and lf_level / flags (word 2); four records share a
    // 128-byte line of the read-only cache, so this is rarely a round trip
    const uint32_t rec_y = __ldg(reinterpret_cast<const uint32_t*>(row_mbs + col) + 1);
    const uint32_t rec_z = __ldg(reinterpret_cast<const uint32_t*>(row_mbs + col) + 2);
    const int mb_tok_cnt = rec_y & 0xFFFF, mb_level = (rec_z >> 16) & 0xFF, mb_flags = rec_z >> 24;
    const int level = J.lf_force ? J.lf_force : mb_level;
    if (level != 0) {
      const vp8m::LfParams lp = vp8m::lf_params(level, J.sharpness, J.key_frame);
      const bool do_inner = !((mb_flags & VP8GPU_MB_HAS_Y2) && mb_tok_cnt == 0);  // macroblock.cc:608
      // lane roles on an edge: 0-15 luma positions, 16-23 U, 24-31 V
      const bool luma = lane < 16;
      uint8_t* const plane_base = luma ? ry : rc[(lane - 16) >> 3];
      const int stride = luma ? YS : CSZ, idx = luma ? lane : (lane & 7), len = luma ? 20 : 12;
      int px[20];
      // ---- vertical edges: one region row (4 + idx) per lane, in registers ----
      {
        const uint32_t* rw = reinterpret_cast<const uint32_t*>(plane_base + (4 + idx) * stride);
#pragma unroll
        for (int k = 0; k < 5; k++) {
          const uint32_t v = (k < 3 || luma) ? rw[k] : 0u;
          px[4 * k] = v & 0xFF, px[4 * k + 1] = (v >> 8) & 0xFF, px[4 * k + 2] = (v >> 16) & 0xFF, px[4 * k + 3] = v >> 24;
        }
        filter_line(px, luma, col > 0, do_inner, lp);
        uint32_t* ww = reinterpret_cast<uint32_t*>(plane_base + (4 + idx) * stride);
#pragma unroll
        for (int k = 0; k < 5; k++)
          if (k < 3 || luma) ww[k] = (uint32_t)px[4 * k] | ((uint32_t)px[4 * k + 1] << 8) | ((uint32_t)px[4 * k + 2] << 16) | ((uint32_t)px[4 * k + 3] << 24);
      }
      __syncwarp();
      // ---- horizontal edges: one region column (4 + idx) per lane ----
      {
        uint8_t* cp = plane_base + 4 + idx;
#pragma unroll
        for (int k = 0; k < 20; k++) px[k] = k < len ? cp[k * stride] : 0;
        filter_line(px, luma, row > 0, do_inner, lp);
#pragma unroll
        for (int k = 1; k < 19; k++)
          if (k < len - 1) cp[k * stride] = (uint8_t)px[k];
      }
      __syncwarp();
    }
    PROF(3);

    // ---- hand the bottom 4 lines of region columns 0..15 to the row below ----
    const bool last_col = col == cols - 1;
    if (!last_row) {
      const uint8_t* src = luma_w ? ry + (16 + mj) * YS : rc[mp] + (8 + mj) * CSZ;
      st_msg(msg_at(row, col), *reinterpret_cast<const uint32_t*>(src + 4 * mw), epoch);
      if (last_col) st_msg(msg_at(row, cols), *reinterpret_cast<const uint32_t*>(src + (luma_w ? 16 : 8)), epoch);
    }
    // ---- write back: region columns 0..15 (x -4..11); the last 4 columns travel with the next macroblock ----
    const int x_lo = col > 0 ? 0 : 1;
    {
      uint8_t* const gy = Y + (size_t)(16 * row - 4) * g.y_pitch + 16 * col - 4;
#pragma unroll
      for (int k = 0; k < 3; k++) {  // luma words 0..79: 20 rows x 4 words
        const int w = lane + 32 * k, r = w >> 2, wx = w & 3;
        if (w < 80 && r >= y_lo && r < y_hi && wx >= x_lo)
          *reinterpret_cast<uint32_t*>(gy + (size_t)r * g.y_pitch + 4 * wx) = *reinterpret_cast<const uint32_t*>(ry + r * YS + 4 * wx);
      }
#pragma unroll
      for (int k = 0; k < 2; k++) {  // chroma words 0..47: 2 planes x 12 rows x 2 words
        const int w = lane + 32 * k, plane = w >= 24, kk = w - 24 * plane, r = kk >> 1, wx = kk & 1;
        if (w < 48 && r >= y_lo && r < yc_hi && wx >= x_lo)
          *reinterpret_cast<uint32_t*>((plane ? V : U) + (size_t)(8 * row - 4 + r) * g.c_pitch + 8 * col - 4 + 4 * wx) =
              *reinterpret_cast<const uint32_t*>(rc[plane] + r * CSZ + 4 * wx);
      }
      if (last_col) {
        if (lane < 20 && lane >= y_lo && lane < y_hi)
          *reinterpret_cast<uint32_t*>(gy + (size_t)lane * g.y_pitch + 16) = *reinterpret_cast<const uint32_t*>(ry + lane * YS + 16);
        if (lane < 24) {
          const int plane = lane >= 12, r = lane - 12 * plane;
          if (r >= y_lo && r < yc_hi)
            *reinterpret_cast<uint32_t*>((plane ? V : U) + (size_t)(8 * row - 4 + r) * g.c_pitch + 8 * col + 4) =
                *reinterpret_cast<const uint32_t*>(rc[plane] + r * CSZ + 8);
        }
      }
    }
    PROF(4);
    PROF(5);
    PROF_COUNT();
  }
  PROF_FLUSH(16);
}
