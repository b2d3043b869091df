// reencode.cuh -- device half of Encoder::update_residues (encoder/reencode.cc:131-313, SURVEY.md 8 row f3):
// the modes, vectors and references of an already coded inter frame are kept, the residues are recomputed
// against the CURRENT references so that the frame decodes as close as possible to a target raster.
// Included by kernels.cu after k_enc_rd (shares its workspace, transforms and wavefront plumbing).
//
// The reference walks the macroblocks in raster order: predict with the frame's own mode, subtract from the
// target, fdct / wht, quantise (truncating division, FIRST_PASS), reconstruct.  Only intra macroblocks depend on
// their neighbours' reconstruction, so the work is split:
//   1. k_inter with empty token lists (the decoder's own kernel)      -> the prediction of every inter macroblock
//   2. k_reenc_inter, one warp per inter macroblock, no dependencies   -> its tokens (luma_mb_apply_inter_prediction
//                                                                         encode_inter.cc:375-435, chroma_mb_inter_predict :437-500)
//   3. k_inter again with those tokens                                 -> its reconstruction (reconstruct_inter)
//   4. k_reenc_intra, one warp per macroblock row, 2-macroblock lag    -> intra macroblocks: prediction from the
//      reconstruction so far with the frame's mode (update_macroblock reencode.cc:143-167, 210-232), tokens,
//      reconstruction (luma_mb_apply_intra_prediction encode_intra.cc:168-221, luma_sb_apply_intra_prediction,
//      chroma_mb_apply_intra_prediction :286-330)
// The loop filter is not part of this (reencode.cc: the frame is written and then decoded like any other).

// quantise the 25 blocks of coef (lane = block; lane 24 = Y2 when has_y2), emit the non-zero values as tokens,
// leave the DEQUANTISED coefficients in coef.  qb != nullptr: the luma blocks were quantised earlier (B_PRED).
// Returns the macroblock's token count; base = its first token.
__device__ __forceinline__ int reenc_quantize_emit(int16_t* coef, const int16_t (*qb)[16], bool has_y2, const vp8gpu_quant& q,
                                                   uint32_t* tok_counter, uint32_t tok_cap, vp8gpu_token* tokens, uint32_t& base,
                                                   int lane) {
  int cnt = 0;
  int16_t qv[16];
  const bool has_blk = lane < 24 || (lane == 24 && has_y2);
  if (has_blk) {
    const int dcq = lane < 16 ? q.y_dc : (lane < 24 ? q.uv_dc : q.y2_dc);
    const int acq = lane < 16 ? q.y_ac : (lane < 24 ? q.uv_ac : q.y2_ac);
#pragma unroll
    for (int k = 0; k < 16; k++) {
      int v;
      if (qb && lane < 16) {
        v = qb[lane][k];
      } else {
        int c = coef[lane * CS + k];
        if (has_y2 && lane < 16 && k == 0) c = 0;  // Y_after_Y2: the luma DCs travel in Y2
        v = vp8m::quantize_trunc(c, k ? acq : dcq);
        v = v > 2047 ? 2047 : (v < -2047 ? -2047 : v);
      }
      qv[k] = (int16_t)v;
      cnt += v != 0;
      coef[lane * CS + k] = (int16_t)(v * (k ? acq : dcq));
    }
  }
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  base = 0;
  if (lane == 0 && total) base = atomicAdd(tok_counter, (uint32_t)total);
  base = __shfl_sync(0xffffffffu, base, 0);
  if (has_blk && cnt && base + total <= tok_cap) {
    uint32_t at = base + incl - cnt;
#pragma unroll
    for (int k = 0; k < 16; k++)
      if (qv[k]) tokens[at++] = VP8GPU_TOKEN(lane, k, qv[k]);
  }
  __syncwarp();
  return total;
}

// forward DCT of the residual target - prediction, one 4x4 block per lane (0-15 luma, 16-23 chroma), then the WHT
// of the sixteen luma DCs by lane 24.  src: Y 16x16 at 0, U 8x8 at 256, V at 320; predY(y, x) / predC(plane, y, x)
template <class PY, class PC>
__device__ __forceinline__ void reenc_forward(const uint8_t* src, PY predY, PC predC, int16_t* coef, bool luma, bool has_y2, int lane) {
  if (lane < 24 && (luma || lane >= 16)) {
    int16_t d[16], o[16];
    if (lane < 16) {
      const int bx = lane & 3, by = lane >> 2;
#pragma unroll
      for (int k = 0; k < 16; k++) d[k] = (int16_t)((int)src[(4 * by + (k >> 2)) * 16 + 4 * bx + (k & 3)] - predY(4 * by + (k >> 2), 4 * bx + (k & 3)));
    } else {
      const int c = lane - 16, plane = c >> 2, bx = c & 1, by = (c >> 1) & 1;
#pragma unroll
      for (int k = 0; k < 16; k++)
        d[k] = (int16_t)((int)src[256 + plane * 64 + (4 * by + (k >> 2)) * 8 + 4 * bx + (k & 3)] - predC(plane, 4 * by + (k >> 2), 4 * bx + (k & 3)));
    }
    vp8m::fdct16(d, o);
#pragma unroll
    for (int k = 0; k < 16; k++) coef[lane * CS + k] = o[k];
  }
  __syncwarp();
  if (has_y2 && lane == 24) {
    int16_t in[16], o[16];
#pragma unroll
    for (int k = 0; k < 16; k++) in[k] = coef[k * CS];
    vp8m::fwht16(in, o);
#pragma unroll
    for (int k = 0; k < 16; k++) coef[24 * CS + k] = o[k];
  }
  __syncwarp();
}

__device__ __forceinline__ void reenc_load_target(const ReencJob& J, const Geom& g, int col, int row, uint8_t* src, int lane) {
  for (int i = lane; i < 96; i += 32) {
    const uint8_t* gp;
    if (i < 64) gp = J.target + (size_t)(16 * row + (i >> 2)) * g.y_pitch + 16 * col + 4 * (i & 3);
    else {
      const int c = i - 64, plane = c >> 4, k = c & 15;
      gp = J.target + (plane ? g.v_off : g.u_off) + (size_t)(8 * row + (k >> 1)) * g.c_pitch + 8 * col + 4 * (k & 1);
    }
    reinterpret_cast<uint32_t*>(src)[i] = __ldg(reinterpret_cast<const uint32_t*>(gp));
  }
}

constexpr int REENC_WARPS = 4;
struct __align__(16) ReencInterSmem {  // per warp
  uint8_t src[384];
  uint8_t pred[384];
  int16_t coef[COEF_I16];
};

// step 2: tokens of every inter macroblock.  J.recon holds the predictions (step 1).  One launch serves njobs frames
// of the context (Encoder::update_residues of several Encoders at once): job blockIdx.y, macroblocks along blockIdx.x.
__global__ void __launch_bounds__(32 * REENC_WARPS) k_reenc_inter(const ReencJob* __restrict__ jobp, int njobs, Geom g) {
  __shared__ ReencInterSmem s_all[REENC_WARPS];
  const ReencJob& J = jobp[blockIdx.y];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mbi = blockIdx.x * REENC_WARPS + warp;
  if (mbi >= J.cols * J.rows) return;
  const MbFields f = load_mb(J.mbs_in + mbi);
  if (f.ref == VP8GPU_REF_CURRENT) return;  // intra macroblocks belong to k_reenc_intra
  const int row = mbi / J.cols, col = mbi - row * J.cols;
  ReencInterSmem& S = s_all[warp];
  reenc_load_target(J, g, col, row, S.src, lane);
  for (int i = lane; i < 96; i += 32) {
    const uint8_t* gp;
    if (i < 64) gp = J.recon + (size_t)(16 * row + (i >> 2)) * g.y_pitch + 16 * col + 4 * (i & 3);
    else {
      const int c = i - 64, plane = c >> 4, k = c & 15;
      gp = J.recon + (plane ? g.v_off : g.u_off) + (size_t)(8 * row + (k >> 1)) * g.c_pitch + 8 * col + 4 * (k & 1);
    }
    reinterpret_cast<uint32_t*>(S.pred)[i] = __ldg(reinterpret_cast<const uint32_t*>(gp));
  }
  __syncwarp();
  const bool has_y2 = f.y_mode != VP8GPU_SPLITMV;  // SPLITMV: set_Y_without_Y2, Y2 not coded (encode_inter.cc:385-404)
  const uint8_t* pred = S.pred;
  reenc_forward(
      S.src, [pred](int y, int x) { return (int)pred[y * 16 + x]; }, [pred](int plane, int y, int x) { return (int)pred[256 + plane * 64 + y * 8 + x]; },
      S.coef, true, has_y2, lane);
  uint32_t base;
  const int total = reenc_quantize_emit(S.coef, nullptr, has_y2, J.q, J.tok_counter, J.tok_cap, J.tokens, base, lane);
  if (lane == 0) {
    vp8gpu_mb m = J.mbs_in[mbi];
    m.tok_off = base;
    m.tok_cnt = (uint16_t)total;
    m.flags = has_y2 ? VP8GPU_MB_HAS_Y2 : 0;
    J.mbs_out[mbi] = m;
  }
}

// step 4: the intra macroblocks, in dependency order.  J.recon holds every inter macroblock reconstructed (step 3).
__global__ void __launch_bounds__(32 * WF_WARPS, 8) k_reenc_intra(const ReencJob* __restrict__ jobp, int njobs, Geom g, int* ticket) {
  __shared__ EncSmem s_all[WF_WARPS];
  __shared__ uint16_t s_lut[128];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 128; i += blockDim.x) s_lut[i] = k_bpred_lut[i];
  __syncthreads();
  EncSmem& S = s_all[warp];
  uint8_t* const W = S.W;
  uint8_t* const Wb = S.Wb;
  uint8_t* const pixc = S.pixc;
  uint8_t* const src = S.src;
  int16_t* const coef = S.coef;
  int t = 0;
  if (lane == 0) t = atomicAdd(ticket, 1);
  t = __shfl_sync(0xffffffffu, t, 0);
  // ticket t -> row t / njobs of job t % njobs (as k_enc_rd): the row a warp waits for, row - 1 of the same job, holds
  // ticket t - njobs, so it was claimed by a warp that is already running; every job has its own progress counters
  const ReencJob& J = jobp[t % njobs];
  const int row = t / njobs;
  const int cols = J.cols, rows = J.rows;
  if (row >= rows) return;
  int* progress = J.progress + row;
  uint8_t* const Y = J.recon;
  uint8_t* const U = J.recon + g.u_off;
  uint8_t* const V = J.recon + g.v_off;
  const vp8gpu_quant q = J.q;

  // Which macroblocks of this row are intra-coded: one mask word per lane (as in k_intra).  The inter-coded ones were
  // reconstructed by step 3 and nothing of them depends on this frame, so the row only stops at its intra macroblocks
  // and publishes "everything left of the next one is done" -- a row without any is finished at once instead of
  // walking (and publishing) every macroblock.
  const int nwords = (cols + 31) >> 5;
  uint32_t my_word = 0;
  for (int w = 0; w < nwords; w++) {
    const int c = w * 32 + lane;
    const bool intra = c < cols && (__ldg(reinterpret_cast<const uint32_t*>(J.mbs_in + row * cols + c) + 2) & 0xFF) == VP8GPU_REF_CURRENT;
    const uint32_t bits = __ballot_sync(0xffffffffu, intra);
    if (lane == w) my_word = bits;
  }
  int col = next_marked(my_word, 0, nwords);
  // progress = P means: every macroblock of this row with column < P is reconstructed
  publish_row(progress, col < 0 ? cols : col, lane);

  while (col >= 0) {
    const int mbi = row * cols + col;
    const MbFields f = load_mb(J.mbs_in + mbi);
    reenc_load_target(J, g, col, row, src, lane);
    __syncwarp();
    // (the above-right macroblock only matters to the sub-blocks of a B_PRED macroblock, prediction.cc:143-167)
    if (row > 0) wait_row(progress - 1, min(col + (f.y_mode == VP8GPU_B_PRED ? 2 : 1), cols), lane);

    // ---- edges of the reconstruction so far (prediction.cc:99-167; same rules as k_intra / k_enc_rd) ----
    {
      const int outside_above = row == 0 ? 127 : 129;
      const uint8_t* pa = Y;
      bool va = false;
      if (lane < 21 && row > 0 && !(lane == 0 && col == 0)) {
        const int x = (lane >= 17 && col == cols - 1) ? 15 : lane - 1;
        pa = Y + (size_t)(16 * row - 1) * g.y_pitch + 16 * col + x;
        va = true;
      }
      const uint8_t* pb = Y;
      if (col > 0) {
        if (lane < 16) pb = Y + (size_t)(16 * row + lane) * g.y_pitch + 16 * col - 1;
        else pb = ((lane & 8) ? V : U) + (size_t)(8 * row + (lane & 7)) * g.c_pitch + 8 * col - 1;
      }
      const uint8_t* pc = Y;
      bool vc = false;
      const int cpl = lane >= 9, ck = lane - 9 * cpl;
      if (lane < 18 && row > 0 && !(ck == 0 && col == 0)) {
        pc = (cpl ? V : U) + (size_t)(8 * row - 1) * g.c_pitch + 8 * col + ck - 1;
        vc = true;
      }
      const int a = va ? (int)ldcg_u8(pa) : outside_above;
      const int b = col > 0 ? (int)ldcg_u8(pb) : 129;
      const int c = vc ? (int)ldcg_u8(pc) : outside_above;
      if (lane < 21) W[15 + lane] = (uint8_t)a;
      if (lane < 16) W[(lane + 1) * WS + 15] = (uint8_t)b;
      else S.leftC[(lane >> 3) & 1][lane & 7] = (uint8_t)b;
      if (lane < 18) S.aboveC[cpl][ck] = (uint8_t)c;
    }
    __syncwarp();
    const uint8_t* A = W + 16;  // above[x]
    const bool bpred = f.y_mode == VP8GPU_B_PRED;

    if (bpred) {
      // ---- sub-blocks in raster order with the frame's own modes, each coded and reconstructed before the next
      //      one is predicted (update_macroblock reencode.cc:152-167 -> luma_sb_apply_intra_prediction) ----
      if (lane < 21) Wb[15 + lane] = W[15 + lane];
      if (lane < 16) Wb[(lane + 1) * WS + 15] = W[(lane + 1) * WS + 15];
      __syncwarp();
      if (lane < 12) Wb[(4 + 4 * (lane >> 2)) * WS + 32 + (lane & 3)] = Wb[32 + (lane & 3)];  // above-right copies
      __syncwarp();
      const unsigned long long bm = (unsigned long long)f.bm_lo | ((unsigned long long)f.bm_hi << 32);
      const int px = lane & 15, x = px & 3, y = px >> 2;
      for (int b = 0; b < 16; b++) {
        const int bx = b & 3, by = b >> 2;
        const int mode = (int)((bm >> (4 * b)) & 15);
        const uint8_t* e0 = Wb + (4 * by) * WS + 15 + 4 * bx;  // = above[-1] of this sub-block
        const int sp = src[(4 * by + y) * 16 + 4 * bx + x];
        int v;
        if (mode == VP8GPU_B_DC_PRED) {
          int s4 = 4;
#pragma unroll
          for (int k = 0; k < 4; k++) s4 += e0[1 + k] + e0[(1 + k) * WS];
          v = s4 >> 3;
        } else if (mode == VP8GPU_B_TM_PRED) {
          v = vp8m::clamp255(e0[(1 + y) * WS] + e0[1 + x] - e0[0]);
        } else {
          const unsigned entry = s_lut[(mode - 2) * 16 + px];
          const int ia = entry & 15, ib = (entry >> 4) & 15, ic = (entry >> 8) & 15;
          const int pa = e0[ia < 4 ? (4 - ia) * WS : ia - 4];
          const int pb = e0[ib < 4 ? (4 - ib) * WS : ib - 4];
          const int pc = e0[ic < 4 ? (4 - ic) * WS : ic - 4];
          v = (entry & 0x1000) ? ((pa + 2 * pb + pc + 2) >> 2) : ((pa + pb + 1) >> 1);
        }
        const int pred = v;
        __syncwarp();
        if (lane < 16) S.tmp[lane] = (int16_t)(sp - pred);
        __syncwarp();
        if (lane == 0) {
          int16_t d[16], o[16];
#pragma unroll
          for (int k = 0; k < 16; k++) d[k] = S.tmp[k];
          vp8m::fdct16(d, o);
#pragma unroll
          for (int k = 0; k < 16; k++) {
            const int fq = k ? q.y_ac : q.y_dc;  // Y without Y2: the DC uses y_dc
            int qv = vp8m::quantize_trunc(o[k], fq);
            qv = qv > 2047 ? 2047 : (qv < -2047 ? -2047 : qv);
            S.qb[b][k] = (int16_t)qv;
            d[k] = (int16_t)(qv * fq);
          }
          vp8m::idct16(d, o);
#pragma unroll
          for (int k = 0; k < 16; k++) S.tmp[k] = o[k];
        }
        __syncwarp();
        if (lane < 16) Wb[(4 * by + y + 1) * WS + 16 + 4 * bx + x] = (uint8_t)vp8m::clamp255(pred + S.tmp[lane]);
        __syncwarp();
      }
    } else {
      // ---- 16x16 prediction with the frame's mode into the workspace (Block<16>::intra_predict) ----
      const int y = lane >> 1, x8 = (lane & 1) * 8;
      const int left = W[(y + 1) * WS + 15];
      uint32_t w0, w1;
      if (f.y_mode == VP8GPU_DC_PRED) {
        int s = 0, n = 0;
        if (row > 0) { for (int k = 0; k < 16; k++) s += A[k]; n += 16; }
        if (col > 0) { for (int k = 0; k < 16; k++) s += W[(k + 1) * WS + 15]; n += 16; }
        w0 = w1 = (uint32_t)(n == 32 ? (s + 16) >> 5 : (n == 16 ? (s + 8) >> 4 : 128)) * 0x01010101u;
      } else if (f.y_mode == VP8GPU_V_PRED) {
        w0 = (uint32_t)A[x8] | ((uint32_t)A[x8 + 1] << 8) | ((uint32_t)A[x8 + 2] << 16) | ((uint32_t)A[x8 + 3] << 24);
        w1 = (uint32_t)A[x8 + 4] | ((uint32_t)A[x8 + 5] << 8) | ((uint32_t)A[x8 + 6] << 16) | ((uint32_t)A[x8 + 7] << 24);
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
      __syncwarp();
      *reinterpret_cast<uint32_t*>(W + (y + 1) * WS + 16 + x8) = w0;
      *reinterpret_cast<uint32_t*>(W + (y + 1) * WS + 20 + x8) = w1;
    }
    // ---- chroma prediction with the frame's mode (Block<8>::intra_predict) ----
    {
      const int cplane = lane >> 4, cy = (lane >> 1) & 7, cx4 = (lane & 1) * 4;
      int cdc[2];
#pragma unroll
      for (int plane = 0; plane < 2; plane++) {
        int s = 0, n = 0;
        if (row > 0) { for (int k = 0; k < 8; k++) s += S.aboveC[plane][1 + k]; n += 8; }
        if (col > 0) { for (int k = 0; k < 8; k++) s += S.leftC[plane][k]; n += 8; }
        cdc[plane] = n == 16 ? (s + 8) >> 4 : (n == 8 ? (s + 4) >> 3 : 128);
      }
      const uint8_t* CA = S.aboveC[cplane] + 1;
      const int cl = S.leftC[cplane][cy], ccorner = CA[-1], cd = cplane ? cdc[1] : cdc[0];
      uint32_t word;
      if (f.uv_mode == VP8GPU_DC_PRED) word = (uint32_t)cd * 0x01010101u;
      else if (f.uv_mode == VP8GPU_V_PRED) word = (uint32_t)CA[cx4] | ((uint32_t)CA[cx4 + 1] << 8) | ((uint32_t)CA[cx4 + 2] << 16) | ((uint32_t)CA[cx4 + 3] << 24);
      else if (f.uv_mode == VP8GPU_H_PRED) word = (uint32_t)cl * 0x01010101u;
      else {
        const int base = cl - ccorner;
        word = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) word |= (uint32_t)vp8m::clamp255(base + CA[cx4 + k]) << (8 * k);
      }
      *reinterpret_cast<uint32_t*>(pixc + cplane * 64 + cy * 8 + cx4) = word;
    }
    __syncwarp();

    // ---- residual, transforms, tokens ----
    reenc_forward(
        src, [W](int y, int x) { return (int)W[(y + 1) * WS + 16 + x]; }, [pixc](int plane, int y, int x) { return (int)pixc[plane * 64 + y * 8 + x]; },
        coef, !bpred, !bpred, lane);
    uint32_t base;
    const int total = reenc_quantize_emit(coef, bpred ? S.qb : nullptr, !bpred, q, J.tok_counter, J.tok_cap, J.tokens, base, lane);

    // ---- reconstruct exactly like a decoder will ----
    if (bpred) {
      for (int i = lane; i < 64; i += 32) {
        const int y = i >> 2, x4 = (i & 3) * 4;
        *reinterpret_cast<uint32_t*>(W + (y + 1) * WS + 16 + x4) = *reinterpret_cast<const uint32_t*>(Wb + (y + 1) * WS + 16 + x4);
      }
      __syncwarp();
      if (total) {
        if (lane < 16) {  // the luma residual is already in the workspace: blank the (dequantised) luma blocks
          uint2* cv = reinterpret_cast<uint2*>(coef + lane * CS);
#pragma unroll
          for (int k = 0; k < 4; k++) cv[k] = make_uint2(0u, 0u);
        }
        __syncwarp();
        inverse_transforms(coef, false, lane);
        add_residuals_intra(W, pixc, coef, lane, false);
      }
    } else if (total) {
      inverse_transforms(coef, true, lane);
      add_residuals_intra(W, pixc, coef, lane, true);
    }
    if (lane < 16) {
      *reinterpret_cast<uint4*>(Y + (size_t)(16 * row + lane) * g.y_pitch + 16 * col) = *reinterpret_cast<const uint4*>(W + (lane + 1) * WS + 16);
    } else {
      const int plane = (lane - 16) >> 3, yy = lane & 7;
      *reinterpret_cast<uint2*>((plane ? V : U) + (size_t)(8 * row + yy) * g.c_pitch + 8 * col) = *reinterpret_cast<const uint2*>(pixc + plane * 64 + yy * 8);
    }
    if (lane == 0) {
      vp8gpu_mb m = J.mbs_in[mbi];
      m.tok_off = base;
      m.tok_cnt = (uint16_t)total;
      m.flags = bpred ? 0 : VP8GPU_MB_HAS_Y2;
      J.mbs_out[mbi] = m;
    }
    const int next = next_marked(my_word, col + 1, nwords);
    publish_row(progress, next < 0 ? cols : next, lane);
    col = next;
  }
}
