// tokens_core.cuh -- the device-side token decoder's logic (see tokens.cu), written so that it also
// compiles as plain host C++: tests/test_tokens_host.py runs exactly this code on the CPU against
// the CPU front end (csrc/parser.cc) on every golden vector before it ever sees a GPU.
//
// What the code is shaped by: one thread walks one frame, so everything is latency.  The decoder
// state lives in registers (nothing here takes its address), and the eleven probabilities of a
// (block type, band, context) position are fetched with ONE 16-byte shared-memory load per token
// instead of one byte load per decision.
#pragma once
#include <stdint.h>

#include "engine.h"

#ifdef __CUDACC__
#define TK_DEV __device__ __forceinline__
#define TK_CONST __constant__
#define TK_LDG(p) __ldg(p)
#define TK_LDCG(p) __ldcg(p)
#define TK_CLZ(x) __clz(x)
#else
#define TK_DEV inline __attribute__((always_inline))
#define TK_CONST static const
#define TK_LDG(p) (*(p))
#define TK_LDCG(p) (*(p))
#define TK_CLZ(x) __builtin_clz(x)
#endif

namespace vp8 {
namespace tok {

// coefficient bands (tokens.hh:59-60)
TK_CONST uint8_t c_band[16] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7};
TK_CONST uint8_t c_zigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
// extra-bit probabilities of DCT_CAT2..6 (tokens.hh:74-78), rows padded to 11
TK_CONST uint8_t c_cat[5][11] = {{165, 145},
                                 {173, 148, 140},
                                 {176, 155, 140, 135},
                                 {180, 157, 141, 134, 130},
                                 {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129}};

// Probability table as the decoder wants it: [type 4][band 8][ctx 3] entries of 16 bytes (11 used).
constexpr int kProbEntries = 4 * 8 * 3;
constexpr int kProbBytes = kProbEntries * 16;
struct alignas(16) Probs16 {
  uint32_t w[4];
  TK_DEV uint32_t at(int k) const { return (w[k >> 2] >> ((k & 3) * 8)) & 0xFF; }
};
// entry e of the 16-byte layout from the 1056-byte table of the frame header (type, band, ctx, node)
TK_DEV void expand_prob_entry(const uint8_t* src, uint8_t* dst, int e) {
  for (int k = 0; k < 11; k++) dst[e * 16 + k] = src[e * 11 + k];
  for (int k = 11; k < 16; k++) dst[e * 16 + k] = 0;
}

// ---- bit reader ----------------------------------------------------------------------------------
// Bit-for-bit the decisions of csrc/parser.cc's BoolReader (and therefore bool_decoder.hh:82-107): past
// the end of the partition only zero bits arrive.  A decode never waits for memory: the stream is fetched
// as aligned 32-bit words ONE REFILL AHEAD (`nxt` is requested when the previous word is consumed, ~30
// decisions before it is needed).  The window is 64 bits, consumed from the top, with `nbits` valid bits
// (the rest zero); it is kept as two words, `hi` and `lo`, because a decision compares and subtracts in
// `hi` alone and normalising is one funnel shift of (hi, lo).  The range is kept as range << 16, so that
// one multiply-add gives the split already in the top byte (lr_decide).  Plain struct, always handled by
// value / reference to a local: stays in registers.
#ifdef __CUDACC__
#define TK_BSWAP(x) __byte_perm((x), 0, 0x0123)
#define TK_FUNNEL_L(lo, hi, s) __funnelshift_l((lo), (hi), (s))
#else
#define TK_BSWAP(x) __builtin_bswap32(x)
#define TK_FUNNEL_L(lo, hi, s) static_cast<uint32_t>(((static_cast<uint64_t>(hi) << 32) | (lo)) << (s) >> 32)
#endif
struct LaneReader {
  const uint8_t* p;    // next word to request (4-byte aligned)
  const uint8_t* end;
  uint32_t hi, lo;     // the window: hi = its top 32 bits
  int nbits;
  uint32_t nxt;        // the next 32 bits of the stream, most significant bit first
  uint32_t rng16;      // range << 16, range in [128, 255] between decisions
};
TK_DEV uint32_t lr_fetch(LaneReader& b) {
  uint32_t w = 0;
  if (b.p + 4 <= b.end) {
    w = TK_BSWAP(TK_LDG(reinterpret_cast<const uint32_t*>(b.p)));
  } else {
    for (int k = 0; k < 4; k++)
      if (b.p + k < b.end) w |= static_cast<uint32_t>(TK_LDG(b.p + k)) << (24 - 8 * k);
  }
  b.p += 4;
  return w;
}
TK_DEV void lr_refill(LaneReader& b) {  // nbits <= 32 on entry, so lo == 0
  const uint64_t v = (static_cast<uint64_t>(b.nxt) << 32) >> b.nbits;
  b.hi |= static_cast<uint32_t>(v >> 32);
  b.lo = static_cast<uint32_t>(v);
  b.nbits += 32;
  b.nxt = lr_fetch(b);
}
TK_DEV void lr_init(LaneReader& b, const uint8_t* data, uint32_t n) {
  b.p = data;
  b.end = data + n;
  uint64_t value = 0;
  b.nbits = 0;
  b.rng16 = 255u << 16;
  while ((reinterpret_cast<uintptr_t>(b.p) & 3) && b.p < b.end) {  // up to three bytes to reach a word boundary
    value |= static_cast<uint64_t>(TK_LDG(b.p++)) << (56 - b.nbits);
    b.nbits += 8;
  }
  b.hi = static_cast<uint32_t>(value >> 32);
  b.lo = static_cast<uint32_t>(value);
  if (b.p >= b.end) b.p = reinterpret_cast<const uint8_t*>((reinterpret_cast<uintptr_t>(b.p) + 3) & ~static_cast<uintptr_t>(3));
  b.nxt = lr_fetch(b);
  lr_refill(b);
  if (b.nbits <= 32) lr_refill(b);
}
// One decision, without a refill test: the 8 compared bits must be valid (nbits >= 8), and the window
// shifts by at most 7.  With M = 0xFFFFFF and t = rng16 * prob + ((256 - prob) << 16), the top byte of t is
// split = 1 + (((range - 1) * prob) >> 8) and t's low 24 bits are below 2^24, so
//   hi >= split << 24          <=>  (hi | M) >= t
//   (range - split) << 24      ==   ((rng16 << 8 | M) - t) & ~M
// and what depends on the previous decision is a multiply-add, a compare, a select, FLO and a shift.  The low
// 24 bits of the selected range do not change its leading zeros; they are dropped before it is shifted.
#ifndef TK_ON_DECISION
#define TK_ON_DECISION()  // host-only hook: tools/tokens_chain_count.cc counts decisions with it
#endif
TK_DEV int lr_decide(LaneReader& b, uint32_t prob) {
  TK_ON_DECISION();
  const uint32_t M = 0xFFFFFFu;
  const uint32_t t = b.rng16 * prob + ((256u - prob) << 16);
  const int bit = (b.hi | M) >= t;
  const uint32_t r = bit ? ((b.rng16 << 8) | M) - t : t;  // (new range << 24) + bits below 2^24
  const uint32_t h = bit ? b.hi - (t & ~M) : b.hi;
#ifdef __CUDACC__
  int shift;  // leading zeros of r (r != 0): FLO.SH gives them directly, __clz adds a subtraction from 31
  asm("bfind.shiftamt.u32 %0, %1;" : "=r"(shift) : "r"(r));
  const uint32_t r16 = __byte_perm(r, 0, 0x4344);  // (r >> 24) << 16
#else
  const int shift = TK_CLZ(r);
  const uint32_t r16 = (r >> 24) << 16;
#endif
  b.rng16 = r16 << shift;
  b.hi = TK_FUNNEL_L(b.lo, h, shift);
  b.lo <<= shift;
  b.nbits -= shift;
  return bit;
}
// Afterwards nbits >= 33: enough for the next FOUR decisions (33 - 3 * 7 >= 8).
TK_DEV void lr_ensure(LaneReader& b) {
  if (b.nbits <= 32) lr_refill(b);
}
// A decision that keeps the window at >= 33 valid bits itself (the lock-step decoder, one decision per step).
TK_DEV int lr_get(LaneReader& b, uint32_t prob) {
  const int bit = lr_decide(b, prob);
  lr_ensure(b);
  return bit;
}

// ---- one thread walks one frame ------------------------------------------------------------------
// Everything here is one dependent chain, so the per-decision work is lr_decide alone: the refill test is
// made once per group of at most four decisions (lr_ensure at the start of a token, after p[2] for the
// larger tokens, before every extra bit and before the sign of a DCT_CAT token), and the probability entry of
// the next coefficient position is loaded as soon as its context is known (after p[2]), while the rest of the
// token is decoded.  c_band as nibbles in a register: the entry's address costs no constant-memory load.
constexpr uint64_t kBandNibbles = 0x7666666665463210ull;  // c_band[i] = nibble i
TK_DEV uint32_t band_off(int i) {  // byte offset of (band of position i & 15, ctx 0) in a block type's entries
  return static_cast<uint32_t>((kBandNibbles >> (4 * (i & 15))) & 15) * 48;
}
// The probability table is addressed by its 32-bit shared-memory offset on the device (ProbAddr): the address
// of an entry is then one integer add, not a generic pointer the compiler rebuilds from the CTA's shared
// window (an S2R on the chain).  The load is volatile asm, so that it is issued where the source puts it --
// ahead of the decision that selects its result -- and not sunk into the branch that uses it, where the next
// decision would wait for it.
#ifdef __CUDACC__
typedef uint32_t ProbAddr;
TK_DEV ProbAddr prob_addr(const uint8_t* p) {
  // through an opaque move: the compiler would otherwise rebuild the address from SR_CgaCtaId at every use
  uint32_t a;
  asm volatile("mov.u32 %0, %1;" : "=r"(a) : "r"(static_cast<uint32_t>(__cvta_generic_to_shared(p))));
  return a;
}
TK_DEV Probs16 ld_probs(ProbAddr a) {
  Probs16 P;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(P.w[0]), "=r"(P.w[1]), "=r"(P.w[2]), "=r"(P.w[3]) : "r"(a));
  return P;
}
#else
typedef const uint8_t* ProbAddr;
TK_DEV ProbAddr prob_addr(const uint8_t* p) { return p; }
TK_DEV Probs16 ld_probs(ProbAddr p) { return *reinterpret_cast<const Probs16*>(p); }
#endif

// One 4x4 block (tokens.cc:50-135).  tp = 16-byte probability entries of the block type,
// i = first coefficient, tag = block number << 20.  Returns has_nonzero.
TK_DEV int parse_block(LaneReader& br, ProbAddr tp, int ctx, int i, uint32_t tag, vp8gpu_token*& out) {
  lr_ensure(br);
  Probs16 P = ld_probs(tp + band_off(i) + ctx * 16);
  if (!lr_decide(br, P.at(0))) return 0;
  int nz = 0;
  for (;;) {
    // group of decisions: p[1], p[2] and, for a ONE token, its sign and the next p[0]
    const uint32_t next = band_off(i + 1);      // position i + 1 (unused when i == 15)
    const Probs16 Pz = ld_probs(tp + next);      // its entry after a ZERO token (ctx 0)
    lr_ensure(br);
    if (!lr_decide(br, P.at(1))) {  // zero token: no end-of-block test after a zero
      if (++i == 16) return nz;
      P = Pz;
      continue;
    }
    int v;
    Probs16 Pn;
    if (!lr_decide(br, P.at(2))) {
      Pn = ld_probs(tp + next + 16);  // ctx 1
      v = 1;
    } else {
      Pn = ld_probs(tp + next + 32);  // ctx 2
      lr_ensure(br);  // the tree below p[2]: at most four decisions
      if (!lr_decide(br, P.at(3))) {
        if (!lr_decide(br, P.at(4))) v = 2;
        else v = 3 + lr_decide(br, P.at(5));
      } else {
        int cat, n, base;
        if (!lr_decide(br, P.at(6))) {
          if (!lr_decide(br, P.at(7))) {
            cat = 0, n = 0, base = 5 + lr_decide(br, 159);
          } else {
            cat = 0, n = 2, base = 7;
          }
        } else if (!lr_decide(br, P.at(8))) {
          if (!lr_decide(br, P.at(9))) cat = 1, n = 3, base = 11;
          else cat = 2, n = 4, base = 19;
        } else {
          if (!lr_decide(br, P.at(10))) cat = 3, n = 5, base = 35;
          else cat = 4, n = 11, base = 67;
        }
        int inc = 0;
        for (int k = 0; k < n; k++) {
          lr_ensure(br);
          inc = (inc << 1) + lr_decide(br, c_cat[cat][k]);
        }
        v = base + inc;
      }
      lr_ensure(br);  // sign and the next p[0]
    }
    if (lr_decide(br, 128)) v = -v;
    *out++ = tag | (static_cast<uint32_t>(c_zigzag[i]) << 16) | static_cast<uint16_t>(v);
    nz = 1;
    if (++i == 16) return 1;
    P = Pn;
    if (!lr_decide(br, P.at(0))) return 1;
  }
}

// One frame, raster order (Frame::parse_tokens, frame.cc:122-137 + Macroblock::parse_tokens,
// macroblock.cc:468-502).  probs: the frame's coefficient probabilities in the 16-byte layout
// (kProbBytes, 16-byte aligned); above_nz: mb_cols zeroed words (Y0-3 | U << 4 | V << 6 | Y2 << 8
// per column).  On the device both live in shared memory.
TK_DEV void decode_frame_tokens(const TokJob& J, const Geom& g, const uint8_t* probs, uint16_t* above_nz) {
  LaneReader parts[8];
  const int nparts = static_cast<int>(J.nparts);
  for (int i = 0; i < nparts; i++) lr_init(parts[i], J.bits + J.part_off[i], J.part_len[i]);

  vp8gpu_mb* const mbs = J.mbs;
  vp8gpu_token* const t_begin = J.tokens;
  vp8gpu_token* t = t_begin;
  const vp8gpu_token* const t_limit = t_begin + J.tok_cap;
  uint32_t overflow = 0;
  const ProbAddr coef_y_after_y2 = prob_addr(probs);
  const ProbAddr coef_y2 = coef_y_after_y2 + 1 * 384;
  const ProbAddr coef_uv = coef_y_after_y2 + 2 * 384;
  const ProbAddr coef_y_full = coef_y_after_y2 + 3 * 384;

  // word 1 of a record = tok_cnt | y_mode << 16 | uv_mode << 24, word 2 = ref | segment | lf | flags << 24
  const uint32_t* rec = reinterpret_cast<const uint32_t*>(mbs);
  uint32_t w1 = TK_LDCG(rec + 1), w2 = TK_LDCG(rec + 2);
  const int n_mbs = g.mb_cols * g.mb_rows;
  int idx = 0;
  for (int row = 0; row < g.mb_rows; row++) {
    unsigned left_nz = 0;
    LaneReader tr = parts[row & (nparts - 1)];  // row r -> partition r % n (frame.cc:131-136)
    for (int col = 0; col < g.mb_cols; col++, idx++) {
      const uint32_t cur1 = w1, cur2 = w2;
      if (idx + 1 < n_mbs) {  // next record: requested now, needed after this macroblock's tokens
        w1 = TK_LDCG(rec + 8 * (idx + 1) + 1);
        w2 = TK_LDCG(rec + 8 * (idx + 1) + 2);
      }
      const int y_mode = (cur1 >> 16) & 0xFF;
      const bool skip = (cur2 >> 24) & VP8GPU_MB_SKIP;
      const bool has_y2 = y_mode != VP8GPU_B_PRED && y_mode != VP8GPU_SPLITMV;
      unsigned a_nz = above_nz[col];
      vp8gpu_token* const t0 = t;
      if (skip) {
        // frame.cc:252-269: a macroblock without Y2 leaves the previous Y2 context in place
        const unsigned keep = has_y2 ? 0u : 0x100u;
        a_nz &= keep;
        left_nz &= keep;
      } else if (t + 400 > t_limit) {
        overflow = 1;  // cannot happen with the capacity rule of the host (engine.cu); stay in bounds
        a_nz = 0;
        left_nz = 0;
      } else {
        ProbAddr y_probs = coef_y_full;
        int first = 0;
        if (has_y2) {
          const int ctx = ((a_nz >> 8) & 1) + ((left_nz >> 8) & 1);
          const unsigned nz = parse_block(tr, coef_y2, ctx, 0, VP8GPU_BLK_Y2 << 20, t);
          a_nz = (a_nz & ~0x100u) | (nz << 8);
          left_nz = (left_nz & ~0x100u) | (nz << 8);
          y_probs = coef_y_after_y2;
          first = 1;
        }
        // 16 luma blocks, then U and V: block b uses context bits (bx, by) of the above / left words
#pragma unroll 1
        for (int b = 0; b < 24; b++) {
          int bx, by;
          ProbAddr tp;
          int f;
          if (b < 16) {
            bx = b & 3, by = b >> 2, tp = y_probs, f = first;
          } else {
            const int sh = 4 + 2 * ((b - 16) >> 2);
            bx = sh + (b & 1), by = sh + ((b >> 1) & 1), tp = coef_uv, f = 0;
          }
          const int ctx = ((a_nz >> bx) & 1) + ((left_nz >> by) & 1);
          const unsigned nz = parse_block(tr, tp, ctx, f, static_cast<uint32_t>(b) << 20, t);
          a_nz = (a_nz & ~(1u << bx)) | (nz << bx);
          left_nz = (left_nz & ~(1u << by)) | (nz << by);
        }
      }
      above_nz[col] = static_cast<uint16_t>(a_nz);
      uint32_t* wr = reinterpret_cast<uint32_t*>(mbs) + 8 * idx;
      wr[0] = static_cast<uint32_t>(t0 - t_begin);
      wr[1] = (cur1 & 0xFFFF0000u) | static_cast<uint32_t>(t - t0);
      wr[2] = cur2 & ~(static_cast<uint32_t>(VP8GPU_MB_SKIP) << 24);
    }
    parts[row & (nparts - 1)] = tr;
  }
  J.result[0] = static_cast<uint32_t>(t - t_begin);
  // sticky: a slot's result words serve all the frames staged in it, and the host reads the flag once for all of them
  if (overflow) J.result[1] = 1;
}


// ------------------------------------------------------------------------------------------------
// The same decoder as a state machine that consumes exactly ONE arithmetic-coded decision per loop
// iteration, so that the 32 lanes of a warp can each walk their OWN frame in lock-step: the expensive
// part of an iteration (probability fetch + bool decode) is the same instruction stream for every
// lane whatever token-tree node it is at, the transition is table driven, and only the rarer block /
// macroblock boundaries diverge.  One thread per frame (above) spends a whole warp instruction on one
// lane's decision; this form spends it on 32.
//   node 0..10 = tree node reading probability p[node] (tokens.cc:50-135), 11 = extra bits of a
//   DCT_CAT token, 12 = sign, 13 = block finished.
// ------------------------------------------------------------------------------------------------
constexpr int kNodeExtra = 11, kNodeSign = 12, kNodeEnd = 13;
// transition on (node, bit): next node | magnitude << 4 | zero-token << 8 | category << 9
#define TK_T(next, setv, zero, cat) static_cast<uint16_t>((next) | ((setv) << 4) | ((zero) << 8) | ((cat) << 9))
TK_CONST uint16_t c_trans[22] = {
    TK_T(kNodeEnd, 0, 0, 0),  TK_T(1, 0, 0, 0),           // p[0]: end of block?
    TK_T(1, 0, 1, 0),         TK_T(2, 0, 0, 0),           // p[1]: zero token?  (no end-of-block test after it)
    TK_T(kNodeSign, 1, 0, 0), TK_T(3, 0, 0, 0),           // p[2]: one?
    TK_T(4, 0, 0, 0),         TK_T(6, 0, 0, 0),           // p[3]
    TK_T(kNodeSign, 2, 0, 0), TK_T(5, 0, 0, 0),           // p[4]: two?
    TK_T(kNodeSign, 3, 0, 0), TK_T(kNodeSign, 4, 0, 0),   // p[5]: three / four
    TK_T(7, 0, 0, 0),         TK_T(8, 0, 0, 0),           // p[6]
    TK_T(kNodeExtra, 0, 0, 1), TK_T(kNodeExtra, 0, 0, 2), // p[7]: DCT_CAT1 / 2
    TK_T(9, 0, 0, 0),         TK_T(10, 0, 0, 0),          // p[8]
    TK_T(kNodeExtra, 0, 0, 3), TK_T(kNodeExtra, 0, 0, 4), // p[9]: DCT_CAT3 / 4
    TK_T(kNodeExtra, 0, 0, 5), TK_T(kNodeExtra, 0, 0, 6), // p[10]: DCT_CAT5 / 6
};
#undef TK_T
// categories 1..6: base value, number of extra bits, their probabilities (tokens.hh:74-78)
TK_CONST uint8_t c_cat_base[7] = {0, 5, 7, 11, 19, 35, 67};
TK_CONST uint8_t c_cat_bits[7] = {0, 1, 2, 3, 4, 5, 11};
TK_CONST uint8_t c_cat_prob[7][11] = {{0},
                                      {159},
                                      {165, 145},
                                      {173, 148, 140},
                                      {176, 155, 140, 135},
                                      {180, 157, 141, 134, 130},
                                      {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129}};

// The small tables above, gathered: lanes index them with different values, which constant memory
// serialises -- the kernel keeps one copy per CTA in shared memory.
struct LockstepTables {
  uint16_t trans[22];
  uint8_t band[16], zigzag[16], cat_base[8], cat_bits[8], cat_prob[7][11];
};
TK_DEV void fill_lockstep_tables(LockstepTables& T, int lane, int nlanes) {
  for (int k = lane; k < 22; k += nlanes) T.trans[k] = c_trans[k];
  for (int k = lane; k < 16; k += nlanes) {
    T.band[k] = c_band[k];
    T.zigzag[k] = c_zigzag[k];
  }
  for (int k = lane; k < 7; k += nlanes) {
    T.cat_base[k] = c_cat_base[k];
    T.cat_bits[k] = c_cat_bits[k];
    for (int j = 0; j < 11; j++) T.cat_prob[k][j] = c_cat_prob[k][j];
  }
}

// The lock-step decoder reads its partitions with the LaneReader above, one lr_get per step: in lock-step a
// lane that waited for memory would stall the other 31.

// One lane = one frame.  P = this lane's column of the transposed probability table ([1056 entries][LS
// lanes] bytes: entry e of this frame at P[e * LS]), above = this lane's column of the transposed row of
// contexts ([mb_cols][LS] words); on the device both live in shared memory, LS = 32.  J.mbinfo = 2 bits
// per macroblock (flags & 3: VP8GPU_MB_HAS_Y2 | VP8GPU_MB_SKIP), 16 macroblocks per word, read one word
// ahead: the decoder never waits for a record.  Records get tok_off / tok_cnt / flags by plain stores.
template <int LS>
TK_DEV void decode_frame_tokens_lockstep(const TokJob& J, const Geom& g, const LockstepTables& T, const uint8_t* P,
                                         uint16_t* above) {
  for (int c = 0; c < g.mb_cols; c++) above[c * LS] = 0;
  LaneReader parts[8];
  const int nparts = static_cast<int>(J.nparts);
  for (int k = 0; k < nparts; k++) lr_init(parts[k], J.bits + J.part_off[k], J.part_len[k]);
  uint8_t* const mbs = reinterpret_cast<uint8_t*>(J.mbs);
  vp8gpu_token* const t_begin = J.tokens;
  vp8gpu_token* t = t_begin;
  vp8gpu_token* t0 = t_begin;
  const vp8gpu_token* const t_limit = t_begin + J.tok_cap;
  uint32_t overflow = 0;
  const int n_mbs = g.mb_cols * g.mb_rows;
  const int n_words = (n_mbs + 15) >> 4;
  uint32_t info = n_words > 0 ? TK_LDG(J.mbinfo) : 0u, info_next = n_words > 1 ? TK_LDG(J.mbinfo + 1) : 0u;

  LaneReader tr = parts[0];
  int idx = 0, col = 0, row = 0;
  unsigned a_nz = 0, left_nz = 0;
  int bq = 0, last_y_type = 0, first_y = 0;  // current block: -1 = Y2, 0..15 Y, 16..23 U V
  int has_y2_cur = 0;
  int type_off = 0, bx = 0, by = 0;
  int i = 0, ctx = 0, node = kNodeEnd, nz = 0;
  int v = 0, acc = 0, cat = 0, nrem = 0, extra_k = 0;
  bool need_mb = true;  // the next thing to do is to start macroblock idx
  bool done = n_mbs == 0;

  while (!done) {
    // ---- boundaries (divergent, comparatively rare): finish a block, finish / start macroblocks ----
    if (node == kNodeEnd) {
      if (!need_mb) {  // a block has just ended
        a_nz = (a_nz & ~(1u << bx)) | (static_cast<unsigned>(nz) << bx);
        left_nz = (left_nz & ~(1u << by)) | (static_cast<unsigned>(nz) << by);
        bq++;
        if (bq == 24) {  // macroblock finished
          above[col * LS] = static_cast<uint16_t>(a_nz);
          uint8_t* rec = mbs + 32 * static_cast<size_t>(idx);
          *reinterpret_cast<uint32_t*>(rec) = static_cast<uint32_t>(t0 - t_begin);
          *reinterpret_cast<uint16_t*>(rec + 4) = static_cast<uint16_t>(t - t0);
          rec[11] = static_cast<uint8_t>(has_y2_cur ? VP8GPU_MB_HAS_Y2 : 0);
          idx++;
          col++;
          need_mb = true;
        }
      }
      // start macroblocks until one has blocks to decode (skipped ones are settled on the spot)
      while (need_mb && !done) {
        if (idx == n_mbs) {
          done = true;
          break;
        }
        if (col == g.mb_cols) {  // next row: its partition is row % n (frame.cc:131-136)
          parts[row & (nparts - 1)] = tr;
          row++;
          col = 0;
          left_nz = 0;
          tr = parts[row & (nparts - 1)];
        }
        const unsigned bits2 = (info >> (2 * (idx & 15))) & 3u;
        if ((idx & 15) == 15) {  // last macroblock of this word: move on, request the word after the next
          info = info_next;
          const int nw = (idx >> 4) + 2;
          info_next = nw < n_words ? TK_LDG(J.mbinfo + nw) : 0u;
        }
        const bool skip = (bits2 & VP8GPU_MB_SKIP) != 0;
        const bool has_y2 = (bits2 & VP8GPU_MB_HAS_Y2) != 0;
        has_y2_cur = has_y2;
        a_nz = above[col * LS];
        t0 = t;
        bool settled = false;
        if (skip) {  // frame.cc:252-269: without Y2 the previous Y2 context stays
          const unsigned keep = has_y2 ? 0u : 0x100u;
          a_nz &= keep;
          left_nz &= keep;
          settled = true;
        } else if (t + 400 > t_limit) {
          overflow = 1;
          a_nz = 0;
          left_nz = 0;
          settled = true;
        }
        if (settled) {
          above[col * LS] = static_cast<uint16_t>(a_nz);
          uint8_t* rec = mbs + 32 * static_cast<size_t>(idx);
          *reinterpret_cast<uint32_t*>(rec) = static_cast<uint32_t>(t0 - t_begin);
          *reinterpret_cast<uint16_t*>(rec + 4) = 0;
          rec[11] = static_cast<uint8_t>(has_y2 ? VP8GPU_MB_HAS_Y2 : 0);
          idx++;
          col++;
          continue;
        }
        need_mb = false;
        bq = has_y2 ? -1 : 0;
        last_y_type = has_y2 ? 0 : 3;  // Y after Y2 / Y with DC
        first_y = has_y2 ? 1 : 0;
      }
      if (done) break;
      // set the block up: type, context bits, first coefficient
      if (bq < 0) {
        type_off = 1 * 264, bx = 8, by = 8, i = 0;
      } else if (bq < 16) {
        type_off = last_y_type * 264, bx = bq & 3, by = bq >> 2, i = first_y;
      } else {
        const int sh = 4 + 2 * ((bq - 16) >> 2);
        type_off = 2 * 264, bx = sh + (bq & 1), by = sh + ((bq >> 1) & 1), i = 0;
      }
      ctx = ((a_nz >> bx) & 1) + ((left_nz >> by) & 1);
      node = 0;
      nz = 0;
    }

    // ---- one decision (the same code for every lane) ----
    const int tree_node = node <= 10 ? node : 0;
    const uint32_t p_tree = P[(type_off + T.band[i & 15] * 33 + ctx * 11 + tree_node) * LS];
    const uint32_t p_extra = T.cat_prob[cat][extra_k];
    const uint32_t prob = node <= 10 ? p_tree : (node == kNodeExtra ? p_extra : 128u);
    const int bit = lr_get(tr, prob);

    // ---- transition ----
    if (node <= 10) {
      const uint32_t e = T.trans[node * 2 + bit];
      node = e & 15;
      const int setv = (e >> 4) & 15;
      v = setv ? setv : v;
      if ((e >> 8) & 1) {  // zero token
        i++;
        ctx = 0;
        if (i == 16) node = kNodeEnd;
      }
      const int c = (e >> 9) & 7;
      if (c) {
        cat = c;
        nrem = T.cat_bits[c];
        acc = 0;
        extra_k = 0;
      }
    } else if (node == kNodeExtra) {
      acc = (acc << 1) + bit;
      extra_k++;
      if (--nrem == 0) {
        v = T.cat_base[cat] + acc;
        extra_k = 0;
        node = kNodeSign;
      }
    } else {  // sign: the token is complete
      const int sv = bit ? -v : v;
      const int blk = bq < 0 ? VP8GPU_BLK_Y2 : bq;
      *t++ = (static_cast<uint32_t>(blk) << 20) | (static_cast<uint32_t>(T.zigzag[i]) << 16) | static_cast<uint16_t>(sv);
      nz = 1;
      ctx = v == 1 ? 1 : 2;
      i++;
      node = i == 16 ? kNodeEnd : 0;
    }
  }
  J.result[0] = static_cast<uint32_t>(t - t_begin);
  if (overflow) J.result[1] = 1;  // sticky, as in decode_frame_tokens
}

}  // namespace tok
}  // namespace vp8
