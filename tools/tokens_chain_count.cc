// Host build of the device token decoder (alfalfa_b200/csrc/tokens_core.cuh) that counts its arithmetic-coded
// decisions per frame, for tools/tokens_chain.py: parse_frame(defer_tokens) + decode_frame_tokens, as k_tokens<1>
// runs them, with TK_ON_DECISION counting every lr_decide.
#include <string.h>

#include <vector>

static unsigned long long g_decisions;
#define TK_ON_DECISION() (++g_decisions)

#include "../alfalfa_b200/csrc/parser.h"
#include "../alfalfa_b200/csrc/tokens_core.cuh"

struct Counter {
  vp8::State st;
  vp8::ParsedFrame pf;
  std::vector<vp8gpu_token> tokens;
  std::vector<uint16_t> above;
  Counter(int w, int h) : st(w, h) {}
};

extern "C" {
void* tc_new(int w, int h) { return new Counter(w, h); }
void tc_free(void* p) { delete static_cast<Counter*>(p); }
// decisions of one frame (out[0]) and its tokens (out[1]); returns the parser's code (0 = ok)
int tc_frame(void* p, const uint8_t* data, size_t len, unsigned long long* out) {
  Counter& C = *static_cast<Counter*>(p);
  const int rc = vp8::parse_frame(C.st, data, len, C.pf, true);
  if (rc != VP8GPU_OK) return rc;
  const vp8gpu_frame_desc& d = C.pf.desc;
  vp8::Geom g{};
  g.mb_cols = d.mb_cols;
  g.mb_rows = d.mb_rows;
  const size_t n_mbs = (size_t)d.mb_cols * d.mb_rows;
  C.tokens.assign(n_mbs * 400, 0);
  C.above.assign(g.mb_cols, 0);
  uint32_t result[2] = {0, 0};
  vp8::TokJob J{};
  J.mbs = C.pf.mbs.data();
  J.tokens = C.tokens.data();
  J.bits = C.pf.tw.bits;
  J.coef_probs = C.pf.tw.coef_probs;
  J.result = result;
  memcpy(J.part_off, C.pf.tw.part_off, sizeof(J.part_off));
  memcpy(J.part_len, C.pf.tw.part_len, sizeof(J.part_len));
  J.nparts = C.pf.tw.nparts;
  J.tok_cap = (uint32_t)(n_mbs * 400);
  alignas(16) uint8_t probs16[vp8::tok::kProbBytes];
  for (int e = 0; e < vp8::tok::kProbEntries; e++) vp8::tok::expand_prob_entry(C.pf.tw.coef_probs, probs16, e);
  g_decisions = 0;
  vp8::tok::decode_frame_tokens(J, g, probs16, C.above.data());
  out[0] = g_decisions;
  out[1] = result[0];
  return 0;
}
}
