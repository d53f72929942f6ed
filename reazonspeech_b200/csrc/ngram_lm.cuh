// The n-gram LM lookup shared by the greedy decode (decode_spec.cu) and the MAES beam search (decode_maes.cu): one lookup, so
// that both decoders add the same fp32 term for the same (state, token).  Tables: reazonspeech_b200/ngram_lm.py.
#pragma once
#include "kernels.h"

namespace rs {

// n-gram LM lookup of one state over vocabulary columns [j0, jn) (the greedy decode's slice, width rows_j <= 128; MAES: one
// token), by one warp: term[j - j0] = the LM term
// of token j, next[j - j0] = the state emitting it leads to.  The root row is written first; then the chain levels, lowest
// first, overwrite the tokens they have arcs for, so the highest level wins (a level's tokens are distinct: no lane conflicts).
// Each level's arc range is narrowed to <= 32 arcs around the first token >= j0 by 32-wide probe rounds, all levels in the
// same rounds; then 32-arc chunks are read from there until a token >= jn.  A state outside [0, n_states) counts as the root.
constexpr int kMaxLmCtx = 5;                 // LM order <= 6
constexpr int kNoTok = 0x7fffffff;
__device__ __forceinline__ void lm_fill_row(const NgramLM& lm, int s, int j0, int jn, float* term, int* next, int lane) {
  const int nctx = lm.order - 1;
  if (static_cast<unsigned int>(s) >= static_cast<unsigned int>(lm.n_states)) s = 0;
  const float cb = __ldg(lm.cb + s);
  const int o = lane < nctx ? __ldg(lm.chain + static_cast<size_t>(s) * nctx + lane) : 0;
  for (int j = j0 + lane; j < jn; j += 32) { term[j - j0] = cb + __ldg(lm.uni_w + j); next[j - j0] = __ldg(lm.uni_to + j); }
  int lo = 0, end = 0;
  if (o > 0) { lo = __ldg(lm.arc_begin + o); end = __ldg(lm.arc_begin + o + 1); }
  int L[kMaxLmCtx], H[kMaxLmCtx], E[kMaxLmCtx];    // level d (chain[s][d]): the first arc with token >= j0 lies in [L, H]
#pragma unroll
  for (int d = 0; d < kMaxLmCtx; ++d) { L[d] = __shfl_sync(0xffffffffu, lo, d); E[d] = __shfl_sync(0xffffffffu, end, d); H[d] = E[d]; }
  for (;;) {
    int v[kMaxLmCtx];
    bool more = false;
#pragma unroll
    for (int d = 0; d < kMaxLmCtx; ++d) {                    // the probes of every level first: independent loads
      v[d] = kNoTok;
      const int n = H[d] - L[d];
      if (n > 32) {
        more = true;
        const int step = (n + 31) >> 5, q = L[d] + lane * step + step - 1;
        if (q < H[d]) v[d] = __ldg(lm.arc_tok + q);
      }
    }
    if (!more) break;                                         // warp-uniform
#pragma unroll
    for (int d = 0; d < kMaxLmCtx; ++d) {
      const int n = H[d] - L[d];
      if (n > 32) {
        const int step = (n + 31) >> 5, c = __popc(__ballot_sync(0xffffffffu, v[d] < j0));
        L[d] += c * step;
        H[d] = min(L[d] + step - 1, H[d]);
      }
    }
  }
  int t0[kMaxLmCtx], n0[kMaxLmCtx];
  float w0[kMaxLmCtx];
#pragma unroll
  for (int d = 0; d < kMaxLmCtx; ++d) {                      // first chunk of every level
    const int i = L[d] + lane;
    const bool ok = i < E[d];
    t0[d] = ok ? __ldg(lm.arc_tok + i) : kNoTok;
    w0[d] = ok ? __ldg(lm.arc_w + i) : 0.f;
    n0[d] = ok ? __ldg(lm.arc_to + i) : 0;
  }
  __syncwarp();                                               // the root row is written before any overwrite
#pragma unroll
  for (int d = kMaxLmCtx - 1; d >= 0; --d) {
    int t = t0[d], nx = n0[d];
    float w = w0[d];
    for (int base = L[d];; base += 32) {
      if (t >= j0 && t < jn) { term[t - j0] = cb + w; next[t - j0] = nx; }
      if (!(__shfl_sync(0xffffffffu, t, 31) < jn && base + 32 < E[d])) break;
      const int i = base + 32 + lane;
      const bool ok = i < E[d];
      t = ok ? __ldg(lm.arc_tok + i) : kNoTok;
      w = ok ? __ldg(lm.arc_w + i) : 0.f;
      nx = ok ? __ldg(lm.arc_to + i) : 0;
    }
    __syncwarp();
  }
}

}  // namespace rs
