// MAES beam search (modified adaptive expansion search, Kim et al. 2020) for the RNN-T head, batched over utterances: NeMo's
// BeamRNNTInfer.modified_adaptive_expansion_search, the transducer beam search NeMo fuses an n-gram LM into.  Semantics restated in
// oracle/maes_restated.py.
//
// The search is frame-synchronous: every utterance advances one encoder frame per host iteration (utterances past their length
// are frozen).  A frame is
//
//   maes_prefix_rows_kernel  kept hypothesis k, depth d < P: relu(enc_proj[b, t] + dec_out_k[-1 - d]) -> three bf16 planes
//   [GEMM]                   logits = planes . [W_out x3]^T + b_out
//   maes_reduce_kernel       log-sum-exp; for d = 0 also the C = beam + beta best of all V + 1 classes (the shared beam_row_reduce)
//   maes_prefix_kernel       per utterance: kept sorted by length (longest first, stable), NeMo's prefix_search
//   num_steps rounds of
//     maes_expand_kernel     per utterance: select_k_expansions (gamma filter, ascending order), blanks -> list_b, tokens whose
//                            sequence is not a kept one (64-bit sequence hash + length) -> list_exp with their LM term; the rows
//                            of list_exp are compacted over the batch (one atomicAdd per utterance) and the host reads the count
//     maes_lstm_in / [GEMM] / maes_cell / [GEMM]    predictor of the new rows (h, c and joint.pred)
//     maes_rows / [GEMM] / maes_reduce              their joint: top-C for the next round, log p(blank) after the last one
//   maes_select_kernel       per utterance: recombine(list_b + list_exp) (first occurrence takes the logaddexp of its duplicates),
//                            the beam best by score (stable), back-pointer nodes for the tokens of this frame of each kept one
//   maes_gather_kernel       predictor state (h, c, the last P dec_out) of the new kept hypotheses
//
// As in ALSD (decode_alsd.cu) the matrix products run on the wgmma GEMM with activations split into three bf16 terms against
// bf16-exact weights: fp32-accurate log-probabilities.  Scores are doubles, log-probabilities fp32.
#include <cfloat>

#include "beam_common.cuh"
#include "common.cuh"
#include "kernels.h"
#include "maes.h"
#include "ngram_lm.cuh"

namespace rs {

namespace {

constexpr unsigned long long kHashSeed = 1469598103934665603ull;
__device__ __forceinline__ unsigned long long hash_push(unsigned long long h, int tok) { return h * 1000003ull + static_cast<unsigned long long>(tok + 1); }

// A hypothesis of this frame: round -1 is a kept slot, round n >= 0 a row of expansion round n
struct Src { const double* score; const unsigned long long* hh; const int* th; const int* u; const int* lm; const float* h; const float* c; const float* pp; size_t pp_plane; };
__device__ __forceinline__ Src src_of(const MaesState& st, int round) {
  if (round < 0) return {st.cur.score, st.cur.hh, st.cur.th, st.cur.u, st.cur.lm, st.cur.h, st.cur.c, st.cur.pp, static_cast<size_t>(st.B) * st.K};
  const MaesRows& r = st.rows[round];
  return {r.score, r.hh, r.th, r.u, r.lm, r.h, r.c, r.pp, static_cast<size_t>(r.cap)};
}

__device__ __forceinline__ void write_planes3(__nv_bfloat16* row, int stride, int j, float x) {
  __nv_bfloat16 hi, mid, lo;
  split3(x, hi, mid, lo);
  row[j] = hi; row[stride + j] = mid; row[2 * stride + j] = lo;
}

// ---------------------------------------------------------------------------------------------- start
// grid (B), block 32: the start hypothesis [blank] of every utterance as row b of round 0 (parent: the zero state), the root node
__global__ void maes_init_kernel(const MaesState st, int blank, int lm_start) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  const MaesRows& r = st.rows[0];
  r.tok[b] = blank; r.par[b] = -1; r.utt[b] = b;
  st.cur.n_hyp[b] = 1;
  const int s = b * st.K;
  st.cur.score[s] = 0.0; st.cur.u[s] = 0; st.cur.node[s] = 0; st.cur.lm[s] = lm_start;
  for (int d = 0; d <= st.P; ++d) st.cur.hh[static_cast<size_t>(s) * (st.P + 1) + d] = kHashSeed;
  st.n_nodes[b] = 1;
  const size_t tree = static_cast<size_t>(b) * st.max_nodes;
  st.node_parent[tree] = -1; st.node_tok[tree] = blank; st.node_frame[tree] = -1;
}

// grid (B), block 128: the predictor state of the start (row b of round 0) into kept slot b * K
__global__ void __launch_bounds__(128) maes_init_kept_kernel(const MaesState st, int Hp, int Hj) {
  const int b = blockIdx.x, s = b * st.K;
  const MaesRows& r = st.rows[0];
  for (int j = threadIdx.x; j < Hp; j += blockDim.x) {
    st.cur.h[static_cast<size_t>(s) * Hp + j] = r.h[static_cast<size_t>(b) * Hp + j];
    st.cur.c[static_cast<size_t>(s) * Hp + j] = r.c[static_cast<size_t>(b) * Hp + j];
  }
  for (int j = threadIdx.x; j < Hj; j += blockDim.x) st.cur.pp[static_cast<size_t>(s) * Hj + j] = r.pp[static_cast<size_t>(b) * Hj + j];
}

// ---------------------------------------------------------------------------------------------- joint rows
// grid (R * P), block 128: row r * P + d = kept slot r against dec_out[-1 - d] at frame t.  Dead rows (no hypothesis, past the
// last frame, or deeper than the hypothesis) are zero-filled and marked prow_t = -1: their logits are never read.
__global__ void __launch_bounds__(128)
maes_prefix_rows_kernel(const MaesState st, const float* __restrict__ encp, const int32_t* __restrict__ enc_len, int T_max, int Hj, int t,
                        __nv_bfloat16* __restrict__ planes) {
  const int row = blockIdx.x, r = row / st.P, d = row % st.P, b = r / st.K, k = r % st.K;
  const bool live = t < enc_len[b] && k < st.cur.n_hyp[b] && d <= st.cur.u[r];
  if (threadIdx.x == 0) st.prow_t[row] = live ? t : -1;
  __nv_bfloat16* out = planes + static_cast<size_t>(row) * 3 * Hj;
  const float* ep = encp + (static_cast<size_t>(b) * T_max + (live ? t : 0)) * Hj;
  const float* pp = st.cur.pp + (static_cast<size_t>(d) * st.B * st.K + r) * Hj;
  for (int j = threadIdx.x; j < Hj; j += blockDim.x) write_planes3(out, Hj, j, live ? fmaxf(ep[j] + pp[j], 0.f) : 0.f);
}

// grid (M), block 128: row i of round n at frame t
__global__ void __launch_bounds__(128)
maes_rows_kernel(const MaesState st, int n, const float* __restrict__ encp, int T_max, int Hj, int t, __nv_bfloat16* __restrict__ planes) {
  const int i = blockIdx.x;
  const MaesRows& r = st.rows[n];
  const float* ep = encp + (static_cast<size_t>(r.utt[i]) * T_max + t) * Hj;
  const float* pp = r.pp + static_cast<size_t>(i) * Hj;
  __nv_bfloat16* out = planes + static_cast<size_t>(i) * 3 * Hj;
  for (int j = threadIdx.x; j < Hj; j += blockDim.x) write_planes3(out, Hj, j, fmaxf(ep[j] + pp[j], 0.f));
}

// grid (M), block 256.  n < 0: the prefix pass (log-sum-exp of every live row; top-C of the depth-0 rows); n < S - 1: top-C of
// round n's rows (the next round expands them); n = S - 1: log p(blank) of the last round's rows.
__global__ void __launch_bounds__(256) maes_reduce_kernel(const MaesState st, int n, const float* __restrict__ logits, int ld, int V) {
  const int i = blockIdx.x;
  const float* x = logits + static_cast<size_t>(i) * ld;
  if (n < 0) {
    if (st.prow_t[i] < 0) return;
    const bool top = i % st.P == 0;
    const int r = i / st.P;
    beam_row_reduce(x, V + 1, V + 1, top ? st.C : 0, st.plse + i, nullptr, st.pcand_lp + static_cast<size_t>(r) * st.C,
                    st.pcand_tok + static_cast<size_t>(r) * st.C);
  } else if (n < st.S - 1) {
    beam_row_reduce(x, V + 1, V + 1, st.C, nullptr, nullptr, st.rcand_lp + static_cast<size_t>(i) * st.C, st.rcand_tok + static_cast<size_t>(i) * st.C);
  } else {
    beam_row_reduce(x, V + 1, V + 1, 0, nullptr, st.rblank + i, nullptr, nullptr);
  }
}

// ---------------------------------------------------------------------------------------------- prefix search
// grid (B), block 32 (lane 0 serial: at most beam (beam - 1) / 2 pairs).  Sorts the kept slots by length (longest first, stable)
// into ord and runs NeMo's prefix_search: for kept j and a later i whose sequence is a strict prefix of j's and at most
// prefix_alpha shorter, score_j = logaddexp(score_j, score_i + log p(the tokens of j after i's)).  Every score read is the one
// before this frame's updates (NeMo reads i's score before its own turn as j comes).
__global__ void __launch_bounds__(32) maes_prefix_kernel(const MaesState st, const float* __restrict__ logits, int ld) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  const int K = st.K, P = st.P;
  st.lb_n[b] = 0;
  const int r0 = b * K;
  if (st.prow_t[r0 * P] < 0) { st.fstate[b] = 2; return; }   // past the last frame (slot 0 is live while the utterance is)
  st.fstate[b] = 0;
  const int n_h = st.cur.n_hyp[b];
  int ord[8];
  for (int k = 0; k < n_h; ++k) {                                            // stable insertion by u descending
    int pos = k;
    while (pos > 0 && st.cur.u[r0 + ord[pos - 1]] < st.cur.u[r0 + k]) { ord[pos] = ord[pos - 1]; --pos; }
    ord[pos] = k;
  }
  for (int k = 0; k < n_h; ++k) st.ord[r0 + k] = r0 + ord[k];
  if (st.alpha == 0) return;
  double sc0[8];
  for (int k = 0; k < n_h; ++k) sc0[k] = st.cur.score[r0 + k];
  auto lp = [&](int r, int d, int tok) {
    const int row = r * P + d;
    return static_cast<double>(logits[static_cast<size_t>(row) * ld + tok] - st.plse[row]);
  };
  for (int jj = 0; jj + 1 < n_h; ++jj) {
    const int j = r0 + ord[jj];
    const int uj = st.cur.u[j];
    double s = sc0[ord[jj]];
    bool changed = false;
    for (int ii = jj + 1; ii < n_h; ++ii) {
      const int i = r0 + ord[ii];
      const int dl = uj - st.cur.u[i];
      if (dl < 1 || dl > st.alpha || st.cur.hh[static_cast<size_t>(j) * (P + 1) + dl] != st.cur.hh[static_cast<size_t>(i) * (P + 1)]) continue;
      const int* th = st.cur.th + static_cast<size_t>(j) * P;                // th[d]: j's d-th token from the end
      double curr = sc0[ord[ii]] + lp(i, 0, th[dl - 1]);
      for (int depth = dl - 1; depth >= 1; --depth) curr += lp(j, depth, th[depth - 1]);
      s = logaddexp(s, curr);
      changed = true;
    }
    if (changed) st.cur.score[j] = s;
  }
}

// ---------------------------------------------------------------------------------------------- expansion round
// grid (B), block 32.  Round n expands the hypotheses of the previous round (n = 0: the kept ones in prefix-search order).  Lane 0
// runs select_k_expansions and the list bookkeeping into the utterance's staging area; the warp then writes the compacted rows
// and adds the LM terms (one lm_fill_row per expansion, over the one column of its token).
__global__ void __launch_bounds__(32) maes_expand_kernel(const MaesState st, int n, int blank, const NgramLM lm) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const MaesRows& out = st.rows[n];
  if (st.fstate[b] != 0) {
    if (lane == 0) out.cnt[b] = 0;
    return;
  }
  const int K = st.K, C = st.C, P = st.P;
  const Src par = src_of(st, n - 1);
  const int n_h = n == 0 ? st.cur.n_hyp[b] : st.rows[n - 1].cnt[b];
  const int h0 = n == 0 ? 0 : st.rows[n - 1].begin[b];
  const size_t sg = static_cast<size_t>(b) * st.W;
  int ne = 0;
  if (lane == 0) {
    const size_t lb = static_cast<size_t>(b) * st.lb_cap;
    int nb = st.lb_n[b];
    for (int q = 0; q < n_h; ++q) {
      const int id = n == 0 ? st.ord[b * K + q] : h0 + q;                   // kept slot, or row of round n - 1
      const float* clp = n == 0 ? st.pcand_lp + static_cast<size_t>(id) * C : st.rcand_lp + static_cast<size_t>(id) * C;
      const int* ctok = n == 0 ? st.pcand_tok + static_cast<size_t>(id) * C : st.rcand_tok + static_cast<size_t>(id) * C;
      const double s0 = par.score[id];
      double v[kMaesMaxC];
      int best = 0;
      for (int c = 0; c < C; ++c) {
        v[c] = s0 + static_cast<double>(clp[c]);
        if (v[c] > v[best]) best = c;
      }
      bool keep[kMaesMaxC];
      int n_keep = 0;
      for (int c = 0; c < C; ++c) { keep[c] = v[best] - st.gamma <= v[c]; n_keep += keep[c]; }
      if (n_keep == 0) keep[best] = true, n_keep = 1;
      const unsigned long long hp = par.hh[static_cast<size_t>(id) * (P + 1)];
      const int up = par.u[id];
      for (int e = 0; e < n_keep; ++e) {                                    // ascending by score, stable (ties: top-C order)
        int c = -1;
        for (int x = 0; x < C; ++x)
          if (keep[x] && (c < 0 || v[x] < v[c])) c = x;
        keep[c] = false;
        const int tok = ctok[c];
        if (tok == blank) {
          st.lb_score[lb + nb] = v[c]; st.lb_round[lb + nb] = n - 1; st.lb_idx[lb + nb] = id; ++nb;
          continue;
        }
        const unsigned long long h2 = hash_push(hp, tok);
        bool dup = false;                                                    // duplication_check: the kept sequences of this frame
        for (int k = 0; k < st.cur.n_hyp[b]; ++k) {
          const int r = b * K + k;
          dup |= st.cur.u[r] == up + 1 && st.cur.hh[static_cast<size_t>(r) * (P + 1)] == h2;
        }
        if (dup) continue;
        st.sg_score[sg + ne] = v[c]; st.sg_par[sg + ne] = id; st.sg_tok[sg + ne] = tok; ++ne;
      }
    }
    st.lb_n[b] = nb;
    if (ne == 0) st.fstate[b] = 1;
  }
  ne = __shfl_sync(0xffffffffu, ne, 0);
  int begin = 0;
  if (lane == 0 && ne > 0) begin = atomicAdd(st.m + n, ne);
  begin = __shfl_sync(0xffffffffu, begin, 0);
  if (lane == 0) { out.begin[b] = begin; out.cnt[b] = ne; }
  __syncwarp();
  for (int e = lane; e < ne; e += 32) {
    const int i = begin + e, id = st.sg_par[sg + e], tok = st.sg_tok[sg + e];
    out.score[i] = st.sg_score[sg + e]; out.par[i] = id; out.tok[i] = tok; out.utt[i] = b;
    out.u[i] = par.u[id] + 1; out.lm[i] = par.lm[id];
    out.hh[static_cast<size_t>(i) * (P + 1)] = hash_push(par.hh[static_cast<size_t>(id) * (P + 1)], tok);
    for (int d = 1; d <= P; ++d) out.hh[static_cast<size_t>(i) * (P + 1) + d] = par.hh[static_cast<size_t>(id) * (P + 1) + d - 1];
    out.th[static_cast<size_t>(i) * P] = tok;
    for (int d = 1; d < P; ++d) out.th[static_cast<size_t>(i) * P + d] = par.th[static_cast<size_t>(id) * P + d - 1];
  }
  if (lm.order == 0) return;
  __shared__ float s_term;
  __shared__ int s_next;
  __syncwarp();
  for (int e = 0; e < ne; ++e) {
    const int i = begin + e, tok = st.sg_tok[sg + e];
    lm_fill_row(lm, out.lm[i], tok, tok + 1, &s_term, &s_next, lane);
    __syncwarp();
    if (lane == 0) { out.score[i] += static_cast<double>(s_term); out.lm[i] = s_next; }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------- predictor of a round's rows
// grid (M), block 128: [embed[token] (blank: the zero vector) | h of the parent (none: zeros)] as three bf16 planes (K = 2 Hp per
// plane); the parent's dec_out history moves one plane deeper.
__global__ void __launch_bounds__(128)
maes_lstm_in_kernel(const MaesState st, int n, const float* __restrict__ embed, int Hp, int Hj, int blank, __nv_bfloat16* __restrict__ planes) {
  const int i = blockIdx.x;
  const MaesRows& r = st.rows[n];
  const int tok = r.tok[i], p = r.par[i];
  const Src par = src_of(st, n - 1);
  const float* e = embed + static_cast<size_t>(tok == blank ? 0 : tok) * Hp;
  const float* h = par.h + static_cast<size_t>(p < 0 ? 0 : p) * Hp;
  __nv_bfloat16* row = planes + static_cast<size_t>(i) * 6 * Hp;
  for (int j = threadIdx.x; j < 2 * Hp; j += blockDim.x) {
    const float x = j < Hp ? (tok == blank ? 0.f : e[j]) : (p < 0 ? 0.f : h[j - Hp]);
    write_planes3(row, 2 * Hp, j, x);
  }
  if (p < 0) return;
  for (int d = 1; d < st.P; ++d)
    for (int j = threadIdx.x; j < Hj; j += blockDim.x)
      r.pp[(static_cast<size_t>(d) * r.cap + i) * Hj + j] = par.pp[(static_cast<size_t>(d - 1) * par.pp_plane + p) * Hj + j];
}

// grid (M), block 128: LSTM cell (gate order i, f, g, o; biases already in `gates`) -> h, c of the row; h as three bf16 planes
__global__ void __launch_bounds__(128)
maes_cell_kernel(const MaesState st, int n, const float* __restrict__ gates, int Hp, __nv_bfloat16* __restrict__ planes) {
  const int i = blockIdx.x;
  const MaesRows& r = st.rows[n];
  const int p = r.par[i];
  const Src par = src_of(st, n - 1);
  const float* g = gates + static_cast<size_t>(i) * 4 * Hp;
  __nv_bfloat16* row = planes + static_cast<size_t>(i) * 3 * Hp;
  for (int j = threadIdx.x; j < Hp; j += blockDim.x) {
    const float ig = sigmoidf_accurate(g[j]), fg = sigmoidf_accurate(g[Hp + j]);
    const float cg = tanhf(g[2 * Hp + j]), og = sigmoidf_accurate(g[3 * Hp + j]);
    const float c0 = p < 0 ? 0.f : par.c[static_cast<size_t>(p) * Hp + j];
    const float c2 = fg * c0 + ig * cg;
    const float h2 = og * tanhf(c2);
    r.h[static_cast<size_t>(i) * Hp + j] = h2;
    r.c[static_cast<size_t>(i) * Hp + j] = c2;
    write_planes3(row, Hp, j, h2);
  }
}

// ---------------------------------------------------------------------------------------------- new kept hypotheses
// grid (B), block 32, the lanes in parallel over the candidates list_b + list_exp (in that order; list_exp scored with its final
// blank).  NeMo's recombine_hypotheses: the first occurrence of a sequence takes the logaddexp of every later duplicate's score in
// order; as recalled it returns its input (duplicates kept, recombine_returns_input) -- otherwise the merged list.  Then the beam
// best by score, stable (Python's sorted), become the kept slots, with one back-pointer node per token this frame added.
__global__ void __launch_bounds__(32) maes_select_kernel(const MaesState st, int t) {
  const int b = blockIdx.x, lane = threadIdx.x, K = st.K, P = st.P;
  const int fs = st.fstate[b];
  if (fs == 2) {                                                              // frozen: the kept slots stay
    if (lane == 0) st.nx.n_hyp[b] = st.cur.n_hyp[b];
    if (lane < K) {
      const int r = b * K + lane;
      st.sel_round[r] = -1; st.sel_idx[r] = r;
      st.nx.score[r] = st.cur.score[r]; st.nx.u[r] = st.cur.u[r]; st.nx.node[r] = st.cur.node[r]; st.nx.lm[r] = st.cur.lm[r];
      for (int d = 0; d <= P; ++d) st.nx.hh[static_cast<size_t>(r) * (P + 1) + d] = st.cur.hh[static_cast<size_t>(r) * (P + 1) + d];
      for (int d = 0; d < P; ++d) st.nx.th[static_cast<size_t>(r) * P + d] = st.cur.th[static_cast<size_t>(r) * P + d];
    }
    return;
  }
  const MaesRows& last = st.rows[st.S - 1];
  const int nb = st.lb_n[b];
  const int ne = fs == 0 ? last.cnt[b] : 0;
  const int e0 = fs == 0 ? last.begin[b] : 0;
  const int nc = nb + ne;
  const size_t co = static_cast<size_t>(b) * (st.lb_cap + st.W), lb = static_cast<size_t>(b) * st.lb_cap;
  double* cs = st.c_score + co;
  unsigned long long* ch = st.c_hash + co;
  int* cu = st.c_u + co;
  int* cf = st.c_first + co;
  for (int x = lane; x < nc; x += 32) {
    if (x < nb) {
      const Src s = src_of(st, st.lb_round[lb + x]);
      const int id = st.lb_idx[lb + x];
      cs[x] = st.lb_score[lb + x]; ch[x] = s.hh[static_cast<size_t>(id) * (P + 1)]; cu[x] = s.u[id];
    } else {
      const int i = e0 + x - nb;
      cs[x] = last.score[i] + static_cast<double>(st.rblank[i]); ch[x] = last.hh[static_cast<size_t>(i) * (P + 1)]; cu[x] = last.u[i];
    }
  }
  __syncwarp();
  for (int x = lane; x < nc; x += 32) {                                       // first occurrence of x's sequence
    int f = x;
    for (int y = 0; y < x; ++y)
      if (ch[y] == ch[x] && cu[y] == cu[x]) { f = y; break; }
    cf[x] = f;
  }
  __syncwarp();
  for (int x = lane; x < nc; x += 32) {                                       // merged in place: only first occurrences are written,
    if (cf[x] != x) continue;                                                 // only later duplicates read
    double s = cs[x];
    for (int y = x + 1; y < nc; ++y)
      if (cf[y] == x) s = logaddexp(s, cs[y]);
    cs[x] = s;
  }
  __syncwarp();
  const bool rri = st.rri != 0;
  int n_live = 0;
  for (int x = lane; x < nc; x += 32) n_live += rri || cf[x] == x;
  for (int o = 16; o > 0; o >>= 1) n_live += __shfl_xor_sync(0xffffffffu, n_live, o);
  const int n_new = n_live < K ? n_live : K;
  for (int x = lane; x < nc; x += 32) {
    if (!rri && cf[x] != x) continue;
    const double s = cs[x];
    int rank = 0;
    for (int y = 0; y < nc && rank < K; ++y)
      if ((rri || cf[y] == y) && (cs[y] > s || (cs[y] == s && y < x))) ++rank;
    if (rank >= K) continue;
    const int r = b * K + rank;
    int round, id;
    if (x < nb) { round = st.lb_round[lb + x]; id = st.lb_idx[lb + x]; }
    else { round = st.S - 1; id = e0 + x - nb; }
    const Src src = src_of(st, round);
    st.sel_round[r] = round; st.sel_idx[r] = id;
    st.nx.score[r] = s; st.nx.u[r] = src.u[id]; st.nx.lm[r] = src.lm[id];
    for (int d = 0; d <= P; ++d) st.nx.hh[static_cast<size_t>(r) * (P + 1) + d] = src.hh[static_cast<size_t>(id) * (P + 1) + d];
    for (int d = 0; d < P; ++d) st.nx.th[static_cast<size_t>(r) * P + d] = src.th[static_cast<size_t>(id) * P + d];
    // the tokens this frame added, newest first, up to the kept parent; then nodes oldest first
    int toks[kMaesMaxSteps];
    int m = 0, slot = id;
    for (int rd = round; rd >= 0; --rd) { toks[m++] = st.rows[rd].tok[slot]; slot = st.rows[rd].par[slot]; }
    int node = st.cur.node[slot];
    const size_t tree = static_cast<size_t>(b) * st.max_nodes;
    for (int q = m - 1; q >= 0; --q) {
      const int nn = atomicAdd(st.n_nodes + b, 1);
      st.node_parent[tree + nn] = node; st.node_tok[tree + nn] = toks[q]; st.node_frame[tree + nn] = t;
      node = nn;
    }
    st.nx.node[r] = node;
  }
  if (lane == 0) st.nx.n_hyp[b] = n_new;
}

// grid (R), block 128: h, c and the dec_out history of each new kept slot from its source
__global__ void __launch_bounds__(128) maes_gather_kernel(const MaesState st, int Hp, int Hj) {
  const int r = blockIdx.x, b = r / st.K, k = r % st.K;
  if (k >= st.nx.n_hyp[b]) return;
  const int round = st.sel_round[r], id = st.sel_idx[r];
  const Src s = src_of(st, round);
  for (int j = threadIdx.x; j < Hp; j += blockDim.x) {
    st.nx.h[static_cast<size_t>(r) * Hp + j] = s.h[static_cast<size_t>(id) * Hp + j];
    st.nx.c[static_cast<size_t>(r) * Hp + j] = s.c[static_cast<size_t>(id) * Hp + j];
  }
  const size_t R = static_cast<size_t>(st.B) * st.K;
  for (int d = 0; d < st.P; ++d)
    for (int j = threadIdx.x; j < Hj; j += blockDim.x)
      st.nx.pp[(d * R + r) * Hj + j] = s.pp[(d * s.pp_plane + id) * Hj + j];
}

// ---------------------------------------------------------------------------------------------- output
// grid (B), block 32: NeMo's sort_nbest of the kept hypotheses (score / len(y) with score_norm, else score; stable) -> the first
// n_best entries: y with the leading blank, each token's encoder frame, token count, score; count[b] = min(n_best, kept).
__global__ void __launch_bounds__(32)
maes_output_kernel(const MaesState st, int n_best, int blank, int32_t* __restrict__ y_out, int32_t* __restrict__ frame_out,
                   int32_t* __restrict__ n_out, double* __restrict__ score_out, int32_t* __restrict__ count_out, int U_cap) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int n_h = st.cur.n_hyp[b];
  if (lane == 0) count_out[b] = n_h < n_best ? n_h : n_best;
  if (lane >= n_h) return;
  auto key = [&](int k) {
    const int r = b * st.K + k;
    return st.score_norm ? st.cur.score[r] / static_cast<double>(st.cur.u[r] + 1) : st.cur.score[r];
  };
  const double mine = key(lane);
  int rank = 0;
  for (int k = 0; k < n_h; ++k) {
    const double other = key(k);
    rank += other > mine || (other == mine && k < lane);
  }
  if (rank >= n_best) return;
  const int r = b * st.K + lane;
  const size_t i = static_cast<size_t>(b) * n_best + rank;
  const int u = st.cur.u[r];
  n_out[i] = u;
  score_out[i] = st.cur.score[r];
  int32_t* y = y_out + i * (U_cap + 1);
  int32_t* fr = frame_out + i * U_cap;
  const size_t tree = static_cast<size_t>(b) * st.max_nodes;
  y[0] = blank;
  int node = st.cur.node[r], pos = u;
  while (node > 0 && pos > 0) {
    if (pos <= U_cap) { y[pos] = st.node_tok[tree + node]; fr[pos - 1] = st.node_frame[tree + node]; }
    node = st.node_parent[tree + node];
    --pos;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
void maes_layout_state(MaesState& st, Arena& a, char* base, int B, int K, int C, int S, int P, int Hp, int Hj, int max_nodes) {
  auto take = [&](size_t bytes) { return reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(base) + a.take(bytes)); };
  const size_t R = static_cast<size_t>(B) * K;
  st.B = B; st.K = K; st.C = C; st.S = S; st.P = P; st.max_nodes = max_nodes;
  int pw = 1, lb = 0;
  for (int n = 0; n < S; ++n) { lb += K * pw; pw *= C; }
  st.W = K * pw; st.lb_cap = lb;
  for (MaesKept* k : {&st.cur, &st.nx}) {
    k->score = static_cast<double*>(take(R * 8)); k->hh = static_cast<unsigned long long*>(take(R * (P + 1) * 8));
    k->th = static_cast<int*>(take(R * P * 4)); k->u = static_cast<int*>(take(R * 4)); k->node = static_cast<int*>(take(R * 4));
    k->lm = static_cast<int*>(take(R * 4));
    k->h = static_cast<float*>(take(R * Hp * 4)); k->c = static_cast<float*>(take(R * Hp * 4)); k->pp = static_cast<float*>(take(P * R * Hj * 4));
    k->n_hyp = static_cast<int*>(take(static_cast<size_t>(B) * 4));
  }
  int w = K;
  size_t cap_max = 0;
  for (int n = 0; n < S; ++n) {
    w *= C;
    MaesRows& r = st.rows[n];
    r.cap = B * w;
    const size_t cap = static_cast<size_t>(r.cap);
    cap_max = cap > cap_max ? cap : cap_max;
    r.score = static_cast<double*>(take(cap * 8)); r.hh = static_cast<unsigned long long*>(take(cap * (P + 1) * 8));
    r.th = static_cast<int*>(take(cap * P * 4));
    int* ints = static_cast<int*>(take(cap * 5 * 4));
    r.u = ints; r.lm = ints + cap; r.par = ints + 2 * cap; r.tok = ints + 3 * cap; r.utt = ints + 4 * cap;
    r.h = static_cast<float*>(take(cap * Hp * 4)); r.c = static_cast<float*>(take(cap * Hp * 4)); r.pp = static_cast<float*>(take(P * cap * Hj * 4));
    r.begin = static_cast<int*>(take(static_cast<size_t>(B) * 4)); r.cnt = static_cast<int*>(take(static_cast<size_t>(B) * 4));
  }
  st.m = static_cast<int*>(take(kMaesMaxSteps * 4));
  st.prow_t = static_cast<int*>(take(R * P * 4)); st.plse = static_cast<float*>(take(R * P * 4));
  st.pcand_lp = static_cast<float*>(take(R * C * 4)); st.pcand_tok = static_cast<int*>(take(R * C * 4));
  st.rcand_lp = static_cast<float*>(take(cap_max * C * 4)); st.rcand_tok = static_cast<int*>(take(cap_max * C * 4));
  st.rblank = static_cast<float*>(take(cap_max * 4));
  st.ord = static_cast<int*>(take(R * 4)); st.fstate = static_cast<int*>(take(static_cast<size_t>(B) * 4));
  const size_t L = static_cast<size_t>(B) * st.lb_cap, G = static_cast<size_t>(B) * st.W, CC = L + G;
  st.lb_score = static_cast<double*>(take(L * 8)); st.lb_round = static_cast<int*>(take(L * 4)); st.lb_idx = static_cast<int*>(take(L * 4));
  st.lb_n = static_cast<int*>(take(static_cast<size_t>(B) * 4));
  st.sg_score = static_cast<double*>(take(G * 8)); st.sg_par = static_cast<int*>(take(G * 4)); st.sg_tok = static_cast<int*>(take(G * 4));
  st.c_score = static_cast<double*>(take(CC * 8)); st.c_hash = static_cast<unsigned long long*>(take(CC * 8));
  st.c_u = static_cast<int*>(take(CC * 4)); st.c_first = static_cast<int*>(take(CC * 4));
  st.sel_round = static_cast<int*>(take(R * 4)); st.sel_idx = static_cast<int*>(take(R * 4));
  st.n_nodes = static_cast<int*>(take(static_cast<size_t>(B) * 4));
  int* tree = static_cast<int*>(take(static_cast<size_t>(B) * max_nodes * 4 * 3));
  st.node_parent = tree; st.node_tok = tree + static_cast<size_t>(B) * max_nodes; st.node_frame = tree + 2 * static_cast<size_t>(B) * max_nodes;
}

cudaError_t maes_launch_init(const MaesState& st, int blank, int lm_start, cudaStream_t s) {
  maes_init_kernel<<<st.B, 32, 0, s>>>(st, blank, lm_start);
  return cudaGetLastError();
}
cudaError_t maes_launch_init_kept(const MaesState& st, int Hp, int Hj, cudaStream_t s) {
  maes_init_kept_kernel<<<st.B, 128, 0, s>>>(st, Hp, Hj);
  return cudaGetLastError();
}
cudaError_t maes_launch_prefix_rows(const MaesState& st, const float* encp, const int32_t* enc_len, int T_max, int Hj, int t, void* planes, cudaStream_t s) {
  maes_prefix_rows_kernel<<<st.B * st.K * st.P, 128, 0, s>>>(st, encp, enc_len, T_max, Hj, t, static_cast<__nv_bfloat16*>(planes));
  return cudaGetLastError();
}
cudaError_t maes_launch_reduce(const MaesState& st, int n, int M, const float* logits, int ld, int V, cudaStream_t s) {
  maes_reduce_kernel<<<M, 256, 0, s>>>(st, n, logits, ld, V);
  return cudaGetLastError();
}
cudaError_t maes_launch_prefix(const MaesState& st, const float* logits, int ld, cudaStream_t s) {
  maes_prefix_kernel<<<st.B, 32, 0, s>>>(st, logits, ld);
  return cudaGetLastError();
}
cudaError_t maes_launch_expand(const MaesState& st, int n, int blank, const NgramLM& lm, cudaStream_t s) {
  maes_expand_kernel<<<st.B, 32, 0, s>>>(st, n, blank, lm);
  return cudaGetLastError();
}
cudaError_t maes_launch_lstm_in(const MaesState& st, int n, int M, const float* embed, int Hp, int Hj, int blank, void* planes, cudaStream_t s) {
  maes_lstm_in_kernel<<<M, 128, 0, s>>>(st, n, embed, Hp, Hj, blank, static_cast<__nv_bfloat16*>(planes));
  return cudaGetLastError();
}
cudaError_t maes_launch_cell(const MaesState& st, int n, int M, const float* gates, int Hp, void* planes, cudaStream_t s) {
  maes_cell_kernel<<<M, 128, 0, s>>>(st, n, gates, Hp, static_cast<__nv_bfloat16*>(planes));
  return cudaGetLastError();
}
cudaError_t maes_launch_rows(const MaesState& st, int n, int M, const float* encp, int T_max, int Hj, int t, void* planes, cudaStream_t s) {
  maes_rows_kernel<<<M, 128, 0, s>>>(st, n, encp, T_max, Hj, t, static_cast<__nv_bfloat16*>(planes));
  return cudaGetLastError();
}
cudaError_t maes_launch_select(const MaesState& st, int t, cudaStream_t s) {
  maes_select_kernel<<<st.B, 32, 0, s>>>(st, t);
  return cudaGetLastError();
}
cudaError_t maes_launch_gather(const MaesState& st, int Hp, int Hj, cudaStream_t s) {
  maes_gather_kernel<<<st.B * st.K, 128, 0, s>>>(st, Hp, Hj);
  return cudaGetLastError();
}
cudaError_t maes_launch_output(const MaesState& st, int n_best, int blank, int32_t* y, int32_t* frames, int32_t* n, double* score, int32_t* count,
                               int U_cap, cudaStream_t s) {
  maes_output_kernel<<<st.B, 32, 0, s>>>(st, n_best, blank, y, frames, n, score, count, U_cap);
  return cudaGetLastError();
}

}  // namespace rs
