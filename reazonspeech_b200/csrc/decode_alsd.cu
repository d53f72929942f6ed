// ALSD beam search (alignment-length synchronous decoding) for the RNN-T head, batched over utterances: NeMo's
// BeamRNNTInfer.align_length_sync_decoding, the strategy the shipped reazonspeech-nemo-v2 checkpoint decodes with by default
// -- the reference's own post-processing is written for its hypotheses (pkg/nemo-asr/src/decode.py:29 "Decode ALSD beam search
// info", :38-40 the leading blank of y_sequence, :48 step - idx - 1).  Semantics restated in oracle/alsd_restated.py.
//
// One step = one anti-diagonal i = t + u of the (frame, token) lattice for every utterance at once.  The three matrix products
// of a step (joint logits of the live hypotheses, LSTM gates and joint.pred of the newly extended ones) go through the wgmma
// GEMM of gemm_wgmma.cu with their fp32 activations split into three bf16 terms (24 mantissa bits against bf16-exact
// weights: fp32-accurate log-probabilities, so that beam decisions move only with the encoder's rounding, not the decoder's);
// this file holds the kernels in between:
//
//   alsd_rows_kernel     live (utterance, hypothesis) rows: relu(enc_proj[b, t] + pred_proj[b, k]) -> three bf16 planes
//   [GEMM]               logits[rows, V + 1] = planes . [W_out | W_out | W_out]^T + b_out
//   alsd_reduce_kernel   per row: log-sum-exp, log p(blank), the `beam` best non-blank classes (ties: lower index)
//   alsd_select_kernel   per utterance: A = [stay, extensions ...] per live hypothesis in beam order, the `beam` best by score
//                        (stable: ties keep A's order, as Python's sorted does), NeMo's recombine_hypotheses, the finished
//                        list (hypotheses that took the blank at the last frame; its n_best best kept sorted), back-pointer
//                        nodes of the extensions
//   alsd_lstm_in_kernel  extended hypotheses: [embed[token] | h_parent] -> three bf16 planes
//   [GEMM]               gates = planes . [W_lstm x3]^T + b
//   alsd_cell_kernel     LSTM cell, new (h, c) (kept hypotheses: copied from the parent); h -> three bf16 planes
//   [GEMM]               pred_proj = planes . [W_pred x3]^T + b_pred, straight into the next beam
//
// The state holds two beams, the current one and the one the step builds; the host swaps them after every predictor pass.
// A kept hypothesis's pred_proj is recomputed from the h it inherits rather than copied: a GEMM row does not depend on the
// other rows or on its position, so the value is the parent's bit for bit.
//
// Scores are doubles (Python floats in NeMo), log-probabilities fp32 (torch.log_softmax of fp32 logits).
#include <cfloat>

#include "alsd.h"
#include "beam_common.cuh"
#include "common.cuh"
#include "kernels.h"

namespace rs {

namespace {

constexpr int kMaxBeam = 8;

// ---------------------------------------------------------------------------------------------- joint rows
// grid (B * beam), block 128.  Row r = b * beam + k.  Dead rows (hypothesis absent, or past the last frame) are zero-filled:
// their logits are never read.
__global__ void __launch_bounds__(128)
alsd_rows_kernel(const AlsdState st, const float* __restrict__ enc_proj, const int32_t* __restrict__ enc_len, int T_max, int Hj,
                 int step, __nv_bfloat16* __restrict__ planes) {
  const int r = blockIdx.x, b = r / st.beam, k = r % st.beam;
  const int n_h = st.cur.n_hyp[b];
  const int T = enc_len[b];
  int t = -1;
  if (!st.done[b] && k < n_h) {
    t = step - st.cur.u[r];
    if (t > T - 1) t = -1;
  }
  if (threadIdx.x == 0) st.row_t[r] = t;
  __nv_bfloat16* row = planes + static_cast<size_t>(r) * 3 * Hj;
  const float* ep = enc_proj + (static_cast<size_t>(b) * T_max + (t >= 0 ? t : 0)) * Hj;
  const float* pp = st.cur.pp + static_cast<size_t>(r) * Hj;
  for (int j = threadIdx.x; j < Hj; j += blockDim.x) {
    const float x = t >= 0 ? fmaxf(ep[j] + pp[j], 0.f) : 0.f;
    __nv_bfloat16 h, m, l;
    split3(x, h, m, l);
    row[j] = h; row[Hj + j] = m; row[2 * Hj + j] = l;
  }
}

// ---------------------------------------------------------------------------------------------- per-row reductions
// grid (B * beam), block 256: log-sum-exp over the V + 1 classes, log p(blank), the `beam` largest non-blank log-probabilities
// (ties -> lower class index).
__global__ void __launch_bounds__(256)
alsd_reduce_kernel(const AlsdState st, const float* __restrict__ logits, int ld, int V) {
  const int r = blockIdx.x;
  if (st.row_t[r] < 0) return;
  beam_row_reduce(logits + static_cast<size_t>(r) * ld, V + 1, V, st.beam, nullptr, st.cand_logp + r * (kMaxBeam + 1),
                  st.cand_logp + r * (kMaxBeam + 1) + 1, st.cand_tok + r * kMaxBeam);
}

// ---------------------------------------------------------------------------------------------- beam update
// grid (B), block 32 (lane 0 does the serial work: at most beam * (beam + 1) <= 72 candidates).
// u_max = int(u_max_ratio * T) in double, as NeMo computes it: in fp32, ratio 1.16 at T = 25 gives 29 instead of 28.
__global__ void __launch_bounds__(32)
alsd_select_kernel(const AlsdState st, const int32_t* __restrict__ enc_len, int step, double u_max_ratio, int recombine_returns_input) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0 || st.done[b]) return;
  const int K = st.beam;
  const int T = enc_len[b];
  const int u_max = static_cast<int>(u_max_ratio * static_cast<double>(T));
  const AlsdBeam& cur = st.cur;
  const int n_h = cur.n_hyp[b];
  // the search of utterance b ends: no kernel writes its beam again, so the next beam becomes a copy of the current one and
  // both halves hold it whichever way later swaps fall (alsd_output_kernel reads it when no hypothesis finished)
  auto finish = [&]() {
    st.nx.n_hyp[b] = n_h;
    for (int k = 0; k < n_h; ++k) {
      const int r = b * K + k;
      st.nx.score[r] = cur.score[r]; st.nx.hash[r] = cur.hash[r]; st.nx.u[r] = cur.u[r]; st.nx.node[r] = cur.node[r];
    }
    st.done[b] = 1;
    atomicAdd(st.n_done, 1);
  };
  if (step >= T + u_max) {                             // the loop of the reference ends here whether or not hypotheses remain
    finish();
    return;
  }
  // A in the reference's order: for every live hypothesis of B: [stay, extension 0 .. K-1]
  double a_score[kMaxBeam * (kMaxBeam + 1)];
  int a_par[kMaxBeam * (kMaxBeam + 1)], a_tok[kMaxBeam * (kMaxBeam + 1)];
  int n_a = 0;
  bool any_final = false;                              // a stay at the last frame in this step
  for (int k = 0; k < n_h; ++k) {
    const int r = b * K + k;
    const int t = st.row_t[r];
    if (t < 0) continue;                               // past the last frame: dropped (it entered `final` when it got there)
    any_final |= t == T - 1;
    const double s0 = cur.score[r];
    const double stay = s0 + static_cast<double>(st.cand_logp[r * (kMaxBeam + 1)]);
    a_score[n_a] = stay; a_par[n_a] = k; a_tok[n_a] = -1; ++n_a;
    for (int c = 0; c < K; ++c) {
      a_score[n_a] = s0 + static_cast<double>(st.cand_logp[r * (kMaxBeam + 1) + 1 + c]);
      a_par[n_a] = k; a_tok[n_a] = st.cand_tok[r * kMaxBeam + c]; ++n_a;
    }
  }
  if (n_a == 0) {                                      // every hypothesis has left the lattice: the reference breaks out of its loop
    finish();
    return;
  }
  // the K best of A by score, stable
  int pick[kMaxBeam];
  bool used[kMaxBeam * (kMaxBeam + 1)];
  for (int i = 0; i < n_a; ++i) used[i] = false;
  const int n_new = n_a < K ? n_a : K;
  for (int j = 0; j < n_new; ++j) {
    int best = -1;
    for (int i = 0; i < n_a; ++i)
      if (!used[i] && (best < 0 || a_score[i] > a_score[best])) best = i;
    used[best] = true;
    pick[j] = best;
  }
  // new beam, written to the `nx` half
  double n_score[kMaxBeam];
  unsigned long long n_hash[kMaxBeam];
  int n_len[kMaxBeam];
  for (int j = 0; j < n_new; ++j) {
    const int a = pick[j], pk = a_par[a], pr = b * K + pk;
    n_score[j] = a_score[a];
    n_hash[j] = a_tok[a] >= 0 ? cur.hash[pr] * 1000003ull + static_cast<unsigned long long>(a_tok[a] + 1) : cur.hash[pr];
    n_len[j] = cur.u[pr] + (a_tok[a] >= 0 ? 1 : 0);
  }
  // NeMo's recombine_hypotheses: the score of a later duplicate is added (logaddexp) into the first occurrence; as recalled, the
  // reference then returns its INPUT list, duplicates included (oracle/alsd_restated.py `recombine_returns_input`)
  bool dropped[kMaxBeam], later[kMaxBeam];                         // later: a duplicate of an earlier pick (merged into it)
  for (int j = 0; j < n_new; ++j) dropped[j] = later[j] = false;
  for (int j = 1; j < n_new; ++j)
    for (int f = 0; f < j; ++f)
      if (!dropped[f] && n_hash[f] == n_hash[j] && n_len[f] == n_len[j]) {        // equal token sequences (64-bit sequence hash + length)
        n_score[f] = logaddexp(n_score[f], n_score[j]);
        later[j] = true;
        if (!recombine_returns_input) dropped[j] = true;
        break;
      }
  // finished hypotheses: the stays at the last frame, appended to `final` in A order and kept sorted by score / len(y)
  // (score_norm) as Python's stable sorted(reverse=True) orders them: a new entry goes after every held entry whose key is >=
  // its own, and the list keeps its first n_best.  In the reference the entry of `final` is the very object that went into
  // the beam, so a stay picked as the first of its sequence carries the score recombination added into it; any other stay
  // keeps its own.  Only this step can change them: a stay at T - 1 is not live at the next one.
  // The held keys are sorted, so the entries whose key is >= the new one are a prefix: counting them over the whole list
  // (independent loads) finds the position without a scan that stops at each load.
  const int N = st.n_best;
  const size_t fo = static_cast<size_t>(b) * N;
  double* __restrict__ f_key = st.fin_key + fo;
  double* __restrict__ f_score = st.fin_score + fo;
  int* __restrict__ f_node = st.fin_node + fo;
  int* __restrict__ f_u = st.fin_u + fo;
  for (int a = 0; any_final && a < n_a; ++a) {
    const int r = b * K + a_par[a];
    if (a_tok[a] >= 0 || st.row_t[r] != T - 1) continue;
    double s = a_score[a];
    for (int j = 0; j < n_new; ++j)
      if (pick[j] == a && !later[j]) s = n_score[j];
    const double key = st.score_norm ? s / static_cast<double>(cur.u[r] + 1) : s;
    ++st.fin_pool[b];
    const int cnt = st.fin_count[b];
    int pos = 0;
    for (int e = 0; e < cnt; ++e) pos += f_key[e] >= key;
    if (pos == N) continue;                            // full, and no held key is below it
    for (int e = cnt < N ? cnt : N - 1; e > pos; --e) {
      f_key[e] = f_key[e - 1]; f_score[e] = f_score[e - 1]; f_node[e] = f_node[e - 1]; f_u[e] = f_u[e - 1];
    }
    f_key[pos] = key; f_score[pos] = s; f_node[pos] = cur.node[r]; f_u[pos] = cur.u[r];
    st.fin_count[b] = cnt < N ? cnt + 1 : N;
  }
  int w = 0;
  for (int j = 0; j < n_new; ++j) {
    if (dropped[j]) continue;
    const int a = pick[j], pk = a_par[a], pr = b * K + pk, nr = b * K + w;
    st.nx.score[nr] = n_score[j];
    st.nx.hash[nr] = n_hash[j];
    st.nx_parent[nr] = pk;
    st.nx_tok[nr] = a_tok[a];
    if (a_tok[a] >= 0) {                               // extension: one more token, emitted at alignment step `step`
      st.nx.u[nr] = cur.u[pr] + 1;
      const int node = st.n_nodes[b]++;
      st.node_parent[static_cast<size_t>(b) * st.max_nodes + node] = cur.node[pr];
      st.node_tok[static_cast<size_t>(b) * st.max_nodes + node] = a_tok[a];
      st.node_step[static_cast<size_t>(b) * st.max_nodes + node] = step;
      st.nx.node[nr] = node;
    } else {
      st.nx.u[nr] = cur.u[pr];
      st.nx.node[nr] = cur.node[pr];
    }
    ++w;
  }
  st.nx.n_hyp[b] = w;
}

// ---------------------------------------------------------------------------------------------- predictor of the extensions
// grid (B * beam), block 128: rows of the NEXT beam.  Extended hypotheses get [embed[token] | h_parent] as three bf16 planes
// (K = 2 * Hp per plane); kept ones (and absent rows) get zeros, and the cell kernel ignores their gates.
__global__ void __launch_bounds__(128)
alsd_lstm_in_kernel(const AlsdState st, const float* __restrict__ embed, int Hp, __nv_bfloat16* __restrict__ planes) {
  const int r = blockIdx.x, b = r / st.beam, k = r % st.beam;
  const bool ext = !st.done[b] && k < st.nx.n_hyp[b] && st.nx_tok[r] >= 0;
  __nv_bfloat16* row = planes + static_cast<size_t>(r) * 6 * Hp;
  const float* e = embed + static_cast<size_t>(ext ? st.nx_tok[r] : 0) * Hp;
  const float* h = st.cur.h + (static_cast<size_t>(b) * st.beam + (ext ? st.nx_parent[r] : 0)) * Hp;
  for (int j = threadIdx.x; j < 2 * Hp; j += blockDim.x) {
    const float x = ext ? (j < Hp ? e[j] : h[j - Hp]) : 0.f;
    __nv_bfloat16 hi, mid, lo;
    split3(x, hi, mid, lo);
    row[j] = hi; row[2 * Hp + j] = mid; row[4 * Hp + j] = lo;
  }
}

// grid (B * beam), block 128: LSTM cell (gate order i, f, g, o; biases already in `gates`), new state into the `nx` half;
// h of every live row as three bf16 planes for joint.pred.  Kept hypotheses copy (h, c) from their parent.
__global__ void __launch_bounds__(128)
alsd_cell_kernel(const AlsdState st, const float* __restrict__ gates, int Hp, __nv_bfloat16* __restrict__ planes) {
  const int r = blockIdx.x, b = r / st.beam, k = r % st.beam;
  const bool live = !st.done[b] && k < st.nx.n_hyp[b];
  const bool ext = live && st.nx_tok[r] >= 0;
  const size_t pr = static_cast<size_t>(b) * st.beam + (live ? st.nx_parent[r] : 0);
  const float* g = gates + static_cast<size_t>(r) * 4 * Hp;
  __nv_bfloat16* row = planes + static_cast<size_t>(r) * 3 * Hp;
  for (int j = threadIdx.x; j < Hp; j += blockDim.x) {
    float h2 = 0.f, c2 = 0.f;
    if (ext) {
      const float ig = sigmoidf_accurate(g[j]), fg = sigmoidf_accurate(g[Hp + j]);
      const float cg = tanhf(g[2 * Hp + j]), og = sigmoidf_accurate(g[3 * Hp + j]);
      c2 = fg * st.cur.c[pr * Hp + j] + ig * cg;
      h2 = og * tanhf(c2);
    } else if (live) {
      h2 = st.cur.h[pr * Hp + j]; c2 = st.cur.c[pr * Hp + j];
    }
    st.nx.h[static_cast<size_t>(r) * Hp + j] = h2;
    st.nx.c[static_cast<size_t>(r) * Hp + j] = c2;
    __nv_bfloat16 hi, mid, lo;
    split3(h2, hi, mid, lo);
    row[j] = hi; row[Hp + j] = mid; row[2 * Hp + j] = lo;
  }
}

// grid (B), block 32, on the zeroed state: initial beam = one hypothesis [blank] with score 0 in the `nx` half (its predictor
// state is computed by one predictor pass with nx_tok = blank -> the zero embedding, from the zero state of the `cur` half)
__global__ void alsd_init_kernel(const AlsdState st, int blank) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  const int K = st.beam;
  st.nx.n_hyp[b] = 1; st.n_nodes[b] = 1;
  st.node_parent[static_cast<size_t>(b) * st.max_nodes] = -1;
  st.node_tok[static_cast<size_t>(b) * st.max_nodes] = blank;
  st.node_step[static_cast<size_t>(b) * st.max_nodes] = -1;
  for (int k = 1; k < K; ++k) st.nx_tok[b * K + k] = -1;
  const int r = b * K;
  st.nx.hash[r] = 1469598103934665603ull; st.nx_tok[r] = blank;
}

// Entry e of utterance b: y_sequence (leading blank) and the alignment steps of its tokens from the back-pointers of `node`;
// n is the full token count u, y / steps hold the first U_cap tokens.
__device__ void alsd_write_entry(const AlsdState& st, int b, int e, int node, int u, double score, int blank, int32_t* __restrict__ y_out,
                                 int32_t* __restrict__ step_out, int32_t* __restrict__ n_out, double* __restrict__ score_out, int U_cap) {
  const size_t i = static_cast<size_t>(b) * st.n_best + e;
  n_out[i] = u;
  score_out[i] = score;
  int32_t* y = y_out + i * (U_cap + 1);
  int32_t* steps = step_out + i * U_cap;
  const size_t tree = static_cast<size_t>(b) * st.max_nodes;
  y[0] = blank;
  int pos = u;
  while (node > 0 && pos > 0) {
    if (pos <= U_cap) {
      y[pos] = st.node_tok[tree + node];
      steps[pos - 1] = st.node_step[tree + node];
    }
    node = st.node_parent[tree + node];
    --pos;
  }
}

// grid (B), block 32: the N-best list of every utterance, one entry per lane.  With a finished hypothesis, the held entries
// of the list; with none, the last beam ranked by the same key, stable in slot order (entry 0 is the winner either way).
__global__ void __launch_bounds__(32)
alsd_output_kernel(const AlsdState st, int blank, int32_t* __restrict__ y_out, int32_t* __restrict__ step_out, int32_t* __restrict__ n_out,
                   double* __restrict__ score_out, int32_t* __restrict__ count_out, int32_t* __restrict__ pool_out,
                   int32_t* __restrict__ from_final_out, int U_cap) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int N = st.n_best;
  const int pool = st.fin_pool[b];
  if (pool > 0) {
    const size_t fo = static_cast<size_t>(b) * N;
    for (int e = lane; e < st.fin_count[b]; e += 32)
      alsd_write_entry(st, b, e, st.fin_node[fo + e], st.fin_u[fo + e], st.fin_score[fo + e], blank, y_out, step_out, n_out, score_out, U_cap);
  } else if (lane < st.cur.n_hyp[b]) {                 // slot `lane` of the last beam goes to entry `rank`
    const AlsdBeam& cur = st.cur;
    auto key = [&](int k) {
      const int r = b * st.beam + k;
      return st.score_norm ? cur.score[r] / static_cast<double>(cur.u[r] + 1) : cur.score[r];
    };
    const double mine = key(lane);
    int rank = 0;
    for (int k = 0; k < cur.n_hyp[b]; ++k) {
      const double other = key(k);
      rank += other > mine || (other == mine && k < lane);
    }
    const int r = b * st.beam + lane;
    if (rank < N) alsd_write_entry(st, b, rank, cur.node[r], cur.u[r], cur.score[r], blank, y_out, step_out, n_out, score_out, U_cap);
  }
  if (lane == 0 && count_out != nullptr) {
    const int n_pool = pool > 0 ? pool : st.cur.n_hyp[b];
    count_out[b] = n_pool < N ? n_pool : N;
    pool_out[b] = n_pool;
    from_final_out[b] = pool > 0 ? 1 : 0;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
void alsd_layout_state(AlsdState& st, Arena& a, char* base, int B, int beam, int Hp, int Hj, int max_nodes, bool score_norm, int n_best) {
  const size_t R = static_cast<size_t>(B) * beam, F = static_cast<size_t>(B) * n_best;
  auto take = [&](size_t bytes) { return reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(base) + a.take(bytes)); };
  st.beam = beam; st.max_nodes = max_nodes; st.score_norm = score_norm ? 1 : 0; st.n_best = n_best;
  for (AlsdBeam* m : {&st.cur, &st.nx}) {
    m->score = static_cast<double*>(take(R * 8)); m->hash = static_cast<unsigned long long*>(take(R * 8));
    m->u = static_cast<int*>(take(R * 4)); m->node = static_cast<int*>(take(R * 4));
    m->h = static_cast<float*>(take(R * Hp * 4)); m->c = static_cast<float*>(take(R * Hp * 4)); m->pp = static_cast<float*>(take(R * Hj * 4));
    m->n_hyp = static_cast<int*>(take(static_cast<size_t>(B) * 4));
  }
  st.nx_parent = static_cast<int*>(take(R * 4)); st.nx_tok = static_cast<int*>(take(R * 4)); st.row_t = static_cast<int*>(take(R * 4));
  st.cand_logp = static_cast<float*>(take(R * (kMaxBeam + 1) * 4)); st.cand_tok = static_cast<int*>(take(R * kMaxBeam * 4));
  int* ints = static_cast<int*>(take(static_cast<size_t>(B) * 4 * 4));
  st.done = ints; st.n_nodes = ints + B; st.fin_count = ints + 2 * B; st.fin_pool = ints + 3 * B;
  st.fin_key = static_cast<double*>(take(F * 8)); st.fin_score = static_cast<double*>(take(F * 8));
  st.fin_node = static_cast<int*>(take(F * 4)); st.fin_u = static_cast<int*>(take(F * 4));
  int* tree = static_cast<int*>(take(static_cast<size_t>(B) * max_nodes * 4 * 3));
  st.node_parent = tree; st.node_tok = tree + static_cast<size_t>(B) * max_nodes; st.node_step = tree + 2 * static_cast<size_t>(B) * max_nodes;
  st.n_done = static_cast<int*>(take(4));
}

cudaError_t alsd_launch_init(const AlsdState& st, int B, int blank, cudaStream_t s) {
  alsd_init_kernel<<<B, 32, 0, s>>>(st, blank);
  return cudaGetLastError();
}
cudaError_t alsd_launch_rows(const AlsdState& st, int B, const float* enc_proj, const int32_t* enc_len, int T_max, int Hj, int step, void* planes, cudaStream_t s) {
  alsd_rows_kernel<<<B * st.beam, 128, 0, s>>>(st, enc_proj, enc_len, T_max, Hj, step, static_cast<__nv_bfloat16*>(planes));
  return cudaGetLastError();
}
cudaError_t alsd_launch_reduce(const AlsdState& st, int B, const float* logits, int ld, int V, cudaStream_t s) {
  alsd_reduce_kernel<<<B * st.beam, 256, 0, s>>>(st, logits, ld, V);
  return cudaGetLastError();
}
cudaError_t alsd_launch_select(const AlsdState& st, int B, const int32_t* enc_len, int step, double u_max_ratio, bool recombine_returns_input, cudaStream_t s) {
  alsd_select_kernel<<<B, 32, 0, s>>>(st, enc_len, step, u_max_ratio, recombine_returns_input ? 1 : 0);
  return cudaGetLastError();
}
cudaError_t alsd_launch_lstm_in(const AlsdState& st, int B, const float* embed, int Hp, void* planes, cudaStream_t s) {
  alsd_lstm_in_kernel<<<B * st.beam, 128, 0, s>>>(st, embed, Hp, static_cast<__nv_bfloat16*>(planes));
  return cudaGetLastError();
}
cudaError_t alsd_launch_cell(const AlsdState& st, int B, const float* gates, int Hp, void* planes, cudaStream_t s) {
  alsd_cell_kernel<<<B * st.beam, 128, 0, s>>>(st, gates, Hp, static_cast<__nv_bfloat16*>(planes));
  return cudaGetLastError();
}
cudaError_t alsd_launch_output(const AlsdState& st, int B, int blank, int32_t* y, int32_t* steps, int32_t* n, double* score, int32_t* count,
                               int32_t* pool, int32_t* from_final, int U_cap, cudaStream_t s) {
  alsd_output_kernel<<<B, 32, 0, s>>>(st, blank, y, steps, n, score, count, pool, from_final, U_cap);
  return cudaGetLastError();
}

}  // namespace rs
