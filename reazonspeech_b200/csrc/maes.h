// Host-side interface of the MAES beam-search kernels (decode_maes.cu); internal to librs_engine.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace rs {

constexpr int kMaesMaxSteps = 4;
constexpr int kMaesMaxC = 12;          // candidates per hypothesis: beam (<= 8) + expansion_beta (<= 4)

// The kept hypotheses of a batched MAES search, R = B * beam slots.  P = max(prefix_alpha, 1) predictor outputs are kept per
// hypothesis (plane d: dec_out[-1 - d]), P + 1 prefix hashes (hh[d]: the sequence without its last d tokens) and its last P tokens
// (th[d]: the d-th from the end), which is what the prefix search reads.
struct MaesKept {
  double* score; unsigned long long* hh; int* th; int* u; int* node; int* lm;   // [R], [R][P + 1], [R][P], [R] x 3
  float* h; float* c; float* pp;                                              // [R, Hp], [R, Hp], [P][R, Hj]
  int* n_hyp;                                                                 // [B]
};

// The hypotheses one expansion round adds (list_exp), compacted over the batch: utterance b's rows are [begin[b], begin[b] + cnt[b]).
// par is the parent: a kept slot in round 0, a row of the previous round after it.
struct MaesRows {
  int cap;
  double* score; unsigned long long* hh; int* th; int* u; int* lm; int* par; int* tok; int* utt;
  float* h; float* c; float* pp;                                              // [cap, Hp], [cap, Hp], [P][cap, Hj]
  int* begin; int* cnt;                                                       // [B]
};

struct MaesState {
  int B, K, C, S, P, alpha, W, lb_cap, max_nodes, score_norm, rri;
  double gamma;
  MaesKept cur, nx;
  MaesRows rows[kMaesMaxSteps];
  int* m;                                                  // [kMaesMaxSteps] rows taken in each round (atomic compaction)
  int* prow_t; float* plse; float* pcand_lp; int* pcand_tok;   // prefix-pass rows [R * P] (slot r, depth d: r * P + d); top-C of d = 0: [R][C]
  float* rcand_lp; int* rcand_tok; float* rblank;          // joint of a round's rows: top-C [cap][C], log p(blank) [cap]
  int* ord;                                                // [R] kept slots by length, longest first (stable)
  int* fstate;                                             // [B] 0: expanding, 1: the frame ended early (no expansion), 2: past enc_len
  double* lb_score; int* lb_round; int* lb_idx; int* lb_n;  // list_b [B][lb_cap] (round -1: a kept slot), [B]
  double* sg_score; int* sg_par; int* sg_tok;              // a round's expansions per utterance before compaction [B][W]
  double* c_score; unsigned long long* c_hash; int* c_u; int* c_first;   // select: candidates [B][lb_cap + W]
  int* sel_round; int* sel_idx;                            // [R] source of each new kept slot
  int* n_nodes; int* node_parent; int* node_tok; int* node_frame;   // [B], [B][max_nodes]: node 0 = the leading blank
};

void maes_layout_state(MaesState& st, Arena& a, char* base, int B, int K, int C, int S, int P, int Hp, int Hj, int max_nodes);
cudaError_t maes_launch_init(const MaesState& st, int blank, int lm_start, cudaStream_t s);
cudaError_t maes_launch_init_kept(const MaesState& st, int Hp, int Hj, cudaStream_t s);
cudaError_t maes_launch_prefix_rows(const MaesState& st, const float* encp, const int32_t* enc_len, int T_max, int Hj, int t, void* planes, cudaStream_t s);
cudaError_t maes_launch_reduce(const MaesState& st, int n, int M, const float* logits, int ld, int V, cudaStream_t s);
cudaError_t maes_launch_prefix(const MaesState& st, const float* logits, int ld, cudaStream_t s);
cudaError_t maes_launch_expand(const MaesState& st, int n, int blank, const NgramLM& lm, cudaStream_t s);
cudaError_t maes_launch_lstm_in(const MaesState& st, int n, int M, const float* embed, int Hp, int Hj, int blank, void* planes, cudaStream_t s);
cudaError_t maes_launch_cell(const MaesState& st, int n, int M, const float* gates, int Hp, void* planes, cudaStream_t s);
cudaError_t maes_launch_rows(const MaesState& st, int n, int M, const float* encp, int T_max, int Hj, int t, void* planes, cudaStream_t s);
cudaError_t maes_launch_select(const MaesState& st, int t, cudaStream_t s);
cudaError_t maes_launch_gather(const MaesState& st, int Hp, int Hj, cudaStream_t s);
cudaError_t maes_launch_output(const MaesState& st, int n_best, int blank, int32_t* y, int32_t* frames, int32_t* n, double* score, int32_t* count,
                               int U_cap, cudaStream_t s);

}  // namespace rs
