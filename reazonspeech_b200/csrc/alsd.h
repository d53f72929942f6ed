// Host-side interface of the ALSD beam-search kernels (decode_alsd.cu); internal to librs_engine.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace rs {

// One beam of a batched ALSD search, R = B * beam rows.
struct AlsdBeam {
  double* score; unsigned long long* hash; int* u; int* node;                 // [R] log-probability, sequence hash, tokens so far, back-pointer node
  float* h; float* c; float* pp;                                              // [R, Hp], [R, Hp], [R, Hj]: predictor state AFTER the last token, joint.pred of it
  int* n_hyp;                                                                 // [B] hypotheses in the beam
};

// Device state of a batched ALSD search.  `cur` is the beam of the current step, `nx` the one being built for the next; the
// host swaps the two after every predictor pass.
struct AlsdState {
  int beam, max_nodes, score_norm, n_best;
  AlsdBeam cur, nx;
  int* nx_parent; int* nx_tok; int* row_t;                                    // [R] parent slot and token (-1: kept) of a new hypothesis; frame of a live row (-1: none)
  float* cand_logp; int* cand_tok;                                            // [R, 9]: log p(blank), then the beam best classes; [R, 8] their indices
  int* done; int* n_nodes;                                                    // [B]
  // The finished hypotheses of utterance b: NeMo's `final` list sorted by key, stable, truncated to n_best.  Entry e of b is
  // [b * n_best + e]; fin_count[b] entries are held, fin_pool[b] hypotheses have finished (the length of NeMo's list).
  double* fin_key; double* fin_score; int* fin_node; int* fin_u;              // [B, n_best]
  int* fin_count; int* fin_pool;                                              // [B]
  int* node_parent; int* node_tok; int* node_step;                            // [B, max_nodes] back-pointer tree: node 0 = the leading blank
  int* n_done;                                                                // utterances whose search has ended
};

// Lays the state out in regions taken from `a`, pointers relative to `base`: with base == nullptr only to size it.
void alsd_layout_state(AlsdState& st, Arena& a, char* base, int B, int beam, int Hp, int Hj, int max_nodes, bool score_norm, int n_best);
cudaError_t alsd_launch_init(const AlsdState& st, int B, int blank, cudaStream_t s);
cudaError_t alsd_launch_rows(const AlsdState& st, int B, const float* enc_proj, const int32_t* enc_len, int T_max, int Hj, int step, void* planes, cudaStream_t s);
cudaError_t alsd_launch_reduce(const AlsdState& st, int B, const float* logits, int ld, int V, cudaStream_t s);
cudaError_t alsd_launch_select(const AlsdState& st, int B, const int32_t* enc_len, int step, double u_max_ratio, bool recombine_returns_input, cudaStream_t s);
cudaError_t alsd_launch_lstm_in(const AlsdState& st, int B, const float* embed, int Hp, void* planes, cudaStream_t s);
cudaError_t alsd_launch_cell(const AlsdState& st, int B, const float* gates, int Hp, void* planes, cudaStream_t s);
// The first fin_count[b] entries (with none finished: the last beam ranked by the same key) -> y [B, n_best, U_cap + 1],
// steps [B, n_best, U_cap], n / score [B, n_best]; count / pool / from_final [B] when not null.
cudaError_t alsd_launch_output(const AlsdState& st, int B, int blank, int32_t* y, int32_t* steps, int32_t* n, double* score, int32_t* count,
                               int32_t* pool, int32_t* from_final, int U_cap, cudaStream_t s);

}  // namespace rs
