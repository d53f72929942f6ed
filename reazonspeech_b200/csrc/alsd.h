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
  int beam, max_nodes, score_norm;
  AlsdBeam cur, nx;
  int* nx_parent; int* nx_tok; int* row_t;                                    // [R] parent slot and token (-1: kept) of a new hypothesis; frame of a live row (-1: none)
  float* cand_logp; int* cand_tok;                                            // [R, 9]: log p(blank), then the beam best classes; [R, 8] their indices
  int* done; int* has_final; int* n_nodes; int* final_node; int* final_u;     // [B]
  double* final_key; double* final_score;                                     // [B]
  int* node_parent; int* node_tok; int* node_step;                            // [B, max_nodes] back-pointer tree: node 0 = the leading blank
  int* n_done;                                                                // utterances whose search has ended
};

// Lays the state out in regions taken from `a`, pointers relative to `base`: with base == nullptr only to size it.
void alsd_layout_state(AlsdState& st, Arena& a, char* base, int B, int beam, int Hp, int Hj, int max_nodes, bool score_norm);
cudaError_t alsd_launch_init(const AlsdState& st, int B, int blank, cudaStream_t s);
cudaError_t alsd_launch_rows(const AlsdState& st, int B, const float* enc_proj, const int32_t* enc_len, int T_max, int Hj, int step, void* planes, cudaStream_t s);
cudaError_t alsd_launch_reduce(const AlsdState& st, int B, const float* logits, int ld, int V, cudaStream_t s);
cudaError_t alsd_launch_select(const AlsdState& st, int B, const int32_t* enc_len, int step, double u_max_ratio, bool recombine_returns_input, cudaStream_t s);
cudaError_t alsd_launch_lstm_in(const AlsdState& st, int B, const float* embed, int Hp, void* planes, cudaStream_t s);
cudaError_t alsd_launch_cell(const AlsdState& st, int B, const float* gates, int Hp, void* planes, cudaStream_t s);
cudaError_t alsd_launch_output(const AlsdState& st, int B, int blank, int32_t* y, int32_t* steps, int32_t* n, double* score, int U_cap, cudaStream_t s);

}  // namespace rs
