// Host-side launch interface of the sm_90a kernels (internal to librs_engine.so).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rs {

// Memory layout: regions taken one after another, each starting 256-byte aligned (offsets from a 256-byte-aligned base).
struct Arena {
  size_t off = 0;
  size_t take(size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~static_cast<size_t>(255); return o; }
};

// out = epi(A[M,K] * W[N,K]^T); the output row pitch is N (N / 2 for RS_EPI_BIAS_GLU_BF16)
struct GemmArgs {
  const void* a;       // bf16 [M,K] row-major
  const void* w;       // bf16 [N,K] row-major (nn.Linear layout)
  const float* bias;   // f32 [N] or nullptr
  const float* resid;  // f32 [M,N] for RS_EPI_RESID_F32 (may be out; otherwise copied to out before the launch)
  void* out;
  int M, N, K;
  int epilogue;        // rs_epilogue
  float alpha;
  // RS_EPI_QKV_VT: columns >= split go, transposed, to out2 (bf16 [N - split, ld2]; ld2 >= M, only columns < M are written)
  void* out2 = nullptr; int split = 0, ld2 = 0;
};

// Returns cudaSuccess or the failing CUDA error; err (>=256 B) receives a description.
cudaError_t launch_gemm(const GemmArgs& g, int num_sms, cudaStream_t stream, char* err);

// bf16 row-major [rows, cols] with a row pitch of ld elements -> 2-D TMA map with a (box_rows x 64) box and 128B swizzle,
// out-of-bounds elements read as zero.  Returns false and writes a description into err (>=256 B) on failure.
bool make_tmap_bf16(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, char* err);

cudaError_t launch_layernorm(const float* x, const float* gamma, const float* beta, float* out_f32,
                             void* out_bf16, const float* gamma2, const float* beta2, int rows, int d,
                             float eps, cudaStream_t stream);

struct SubsampleArgs {
  const float* mel; const int32_t* mel_len;   // un-normalised log-mel [B, F_max, n_mels] and valid frames
  const float* mel_stats;                     // [B, n_mels, 2] (mean, 1 / (std + eps)) from the log-mel kernel
  int B, F_max, n_mels, C;
  const float* w0; const float* b0;      // conv.0  [C,9], [C]
  const float* wd1; const float* bd1;    // conv.2  [C,9], [C]
  void* out1;                            // bf16 [B,T2,F2,C]
  int T1, F1, T2, F2;
};
cudaError_t launch_sub_conv0_dw1(const SubsampleArgs& a, cudaStream_t stream);
// depthwise 3x3 s2 on channels-last bf16 [B,Tin,Fin,C] (rows t >= len_in(b) read as zero)
cudaError_t launch_sub_dw(const void* in, void* out, const float* w, const float* b, const int32_t* mel_len,
                          int len_shift, int B, int Tin, int Fin, int Tout, int Fout, int C, cudaStream_t stream);

// GLU output u bf16 [B*T_max, d] -> depthwise conv (k taps, BN folded) -> swish -> bf16
cudaError_t launch_conv_dw(const void* u, void* out, const float* w /*[k,d]*/, const float* shift /*[d]*/,
                           const int32_t* enc_len, int B, int T_max, int d, int k, cudaStream_t stream);

struct AttnArgs {
  const void* qkv;       // bf16 [B*T_max, 3*d]: q + pos_bias_u | k | (unused; V goes to vt)
  const void* pos;       // bf16 [H, n_rel_pad, dk]: linear_pos(pos_emb) per head, rows beyond the 2w+1 offsets zero (packed at load)
  const float* bd_bias;  // f32 [H, n_rel_pad]: (pos_bias_v - pos_bias_u) . pos[h][c]
  int n_rel_pad;
  const float* bias_u;   // f32 [H, dk]
  void* out;             // bf16 [B*T_max, d]
  const int32_t* enc_len;
  int B, T_max, H, dk, w_left, w_right, n_global;
  const void* vt = nullptr; int ld_vt = 0;   // V^T bf16 [H*dk, ld_vt] written by the QKV GEMM (RS_EPI_QKV_VT)
};
bool attention_tc_supported(const AttnArgs& a);
cudaError_t launch_attention_tc(const AttnArgs& a, cudaStream_t stream);

// n-gram LM of the greedy decode's shallow fusion (reazonspeech_b200/ngram_lm.py builds it; decode_spec.cu describes the
// layout).  Device arrays, 16-byte aligned; order == 0: no LM.
struct NgramLM {
  const float* cb = nullptr;            // [n_states] summed back-off weight of the state's chain (root excluded), nats x alpha
  const int32_t* chain = nullptr;       // [n_states][order - 1] the state, its back-off state, ... (0 = root pads)
  const int32_t* arc_begin = nullptr;   // [n_states + 1] CSR of the arcs, sorted by token within a state
  const int32_t* arc_tok = nullptr;     // [n_arcs]
  const int32_t* arc_to = nullptr;      // [n_arcs] state reached by emitting arc_tok from the arc's state
  const float* arc_w = nullptr;         // [n_arcs] LM term of the arc minus cb of its state
  const float* uni_w = nullptr;         // [pitch] root row: LM term of every token in the empty context
  const int32_t* uni_to = nullptr;      // [pitch] root row: state reached from the empty context
  int order = 0, n_states = 0, n_arcs = 0, pitch = 0, start_state = 0;
};

struct DecodeArgs {
  const float* enc_proj;      // f32 [B*T_max, Hj]  (joint.enc applied to every frame)
  const int32_t* enc_len;
  const void* w_out;          // bf16 [V+1, Hj]
  const float* b_out;         // f32 [V+1]
  const void* w_lstm;         // bf16 [4*Hp, 2*Hp]  (W_ih | W_hh, gate order i,f,g,o)
  const float* gate_tab;      // f32 [V+1, 4*Hp]: W_ih . embed[k] + b_ih + b_hh (the input half of the gates, per token)
  const void* w_pred;         // bf16 [Hj, Hp]
  const float* b_pred;        // f32 [Hj]
  int32_t* tokens; int32_t* frames; int32_t* n_tok;
  int B, T_max, Hj, Hp, V, U_max, max_symbols;
  float* stats = nullptr;     // f32 [B, U_max, 4] (lp, H1, A_alpha, G_alpha) per stored token; nullptr: no confidence statistics
  float alpha = 0.f;          // > 0 and finite when stats is set
  // phrase boosting (boosting.py): f32 bonus / i32 next [boost_states, boost_pitch], pitch >= V and a multiple of 4, both
  // 16-byte aligned; nullptr: no boosting
  const float* boost_bonus = nullptr;
  const int32_t* boost_next = nullptr;
  int boost_states = 0, boost_pitch = 0;
  NgramLM lm;                 // n-gram LM shallow fusion; lm.order == 0: none
  // resume (streaming): states != nullptr makes row b decode frames [dec_begin[b] (nullptr: 0), enc_len[b]) from the record
  // slot[b] of states (stream_state_bytes each, 16-byte aligned, distinct slots) and store its state there; nullptr: every row
  // starts fresh at frame 0
  const int32_t* dec_begin = nullptr;
  const int32_t* slot = nullptr;
  void* states = nullptr;
  // phrase boosting per row: [B] row b's root state, in [0, boost_states) (checked by the caller); nullptr: the root is 0
  const int32_t* boost_root = nullptr;
};
// Bytes of one stream record of the resumed decode (decode_spec.cu describes the layout)
size_t stream_state_bytes(int Hj, int Hp);
// Byte offsets of the decode workspace's regions and its size (decode_spec.cu describes the regions)
struct SpecWorkspace { size_t hbuf, rec, ppbuf, counters, prof, best, conf, lm_ring, total; };
SpecWorkspace rnnt_spec_workspace(int B, int Hj, int Hp, int num_sms);
// windowed (kFrames per iteration) persistent decode, joint on wgmma (decode_spec.cu); workspace laid out by rnnt_spec_workspace();
// a.stats != nullptr selects the instance that also reduces the softmax statistics of every emitted token,
// a.boost_bonus != nullptr the one that adds the phrase-boosting bonus before the argmax, a.lm.order != 0 the one that adds the
// n-gram LM term
cudaError_t launch_rnnt_greedy_spec(const DecodeArgs& a, void* workspace, int num_sms, cudaStream_t stream);
// The decode kernel's own LM lookup on n arbitrary (state, token) pairs (device arrays): score[i] = the LM term the decode adds to
// token tokens[i]'s logit in state states[i], next[i] = the state emitting it leads to (decode_spec.cu)
cudaError_t launch_ngram_lm_eval(const NgramLM& lm, int V, int num_sms, const int32_t* states, const int32_t* tokens, int n,
                                 float* score, int32_t* next, cudaStream_t stream);

// Forced alignment on the RNN-T lattice (align.cu; semantics: reazonspeech_b200/alignment.py).  Lattice arrays are
// [B][T_max][U_max + 1]; labels [B][U_max]; h / pred_proj [B][U_max + 1][Hp / Hj]; c [B][Hp].
struct AlignArgs {
  const float* enc_proj;      // f32 [B*T_max, Hj]  (joint.enc applied to every frame)
  const int32_t* enc_len;
  const int32_t* labels;
  const int32_t* label_len;
  const void* w_out;          // bf16 [V+1, Hj]
  const float* b_out;         // f32 [V+1]
  const void* w_lstm;         // bf16 [4*Hp, 2*Hp]  (W_ih | W_hh, gate order i,f,g,o)
  const float* gate_tab;      // f32 [V+1, 4*Hp]
  const void* w_pred;         // bf16 [Hj, Hp]
  const float* b_pred;        // f32 [Hj]
  int B, T_max, U_max, Hj, Hp, V;
  float* h; float* c; float* pred_proj;
  float* lp_blank; float* lp_emit;
  uint8_t* choice;            // Viterbi predecessor of every cell (1: the emission from (t, u - 1))
  int32_t* frames; float* token_lp; float* viterbi; float* loglik;
  int32_t* seg; float* frame_lp;  // segment alignment only: (s, e) [B][2], f32 [B][T_max]
  // banded alignment only: row (b, u) holds the frames [band_lo, band_hi) at band_off + (t - band_lo) of lp_blank / lp_emit /
  // choice ([B][U_max + 1] each); band_tiles lists the (utterance, t0, u0) lattice tiles that meet the band; the DP keeps
  // band_pitch cells per live diagonal and writes edge [B]
  const int32_t* band_lo; const int32_t* band_hi; const int64_t* band_off; const int4* band_tiles;
  int band_pitch; int32_t* edge;
};
// shapes the kernels implement (false: err, >= 256 B, says why)
bool align_supported(int Hj, int Hp, int V, int U_max, char* err);
// teacher-forced predictor step u (h, c) and then joint.pred of every row
cudaError_t launch_align_lstm_step(const AlignArgs& a, int u, cudaStream_t stream);
cudaError_t launch_align_pred_proj(const AlignArgs& a, cudaStream_t stream);
// lp_blank / lp_emit of every valid cell (err >= 256 B receives a tensor-map failure)
cudaError_t launch_rnnt_lattice(const AlignArgs& a, cudaStream_t stream, char* err);
// forward + Viterbi recursions and backtrace -> frames, token_lp, viterbi, loglik
cudaError_t launch_rnnt_align_dp(const AlignArgs& a, cudaStream_t stream);
// segment alignment (free start and end) -> seg, frames, token_lp, frame_lp, viterbi, loglik
cudaError_t launch_rnnt_segment_dp(const AlignArgs& a, cudaStream_t stream);
// banded alignment: the n_tiles tiles of a.band_tiles into banded storage; then the recursions and backtrace on the band's
// cells -> frames, token_lp, viterbi, loglik, edge (band_dp_smem: shared memory for a.band_pitch)
cudaError_t launch_rnnt_lattice_band(const AlignArgs& a, int n_tiles, cudaStream_t stream, char* err);
cudaError_t launch_rnnt_band_dp(const AlignArgs& a, cudaStream_t stream);
size_t band_dp_smem(int pitch);

// Keyword spotting (align.cu, spot.cu; semantics: reazonspeech_b200/keywords.py): the AlignArgs of the B keywords, whose enc_proj
// and enc_len are the n_rec recordings'; pair p = r * B + k, and the lattice arrays are the pairs'.
struct SpotArgs {
  int n_rec;
  float threshold; int max_hits;
  float* E; int32_t* S;                       // [pairs][T_max]: E(e), S(e) (NaN, -1 where no segment ends)
  int32_t* span; float* score; float* conf;   // [pairs][max_hits] (x2: s, e), E(e), m(e)
  int32_t* frames; float* token_lp;           // [pairs][max_hits][U_max]
  int32_t* count;                             // [pairs]
};
constexpr int kSpotMaxLabels = 32;
constexpr int kSpotMaxHits = 256;
// the lattice of every (recording, keyword) pair
cudaError_t launch_rnnt_lattice_pairs(const AlignArgs& a, int n_rec, cudaStream_t stream, char* err);
// the free-start recursion of every pair -> E, S and a.choice; then the hits of every pair -> span ... count
cudaError_t launch_rnnt_spot_dp(const AlignArgs& a, const SpotArgs& sp, cudaStream_t stream);
cudaError_t launch_rnnt_spot_pick(const AlignArgs& a, const SpotArgs& sp, cudaStream_t stream);
// shared memory of the pick kernel (false when T_max frames do not fit)
bool spot_pick_fits(int T_max, int max_hits);

// Streaming keyword spotting (spot_stream.cu; semantics: keywords.py, "Streaming").  One record per (stream slot, keyword) of
// spot_record(U_max, ring_cap).total bytes; pair p = b * n_kw + k of a call is row b's stream (record slot[b]) and keyword k.
struct SpotRecord { size_t column, lists, ring, total; };
__host__ __device__ inline size_t spot_entry_bytes(int U_max) { return 12 + static_cast<size_t>(8) * U_max; }
__host__ __device__ inline SpotRecord spot_record(int U_max, int ring_cap) {
  SpotRecord r;
  r.column = 32;                                                    // header int32[8]
  r.lists = r.column + static_cast<size_t>(12) * U_max;
  r.ring = r.lists + static_cast<size_t>(8) * U_max * U_max;
  r.total = (r.ring + ring_cap * spot_entry_bytes(U_max) + 15) & ~static_cast<size_t>(15);
  return r;
}
constexpr int kSpotHitInts = 5;                                     // a decided hit: row, keyword, s, e, forced
struct SpotStreamArgs {
  const int32_t* dec_begin; const int32_t* dec_end; const int32_t* slot; const int32_t* last;   // device [B]
  int B, n_kw, U_max, C;                      // C: the compact block's frames per row (>= every dec_end - dec_begin)
  int delay, ring_cap;                        // D frames; ring entries per pair
  float threshold;
  const int32_t* label_len;                   // [n_kw]
  uint8_t* records;                           // [n_slots][n_kw] records
  int32_t* len;                               // [B] dec_end - dec_begin (written by the gather)
  float* E_out; int32_t* S_out; int T_out;    // optional [B][n_kw][T_out] at buffer frames [dec_begin, dec_end)
  int32_t* sigma_out;                         // optional [B][n_kw]: sigma(t) after the step (-1: no frame seen)
  int32_t* n_hits; int hit_cap;               // the decided hits: [hit_cap] x (meta i32[5], (score, confidence) f32[2],
  int32_t* hit_meta; float* hit_val;          //   frames i32[U_max], token_lp f32[U_max])
  int32_t* hit_frames; float* hit_lp;
};
// rows [dec_begin, dec_end) of encp f32 [B][T_max][Hj] -> out f32 [B][C][Hj], len
cudaError_t launch_spot_gather(const float* encp, int T_max, int Hj, const SpotStreamArgs& s, float* out, cudaStream_t stream);
// a: the pairs' lattice (rnnt_lattice_kernel<true> over the gathered block: B = n_kw keywords, T_max = C, enc_len = s.len)
cudaError_t launch_rnnt_spot_resume_dp(const AlignArgs& a, const SpotStreamArgs& s, cudaStream_t stream);
cudaError_t launch_rnnt_spot_resume_pick(const SpotStreamArgs& s, cudaStream_t stream);
size_t spot_pick_stream_smem(int ring_cap);

// norm_audio on the device: polyphase resampling to 16 kHz + channel average + transcribe()'s zero padding (resample.cu)
struct ResampleArgs {
  const void* in; bool in_i16;          // [B, C, L_in_max] f32, or int16 PCM (scaled by 2^-15)
  const int32_t* len_in;                // [B] valid samples per utterance (per channel)
  int B, C, L_in_max;
  const float* taps; int taps_per_phase, up, down, n_pre_remove;   // polyphase FIR from engine.py::resample_taps: taps[up][taps_per_phase]
  int pad;                              // zero samples in front of and behind every resampled utterance
  float* out; int L_out_row;            // [B, L_out_row] f32, fully written (zeros outside the utterance)
  int32_t* len_out;                     // [B] resampled length + 2 * pad
};
cudaError_t launch_resample_mono(const ResampleArgs& a, cudaStream_t stream);

// small utility kernels
cudaError_t launch_f32_to_bf16(const float* in, void* out, int64_t n, cudaStream_t stream);
cudaError_t launch_zero_pad_rows(float* x, const int32_t* len, int B, int T_max, int d, cudaStream_t stream);

}  // namespace rs
