/*
 * rs_engine.h -- C ABI of the H100-native FastConformer-RNNT engine.
 *
 * The reference (reazon-research/ReazonSpeech) has no native layer: its hot path is one
 * opaque Python call into NeMo,
 *     model.transcribe([waveform], batch_size=1, return_hypotheses=True, verbose=...)
 *                                              pkg/nemo-asr/src/transcribe.py:48-53
 * whose result is consumed as hyp.y_sequence / hyp.timestamp (pkg/nemo-asr/src/decode.py:40,44).
 * This header is the boundary a binding for that call site would target (INTEGRATION.md shows
 * the ctypes stub).  Each entry point names the NeMo stage it replaces (SURVEY.md section 8a).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch / C++ types.
 *   - every function returns RS_OK (0) or a negative rs_status; rs_last_error() gives the text.
 *   - "dev" pointers are CUDA device pointers on the engine's device, caller-allocated unless
 *     stated; "host" pointers are host memory (pinned for best throughput).
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*); no hidden synchronisation
 *     except where stated (rs_transcribe_batch synchronises before returning).
 *   - an engine is bound to one device and is not re-entrant; distinct engines are independent.
 *   - batched activations are padded row-major [B, T_max, ...] with a per-utterance length
 *     vector; rows at or beyond an utterance's length never influence valid rows.
 */
#ifndef RS_ENGINE_H_
#define RS_ENGINE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum rs_status {
  RS_OK = 0,
  RS_ERR_INVALID_ARG = -1,
  RS_ERR_CUDA = -2,
  RS_ERR_MISSING_WEIGHT = -3,
  RS_ERR_WORKSPACE = -4,
  RS_ERR_UNSUPPORTED = -5
} rs_status;

/* Mirrors the fields of the .nemo model_config.yaml the path consumes (SURVEY.md App. A.1). */
typedef struct rs_model_config {
  int32_t sample_rate, n_window_size, n_window_stride, n_fft, n_mels;
  float preemph, log_zero_guard, norm_eps;
  int32_t n_layers, d_model, n_heads, d_ff, conv_kernel, sub_channels;
  int32_t att_left, att_right, global_tokens;
  float xscale, ln_eps;
  int32_t vocab_size;   /* blank id == vocab_size; classes == vocab_size + 1 */
  int32_t pred_hidden, joint_hidden, max_symbols;
} rs_model_config;

/* One packed weight tensor, resident on the device (packing: reazonspeech_b200/engine.py::pack_weights is the definition of
 * the names, shapes and value transforms -- e.g. "pred.gate_tab" f32 [V+1, 4*pred_hidden] = W_ih . embed[k] + b_ih + b_hh,
 * the per-token input half of the LSTM gates; rs_engine_create names the first tensor it misses in rs_last_error). */
typedef enum rs_dtype { RS_F32 = 0, RS_BF16 = 1, RS_I32 = 2 } rs_dtype;
typedef struct rs_tensor {
  const char* name;
  const void* dev_ptr;
  int32_t dtype;     /* rs_dtype */
  int64_t numel;
} rs_tensor;

typedef struct rs_engine rs_engine;

/* Epilogues of the wgmma GEMM  out = epi(A[M,K] * W[N,K]^T)  (SURVEY.md App. A.3). */
typedef enum rs_epilogue {
  RS_EPI_BIAS_BF16 = 0,       /* out_bf16[M,N]   = acc + bias                                  */
  RS_EPI_BIAS_RELU_BF16 = 1,  /* out_bf16[M,N]   = relu(acc + bias)                            */
  RS_EPI_BIAS_SWISH_BF16 = 2, /* out_bf16[M,N]   = swish(acc + bias)                           */
  RS_EPI_BIAS_GLU_BF16 = 3,   /* out_bf16[M,N/2] = a * sigmoid(g); W rows interleaved 16/16    */
  RS_EPI_RESID_F32 = 4,       /* out_f32[M,N]    = resid + alpha * (acc + bias), added into out in L2 by a TMA f32
                                 reduction (out may alias resid; a separate resid is first copied to out on the same
                                 stream).  Rounded twice, fl(fl(alpha * s) + resid) with s = fl(acc + bias): bit-equal
                                 to resid + RS_EPI_BIAS_F32(alpha) computed in fp32, and to a fused multiply-add
                                 whenever alpha is a power of two.  Subnormal residuals and sums are kept, not
                                 flushed to zero.                                                                     */
  RS_EPI_BIAS_F32 = 5,        /* out_f32[M,N]    = alpha * (acc + bias)                        */
  RS_EPI_BIAS_F16 = 6,        /* out_f16[M,N]    = acc + bias  (IEEE half)                          */
  RS_EPI_QKV_VT = 7           /* fused QKV projection: columns [0, split) -> out_bf16[M, ldo] as RS_EPI_BIAS_BF16,
                                 columns [split, N) -> TRANSPOSED into out2_bf16[N - split, ld2] (V^T, keys contiguous:
                                 the K-major B operand of the attention kernel's P.V product)               */
} rs_epilogue;

/* ---- lifetime -------------------------------------------------------------------------- */
/* Replaces EncDecRNNTBPEModel.from_pretrained (transcribe.py:26-28) below the Python loader. */
int rs_engine_create(const rs_model_config* cfg, const rs_tensor* weights, int n_weights,
                     int device, rs_engine** out);
void rs_engine_destroy(rs_engine* e);
/* Text of the last failure on `e` (or of the last failed rs_engine_create when e == NULL). */
const char* rs_last_error(const rs_engine* e);

/* Scratch the engine needs for a batch of B utterances of at most L_max samples.  It includes the ring of the n-gram LM
 * fusion (96 * B * (multiprocessors / 4) bytes: about 100 KB for B = 32 on 132 multiprocessors) whether or not an LM is set,
 * so that rs_set_ngram_lm never invalidates a workspace already set. */
int rs_workspace_bytes(const rs_engine* e, int B, int L_max, size_t* bytes);
int rs_set_workspace(rs_engine* e, void* dev_ptr, size_t bytes);

/* ---- shape arithmetic --------------------------------------------------------------------
 * rs_mel_frames / rs_enc_frames: TENSOR time sizes for a buffer of n_samples (frames of the centred
 * STFT = n/hop + 1; ConvSubsampling.calc_length applied to it three times, rounded up to a multiple of 8):
 * what callers allocate.
 * rs_mel_valid / rs_enc_valid: the VALID lengths of an utterance of n_samples
 * (FilterbankFeatures.get_seq_len = n/hop, then calc_length x3): what mel_len / enc_len will hold. */
int rs_mel_frames(const rs_engine* e, int n_samples);
int rs_enc_frames(const rs_engine* e, int n_samples);
int rs_mel_valid(const rs_engine* e, int n_samples);
int rs_enc_valid(const rs_engine* e, int n_samples);

/* ---- stages (each is also a parity-test seam) --------------------------------------------- */
/* N1 AudioToMelSpectrogramPreprocessor: wav f32[B,L_max] + len -> mel f32[B,F_max,n_mels]
 * (time-major, per-feature normalised, rows >= mel_len zero) + mel_len i32[B].  Needs the workspace
 * (rs_set_workspace) for the per-feature statistics.  On the fused paths below the features stay
 * un-normalised in the workspace and the normalisation is applied by the first subsampling kernel's load. */
int rs_logmel(rs_engine* e, const float* wav_dev, const int32_t* len_dev, int B, int L_max,
              float* mel_dev, int32_t* mel_len_dev, void* stream);
/* N2-N7 ConformerEncoder: mel -> enc f32[B,T_max,d_model] + enc_len i32[B].
 * n_layers < 0 runs the configured depth (smaller values are for stage tests). */
int rs_encode(rs_engine* e, const float* mel_dev, const int32_t* mel_len_dev, int B, int F_max,
              float* enc_dev, int32_t* enc_len_dev, int n_layers, void* stream);
/* N8-N9 RNNTDecoder + RNNTJoint + greedy loop: enc -> tokens/frames i32[B,U_max], n_tok i32[B].
 * n_tok[b] is the true emission count (may exceed U_max; only U_max entries are stored). */
int rs_rnnt_greedy(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B,
                   int T_max, int32_t* tokens_dev, int32_t* frames_dev, int32_t* n_tok_dev,
                   int U_max, void* stream);
/* Device-resident whole path (what bench.py's `value` times). */
int rs_transcribe_device(rs_engine* e, const float* wav_dev, const int32_t* len_dev, int B,
                         int L_max, int32_t* tokens_dev, int32_t* frames_dev, int32_t* n_tok_dev,
                         int U_max, void* stream);
/* The model.transcribe seam with HOST buffers: H2D + whole path + D2H; synchronises. */
int rs_transcribe_batch(rs_engine* e, const float* wav_host, const int32_t* len_host, int B,
                        int L_max, int32_t* tokens_host, int32_t* frames_host,
                        int32_t* n_tok_host, int U_max, void* stream);
/* The same two entry points for 16-bit PCM (what audio files hold): samples are scaled by 2^-15 inside the
 * log-mel kernel's staging load -- the value decoding a 16-bit WAV to float32 gives (the reference loads files
 * through librosa.load, pkg/nemo-asr/src/audio.py:32-42) -- so the results equal the float entry points' on
 * the converted samples, for half the host-to-device and HBM bytes.  L_max must be a multiple of 4 for the
 * vectorised load (any value works, unaligned rows fall back to scalar loads). */
int rs_transcribe_device_pcm16(rs_engine* e, const int16_t* wav_dev, const int32_t* len_dev, int B,
                               int L_max, int32_t* tokens_dev, int32_t* frames_dev,
                               int32_t* n_tok_dev, int U_max, void* stream);
int rs_transcribe_batch_pcm16(rs_engine* e, const int16_t* wav_host, const int32_t* len_host, int B,
                              int L_max, int32_t* tokens_host, int32_t* frames_host,
                              int32_t* n_tok_host, int U_max, void* stream);

/* Confidence statistics of the greedy decode (what NeMo's ConfidenceConfig turns into token / word confidence): the three
 * calls above plus `alpha` (> 0, finite; RS_ERR_INVALID_ARG otherwise) and `stats` f32 [B, U_max, 4].  For every stored
 * token n of utterance b, stats[b][n] = (lp, H1, A, G) of the softmax p over all vocab_size + 1 classes (blank included) of
 * the joint evaluation that emitted it: lp = log p of the emitted (argmax) token, H1 = sum p log p, A = sum p^alpha,
 * G = sum p^alpha log p.  Every confidence measure NeMo defines is a function of these four numbers and the class count
 * (reazonspeech_b200/confidence.py).  Blank decisions and tokens at or beyond U_max store nothing.  Tokens, frames and n_tok
 * are exactly those of the calls without statistics.  wav_is_pcm16: the samples are int16 PCM (as in the _pcm16 calls).
 * rs_transcribe_batch_confidence synchronises; its statistics are copied back with the tokens. */
int rs_rnnt_greedy_confidence(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B,
                              int T_max, int32_t* tokens_dev, int32_t* frames_dev, int32_t* n_tok_dev,
                              int U_max, float alpha, float* stats_dev, void* stream);
int rs_transcribe_device_confidence(rs_engine* e, const void* wav_dev, int wav_is_pcm16, const int32_t* len_dev,
                                    int B, int L_max, int32_t* tokens_dev, int32_t* frames_dev,
                                    int32_t* n_tok_dev, int U_max, float alpha, float* stats_dev, void* stream);
int rs_transcribe_batch_confidence(rs_engine* e, const void* wav_host, int wav_is_pcm16, const int32_t* len_host,
                                   int B, int L_max, int32_t* tokens_host, int32_t* frames_host,
                                   int32_t* n_tok_host, int U_max, float alpha, float* stats_host, void* stream);

/* Streaming: the greedy decode resumed from, and returning, a per-stream decoder state (semantics, frame grid and chunk
 * schedule: reazonspeech_b200/streaming.py).  A stream's state is one record of rs_stream_state_bytes() bytes in caller-owned
 * device memory (about 15 KB at the production size; records 16-byte aligned).  The record is opaque apart from its three
 * leading int32 words: started, boost_state, lm_state.  An all-zero record is a stream that has not started: its first call
 * runs the start (SOS) step, exactly as rs_rnnt_greedy does.  A boost_state / lm_state outside the current table counts as
 * the root / the LM's start_state: writing -1 there makes a stream start over in a table set while it was open.
 *
 * rs_rnnt_greedy_resume: enc f32[B,T_max,d_model] (device); row b decodes its frames [dec_begin[b], dec_end[b]) from record
 * slot[b] of `states` (device arrays i32[B]) and stores its state there.  Slots must be distinct (not checked: they are on
 * the device).  tokens / frames / n_tok / stats as rs_rnnt_greedy_confidence, for this call's emissions only; frames are
 * frames of `enc`.  stats may be NULL (alpha is then ignored).  Asynchronous on stream.
 * rs_stream_step: the whole path with HOST buffers, shaped like rs_transcribe_batch_confidence: H2D, log-mel, encoder,
 * joint.enc, the resumed decode, D2H; synchronises.  Row b is a buffer of len_host[b] samples; dec_begin / dec_end / slot are
 * host arrays.  Checks on the host that the slots are distinct and >= 0 and that 0 <= dec_begin <= dec_end <=
 * rs_enc_valid(len) (and len <= L_max), RS_ERR_INVALID_ARG before any launch otherwise.  stats_host may be NULL.
 * Phrase boosting and the n-gram LM apply to both as to every greedy entry point. */
size_t rs_stream_state_bytes(const rs_engine* e);
int rs_rnnt_greedy_resume(rs_engine* e, const float* enc_dev, const int32_t* dec_begin_dev, const int32_t* dec_end_dev,
                          const int32_t* slot_dev, void* states_dev, int B, int T_max, int32_t* tokens_dev, int32_t* frames_dev,
                          int32_t* n_tok_dev, int U_max, float alpha, float* stats_dev, void* stream);
int rs_stream_step(rs_engine* e, const void* wav_host, int wav_is_pcm16, const int32_t* len_host, const int32_t* dec_begin_host,
                   const int32_t* dec_end_host, const int32_t* slot_host, void* states_dev, int B, int L_max, int32_t* tokens_host,
                   int32_t* frames_host, int32_t* n_tok_host, int U_max, float alpha, float* stats_host, void* stream);

/* Phrase boosting (context biasing) of the greedy decode.  bonus f32 and next i32, both [n_states, pitch] in device memory
 * and 16-byte aligned, are the tables of a phrase automaton (reazonspeech_b200/boosting.py builds them): emitting non-blank
 * token k from state n adds bonus[n][k] to token k's logit before the argmax and moves the utterance to next[n][k] (a value
 * outside [0, n_states) counts as the root: state 0, or the row's root with rs_set_boost_roots).  Every utterance starts at
 * the root in every call; blank is never boosted.  pitch >= vocab_size and a multiple of 4; 1 <= n_states <= RS_MAX_BOOST_STATES; otherwise RS_ERR_INVALID_ARG and
 * the previous setting stays.  n_states = 0 clears the setting (the pointers are then ignored).  While a table is set, every
 * greedy entry point (rs_rnnt_greedy, rs_transcribe_device / _batch and their _pcm16 / _confidence forms) decodes with it; the
 * confidence statistics stay those of the unboosted softmax at the boosted decisions.  The tables stay owned by the caller
 * and must outlive every call that uses them; the engine keeps only the pointers.  rs_rnnt_alsd ignores them. */
#define RS_MAX_BOOST_STATES 8192
int rs_set_phrase_boosting(rs_engine* e, const float* bonus_dev, const int32_t* next_dev, int n_states, int pitch);

/* Phrase boosting per row: each row of a greedy batch decodes against its own phrase list.  The table set by
 * rs_set_phrase_boosting then holds several automata laid one after another, each with its next entries offset to its own
 * region (reazonspeech_b200/boosting.py combine_tables builds it); a row's root is the first state of its region.
 * roots_host is a HOST array of n entries; each must lie in [0, n_states) of the current table, and a table must be set,
 * otherwise RS_ERR_INVALID_ARG and the previous roots stay.  The engine keeps a copy and stages it into an engine-owned
 * device buffer on each decode's stream, ordered like the workspace (the call waits for the device only when that buffer
 * has to grow).  From then on row b of every greedy
 * entry point (rs_rnnt_greedy, rs_transcribe_device / _batch in their _pcm16 / _confidence forms, rs_rnnt_greedy_resume and
 * rs_stream_step) starts at roots[b] instead of state 0, and a state outside [0, n_states) -- a transition or a stream
 * record's boost_state -- counts as roots[b].  A call with more rows than roots (B > n) returns RS_ERR_INVALID_ARG before any
 * launch.  n = 0 clears the roots (every row starts at 0 again); setting or clearing a table with rs_set_phrase_boosting also
 * clears them. */
int rs_set_boost_roots(rs_engine* e, const int32_t* roots_host, int n);

/* n-gram language-model shallow fusion of the greedy decode and of rs_rnnt_maes (reazonspeech_b200/ngram_lm.py builds the
 * tables from an ARPA file over BPE token ids and states the semantics).  In the greedy decode the decision of every (utterance, frame) is the argmax of
 * logit_k + [k != blank] * (boosting bonus + LM term of k in the utterance's LM state); the state moves on emissions only and
 * starts at start_state in every call.  The LM term of token k in state s is cb[s] + arc_w[a] for the highest-level arc a of
 * token k on s's chain chain[s][0 .. order-1) (arcs of state o: arc_begin[o] .. arc_begin[o+1], sorted by arc_tok), or
 * cb[s] + uni_w[k] when there is none; the state reached is arc_to[a] (or uni_to[k]).  State 0 is the empty context.  All
 * arrays live in device memory, 16-byte aligned, owned by the caller, and must outlive every call that uses them; the engine
 * keeps only the pointers.  2 <= order <= RS_MAX_LM_ORDER, n_states >= 1, n_arcs >= 0, pitch >= vocab_size and a multiple of
 * 4, 0 <= start_state < n_states, no NULL array; otherwise RS_ERR_INVALID_ARG and the previous setting stays.  lm == NULL
 * clears the setting.  While a table is set, every greedy entry point (rs_rnnt_greedy, rs_transcribe_device / _batch and
 * their _pcm16 / _confidence forms) decodes with it; the confidence
 * statistics stay those of the unfused softmax at the fused decisions.  rs_rnnt_alsd ignores it. */
#define RS_MAX_LM_ORDER 6
typedef struct rs_ngram_lm {
  int order, n_states, n_arcs, pitch, start_state;
  const float* cb;          /* [n_states] */
  const int32_t* chain;     /* [n_states][order - 1] */
  const int32_t* arc_begin; /* [n_states + 1] */
  const int32_t* arc_tok;   /* [n_arcs] */
  const int32_t* arc_to;    /* [n_arcs] */
  const float* arc_w;       /* [n_arcs] */
  const float* uni_w;       /* [pitch] */
  const int32_t* uni_to;    /* [pitch] */
} rs_ngram_lm;
int rs_set_ngram_lm(rs_engine* e, const rs_ngram_lm* lm);
/* The decode kernel's own LM lookup on n (state, token) pairs, device arrays states / tokens i32[n] -> score f32[n] (the LM
 * term the decode adds to the token's logit in that state) and next i32[n] (the state emitting it leads to); a token outside
 * [0, vocab_size) gives NaN and -1.  Needs a table set by rs_set_ngram_lm.  Asynchronous on stream.  A test seam. */
int rs_ngram_lm_eval(rs_engine* e, const int32_t* states_dev, const int32_t* tokens_dev, int n, float* score_dev, int32_t* next_dev,
                     void* stream);

/* ALSD beam search (NeMo BeamRNNTInfer.align_length_sync_decoding, the shipped checkpoint's default strategy; the reference's
 * decode.py is written for its hypotheses, pkg/nemo-asr/src/decode.py:29,38-40,48): enc f32[B,T_max,d_model] + enc_len ->
 * y i32[B, U_cap + 1] (leading blank, then the tokens), step i32[B, U_cap] (alignment step t + u of every token =
 * Hypothesis.timestamp after NeMo's pack_hypotheses), n i32[B] tokens, score f64[B] (log-probability of the winner).
 * beam 1..8; u_max_ratio = alsd_max_target_len (NeMo: 2.0); score_norm: rank finished hypotheses by score / len(y);
 * recombine_returns_input: NeMo's recombine_hypotheses as recalled (adds duplicate scores, keeps the duplicates).
 * u_max = int(u_max_ratio * T) is computed in double, as NeMo does (in float, 1.16 * 25 would round to 29 instead of 28).
 * A finished hypothesis is ranked with the score recombination added into it in the step it finished, as NeMo's `final`
 * list holds the same object as its beam.  n[b] is the winner's full length even when it exceeds U_cap; y and step then
 * hold its first U_cap tokens.  enc_len[b] = 0 gives y = [blank], n = 0, score 0.
 * Needs the "alsd.*" weight tensors at rs_engine_create.  Synchronises before returning. */
int rs_rnnt_alsd(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, int beam,
                 double u_max_ratio, int score_norm, int recombine_returns_input, int32_t* y_dev, int32_t* step_dev,
                 int32_t* n_dev, double* score_dev, int U_cap, void* stream);
/* The N-best list of the same search (NeMo's BeamRNNTInfer with return_best_hypothesis=False): the same launches as
 * rs_rnnt_alsd, and every beam, scored row and winner bit-identical to it.  The N-best list of an utterance is the first
 * n_best entries of Python's stable sorted(pool, key, reverse=True), where
 *   pool = NeMo's `final`: every stay at the last frame, in append order (A order within a step, steps ascending),
 *          duplicates included; if nothing finished, the last beam in slot order;
 *   key  = score / len(y) with score_norm (len(y) counts the leading blank), else score; equal keys keep pool order.
 * A finished entry carries the score recombination added into it in the step it finished, as for rs_rnnt_alsd.  Entry 0 is
 * always what rs_rnnt_alsd returns.  Entry e of utterance b is row b * n_best + e of y [B][n_best][U_cap + 1] (leading
 * blank), step [B][n_best][U_cap], n [B][n_best] (its full token count; y and step hold the first U_cap tokens) and
 * score [B][n_best].  count[b] = min(n_best, pool[b]) entries are written, and entries at or past count[b] are left
 * untouched; pool[b] is the size of NeMo's whole list; from_final[b] is 0 when nothing finished and the last beam was ranked.
 * enc_len[b] = 0 gives one entry: [blank], n 0, score 0, pool 1, from_final 0.  n_best outside 1..RS_MAX_NBEST, or any
 * argument rs_rnnt_alsd rejects, gives RS_ERR_INVALID_ARG before any launch.  The list lives in the engine-owned ALSD
 * workspace (24 bytes per entry); rs_workspace_bytes is unchanged.  Synchronises before returning. */
#define RS_MAX_NBEST 64
int rs_rnnt_alsd_nbest(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, int beam,
                       double u_max_ratio, int score_norm, int recombine_returns_input, int n_best,
                       int32_t* y_dev,          /* [B][n_best][U_cap + 1] */
                       int32_t* step_dev,       /* [B][n_best][U_cap]     */
                       int32_t* n_dev,          /* [B][n_best] full token count */
                       double* score_dev,       /* [B][n_best]            */
                       int32_t* count_dev,      /* [B] entries written = min(n_best, pool) */
                       int32_t* pool_dev,       /* [B] size of NeMo's whole list */
                       int32_t* from_final_dev, /* [B] 0: nothing finished, the last beam was ranked */
                       int U_cap, void* stream);
/* Test seam: rs_rnnt_alsd (the same launches and results) that also copies the search state into caller-owned device
 * buffers.  R = B * beam rows; row r = b * beam + k is slot k of utterance b.  After the beam update of step i (the
 * anti-diagonal t + u = i), for i < max_steps (later steps are not recorded; steps the search never ran are untouched):
 *   n_hyp [i][b], beam_score / beam_u / beam_node [i][r]: the new beam (slot k < n_hyp: its log-probability, token count, back-pointer node);
 *   row_t [i][r]: frame of the hypothesis in slot k of the previous beam scored at step i (-1: not scored);
 *   cand_logp [i][r][9]: its log p(blank), then the beam best non-blank log-probabilities; cand_tok [i][r][8]: their classes;
 *   has_final / final_key / final_score [i][b]: the best finished hypothesis so far (key = score / (u + 1) with score_norm),
 *   entry 0 of rs_rnnt_alsd_nbest's list.
 * Once at the end, the back-pointer tree [B][node_pitch]: node 0 is the leading blank; node n > 0 is a token node_tok[n]
 * emitted at step node_step[n] after node_parent[n].  node_pitch >= 1 + beam * (T_max + int(u_max_ratio * T_max) + 1);
 * RS_ERR_INVALID_ARG before any launch otherwise, or when a buffer is NULL or max_steps < 0. */
typedef struct rs_alsd_trace {
  int32_t max_steps, node_pitch;
  int32_t* n_hyp;         /* [max_steps][B] */
  double* beam_score;     /* [max_steps][R] */
  int32_t* beam_u;        /* [max_steps][R] */
  int32_t* beam_node;     /* [max_steps][R] */
  int32_t* row_t;         /* [max_steps][R] */
  float* cand_logp;       /* [max_steps][R][9] */
  int32_t* cand_tok;      /* [max_steps][R][8] */
  int32_t* has_final;     /* [max_steps][B] */
  double* final_key;      /* [max_steps][B] */
  double* final_score;    /* [max_steps][B] */
  int32_t* node_parent;   /* [B][node_pitch] */
  int32_t* node_tok;      /* [B][node_pitch] */
  int32_t* node_step;     /* [B][node_pitch] */
} rs_alsd_trace;
int rs_rnnt_alsd_trace(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, int beam,
                       double u_max_ratio, int score_norm, int recombine_returns_input, int32_t* y_dev, int32_t* step_dev,
                       int32_t* n_dev, double* score_dev, int U_cap, const rs_alsd_trace* trace, void* stream);

/* MAES beam search (NeMo BeamRNNTInfer.modified_adaptive_expansion_search, Kim et al. 2020; semantics restated in
 * oracle/maes_restated.py): enc f32[B,T_max,d_model] + enc_len -> NeMo's sort_nbest of the kept hypotheses after the last
 * frame, best first.  Entry e of utterance b is row b * n_best + e of y [B][n_best][U_cap + 1] (leading blank, then the
 * tokens), frames [B][n_best][U_cap] (the encoder frame that emitted each token), n [B][n_best] (its full token count; y and
 * frames hold the first U_cap tokens) and score [B][n_best] (log-probability, with the LM terms when an LM is set).
 * count[b] = min(n_best, kept hypotheses) entries are written; entries at or past count[b] are left untouched.  The ranking
 * key is score / len(y) with score_norm (len(y) counts the leading blank), else score; equal keys keep the beam's order.
 * enc_len[b] = 0 gives one entry: [blank], n 0, score 0.
 * Parameters (NeMo's defaults in brackets): beam 1..8 (K = min(beam, vocab_size)); num_steps 2..4 [2] expansion rounds per
 * frame; prefix_alpha 0..4 [1]; expansion_beta 0..4 [2] (C = K + beta candidates per hypothesis; K + beta <= vocab_size);
 * expansion_gamma > 0 [2.3]; recombine_returns_input as for rs_rnnt_alsd; n_best 1..K.  An out-of-range parameter gives
 * RS_ERR_INVALID_ARG, and a worst case of W = K * C^num_steps expansion rows per utterance above RS_MAX_MAES_ROWS gives
 * RS_ERR_UNSUPPORTED, both before any launch (NeMo's defaults fit at every beam <= 8: 8 * 10^2 = 800).
 * With an n-gram LM set (rs_set_ngram_lm) every token expansion adds the LM term of its token in the hypothesis's LM context
 * (the greedy decode's lookup; the context starts at the LM's start state).  Phrase boosting is ignored.
 * The host learns the number of live expansion rows of each round (their GEMMs' M) by one pinned 4-byte read per round.
 * Needs the "alsd.*" weight tensors at rs_engine_create.  The workspace is engine-owned and grown on demand (the ALSD one).
 * Synchronises before returning. */
#define RS_MAX_MAES_ROWS 1024
typedef struct rs_maes_params {
  int32_t beam, num_steps, prefix_alpha, expansion_beta;
  float expansion_gamma;
  int32_t score_norm, recombine_returns_input;
} rs_maes_params;
int rs_rnnt_maes(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max,
                 const rs_maes_params* p, int n_best,
                 int32_t* y_dev,       /* [B][n_best][U_cap + 1] */
                 int32_t* frames_dev,  /* [B][n_best][U_cap]     */
                 int32_t* n_dev,       /* [B][n_best] full token count */
                 double* score_dev,    /* [B][n_best]            */
                 int32_t* count_dev,   /* [B] entries written = min(n_best, kept) */
                 int U_cap, void* stream);
/* Expansion rows of the last rs_rnnt_maes call on this engine: the sum over frames of the rows the expansion rounds ran
 * through the predictor (*rows), and the frames searched (*frames: T_max of that call). */
int rs_maes_last_rows(const rs_engine* e, int64_t* rows, int64_t* frames);

/* Forced alignment of given label sequences on the standard RNN-T lattice (semantics: reazonspeech_b200/alignment.py):
 * enc f32[B,T_max,d_model] + enc_len, labels i32[B,U_max] + label_len i32[B] (device) ->
 * frames i32[B,U_max] (emission frame of each token on the Viterbi path), token_lp f32[B,U_max] (the token's lattice
 * log-probability lp_emit[frame][u - 1] on that path), viterbi f32[B] (the Viterbi path's log-probability), loglik f32[B]
 * (log P(y|x) = -RNN-T loss).  Entries at or beyond label_len[b] hold frame -1 and NaN.  An utterance with a label outside
 * [0, vocab_size), label_len outside [0, U_max] or enc_len outside [1, T_max] gets NaN scores and frames -1; the others are
 * unaffected.  Scratch (the lattice, 8 bytes + 1 per cell of B x T_max x (U_max + 1), and the predictor rows) is engine-owned
 * and grown on demand like the ALSD workspace (RS_ERR_WORKSPACE when that allocation fails: a 10-minute clip is about 200 MB;
 * callers chunk longer inputs); rs_workspace_bytes is unchanged.  U_max <= 14527 (the DP keeps two anti-diagonals in shared
 * memory; RS_ERR_UNSUPPORTED beyond).  Works with or without the alsd.* tensors, and ignores phrase boosting and the LM.
 * Asynchronous on stream, except that growing the scratch synchronises it. */
int rs_rnnt_align(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max,
                  const int32_t* labels_dev, const int32_t* label_len_dev, int U_max,
                  int32_t* frames_dev, float* token_lp_dev, float* viterbi_dev, float* loglik_dev, void* stream);
/* Test seam: the lattice alone -> lp_blank / lp_emit f32[B, T_max, U_max + 1] (cells outside an utterance untouched;
 * lp_emit[t][label_len] = -inf: no label left to emit). */
int rs_rnnt_align_lattice(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max,
                          const int32_t* labels_dev, const int32_t* label_len_dev, int U_max,
                          float* lp_blank_dev, float* lp_emit_dev, void* stream);

/* Segment alignment of given label sequences inside longer windows (semantics: reazonspeech_b200/alignment.py, "Segment
 * alignment"): the same lattice as rs_rnnt_align, but the tokens may start and end at any frame and the frames outside
 * the segment are not charged.  enc f32[B,T_max,d_model] + enc_len, labels i32[B,U_max] + label_len i32[B] (device) ->
 * seg i32[B,2] (s, e: the segment's first and last frame), frames i32[B,U_max] (each token's emission frame on the best
 * segment path), token_lp f32[B,U_max] (lp_emit[frame][u - 1] on that path), frame_lp f32[B,T_max] (for t in [s, e] the
 * path's emissions at t plus the blank that leaves t, sum = viterbi; NaN outside [s, e]), viterbi f32[B] (the best segment
 * path's log-probability), loglik f32[B] (log P(y | the frames [s, e])).  Entries at or beyond label_len[b] hold frame -1
 * and NaN.  An utterance with label_len outside [1, U_max], a label outside [0, vocab_size) or enc_len outside [1, T_max]
 * gets s = e = -1, frames -1 and NaN scores; the others are unaffected.  Scratch, limits (U_max <= 14527) and argument checks
 * are rs_rnnt_align's; bad host arguments are rejected before any launch. */
int rs_rnnt_align_segment(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max,
                          const int32_t* labels_dev, const int32_t* label_len_dev, int U_max, int32_t* seg_dev,
                          int32_t* frames_dev, float* token_lp_dev, float* frame_lp_dev, float* viterbi_dev,
                          float* loglik_dev, void* stream);

/* norm_audio on the device (pkg/nemo-asr/src/audio.py:54-68: resample to 16 kHz, then average the channels) fused with
 * transcribe()'s padding (audio.py:70-83): in [B, channels, L_in_max] f32 or int16 PCM at the native rate ->
 * out f32 [B, L_out_row], row b = pad zeros | resampled mono utterance | zeros, len_out[b] = resampled length + 2 pad;
 * feed out / len_out to rs_transcribe_device.  The polyphase FIR (taps [up][taps_per_phase], n_pre_remove) is
 * scipy.signal.resample_poly's, designed by the host binding (reazonspeech_b200/engine.py::resample_taps). */
int rs_resample_mono(rs_engine* e, const void* in_dev, int in_is_pcm16, const int32_t* len_in_dev, int B,
                     int channels, int L_in_max, const float* taps_dev, int taps_per_phase, int up, int down,
                     int n_pre_remove, int pad, float* out_dev, int L_out_row, int32_t* len_out_dev, void* stream);

/* Host-side half of transcribe()'s padding (pkg/nemo-asr/src/audio.py:70-83) for a batch: row r of dst[B][L] (pinned host
 * memory the caller then hands to rs_transcribe_batch / _pcm16) = zeros(pad) | src[r][0 .. n[r]) | zeros to L.
 * dst_is_pcm16: rows are int16 and every source must be int16; otherwise rows are float32 and an int16 source
 * (src_is_pcm16[r] != 0; the array may be NULL = all float32) is scaled by 1/32768.  No engine, no CUDA call: plain
 * copies split over `threads` host threads, so a binding can stage a batch without holding its interpreter lock. */
int rs_stage_rows(void* dst, int64_t L, const void* const* src, const int64_t* n, const int32_t* src_is_pcm16,
                  int dst_is_pcm16, int B, int64_t pad, int threads);

/* ---- kernel-level seams (parity tests and roofline measurement) ---------------------------
 * Each calls one kernel launcher with the shapes given (not the engine's configuration); none needs the workspace.
 * A shape or parameter the kernel does not implement is rejected before any launch (RS_ERR_UNSUPPORTED /
 * RS_ERR_INVALID_ARG). */
/* out2 / split / ld2: RS_EPI_QKV_VT only (columns >= split go transposed to out2 bf16 [N - split, ld2], ld2 >= M). */
int rs_gemm_bf16(rs_engine* e, const void* a_bf16, const void* w_bf16, const float* bias,
                 const float* resid, void* out, int M, int N, int K, int epilogue, float alpha,
                 void* out2, int split, int ld2, void* stream);
/* gamma2 / beta2 (nullable): a second LayerNorm chained on the first's result, written to out_bf16 (norm_out of one layer
 * feeding the next layer's first pre-norm); out_f32 may be x (in place). */
int rs_layernorm(rs_engine* e, const float* x, const float* gamma, const float* beta,
                 float* out_f32 /*nullable*/, void* out_bf16 /*nullable*/, const float* gamma2,
                 const float* beta2, int rows, int d, void* stream);
/* Local attention + global token (head dim 128): qkv bf16 [B*T_max, 3*H*128] with q + pos_bias_u in the q columns and k
 * after them, V^T bf16 [H*128, ld_vt] (column = b*T_max + t), pos bf16 [H, n_rel_pad, 128], bd_bias f32 [H, n_rel_pad],
 * bias_u f32 [H, 128] -> out bf16 [B*T_max, H*128] (rows >= enc_len[b] zero). */
int rs_attention(rs_engine* e, const void* qkv_bf16, const void* vt_bf16, int ld_vt, const void* pos_bf16,
                 const float* bd_bias, int n_rel_pad, const float* bias_u, void* out_bf16, const int32_t* enc_len,
                 int B, int T_max, int H, int w_left, int w_right, int n_global, void* stream);
/* Depthwise conv (k taps, BatchNorm folded into w [k, d] and shift [d]) + Swish on bf16 [B*T_max, d]; input rows
 * t >= enc_len[b] read as zero. */
int rs_conv_dw(rs_engine* e, const void* u_bf16, void* out_bf16, const float* w_f32, const float* shift_f32,
               const int32_t* enc_len, int B, int T_max, int d, int k, void* stream);
/* Subsampling conv.0 (1 -> C, 3x3 s2) + ReLU + conv.2 (depthwise 3x3 s2) on mel f32 [B, F_max, n_mels] -> bf16
 * [B, T2, F2, C] with T1 = conv_len(F_max), T2 = conv_len(T1), F2 = conv_len(conv_len(n_mels)).  mel_stats
 * [B, n_mels, 2] = (mean, 1 / (std + eps)) normalises the features on load; NULL: they are already normalised. */
int rs_sub_conv0_dw1(rs_engine* e, const float* mel, const int32_t* mel_len, const float* mel_stats, int B, int F_max,
                     int n_mels, int C, const float* w0, const float* b0, const float* wd, const float* bd,
                     void* out_bf16, void* stream);
/* Depthwise 3x3 s2 on channels-last bf16 [B, Tin, Fin, C] -> [B, Tout, Fout, C]; the valid input length of utterance b
 * is conv_len applied len_shift times to mel_len[b]. */
int rs_sub_dw(rs_engine* e, const void* in_bf16, void* out_bf16, const float* w, const float* b, const int32_t* mel_len,
              int len_shift, int B, int Tin, int Fin, int Tout, int Fout, int C, void* stream);
/* Counters: kernels launched by this engine since creation (bench.py's gpu_launches). */
int64_t rs_launch_count(const rs_engine* e);
/* Per-stage device time of the last rs_transcribe_* call when timing was enabled. */
int rs_enable_stage_timing(rs_engine* e, int on);
int rs_stage_times_ms(const rs_engine* e, float* ms /*[8]*/);
int rs_debug_decode_cycles(rs_engine* e, int B, int L_max, int U_max, int64_t* out12);  /* profiling aid, see engine.cu */
/* Per-launch CUDA-event timing of the wgmma GEMM (the dominant kernel): while enabled every GEMM
 * launch is bracketed by two events on its stream.  rs_gemm_timing() synchronises, returns the summed
 * device time, the summed algorithmic FLOPs (2*M*N*K) and the launch count since it was enabled or
 * last read, and resets the log. */
int rs_enable_gemm_timing(rs_engine* e, int on);
int rs_gemm_timing(rs_engine* e, double* ms, double* flops, int64_t* launches);
/* Per-kernel CUDA-event timing of EVERY launch inside the real pipeline (warm caches, back-to-back launches, unlike
 * the cold, serialised launches ncu reports).  rs_kernel_timing() synchronises the device and writes one line per
 * kernel name, "name<TAB>launches<TAB>total_ms", into buf; the log is reset. */
int rs_enable_kernel_timing(rs_engine* e, int on);
int rs_kernel_timing(rs_engine* e, char* buf, int buf_bytes);

#ifdef __cplusplus
}
#endif
#endif /* RS_ENGINE_H_ */
