// C ABI of the engine (include/rs_engine.h): weight table lookup, workspace planning and the
// launch sequence of the FastConformer-RNNT path.  Host-side orchestration only; every device
// operation is one of the sm_90a kernels declared in kernels.h.
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <map>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/rs_engine.h"
#include "alsd.h"
#include "kernels.h"
#include "logmel.h"
#include "maes.h"

namespace {

thread_local char g_create_error[512] = "";

// NVTX range around the ENQUEUE of a stage (SURVEY.md section 5: per-stage ranges for Nsight Systems / Compute).  Header-only
// NVTX v3: a no-op unless a tool has injected itself into the process.
struct Nvtx {
  explicit Nvtx(const char* name) { nvtxRangePushA(name); }
  ~Nvtx() { nvtxRangePop(); }
  Nvtx(const Nvtx&) = delete;
  Nvtx& operator=(const Nvtx&) = delete;
};

struct Tensor { const void* p = nullptr; int dtype = 0; int64_t numel = 0; };

struct LayerW {
  const float *ln_ff1_g, *ln_ff1_b, *ff1_b1, *ff1_b2;
  const void *ff1_w1, *ff1_w2;
  const float *ln_att_g, *ln_att_b, *bqkv, *att_u, *att_bdbias, *bo;
  const void *wqkv, *att_pos, *wo;
  const float *ln_conv_g, *ln_conv_b, *pw1_b, *dw_w, *dw_shift, *pw2_b;
  const void *pw1_w, *pw2_w;
  const float *ln_ff2_g, *ln_ff2_b, *ff2_b1, *ff2_b2;
  const void *ff2_w1, *ff2_w2;
  const float *ln_out_g, *ln_out_b;
};

struct Plan {           // workspace offsets (bytes) for one (B, L_max)
  int B, L_max, F_max, T1, F1, T2, F2, T3, F3, M;
  size_t wav, len, mel, mel_len, mel_part, mel_stats, enc_len, sub1, sub2, sub3, sub4, x, xn, hbuf, abuf, cbuf, vt, enc, encp;
  int n_rel_pad, ld_vt;
  size_t tokens, frames, ntok, stats, dec_ws, total;
};

inline int conv_len(int n) { return n > 0 ? (n - 1) / 2 + 1 : 0; }   // floor division as in NeMo's calc_length: 0 stays 0
// Encoder-frame capacity of the padded activation tensors: the subsampled length rounded up to a multiple of 8, so that
// every utterance starts at a 16-byte-aligned column of the transposed V buffer (TMA wants the innermost coordinate
// 16-byte aligned: an odd T_max raised "illegal instruction" on the V^T tile loads of the attention kernel).
inline int enc_capacity(int mel_frames) { return (conv_len(conv_len(conv_len(mel_frames))) + 7) & ~7; }

}  // namespace

struct rs_engine {
  rs_model_config cfg;
  int device = 0;
  int num_sms = 132;
  std::map<std::string, Tensor> w;
  rs::LmTables fe{};          // tables of the fused log-mel kernel (logmel_tables.py)
  // ALSD beam search (decode_alsd.cu): fp32-accurate tripled weights (optional: present when the engine was created with them),
  // an engine-owned workspace grown on demand, a pinned word for the periodic "all utterances finished" check
  struct { const void *out_w3 = nullptr, *lstm_w3 = nullptr, *pred_w3 = nullptr; const float* out_b = nullptr; int n_pad = 0; } alsd;
  void* alsd_ws = nullptr;
  size_t alsd_ws_bytes = 0;
  int* alsd_done_host = nullptr;       // also the per-round row count of MAES (rs_rnnt_maes)
  int64_t maes_rows = 0, maes_frames = 0;   // rs_maes_last_rows
  // forced alignment (align.cu): scratch grown on demand like the ALSD workspace
  void* align_ws = nullptr;
  size_t align_ws_bytes = 0;
  // rs_stream_step: device copies of the step's dec_begin | dec_end | slot, grown on demand
  void* stream_args = nullptr;
  size_t stream_args_bytes = 0;
  // streaming keyword spotting (rs_set_spot_keywords): the installed keyword set, its labels and its teacher-forced predictor
  // rows (pred_proj [n_kw][U_max + 1][Hj]) in one engine-owned allocation; the calls' scratch grown on demand
  struct { int n_kw = 0, U_max = 0, delay = 0, chunk = 0, ring_cap = 0; float threshold = 0.f; void* mem = nullptr;
           const int32_t* labels = nullptr; const int32_t* label_len = nullptr; float* pred_proj = nullptr; } spot;
  void* spot_ws = nullptr;
  size_t spot_ws_bytes = 0;
  unsigned int* lm_tickets = nullptr;   // per-utterance CTA tickets of the log-mel statistics (engine-owned, kept zero between launches)
  static constexpr int kMaxBatch = 1 << 16;
  struct { const float *c0w, *c0b, *d1w, *d1b, *p1b, *d2w, *d2b, *p2b, *ob; const void *p1w, *p2w, *ow; } sub;
  std::vector<LayerW> layers;
  struct { const void *enc_w, *out_w, *lstm_w, *pred_w; const float *enc_b, *out_b, *embed, *lstm_b, *pred_b, *gate_tab; } dec;
  // phrase boosting (rs_set_phrase_boosting): caller-owned device tables used by every greedy decode while set
  struct { const float* bonus = nullptr; const int32_t* next = nullptr; int n_states = 0, pitch = 0; } boost;
  // per-row roots of that table (rs_set_boost_roots): n_roots host entries, copied on the call's stream into an engine-owned
  // device buffer (grown on demand) before each decode; 0: none
  std::vector<int32_t> roots_host;
  int32_t* boost_roots = nullptr;
  int n_roots = 0, roots_cap = 0;
  // n-gram LM shallow fusion (rs_set_ngram_lm): caller-owned device tables used by every greedy decode and rs_rnnt_maes while set; order 0: none
  rs::NgramLM lm;
  void* ws = nullptr;
  size_t ws_bytes = 0;
  mutable char err[512] = "";
  int64_t launches = 0;
  bool timing = false;                  // stage marks (mark)
  cudaEvent_t ev[6] = {};
  // launch log (launch): one {tag, flops} entry per timed launch, timed by the event pair log_ev[2i], log_ev[2i + 1]
  struct Timed { std::string tag; double flops; };
  bool ktiming = false, gemm_timing = false;
  std::vector<Timed> log;
  std::vector<cudaEvent_t> log_ev;
  // rs_transcribe_batch: host->device copies run on their own stream in utterance chunks so the frontend of
  // chunk i overlaps the copy of chunk i+1
  static constexpr int kCopyChunks = 8;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t copy_ev[kCopyChunks + 1] = {};
};

namespace {

int fail(const rs_engine* e, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(e ? e->err : g_create_error, 512, fmt, ap);
  va_end(ap);
  return code;
}

#define RS_CUDA(e, call)                                                                   \
  do {                                                                                     \
    cudaError_t _c = (call);                                                               \
    if (_c != cudaSuccess) return fail((e), RS_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(_c)); \
  } while (0)

#define RS_TRY(x) do { int _r = (x); if (_r != RS_OK) return _r; } while (0)

// Every device enqueue of the engine goes through launch(): `enqueue()` issues `n` launches (a memset counts as one) on
// stream `s` and returns the first error.  The launches are counted (rs_launch_count).  While kernel timing is on, or GEMM
// timing is on and the call is a GEMM (flops = 2*M*N*K > 0), the call is bracketed by an event pair on `s` and logged as
// {tag, flops}.  `what` is the call's source text, quoted by the error message; the tag is its name without the rs::
// namespace and the arguments.
template <typename F>
int launch(rs_engine* e, cudaStream_t s, const char* what, int n, double flops, F&& enqueue) {
  const bool timed = e->ktiming || (e->gemm_timing && flops > 0.0);
  const size_t i = 2 * e->log.size();
  if (timed) {
    while (e->log_ev.size() < i + 2) {
      cudaEvent_t ev;
      RS_CUDA(e, cudaEventCreate(&ev));
      e->log_ev.push_back(ev);
    }
    RS_CUDA(e, cudaEventRecord(e->log_ev[i], s));
  }
  const cudaError_t c = enqueue();
  if (c != cudaSuccess) return fail(e, RS_ERR_CUDA, "%s: %s", what, cudaGetErrorString(c));
  if (timed) {
    RS_CUDA(e, cudaEventRecord(e->log_ev[i + 1], s));
    std::string tag(what);
    if (tag.rfind("rs::", 0) == 0) tag = tag.substr(4);
    e->log.push_back({tag.substr(0, tag.find('(')), flops});
  }
  e->launches += n;
  return RS_OK;
}
#define RS_LAUNCH(e, s, n, call) RS_TRY(launch((e), (s), #call, (n), 0.0, [&] { return (call); }))

int gemm(rs_engine* e, const rs::GemmArgs& g, cudaStream_t s) {
  char what[64], msg[256] = "";
  snprintf(what, sizeof what, "gemm N=%d K=%d epi=%d", g.N, g.K, g.epilogue);
  const int r = launch(e, s, what, 1, 2.0 * g.M * static_cast<double>(g.N) * g.K, [&] { return rs::launch_gemm(g, e->num_sms, s, msg); });
  if (r != RS_OK && msg[0] != '\0') return fail(e, r, "gemm: %s", msg);
  return r;
}

// Synchronises the engine's device, passes every logged launch with its device time to visit(entry, ms), clears the log.
template <typename F>
int drain_log(rs_engine* e, F&& visit) {
  RS_CUDA(e, cudaSetDevice(e->device));
  RS_CUDA(e, cudaDeviceSynchronize());
  for (size_t i = 0; i < e->log.size(); ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e->log_ev[2 * i], e->log_ev[2 * i + 1]);
    visit(e->log[i], ms);
  }
  e->log.clear();
  return RS_OK;
}

inline rs::SpecWorkspace dec_ws(const rs_engine* e, int B) { return rs::rnnt_spec_workspace(B, e->cfg.joint_hidden, e->cfg.pred_hidden, e->num_sms); }

Plan make_plan(const rs_engine* e, int B, int L_max, int U_max) {
  const rs_model_config& c = e->cfg;
  Plan p{};
  p.B = B; p.L_max = L_max;
  p.F_max = L_max / c.n_window_stride + 1;
  p.T1 = conv_len(p.F_max); p.F1 = conv_len(c.n_mels);
  p.T2 = conv_len(p.T1); p.F2 = conv_len(p.F1);
  p.T3 = enc_capacity(p.F_max); p.F3 = conv_len(p.F2);
  p.M = B * p.T3;
  const size_t C = c.sub_channels, d = c.d_model;
  const size_t wide = static_cast<size_t>(c.d_ff) > 3 * d ? c.d_ff : 3 * d;
  rs::Arena a;
  p.wav = a.take(static_cast<size_t>(B) * L_max * 4);
  p.len = a.take(static_cast<size_t>(B) * 4);
  p.mel = a.take(static_cast<size_t>(B) * p.F_max * c.n_mels * 4);
  p.mel_len = a.take(static_cast<size_t>(B) * 4);
  p.mel_part = a.take(static_cast<size_t>(B) * rs::logmel_tiles(L_max, c.n_window_stride) * c.n_mels * 2 * 4);   // per-CTA (sum, sum of squares)
  p.mel_stats = a.take(static_cast<size_t>(B) * c.n_mels * 2 * 4);                                               // (mean, 1 / (std + eps))
  p.enc_len = a.take(static_cast<size_t>(B) * 4);
  p.sub1 = a.take(static_cast<size_t>(B) * p.T2 * p.F2 * C * 2);
  p.sub2 = a.take(static_cast<size_t>(B) * p.T2 * p.F2 * C * 2);
  p.sub3 = a.take(static_cast<size_t>(B) * p.T3 * p.F3 * C * 2);
  p.sub4 = a.take(static_cast<size_t>(B) * p.T3 * p.F3 * C * 2);
  p.x = a.take(static_cast<size_t>(p.M) * d * 4);
  p.xn = a.take(static_cast<size_t>(p.M) * d * 2);
  p.hbuf = a.take(static_cast<size_t>(p.M) * wide * 2);
  p.abuf = a.take(static_cast<size_t>(p.M) * d * 2);
  p.cbuf = a.take(static_cast<size_t>(p.M) * d * 2);
  p.n_rel_pad = ((c.att_left + c.att_right + 1 + 31) / 32) * 32;
  p.ld_vt = ((p.M + 255) / 256) * 256 + 64;                               // V^T row pitch (the GEMM writes columns < M only; any ld_vt >= M works)
  p.vt = a.take(static_cast<size_t>(d) * p.ld_vt * 2);
  p.enc = a.take(static_cast<size_t>(p.M) * d * 4);
  p.encp = a.take(static_cast<size_t>(p.M) * c.joint_hidden * 4);
  p.tokens = a.take(static_cast<size_t>(B) * U_max * 4);
  p.frames = a.take(static_cast<size_t>(B) * U_max * 4);
  p.ntok = a.take(static_cast<size_t>(B) * 4);
  p.stats = a.take(static_cast<size_t>(B) * U_max * 4 * 4);                // rs_transcribe_batch_confidence's statistics
  p.dec_ws = a.take(dec_ws(e, B).total);
  p.total = a.off;
  return p;
}

template <typename T>
T* at(const rs_engine* e, size_t off) { return reinterpret_cast<T*>(static_cast<char*>(e->ws) + off); }

int need(rs_engine* e, const char* name, int dtype, int64_t numel, const void** out) {
  auto it = e->w.find(name);
  if (it == e->w.end()) return fail(e, RS_ERR_MISSING_WEIGHT, "weight '%s' missing from the table", name);
  if (it->second.dtype != dtype || it->second.numel != numel)
    return fail(e, RS_ERR_MISSING_WEIGHT, "weight '%s': dtype/numel (%d, %lld) != expected (%d, %lld)", name,
                it->second.dtype, (long long)it->second.numel, dtype, (long long)numel);
  *out = it->second.p;
  return RS_OK;
}

#define NEED(field, name, dt, n)                                                   \
  do {                                                                             \
    const void* _p;                                                                \
    int _r = need(e, (name), (dt), (n), &_p);                                      \
    if (_r != RS_OK) return _r;                                                    \
    field = static_cast<decltype(field)>(_p);                                      \
  } while (0)

int bind_weights(rs_engine* e) {
  const rs_model_config& c = e->cfg;
  const int64_t d = c.d_model, ff = c.d_ff, C = c.sub_channels, H = c.n_heads, dk = d / H;
  const int64_t n_rel_pad = ((c.att_left + c.att_right + 1 + 31) / 32) * 32, k = c.conv_kernel;
  const int64_t F3 = conv_len(conv_len(conv_len(c.n_mels)));
  NEED(e->fe.window, "fe.window", RS_F32, c.n_fft);
  NEED(e->fe.tw_b, "fe.tw_b", RS_F32, 512);
  NEED(e->fe.tw_x, "fe.tw_x", RS_F32, 256);
  NEED(e->fe.mel_meta, "fe.mel_meta", RS_I32, rs::kLmMetaInts);
  {
    auto it = e->w.find("fe.mel_w");
    if (it == e->w.end() || it->second.dtype != RS_F32 || it->second.numel <= 0 || it->second.numel % 16)
      return fail(e, RS_ERR_MISSING_WEIGHT, "weight 'fe.mel_w' (f32 [taps, 16]) missing from the table or misshapen");
    e->fe.mel_w = static_cast<const float*>(it->second.p);
    e->fe.n_taps = static_cast<int>(it->second.numel / 16);
  }
  NEED(e->sub.c0w, "sub.conv0.w", RS_F32, C * 9); NEED(e->sub.c0b, "sub.conv0.b", RS_F32, C);
  NEED(e->sub.d1w, "sub.dw1.w", RS_F32, C * 9); NEED(e->sub.d1b, "sub.dw1.b", RS_F32, C);
  NEED(e->sub.p1w, "sub.pw1.w", RS_BF16, C * C); NEED(e->sub.p1b, "sub.pw1.b", RS_F32, C);
  NEED(e->sub.d2w, "sub.dw2.w", RS_F32, C * 9); NEED(e->sub.d2b, "sub.dw2.b", RS_F32, C);
  NEED(e->sub.p2w, "sub.pw2.w", RS_BF16, C * C); NEED(e->sub.p2b, "sub.pw2.b", RS_F32, C);
  NEED(e->sub.ow, "sub.out.w", RS_BF16, d * F3 * C); NEED(e->sub.ob, "sub.out.b", RS_F32, d);
  e->layers.resize(c.n_layers);
  for (int i = 0; i < c.n_layers; ++i) {
    LayerW& L = e->layers[i];
    char nm[64];
    auto N = [&](const char* s) { snprintf(nm, sizeof nm, "L%d.%s", i, s); return nm; };
    NEED(L.ln_ff1_g, N("ln_ff1.g"), RS_F32, d); NEED(L.ln_ff1_b, N("ln_ff1.b"), RS_F32, d);
    NEED(L.ff1_w1, N("ff1.w1"), RS_BF16, ff * d); NEED(L.ff1_b1, N("ff1.b1"), RS_F32, ff);
    NEED(L.ff1_w2, N("ff1.w2"), RS_BF16, d * ff); NEED(L.ff1_b2, N("ff1.b2"), RS_F32, d);
    NEED(L.ln_att_g, N("ln_att.g"), RS_F32, d); NEED(L.ln_att_b, N("ln_att.b"), RS_F32, d);
    NEED(L.wqkv, N("att.wqkv"), RS_BF16, 3 * d * d); NEED(L.bqkv, N("att.bqkv"), RS_F32, 3 * d);
    NEED(L.att_pos, N("att.pos"), RS_BF16, H * n_rel_pad * dk);
    NEED(L.att_u, N("att.u"), RS_F32, d); NEED(L.att_bdbias, N("att.bdbias"), RS_F32, H * n_rel_pad);
    NEED(L.wo, N("att.wo"), RS_BF16, d * d); NEED(L.bo, N("att.bo"), RS_F32, d);
    NEED(L.ln_conv_g, N("ln_conv.g"), RS_F32, d); NEED(L.ln_conv_b, N("ln_conv.b"), RS_F32, d);
    NEED(L.pw1_w, N("conv.pw1.w"), RS_BF16, 2 * d * d); NEED(L.pw1_b, N("conv.pw1.b"), RS_F32, 2 * d);
    NEED(L.dw_w, N("conv.dw.w"), RS_F32, k * d); NEED(L.dw_shift, N("conv.dw.shift"), RS_F32, d);
    NEED(L.pw2_w, N("conv.pw2.w"), RS_BF16, d * d); NEED(L.pw2_b, N("conv.pw2.b"), RS_F32, d);
    NEED(L.ln_ff2_g, N("ln_ff2.g"), RS_F32, d); NEED(L.ln_ff2_b, N("ln_ff2.b"), RS_F32, d);
    NEED(L.ff2_w1, N("ff2.w1"), RS_BF16, ff * d); NEED(L.ff2_b1, N("ff2.b1"), RS_F32, ff);
    NEED(L.ff2_w2, N("ff2.w2"), RS_BF16, d * ff); NEED(L.ff2_b2, N("ff2.b2"), RS_F32, d);
    NEED(L.ln_out_g, N("ln_out.g"), RS_F32, d); NEED(L.ln_out_b, N("ln_out.b"), RS_F32, d);
  }
  const int64_t Hj = c.joint_hidden, Hp = c.pred_hidden, NC = c.vocab_size + 1;
  if (e->w.count("alsd.out.w3") != 0) {                  // optional: only an engine that was asked for beam search carries these
    const int64_t n_pad = (NC + 63) / 64 * 64;
    NEED(e->alsd.out_w3, "alsd.out.w3", RS_BF16, n_pad * 3 * Hj); NEED(e->alsd.out_b, "alsd.out.b", RS_F32, n_pad);
    NEED(e->alsd.lstm_w3, "alsd.lstm.w3", RS_BF16, 4 * Hp * 6 * Hp); NEED(e->alsd.pred_w3, "alsd.pred.w3", RS_BF16, Hj * 3 * Hp);
    e->alsd.n_pad = static_cast<int>(n_pad);
  }
  NEED(e->dec.enc_w, "joint.enc.w", RS_BF16, Hj * d); NEED(e->dec.enc_b, "joint.enc.b", RS_F32, Hj);
  NEED(e->dec.out_w, "joint.out.w", RS_BF16, NC * Hj); NEED(e->dec.out_b, "joint.out.b", RS_F32, NC);
  NEED(e->dec.embed, "pred.embed", RS_F32, NC * Hp);
  NEED(e->dec.lstm_w, "pred.lstm.w", RS_BF16, 4 * Hp * 2 * Hp); NEED(e->dec.lstm_b, "pred.lstm.b", RS_F32, 4 * Hp);
  NEED(e->dec.gate_tab, "pred.gate_tab", RS_F32, NC * 4 * Hp);     // W_ih . embed[k] + b_ih + b_hh per token k (decode_spec.cu)
  NEED(e->dec.pred_w, "joint.pred.w", RS_BF16, Hj * Hp); NEED(e->dec.pred_b, "joint.pred.b", RS_F32, Hj);
  return RS_OK;
}

__global__ void enc_len_kernel(const int32_t* __restrict__ mel_len, int32_t* __restrict__ enc_len, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int n = mel_len[b];
  for (int i = 0; i < 3; ++i) n = n > 0 ? (n - 1) / 2 + 1 : 0;
  enc_len[b] = n;
}

int check_ws(rs_engine* e, const Plan& p) {
  if (e->ws == nullptr) return fail(e, RS_ERR_WORKSPACE, "no workspace set (rs_set_workspace)");
  if (p.total > e->ws_bytes)
    return fail(e, RS_ERR_WORKSPACE, "workspace too small: need %zu bytes for B=%d L_max=%d, have %zu", p.total, p.B, p.L_max, e->ws_bytes);
  return RS_OK;
}

void mark(rs_engine* e, int i, cudaStream_t s) {
  if (e->timing) cudaEventRecord(e->ev[i], s);
}

// Log-mel of utterances [b0, b0 + nb) of a batch whose statistics live at plan offsets (absolute utterance index).
// normalise = false leaves `mel` un-normalised for sub_conv0_dw1_kernel (the transcribe path); rs_logmel passes true.
int do_logmel(rs_engine* e, const void* wav, bool i16, const int32_t* len, int nb, int L_max, float* mel, int32_t* mel_len,
              float* partials, float* stats, int b0, bool normalise, cudaStream_t s) {
  Nvtx range("rs::logmel");
  const rs_model_config& c = e->cfg;
  if (b0 + nb > rs_engine::kMaxBatch) return fail(e, RS_ERR_INVALID_ARG, "batch of %d utterances exceeds the engine limit of %d", b0 + nb, rs_engine::kMaxBatch);
  rs::LogmelArgs a{};
  a.wav = wav; a.wav_i16 = i16; a.len = len; a.B = nb; a.L_max = L_max; a.mel = mel; a.mel_len = mel_len;
  a.partials = partials + static_cast<size_t>(b0) * rs::logmel_tiles(L_max, c.n_window_stride) * c.n_mels * 2;
  a.stats = stats + static_cast<size_t>(b0) * c.n_mels * 2;
  a.tickets = e->lm_tickets + b0;
  a.tb = e->fe; a.n_mels = c.n_mels; a.hop = c.n_window_stride; a.n_fft = c.n_fft; a.win = c.n_window_size;
  a.preemph = c.preemph; a.guard = c.log_zero_guard; a.eps = c.norm_eps; a.normalise_in_place = normalise;
  RS_LAUNCH(e, s, normalise ? 2 : 1, rs::launch_logmel_fused(a, s));
  return RS_OK;
}

// mel_stats == nullptr: `mel` is already normalised (rs_encode takes rs_logmel's output)
int do_sub_conv0(rs_engine* e, const Plan& p, const float* mel, const int32_t* mel_len, const float* mel_stats, int b0, int nb, cudaStream_t s) {
  Nvtx range("rs::subsampling.conv0_dw1");
  const rs_model_config& c = e->cfg;
  const int C = c.sub_channels;
  rs::SubsampleArgs sa{mel + static_cast<size_t>(b0) * p.F_max * c.n_mels, mel_len + b0,
                       mel_stats ? mel_stats + static_cast<size_t>(b0) * c.n_mels * 2 : nullptr, nb, p.F_max, c.n_mels, C,
                       e->sub.c0w, e->sub.c0b, e->sub.d1w, e->sub.d1b,
                       at<uint16_t>(e, p.sub1) + static_cast<size_t>(b0) * p.T2 * p.F2 * C, p.T1, p.F1, p.T2, p.F2};
  RS_LAUNCH(e, s, 1, rs::launch_sub_conv0_dw1(sa, s));
  return RS_OK;
}

// The encoder after the first (fused) subsampling conv, which do_sub_conv0 has enqueued on `s`.
int do_encode(rs_engine* e, const Plan& p, const int32_t* mel_len, float* enc, int32_t* enc_len, int n_layers, cudaStream_t s) {
  const rs_model_config& c = e->cfg;
  const int d = c.d_model, C = c.sub_channels, M = p.M, B = p.B;
  if (n_layers < 0 || n_layers > c.n_layers) n_layers = c.n_layers;
  RS_TRY(launch(e, s, "enc_len_kernel", 1, 0.0, [&] {
    enc_len_kernel<<<(B + 127) / 128, 128, 0, s>>>(mel_len, enc_len, B);
    return cudaGetLastError();
  }));
  // ---- ConvSubsampling
  RS_TRY(gemm(e, {at<void>(e, p.sub1), e->sub.p1w, e->sub.p1b, nullptr, at<void>(e, p.sub2), B * p.T2 * p.F2, C, C, RS_EPI_BIAS_RELU_BF16, 1.f}, s));
  RS_LAUNCH(e, s, 1, rs::launch_sub_dw(at<void>(e, p.sub2), at<void>(e, p.sub3), e->sub.d2w, e->sub.d2b, mel_len, 2, B, p.T2, p.F2,
                                       p.T3, p.F3, C, s));
  RS_TRY(gemm(e, {at<void>(e, p.sub3), e->sub.p2w, e->sub.p2b, nullptr, at<void>(e, p.sub4), B * p.T3 * p.F3, C, C, RS_EPI_BIAS_RELU_BF16, 1.f}, s));
  float* x = at<float>(e, p.x);
  Nvtx layers_range("rs::conformer_layers");
  RS_TRY(gemm(e, {at<void>(e, p.sub4), e->sub.ow, e->sub.ob, nullptr, x, M, d, p.F3 * C, RS_EPI_BIAS_F32, c.xscale}, s));
  mark(e, 2, s);
  // ---- Conformer layers
  void* xn = at<void>(e, p.xn); void* hb = at<void>(e, p.hbuf); void* ab = at<void>(e, p.abuf); void* cb = at<void>(e, p.cbuf);
  if (n_layers > 0) {
    const LayerW& L0 = e->layers[0];
    RS_LAUNCH(e, s, 1, rs::launch_layernorm(x, L0.ln_ff1_g, L0.ln_ff1_b, nullptr, xn, nullptr, nullptr, M, d, c.ln_eps, s));
  }
  auto resid_gemm = [&](const void* a, const void* w, const float* bias, int K, float alpha) -> int {
    return gemm(e, {a, w, bias, x, x, M, d, K, RS_EPI_RESID_F32, alpha}, s);
  };
  for (int i = 0; i < n_layers; ++i) {
    const LayerW& L = e->layers[i];
    char layer_name[32];
    snprintf(layer_name, sizeof layer_name, "rs::conformer_layer[%d]", i);
    Nvtx layer_range(layer_name);
    RS_TRY(gemm(e, {xn, L.ff1_w1, L.ff1_b1, nullptr, hb, M, c.d_ff, d, RS_EPI_BIAS_SWISH_BF16, 1.f}, s));
    RS_TRY(resid_gemm(hb, L.ff1_w2, L.ff1_b2, c.d_ff, 0.5f));
    RS_LAUNCH(e, s, 1, rs::launch_layernorm(x, L.ln_att_g, L.ln_att_b, nullptr, xn, nullptr, nullptr, M, d, c.ln_eps, s));
    // the relative-position term (q + pos_bias_v) . p[c] is a wgmma product inside the attention kernel (attention_tc.cu): no score tensor in HBM
    rs::AttnArgs aa{hb, L.att_pos, L.att_bdbias, p.n_rel_pad, L.att_u, ab, enc_len, B, p.T3, c.n_heads, d / c.n_heads, c.att_left, c.att_right, c.global_tokens};
    aa.vt = at<void>(e, p.vt); aa.ld_vt = p.ld_vt;
    // q | k row-major, V transposed (keys contiguous) for the attention's P.V product
    RS_TRY(gemm(e, {xn, L.wqkv, L.bqkv, nullptr, hb, M, 3 * d, d, RS_EPI_QKV_VT, 1.f, at<void>(e, p.vt), 2 * d, p.ld_vt}, s));
    RS_LAUNCH(e, s, c.global_tokens > 0 ? 2 : 1, rs::launch_attention_tc(aa, s));
    RS_TRY(resid_gemm(ab, L.wo, L.bo, d, 1.f));
    RS_LAUNCH(e, s, 1, rs::launch_layernorm(x, L.ln_conv_g, L.ln_conv_b, nullptr, xn, nullptr, nullptr, M, d, c.ln_eps, s));
    RS_TRY(gemm(e, {xn, L.pw1_w, L.pw1_b, nullptr, ab, M, 2 * d, d, RS_EPI_BIAS_GLU_BF16, 1.f}, s));
    RS_LAUNCH(e, s, 1, rs::launch_conv_dw(ab, cb, L.dw_w, L.dw_shift, enc_len, B, p.T3, d, c.conv_kernel, s));
    RS_TRY(resid_gemm(cb, L.pw2_w, L.pw2_b, d, 1.f));
    RS_LAUNCH(e, s, 1, rs::launch_layernorm(x, L.ln_ff2_g, L.ln_ff2_b, nullptr, xn, nullptr, nullptr, M, d, c.ln_eps, s));
    RS_TRY(gemm(e, {xn, L.ff2_w1, L.ff2_b1, nullptr, hb, M, c.d_ff, d, RS_EPI_BIAS_SWISH_BF16, 1.f}, s));
    RS_TRY(resid_gemm(hb, L.ff2_w2, L.ff2_b2, c.d_ff, 0.5f));
    if (i + 1 < n_layers) {   // norm_out chained with the next layer's norm_feed_forward1
      const LayerW& Ln = e->layers[i + 1];
      RS_LAUNCH(e, s, 1, rs::launch_layernorm(x, L.ln_out_g, L.ln_out_b, x, xn, Ln.ln_ff1_g, Ln.ln_ff1_b, M, d, c.ln_eps, s));
    } else {
      RS_LAUNCH(e, s, 1, rs::launch_layernorm(x, L.ln_out_g, L.ln_out_b, enc, nullptr, nullptr, nullptr, M, d, c.ln_eps, s));
    }
  }
  if (n_layers == 0) RS_CUDA(e, cudaMemcpyAsync(enc, x, static_cast<size_t>(M) * d * 4, cudaMemcpyDeviceToDevice, s));
  RS_LAUNCH(e, s, 1, rs::launch_zero_pad_rows(enc, enc_len, B, p.T3, d, s));
  return RS_OK;
}

// The resumed decode of streaming (rs_rnnt_greedy_resume, rs_stream_step): device arrays; the decode runs frames
// [dec_begin[b], dec_end[b]) of row b from record slot[b] of states
struct Resume { const int32_t* dec_begin; const int32_t* dec_end; const int32_t* slot; void* states; };

// stats == nullptr: tokens only; otherwise stats f32 [B, U_max, 4] receives (lp, H1, A_alpha, G_alpha) of every stored token.
// rs != nullptr: the resumed decode (enc_len stays the encoder's valid length; the decode ends at rs->dec_end)
int do_greedy(rs_engine* e, const Plan& p, const float* enc, const int32_t* enc_len, int T_max, int32_t* tokens,
              int32_t* frames, int32_t* ntok, int U_max, float* stats, float alpha, cudaStream_t s, const Resume* rs = nullptr) {
  Nvtx range("rs::rnnt_greedy (joint.enc projection + persistent decode)");
  const rs_model_config& c = e->cfg;
  const int M = p.B * T_max;
  RS_LAUNCH(e, s, 1, rs::launch_f32_to_bf16(enc, at<void>(e, p.xn), static_cast<int64_t>(M) * c.d_model, s));
  RS_TRY(gemm(e, {at<void>(e, p.xn), e->dec.enc_w, e->dec.enc_b, nullptr, at<void>(e, p.encp), M, c.joint_hidden, c.d_model, RS_EPI_BIAS_F32, 1.f}, s));
  mark(e, 4, s);
  rs::DecodeArgs da{at<float>(e, p.encp), rs ? rs->dec_end : enc_len, e->dec.out_w, e->dec.out_b, e->dec.lstm_w, e->dec.gate_tab, e->dec.pred_w,
                    e->dec.pred_b, tokens, frames, ntok, p.B, T_max, c.joint_hidden, c.pred_hidden, c.vocab_size, U_max, c.max_symbols,
                    stats, alpha, e->boost.bonus, e->boost.next, e->boost.n_states, e->boost.pitch, e->lm};
  if (rs) { da.dec_begin = rs->dec_begin; da.slot = rs->slot; da.states = rs->states; }
  if (e->n_roots > 0) {             // ordered on s like the workspace: the previous decode has read the previous roots
    RS_CUDA(e, cudaMemcpyAsync(e->boost_roots, e->roots_host.data(), static_cast<size_t>(p.B) * 4, cudaMemcpyHostToDevice, s));
    da.boost_root = e->boost_roots;
  }
  // One decode kernel for every batch size (windowed, weights-stationary, joint on wgmma: decode_spec.cu): an utterance's
  // logits are accumulated in the same order whether it is decoded alone or inside a batch, so results do not depend on
  // batch composition.
  RS_LAUNCH(e, s, 2, rs::launch_rnnt_greedy_spec(da, at<void>(e, p.dec_ws), e->num_sms, s));   // workspace memset + kernel
  return RS_OK;
}

}  // namespace

extern "C" {

int rs_engine_create(const rs_model_config* cfg, const rs_tensor* weights, int n_weights, int device, rs_engine** out) {
  if (cfg == nullptr || weights == nullptr || out == nullptr) return fail(nullptr, RS_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  if (cfg->n_fft != 512) return fail(nullptr, RS_ERR_UNSUPPORTED, "n_fft=%d unsupported (frontend kernel is built for 512)", cfg->n_fft);
  if (cfg->d_model % cfg->n_heads || cfg->d_model / cfg->n_heads != 128)
    return fail(nullptr, RS_ERR_UNSUPPORTED, "d_model/n_heads must be 128 (got %d/%d)", cfg->d_model, cfg->n_heads);
  if (cfg->d_model != 256 && cfg->d_model != 512 && cfg->d_model != 1024)
    return fail(nullptr, RS_ERR_UNSUPPORTED, "d_model=%d unsupported (256/512/1024)", cfg->d_model);
  if (cfg->conv_kernel != 9) return fail(nullptr, RS_ERR_UNSUPPORTED, "conv_kernel=%d unsupported (9)", cfg->conv_kernel);
  if (cfg->global_tokens < 0 || cfg->global_tokens > 1)
    return fail(nullptr, RS_ERR_UNSUPPORTED, "global_tokens=%d unsupported (the attention kernels implement 0 or 1)", cfg->global_tokens);
  if (cfg->att_left < 0 || cfg->att_right < 0 || cfg->att_left > 128 || cfg->att_right > 128 || (cfg->att_left & 7))
    return fail(nullptr, RS_ERR_UNSUPPORTED, "att context (%d, %d) unsupported: the attention kernel covers limited local context with 0 <= left, right <= 128 and left %% 8 == 0 (the shipped model is [128, 128])", cfg->att_left, cfg->att_right);
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(nullptr, RS_ERR_CUDA, "no CUDA device available (%s); this engine has no CPU path", cudaGetErrorString(ce));
  if (device < 0 || device >= ndev) return fail(nullptr, RS_ERR_INVALID_ARG, "device %d out of range (%d devices)", device, ndev);
  ce = cudaSetDevice(device);
  if (ce != cudaSuccess) return fail(nullptr, RS_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(ce));
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9) return fail(nullptr, RS_ERR_UNSUPPORTED, "device %d is sm_%d%d; kernels are built for sm_90a only", device, prop.major, prop.minor);
  rs_engine* e = new rs_engine();
  e->cfg = *cfg; e->device = device; e->num_sms = prop.multiProcessorCount;
  for (int i = 0; i < n_weights; ++i) e->w[weights[i].name] = Tensor{weights[i].dev_ptr, weights[i].dtype, weights[i].numel};
  int r = bind_weights(e);
  if (r != RS_OK) { snprintf(g_create_error, sizeof g_create_error, "%s", e->err); delete e; return r; }
  ce = cudaMalloc(&e->lm_tickets, rs_engine::kMaxBatch * sizeof(unsigned int));
  if (ce == cudaSuccess) ce = cudaMemset(e->lm_tickets, 0, rs_engine::kMaxBatch * sizeof(unsigned int));
  if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking);
  for (auto& ev : e->ev) if (ce == cudaSuccess) ce = cudaEventCreate(&ev);
  for (auto& ev : e->copy_ev) if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
  if (ce != cudaSuccess) {
    snprintf(g_create_error, sizeof g_create_error, "cannot create the log-mel ticket array, copy stream or events (%s)", cudaGetErrorString(ce));
    rs_engine_destroy(e);
    return RS_ERR_CUDA;
  }
  *out = e;
  return RS_OK;
}

void rs_engine_destroy(rs_engine* e) {
  if (e == nullptr) return;
  for (auto& ev : e->ev) if (ev) cudaEventDestroy(ev);
  for (auto& ev : e->copy_ev) if (ev) cudaEventDestroy(ev);
  if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
  for (auto& ev : e->log_ev) cudaEventDestroy(ev);
  cudaFree(e->lm_tickets);
  cudaFree(e->alsd_ws);
  cudaFree(e->align_ws);
  cudaFree(e->stream_args);
  cudaFree(e->spot.mem);
  cudaFree(e->spot_ws);
  cudaFree(e->boost_roots);
  if (e->alsd_done_host) cudaFreeHost(e->alsd_done_host);
  delete e;
}

const char* rs_last_error(const rs_engine* e) { return e ? e->err : g_create_error; }

int rs_set_phrase_boosting(rs_engine* e, const float* bonus_dev, const int32_t* next_dev, int n_states, int pitch) {
  if (e == nullptr) return RS_ERR_INVALID_ARG;
  if (n_states == 0) {
    e->boost = {};
    e->n_roots = 0;
    return RS_OK;
  }
  if (n_states < 1 || n_states > RS_MAX_BOOST_STATES)
    return fail(e, RS_ERR_INVALID_ARG, "rs_set_phrase_boosting: n_states=%d outside [1, %d]", n_states, RS_MAX_BOOST_STATES);
  if (pitch < e->cfg.vocab_size || pitch % 4 != 0)
    return fail(e, RS_ERR_INVALID_ARG, "rs_set_phrase_boosting: pitch=%d must be >= vocab_size (%d) and a multiple of 4", pitch, e->cfg.vocab_size);
  if (bonus_dev == nullptr || next_dev == nullptr || ((reinterpret_cast<uintptr_t>(bonus_dev) | reinterpret_cast<uintptr_t>(next_dev)) & 15u))
    return fail(e, RS_ERR_INVALID_ARG, "rs_set_phrase_boosting: bonus and next must be non-null and 16-byte aligned");
  e->boost.bonus = bonus_dev; e->boost.next = next_dev; e->boost.n_states = n_states; e->boost.pitch = pitch;
  e->n_roots = 0;                         // roots index the table they were set for
  return RS_OK;
}

int rs_set_boost_roots(rs_engine* e, const int32_t* roots_host, int n) {
  if (e == nullptr) return RS_ERR_INVALID_ARG;
  if (n == 0) {
    e->n_roots = 0;
    return RS_OK;
  }
  if (n < 0 || roots_host == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_set_boost_roots: n=%d must be >= 0 and roots non-null", n);
  if (e->boost.bonus == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_set_boost_roots: no phrase-boosting table is set (rs_set_phrase_boosting)");
  for (int b = 0; b < n; ++b)
    if (roots_host[b] < 0 || roots_host[b] >= e->boost.n_states)
      return fail(e, RS_ERR_INVALID_ARG, "rs_set_boost_roots: roots[%d] = %d outside [0, %d)", b, roots_host[b], e->boost.n_states);
  if (n > e->roots_cap) {                 // growing: a decode still queued may read the old buffer
    RS_CUDA(e, cudaSetDevice(e->device));
    RS_CUDA(e, cudaDeviceSynchronize());
    cudaFree(e->boost_roots); e->boost_roots = nullptr; e->roots_cap = 0; e->n_roots = 0;
    RS_CUDA(e, cudaMalloc(&e->boost_roots, static_cast<size_t>(n) * 4));
    e->roots_cap = n;
  }
  e->roots_host.assign(roots_host, roots_host + n);
  e->n_roots = n;
  return RS_OK;
}

int rs_set_ngram_lm(rs_engine* e, const rs_ngram_lm* lm) {
  if (e == nullptr) return RS_ERR_INVALID_ARG;
  if (lm == nullptr) {
    e->lm = {};
    return RS_OK;
  }
  if (lm->order < 2 || lm->order > RS_MAX_LM_ORDER)
    return fail(e, RS_ERR_INVALID_ARG, "rs_set_ngram_lm: order=%d outside [2, %d]", lm->order, RS_MAX_LM_ORDER);
  if (lm->n_states < 1 || lm->n_arcs < 0 || lm->start_state < 0 || lm->start_state >= lm->n_states)
    return fail(e, RS_ERR_INVALID_ARG, "rs_set_ngram_lm: n_states=%d, n_arcs=%d, start_state=%d (need n_states >= 1, n_arcs >= 0, "
                "0 <= start_state < n_states)", lm->n_states, lm->n_arcs, lm->start_state);
  if (lm->pitch < e->cfg.vocab_size || lm->pitch % 4 != 0)
    return fail(e, RS_ERR_INVALID_ARG, "rs_set_ngram_lm: pitch=%d must be >= vocab_size (%d) and a multiple of 4", lm->pitch, e->cfg.vocab_size);
  const void* arrays[] = {lm->cb, lm->chain, lm->arc_begin, lm->arc_tok, lm->arc_to, lm->arc_w, lm->uni_w, lm->uni_to};
  for (const void* a : arrays)
    if (a == nullptr || (reinterpret_cast<uintptr_t>(a) & 15u))
      return fail(e, RS_ERR_INVALID_ARG, "rs_set_ngram_lm: every array must be non-null and 16-byte aligned");
  rs::NgramLM t;
  t.cb = lm->cb; t.chain = lm->chain; t.arc_begin = lm->arc_begin; t.arc_tok = lm->arc_tok; t.arc_to = lm->arc_to; t.arc_w = lm->arc_w;
  t.uni_w = lm->uni_w; t.uni_to = lm->uni_to;
  t.order = lm->order; t.n_states = lm->n_states; t.n_arcs = lm->n_arcs; t.pitch = lm->pitch; t.start_state = lm->start_state;
  e->lm = t;
  return RS_OK;
}

int rs_ngram_lm_eval(rs_engine* e, const int32_t* states_dev, const int32_t* tokens_dev, int n, float* score_dev, int32_t* next_dev,
                     void* stream) {
  if (e == nullptr || n < 0 || (n > 0 && (!states_dev || !tokens_dev || !score_dev || !next_dev)))
    return fail(e, RS_ERR_INVALID_ARG, "rs_ngram_lm_eval: bad arguments");
  if (e->lm.order == 0) return fail(e, RS_ERR_INVALID_ARG, "rs_ngram_lm_eval: no n-gram LM is set (rs_set_ngram_lm)");
  RS_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RS_LAUNCH(e, s, 1, rs::launch_ngram_lm_eval(e->lm, e->cfg.vocab_size, e->num_sms, states_dev, tokens_dev, n, score_dev, next_dev, s));
  return RS_OK;
}

int rs_workspace_bytes(const rs_engine* e, int B, int L_max, size_t* bytes) {
  if (e == nullptr || bytes == nullptr || B <= 0 || L_max <= 0) return fail(e, RS_ERR_INVALID_ARG, "bad arguments");
  // token capacity: max_symbols per encoder frame is the hard upper bound of the greedy loop
  const int T = enc_capacity(L_max / e->cfg.n_window_stride + 1);
  *bytes = make_plan(e, B, L_max, T * e->cfg.max_symbols).total;
  return RS_OK;
}

int rs_set_workspace(rs_engine* e, void* dev_ptr, size_t bytes) {
  if (e == nullptr) return RS_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(dev_ptr) & 255) return fail(e, RS_ERR_INVALID_ARG, "workspace must be 256-byte aligned");
  e->ws = dev_ptr; e->ws_bytes = bytes;
  return RS_OK;
}

int rs_mel_frames(const rs_engine* e, int n) { return n / e->cfg.n_window_stride + 1; }
int rs_enc_frames(const rs_engine* e, int n) { return enc_capacity(rs_mel_frames(e, n)); }
int rs_mel_valid(const rs_engine* e, int n) { return (n + 2 * (e->cfg.n_fft / 2) - e->cfg.n_fft) / e->cfg.n_window_stride; }
int rs_enc_valid(const rs_engine* e, int n) { return conv_len(conv_len(conv_len(rs_mel_valid(e, n)))); }

int rs_logmel(rs_engine* e, const float* wav, const int32_t* len, int B, int L_max, float* mel, int32_t* mel_len, void* stream) {
  if (!e || !wav || !len || !mel || !mel_len || B <= 0 || L_max <= 0) return fail(e, RS_ERR_INVALID_ARG, "rs_logmel: bad arguments");
  RS_CUDA(e, cudaSetDevice(e->device));
  Plan p = make_plan(e, B, L_max, 1);               // the statistics scratch lives in the workspace
  RS_TRY(check_ws(e, p));
  return do_logmel(e, wav, false, len, B, L_max, mel, mel_len, at<float>(e, p.mel_part), at<float>(e, p.mel_stats), 0, true,
                   static_cast<cudaStream_t>(stream));
}

int rs_encode(rs_engine* e, const float* mel, const int32_t* mel_len, int B, int F_max, float* enc, int32_t* enc_len,
              int n_layers, void* stream) {
  if (!e || !mel || !mel_len || !enc || !enc_len || B <= 0 || F_max <= 0) return fail(e, RS_ERR_INVALID_ARG, "rs_encode: bad arguments");
  RS_CUDA(e, cudaSetDevice(e->device));
  const int L_max = (F_max - 1) * e->cfg.n_window_stride;
  Plan p = make_plan(e, B, L_max, 1);
  RS_TRY(check_ws(e, p));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RS_TRY(do_sub_conv0(e, p, mel, mel_len, nullptr, 0, B, s));
  return do_encode(e, p, mel_len, enc, enc_len, n_layers, s);
}

}  // extern "C"

namespace {

bool alpha_ok(float alpha) { return alpha > 0.f && std::isfinite(alpha); }

// Per-row boosting roots, when set, must cover every row of the batch
int check_roots(rs_engine* e, const char* fn, int B) {
  if (e->n_roots > 0 && B > e->n_roots)
    return fail(e, RS_ERR_INVALID_ARG, "%s: B=%d rows but only %d boosting roots are set (rs_set_boost_roots)", fn, B, e->n_roots);
  return RS_OK;
}

int rnnt_greedy(rs_engine* e, const char* fn, const float* enc, const int32_t* enc_len, int B, int T_max, int32_t* tokens,
                int32_t* frames, int32_t* n_tok, int U_max, float* stats, float alpha, cudaStream_t s, const Resume* rs = nullptr) {
  if (!e || !enc || !enc_len || !tokens || !frames || !n_tok || B <= 0 || T_max <= 0 || U_max <= 0)
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments", fn);
  RS_TRY(check_roots(e, fn, B));
  RS_CUDA(e, cudaSetDevice(e->device));
  Plan p{};
  // only xn / encp / dec_ws are touched: size them for M = B*T_max rows
  p.B = B; p.M = B * T_max;
  rs::Arena a;
  p.xn = a.take(static_cast<size_t>(p.M) * e->cfg.d_model * 2);
  p.encp = a.take(static_cast<size_t>(p.M) * e->cfg.joint_hidden * 4);
  p.dec_ws = a.take(dec_ws(e, B).total);
  p.total = a.off;
  RS_TRY(check_ws(e, p));
  return do_greedy(e, p, enc, enc_len, T_max, tokens, frames, n_tok, U_max, stats, alpha, s, rs);
}

}  // namespace

extern "C" {

int rs_rnnt_greedy(rs_engine* e, const float* enc, const int32_t* enc_len, int B, int T_max, int32_t* tokens,
                   int32_t* frames, int32_t* n_tok, int U_max, void* stream) {
  return rnnt_greedy(e, "rs_rnnt_greedy", enc, enc_len, B, T_max, tokens, frames, n_tok, U_max, nullptr, 0.f, static_cast<cudaStream_t>(stream));
}

int rs_rnnt_greedy_confidence(rs_engine* e, const float* enc, const int32_t* enc_len, int B, int T_max, int32_t* tokens,
                              int32_t* frames, int32_t* n_tok, int U_max, float alpha, float* stats, void* stream) {
  if (!stats || !alpha_ok(alpha)) return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_greedy_confidence: bad arguments (stats must be set, alpha > 0 and finite)");
  return rnnt_greedy(e, "rs_rnnt_greedy_confidence", enc, enc_len, B, T_max, tokens, frames, n_tok, U_max, stats, alpha,
                     static_cast<cudaStream_t>(stream));
}

size_t rs_stream_state_bytes(const rs_engine* e) {
  return e ? rs::stream_state_bytes(e->cfg.joint_hidden, e->cfg.pred_hidden) : 0;
}

int rs_rnnt_greedy_resume(rs_engine* e, const float* enc, const int32_t* dec_begin, const int32_t* dec_end, const int32_t* slot,
                          void* states, int B, int T_max, int32_t* tokens, int32_t* frames, int32_t* n_tok, int U_max, float alpha,
                          float* stats, void* stream) {
  if (!dec_begin || !dec_end || !slot || !states || (stats && !alpha_ok(alpha)))
    return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_greedy_resume: bad arguments (dec_begin, dec_end, slot and states must be set; with stats, alpha > 0 and finite)");
  if (reinterpret_cast<uintptr_t>(states) & 15u) return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_greedy_resume: states must be 16-byte aligned");
  const Resume rs{dec_begin, dec_end, slot, states};
  return rnnt_greedy(e, "rs_rnnt_greedy_resume", enc, dec_end, B, T_max, tokens, frames, n_tok, U_max, stats, alpha,
                     static_cast<cudaStream_t>(stream), &rs);
}

}  // extern "C"

namespace {

int grow_align_ws(rs_engine* e, const char* fn, size_t bytes, cudaStream_t s);

// Streaming keyword spotting (spot_stream.cu; semantics: reazonspeech_b200/keywords.py, "Streaming").  One call's rows: host
// copies of dec_begin / dec_end / slot / last (checked before any launch), the records, and the host outputs.
struct SpotCall {
  const int32_t *dec_begin, *dec_end, *slot, *last;
  void* records; int n_slots;
  int max_out; int32_t* meta; float* val; int32_t* frames; float* token_lp; int32_t* n_out;
  float* E; int32_t* S; int32_t* sigma;          // device, optional (the test seam)
};

int spot_capacity(const rs_engine* e, int B) {
  const int64_t n = static_cast<int64_t>(B) * e->spot.n_kw * e->spot.ring_cap;
  return n > INT32_MAX ? -1 : static_cast<int>(n);
}

// Rows bounded by T_lim frames (the seam: T_max; a step: rs_stream_step's own checks come first).
int check_spot_call(rs_engine* e, const char* fn, int B, int T_lim, const SpotCall& c) {
  if (e->spot.n_kw == 0) return fail(e, RS_ERR_INVALID_ARG, "%s: no keyword set is installed (rs_set_spot_keywords)", fn);
  if (!c.records || (reinterpret_cast<uintptr_t>(c.records) & 15u) || c.n_slots < 1 || !c.meta || !c.val || !c.frames || !c.token_lp ||
      !c.n_out || ((c.E != nullptr) != (c.S != nullptr)))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments (records 16-byte aligned, n_slots >= 1, every hit output set, E and S both or neither)", fn);
  const int cap = spot_capacity(e, B);
  if (cap < 0)
    return fail(e, RS_ERR_INVALID_ARG, "%s: B=%d rows x %d keywords x %d ring entries exceed one call's hit list: fewer rows per call", fn, B,
                e->spot.n_kw, e->spot.ring_cap);
  if (c.max_out < cap)
    return fail(e, RS_ERR_INVALID_ARG, "%s: max_out=%d is below rs_spot_max_hits(B=%d) = %d", fn, c.max_out, B, cap);
  std::vector<int32_t> seen(c.slot, c.slot + B);
  std::sort(seen.begin(), seen.end());
  if (seen[0] < 0 || seen.back() >= c.n_slots || std::adjacent_find(seen.begin(), seen.end()) != seen.end())
    return fail(e, RS_ERR_INVALID_ARG, "%s: slots must be distinct and in [0, n_slots = %d)", fn, c.n_slots);
  for (int b = 0; b < B; ++b)
    if (c.dec_begin[b] < 0 || c.dec_begin[b] > c.dec_end[b] || c.dec_end[b] > T_lim || c.dec_end[b] - c.dec_begin[b] > e->spot.chunk)
      return fail(e, RS_ERR_INVALID_ARG, "%s: row %d: need 0 <= dec_begin (%d) <= dec_end (%d) <= %d and at most %d frames (the installed chunk)",
                  fn, b, c.dec_begin[b], c.dec_end[b], T_lim, e->spot.chunk);
  return RS_OK;
}

// The compact block's frames per row: the longest range (at least 1)
int spot_frames(int B, const SpotCall& c) {
  int C = 1;
  for (int b = 0; b < B; ++b) C = std::max(C, c.dec_end[b] - c.dec_begin[b]);
  return C;
}

// The scratch of one call: staged row arguments, the gathered block and lengths, the pairs' lattice, and the hit list
struct SpotLayout { size_t args, blk, len, lpb, lpe, n, meta, val, fr, lp, total; int cap; };
SpotLayout spot_layout(const rs_engine* e, int B, int C) {
  const auto& ks = e->spot;
  const size_t cells = static_cast<size_t>(B) * ks.n_kw * C * (ks.U_max + 1);
  SpotLayout L;
  L.cap = spot_capacity(e, B);
  const size_t cap = static_cast<size_t>(L.cap);
  rs::Arena a;
  L.args = a.take(static_cast<size_t>(4) * B * 4); L.blk = a.take(static_cast<size_t>(B) * C * e->cfg.joint_hidden * 4);
  L.len = a.take(static_cast<size_t>(B) * 4); L.lpb = a.take(cells * 4); L.lpe = a.take(cells * 4); L.n = a.take(4);
  L.meta = a.take(cap * rs::kSpotHitInts * 4); L.val = a.take(cap * 8);
  L.fr = a.take(cap * ks.U_max * 4); L.lp = a.take(cap * ks.U_max * 4);
  L.total = a.off;
  return L;
}

// Enqueues the gather, the pairs' lattice, the resumed recursion and the streaming pick on `encp` (joint.enc of every frame,
// f32 [B][T_max][Hj]).  args_dev: dec_begin | dec_end | slot | last on the device, or nullptr to stage the host copies.
int spot_enqueue(rs_engine* e, const char* fn, const float* encp, int T_max, int B, const SpotCall& c, const int32_t* args_dev,
                 cudaStream_t s) {
  const rs_model_config& cfg = e->cfg;
  const auto& ks = e->spot;
  const int Hj = cfg.joint_hidden, C = spot_frames(B, c);
  const SpotLayout L = spot_layout(e, B, C);
  if (L.total > e->spot_ws_bytes) {
    RS_CUDA(e, cudaStreamSynchronize(s));
    cudaFree(e->spot_ws); e->spot_ws = nullptr; e->spot_ws_bytes = 0;
    if (cudaMalloc(&e->spot_ws, L.total) != cudaSuccess) {
      cudaGetLastError();
      return fail(e, RS_ERR_WORKSPACE, "%s: cannot allocate %zu bytes of keyword scratch", fn, L.total);
    }
    e->spot_ws_bytes = L.total;
  }
  char* ws = static_cast<char*>(e->spot_ws);
  if (args_dev == nullptr) {                       // pageable sources: each copy has read its source when it returns
    int32_t* d = reinterpret_cast<int32_t*>(ws + L.args);
    const int32_t* src[4] = {c.dec_begin, c.dec_end, c.slot, c.last};
    for (int i = 0; i < 4; ++i) RS_CUDA(e, cudaMemcpyAsync(d + i * B, src[i], static_cast<size_t>(B) * 4, cudaMemcpyHostToDevice, s));
    args_dev = d;
  }
  rs::SpotStreamArgs sa{};
  sa.dec_begin = args_dev; sa.dec_end = args_dev + B; sa.slot = args_dev + 2 * B; sa.last = args_dev + 3 * B;
  sa.B = B; sa.n_kw = ks.n_kw; sa.U_max = ks.U_max; sa.C = C; sa.delay = ks.delay; sa.ring_cap = ks.ring_cap; sa.threshold = ks.threshold;
  sa.label_len = ks.label_len; sa.records = static_cast<uint8_t*>(c.records); sa.len = reinterpret_cast<int32_t*>(ws + L.len);
  sa.E_out = c.E; sa.S_out = c.S; sa.T_out = T_max; sa.sigma_out = c.sigma;
  sa.n_hits = reinterpret_cast<int32_t*>(ws + L.n); sa.hit_cap = L.cap;
  sa.hit_meta = reinterpret_cast<int32_t*>(ws + L.meta); sa.hit_val = reinterpret_cast<float*>(ws + L.val);
  sa.hit_frames = reinterpret_cast<int32_t*>(ws + L.fr); sa.hit_lp = reinterpret_cast<float*>(ws + L.lp);
  float* blk = reinterpret_cast<float*>(ws + L.blk);
  rs::AlignArgs g{};
  g.enc_proj = blk; g.enc_len = sa.len; g.labels = ks.labels; g.label_len = ks.label_len;
  g.w_out = e->dec.out_w; g.b_out = e->dec.out_b;
  g.B = ks.n_kw; g.T_max = C; g.U_max = ks.U_max; g.Hj = Hj; g.Hp = cfg.pred_hidden; g.V = cfg.vocab_size;
  g.pred_proj = ks.pred_proj; g.lp_blank = reinterpret_cast<float*>(ws + L.lpb); g.lp_emit = reinterpret_cast<float*>(ws + L.lpe);
  Nvtx range("rs::rnnt_spot_resume");
  RS_CUDA(e, cudaMemsetAsync(sa.n_hits, 0, 4, s));
  RS_LAUNCH(e, s, 1, rs::launch_spot_gather(encp, T_max, Hj, sa, blk, s));
  {
    char msg[256] = "";
    const int r = launch(e, s, "rnnt_lattice_kernel<pairs>", 1, 0.0, [&] { return rs::launch_rnnt_lattice_pairs(g, B, s, msg); });
    if (r != RS_OK && msg[0] != '\0') return fail(e, r, "%s: %s", fn, msg);
    RS_TRY(r);
  }
  RS_LAUNCH(e, s, 1, rs::launch_rnnt_spot_resume_dp(g, sa, s));
  RS_LAUNCH(e, s, 1, rs::launch_rnnt_spot_resume_pick(sa, s));
  return RS_OK;
}

// Copies the decided hits back, sorted by (row, keyword, e); synchronises.
int spot_collect(rs_engine* e, int B, const SpotCall& c, cudaStream_t s) {
  const int UM = e->spot.U_max;
  const SpotLayout L = spot_layout(e, B, spot_frames(B, c));
  const int cap = L.cap;
  const char* ws = static_cast<const char*>(e->spot_ws);
  int32_t n = 0;
  RS_CUDA(e, cudaMemcpyAsync(&n, ws + L.n, 4, cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaStreamSynchronize(s));
  n = std::min(n, cap);
  std::vector<int32_t> meta(static_cast<size_t>(n) * rs::kSpotHitInts), fr(static_cast<size_t>(n) * UM);
  std::vector<float> val(static_cast<size_t>(n) * 2), lp(static_cast<size_t>(n) * UM);
  if (n > 0) {
    RS_CUDA(e, cudaMemcpyAsync(meta.data(), ws + L.meta, meta.size() * 4, cudaMemcpyDeviceToHost, s));
    RS_CUDA(e, cudaMemcpyAsync(val.data(), ws + L.val, val.size() * 4, cudaMemcpyDeviceToHost, s));
    RS_CUDA(e, cudaMemcpyAsync(fr.data(), ws + L.fr, fr.size() * 4, cudaMemcpyDeviceToHost, s));
    RS_CUDA(e, cudaMemcpyAsync(lp.data(), ws + L.lp, lp.size() * 4, cudaMemcpyDeviceToHost, s));
    RS_CUDA(e, cudaStreamSynchronize(s));
  }
  std::vector<int> order(n);
  for (int i = 0; i < n; ++i) order[i] = i;
  const auto key = [&](int i) { const int32_t* m = &meta[static_cast<size_t>(i) * rs::kSpotHitInts]; return std::make_tuple(m[0], m[1], m[3]); };
  std::sort(order.begin(), order.end(), [&](int x, int y) { return key(x) < key(y); });
  for (int j = 0; j < n; ++j) {
    const size_t i = order[j];
    std::copy_n(&meta[i * rs::kSpotHitInts], rs::kSpotHitInts, c.meta + static_cast<size_t>(j) * rs::kSpotHitInts);
    std::copy_n(&val[i * 2], 2, c.val + static_cast<size_t>(j) * 2);
    std::copy_n(&fr[i * UM], UM, c.frames + static_cast<size_t>(j) * UM);
    std::copy_n(&lp[i * UM], UM, c.token_lp + static_cast<size_t>(j) * UM);
  }
  *c.n_out = n;
  return RS_OK;
}

int check_transcribe_args(rs_engine* e, const char* fn, const void* wav, const int32_t* len, int B, int L_max, const int32_t* tokens,
                          const int32_t* frames, const int32_t* n_tok, int U_max) {
  if (!e || !wav || !len || !tokens || !frames || !n_tok || B <= 0 || L_max <= 0 || U_max <= 0)
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments", fn);
  RS_TRY(check_roots(e, fn, B));
  RS_CUDA(e, cudaSetDevice(e->device));
  return RS_OK;
}

// The whole path over plan `p`, the batch's utterances taken in n_chunks equal chunks (the last may be shorter): per chunk
// log-mel and the fused first subsampling conv, then the rest of the encoder and the greedy decode over the whole batch.
// landed[c] (when not null) is recorded once chunk c's samples have been copied in.  `wav` holds f32 samples, or int16 PCM
// (scaled by 2^-15 inside the log-mel kernel) when i16.
int run_pipeline(rs_engine* e, const Plan& p, const void* wav, bool i16, const int32_t* len, int n_chunks, const cudaEvent_t* landed,
                 int32_t* tokens, int32_t* frames, int32_t* n_tok, int U_max, float* conf_stats, float alpha, cudaStream_t s,
                 const Resume* rs = nullptr) {
  const int B = p.B, per = (B + n_chunks - 1) / n_chunks;
  const size_t row_bytes = static_cast<size_t>(p.L_max) * (i16 ? 2 : 4);
  float* mel = at<float>(e, p.mel);
  int32_t* mel_len = at<int32_t>(e, p.mel_len);
  float* stats = at<float>(e, p.mel_stats);
  mark(e, 0, s);
  for (int c = 0, b0 = 0; b0 < B; ++c, b0 += per) {
    const int nb = (B - b0 < per) ? B - b0 : per;
    if (landed != nullptr) RS_CUDA(e, cudaStreamWaitEvent(s, landed[c], 0));
    RS_TRY(do_logmel(e, static_cast<const char*>(wav) + b0 * row_bytes, i16, len + b0, nb, p.L_max,
                     mel + static_cast<size_t>(b0) * p.F_max * e->cfg.n_mels, mel_len + b0, at<float>(e, p.mel_part), stats, b0, false, s));
    mark(e, 1, s);                                      // of several chunks, the last one's record counts
    RS_TRY(do_sub_conv0(e, p, mel, mel_len, stats, b0, nb, s));
  }
  RS_TRY(do_encode(e, p, mel_len, at<float>(e, p.enc), at<int32_t>(e, p.enc_len), -1, s));
  mark(e, 3, s);
  RS_TRY(do_greedy(e, p, at<float>(e, p.enc), at<int32_t>(e, p.enc_len), p.T3, tokens, frames, n_tok, U_max, conf_stats, alpha, s, rs));
  mark(e, 5, s);
  return RS_OK;
}

int transcribe_device(rs_engine* e, const char* fn, const void* wav, bool i16, const int32_t* len, int B, int L_max, int32_t* tokens,
                      int32_t* frames, int32_t* n_tok, int U_max, float* stats, float alpha, cudaStream_t s) {
  RS_TRY(check_transcribe_args(e, fn, wav, len, B, L_max, tokens, frames, n_tok, U_max));
  Plan p = make_plan(e, B, L_max, U_max);
  RS_TRY(check_ws(e, p));
  return run_pipeline(e, p, wav, i16, len, 1, nullptr, tokens, frames, n_tok, U_max, stats, alpha, s);
}

// Host buffers in, host buffers out (the model.transcribe seam): H2D in utterance chunks on the copy stream, overlapped with
// the frontend of the chunks that have landed; D2H of the tokens (and of the statistics when stats_host is set); synchronises
// before returning.
// rs (host arrays dec_begin / dec_end / slot, device states): the resumed decode of rs_stream_step; the three arrays are copied
// into an engine-owned device buffer first.
int transcribe_batch(rs_engine* e, const char* fn, const void* wav_host, bool i16, const int32_t* len_host, int B, int L_max,
                     int32_t* tokens_host, int32_t* frames_host, int32_t* n_tok_host, int U_max, float* stats_host, float alpha,
                     cudaStream_t s, const Resume* rs_host = nullptr, const SpotCall* spot = nullptr) {
  RS_TRY(check_transcribe_args(e, fn, wav_host, len_host, B, L_max, tokens_host, frames_host, n_tok_host, U_max));
  Plan p = make_plan(e, B, L_max, U_max);
  RS_TRY(check_ws(e, p));
  Resume rs_dev{};
  if (rs_host) {
    const size_t need_bytes = static_cast<size_t>(3) * B * 4;
    if (need_bytes > e->stream_args_bytes) {
      RS_CUDA(e, cudaStreamSynchronize(s));
      cudaFree(e->stream_args); e->stream_args = nullptr; e->stream_args_bytes = 0;
      RS_CUDA(e, cudaMalloc(&e->stream_args, need_bytes));
      e->stream_args_bytes = need_bytes;
    }
    int32_t* d = static_cast<int32_t*>(e->stream_args);
    RS_CUDA(e, cudaMemcpyAsync(d, rs_host->dec_begin, static_cast<size_t>(B) * 4, cudaMemcpyHostToDevice, s));
    RS_CUDA(e, cudaMemcpyAsync(d + B, rs_host->dec_end, static_cast<size_t>(B) * 4, cudaMemcpyHostToDevice, s));
    RS_CUDA(e, cudaMemcpyAsync(d + 2 * B, rs_host->slot, static_cast<size_t>(B) * 4, cudaMemcpyHostToDevice, s));
    rs_dev = {d, d + B, d + 2 * B, rs_host->states};
  }
  const size_t row_bytes = static_cast<size_t>(L_max) * (i16 ? 2 : 4);   // the waveform region of the workspace is sized for f32
  char* wav = at<char>(e, p.wav);
  const char* wav_h = static_cast<const char*>(wav_host);
  int32_t* len = at<int32_t>(e, p.len);
  const int n_chunks = B >= 2 * rs_engine::kCopyChunks ? rs_engine::kCopyChunks : 1;
  if (n_chunks == 1) {
    RS_CUDA(e, cudaMemcpyAsync(wav, wav_h, B * row_bytes, cudaMemcpyHostToDevice, s));
    RS_CUDA(e, cudaMemcpyAsync(len, len_host, static_cast<size_t>(B) * 4, cudaMemcpyHostToDevice, s));
  } else {
    // copies on the copy stream, chunk by chunk; log-mel and the first (fused) subsampling conv of a chunk start as
    // soon as its samples have landed.  The copy stream first waits for everything already queued on the caller's
    // stream (the workspace may still be in use by an earlier asynchronous call).
    const int per = (B + n_chunks - 1) / n_chunks;
    RS_CUDA(e, cudaEventRecord(e->copy_ev[n_chunks], s));
    RS_CUDA(e, cudaStreamWaitEvent(e->copy_stream, e->copy_ev[n_chunks], 0));
    RS_CUDA(e, cudaMemcpyAsync(len, len_host, static_cast<size_t>(B) * 4, cudaMemcpyHostToDevice, e->copy_stream));
    for (int c = 0, b0 = 0; b0 < B; ++c, b0 += per) {
      const int nb = (B - b0 < per) ? B - b0 : per;
      RS_CUDA(e, cudaMemcpyAsync(wav + b0 * row_bytes, wav_h + b0 * row_bytes, nb * row_bytes, cudaMemcpyHostToDevice, e->copy_stream));
      RS_CUDA(e, cudaEventRecord(e->copy_ev[c], e->copy_stream));
    }
  }
  RS_TRY(run_pipeline(e, p, wav, i16, len, n_chunks, n_chunks > 1 ? e->copy_ev : nullptr, at<int32_t>(e, p.tokens),
                      at<int32_t>(e, p.frames), at<int32_t>(e, p.ntok), U_max, stats_host ? at<float>(e, p.stats) : nullptr, alpha, s,
                      rs_host ? &rs_dev : nullptr));
  if (spot) RS_TRY(spot_enqueue(e, fn, at<float>(e, p.encp), p.T3, B, *spot, nullptr, s));   // on the decode's joint.enc rows
  RS_CUDA(e, cudaMemcpyAsync(tokens_host, at<int32_t>(e, p.tokens), static_cast<size_t>(B) * U_max * 4, cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaMemcpyAsync(frames_host, at<int32_t>(e, p.frames), static_cast<size_t>(B) * U_max * 4, cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaMemcpyAsync(n_tok_host, at<int32_t>(e, p.ntok), static_cast<size_t>(B) * 4, cudaMemcpyDeviceToHost, s));
  if (stats_host)
    RS_CUDA(e, cudaMemcpyAsync(stats_host, at<float>(e, p.stats), static_cast<size_t>(B) * U_max * 4 * 4, cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaStreamSynchronize(s));
  if (spot) RS_TRY(spot_collect(e, B, *spot, s));
  return RS_OK;
}

}  // namespace

extern "C" {

int rs_transcribe_device(rs_engine* e, const float* wav, const int32_t* len, int B, int L_max, int32_t* tokens,
                         int32_t* frames, int32_t* n_tok, int U_max, void* stream) {
  return transcribe_device(e, "rs_transcribe_device", wav, false, len, B, L_max, tokens, frames, n_tok, U_max, nullptr, 0.f, static_cast<cudaStream_t>(stream));
}

int rs_transcribe_device_pcm16(rs_engine* e, const int16_t* wav, const int32_t* len, int B, int L_max, int32_t* tokens,
                               int32_t* frames, int32_t* n_tok, int U_max, void* stream) {
  return transcribe_device(e, "rs_transcribe_device_pcm16", wav, true, len, B, L_max, tokens, frames, n_tok, U_max, nullptr, 0.f,
                           static_cast<cudaStream_t>(stream));
}

int rs_transcribe_device_confidence(rs_engine* e, const void* wav, int wav_is_pcm16, const int32_t* len, int B, int L_max, int32_t* tokens,
                                    int32_t* frames, int32_t* n_tok, int U_max, float alpha, float* stats, void* stream) {
  if (!stats || !alpha_ok(alpha)) return fail(e, RS_ERR_INVALID_ARG, "rs_transcribe_device_confidence: bad arguments (stats must be set, alpha > 0 and finite)");
  return transcribe_device(e, "rs_transcribe_device_confidence", wav, wav_is_pcm16 != 0, len, B, L_max, tokens, frames, n_tok, U_max, stats, alpha,
                           static_cast<cudaStream_t>(stream));
}

int rs_transcribe_batch(rs_engine* e, const float* wav_host, const int32_t* len_host, int B, int L_max,
                        int32_t* tokens_host, int32_t* frames_host, int32_t* n_tok_host, int U_max, void* stream) {
  return transcribe_batch(e, "rs_transcribe_batch", wav_host, false, len_host, B, L_max, tokens_host, frames_host, n_tok_host, U_max,
                          nullptr, 0.f, static_cast<cudaStream_t>(stream));
}

int rs_transcribe_batch_pcm16(rs_engine* e, const int16_t* wav_host, const int32_t* len_host, int B, int L_max,
                              int32_t* tokens_host, int32_t* frames_host, int32_t* n_tok_host, int U_max, void* stream) {
  return transcribe_batch(e, "rs_transcribe_batch_pcm16", wav_host, true, len_host, B, L_max, tokens_host, frames_host, n_tok_host, U_max,
                          nullptr, 0.f, static_cast<cudaStream_t>(stream));
}

int rs_transcribe_batch_confidence(rs_engine* e, const void* wav_host, int wav_is_pcm16, const int32_t* len_host, int B, int L_max,
                                   int32_t* tokens_host, int32_t* frames_host, int32_t* n_tok_host, int U_max, float alpha,
                                   float* stats_host, void* stream) {
  if (!stats_host || !alpha_ok(alpha)) return fail(e, RS_ERR_INVALID_ARG, "rs_transcribe_batch_confidence: bad arguments (stats must be set, alpha > 0 and finite)");
  return transcribe_batch(e, "rs_transcribe_batch_confidence", wav_host, wav_is_pcm16 != 0, len_host, B, L_max, tokens_host, frames_host, n_tok_host,
                          U_max, stats_host, alpha, static_cast<cudaStream_t>(stream));
}

int rs_stream_step(rs_engine* e, const void* wav_host, int wav_is_pcm16, const int32_t* len_host, const int32_t* dec_begin_host,
                   const int32_t* dec_end_host, const int32_t* slot_host, void* states, int B, int L_max, int32_t* tokens_host,
                   int32_t* frames_host, int32_t* n_tok_host, int U_max, float alpha, float* stats_host, void* stream) {
  const char* fn = "rs_stream_step";
  if (!e || !dec_begin_host || !dec_end_host || !slot_host || !states || !len_host || B <= 0 || (stats_host && !alpha_ok(alpha)))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments (dec_begin, dec_end, slot, len and states must be set; with stats, alpha > 0 and finite)", fn);
  if (reinterpret_cast<uintptr_t>(states) & 15u) return fail(e, RS_ERR_INVALID_ARG, "%s: states must be 16-byte aligned", fn);
  std::vector<int32_t> seen(slot_host, slot_host + B);
  std::sort(seen.begin(), seen.end());
  if (seen[0] < 0 || std::adjacent_find(seen.begin(), seen.end()) != seen.end())
    return fail(e, RS_ERR_INVALID_ARG, "%s: slots must be distinct and >= 0", fn);
  for (int b = 0; b < B; ++b) {
    const int n = len_host[b] < 0 || len_host[b] > L_max ? -1 : rs_enc_valid(e, len_host[b]);
    if (n < 0 || dec_begin_host[b] < 0 || dec_begin_host[b] > dec_end_host[b] || dec_end_host[b] > n)
      return fail(e, RS_ERR_INVALID_ARG, "%s: row %d: need 0 <= dec_begin (%d) <= dec_end (%d) <= rs_enc_valid(len = %d) = %d and len <= L_max",
                  fn, b, dec_begin_host[b], dec_end_host[b], len_host[b], n);
  }
  const Resume rs{dec_begin_host, dec_end_host, slot_host, states};
  return transcribe_batch(e, fn, wav_host, wav_is_pcm16 != 0, len_host, B, L_max, tokens_host, frames_host, n_tok_host, U_max,
                          stats_host, alpha, static_cast<cudaStream_t>(stream), &rs);
}

int rs_set_spot_keywords(rs_engine* e, const int32_t* labels_host, const int32_t* label_len_host, int n_kw, int U_max, float threshold,
                         int delay_frames, int chunk_frames, void* stream) {
  const char* fn = "rs_set_spot_keywords";
  if (e == nullptr) return RS_ERR_INVALID_ARG;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n_kw == 0) {
    if (e->spot.mem) {                       // a call still queued may read the old set
      RS_CUDA(e, cudaSetDevice(e->device));
      RS_CUDA(e, cudaDeviceSynchronize());
      cudaFree(e->spot.mem);
    }
    e->spot = {};
    return RS_OK;
  }
  if (n_kw < 0 || !labels_host || !label_len_host || U_max < 1 || U_max > rs::kSpotMaxLabels)
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments (n_kw >= 0, labels and lengths set, U_max=%d in [1, %d])", fn, U_max, rs::kSpotMaxLabels);
  if (std::isnan(threshold) || threshold == INFINITY) return fail(e, RS_ERR_INVALID_ARG, "%s: threshold must be finite or -inf", fn);
  if (delay_frames < 0 || chunk_frames < 1) return fail(e, RS_ERR_INVALID_ARG, "%s: delay_frames=%d must be >= 0 and chunk_frames=%d >= 1", fn, delay_frames, chunk_frames);
  const int64_t ring = static_cast<int64_t>(delay_frames) + chunk_frames;
  if (ring > 227 * 1024 / 16 || rs::spot_pick_stream_smem(static_cast<int>(ring)) > 227 * 1024)
    return fail(e, RS_ERR_INVALID_ARG, "%s: a ring of delay + chunk = %lld entries does not fit the pick kernel's shared memory (at most %d)", fn,
                static_cast<long long>(ring), 227 * 1024 / 16);
  if (static_cast<int64_t>(n_kw) * ring > INT32_MAX / 64)
    return fail(e, RS_ERR_INVALID_ARG, "%s: n_kw x (delay + chunk) = %lld pending entries per stream exceed the hit list of one call (at most %d)", fn,
                static_cast<long long>(n_kw) * ring, INT32_MAX / 64);
  const rs_model_config& c = e->cfg;
  for (int k = 0; k < n_kw; ++k) {
    if (label_len_host[k] < 1 || label_len_host[k] > U_max)
      return fail(e, RS_ERR_INVALID_ARG, "%s: keyword %d: length %d outside [1, %d]", fn, k, label_len_host[k], U_max);
    for (int u = 0; u < label_len_host[k]; ++u) {
      const int y = labels_host[static_cast<size_t>(k) * U_max + u];
      if (y < 0 || y >= c.vocab_size) return fail(e, RS_ERR_INVALID_ARG, "%s: keyword %d: label %d = %d outside [0, %d)", fn, k, u, y, c.vocab_size);
    }
  }
  char msg[256] = "";
  if (!rs::align_supported(c.joint_hidden, c.pred_hidden, c.vocab_size, U_max, msg)) return fail(e, RS_ERR_UNSUPPORTED, "%s: %s", fn, msg);
  RS_CUDA(e, cudaSetDevice(e->device));
  const int U1 = U_max + 1, Hj = c.joint_hidden, Hp = c.pred_hidden;
  rs::Arena a;
  const size_t o_lab = a.take(static_cast<size_t>(n_kw) * U_max * 4), o_len = a.take(static_cast<size_t>(n_kw) * 4);
  const size_t o_h = a.take(static_cast<size_t>(n_kw) * U1 * Hp * 4), o_c = a.take(static_cast<size_t>(n_kw) * Hp * 4);
  const size_t o_pp = a.take(static_cast<size_t>(n_kw) * U1 * Hj * 4);
  // the new set is built next to the old one, so a failure below leaves the installed set as it was
  void* mem = nullptr;
  if (cudaMalloc(&mem, a.off) != cudaSuccess) {
    cudaGetLastError();
    return fail(e, RS_ERR_WORKSPACE, "%s: cannot allocate %zu bytes for %d keywords (the installed set is kept)", fn, a.off, n_kw);
  }
  char* m = static_cast<char*>(mem);
  rs::AlignArgs g{};
  g.labels = reinterpret_cast<int32_t*>(m + o_lab); g.label_len = reinterpret_cast<int32_t*>(m + o_len);
  g.w_lstm = e->dec.lstm_w; g.gate_tab = e->dec.gate_tab; g.w_pred = e->dec.pred_w; g.b_pred = e->dec.pred_b;
  g.B = n_kw; g.U_max = U_max; g.Hj = Hj; g.Hp = Hp; g.V = c.vocab_size;
  g.h = reinterpret_cast<float*>(m + o_h); g.c = reinterpret_cast<float*>(m + o_c); g.pred_proj = reinterpret_cast<float*>(m + o_pp);
  const auto predictor = [&]() -> int {        // the teacher-forced predictor of every keyword, once, as rs_rnnt_spot runs it per call
    RS_CUDA(e, cudaMemcpyAsync(m + o_lab, labels_host, static_cast<size_t>(n_kw) * U_max * 4, cudaMemcpyHostToDevice, s));
    RS_CUDA(e, cudaMemcpyAsync(m + o_len, label_len_host, static_cast<size_t>(n_kw) * 4, cudaMemcpyHostToDevice, s));
    for (int u = 0; u <= U_max; ++u) RS_LAUNCH(e, s, 1, rs::launch_align_lstm_step(g, u, s));
    RS_LAUNCH(e, s, 1, rs::launch_align_pred_proj(g, s));
    RS_CUDA(e, cudaStreamSynchronize(s));
    return RS_OK;
  };
  const int r = predictor();
  if (r != RS_OK) {
    cudaStreamSynchronize(s);
    cudaFree(mem);
    return r;
  }
  if (e->spot.mem) {
    RS_CUDA(e, cudaDeviceSynchronize());     // a call still queued may read the old set
    cudaFree(e->spot.mem);
  }
  e->spot = {};
  e->spot.mem = mem;
  e->spot.n_kw = n_kw; e->spot.U_max = U_max; e->spot.delay = delay_frames; e->spot.chunk = chunk_frames;
  e->spot.ring_cap = static_cast<int>(ring); e->spot.threshold = threshold;
  e->spot.labels = g.labels; e->spot.label_len = g.label_len; e->spot.pred_proj = g.pred_proj;
  return RS_OK;
}

size_t rs_spot_state_bytes(const rs_engine* e) {
  return e && e->spot.n_kw > 0 ? rs::spot_record(e->spot.U_max, e->spot.ring_cap).total : 0;
}

int rs_spot_max_hits(const rs_engine* e, int B) { return e && e->spot.n_kw > 0 && B > 0 ? spot_capacity(e, B) : 0; }

int rs_rnnt_spot_resume(rs_engine* e, const float* enc_dev, const int32_t* dec_begin_dev, const int32_t* dec_end_dev, const int32_t* slot_dev,
                        const int32_t* last_dev, void* records_dev, int n_slots, int B, int T_max, int max_out, int32_t* hit_meta_host,
                        float* hit_val_host, int32_t* hit_frames_host, float* hit_token_lp_host, int32_t* n_hits_host, float* E_dev,
                        int32_t* S_dev, int32_t* sigma_dev, void* stream) {
  const char* fn = "rs_rnnt_spot_resume";
  if (!e || !enc_dev || !dec_begin_dev || !dec_end_dev || !slot_dev || !last_dev || B <= 0 || T_max <= 0)
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments", fn);
  RS_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<int32_t> h(static_cast<size_t>(4) * B);
  const int32_t* src[4] = {dec_begin_dev, dec_end_dev, slot_dev, last_dev};
  for (int i = 0; i < 4; ++i) RS_CUDA(e, cudaMemcpyAsync(h.data() + i * B, src[i], static_cast<size_t>(B) * 4, cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaStreamSynchronize(s));
  const SpotCall c{h.data(), h.data() + B, h.data() + 2 * B, h.data() + 3 * B, records_dev, n_slots, max_out, hit_meta_host, hit_val_host,
                   hit_frames_host, hit_token_lp_host, n_hits_host, E_dev, S_dev, sigma_dev};
  RS_TRY(check_spot_call(e, fn, B, T_max, c));
  const rs_model_config& cfg = e->cfg;
  const size_t M = static_cast<size_t>(B) * T_max;
  rs::Arena a;
  const size_t o_xn = a.take(M * cfg.d_model * 2), o_encp = a.take(M * cfg.joint_hidden * 4), o_args = a.take(static_cast<size_t>(4) * B * 4);
  RS_TRY(grow_align_ws(e, fn, a.off, s));
  char* ws = static_cast<char*>(e->align_ws);
  int32_t* args = reinterpret_cast<int32_t*>(ws + o_args);
  for (int i = 0; i < 4; ++i) RS_CUDA(e, cudaMemcpyAsync(args + i * B, src[i], static_cast<size_t>(B) * 4, cudaMemcpyDeviceToDevice, s));
  // joint.enc over every frame, as in the greedy path
  RS_LAUNCH(e, s, 1, rs::launch_f32_to_bf16(enc_dev, ws + o_xn, static_cast<int64_t>(M) * cfg.d_model, s));
  RS_TRY(gemm(e, {ws + o_xn, e->dec.enc_w, e->dec.enc_b, nullptr, ws + o_encp, static_cast<int>(M), cfg.joint_hidden, cfg.d_model, RS_EPI_BIAS_F32, 1.f}, s));
  RS_TRY(spot_enqueue(e, fn, reinterpret_cast<float*>(ws + o_encp), T_max, B, c, args, s));
  return spot_collect(e, B, c, s);
}

int rs_stream_step_spot(rs_engine* e, const void* wav_host, int wav_is_pcm16, const int32_t* len_host, const int32_t* dec_begin_host,
                        const int32_t* dec_end_host, const int32_t* slot_host, void* states, int B, int L_max, int32_t* tokens_host,
                        int32_t* frames_host, int32_t* n_tok_host, int U_max, float alpha, float* stats_host, const int32_t* last_host,
                        void* spot_records_dev, int n_slots, int max_out, int32_t* hit_meta_host, float* hit_val_host,
                        int32_t* hit_frames_host, float* hit_token_lp_host, int32_t* n_hits_host, void* stream) {
  const char* fn = "rs_stream_step_spot";
  if (!e || !dec_begin_host || !dec_end_host || !slot_host || !states || !len_host || !last_host || B <= 0 || (stats_host && !alpha_ok(alpha)))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments (dec_begin, dec_end, slot, last, len and states must be set; with stats, alpha > 0 and finite)", fn);
  if (reinterpret_cast<uintptr_t>(states) & 15u) return fail(e, RS_ERR_INVALID_ARG, "%s: states must be 16-byte aligned", fn);
  for (int b = 0; b < B; ++b) {
    const int n = len_host[b] < 0 || len_host[b] > L_max ? -1 : rs_enc_valid(e, len_host[b]);
    if (n < 0 || dec_begin_host[b] < 0 || dec_begin_host[b] > dec_end_host[b] || dec_end_host[b] > n)
      return fail(e, RS_ERR_INVALID_ARG, "%s: row %d: need 0 <= dec_begin (%d) <= dec_end (%d) <= rs_enc_valid(len = %d) = %d and len <= L_max",
                  fn, b, dec_begin_host[b], dec_end_host[b], len_host[b], n);
  }
  const SpotCall c{dec_begin_host, dec_end_host, slot_host, last_host, spot_records_dev, n_slots, max_out, hit_meta_host, hit_val_host,
                   hit_frames_host, hit_token_lp_host, n_hits_host, nullptr, nullptr, nullptr};
  RS_TRY(check_spot_call(e, fn, B, INT32_MAX, c));   // also: the slots are distinct and >= 0, as rs_stream_step requires
  const Resume rs{dec_begin_host, dec_end_host, slot_host, states};
  return transcribe_batch(e, fn, wav_host, wav_is_pcm16 != 0, len_host, B, L_max, tokens_host, frames_host, n_tok_host, U_max,
                          stats_host, alpha, static_cast<cudaStream_t>(stream), &rs, &c);
}

}  // extern "C"

namespace {

// ALSD beam search over encoder outputs (decode_alsd.cu; semantics: oracle/alsd_restated.py).  Synchronises: the host checks every
// 32 steps whether every utterance's search has ended.  The search keeps the n_best best finished hypotheses and writes them
// all; rs_rnnt_alsd and the trace seam run it with n_best = 1 and without the per-utterance list sizes (count == nullptr).
// tr set: the trace seam (rs_rnnt_alsd_trace), which copies the state of every step out after the beam update; rs_rnnt_alsd
// passes nullptr, so the two run the same launches.
int rnnt_alsd(rs_engine* e, const char* fn, const float* enc, const int32_t* enc_len, int B, int T_max, int beam, double u_max_ratio,
              int score_norm, int recombine_returns_input, int n_best, int32_t* y_dev, int32_t* step_dev, int32_t* n_dev, double* score_dev,
              int32_t* count_dev, int32_t* pool_dev, int32_t* from_final_dev, int U_cap, const rs_alsd_trace* tr, cudaStream_t s) {
  if (!e || !enc || !enc_len || !y_dev || !step_dev || !n_dev || !score_dev || B <= 0 || T_max <= 0 || U_cap <= 0 || beam < 1 || beam > 8 ||
      !(u_max_ratio >= 0.0) || n_best < 1 || n_best > RS_MAX_NBEST || (count_dev != nullptr) != (pool_dev != nullptr) ||
      (count_dev != nullptr) != (from_final_dev != nullptr))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments (beam must be 1..8, n_best 1..%d)", fn, RS_MAX_NBEST);
  const int total_steps = T_max + static_cast<int>(u_max_ratio * static_cast<double>(T_max));
  const int max_nodes = 1 + beam * (total_steps + 1);
  if (tr && (tr->max_steps < 0 || tr->node_pitch < max_nodes || !tr->n_hyp || !tr->beam_score || !tr->beam_u || !tr->beam_node || !tr->row_t ||
             !tr->cand_logp || !tr->cand_tok || !tr->has_final || !tr->final_key || !tr->final_score || !tr->node_parent ||
             !tr->node_tok || !tr->node_step))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad trace buffers (every pointer set, max_steps >= 0, node_pitch >= %d)", fn, max_nodes);
  if (e->alsd.out_w3 == nullptr)
    return fail(e, RS_ERR_UNSUPPORTED, "%s: the engine was created without the beam-search weight tensors (alsd.*)", fn);
  RS_CUDA(e, cudaSetDevice(e->device));
  Nvtx range("rs::rnnt_alsd");
  const rs_model_config& c = e->cfg;
  const int Hj = c.joint_hidden, Hp = c.pred_hidden, d = c.d_model, V = c.vocab_size, blank = c.vocab_size, n_pad = e->alsd.n_pad;
  const int M = B * T_max, R = B * beam;
  // ---- workspace: scratch, then the search state, laid out once to size it and once more to bind it
  rs::Arena a;
  const size_t o_xn = a.take(static_cast<size_t>(M) * d * 2), o_encp = a.take(static_cast<size_t>(M) * Hj * 4);
  const size_t plane_cols = static_cast<size_t>(3 * Hj > 6 * Hp ? 3 * Hj : 6 * Hp);
  const size_t o_planes = a.take(static_cast<size_t>(R) * plane_cols * 2), o_logits = a.take(static_cast<size_t>(R) * n_pad * 4);
  const size_t o_gates = a.take(static_cast<size_t>(R) * 4 * Hp * 4);
  const size_t o_state = a.off;
  rs::AlsdState st{};
  rs::Arena state_plan = a;
  rs::alsd_layout_state(st, state_plan, nullptr, B, beam, Hp, Hj, max_nodes, score_norm != 0, n_best);
  const size_t need_bytes = state_plan.off;
  if (need_bytes > e->alsd_ws_bytes) {
    RS_CUDA(e, cudaStreamSynchronize(s));
    cudaFree(e->alsd_ws); e->alsd_ws = nullptr; e->alsd_ws_bytes = 0;
    RS_CUDA(e, cudaMalloc(&e->alsd_ws, need_bytes));
    e->alsd_ws_bytes = need_bytes;
  }
  if (e->alsd_done_host == nullptr) RS_CUDA(e, cudaMallocHost(reinterpret_cast<void**>(&e->alsd_done_host), sizeof(int)));
  char* ws = static_cast<char*>(e->alsd_ws);
  void* xn = ws + o_xn; float* encp = reinterpret_cast<float*>(ws + o_encp); void* planes = ws + o_planes;
  float* logits = reinterpret_cast<float*>(ws + o_logits); float* gates = reinterpret_cast<float*>(ws + o_gates);
  RS_CUDA(e, cudaMemsetAsync(ws + o_state, 0, need_bytes - o_state, s));
  rs::alsd_layout_state(st, a, ws, B, beam, Hp, Hj, max_nodes, score_norm != 0, n_best);
  // ---- joint.enc over every frame (as in the greedy path)
  RS_LAUNCH(e, s, 1, rs::launch_f32_to_bf16(enc, xn, static_cast<int64_t>(M) * d, s));
  RS_TRY(gemm(e, {xn, e->dec.enc_w, e->dec.enc_b, nullptr, encp, M, Hj, d, RS_EPI_BIAS_F32, 1.f}, s));
  // predictor of the beam being built (also the start: [blank] from the zero state), which then becomes the current one
  auto predictor = [&]() -> int {
    RS_LAUNCH(e, s, 1, rs::alsd_launch_lstm_in(st, B, e->dec.embed, Hp, planes, s));
    RS_TRY(gemm(e, {planes, e->alsd.lstm_w3, e->dec.lstm_b, nullptr, gates, R, 4 * Hp, 6 * Hp, RS_EPI_BIAS_F32, 1.f}, s));
    RS_LAUNCH(e, s, 1, rs::alsd_launch_cell(st, B, gates, Hp, planes, s));
    RS_TRY(gemm(e, {planes, e->alsd.pred_w3, e->dec.pred_b, nullptr, st.nx.pp, R, Hj, 3 * Hp, RS_EPI_BIAS_F32, 1.f}, s));
    std::swap(st.cur, st.nx);
    return RS_OK;
  };
  RS_LAUNCH(e, s, 1, rs::alsd_launch_init(st, B, blank, s));
  RS_TRY(predictor());
  for (int step = 0; step <= total_steps; ++step) {
    RS_LAUNCH(e, s, 1, rs::alsd_launch_rows(st, B, encp, enc_len, T_max, Hj, step, planes, s));
    RS_TRY(gemm(e, {planes, e->alsd.out_w3, e->alsd.out_b, nullptr, logits, R, n_pad, 3 * Hj, RS_EPI_BIAS_F32, 1.f}, s));
    RS_LAUNCH(e, s, 1, rs::alsd_launch_reduce(st, B, logits, n_pad, V, s));
    RS_LAUNCH(e, s, 1, rs::alsd_launch_select(st, B, enc_len, step, u_max_ratio, recombine_returns_input != 0, s));
    if (tr && step < tr->max_steps) {                   // the new beam is the `nx` half until the predictor pass swaps it in
      const size_t o = static_cast<size_t>(step) * R, ob = static_cast<size_t>(step) * B;
      auto copy = [&](void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s); };
      RS_CUDA(e, copy(tr->n_hyp + ob, st.nx.n_hyp, B * 4));
      RS_CUDA(e, copy(tr->beam_score + o, st.nx.score, R * 8));
      RS_CUDA(e, copy(tr->beam_u + o, st.nx.u, R * 4));
      RS_CUDA(e, copy(tr->beam_node + o, st.nx.node, R * 4));
      RS_CUDA(e, copy(tr->row_t + o, st.row_t, R * 4));
      RS_CUDA(e, copy(tr->cand_logp + o * 9, st.cand_logp, R * 9 * 4));
      RS_CUDA(e, copy(tr->cand_tok + o * 8, st.cand_tok, R * 8 * 4));
      // entry 0 of each utterance's finished list (n_best = 1 here, so fin_count is 0 or 1)
      RS_CUDA(e, copy(tr->has_final + ob, st.fin_count, B * 4));
      const size_t fp = static_cast<size_t>(n_best) * 8;
      RS_CUDA(e, cudaMemcpy2DAsync(tr->final_key + ob, 8, st.fin_key, fp, 8, B, cudaMemcpyDeviceToDevice, s));
      RS_CUDA(e, cudaMemcpy2DAsync(tr->final_score + ob, 8, st.fin_score, fp, 8, B, cudaMemcpyDeviceToDevice, s));
    }
    RS_TRY(predictor());
    if ((step & 31) == 31) {
      RS_CUDA(e, cudaMemcpyAsync(e->alsd_done_host, st.n_done, sizeof(int), cudaMemcpyDeviceToHost, s));
      RS_CUDA(e, cudaStreamSynchronize(s));
      if (*e->alsd_done_host >= B) break;
    }
  }
  RS_LAUNCH(e, s, 1, rs::alsd_launch_output(st, B, blank, y_dev, step_dev, n_dev, score_dev, count_dev, pool_dev, from_final_dev, U_cap, s));
  if (tr) {
    const size_t dp = static_cast<size_t>(tr->node_pitch) * 4, sp = static_cast<size_t>(max_nodes) * 4;
    RS_CUDA(e, cudaMemcpy2DAsync(tr->node_parent, dp, st.node_parent, sp, sp, B, cudaMemcpyDeviceToDevice, s));
    RS_CUDA(e, cudaMemcpy2DAsync(tr->node_tok, dp, st.node_tok, sp, sp, B, cudaMemcpyDeviceToDevice, s));
    RS_CUDA(e, cudaMemcpy2DAsync(tr->node_step, dp, st.node_step, sp, sp, B, cudaMemcpyDeviceToDevice, s));
  }
  RS_CUDA(e, cudaStreamSynchronize(s));
  return RS_OK;
}

}  // namespace

extern "C" {

int rs_rnnt_alsd(rs_engine* e, const float* enc, const int32_t* enc_len, int B, int T_max, int beam, double u_max_ratio, int score_norm,
                 int recombine_returns_input, int32_t* y_dev, int32_t* step_dev, int32_t* n_dev, double* score_dev, int U_cap, void* stream) {
  return rnnt_alsd(e, "rs_rnnt_alsd", enc, enc_len, B, T_max, beam, u_max_ratio, score_norm, recombine_returns_input, 1, y_dev, step_dev, n_dev,
                   score_dev, nullptr, nullptr, nullptr, U_cap, nullptr, static_cast<cudaStream_t>(stream));
}

int rs_rnnt_alsd_nbest(rs_engine* e, const float* enc, const int32_t* enc_len, int B, int T_max, int beam, double u_max_ratio, int score_norm,
                       int recombine_returns_input, int n_best, int32_t* y_dev, int32_t* step_dev, int32_t* n_dev, double* score_dev,
                       int32_t* count_dev, int32_t* pool_dev, int32_t* from_final_dev, int U_cap, void* stream) {
  if (!count_dev || !pool_dev || !from_final_dev)
    return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_alsd_nbest: bad arguments (count, pool and from_final are required)");
  return rnnt_alsd(e, "rs_rnnt_alsd_nbest", enc, enc_len, B, T_max, beam, u_max_ratio, score_norm, recombine_returns_input, n_best, y_dev,
                   step_dev, n_dev, score_dev, count_dev, pool_dev, from_final_dev, U_cap, nullptr, static_cast<cudaStream_t>(stream));
}

int rs_rnnt_alsd_trace(rs_engine* e, const float* enc, const int32_t* enc_len, int B, int T_max, int beam, double u_max_ratio, int score_norm,
                       int recombine_returns_input, int32_t* y_dev, int32_t* step_dev, int32_t* n_dev, double* score_dev, int U_cap,
                       const rs_alsd_trace* trace, void* stream) {
  if (trace == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_alsd_trace: bad arguments (no trace)");
  return rnnt_alsd(e, "rs_rnnt_alsd_trace", enc, enc_len, B, T_max, beam, u_max_ratio, score_norm, recombine_returns_input, 1, y_dev, step_dev,
                   n_dev, score_dev, nullptr, nullptr, nullptr, U_cap, trace, static_cast<cudaStream_t>(stream));
}

// MAES beam search over encoder outputs (decode_maes.cu; semantics: oracle/maes_restated.py).  Exactly T_max frames; each
// expansion round's live rows are compacted on the device and their count read back through a pinned word, so every GEMM of the
// round runs over the live rows only.
int rs_rnnt_maes(rs_engine* e, const float* enc, const int32_t* enc_len, int B, int T_max, const rs_maes_params* p, int n_best,
                 int32_t* y_dev, int32_t* frames_dev, int32_t* n_dev, double* score_dev, int32_t* count_dev, int U_cap, void* stream) {
  static const char* fn = "rs_rnnt_maes";
  if (!e || !enc || !enc_len || !p || !y_dev || !frames_dev || !n_dev || !score_dev || !count_dev || B <= 0 || T_max <= 0 || U_cap <= 0)
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments", fn);
  const int V = e->cfg.vocab_size;
  const int K = std::min(p->beam, V), S = p->num_steps, alpha = p->prefix_alpha, beta = p->expansion_beta;
  if (p->beam < 1 || p->beam > 8 || S < 2 || S > rs::kMaesMaxSteps || alpha < 0 || alpha > 4 || beta < 0 || beta > 4 ||
      !(p->expansion_gamma > 0.f) || !std::isfinite(p->expansion_gamma) || K + beta > V || n_best < 1 || n_best > K)
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad parameters (beam 1..8, num_steps 2..4, prefix_alpha 0..4, expansion_beta 0..4, "
                "expansion_gamma > 0, beam + expansion_beta <= vocab_size, n_best 1..beam)", fn);
  const int C = K + beta;
  int64_t W = K;
  for (int n = 0; n < S; ++n) W *= C;
  if (W > RS_MAX_MAES_ROWS)
    return fail(e, RS_ERR_UNSUPPORTED, "%s: beam * (beam + expansion_beta)^num_steps = %lld expansion rows per utterance exceed %d", fn,
                static_cast<long long>(W), RS_MAX_MAES_ROWS);
  if (e->alsd.out_w3 == nullptr)
    return fail(e, RS_ERR_UNSUPPORTED, "%s: the engine was created without the beam-search weight tensors (alsd.*)", fn);
  RS_CUDA(e, cudaSetDevice(e->device));
  Nvtx range("rs::rnnt_maes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const rs_model_config& c = e->cfg;
  const int Hj = c.joint_hidden, Hp = c.pred_hidden, d = c.d_model, blank = V, n_pad = e->alsd.n_pad;
  const int M_enc = B * T_max, R = B * K, P = std::max(alpha, 1);
  const int max_nodes = 1 + T_max * K * S;
  const int rows_max = std::max(R * P, B * static_cast<int>(W));
  // ---- workspace: scratch, then the search state, laid out once to size it and once more to bind it
  rs::Arena a;
  const size_t o_xn = a.take(static_cast<size_t>(M_enc) * d * 2), o_encp = a.take(static_cast<size_t>(M_enc) * Hj * 4);
  const size_t plane_cols = static_cast<size_t>(3 * Hj > 6 * Hp ? 3 * Hj : 6 * Hp);
  const size_t o_planes = a.take(static_cast<size_t>(rows_max) * plane_cols * 2), o_logits = a.take(static_cast<size_t>(rows_max) * n_pad * 4);
  const size_t o_gates = a.take(static_cast<size_t>(rows_max) * 4 * Hp * 4);
  const size_t o_state = a.off;
  rs::MaesState st{};
  rs::Arena state_plan = a;
  rs::maes_layout_state(st, state_plan, nullptr, B, K, C, S, P, Hp, Hj, max_nodes);
  const size_t need_bytes = state_plan.off;
  if (need_bytes > e->alsd_ws_bytes) {
    RS_CUDA(e, cudaStreamSynchronize(s));
    cudaFree(e->alsd_ws); e->alsd_ws = nullptr; e->alsd_ws_bytes = 0;
    if (cudaMalloc(&e->alsd_ws, need_bytes) != cudaSuccess) {
      cudaGetLastError();
      e->alsd_ws = nullptr;
      return fail(e, RS_ERR_WORKSPACE, "%s: could not allocate %zu bytes of search workspace", fn, need_bytes);
    }
    e->alsd_ws_bytes = need_bytes;
  }
  if (e->alsd_done_host == nullptr) RS_CUDA(e, cudaMallocHost(reinterpret_cast<void**>(&e->alsd_done_host), sizeof(int)));
  char* ws = static_cast<char*>(e->alsd_ws);
  void* xn = ws + o_xn; float* encp = reinterpret_cast<float*>(ws + o_encp); void* planes = ws + o_planes;
  float* logits = reinterpret_cast<float*>(ws + o_logits); float* gates = reinterpret_cast<float*>(ws + o_gates);
  RS_CUDA(e, cudaMemsetAsync(ws + o_state, 0, need_bytes - o_state, s));
  rs::maes_layout_state(st, a, ws, B, K, C, S, P, Hp, Hj, max_nodes);
  st.alpha = alpha; st.gamma = static_cast<double>(p->expansion_gamma); st.score_norm = p->score_norm != 0; st.rri = p->recombine_returns_input != 0;
  rs::NgramLM lm = e->lm;
  // ---- joint.enc over every frame (as in the greedy path)
  RS_LAUNCH(e, s, 1, rs::launch_f32_to_bf16(enc, xn, static_cast<int64_t>(M_enc) * d, s));
  RS_TRY(gemm(e, {xn, e->dec.enc_w, e->dec.enc_b, nullptr, encp, M_enc, Hj, d, RS_EPI_BIAS_F32, 1.f}, s));
  // predictor of round n's M rows (h, c, then joint.pred into plane 0 of the rows' dec_out history)
  auto predictor = [&](int n, int M) -> int {
    RS_LAUNCH(e, s, 1, rs::maes_launch_lstm_in(st, n, M, e->dec.embed, Hp, Hj, blank, planes, s));
    RS_TRY(gemm(e, {planes, e->alsd.lstm_w3, e->dec.lstm_b, nullptr, gates, M, 4 * Hp, 6 * Hp, RS_EPI_BIAS_F32, 1.f}, s));
    RS_LAUNCH(e, s, 1, rs::maes_launch_cell(st, n, M, gates, Hp, planes, s));
    RS_TRY(gemm(e, {planes, e->alsd.pred_w3, e->dec.pred_b, nullptr, st.rows[n].pp, M, Hj, 3 * Hp, RS_EPI_BIAS_F32, 1.f}, s));
    return RS_OK;
  };
  auto joint = [&](int M) { return gemm(e, {planes, e->alsd.out_w3, e->alsd.out_b, nullptr, logits, M, n_pad, 3 * Hj, RS_EPI_BIAS_F32, 1.f}, s); };
  RS_LAUNCH(e, s, 1, rs::maes_launch_init(st, blank, lm.order != 0 ? lm.start_state : 0, s));
  RS_TRY(predictor(0, B));
  RS_LAUNCH(e, s, 1, rs::maes_launch_init_kept(st, Hp, Hj, s));
  int64_t live_rows = 0;
  for (int t = 0; t < T_max; ++t) {
    RS_CUDA(e, cudaMemsetAsync(st.m, 0, rs::kMaesMaxSteps * sizeof(int), s));
    RS_LAUNCH(e, s, 1, rs::maes_launch_prefix_rows(st, encp, enc_len, T_max, Hj, t, planes, s));
    RS_TRY(joint(R * P));
    RS_LAUNCH(e, s, 1, rs::maes_launch_reduce(st, -1, R * P, logits, n_pad, V, s));
    RS_LAUNCH(e, s, 1, rs::maes_launch_prefix(st, logits, n_pad, s));
    for (int n = 0; n < S; ++n) {
      RS_LAUNCH(e, s, 1, rs::maes_launch_expand(st, n, blank, lm, s));
      RS_CUDA(e, cudaMemcpyAsync(e->alsd_done_host, st.m + n, sizeof(int), cudaMemcpyDeviceToHost, s));
      RS_CUDA(e, cudaStreamSynchronize(s));
      const int M = *e->alsd_done_host;
      if (M == 0) break;                               // every utterance's frame ended in this round
      live_rows += M;
      RS_TRY(predictor(n, M));
      RS_LAUNCH(e, s, 1, rs::maes_launch_rows(st, n, M, encp, T_max, Hj, t, planes, s));
      RS_TRY(joint(M));
      RS_LAUNCH(e, s, 1, rs::maes_launch_reduce(st, n, M, logits, n_pad, V, s));
    }
    RS_LAUNCH(e, s, 1, rs::maes_launch_select(st, t, s));
    RS_LAUNCH(e, s, 1, rs::maes_launch_gather(st, Hp, Hj, s));
    std::swap(st.cur, st.nx);
  }
  RS_LAUNCH(e, s, 1, rs::maes_launch_output(st, n_best, blank, y_dev, frames_dev, n_dev, score_dev, count_dev, U_cap, s));
  RS_CUDA(e, cudaStreamSynchronize(s));
  e->maes_rows = live_rows;
  e->maes_frames = T_max;
  return RS_OK;
}

int rs_maes_last_rows(const rs_engine* e, int64_t* rows, int64_t* frames) {
  if (e == nullptr || rows == nullptr || frames == nullptr) return RS_ERR_INVALID_ARG;
  *rows = e->maes_rows;
  *frames = e->maes_frames;
  return RS_OK;
}

}  // extern "C"

namespace {

// The forced alignment's scratch holds at least `bytes` (growing it synchronises s).
int grow_align_ws(rs_engine* e, const char* fn, size_t bytes, cudaStream_t s) {
  if (bytes > e->align_ws_bytes) {
    RS_CUDA(e, cudaStreamSynchronize(s));
    cudaFree(e->align_ws); e->align_ws = nullptr; e->align_ws_bytes = 0;
    if (cudaMalloc(&e->align_ws, bytes) != cudaSuccess) {
      cudaGetLastError();
      return fail(e, RS_ERR_WORKSPACE, "%s: cannot allocate %zu bytes of alignment scratch (chunk long inputs)", fn, bytes);
    }
    e->align_ws_bytes = bytes;
  }
  return RS_OK;
}

// Forced alignment (align.cu; semantics: reazonspeech_b200/alignment.py).  lp_blank / lp_emit set: the lattice seam (the
// caller's buffers, no DP); otherwise the lattice lives in the scratch and the DP writes frames / token_lp / viterbi / loglik.
// seg set: the segment alignment (rnnt_segment_dp_kernel), which also writes seg and frame_lp.
int rnnt_align(rs_engine* e, const char* fn, const float* enc, const int32_t* enc_len, int B, int T_max, const int32_t* labels,
               const int32_t* label_len, int U_max, float* lp_blank, float* lp_emit, int32_t* frames, float* token_lp, float* viterbi,
               float* loglik, cudaStream_t s, int32_t* seg = nullptr, float* frame_lp = nullptr) {
  const bool seam = lp_blank != nullptr;
  if (!e || !enc || !enc_len || !labels || !label_len || B <= 0 || T_max <= 0 || U_max <= 0 ||
      (seam ? lp_emit == nullptr : (!frames || !token_lp || !viterbi || !loglik)) || (seg != nullptr && (seam || frame_lp == nullptr)))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments", fn);
  const rs_model_config& c = e->cfg;
  char msg[256] = "";
  if (!rs::align_supported(c.joint_hidden, c.pred_hidden, c.vocab_size, U_max, msg)) return fail(e, RS_ERR_UNSUPPORTED, "%s: %s", fn, msg);
  RS_CUDA(e, cudaSetDevice(e->device));
  Nvtx range("rs::rnnt_align");
  const int M = B * T_max, U1 = U_max + 1, Hj = c.joint_hidden, Hp = c.pred_hidden;
  const size_t cells = static_cast<size_t>(M) * U1;
  rs::Arena a;
  const size_t o_xn = a.take(static_cast<size_t>(M) * c.d_model * 2), o_encp = a.take(static_cast<size_t>(M) * Hj * 4);
  const size_t o_h = a.take(static_cast<size_t>(B) * U1 * Hp * 4), o_c = a.take(static_cast<size_t>(B) * Hp * 4);
  const size_t o_pp = a.take(static_cast<size_t>(B) * U1 * Hj * 4);
  size_t o_lpb = 0, o_lpe = 0, o_ch = 0;
  if (!seam) { o_lpb = a.take(cells * 4); o_lpe = a.take(cells * 4); o_ch = a.take(cells); }
  RS_TRY(grow_align_ws(e, fn, a.off, s));
  char* ws = static_cast<char*>(e->align_ws);
  rs::AlignArgs g{reinterpret_cast<float*>(ws + o_encp), enc_len, labels, label_len, e->dec.out_w, e->dec.out_b, e->dec.lstm_w,
                  e->dec.gate_tab, e->dec.pred_w, e->dec.pred_b, B, T_max, U_max, Hj, Hp, c.vocab_size,
                  reinterpret_cast<float*>(ws + o_h), reinterpret_cast<float*>(ws + o_c), reinterpret_cast<float*>(ws + o_pp),
                  seam ? lp_blank : reinterpret_cast<float*>(ws + o_lpb), seam ? lp_emit : reinterpret_cast<float*>(ws + o_lpe),
                  reinterpret_cast<uint8_t*>(ws + o_ch), frames, token_lp, viterbi, loglik, seg, frame_lp};
  // joint.enc over every frame, as in the greedy path
  RS_LAUNCH(e, s, 1, rs::launch_f32_to_bf16(enc, ws + o_xn, static_cast<int64_t>(M) * c.d_model, s));
  RS_TRY(gemm(e, {ws + o_xn, e->dec.enc_w, e->dec.enc_b, nullptr, ws + o_encp, M, Hj, c.d_model, RS_EPI_BIAS_F32, 1.f}, s));
  for (int u = 0; u <= U_max; ++u) RS_LAUNCH(e, s, 1, rs::launch_align_lstm_step(g, u, s));
  RS_LAUNCH(e, s, 1, rs::launch_align_pred_proj(g, s));
  {
    const int r = launch(e, s, "rnnt_lattice_kernel", 1, 0.0, [&] { return rs::launch_rnnt_lattice(g, s, msg); });
    if (r != RS_OK && msg[0] != '\0') return fail(e, r, "%s: %s", fn, msg);
    RS_TRY(r);
  }
  if (seg != nullptr) RS_LAUNCH(e, s, 1, rs::launch_rnnt_segment_dp(g, s));
  else if (!seam) RS_LAUNCH(e, s, 1, rs::launch_rnnt_align_dp(g, s));
  return RS_OK;
}

// Banded alignment (align.cu; semantics: reazonspeech_b200/alignment.py, "Banded alignment").  The lengths and labels are read
// back and checked with the host band before anything is launched; the host also lays out the banded storage (row (b, u) at
// off[b][u], the prefix sum of the band widths), finds every diagonal's extent and lists the lattice tiles that meet the band.
// lp_blank / lp_emit set: the lattice seam (the caller's banded buffers, no DP).
int rnnt_align_banded(rs_engine* e, const char* fn, const float* enc, const int32_t* enc_len, int B, int T_max, const int32_t* labels,
                      const int32_t* label_len, int U_max, const int32_t* band_lo, const int32_t* band_hi, float* lp_blank, float* lp_emit,
                      int32_t* frames, float* token_lp, float* viterbi, float* loglik, int32_t* edge, cudaStream_t s) {
  const bool seam = lp_blank != nullptr;
  if (!e || !enc || !enc_len || !labels || !label_len || !band_lo || !band_hi || B <= 0 || T_max <= 0 || U_max <= 0 ||
      (seam ? lp_emit == nullptr : (!frames || !token_lp || !viterbi || !loglik || !edge)))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments", fn);
  const rs_model_config& c = e->cfg;
  char msg[256] = "";
  if (!rs::align_supported(c.joint_hidden, c.pred_hidden, c.vocab_size, 1, msg)) return fail(e, RS_ERR_UNSUPPORTED, "%s: %s", fn, msg);
  RS_CUDA(e, cudaSetDevice(e->device));
  const int U1 = U_max + 1, Hj = c.joint_hidden, Hp = c.pred_hidden;
  std::vector<int32_t> T(B), U(B), y(static_cast<size_t>(B) * U_max);
  RS_CUDA(e, cudaMemcpyAsync(T.data(), enc_len, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaMemcpyAsync(U.data(), label_len, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaMemcpyAsync(y.data(), labels, y.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  RS_CUDA(e, cudaStreamSynchronize(s));
  std::vector<int64_t> off(static_cast<size_t>(B) * U1, 0);
  std::vector<int4> tiles;
  int64_t cells = 0;
  int pitch = 1, U_top = 0;
  for (int b = 0; b < B; ++b) {
    const int Tb = T[b], Ub = U[b];
    if (Tb < 1 || Tb > T_max || Ub < 0 || Ub > U_max)
      return fail(e, RS_ERR_INVALID_ARG, "%s: utterance %d: enc_len=%d outside [1, %d] or label_len=%d outside [0, %d]", fn, b, Tb, T_max, Ub, U_max);
    for (int u = 0; u < Ub; ++u) {
      const int k = y[static_cast<size_t>(b) * U_max + u];
      if (k < 0 || k >= c.vocab_size) return fail(e, RS_ERR_INVALID_ARG, "%s: utterance %d: label %d = %d outside [0, %d)", fn, b, u, k, c.vocab_size);
    }
    const int32_t* lo = band_lo + static_cast<size_t>(b) * U1;
    const int32_t* hi = band_hi + static_cast<size_t>(b) * U1;
    if (lo[0] != 0 || hi[Ub] != Tb)
      return fail(e, RS_ERR_INVALID_ARG, "%s: utterance %d: the band must start at frame 0 in row 0 (got %d) and end at enc_len=%d in row %d (got %d)",
                  fn, b, lo[0], Tb, Ub, hi[Ub]);
    for (int u = 0; u <= Ub; ++u) {
      if (lo[u] < 0 || lo[u] >= hi[u] || hi[u] > Tb)
        return fail(e, RS_ERR_INVALID_ARG, "%s: utterance %d row %d: band [%d, %d) is empty or outside [0, %d)", fn, b, u, lo[u], hi[u], Tb);
      if (u > 0 && (lo[u] < lo[u - 1] || hi[u] < hi[u - 1]))
        return fail(e, RS_ERR_INVALID_ARG, "%s: utterance %d row %d: band [%d, %d) decreases from row %d's [%d, %d)", fn, b, u, lo[u], hi[u], u - 1,
                    lo[u - 1], hi[u - 1]);
      if (u > 0 && lo[u] >= hi[u - 1])
        return fail(e, RS_ERR_INVALID_ARG, "%s: utterance %d: rows %d [%d, %d) and %d [%d, %d) do not overlap", fn, b, u - 1, lo[u - 1], hi[u - 1], u,
                    lo[u], hi[u]);
      off[static_cast<size_t>(b) * U1 + u] = cells;
      cells += hi[u] - lo[u];
    }
    for (int d = 0, u0 = 0, u1 = 0; d < Tb + Ub; ++d) {        // diagonal d meets the rows [u0, u1]
      while (u1 < Ub && u1 + 1 + lo[u1 + 1] <= d) ++u1;
      while (u0 + hi[u0] <= d) ++u0;
      pitch = std::max(pitch, u1 - u0 + 1);
    }
    for (int u0 = 0; u0 <= Ub; u0 += 8) {                       // rows [u0, u0 + 8) cover the frames [lo[u0], hi[last row])
      const int ul = std::min(u0 + 7, Ub);
      for (int t0 = lo[u0] / 16 * 16; t0 < hi[ul]; t0 += 16) tiles.push_back(make_int4(b, t0, u0, 0));
    }
    U_top = std::max(U_top, Ub);
  }
  if (tiles.size() > static_cast<size_t>(INT32_MAX)) return fail(e, RS_ERR_INVALID_ARG, "%s: %zu lattice tiles exceed one launch", fn, tiles.size());
  if (!seam && rs::band_dp_smem(pitch) > 227 * 1024)
    return fail(e, RS_ERR_UNSUPPORTED, "%s: a diagonal meets %d rows of the band, more than the DP's shared memory holds (%d)", fn, pitch,
                static_cast<int>(227 * 1024 / rs::band_dp_smem(1)));
  Nvtx range("rs::rnnt_align_banded");
  const size_t M = static_cast<size_t>(B) * T_max, rows = static_cast<size_t>(B) * U1;
  rs::Arena a;
  const size_t o_xn = a.take(M * c.d_model * 2), o_encp = a.take(M * Hj * 4);
  const size_t o_h = a.take(rows * Hp * 4), o_c = a.take(static_cast<size_t>(B) * Hp * 4), o_pp = a.take(rows * Hj * 4);
  const size_t o_lo = a.take(rows * 4), o_hi = a.take(rows * 4), o_off = a.take(rows * 8), o_tiles = a.take(tiles.size() * sizeof(int4));
  size_t o_lpb = 0, o_lpe = 0, o_ch = 0;
  if (!seam) { o_lpb = a.take(cells * 4); o_lpe = a.take(cells * 4); o_ch = a.take(cells); }
  RS_TRY(grow_align_ws(e, fn, a.off, s));
  char* ws = static_cast<char*>(e->align_ws);
  // pageable sources: each copy has read its source when it returns
  RS_CUDA(e, cudaMemcpyAsync(ws + o_lo, band_lo, rows * 4, cudaMemcpyHostToDevice, s));
  RS_CUDA(e, cudaMemcpyAsync(ws + o_hi, band_hi, rows * 4, cudaMemcpyHostToDevice, s));
  RS_CUDA(e, cudaMemcpyAsync(ws + o_off, off.data(), rows * 8, cudaMemcpyHostToDevice, s));
  RS_CUDA(e, cudaMemcpyAsync(ws + o_tiles, tiles.data(), tiles.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
  rs::AlignArgs g{};
  g.enc_proj = reinterpret_cast<float*>(ws + o_encp); g.enc_len = enc_len; g.labels = labels; g.label_len = label_len;
  g.w_out = e->dec.out_w; g.b_out = e->dec.out_b; g.w_lstm = e->dec.lstm_w; g.gate_tab = e->dec.gate_tab;
  g.w_pred = e->dec.pred_w; g.b_pred = e->dec.pred_b;
  g.B = B; g.T_max = T_max; g.U_max = U_max; g.Hj = Hj; g.Hp = Hp; g.V = c.vocab_size;
  g.h = reinterpret_cast<float*>(ws + o_h); g.c = reinterpret_cast<float*>(ws + o_c); g.pred_proj = reinterpret_cast<float*>(ws + o_pp);
  g.lp_blank = seam ? lp_blank : reinterpret_cast<float*>(ws + o_lpb); g.lp_emit = seam ? lp_emit : reinterpret_cast<float*>(ws + o_lpe);
  g.choice = reinterpret_cast<uint8_t*>(ws + o_ch);
  g.frames = frames; g.token_lp = token_lp; g.viterbi = viterbi; g.loglik = loglik;
  g.band_lo = reinterpret_cast<int32_t*>(ws + o_lo); g.band_hi = reinterpret_cast<int32_t*>(ws + o_hi);
  g.band_off = reinterpret_cast<int64_t*>(ws + o_off); g.band_tiles = reinterpret_cast<int4*>(ws + o_tiles);
  g.band_pitch = pitch; g.edge = edge;
  // joint.enc over every frame and the teacher-forced predictor, as in the forced alignment
  RS_LAUNCH(e, s, 1, rs::launch_f32_to_bf16(enc, ws + o_xn, static_cast<int64_t>(M) * c.d_model, s));
  RS_TRY(gemm(e, {ws + o_xn, e->dec.enc_w, e->dec.enc_b, nullptr, ws + o_encp, static_cast<int>(M), Hj, c.d_model, RS_EPI_BIAS_F32, 1.f}, s));
  for (int u = 0; u <= U_top; ++u) RS_LAUNCH(e, s, 1, rs::launch_align_lstm_step(g, u, s));
  RS_LAUNCH(e, s, 1, rs::launch_align_pred_proj(g, s));
  {
    const int n = static_cast<int>(tiles.size());
    const int r = launch(e, s, "rnnt_lattice_kernel<band>", 1, 0.0, [&] { return rs::launch_rnnt_lattice_band(g, n, s, msg); });
    if (r != RS_OK && msg[0] != '\0') return fail(e, r, "%s: %s", fn, msg);
    RS_TRY(r);
  }
  if (!seam) RS_LAUNCH(e, s, 1, rs::launch_rnnt_band_dp(g, s));
  return RS_OK;
}

// Keyword spotting (align.cu, spot.cu; semantics: reazonspeech_b200/keywords.py): joint.enc once per recording, the
// predictor once per keyword, then the lattice, the recursion and the hits of every (recording, keyword) pair.
int rnnt_spot(rs_engine* e, const float* enc, const int32_t* enc_len, int n_rec, int T_max, const int32_t* labels,
              const int32_t* label_len, int n_kw, int U_max, float threshold, int max_hits, int32_t* span, float* score, float* conf,
              int32_t* frames, float* token_lp, int32_t* count, float* E_out, int32_t* S_out, cudaStream_t s,
              float* lp_blank = nullptr, float* lp_emit = nullptr) {
  const bool seam = lp_blank != nullptr;
  const char* fn = seam ? "rs_rnnt_spot_lattice" : "rs_rnnt_spot";
  if (!e || !enc || !enc_len || !labels || !label_len ||
      (seam ? lp_emit == nullptr : (!span || !score || !conf || !frames || !token_lp || !count)))
    return fail(e, RS_ERR_INVALID_ARG, "%s: bad arguments", fn);
  if (n_rec < 1 || T_max < 1 || n_kw < 1 || U_max < 1 || U_max > rs::kSpotMaxLabels)
    return fail(e, RS_ERR_INVALID_ARG, "%s: n_rec=%d, T_max=%d, n_kw=%d must be >= 1 and U_max=%d in [1, %d]", fn, n_rec, T_max, n_kw, U_max,
                rs::kSpotMaxLabels);
  if (max_hits < 1 || max_hits > rs::kSpotMaxHits)
    return fail(e, RS_ERR_INVALID_ARG, "%s: max_hits=%d outside [1, %d]", fn, max_hits, rs::kSpotMaxHits);
  if (std::isnan(threshold) || threshold == INFINITY)
    return fail(e, RS_ERR_INVALID_ARG, "%s: threshold must be finite or -inf", fn);
  const rs_model_config& c = e->cfg;
  const int U1 = U_max + 1, Hj = c.joint_hidden, Hp = c.pred_hidden;
  const int64_t pairs = static_cast<int64_t>(n_rec) * n_kw;
  const int64_t tiles = ((T_max + 15) / 16) * static_cast<int64_t>((U1 + 7) / 8);
  if (pairs * tiles > INT32_MAX || static_cast<int64_t>(n_rec) * T_max > INT32_MAX)
    return fail(e, RS_ERR_INVALID_ARG, "%s: %lld pairs of %d frames exceed one launch (fewer keywords per call)", fn, static_cast<long long>(pairs), T_max);
  char msg[256] = "";
  if (!rs::align_supported(Hj, Hp, c.vocab_size, U_max, msg)) return fail(e, RS_ERR_UNSUPPORTED, "%s: %s", fn, msg);
  if (!rs::spot_pick_fits(T_max, max_hits)) return fail(e, RS_ERR_UNSUPPORTED, "%s: T_max=%d exceeds the pick kernel's shared memory", fn, T_max);
  RS_CUDA(e, cudaSetDevice(e->device));
  Nvtx range("rs::rnnt_spot");
  const size_t M = static_cast<size_t>(n_rec) * T_max, cells = static_cast<size_t>(pairs) * T_max * U1;
  rs::Arena a;
  const size_t o_xn = a.take(M * c.d_model * 2), o_encp = a.take(M * Hj * 4);
  const size_t o_h = a.take(static_cast<size_t>(n_kw) * U1 * Hp * 4), o_c = a.take(static_cast<size_t>(n_kw) * Hp * 4);
  const size_t o_pp = a.take(static_cast<size_t>(n_kw) * U1 * Hj * 4);
  size_t o_lpb = 0, o_lpe = 0, o_ch = 0, o_E = 0, o_S = 0;
  if (!seam) {
    o_lpb = a.take(cells * 4); o_lpe = a.take(cells * 4); o_ch = a.take(cells);
    if (!E_out) o_E = a.take(static_cast<size_t>(pairs) * T_max * 4);
    if (!S_out) o_S = a.take(static_cast<size_t>(pairs) * T_max * 4);
  }
  RS_TRY(grow_align_ws(e, fn, a.off, s));
  char* ws = static_cast<char*>(e->align_ws);
  rs::AlignArgs g{};
  g.enc_proj = reinterpret_cast<float*>(ws + o_encp); g.enc_len = enc_len; g.labels = labels; g.label_len = label_len;
  g.w_out = e->dec.out_w; g.b_out = e->dec.out_b; g.w_lstm = e->dec.lstm_w; g.gate_tab = e->dec.gate_tab;
  g.w_pred = e->dec.pred_w; g.b_pred = e->dec.pred_b;
  g.B = n_kw; g.T_max = T_max; g.U_max = U_max; g.Hj = Hj; g.Hp = Hp; g.V = c.vocab_size;
  g.h = reinterpret_cast<float*>(ws + o_h); g.c = reinterpret_cast<float*>(ws + o_c); g.pred_proj = reinterpret_cast<float*>(ws + o_pp);
  g.lp_blank = seam ? lp_blank : reinterpret_cast<float*>(ws + o_lpb); g.lp_emit = seam ? lp_emit : reinterpret_cast<float*>(ws + o_lpe);
  g.choice = reinterpret_cast<uint8_t*>(ws + o_ch);
  const rs::SpotArgs sp{n_rec, threshold, max_hits, E_out ? E_out : reinterpret_cast<float*>(ws + o_E),
                        S_out ? S_out : reinterpret_cast<int32_t*>(ws + o_S), span, score, conf, frames, token_lp, count};
  // joint.enc over every frame of every recording, as in the forced alignment
  RS_LAUNCH(e, s, 1, rs::launch_f32_to_bf16(enc, ws + o_xn, static_cast<int64_t>(M) * c.d_model, s));
  RS_TRY(gemm(e, {ws + o_xn, e->dec.enc_w, e->dec.enc_b, nullptr, ws + o_encp, static_cast<int>(M), Hj, c.d_model, RS_EPI_BIAS_F32, 1.f}, s));
  for (int u = 0; u <= U_max; ++u) RS_LAUNCH(e, s, 1, rs::launch_align_lstm_step(g, u, s));
  RS_LAUNCH(e, s, 1, rs::launch_align_pred_proj(g, s));
  {
    const int r = launch(e, s, "rnnt_lattice_kernel<pairs>", 1, 0.0, [&] { return rs::launch_rnnt_lattice_pairs(g, n_rec, s, msg); });
    if (r != RS_OK && msg[0] != '\0') return fail(e, r, "%s: %s", fn, msg);
    RS_TRY(r);
  }
  if (seam) return RS_OK;
  RS_LAUNCH(e, s, 1, rs::launch_rnnt_spot_dp(g, sp, s));
  RS_LAUNCH(e, s, 1, rs::launch_rnnt_spot_pick(g, sp, s));
  return RS_OK;
}

}  // namespace

extern "C" {

int rs_rnnt_spot(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int n_rec, int T_max, const int32_t* labels_dev,
                 const int32_t* label_len_dev, int n_kw, int U_max, float threshold, int max_hits, int32_t* span_dev, float* score_dev,
                 float* confidence_dev, int32_t* frames_dev, float* token_lp_dev, int32_t* count_dev, float* E_dev, int32_t* S_dev,
                 void* stream) {
  return rnnt_spot(e, enc_dev, enc_len_dev, n_rec, T_max, labels_dev, label_len_dev, n_kw, U_max, threshold, max_hits, span_dev, score_dev,
                   confidence_dev, frames_dev, token_lp_dev, count_dev, E_dev, S_dev, static_cast<cudaStream_t>(stream));
}

int rs_rnnt_spot_lattice(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int n_rec, int T_max, const int32_t* labels_dev,
                         const int32_t* label_len_dev, int n_kw, int U_max, float* lp_blank_dev, float* lp_emit_dev, void* stream) {
  if (lp_blank_dev == nullptr || lp_emit_dev == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_spot_lattice: bad arguments");
  return rnnt_spot(e, enc_dev, enc_len_dev, n_rec, T_max, labels_dev, label_len_dev, n_kw, U_max, -1.f, 1, nullptr, nullptr, nullptr, nullptr,
                   nullptr, nullptr, nullptr, nullptr, static_cast<cudaStream_t>(stream), lp_blank_dev, lp_emit_dev);
}

int rs_rnnt_align(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, const int32_t* labels_dev,
                  const int32_t* label_len_dev, int U_max, int32_t* frames_dev, float* token_lp_dev, float* viterbi_dev,
                  float* loglik_dev, void* stream) {
  return rnnt_align(e, "rs_rnnt_align", enc_dev, enc_len_dev, B, T_max, labels_dev, label_len_dev, U_max, nullptr, nullptr, frames_dev,
                    token_lp_dev, viterbi_dev, loglik_dev, static_cast<cudaStream_t>(stream));
}

int rs_rnnt_align_lattice(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, const int32_t* labels_dev,
                          const int32_t* label_len_dev, int U_max, float* lp_blank_dev, float* lp_emit_dev, void* stream) {
  if (lp_blank_dev == nullptr || lp_emit_dev == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_align_lattice: bad arguments");
  return rnnt_align(e, "rs_rnnt_align_lattice", enc_dev, enc_len_dev, B, T_max, labels_dev, label_len_dev, U_max, lp_blank_dev, lp_emit_dev,
                    nullptr, nullptr, nullptr, nullptr, static_cast<cudaStream_t>(stream));
}

int rs_rnnt_align_banded(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, const int32_t* labels_dev,
                         const int32_t* label_len_dev, int U_max, const int32_t* band_lo_host, const int32_t* band_hi_host, int32_t* frames_dev,
                         float* token_lp_dev, float* viterbi_dev, float* loglik_dev, int32_t* edge_dev, void* stream) {
  return rnnt_align_banded(e, "rs_rnnt_align_banded", enc_dev, enc_len_dev, B, T_max, labels_dev, label_len_dev, U_max, band_lo_host,
                           band_hi_host, nullptr, nullptr, frames_dev, token_lp_dev, viterbi_dev, loglik_dev, edge_dev,
                           static_cast<cudaStream_t>(stream));
}

int rs_rnnt_align_banded_lattice(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, const int32_t* labels_dev,
                                 const int32_t* label_len_dev, int U_max, const int32_t* band_lo_host, const int32_t* band_hi_host,
                                 float* lp_blank_dev, float* lp_emit_dev, void* stream) {
  if (lp_blank_dev == nullptr || lp_emit_dev == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_align_banded_lattice: bad arguments");
  return rnnt_align_banded(e, "rs_rnnt_align_banded_lattice", enc_dev, enc_len_dev, B, T_max, labels_dev, label_len_dev, U_max, band_lo_host,
                           band_hi_host, lp_blank_dev, lp_emit_dev, nullptr, nullptr, nullptr, nullptr, nullptr,
                           static_cast<cudaStream_t>(stream));
}

int rs_rnnt_align_segment(rs_engine* e, const float* enc_dev, const int32_t* enc_len_dev, int B, int T_max, const int32_t* labels_dev,
                          const int32_t* label_len_dev, int U_max, int32_t* seg_dev, int32_t* frames_dev, float* token_lp_dev,
                          float* frame_lp_dev, float* viterbi_dev, float* loglik_dev, void* stream) {
  if (seg_dev == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_rnnt_align_segment: bad arguments");
  return rnnt_align(e, "rs_rnnt_align_segment", enc_dev, enc_len_dev, B, T_max, labels_dev, label_len_dev, U_max, nullptr, nullptr, frames_dev,
                    token_lp_dev, viterbi_dev, loglik_dev, static_cast<cudaStream_t>(stream), seg_dev, frame_lp_dev);
}

int rs_resample_mono(rs_engine* e, const void* in_dev, int in_is_pcm16, const int32_t* len_in_dev, int B, int channels, int L_in_max,
                     const float* taps_dev, int taps_per_phase, int up, int down, int n_pre_remove, int pad, float* out_dev,
                     int L_out_row, int32_t* len_out_dev, void* stream) {
  if (!e || !in_dev || !len_in_dev || !taps_dev || !out_dev || !len_out_dev) return fail(e, RS_ERR_INVALID_ARG, "rs_resample_mono: bad arguments");
  RS_CUDA(e, cudaSetDevice(e->device));
  Nvtx range("rs::resample_mono");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  rs::ResampleArgs a{in_dev, in_is_pcm16 != 0, len_in_dev, B, channels, L_in_max, taps_dev, taps_per_phase, up, down, n_pre_remove, pad,
                     out_dev, L_out_row, len_out_dev};
  RS_LAUNCH(e, s, 1, rs::launch_resample_mono(a, s));
  return RS_OK;
}

int rs_gemm_bf16(rs_engine* e, const void* a, const void* w, const float* bias, const float* resid, void* out, int M,
                 int N, int K, int epilogue, float alpha, void* out2, int split, int ld2, void* stream) {
  if (!e || !a || !w || !out) return fail(e, RS_ERR_INVALID_ARG, "rs_gemm_bf16: bad arguments");
  if (epilogue == RS_EPI_QKV_VT && (!out2 || split <= 0 || split >= N || split % 32 || M % 8 || ld2 % 8 || ld2 < M))
    return fail(e, RS_ERR_INVALID_ARG, "rs_gemm_bf16: RS_EPI_QKV_VT needs out2, 0 < split < N, split %% 32 == 0, M %% 8 == 0, ld2 %% 8 == 0, ld2 >= M");
  RS_CUDA(e, cudaSetDevice(e->device));
  return gemm(e, {a, w, bias, resid, out, M, N, K, epilogue, alpha, out2, split, ld2}, static_cast<cudaStream_t>(stream));
}

int rs_layernorm(rs_engine* e, const float* x, const float* gamma, const float* beta, float* out_f32, void* out_bf16,
                 const float* gamma2, const float* beta2, int rows, int d, void* stream) {
  if (!e || !x || !gamma || !beta || (gamma2 == nullptr) != (beta2 == nullptr)) return fail(e, RS_ERR_INVALID_ARG, "rs_layernorm: bad arguments");
  if (gamma2 != nullptr && out_bf16 == nullptr) return fail(e, RS_ERR_INVALID_ARG, "rs_layernorm: the chained LayerNorm writes out_bf16");
  if (d != 256 && d != 512 && d != 1024) return fail(e, RS_ERR_UNSUPPORTED, "rs_layernorm: d=%d unsupported (256/512/1024)", d);
  RS_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RS_LAUNCH(e, s, 1, rs::launch_layernorm(x, gamma, beta, out_f32, out_bf16, gamma2, beta2, rows, d, e->cfg.ln_eps, s));
  return RS_OK;
}

int rs_attention(rs_engine* e, const void* qkv, const void* vt, int ld_vt, const void* pos, const float* bd_bias, int n_rel_pad,
                 const float* bias_u, void* out, const int32_t* enc_len, int B, int T_max, int H, int w_left, int w_right,
                 int n_global, void* stream) {
  if (!e || !qkv || !vt || !pos || !bd_bias || !bias_u || !out || !enc_len || B <= 0 || T_max <= 0 || H <= 0)
    return fail(e, RS_ERR_INVALID_ARG, "rs_attention: bad arguments");
  rs::AttnArgs aa{qkv, pos, bd_bias, n_rel_pad, bias_u, out, enc_len, B, T_max, H, 128, w_left, w_right, n_global};
  aa.vt = vt; aa.ld_vt = ld_vt;
  if (!rs::attention_tc_supported(aa))
    return fail(e, RS_ERR_UNSUPPORTED, "rs_attention: unsupported geometry (0 <= w_left, w_right <= 128, w_left %% 8 == 0, n_global 0/1, "
                "T_max %% 8 == 0, n_rel_pad a multiple of 32 in [w_left + w_right + 1, 288])");
  // the global-row kernel keeps max(T_max, 1024) scores in at most 200 KB of shared memory
  if (ld_vt % 8 || static_cast<int64_t>(ld_vt) < static_cast<int64_t>(B) * T_max || (n_global > 0 && (T_max + 8 + 128) * 4 > 200 * 1024))
    return fail(e, RS_ERR_INVALID_ARG, "rs_attention: ld_vt must be a multiple of 8 and >= B*T_max; T_max too large for the global row");
  RS_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RS_LAUNCH(e, s, n_global > 0 ? 2 : 1, rs::launch_attention_tc(aa, s));
  return RS_OK;
}

int rs_conv_dw(rs_engine* e, const void* u, void* out, const float* w, const float* shift, const int32_t* enc_len, int B, int T_max,
               int d, int k, void* stream) {
  if (!e || !u || !out || !w || !shift || !enc_len || B <= 0 || T_max <= 0 || d <= 0) return fail(e, RS_ERR_INVALID_ARG, "rs_conv_dw: bad arguments");
  if (k != 9) return fail(e, RS_ERR_UNSUPPORTED, "rs_conv_dw: k=%d unsupported (9)", k);
  if (d % 4) return fail(e, RS_ERR_INVALID_ARG, "rs_conv_dw: d %% 4 != 0");
  RS_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RS_LAUNCH(e, s, 1, rs::launch_conv_dw(u, out, w, shift, enc_len, B, T_max, d, k, s));
  return RS_OK;
}

int rs_sub_conv0_dw1(rs_engine* e, const float* mel, const int32_t* mel_len, const float* mel_stats, int B, int F_max, int n_mels, int C,
                     const float* w0, const float* b0, const float* wd, const float* bd, void* out, void* stream) {
  if (!e || !mel || !mel_len || !w0 || !b0 || !wd || !bd || !out || B <= 0 || F_max <= 0 || n_mels <= 0 || C <= 0)
    return fail(e, RS_ERR_INVALID_ARG, "rs_sub_conv0_dw1: bad arguments");
  // the kernel stages 19 rows of n_mels + 8 floats in the default 48 KB of shared memory
  if (n_mels > 600) return fail(e, RS_ERR_UNSUPPORTED, "rs_sub_conv0_dw1: n_mels=%d unsupported (<= 600)", n_mels);
  RS_CUDA(e, cudaSetDevice(e->device));
  const int T1 = conv_len(F_max), F1 = conv_len(n_mels);
  rs::SubsampleArgs sa{mel, mel_len, mel_stats, B, F_max, n_mels, C, w0, b0, wd, bd, out, T1, F1, conv_len(T1), conv_len(F1)};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RS_LAUNCH(e, s, 1, rs::launch_sub_conv0_dw1(sa, s));
  return RS_OK;
}

int rs_sub_dw(rs_engine* e, const void* in, void* out, const float* w, const float* b, const int32_t* mel_len, int len_shift, int B,
              int Tin, int Fin, int Tout, int Fout, int C, void* stream) {
  if (!e || !in || !out || !w || !b || !mel_len || len_shift < 0 || B <= 0 || Tin <= 0 || Fin <= 0 || Tout <= 0 || Fout <= 0 || C <= 0)
    return fail(e, RS_ERR_INVALID_ARG, "rs_sub_dw: bad arguments");
  if (C % 8 || C / 8 > 128 || 128 % (C / 8)) return fail(e, RS_ERR_UNSUPPORTED, "rs_sub_dw: C=%d unsupported (C / 8 must divide 128)", C);
  RS_CUDA(e, cudaSetDevice(e->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  RS_LAUNCH(e, s, 1, rs::launch_sub_dw(in, out, w, b, mel_len, len_shift, B, Tin, Fin, Tout, Fout, C, s));
  return RS_OK;
}

int64_t rs_launch_count(const rs_engine* e) { return e ? e->launches : 0; }

int rs_enable_stage_timing(rs_engine* e, int on) {
  if (!e) return RS_ERR_INVALID_ARG;
  e->timing = on != 0;
  return RS_OK;
}

// Stages: [0] log-mel, [1] subsampling, [2] conformer layers, [3] f32->bf16 + joint.enc GEMM, [4] greedy decode.
int rs_stage_times_ms(const rs_engine* e, float* ms) {
  if (!e || !ms) return RS_ERR_INVALID_ARG;
  for (int i = 0; i < 8; ++i) ms[i] = 0.f;
  if (cudaEventSynchronize(e->ev[5]) != cudaSuccess) return RS_ERR_CUDA;
  for (int i = 0; i < 5; ++i) cudaEventElapsedTime(&ms[i], e->ev[i], e->ev[i + 1]);
  return RS_OK;
}

// Debug: the 12 cycle counters of the batched decode kernel's CTA 0 from the last rs_transcribe_* call for (B, L_max):
// phase J, barrier, token reduce, phase L, barrier, phase P, barrier, iterations, three sub-timers of phase J, one unused slot.
// Synchronises the device.
int rs_debug_decode_cycles(rs_engine* e, int B, int L_max, int U_max, int64_t* out12) {
  if (!e || !out12) return RS_ERR_INVALID_ARG;
  Plan p = make_plan(e, B, L_max, U_max);
  RS_CUDA(e, cudaDeviceSynchronize());
  const size_t off = p.dec_ws + dec_ws(e, B).prof;
  RS_CUDA(e, cudaMemcpy(out12, static_cast<char*>(e->ws) + off, 12 * sizeof(int64_t), cudaMemcpyDeviceToHost));
  return RS_OK;
}

int rs_enable_kernel_timing(rs_engine* e, int on) {
  if (!e) return RS_ERR_INVALID_ARG;
  e->ktiming = on != 0;
  e->log.clear();
  return RS_OK;
}

// Text summary "name\tcount\ttotal_ms\n..." of every launch logged since rs_enable_kernel_timing(e, 1); clears the log.
int rs_kernel_timing(rs_engine* e, char* buf, int buf_bytes) {
  if (!e || !buf || buf_bytes <= 0) return RS_ERR_INVALID_ARG;
  std::map<std::string, std::pair<int, double>> agg;
  RS_TRY(drain_log(e, [&](const rs_engine::Timed& t, float ms) {
    auto& a = agg[t.tag];
    a.first += 1; a.second += ms;
  }));
  std::string out;
  char line[160];
  for (const auto& kv : agg) {
    snprintf(line, sizeof line, "%s\t%d\t%.4f\n", kv.first.c_str(), kv.second.first, kv.second.second);
    out += line;
  }
  snprintf(buf, static_cast<size_t>(buf_bytes), "%s", out.c_str());
  return RS_OK;
}

int rs_enable_gemm_timing(rs_engine* e, int on) {
  if (!e) return RS_ERR_INVALID_ARG;
  e->gemm_timing = on != 0;
  e->log.clear();
  return RS_OK;
}

// The GEMM entries of the launch log: summed device time, summed 2*M*N*K, count; clears the log.
int rs_gemm_timing(rs_engine* e, double* ms, double* flops, int64_t* launches) {
  if (!e || !ms || !flops || !launches) return RS_ERR_INVALID_ARG;
  double total = 0.0, fl = 0.0;
  int64_t n = 0;
  RS_TRY(drain_log(e, [&](const rs_engine::Timed& t, float t_ms) {
    if (t.flops > 0.0) { total += t_ms; fl += t.flops; ++n; }
  }));
  *ms = total; *flops = fl; *launches = n;
  return RS_OK;
}

}  // extern "C"
