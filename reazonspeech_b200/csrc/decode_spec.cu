// Windowed ("blank-run speculative") batched RNN-T greedy decode: NeMo GreedyRNNTInfer._greedy_decode, RNNTDecoder.predict
// and RNNTJoint.joint (the reference reaches them at pkg/nemo-asr/src/transcribe.py:48-53) as ONE persistent cooperative
// kernel, organised around two facts about greedy transducer decoding:
//
//  1. A blank leaves the prediction-network state untouched, so the joint of the NEXT frames can be
//     evaluated against the same state before the current decision is known.  Every iteration scores a
//     window of kFrames consecutive frames per utterance; the utterance then consumes the window up to and
//     including its first non-blank frame (all-blank window: kFrames frames in one iteration).  The decision
//     sequence is exactly the sequential one; the number of lock-step iterations drops from max(T + U) to
//     about max(U + (T - U)/kFrames).
//  2. With kFrames x B rows per iteration the joint is a real (small) GEMM.  The CTAs form a 2-D grid,
//     kGroups utterance groups x S vocabulary slices: a CTA keeps its ~82 rows of W_out in shared memory
//     for the whole decode and multiplies them with the relu(enc_proj + pred_proj) rows of its group
//     (32 rows per pass) on wgmma (see the kernel's comment).  Activations keep 22 mantissa bits: every fp32 value is
//     split into two IEEE-half terms (hi + lo), the bf16 weights are exact in half, accumulation is fp32.
//     joint.pred and the recurrent half of the LSTM of the utterances that emitted are the same kind of GEMM (rows =
//     utterances, K split over the warps, A fragments loaded straight from L2) on mma.sync m16n8k16.
//  3. The input half of the LSTM gates depends on the emitted token only: W_ih . embed[k] + b_ih + b_hh is a table
//     [V+1, 4*Hp] built once at load time (pred.gate_tab).  The recurrent half W_hh . h does not depend on the token at
//     all, so it is computed as soon as h is known: phase P, which has to pull every emitting utterance's full new h
//     through L2 for joint.pred anyway (that traffic, not the arithmetic, is what the phase costs), multiplies the same
//     fragments by the CTA's W_hh rows too and keeps the result (rec) for the utterance's next step.  That step is then
//     elementwise: gates = rec + gate_tab[token].
//
//   phase J  kGroups x S CTAs: window logits of the CTA's vocabulary slice -> per (utterance, frame) a grid-wide
//            64-bit red.max of (ordered logit bits | ~row)
//   barrier  -> every CTA reads the window's tokens, advances (t, symbols), emits; requests the next window's enc_proj rows
//   phase L  utterances that emitted: gates = rec + gate_tab[token] of the CTA's units -> new h slice
//   barrier
//   phase P  utterances that emitted: pred_proj rows and rec = W_hh . h of the CTA from the new h
//   barrier
//
// Confidence (kConf = true; the decisions never depend on it).  Phase J also reduces, over the same fp32 logits l of the CTA's
// vocabulary slice, one softmax tuple per (utterance, frame): m = max l, s = sum e^(l-m), g = sum e^(l-m) (l-m),
// a = sum e^(alpha (l-m)), ga = sum e^(alpha (l-m)) (l-m), and stores it in the conf ring (one slot per slice).  After the
// consume step every emission below U_max is merged over the S slices by one warp (emission e: CTA e % G) into
// stats[b][n] = (log p of the emitted token, sum p log p, sum p^alpha, sum p^alpha log p) over all V + 1 classes.
//
// Phrase boosting (kBoost = true; tables built by reazonspeech_b200/boosting.py).  Every utterance carries a state of the
// phrase automaton, s_state[b], advanced identically by every CTA in the consume step: s_state = next[s_state][token] on
// every emission (a value outside [0, n_states) becomes the row's root).  Row b starts at its root boost_root[b] (0 without
// roots): with several automata laid one after another in one table, each with next offset to its own region, each row
// decodes against its own phrase list.  The root is re-read from global memory where it is needed (the start, and the
// out-of-range case), which keeps it out of the register budget.  The decision for a (utterance, frame) is the argmax of
// logit_k + bonus[s_state][k], blank never boosted.  The four frames of a window share the utterance's state, so a pass needs
// the bonus rows of its <= 8 utterances over the CTA's vocabulary slice: cp.async'd into a shared tile when the pass's
// rows are fetched (pass 0: under phases L and P) and added to the logits in the argmax epilogue.  With kConf as well, the
// statistics stay those of the UNBOOSTED softmax at the boosted decision: log p = (l_emit - m) - log s, l_emit = the winner's
// boosted value (recovered from its ordered bits) - its bonus, which is the raw logit to within one fp32 rounding.
//
// n-gram LM shallow fusion (kLM = true; tables built by reazonspeech_b200/ngram_lm.py, which states the semantics).  Every
// utterance carries an LM state s_lm[b] (a context of the ARPA).  The LM term of token k in state s is cb[s] + w, w = arc_w of
// the highest-level arc for k on s's back-off chain chain[s][0..order-1), or uni_w[k] (the dense root row) when there is none;
// the state reached is that arc's arc_to (or uni_to[k]).  A pass fills, per utterance (one warp each), an LM tile of terms and
// next states over the CTA's vocabulary slice: the root row first, then every chain level from the lowest to the highest
// overwrites the tokens of its arcs (sorted, so a few 32-wide probe rounds narrow each level to the slice; all levels probe in
// the same rounds).  The term is added to the logits next to the boosting bonus (the sum bonus + term when both are on).  The
// transition costs no search: for the best token of every (row, slice), warp 0 writes (next state, added term) into the LM ring
// ([3][B][kFrames][S], like conf); after the consume step the ring slot of the emitted token's slice holds the new state, which
// phase L reads.  Pass 0's tile is filled between the arrival at and the release from the grid barrier that ends phase L,
// i.e. under the barrier's latency.  With kConf the emitted token's unfused logit is its fused value - the added term.
//
// Resume (streaming; semantics: reazonspeech_b200/streaming.py), rnnt_greedy_resume_kernel: the same body with the load at the
// start and the store at the end compiled in (kResume), its own 16 instances: as a runtime branch the same code moved the
// register allocation of the offline instances.  With p.states set, row b
// decodes frames [dec_begin[b], enc_len[b]) from record slot[b]: int32 started, boost_state, lm_state, reserved, then f32 c[HP],
// rec[HP][4], pp[HJ].  h itself is not needed: the next LSTM step reads only rec = W_hh . h, c and the token's gate_tab row, and
// pp feeds the joint.  sym is not needed either: a row leaves the loop only at t == enc_len, reached by a blank or a max_symbols
// advance, both of which reset it.  An unstarted record (all zero) runs the SOS step exactly as a fresh decode does.
#include "common.cuh"
#include "kernels.h"
#include "ngram_lm.cuh"

namespace rs {

constexpr int kStateHead = 16;                   // bytes of a stream record's header (three documented int32 words + one reserved)
size_t stream_state_bytes(int Hj, int Hp) { return (kStateHead + (static_cast<size_t>(Hp) * 5 + Hj) * 4 + 15) & ~static_cast<size_t>(15); }

constexpr int kSpThreads = 256;
constexpr int kSpWarps = kSpThreads / 32;
constexpr int kFrames = 4;                       // frames scored per utterance and iteration
constexpr int kGroups = 4;                       // utterance groups (utterance b belongs to group b % kGroups)
constexpr int kPassRows = 32;                    // (utterance, frame) rows per pass: two m16 tiles
constexpr int kPassUtts = kPassRows / kFrames;

struct SpecDev {
  const float* enc_proj; const int32_t* enc_len;
  const __nv_bfloat16* w_out; const float* b_out;
  const __nv_bfloat16* w_lstm; const float* gate_tab; const __nv_bfloat16* w_pred; const float* b_pred;
  int32_t* tokens; int32_t* frames; int32_t* n_tok;
  unsigned long long* best;   // [3][B][kFrames] packed (ordered logit bits << 32 | ~row), 3-deep ring
  float* hbuf;                // [B][Hp]
  float* rec;                 // [B][Hp][4 gates] W_hh . h, written and read only by the CTA that owns the unit
  float* ppbuf;               // [B][Hj]
  unsigned int* counter;      // grid barrier: kBarCounters arrival counters, one per 128-byte line
  long long* prof;            // [12] cycle counters of CTA 0
  float* conf;                // [3][B][kFrames][S][5] softmax tuples of each vocabulary slice, 3-deep ring like best (kConf)
  float* stats;               // [B][U_max][4] (lp, H1, A_alpha, G_alpha) of every stored token (kConf)
  float alpha, alpha_l2;      // alpha and alpha * log2(e) (kConf)
  const float* boost_bonus;   // [n_states][boost_pitch] bonus of each non-blank token per automaton state (kBoost)
  const int32_t* boost_next;  // [n_states][boost_pitch] automaton transition on each non-blank token (kBoost)
  int boost_states, boost_pitch;
  NgramLM lm;                 // (kLM)
  int2* lm_ring;              // [3][B][kFrames][S] (next LM state, added term bits) of each slice's best token (kLM)
  int B, T_max, V, U_max, max_symbols;
  int S, rows_j, units, rows_p;
  // resume (rnnt_greedy_resume_kernel): row b decodes frames [dec_begin[b], enc_len[b]) from record slot[b] of `states` and
  // writes its state back there
  const int32_t* dec_begin; const int32_t* slot; uint8_t* states; int state_bytes;
  // kBoost: root state of each row ([B]; nullptr: state 0 for every row).  Last, so that the other fields keep their offsets
  // and the instances without kBoost their code.
  const int32_t* boost_root;
};

// Row b's root of the phrase automaton: where it starts, and where a state outside the table sends it (kBoost)
__device__ __forceinline__ int boost_root_of(const SpecDev& p, int b) { return p.boost_root != nullptr ? __ldg(p.boost_root + b) : 0; }

// Softmax statistics of a set of logits relative to its maximum m (an empty set: m = -inf, all sums zero):
// s = sum e^(l-m), g = sum e^(l-m) (l-m), a = sum e^(alpha (l-m)), ga = sum e^(alpha (l-m)) (l-m).
struct SoftStat { float m, s, g, a, ga; };
constexpr float kLog2e = 1.4426950408889634f;
__device__ __forceinline__ SoftStat soft_one(float l) { return {l, 1.f, 0.f, 1.f, 0.f}; }
__device__ __forceinline__ SoftStat soft_empty() { return {-INFINITY, 0.f, 0.f, 0.f, 0.f}; }
// union of two disjoint sets: the smaller-maximum side is rescaled by e^d (resp. e^(alpha d)), d = its m - the larger m
__device__ __forceinline__ SoftStat soft_merge(SoftStat x, SoftStat y, float alpha_l2) {
  if (y.m > x.m) { const SoftStat t = x; x = y; y = t; }
  if (y.m == -INFINITY) return x;
  const float d = y.m - x.m;
  const float r = exp2f(d * kLog2e), ra = exp2f(d * alpha_l2);
  x.s += r * y.s; x.g += r * (y.g + y.s * d);
  x.a += ra * y.a; x.ga += ra * (y.ga + y.a * d);
  return x;
}
__device__ __forceinline__ SoftStat soft_shfl_xor(const SoftStat& x, int o) {
  return {__shfl_xor_sync(0xffffffffu, x.m, o), __shfl_xor_sync(0xffffffffu, x.s, o), __shfl_xor_sync(0xffffffffu, x.g, o),
          __shfl_xor_sync(0xffffffffu, x.a, o), __shfl_xor_sync(0xffffffffu, x.ga, o)};
}

// Grid barrier over kBarCounters arrival counters, each in its own 128-byte line: CTA i arrives on counter i % kBarCounters,
// threads 0..kBarCounters-1 each poll one counter.  Arrivals of every CTA on ONE address are serialised by the L2 slice that
// owns it, three times per decode iteration; spread over several lines they proceed in parallel.  `round` counts the barriers passed; counter c has seen round * (number of CTAs with i % kBarCounters == c) arrivals.
constexpr int kBarCounters = 8;
constexpr int kBarStride = 32;            // unsigned ints between counters
// `during` runs CTA-local work between the arrival and the wait: it may touch only shared memory and read-only global data
// (other CTAs' writes of the phase are not visible to it)
template <class F>
__device__ __forceinline__ void sp_grid_barrier_with(unsigned int* counters, unsigned int& round, unsigned int nblocks, F&& during) {
  __syncthreads();
  ++round;
  if (threadIdx.x == 0)
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counters + (blockIdx.x % kBarCounters) * kBarStride) : "memory");
  during();
  if (threadIdx.x < kBarCounters) {
    const unsigned int c = threadIdx.x;
    const unsigned int target = round * ((nblocks + kBarCounters - 1 - c) / kBarCounters);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counters + c * kBarStride) : "memory");
    } while (v < target);
  }
  __syncthreads();
}

__device__ __forceinline__ void sp_grid_barrier(unsigned int* counters, unsigned int& round, unsigned int nblocks) {
  sp_grid_barrier_with(counters, round, nblocks, [] {});
}

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void mma_f16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float2 ldcg2(const float* p) { return __ldcg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ float4 ldcg4s(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ unsigned long long pack_best(float v, int row) {
  unsigned int fb = __float_as_uint(v);
  fb = (fb & 0x80000000u) ? ~fb : (fb | 0x80000000u);           // order-preserving
  return (static_cast<unsigned long long>(fb) << 32) | (0xffffffffu - static_cast<unsigned int>(row));   // ties -> lower row
}
// the value pack_best ordered (inverse of its bit transform)
__device__ __forceinline__ float best_value(unsigned long long v) {
  const unsigned int fb = static_cast<unsigned int>(v >> 32);
  return __uint_as_float((fb & 0x80000000u) ? (fb & 0x7fffffffu) : ~fb);
}

// Phrase-boosting tile: one bonus row per utterance of a pass, the CTA's vocabulary slice starting at the 16-byte boundary at or
// below j0 (<= 3 + 128 + 3 floats copied)
constexpr int kTileLd = 136;

// The joint window runs on wgmma.  A = the CTA's W_out rows as IEEE half in 128B-swizzled K-major slabs of 64 columns
// (88 rows stored per slab; the two warpgroups' m64 instructions cover 128 rows and read on into the next slab / region,
// whose rows land in accumulator rows nobody looks at), B = the 32 (utterance, frame) activation rows as two half planes
// (hi, lo) staged one k-half at a time, D = [128 vocabulary rows x (32 hi | 32 lo)] fp32 in registers.
// The hi and lo planes of the activations sit side by side as ONE B tile of 64 rows (rows 0-31 hi, 32-63 lo), so a k16 step
// is one m64n64k16 per warpgroup and the two halves of D are added in the epilogue.
static_assert(kSpThreads == 256, "the joint is issued by two warpgroups");

template <int HJ, int HP, bool kConf, bool kBoost, bool kLM, bool kResume>
__device__ __forceinline__ void greedy_spec_body(const SpecDev& p) {
  constexpr int KH = HJ / 2;                 // joint k-half staged in shared memory at a time
  constexpr int LS = HP + 8;                 // W_hh row stride in halves
  constexpr int KSW = (HP / 16) / kSpWarps;  // k16 steps per warp of phase P
  constexpr int V4_ROW = KH / 4;             // float4 per staged row
  constexpr int ITEMS = kPassUtts * V4_ROW;  // loader items per k-half: (utterance, float4 column)
  constexpr int PERU = (ITEMS + kSpThreads - 1) / kSpThreads;
  static_assert(HJ % 32 == 0 && (HP / 16) % kSpWarps == 0, "shape");

  extern __shared__ __align__(16) uint8_t ssm[];
  const int G = gridDim.x, cta = blockIdx.x;
  const int NC = p.V + 1, blank = p.V, B = p.B;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gid = lane >> 2, tig = lane & 3;

  // ---- slices owned by this CTA
  const int grp = cta / p.S, slice = cta % p.S;
  const bool has_j = grp < kGroups;
  const int j0 = min(NC, slice * p.rows_j), j1 = min(NC, j0 + p.rows_j);
  const int nj = has_j ? j1 - j0 : 0;
  const int u0 = min(HP, cta * p.units), u1 = min(HP, u0 + p.units);
  const int nu = u1 - u0;
  const int p0 = min(HJ, cta * p.rows_p), p1 = min(HJ, p0 + p.rows_p);
  const int np = p1 - p0;

  // ---- shared memory carve-up.  B fragments of a partial last n8-tile read past the end of a weight array
  // into the next one; those columns are masked, and every array is followed by at least 8 more rows of bytes.
  constexpr int KSLABS = HJ / 64;                                  // 64-column slabs of A
  constexpr int NSLAB_H = KH / 64;                                 // slabs per staged k-half
  const int rows_a8 = (p.rows_j + 7) & ~7;
  const uint32_t a_slab = static_cast<uint32_t>(rows_a8) * 128u;   // bytes per A slab
  constexpr uint32_t kBSlab = 8192u;                               // B slab: 64 rows x 128 B = hi plane (rows 0-31) | lo plane (rows 32-63)
  constexpr uint32_t kBRegion = (NSLAB_H * kBSlab > 32768u) ? NSLAB_H * kBSlab : 32768u;   // >= what an M = 128 read of the last A slab overruns, and the P reduction buffer
  // Order: [A slabs | W_lstm | W_pred | pad to 1024 | B slabs (also the P reduction buffer) | bias, state ...].  The mma.sync B fragments of the LSTM /
  // joint.pred phases read up to 8 rows past the end of their (5- or 20-row) arrays: those reads must land inside the
  // allocation, so the big B region follows the weight arrays (a 2-utterance batch otherwise read past the end of shared memory).
  const uint32_t wlp_bytes = static_cast<uint32_t>((static_cast<size_t>(4 * p.units) * LS + static_cast<size_t>(p.rows_p) * (HP + 8)) * 2);   // LS = HP + 8
  const uint32_t tc_base = (smem_u32(ssm) + 1023u) & ~1023u;
  const uint32_t b_off = (KSLABS * a_slab + wlp_bytes + 1023u) & ~1023u;
  uint8_t* gA = ssm + (tc_base - smem_u32(ssm));                   // generic pointers to the A slabs / B slabs
  uint8_t* gB = gA + b_off;
  __nv_bfloat16* s_wlstm = reinterpret_cast<__nv_bfloat16*>(gA + KSLABS * a_slab);    // [4*units][LS] gate-major
  __nv_bfloat16* s_wpred = s_wlstm + static_cast<size_t>(4 * p.units) * LS;           // [rows_p][HP + 8]
  float* s_g = reinterpret_cast<float*>(gB);                                          // B planes; also the P reduction buffer
  float* s_bout = reinterpret_cast<float*>(gB + kBRegion);                            // -inf beyond nj
  constexpr int n_bout = 128;
  float* s_c = s_bout + n_bout;                                                      // [B][units]
  unsigned long long* s_best = reinterpret_cast<unsigned long long*>(s_c + ((static_cast<size_t>(B) * p.units + 1) & ~static_cast<size_t>(1)));   // [32][kSpWarps]
  long long* s_prof = reinterpret_cast<long long*>(s_best + kPassRows * kSpWarps);    // [12] cycle counters of CTA 0 (rs_debug_decode_cycles)
  int* s_t = reinterpret_cast<int*>(s_prof + 12);
  int* s_sym = s_t + B; int* s_n = s_sym + B; int* s_tok = s_n + B;
  int* s_emit = s_tok + B; int* s_len = s_emit + B;
  int* s_act = s_len + B;                                                            // ordered list of the utterances with frames left
  int* s_cnt = s_act + B;                                                            // [0] n_emit, [1] n_active, [2..2+8) warp counts x2
  int* s_cj = s_cnt + 2 + 2 * kSpWarps;                                              // kConf: window frame of b's stored emission, -1: none
  float* s_conf = reinterpret_cast<float*>(s_cj + B);                                // kConf: [32 rows][kSpWarps][5] per-warp softmax tuples
  // kBoost: [kPassUtts][kTileLd] bonus tile (16-byte aligned, after the kConf arrays when they exist), automaton state per
  // utterance, and with kConf the emitted token's unboosted logit per utterance
  float* s_tile = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(kConf ? s_conf + kPassRows * kSpWarps * 5 : reinterpret_cast<float*>(s_cj)) + 15) & ~static_cast<uintptr_t>(15));
  int* s_state = reinterpret_cast<int*>(s_tile + kPassUtts * kTileLd);
  float* s_le = reinterpret_cast<float*>(s_state + B);
  // kLM (after the kBoost arrays, which then always exist): [kPassUtts][kTileLd] LM term and next-state tiles, the per-warp
  // (next state, added term) of each row's best token [kPassRows][kSpWarps] (8-byte aligned), LM state and LM ring slot of the
  // window's emission (-1: none) per utterance
  float* s_lmw = reinterpret_cast<float*>(s_le + B);
  int* s_lmn = reinterpret_cast<int*>(s_lmw + kPassUtts * kTileLd);
  int2* s_lmb = reinterpret_cast<int2*>((reinterpret_cast<uintptr_t>(s_lmn + kPassUtts * kTileLd) + 7) & ~static_cast<uintptr_t>(7));
  int* s_lm = reinterpret_cast<int*>(s_lmb + kPassRows * kSpWarps);
  int* s_lslot = s_lm + B;

  {
    const uint32_t zero = 0;
    // W_out slice (rows beyond nj zero-filled)
    {
      for (int i = tid; i < rows_a8 * (HJ / 8); i += kSpThreads) {
        const int r = i / (HJ / 8), c = i % (HJ / 8);          // c: 16-byte chunk (8 columns) of the row
        uint4 v = make_uint4(zero, zero, zero, zero);
        if (r < nj) v = bf16x8_to_f16x8(reinterpret_cast<const uint4*>(p.w_out + static_cast<size_t>(j0 + r) * HJ)[c]);
        *reinterpret_cast<uint4*>(gA + (c >> 3) * a_slab + (r >> 3) * 1024 + (r & 7) * 128 + (((c & 7) ^ (r & 7)) << 4)) = v;
      }
    }
    for (int i = tid; i < 4 * p.units * (HP / 8); i += kSpThreads) {      // the W_hh half of [W_ih | W_hh]
      const int r = i / (HP / 8), c = i % (HP / 8);
      const int gate = r / p.units, u = r % p.units;
      uint4 v = make_uint4(zero, zero, zero, zero);
      if (u < nu) v = bf16x8_to_f16x8(reinterpret_cast<const uint4*>(p.w_lstm + (static_cast<size_t>(gate) * HP + u0 + u) * 2 * HP + HP)[c]);
      *reinterpret_cast<uint4*>(s_wlstm + static_cast<size_t>(r) * LS + c * 8) = v;
    }
    for (int i = tid; i < p.rows_p * (HP / 8); i += kSpThreads) {
      const int r = i / (HP / 8), c = i % (HP / 8);
      uint4 v = make_uint4(zero, zero, zero, zero);
      if (r < np) v = bf16x8_to_f16x8(reinterpret_cast<const uint4*>(p.w_pred + static_cast<size_t>(p0 + r) * HP)[c]);
      *reinterpret_cast<uint4*>(s_wpred + static_cast<size_t>(r) * (HP + 8) + c * 8) = v;
    }
    for (int i = tid; i < n_bout; i += kSpThreads) s_bout[i] = i < nj ? p.b_out[j0 + i] : -INFINITY;
    for (int i = tid; i < B * p.units; i += kSpThreads) s_c[i] = 0.f;
    for (int b = tid; b < B; b += kSpThreads) {
      s_t[b] = 0; s_sym[b] = 0; s_n[b] = 0; s_tok[b] = blank; s_len[b] = p.enc_len[b];
      if constexpr (kBoost) s_state[b] = boost_root_of(p, b);
      if constexpr (kLM) { s_lm[b] = p.lm.start_state; s_lslot[b] = -1; }
    }
    if constexpr (kResume) {
      // resume: a started row continues from its record (no SOS step: s_tok = -1), an unstarted one starts as above.  Each CTA
      // loads what it owns -- the cell state and rec of its units, the pred_proj rows of joint.pred it computes -- and every
      // CTA the automaton and LM states.  Out-of-range states count as the row's root / start_state.
      for (int b = tid; b < B; b += kSpThreads) {
        const int32_t* hd = reinterpret_cast<const int32_t*>(p.states + static_cast<size_t>(p.slot[b]) * p.state_bytes);
        if (p.dec_begin != nullptr) s_t[b] = p.dec_begin[b];
        if (hd[0] != 0) {
          s_tok[b] = -1;
          if constexpr (kBoost) s_state[b] = static_cast<unsigned int>(hd[1]) < static_cast<unsigned int>(p.boost_states) ? hd[1] : boost_root_of(p, b);
          if constexpr (kLM) s_lm[b] = static_cast<unsigned int>(hd[2]) < static_cast<unsigned int>(p.lm.n_states) ? hd[2] : p.lm.start_state;
        }
      }
      for (int i = tid; i < B * p.units; i += kSpThreads) {
        const int b = i / p.units, u = i % p.units;
        const uint8_t* r = p.states + static_cast<size_t>(p.slot[b]) * p.state_bytes;
        if (u < nu && reinterpret_cast<const int32_t*>(r)[0] != 0) {
          s_c[i] = reinterpret_cast<const float*>(r + kStateHead)[u0 + u];
          __stcg(reinterpret_cast<float4*>(p.rec + (static_cast<size_t>(b) * HP + u0 + u) * 4),
                 reinterpret_cast<const float4*>(r + kStateHead + HP * 4)[u0 + u]);
        }
      }
      for (int i = tid; i < B * np; i += kSpThreads) {
        const int b = i / np, r = i % np;
        const uint8_t* rc = p.states + static_cast<size_t>(p.slot[b]) * p.state_bytes;
        if (reinterpret_cast<const int32_t*>(rc)[0] != 0)
          __stcg(p.ppbuf + static_cast<size_t>(b) * HJ + p0 + r, reinterpret_cast<const float*>(rc + kStateHead + HP * 20)[p0 + r]);
      }
    }
    if (tid < 12) s_prof[tid] = 0;
  }
  __syncthreads();

  unsigned int target = 0;
  int iter = 0;
  // per-phase cycle counters, kept by thread 0 of CTA 0 in shared memory (in registers they would cost every thread 24)
  auto tick = [&](int slot, long long& t0) { if (cta == 0 && tid == 0) { const long long t1 = clock64(); s_prof[slot] += t1 - t0; t0 = t1; } };
  long long tk = clock64();

  // ------------------------------------------------------------------------------------------------
  // LSTM step + joint.pred for the utterances listed in s_emit[0..n_emit), which emitted token s_tok[b]
  // ------------------------------------------------------------------------------------------------
  // kLM: the LM tile rows of a pass's utterances over the CTA's vocabulary slice, warp e filling the pass's utterance e
  static_assert(kPassUtts == kSpWarps, "one warp per utterance of a pass fills its LM tile row");
  auto lm_fill = [&](int pass) {
    const int ai = grp + kGroups * (pass * kPassUtts + warp);
    if (ai < s_cnt[1]) lm_fill_row(p.lm, s_lm[s_act[ai]], j0, min(j1, p.V), s_lmw + warp * kTileLd, s_lmn + warp * kTileLd, lane);
  };

  auto lstm_and_pred = [&]() {
    const int n_emit = s_cnt[0];
    // kLM: the new LM state of utterance tid's emission, requested now and stored after the elementwise work
    int lm_nx = -1;
    if constexpr (kLM) if (tid < B && s_lslot[tid] >= 0) lm_nx = __ldcg(&p.lm_ring[s_lslot[tid]].x);
    // ---- phase L: gates = rec + gate_tab[token] per (utterance, unit of the CTA) -> cell -> h.  rec = W_hh . h of the
    // utterance's previous step came from this CTA's phase P (zero before the first step, as h is).
    if (nu > 0) {
      for (int i = tid; i < n_emit * nu; i += kSpThreads) {
        const int b = s_emit[i / nu], u = i % nu, unit = u0 + u;
        const float* tr = p.gate_tab + static_cast<size_t>(s_tok[b]) * 4 * HP + unit;
        const float4 r = __ldcg(reinterpret_cast<const float4*>(p.rec + (static_cast<size_t>(b) * HP + unit) * 4));
        float tab[4];
#pragma unroll
        for (int gate = 0; gate < 4; ++gate) tab[gate] = __ldg(tr + gate * HP);
        const float ig = sigmoidf_accurate(r.x + tab[0]), fg = sigmoidf_accurate(r.y + tab[1]);
        const float cg = tanhf(r.z + tab[2]), og = sigmoidf_accurate(r.w + tab[3]);
        const float c2 = fg * s_c[b * p.units + u] + ig * cg;
        s_c[b * p.units + u] = c2;
        __stcg(p.hbuf + static_cast<size_t>(b) * HP + unit, og * tanhf(c2));
      }
    }
    if constexpr (kLM) {
      if (lm_nx >= 0) s_lm[tid] = lm_nx;
      for (int b = tid + kSpThreads; b < B; b += kSpThreads) if (s_lslot[b] >= 0) s_lm[b] = __ldcg(&p.lm_ring[s_lslot[b]].x);
    }
    tick(3, tk);
    if constexpr (kLM) sp_grid_barrier_with(p.counter, target, G, [&] { if (has_j) lm_fill(0); });   // pass 0's LM tile
    else sp_grid_barrier(p.counter, target, G);
    tick(4, tk);
    // ---- phase P: one load of the new h of every emitting utterance feeds both products of the CTA, K split over the
    // warps: its rows_p rows of W_pred (-> ppbuf) and its 4 * units rows of W_hh (-> rec, the recurrent half of the
    // utterance's next step).  Both 16-row tiles of a step (up to 32 emitting utterances) are loaded before the first MMA:
    // one L2 round trip, one reduction.
    if (nu + np > 0) {
      float* red = s_g;                                // [warps][32 utterances][32]: columns 0-23 W_hh rows, 24-31 W_pred rows
      const int kw = (warp + cta) % kSpWarps;          // which k-range this warp takes (rotated per CTA against L2 hot-spotting)
      for (int m0 = 0; m0 < n_emit; m0 += 32) {
        const bool two = m0 + 16 < n_emit;             // block-uniform
        float2 x[2][KSW][4];                           // [tile][k-step][row a lo, row b lo, row a hi, row b hi]
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          if (mt == 1 && !two) break;
          const int ea = m0 + 16 * mt + gid, eb = ea + 8;
          const bool va = ea < n_emit, vb = eb < n_emit;
          const float* h_a = p.hbuf + static_cast<size_t>(va ? s_emit[ea] : 0) * HP;
          const float* h_b = p.hbuf + static_cast<size_t>(vb ? s_emit[eb] : 0) * HP;
#pragma unroll
          for (int i = 0; i < KSW; ++i) {
            const int off = (kw * KSW + i) * 16 + tig * 2;
            x[mt][i][0] = va ? ldcg2(h_a + off) : make_float2(0.f, 0.f); x[mt][i][2] = va ? ldcg2(h_a + off + 8) : make_float2(0.f, 0.f);
            x[mt][i][1] = vb ? ldcg2(h_b + off) : make_float2(0.f, 0.f); x[mt][i][3] = vb ? ldcg2(h_b + off + 8) : make_float2(0.f, 0.f);
          }
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          if (mt == 1 && !two) break;
          float acc[4][4];                               // n8 tiles 0-2: W_hh rows, 3: W_pred rows
#pragma unroll
          for (int n = 0; n < 4; ++n) { acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f; }
#pragma unroll
          for (int i = 0; i < KSW; ++i) {
            const int ks = kw * KSW + i;
            uint32_t ah[4], al[4];
            split2(x[mt][i][0], ah[0], al[0]); split2(x[mt][i][1], ah[1], al[1]);
            split2(x[mt][i][2], ah[2], al[2]); split2(x[mt][i][3], ah[3], al[3]);
#pragma unroll
            for (int n = 0; n < 3; ++n) {
              if (n * 8 < 4 * p.units) {                 // warp-uniform
                // rows beyond the CTA's 4 * units gate rows feed accumulator columns nobody reads: clamped so the fragment load stays
                // inside the array (it used to run on into the reduction buffer, which compute-sanitizer racecheck rightly flags)
                const __nv_bfloat16* wr = s_wlstm + static_cast<size_t>(min(n * 8 + gid, 4 * p.units - 1)) * LS + ks * 16 + tig * 2;
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(wr), b1 = *reinterpret_cast<const uint32_t*>(wr + 8);
                mma_f16_16816(acc[n], ah, b0, b1); mma_f16_16816(acc[n], al, b0, b1);
              }
            }
            const __nv_bfloat16* wr = s_wpred + static_cast<size_t>(min(gid, p.rows_p - 1)) * (HP + 8) + ks * 16 + tig * 2;   // clamped like the LSTM rows
            const uint32_t b0 = *reinterpret_cast<const uint32_t*>(wr), b1 = *reinterpret_cast<const uint32_t*>(wr + 8);
            mma_f16_16816(acc[3], ah, b0, b1); mma_f16_16816(acc[3], al, b0, b1);
          }
#pragma unroll
          for (int n = 0; n < 4; ++n) {
            float* r0 = red + ((warp * 32 + 16 * mt + gid) * 32) + n * 8 + tig * 2;
            r0[0] = acc[n][0]; r0[1] = acc[n][1]; r0[8 * 32] = acc[n][2]; r0[8 * 32 + 1] = acc[n][3];
          }
        }
        __syncthreads();
        // reducers: (utterance, unit) items write the unit's four gate sums, then (utterance, W_pred row) items
        for (int i = tid; i < 32 * (nu + np); i += kSpThreads) {
          if (i < 32 * nu) {
            const int el = i / nu, u = i % nu, e = m0 + el;
            if (e < n_emit) {
              float s[4];
#pragma unroll
              for (int gate = 0; gate < 4; ++gate) {
                s[gate] = 0.f;
#pragma unroll
                for (int w = 0; w < kSpWarps; ++w) s[gate] += red[(w * 32 + el) * 32 + gate * p.units + u];
              }
              __stcg(reinterpret_cast<float4*>(p.rec + (static_cast<size_t>(s_emit[e]) * HP + u0 + u) * 4), make_float4(s[0], s[1], s[2], s[3]));
            }
          } else {
            const int el = (i - 32 * nu) / np, r = (i - 32 * nu) % np, e = m0 + el;
            if (e < n_emit) {
              float s = 0.f;
#pragma unroll
              for (int w = 0; w < kSpWarps; ++w) s += red[(w * 32 + el) * 32 + 24 + r];
              __stcg(p.ppbuf + static_cast<size_t>(s_emit[e]) * HJ + p0 + r, s + __ldg(p.b_pred + p0 + r));
            }
          }
        }
        __syncthreads();
      }
    }
    tick(5, tk);
    sp_grid_barrier(p.counter, target, G);
    tick(6, tk);
  };

  // ordered compaction of the utterances that emitted (s_emit) and of those with frames left (s_act)
  auto compact = [&]() {
    int run_e = 0, run_a = 0;
    for (int base = 0; base < B; base += kSpThreads) {
      const int b = base + tid;
      const bool em = b < B && s_tok[b] >= 0, ac = b < B && s_t[b] < s_len[b];
      const unsigned me = __ballot_sync(0xffffffffu, em), ma = __ballot_sync(0xffffffffu, ac);
      if (lane == 0) { s_cnt[2 + warp] = __popc(me); s_cnt[2 + kSpWarps + warp] = __popc(ma); }
      __syncthreads();
      int bef_e = 0, bef_a = 0, tot_e = 0, tot_a = 0;
#pragma unroll
      for (int w = 0; w < kSpWarps; ++w) {
        const int ce = s_cnt[2 + w], ca = s_cnt[2 + kSpWarps + w];
        if (w < warp) { bef_e += ce; bef_a += ca; }
        tot_e += ce; tot_a += ca;
      }
      const unsigned below = (1u << lane) - 1u;
      if (em) s_emit[run_e + bef_e + __popc(me & below)] = b;
      if (ac) s_act[run_a + bef_a + __popc(ma & below)] = b;
      run_e += tot_e; run_a += tot_a;
      __syncthreads();
    }
    if (tid == 0) { s_cnt[0] = run_e; s_cnt[1] = run_a; }
    __syncthreads();
  };

  // ---- operand rows of a joint pass.  Row r = (utterance r / kFrames of the pass, frame r % kFrames of its window); lane r of
  // every warp holds row r's utterance (-1: none) and frame.  Loader item = (utterance of the pass, float4 column):
  // pred_proj is fetched once for the four frames of a window, and the item order is rotated by the vocabulary-slice
  // index so the CTAs of a group, which all need the same rows, do not ask L2 for the same lines at the same instant.
  int row_b = -1, row_t = 0;
  float4 gv[2][PERU][kFrames];                     // [k-half][item][frame]: enc_proj, then relu(enc_proj + pred_proj)
  auto item_rows = [&](int i, int& c4, int (&rb)[kFrames], int (&rt)[kFrames]) {
    int it = tid + kSpThreads * i;
    const bool in_range = it < ITEMS;
    it = (it + slice * 29) % ITEMS;
    const int ul = it / V4_ROW;
    c4 = it % V4_ROW;
#pragma unroll
    for (int j = 0; j < kFrames; ++j) {
      rb[j] = __shfl_sync(0xffffffffu, row_b, ul * kFrames + j);
      rt[j] = __shfl_sync(0xffffffffu, row_t, ul * kFrames + j);
    }
    return in_range;
  };
  auto enc_row = [&](int h, int b, int t, int c4) {
    return __ldg(reinterpret_cast<const float4*>(p.enc_proj + (static_cast<size_t>(b) * p.T_max + t) * HJ + h * KH) + c4);
  };
  // the rows of a pass and their enc_proj values of k-half 0.  They depend only on the consumed windows and the active
  // list, and enc_proj is read-only during the decode, so pass 0 is requested right after compact(): those loads are in
  // flight during phases L and P.  (Holding k-half 1 across phase P as well would need more than 255 registers.)
  auto fetch_enc = [&](int pass) {
    // the active utterances are dealt round-robin to the groups every iteration (any group can serve any utterance:
    // all hold the full vocabulary), so the groups stay balanced while utterances finish at different times
    const int n_act = s_cnt[1];
    {
      const int e = pass * kPassUtts + lane / kFrames, ai = grp + kGroups * e, j = lane % kFrames;
      const int b = ai < n_act ? s_act[ai] : 0;
      const bool ok = ai < n_act && s_t[b] + j < s_len[b];
      row_b = ok ? b : -1; row_t = ok ? s_t[b] + j : 0;
    }
    if constexpr (kBoost) {
      // bonus rows [a0, min(j1, V)) of the pass's utterances in 16-byte pieces (rows are boost_pitch floats, a multiple of 4;
      // the blank's column is never read); waited for before the argmax epilogue
      const int a0 = j0 & ~3, n4 = (min(j1, p.V) - a0 + 3) >> 2;
      for (int i = tid; i < kPassUtts * n4; i += kSpThreads) {
        const int u = i / n4, c = i % n4, ai = grp + kGroups * (pass * kPassUtts + u);
        if (ai < n_act)
          cp_async16(s_tile + u * kTileLd + 4 * c, p.boost_bonus + static_cast<size_t>(s_state[s_act[ai]]) * p.boost_pitch + a0 + 4 * c);
      }
    }
    if constexpr (kLM) if (pass > 0) lm_fill(pass);   // pass 0's tile is filled under the barrier that ends phase L
#pragma unroll
    for (int i = 0; i < PERU; ++i) {
      int c4, rb[kFrames], rt[kFrames];
      const bool in_range = item_rows(i, c4, rb, rt);
#pragma unroll
      for (int j = 0; j < kFrames; ++j) gv[0][i][j] = in_range && rb[j] >= 0 ? enc_row(0, rb[j], rt[j], c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  // pred_proj rows of both k-halves and the enc_proj values of k-half 1, all requested before the first is used
  // -> relu(enc_proj + pred_proj); rows without a frame stay zero
  auto add_pred = [&]() {
    float4 q4[PERU][2];
    unsigned ok[PERU];                             // bit j: the item's frame j is a row
#pragma unroll
    for (int i = 0; i < PERU; ++i) {
      int c4, rb[kFrames], rt[kFrames];
      const bool in_range = item_rows(i, c4, rb, rt);
      ok[i] = 0u;
#pragma unroll
      for (int j = 0; j < kFrames; ++j) ok[i] |= (in_range && rb[j] >= 0 ? 1u : 0u) << j;
      q4[i][0] = q4[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok[i] & 1u) {
        const float* q = p.ppbuf + static_cast<size_t>(rb[0]) * HJ + 4 * c4;
        q4[i][0] = ldcg4s(q); q4[i][1] = ldcg4s(q + KH);
      }
#pragma unroll
      for (int j = 0; j < kFrames; ++j) gv[1][i][j] = (ok[i] >> j) & 1u ? enc_row(1, rb[j], rt[j], c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < PERU; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int j = 0; j < kFrames; ++j) {
          if ((ok[i] >> j) & 1u) {
            const float4 e4 = gv[h][i][j], q = q4[i][h];
            gv[h][i][j] = make_float4(fmaxf(e4.x + q.x, 0.f), fmaxf(e4.y + q.y, 0.f), fmaxf(e4.z + q.z, 0.f), fmaxf(e4.w + q.w, 0.f));
          }
        }
      }
    }
  };

  compact();                                      // SOS: every unstarted utterance steps once on the blank (zero) embedding
  if (has_j) fetch_enc(0);
  if constexpr (kResume) {
    if (s_cnt[0] > 0) {
      lstm_and_pred();
    } else {                                      // every row resumes (same decision in every CTA): one barrier publishes the loaded ppbuf
      if constexpr (kLM) sp_grid_barrier_with(p.counter, target, G, [&] { if (has_j) lm_fill(0); });
      else sp_grid_barrier(p.counter, target, G);
    }
  } else {
    lstm_and_pred();
  }

  for (;;) {
    // ---- phase J
    if (has_j) {
      const int n_act = s_cnt[1];
      const int n_pass = ((n_act + kGroups - 1) / kGroups + kPassUtts - 1) / kPassUtts;
      for (int pass = 0; pass < n_pass; ++pass) {
        if (pass > 0) fetch_enc(pass);                        // pass 0 was requested when the window was consumed
        const unsigned mask = __ballot_sync(0xffffffffu, row_b >= 0);
        if (mask == 0u) continue;                             // identical in every warp of the CTA
        long long tj = 0;
        if (cta == 0 && tid == 0) tj = clock64();
        auto jtick = [&](int slot) { if (cta == 0 && tid == 0) { const long long t1 = clock64(); s_prof[slot] += t1 - tj; tj = t1; } };
        {
          // ---- wgmma joint: D[vocabulary row, (utterance, frame) row]; warpgroup wgi holds vocabulary rows [64 wgi, +64)
          auto write_planes = [&](int h) {                    // gv[h] -> two IEEE-half planes, 128B-swizzled K-major, 32 rows per slab
#pragma unroll
            for (int i = 0; i < PERU; ++i) {
              int it = tid + kSpThreads * i;
              if (it < ITEMS) {
                it = (it + slice * 29) % ITEMS;
                const int ul = it / V4_ROW, c4 = it % V4_ROW;
                const int kcol = 4 * c4;                      // column inside the k-half
                const uint32_t off_k = static_cast<uint32_t>(kcol >> 6) * kBSlab, chunk = (kcol & 63) >> 3, sub = (kcol & 7) * 2;
#pragma unroll
                for (int j = 0; j < kFrames; ++j) {
                  const int row = ul * kFrames + j;
                  uint32_t h0, l0, h1, l1;
                  split2(make_float2(gv[h][i][j].x, gv[h][i][j].y), h0, l0);
                  split2(make_float2(gv[h][i][j].z, gv[h][i][j].w), h1, l1);
                  uint8_t* dst = gB + off_k + (row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4) + sub;
                  *reinterpret_cast<uint2*>(dst) = make_uint2(h0, h1);
                  *reinterpret_cast<uint2*>(dst + 4096) = make_uint2(l0, l1);       // row + 32 of the same slab
                }
              }
            }
          };
          float dj[32];
          const uint32_t a_rows = static_cast<uint32_t>(warp >> 2) * (64u * 128u);
          auto issue_half = [&](int h) {                      // both warpgroups: NSLAB_H slabs x 4 k16 steps, N = 64 (hi | lo)
            wgmma_fence();
#pragma unroll 1
            for (int sl = 0; sl < NSLAB_H; ++sl) {
              const uint64_t da = wgmma_desc_k_sw128(tc_base + static_cast<uint32_t>(h * NSLAB_H + sl) * a_slab + a_rows);
              const uint64_t db = wgmma_desc_k_sw128(tc_base + b_off + sl * kBSlab);
#pragma unroll
              for (int k = 0; k < 4; ++k)
                wgmma_f16_ss_n64(dj, da + 2u * k, db + 2u * k, (h | sl | k) != 0 ? 1u : 0u);
            }
            wgmma_commit();
          };
          add_pred();
          write_planes(0);
          fence_proxy_async();
          __syncthreads();
          jtick(8);
          issue_half(0);
          wgmma_wait<0>();
          __syncthreads();                                    // half 0 consumed by both warpgroups: the planes may be rewritten
          write_planes(1);
          if constexpr (kBoost) cp_async_wait_all();          // the bonus tile: visible to every thread after the barrier
          fence_proxy_async();
          __syncthreads();
          issue_half(1);
          wgmma_wait<0>();
          jtick(9);
          // ---- argmax over the vocabulary rows per (utterance, frame) column.  A lane holds rows rr and rr + 8 of its warp's
          // 16 and columns 8j + 2t, +1 (j < 4: A . hi, j + 4: A . lo); the eight lanes with the same t cover the warp's rows.
          {
            const int rr = (warp >> 2) * 64 + (warp & 3) * 16 + gid;
            const bool v0 = rr < nj, v1 = rr + 8 < nj;
            const float bias0 = s_bout[rr], bias1 = s_bout[rr + 8];
            // kBoost: column 8j + 2t + e is frame (2t + e) % 4 of the pass's utterance 2j + t / 2, so both e share the bonus of
            // rows rr, rr + 8; the eight values are read up front (blank, row V, gets none)
            float bon[4][2];
            if constexpr (kBoost) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float* tr = s_tile + (2 * j + (tig >> 1)) * kTileLd + (j0 & 3) + rr;
                bon[j][0] = j0 + rr < p.V ? tr[0] : 0.f;
                bon[j][1] = j0 + rr + 8 < p.V ? tr[8] : 0.f;
              }
            }
            if constexpr (kLM) {                              // the LM terms of the same rows, summed with the bonus
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float* tr = s_lmw + (2 * j + (tig >> 1)) * kTileLd + rr;
                const float lm0 = j0 + rr < p.V ? tr[0] : 0.f, lm1 = j0 + rr + 8 < p.V ? tr[8] : 0.f;
                if constexpr (kBoost) { bon[j][0] += lm0; bon[j][1] += lm1; } else { bon[j][0] = lm0; bon[j][1] = lm1; }
              }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float l0 = (dj[4 * j + e] + dj[4 * (j + 4) + e]) + bias0, l1 = (dj[4 * j + 2 + e] + dj[4 * (j + 4) + 2 + e]) + bias1;
                float s0 = l0, s1 = l1;                       // the scores the argmax ranks
                if constexpr (kBoost || kLM) { s0 += bon[j][0]; s1 += bon[j][1]; }
                unsigned long long k0 = v0 ? pack_best(s0, j0 + rr) : 0ull;
                const unsigned long long k1 = v1 ? pack_best(s1, j0 + rr + 8) : 0ull;
                k0 = k1 > k0 ? k1 : k0;                       // higher logit first, ties -> lower row
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) { const unsigned long long ot = __shfl_xor_sync(0xffffffffu, k0, o); k0 = ot > k0 ? ot : k0; }
                if (gid == 0) s_best[(8 * j + 2 * tig + e) * kSpWarps + warp] = k0;
                if constexpr (kLM) {                          // (next LM state, added term) of the warp's best token of the column
                  if (gid == 0) {
                    const int k = static_cast<int>(0xffffffffu - static_cast<unsigned int>(k0 & 0xffffffffull)), u = 2 * j + (tig >> 1);
                    int2 r = make_int2(0, 0);
                    if (static_cast<unsigned int>(k) < static_cast<unsigned int>(p.V)) {   // k0 == 0 (no row): none
                      float add = s_lmw[u * kTileLd + k - j0];
                      if constexpr (kBoost) add = s_tile[u * kTileLd + (j0 & 3) + k - j0] + add;
                      r = make_int2(s_lmn[u * kTileLd + k - j0], __float_as_int(add));
                    }
                    s_lmb[(8 * j + 2 * tig + e) * kSpWarps + warp] = r;
                  }
                }
                if constexpr (kConf) {                        // the same logits and lanes -> the warp's softmax tuple of the column
                  SoftStat c = soft_merge(v0 ? soft_one(l0) : soft_empty(), v1 ? soft_one(l1) : soft_empty(), p.alpha_l2);
#pragma unroll
                  for (int o = 4; o < 32; o <<= 1) c = soft_merge(c, soft_shfl_xor(c, o), p.alpha_l2);
                  if (gid == 0) {
                    float* d = s_conf + ((8 * j + 2 * tig + e) * kSpWarps + warp) * 5;
                    d[0] = c.m; d[1] = c.s; d[2] = c.g; d[3] = c.a; d[4] = c.ga;
                  }
                }
              }
            }
          }
        }
        __syncthreads();
        if (warp == 0 && row_b >= 0) {
          unsigned long long m = s_best[lane * kSpWarps];
#pragma unroll
          for (int q = 1; q < kSpWarps; ++q) { const unsigned long long o = s_best[lane * kSpWarps + q]; m = o > m ? o : m; }
          asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" ::"l"(p.best + (static_cast<size_t>(iter % 3) * B + row_b) * kFrames + (lane % kFrames)), "l"(m) : "memory");
          if constexpr (kLM) {                                // the slice's best token's (next state, term): its own ring slot
            int q = 0;
            while (s_best[lane * kSpWarps + q] != m) ++q;
            __stcg(p.lm_ring + ((static_cast<size_t>(iter % 3) * B + row_b) * kFrames + (lane % kFrames)) * p.S + slice, s_lmb[lane * kSpWarps + q]);
          }
          if constexpr (kConf) {                              // the slice's tuple: a plain store into the slot it owns
            const float* sc = s_conf + lane * kSpWarps * 5;
            SoftStat c = {sc[0], sc[1], sc[2], sc[3], sc[4]};
#pragma unroll
            for (int q = 1; q < kSpWarps; ++q) c = soft_merge(c, {sc[5 * q], sc[5 * q + 1], sc[5 * q + 2], sc[5 * q + 3], sc[5 * q + 4]}, p.alpha_l2);
            float* d = p.conf + ((((static_cast<size_t>(iter % 3) * B + row_b) * kFrames + (lane % kFrames)) * p.S) + slice) * 5;
            __stcg(d, c.m); __stcg(d + 1, c.s); __stcg(d + 2, c.g); __stcg(d + 3, c.a); __stcg(d + 4, c.ga);
          }
        }
        jtick(10);
        // s_best / s_conf / s_g are rewritten only after the next pass's first __syncthreads pair; the reads above are by warp 0
        // before it reaches that barrier
      }
    }
    tick(0, tk);
    sp_grid_barrier(p.counter, target, G);
    tick(1, tk);
    // ---- consume the window (identically in every CTA): blanks advance t, the first non-blank emits and ends the window
    for (int b = tid; b < B; b += kSpThreads) {
      int t = s_t[b];
      const int len = s_len[b];
      int tok = -1, cj = -1, lslot = -1;
      if (t < len) {
        const int nv = min(kFrames, len - t);
        int sym = s_sym[b];
        const ulonglong2* bp = reinterpret_cast<const ulonglong2*>(p.best + (static_cast<size_t>(iter % 3) * B + b) * kFrames);
        static_assert(kFrames == 4, "window read as two 16-byte loads");
        const ulonglong2 w01 = __ldcg(bp), w23 = __ldcg(bp + 1);
        const unsigned long long win[kFrames] = {w01.x, w01.y, w23.x, w23.y};
#pragma unroll
        for (int j = 0; j < kFrames; ++j) {
          if (j >= nv) break;
          const unsigned long long v = win[j];
          const int k = static_cast<int>(0xffffffffu - static_cast<unsigned int>(v & 0xffffffffull));
          if (k == blank) { t += 1; sym = 0; continue; }
          const int n = s_n[b];
          if (cta == 0 && n < p.U_max) {
            p.tokens[static_cast<size_t>(b) * p.U_max + n] = k;
            p.frames[static_cast<size_t>(b) * p.U_max + n] = t;
          }
          if (kConf && n < p.U_max) cj = j;
          if constexpr (kBoost) {
            const size_t at = static_cast<size_t>(s_state[b]) * p.boost_pitch + k;
            const int nx = __ldg(p.boost_next + at);
            if constexpr (kConf && !kLM) if (n < p.U_max) s_le[b] = best_value(v) - __ldg(p.boost_bonus + at);
            s_state[b] = static_cast<unsigned int>(nx) < static_cast<unsigned int>(p.boost_states) ? nx : boost_root_of(p, b);
          }
          if constexpr (kLM) {                                // the ring slot of k's slice; read in phase L (the new state)
            lslot = static_cast<int>(((static_cast<size_t>(iter % 3) * B + b) * kFrames + j) * p.S + k / p.rows_j);
            if constexpr (kConf) if (n < p.U_max) s_le[b] = best_value(v);   // fused; the term comes from the ring
          }
          s_n[b] = n + 1;
          tok = k;
          if (++sym >= p.max_symbols) { t += 1; sym = 0; }
          break;
        }
        s_t[b] = t; s_sym[b] = sym;
      }
      s_tok[b] = tok;
      if constexpr (kConf) s_cj[b] = cj;
      if constexpr (kLM) s_lslot[b] = lslot;
    }
    // the slot that iteration iter+2 will use was last read two barriers ago: clear it now (visible through the
    // next barrier, which precedes that iteration's red.max)
    if (cta == 0) for (int i = tid; i < B * kFrames; i += kSpThreads) __stcg(p.best + static_cast<size_t>((iter + 2) % 3) * B * kFrames + i, 0ull);
    ++iter;
    __syncthreads();
    compact();
    const int n_active = s_cnt[1];
    tick(2, tk);
    if (cta == 0 && tid == 0) s_prof[7] += 1;
    if (has_j) fetch_enc(0);                      // the next window's enc_proj rows, in flight under phases L and P
    if constexpr (kConf) {
      // statistics of the emissions just consumed: emission e (in s_emit order) is merged by warp e / G of CTA e % G, lane
      // i taking slices i, i + 32, ...; the slot was written before the barrier that preceded the consume step
      const int n_emit = s_cnt[0], slot = (iter + 2) % 3;
      for (int e = cta + G * warp; e < n_emit; e += G * kSpWarps) {
        const int b = s_emit[e], j = s_cj[b];
        if (j < 0) continue;                                  // beyond U_max: nothing is stored
        const float* src = p.conf + ((static_cast<size_t>(slot) * B + b) * kFrames + j) * p.S * 5;
        SoftStat c = soft_empty();
        for (int s = lane; s < p.S; s += 32)
          c = soft_merge(c, {__ldcg(src + 5 * s), __ldcg(src + 5 * s + 1), __ldcg(src + 5 * s + 2), __ldcg(src + 5 * s + 3), __ldcg(src + 5 * s + 4)}, p.alpha_l2);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c = soft_merge(c, soft_shfl_xor(c, o), p.alpha_l2);
        if (lane == 0) {                                      // c is relative to the maximum logit m: log p = (l - m) - log s
          const float log_s = logf(c.s), inv_s = 1.f / c.s, s_ma = expf(-p.alpha * log_s), a_alpha = s_ma * c.a;
          float lp = kBoost ? (s_le[b] - c.m) - log_s : -log_s;   // unboosted, the emitted token is the maximum
          if constexpr (kLM) lp = ((s_le[b] - __int_as_float(__ldcg(&p.lm_ring[s_lslot[b]].y))) - c.m) - log_s;   // unfused
          const float4 st = make_float4(lp, c.g * inv_s - log_s, a_alpha, s_ma * c.ga - log_s * a_alpha);
          __stcg(reinterpret_cast<float4*>(p.stats + (static_cast<size_t>(b) * p.U_max + (s_n[b] - 1)) * 4), st);
        }
      }
    }
    if (s_cnt[0] > 0) lstm_and_pred();
    if constexpr (kLM) if (s_cnt[0] == 0 && has_j) lm_fill(0);   // no emission: the states stand, the pass's rows may not
    if (n_active == 0) break;
  }
  if (cta == 0) for (int b = tid; b < B; b += kSpThreads) p.n_tok[b] = s_n[b];
  if (cta == 0 && tid == 0) for (int i = 0; i < 12; ++i) p.prof[i] = s_prof[i];
  if constexpr (kResume) {
    // store back what this CTA owns.  The last lstm_and_pred ran for the last emissions, so the record holds the state after
    // the last token's step; rec / ppbuf of the CTA's units / rows were written by this CTA (before the barrier that ended it).
    for (int i = tid; i < B * p.units; i += kSpThreads) {
      const int b = i / p.units, u = i % p.units;
      uint8_t* r = p.states + static_cast<size_t>(p.slot[b]) * p.state_bytes;
      if (u < nu) {
        reinterpret_cast<float*>(r + kStateHead)[u0 + u] = s_c[i];
        reinterpret_cast<float4*>(r + kStateHead + HP * 4)[u0 + u] = __ldcg(reinterpret_cast<const float4*>(p.rec + (static_cast<size_t>(b) * HP + u0 + u) * 4));
      }
    }
    for (int i = tid; i < B * np; i += kSpThreads) {
      const int b = i / np, r = i % np;
      uint8_t* rc = p.states + static_cast<size_t>(p.slot[b]) * p.state_bytes;
      reinterpret_cast<float*>(rc + kStateHead + HP * 20)[p0 + r] = __ldcg(p.ppbuf + static_cast<size_t>(b) * HJ + p0 + r);
    }
    if (cta == 0) {                               // every CTA read the headers before the first grid barrier
      for (int b = tid; b < B; b += kSpThreads) {
        int32_t* hd = reinterpret_cast<int32_t*>(p.states + static_cast<size_t>(p.slot[b]) * p.state_bytes);
        hd[0] = 1;
        if constexpr (kBoost) hd[1] = s_state[b];
        if constexpr (kLM) hd[2] = s_lm[b];
      }
    }
  }
}

template <int HJ, int HP, bool kConf, bool kBoost, bool kLM>
__global__ void __launch_bounds__(kSpThreads, 1)
rnnt_greedy_spec_kernel(const SpecDev p) { greedy_spec_body<HJ, HP, kConf, kBoost, kLM, false>(p); }

// the resumed decode: its own instances, so that the offline ones compile from unchanged code (same registers, same results)
template <int HJ, int HP, bool kConf, bool kBoost, bool kLM>
__global__ void __launch_bounds__(kSpThreads, 1)
rnnt_greedy_resume_kernel(const SpecDev p) { greedy_spec_body<HJ, HP, kConf, kBoost, kLM, true>(p); }

// workspace (SpecDev's global buffers): hbuf | rec | ppbuf | barrier counters (kBarCounters 128-byte lines) | prof | best | conf |
// lm_ring.  Everything before conf is zeroed by the launch; every conf / lm_ring slot that is read was written first.
SpecWorkspace rnnt_spec_workspace(int B, int Hj, int Hp, int num_sms) {
  Arena a;
  SpecWorkspace w;
  w.hbuf = a.take(static_cast<size_t>(B) * Hp * 4);
  w.rec = a.take(static_cast<size_t>(B) * Hp * 4 * 4);
  w.ppbuf = a.take(static_cast<size_t>(B) * Hj * 4);
  w.counters = a.take(static_cast<size_t>(kBarCounters) * kBarStride * 4);
  w.prof = a.take(12 * 8);
  w.best = a.take(static_cast<size_t>(3) * B * kFrames * 8);
  w.conf = a.take(static_cast<size_t>(3) * B * kFrames * (num_sms / kGroups) * 5 * 4);
  w.lm_ring = a.take(static_cast<size_t>(3) * B * kFrames * (num_sms / kGroups) * 8);
  w.total = a.off;
  return w;
}

template <int HJ, int HP, bool kConf, bool kBoost, bool kLM>
static cudaError_t launch_sp(SpecDev p, int grid, size_t smem, cudaStream_t stream) {
  const auto kernel = p.states != nullptr ? rnnt_greedy_resume_kernel<HJ, HP, kConf, kBoost, kLM> : rnnt_greedy_spec_kernel<HJ, HP, kConf, kBoost, kLM>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kSpThreads, smem);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) return cudaErrorLaunchOutOfResources;
  void* args[] = {&p};
  return cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kernel), dim3(grid), dim3(kSpThreads), args, smem, stream);
}

template <int HJ, int HP, bool kLM>
static cudaError_t launch_sp(SpecDev p, int grid, size_t smem, cudaStream_t stream) {
  if (p.boost_bonus != nullptr)
    return p.stats != nullptr ? launch_sp<HJ, HP, true, true, kLM>(p, grid, smem, stream) : launch_sp<HJ, HP, false, true, kLM>(p, grid, smem, stream);
  return p.stats != nullptr ? launch_sp<HJ, HP, true, false, kLM>(p, grid, smem, stream) : launch_sp<HJ, HP, false, false, kLM>(p, grid, smem, stream);
}

template <int HJ, int HP>
static cudaError_t launch_sp(SpecDev p, int grid, size_t smem, cudaStream_t stream) {
  return p.lm.order != 0 ? launch_sp<HJ, HP, true>(p, grid, smem, stream) : launch_sp<HJ, HP, false>(p, grid, smem, stream);
}

// The LM table contract the kernels rely on (rs_set_ngram_lm checks the same before it accepts a table)
static bool lm_tables_ok(const NgramLM& lm, int V) {
  const uintptr_t ptrs = reinterpret_cast<uintptr_t>(lm.cb) | reinterpret_cast<uintptr_t>(lm.chain) | reinterpret_cast<uintptr_t>(lm.arc_begin) |
                         reinterpret_cast<uintptr_t>(lm.arc_tok) | reinterpret_cast<uintptr_t>(lm.arc_to) | reinterpret_cast<uintptr_t>(lm.arc_w) |
                         reinterpret_cast<uintptr_t>(lm.uni_w) | reinterpret_cast<uintptr_t>(lm.uni_to);
  return lm.order >= 2 && lm.order <= kMaxLmCtx + 1 && lm.n_states >= 1 && lm.n_arcs >= 0 && lm.pitch >= V && lm.pitch % 4 == 0 &&
         lm.start_state >= 0 && lm.start_state < lm.n_states && lm.cb && lm.chain && lm.arc_begin && lm.arc_tok && lm.arc_to && lm.arc_w &&
         lm.uni_w && lm.uni_to && (ptrs & 15u) == 0;
}

cudaError_t launch_rnnt_greedy_spec(const DecodeArgs& a, void* workspace, int num_sms, cudaStream_t stream) {
  if (a.B <= 0 || num_sms < kGroups) return cudaErrorInvalidValue;
  const int G = num_sms;
  SpecDev p;
  p.enc_proj = a.enc_proj; p.enc_len = a.enc_len;
  p.w_out = static_cast<const __nv_bfloat16*>(a.w_out); p.b_out = a.b_out;
  p.w_lstm = static_cast<const __nv_bfloat16*>(a.w_lstm); p.gate_tab = a.gate_tab;
  p.w_pred = static_cast<const __nv_bfloat16*>(a.w_pred); p.b_pred = a.b_pred;
  p.tokens = a.tokens; p.frames = a.frames; p.n_tok = a.n_tok;
  if (reinterpret_cast<uintptr_t>(workspace) & 15u) return cudaErrorInvalidValue;   // the window is read with 16-byte loads
  char* ws = static_cast<char*>(workspace);
  const SpecWorkspace w = rnnt_spec_workspace(a.B, a.Hj, a.Hp, num_sms);
  p.hbuf = reinterpret_cast<float*>(ws + w.hbuf);
  p.rec = reinterpret_cast<float*>(ws + w.rec);
  p.ppbuf = reinterpret_cast<float*>(ws + w.ppbuf);
  p.counter = reinterpret_cast<unsigned int*>(ws + w.counters);
  p.prof = reinterpret_cast<long long*>(ws + w.prof);
  p.best = reinterpret_cast<unsigned long long*>(ws + w.best);
  p.conf = reinterpret_cast<float*>(ws + w.conf);
  p.stats = a.stats;
  if (a.stats != nullptr && !(a.alpha > 0.f && a.alpha < INFINITY)) return cudaErrorInvalidValue;
  p.alpha = a.alpha; p.alpha_l2 = a.alpha * kLog2e;
  p.boost_bonus = a.boost_bonus; p.boost_next = a.boost_next; p.boost_states = a.boost_states; p.boost_pitch = a.boost_pitch;
  p.boost_root = a.boost_root;
  const bool boost = a.boost_bonus != nullptr;
  if (boost && (a.boost_next == nullptr || a.boost_states < 1 || a.boost_pitch < a.V || (a.boost_pitch & 3) ||
                ((reinterpret_cast<uintptr_t>(a.boost_bonus) | reinterpret_cast<uintptr_t>(a.boost_next)) & 15u)))
    return cudaErrorInvalidValue;                                  // the tile is copied in 16-byte pieces
  p.lm = a.lm;
  const bool lm = a.lm.order != 0;
  if (lm && !lm_tables_ok(a.lm, a.V)) return cudaErrorInvalidValue;
  p.lm_ring = reinterpret_cast<int2*>(ws + w.lm_ring);
  p.dec_begin = a.dec_begin; p.slot = a.slot; p.states = static_cast<uint8_t*>(a.states);
  p.state_bytes = static_cast<int>(stream_state_bytes(a.Hj, a.Hp));
  if (a.states != nullptr && (a.slot == nullptr || (reinterpret_cast<uintptr_t>(a.states) & 15u))) return cudaErrorInvalidValue;
  p.B = a.B; p.T_max = a.T_max; p.V = a.V; p.U_max = a.U_max; p.max_symbols = a.max_symbols;
  p.S = G / kGroups;
  p.rows_j = (a.V + 1 + p.S - 1) / p.S;
  p.units = (a.Hp + G - 1) / G;
  p.rows_p = (a.Hj + G - 1) / G;
  if (4 * p.units > 24 || p.rows_p > 8 || a.gate_tab == nullptr) return cudaErrorInvalidValue;   // the n8 tiles of phase P
  cudaError_t e = cudaMemsetAsync(workspace, 0, w.conf, stream);
  if (e != cudaSuccess) return e;
  const size_t state = ((static_cast<size_t>(a.B) * p.units + 1) & ~static_cast<size_t>(1)) * 4 + (kPassRows * kSpWarps + 12) * 8 + static_cast<size_t>(a.B) * 7 * 4 +
                       (2 + 2 * kSpWarps) * 4 + 64 +
                       (a.stats != nullptr ? static_cast<size_t>(a.B) * 4 + kPassRows * kSpWarps * 5 * 4 : 0) +   // kConf: s_cj, s_conf
                       (boost && !lm ? 16 + kPassUtts * kTileLd * 4 + static_cast<size_t>(a.B) * 4 * (a.stats != nullptr ? 2 : 1) : 0) +   // kBoost: align, s_tile, s_state (, s_le)
                       (lm ? 16 + kPassUtts * kTileLd * 4 + static_cast<size_t>(a.B) * 8 +                 // kLM: the kBoost arrays,
                             2 * kPassUtts * kTileLd * 4 + 8 + kPassRows * kSpWarps * 8 + static_cast<size_t>(a.B) * 8 : 0);   // s_lmw, s_lmn, s_lmb, s_lm, s_lslot
  const size_t w_lp = (static_cast<size_t>(4 * p.units) * (a.Hp + 8) + static_cast<size_t>(p.rows_p) * (a.Hp + 8)) * 2;
  if (p.rows_j > 128) return cudaErrorInvalidValue;                // also the LM tile / lm_fill_row's slice bound
  const size_t rows_a8 = (p.rows_j + 7) & ~7;
  const size_t b_bytes = static_cast<size_t>(a.Hj / 2 / 64) * 8192;
  const size_t b_region = b_bytes > 32768 ? b_bytes : 32768;     // also the [8 warps][32][32] fp32 reduction buffer of phase P
  const size_t ab = ((static_cast<size_t>(a.Hj / 64) * rows_a8 * 128 + w_lp + 1023) & ~static_cast<size_t>(1023));   // A slabs, W_lstm, W_pred, pad
  const size_t smem = 1024 + ab + b_region + 128 * 4 + state + 16;
  if (smem > 227 * 1024) return cudaErrorInvalidValue;
  if (a.Hj == 640 && a.Hp == 640) return launch_sp<640, 640>(p, G, smem, stream);
  if (a.Hj == 128 && a.Hp == 128) return launch_sp<128, 128>(p, G, smem, stream);
  return cudaErrorInvalidValue;
}

// rs_ngram_lm_eval: one warp per (state, token) pair runs lm_fill_row over the slice the decode gives the token (S = num_sms /
// kGroups slices of rows_j columns) and reads the token's term and next state, as the decode's epilogue and ring do
__global__ void __launch_bounds__(kSpThreads) ngram_lm_eval_kernel(const NgramLM lm, int V, int rows_j, const int32_t* states,
                                                                   const int32_t* tokens, int n, float* score, int32_t* next) {
  __shared__ float s_w[kSpWarps][kTileLd];
  __shared__ int s_n[kSpWarps][kTileLd];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = blockIdx.x * kSpWarps + warp; i < n; i += gridDim.x * kSpWarps) {
    const int k = tokens[i];
    if (static_cast<unsigned int>(k) >= static_cast<unsigned int>(V)) {
      if (lane == 0) { score[i] = __int_as_float(0x7fc00000); next[i] = -1; }
      continue;
    }
    const int j0 = (k / rows_j) * rows_j;
    lm_fill_row(lm, states[i], j0, min(j0 + rows_j, V), s_w[warp], s_n[warp], lane);
    __syncwarp();
    if (lane == 0) { score[i] = s_w[warp][k - j0]; next[i] = s_n[warp][k - j0]; }
    __syncwarp();
  }
}

cudaError_t launch_ngram_lm_eval(const NgramLM& lm, int V, int num_sms, const int32_t* states, const int32_t* tokens, int n,
                                 float* score, int32_t* next, cudaStream_t stream) {
  if (n < 0 || num_sms < kGroups || !lm_tables_ok(lm, V)) return cudaErrorInvalidValue;
  if (n == 0) return cudaSuccess;
  const int S = num_sms / kGroups, rows_j = (V + 1 + S - 1) / S;
  if (rows_j > 128) return cudaErrorInvalidValue;
  const int grid = min((n + kSpWarps - 1) / kSpWarps, 4096);
  ngram_lm_eval_kernel<<<grid, kSpThreads, 0, stream>>>(lm, V, rows_j, states, tokens, n, score, next);
  return cudaGetLastError();
}

}  // namespace rs
