// Forced alignment of known label sequences on the standard RNN-T lattice (semantics: reazonspeech_b200/alignment.py).
//
//   align_lstm_step_kernel   teacher-forced predictor, one launch per label position u: every utterance's LSTM input is
//                            known in advance (blank = the zero embedding at u = 0, then y_u), so step u's gates are
//                            pred.gate_tab[y_u] + W_hh . h_{u-1}; one warp per (utterance, unit), fp32 SIMT
//   align_pred_proj_kernel   pred_proj[b][u] = joint.pred(h_u) for all B * (U_max + 1) rows
//   rnnt_lattice_kernel      log softmax of the joint at every (t, u) cell of every utterance -> lp_blank, lp_emit (wgmma)
//   rnnt_align_dp_kernel     forward (logaddexp) and Viterbi (max) recursions over the anti-diagonals + backtrace
//
// The lattice kernel.  A CTA owns a tile of 128 cells of one utterance, 16 frames x 8 labels; row r of the tile is cell
// (t0 + r / 8, u0 + r % 8).  The 24 fp32 source rows (16 enc_proj + 8 pred_proj) stay in shared memory for the whole tile,
// and the A operand is generated in registers one k16 step at a time: relu(enc_proj[t] + pred_proj[u]) split into two
// IEEE-half terms hi + lo (22 mantissa bits, as the greedy decode's joint), fed to wgmma straight from registers.  The
// activation never exists anywhere else.  W_out (L2-resident) streams through a ring of 64-column k-chunks of 128 rows
// loaded by TMA as bf16 and converted in place to half (exact: bf16 weights are exact in half), each chunk used by both
// terms.  Each warpgroup holds 64 rows x 128 vocabulary columns of fp32 accumulators per N-tile; the epilogue adds b_out,
// folds the tile into a running (max, sum) per row (an online log-sum-exp on exp2f) and picks up the blank column and the
// row's own target column y_{u+1}.  After the last N-tile the cell's log-probabilities are written.
#include <cmath>
#include <cstdio>

#include "common.cuh"
#include "kernels.h"

namespace rs {

namespace {

constexpr int kLatThreads = 256;        // two consumer warpgroups, 64 rows each
constexpr int kTileT = 16, kTileU = 8;  // 128 cells per tile
constexpr int kBN = 128;                // vocabulary columns per N-tile
constexpr int kBK = 64;                 // k-chunk: one 128-byte swizzle row of halves
constexpr int kStages = 4;
constexpr uint32_t kStageBytes = kBN * kBK * 2;
constexpr float kL2e = 1.4426950408889634f;

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, f16 inputs, fp32 accumulate; A from registers (mma.sync m16k16 fragment layout)
__device__ __forceinline__ void wgmma_f16_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

// Valid label count of utterance b: label_len clamped to [0, U_max] (an out-of-range length is reported by the DP kernel)
__device__ __forceinline__ int utt_labels(const AlignArgs& a, int b) { return min(max(a.label_len[b], 0), a.U_max); }

__global__ void __launch_bounds__(256) align_lstm_step_kernel(const AlignArgs a, int u) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = blockIdx.x * 8 + warp;
  if (w >= a.B * a.Hp) return;
  const int b = w / a.Hp, j = w % a.Hp, Hp = a.Hp;
  if (u > utt_labels(a, b)) return;
  int tok = a.V;                                               // u = 0: the blank / SOS input (zero embedding)
  if (u > 0) {
    tok = a.labels[static_cast<size_t>(b) * a.U_max + u - 1];
    if (tok < 0 || tok >= a.V) tok = a.V;                      // the utterance's scores become NaN; keep the reads in bounds
  }
  const size_t row = static_cast<size_t>(b) * (a.U_max + 1) + u;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (u > 0) {
    const float* hp = a.h + (row - 1) * Hp;
    for (int k = 2 * lane; k < Hp; k += 64) {
      const float2 hv = *reinterpret_cast<const float2*>(hp + k);
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const float2 wv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(static_cast<const __nv_bfloat16*>(a.w_lstm) + (static_cast<size_t>(g) * Hp + j) * 2 * Hp + Hp + k));
        acc[g] = fmaf(wv.x, hv.x, fmaf(wv.y, hv.y, acc[g]));
      }
    }
  }
#pragma unroll
  for (int g = 0; g < 4; ++g) acc[g] = warp_sum(acc[g]);
  if (lane == 0) {
    const float* tr = a.gate_tab + static_cast<size_t>(tok) * 4 * Hp + j;
    const float ig = sigmoidf_accurate(acc[0] + tr[0]), fg = sigmoidf_accurate(acc[1] + tr[Hp]);
    const float cg = tanhf(acc[2] + tr[2 * Hp]), og = sigmoidf_accurate(acc[3] + tr[3 * Hp]);
    float* cp = a.c + static_cast<size_t>(b) * Hp + j;
    const float c2 = fg * (u > 0 ? *cp : 0.f) + ig * cg;
    *cp = c2;
    a.h[row * Hp + j] = og * tanhf(c2);
  }
}

// 8 rows of h per CTA (in shared memory); warp w computes outputs w, w + 8, ... with the lanes over k
constexpr int kPpRows = 8;
__global__ void __launch_bounds__(256) align_pred_proj_kernel(const AlignArgs a) {
  extern __shared__ __align__(16) float s_h[];                  // [kPpRows][Hp]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, Hp = a.Hp, Hj = a.Hj, U1 = a.U_max + 1;
  const int n_rows = a.B * U1, r0 = blockIdx.x * kPpRows;
  bool ok[kPpRows];
#pragma unroll
  for (int i = 0; i < kPpRows; ++i) {
    const int r = r0 + i;
    ok[i] = r < n_rows && r % U1 <= utt_labels(a, r / U1);
  }
  for (int i = threadIdx.x; i < kPpRows * Hp; i += blockDim.x) {
    const int rr = i / Hp;
    s_h[i] = ok[rr] ? a.h[static_cast<size_t>(r0 + rr) * Hp + i % Hp] : 0.f;
  }
  __syncthreads();
  for (int o = warp; o < Hj; o += 8) {
    float acc[kPpRows];
#pragma unroll
    for (int i = 0; i < kPpRows; ++i) acc[i] = 0.f;
    const __nv_bfloat16* wr = static_cast<const __nv_bfloat16*>(a.w_pred) + static_cast<size_t>(o) * Hp;
    for (int k = 2 * lane; k < Hp; k += 64) {
      const float2 wv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(wr + k));
#pragma unroll
      for (int i = 0; i < kPpRows; ++i) {
        const float2 hv = *reinterpret_cast<const float2*>(s_h + i * Hp + k);
        acc[i] = fmaf(wv.x, hv.x, fmaf(wv.y, hv.y, acc[i]));
      }
    }
    const float bias = a.b_pred[o];
#pragma unroll
    for (int i = 0; i < kPpRows; ++i) {
      const float s = warp_sum(acc[i]);
      if (lane == 0 && ok[i]) a.pred_proj[static_cast<size_t>(r0 + i) * Hj + o] = s + bias;
    }
  }
}

__global__ void __launch_bounds__(kLatThreads, 1)
rnnt_lattice_kernel(const __grid_constant__ CUtensorMap tm_w, const AlignArgs a) {
  extern __shared__ __align__(16) uint8_t ssm[];
  const int Hj = a.Hj, NC = a.V + 1, LDS = Hj + 8;
  const int tiles_t = (a.T_max + kTileT - 1) / kTileT, tiles_u = (a.U_max + 1 + kTileU - 1) / kTileU;
  const int b = blockIdx.x / (tiles_t * tiles_u), rem = blockIdx.x % (tiles_t * tiles_u);
  const int t0 = (rem / tiles_u) * kTileT, u0 = (rem % tiles_u) * kTileU;
  const int Tb = min(max(a.enc_len[b], 0), a.T_max), Ub = utt_labels(a, b);
  if (t0 >= Tb || u0 > Ub || a.label_len[b] < 0 || a.label_len[b] > a.U_max) return;   // no valid cell: nothing to write

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3, wg = warp >> 2;
  // ---- shared memory: [stages (1024-aligned) | enc rows | pred rows | b_out | targets | mbarriers]
  const uint32_t base = (smem_u32(ssm) + 1023u) & ~1023u;
  uint8_t* gbase = ssm + (base - smem_u32(ssm));
  const int n_tiles = (NC + kBN - 1) / kBN, KC = Hj / kBK, total = n_tiles * KC;
  float* s_enc = reinterpret_cast<float*>(gbase + kStages * kStageBytes);   // [16][LDS]
  float* s_pred = s_enc + kTileT * LDS;                                     // [8][LDS]
  float* s_bias = s_pred + kTileU * LDS;                                    // [n_tiles * 128], -inf beyond NC
  int* s_tgt = reinterpret_cast<int*>(s_bias + n_tiles * kBN);              // [8] target class of row u % 8, -1: none
  uint64_t* s_full = reinterpret_cast<uint64_t*>(s_tgt + kTileU);
  const uint32_t full0 = smem_u32(s_full);

  if (tid == 0) {
    tma_prefetch_desc(&tm_w);
    for (int s = 0; s < kStages; ++s) mbar_init(full0 + 8 * s, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    for (int c = 0; c < kStages && c < total; ++c) {
      mbar_arrive_expect_tx(full0 + 8 * c, kStageBytes);
      tma_load_2d(base + c * kStageBytes, &tm_w, (c % KC) * kBK, (c / KC) * kBN, full0 + 8 * c);
    }
  }
  // source rows (rows outside the utterance are zero; their cells are never written)
  for (int i = tid; i < (kTileT + kTileU) * (Hj / 4); i += kLatThreads) {
    const int r = i / (Hj / 4), c4 = i % (Hj / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < kTileT) {
      if (t0 + r < Tb) v = reinterpret_cast<const float4*>(a.enc_proj + (static_cast<size_t>(b) * a.T_max + t0 + r) * Hj)[c4];
      *reinterpret_cast<float4*>(s_enc + r * LDS + 4 * c4) = v;
    } else {
      const int u = u0 + r - kTileT;
      if (u <= Ub) v = reinterpret_cast<const float4*>(a.pred_proj + (static_cast<size_t>(b) * (a.U_max + 1) + u) * Hj)[c4];
      *reinterpret_cast<float4*>(s_pred + (r - kTileT) * LDS + 4 * c4) = v;
    }
  }
  for (int i = tid; i < n_tiles * kBN; i += kLatThreads) s_bias[i] = i < NC ? a.b_out[i] : -INFINITY;
  if (tid < kTileU) {
    const int u = u0 + tid;
    s_tgt[tid] = u < Ub ? a.labels[static_cast<size_t>(b) * a.U_max + u] : -1;
  }
  __syncthreads();

  // this thread's rows: r = 64 wg + 16 (warp % 4) + g (+ 8) -> frames t0 + r / 8, both at label u0 + g
  const int tA = 8 * wg + 2 * (warp & 3), tB = tA + 1;
  const float* pe0 = s_enc + tA * LDS + 2 * tq;
  const float* pe1 = s_enc + tB * LDS + 2 * tq;
  const float* pq = s_pred + g * LDS + 2 * tq;
  const int tgt = s_tgt[g];
  float m[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f}, lb[2] = {-INFINITY, -INFINITY}, le[2] = {-INFINITY, -INFINITY};
  float acc[64];

  for (int n = 0; n < n_tiles; ++n) {
    for (int kc = 0; kc < KC; ++kc) {
      const int c = n * KC + kc, s = c % kStages;
      const uint32_t stage = base + s * kStageBytes;
      mbar_wait(full0 + 8 * s, (c / kStages) & 1);
      {   // bf16 -> half in place (the 128-byte swizzle is a permutation of 16-byte chunks: unaffected)
        uint4* st = reinterpret_cast<uint4*>(gbase + s * kStageBytes);
#pragma unroll
        for (int i = 0; i < static_cast<int>(kStageBytes / 16) / kLatThreads; ++i) st[tid + i * kLatThreads] = bf16x8_to_f16x8(st[tid + i * kLatThreads]);
      }
      fence_proxy_async();
      __syncthreads();
      const uint64_t db = wgmma_desc_k_sw128(stage);
      uint32_t hi[4][4], lo[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int k = kc * kBK + ks * 16;
        const float2 ea = *reinterpret_cast<const float2*>(pe0 + k), eb = *reinterpret_cast<const float2*>(pe0 + k + 8);
        const float2 fa = *reinterpret_cast<const float2*>(pe1 + k), fb = *reinterpret_cast<const float2*>(pe1 + k + 8);
        const float2 qa = *reinterpret_cast<const float2*>(pq + k), qb = *reinterpret_cast<const float2*>(pq + k + 8);
        split2(make_float2(fmaxf(ea.x + qa.x, 0.f), fmaxf(ea.y + qa.y, 0.f)), hi[ks][0], lo[ks][0]);
        split2(make_float2(fmaxf(fa.x + qa.x, 0.f), fmaxf(fa.y + qa.y, 0.f)), hi[ks][1], lo[ks][1]);
        split2(make_float2(fmaxf(eb.x + qb.x, 0.f), fmaxf(eb.y + qb.y, 0.f)), hi[ks][2], lo[ks][2]);
        split2(make_float2(fmaxf(fb.x + qb.x, 0.f), fmaxf(fb.y + qb.y, 0.f)), hi[ks][3], lo[ks][3]);
      }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        wgmma_f16_rs_n128(acc, hi[ks], db + 2u * ks, (kc | ks) != 0 ? 1u : 0u);
        wgmma_f16_rs_n128(acc, lo[ks], db + 2u * ks, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncthreads();                                   // both warpgroups are done with the stage
      if (tid == 0 && c + kStages < total) {
        const int cn = c + kStages;
        mbar_arrive_expect_tx(full0 + 8 * s, kStageBytes);
        tma_load_2d(stage, &tm_w, (cn % KC) * kBK, (cn / KC) * kBN, full0 + 8 * s);
      }
    }
    // ---- epilogue of the N-tile: d[4j + e] = (row g, column 8j + 2tq + e), d[4j + 2 + e] = (row g + 8, same column)
    const int n0 = n * kBN;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = n0 + 8 * j + 2 * tq + e;
        const float bias = s_bias[col];                  // -inf beyond the classes
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float l = acc[4 * j + 2 * h + e] + bias;
          acc[4 * j + 2 * h + e] = l;
          mx[h] = fmaxf(mx[h], l);
          if (col == a.V) lb[h] = l;
          if (col == tgt) le[h] = l;
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float nm = fmaxf(m[h], mx[h]), nml = nm * kL2e;
      float sh = sum[h] * exp2f(fmaf(m[h], kL2e, -nml));
#pragma unroll
      for (int j = 0; j < 16; ++j) sh += exp2f(fmaf(acc[4 * j + 2 * h], kL2e, -nml)) + exp2f(fmaf(acc[4 * j + 2 * h + 1], kL2e, -nml));
      sum[h] = sh;
      m[h] = nm;
    }
  }
  // ---- the cells: lse = m + log(sum over the quad); lp = logit - lse
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float s = sum[h];
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    float vb = lb[h], ve = le[h];
    vb = fmaxf(vb, __shfl_xor_sync(0xffffffffu, vb, 1)); vb = fmaxf(vb, __shfl_xor_sync(0xffffffffu, vb, 2));
    ve = fmaxf(ve, __shfl_xor_sync(0xffffffffu, ve, 1)); ve = fmaxf(ve, __shfl_xor_sync(0xffffffffu, ve, 2));
    const int t = t0 + (h == 0 ? tA : tB), u = u0 + g;
    if (tq == 0 && t < Tb && u <= Ub) {
      const float lse = m[h] + logf(s);
      const size_t cell = (static_cast<size_t>(b) * a.T_max + t) * (a.U_max + 1) + u;
      a.lp_blank[cell] = vb - lse;
      a.lp_emit[cell] = u < Ub ? ve - lse : -INFINITY;
    }
  }
}

__device__ __forceinline__ float logaddexp(float x, float y) {
  const float mx = fmaxf(x, y), mn = fminf(x, y);
  return mx == -INFINITY ? mx : mx + log1pf(expf(mn - mx));
}

// One CTA per utterance.  Diagonal d = t + u: cell (t, u) needs (t - 1, u) and (t, u - 1), both on diagonal d - 1 at
// label index u and u - 1, so two shared rows indexed by u (previous / current diagonal) carry the recursion.
__global__ void __launch_bounds__(256) rnnt_align_dp_kernel(const AlignArgs a) {
  extern __shared__ __align__(16) float s_dp[];                // [2 diagonals][2 (forward, Viterbi)][U_max + 1]
  const int b = blockIdx.x, tid = threadIdx.x, U1 = a.U_max + 1;
  const int T = a.enc_len[b], U = a.label_len[b];
  int bad = T < 1 || T > a.T_max || U < 0 || U > a.U_max;
  if (!bad)
    for (int i = tid; i < U; i += blockDim.x) {
      const int y = a.labels[static_cast<size_t>(b) * a.U_max + i];
      if (y < 0 || y >= a.V) bad = 1;
    }
  bad = __syncthreads_or(bad);
  int32_t* frames = a.frames + static_cast<size_t>(b) * a.U_max;
  float* token_lp = a.token_lp + static_cast<size_t>(b) * a.U_max;
  for (int i = tid; i < a.U_max; i += blockDim.x)
    if (bad || i >= U) { frames[i] = -1; token_lp[i] = NAN; }
  if (bad) {
    if (tid == 0) { a.viterbi[b] = NAN; a.loglik[b] = NAN; }
    return;
  }
  const size_t base = static_cast<size_t>(b) * a.T_max * U1;
  const float* lpb = a.lp_blank + base;
  const float* lpe = a.lp_emit + base;
  uint8_t* choice = a.choice + base;
  float* cur = s_dp;
  float* prev = s_dp + 2 * U1;
  for (int d = 0; d < T + U; ++d) {
    for (int u = tid; u <= U; u += blockDim.x) {
      const int t = d - u;
      if (t < 0 || t >= T) continue;
      float f = 0.f, v = 0.f;
      uint8_t ch = 0;                                          // 1: the Viterbi predecessor is (t, u - 1), an emission
      if (d > 0) {
        float fb = -INFINITY, vb = -INFINITY, fe = -INFINITY, ve = -INFINITY;
        if (t > 0) {
          const float l = lpb[static_cast<size_t>(t - 1) * U1 + u];
          fb = prev[u] + l; vb = prev[U1 + u] + l;
        }
        if (u > 0) {
          const float l = lpe[static_cast<size_t>(t) * U1 + u - 1];
          fe = prev[u - 1] + l; ve = prev[U1 + u - 1] + l;
        }
        f = logaddexp(fb, fe);
        ch = (t == 0 || ve > vb) ? 1 : 0;                      // an exact tie goes to the blank predecessor
        v = ch ? ve : vb;
      }
      choice[static_cast<size_t>(t) * U1 + u] = ch;
      cur[u] = f; cur[U1 + u] = v;
    }
    __syncthreads();
    float* x = cur; cur = prev; prev = x;
  }
  if (tid == 0) {
    const float l = lpb[static_cast<size_t>(T - 1) * U1 + U];
    a.loglik[b] = prev[U] + l;
    a.viterbi[b] = prev[U1 + U] + l;
    int t = T - 1, u = U;
    while (u > 0) {
      if (choice[static_cast<size_t>(t) * U1 + u]) {
        frames[u - 1] = t;
        token_lp[u - 1] = lpe[static_cast<size_t>(t) * U1 + u - 1];
        --u;
      } else {
        --t;
      }
    }
  }
}

}  // namespace

size_t align_dp_smem(int U_max) { return static_cast<size_t>(4) * (U_max + 1) * sizeof(float); }

static size_t lattice_smem(int Hj, int V) {
  const int n_tiles = (V + 1 + kBN - 1) / kBN;
  return 1024 + kStages * kStageBytes + static_cast<size_t>(kTileT + kTileU) * (Hj + 8) * 4 + static_cast<size_t>(n_tiles) * kBN * 4 +
         kTileU * 4 + kStages * 8;
}

bool align_supported(int Hj, int Hp, int V, int U_max, char* err) {
  if (Hj % kBK != 0 || Hp % 2 != 0 || Hp > 1536) {
    snprintf(err, 256, "joint_hidden %% %d == 0 and an even pred_hidden <= 1536 required (got %d, %d)", kBK, Hj, Hp);
    return false;
  }
  if (lattice_smem(Hj, V) > 227 * 1024) { snprintf(err, 256, "joint_hidden=%d / vocab_size=%d exceed the lattice kernel's shared memory", Hj, V); return false; }
  if (align_dp_smem(U_max) > 227 * 1024) { snprintf(err, 256, "U_max=%d exceeds the alignment DP's shared memory (at most %d labels)", U_max, 227 * 1024 / 16 - 1); return false; }
  return true;
}

cudaError_t launch_align_lstm_step(const AlignArgs& a, int u, cudaStream_t stream) {
  const int warps = a.B * a.Hp;
  align_lstm_step_kernel<<<(warps + 7) / 8, 256, 0, stream>>>(a, u);
  return cudaGetLastError();
}

cudaError_t launch_align_pred_proj(const AlignArgs& a, cudaStream_t stream) {
  const int rows = a.B * (a.U_max + 1);
  const size_t smem = static_cast<size_t>(kPpRows) * a.Hp * 4;   // <= 48 KB for pred_hidden <= 1536 (align_supported)
  align_pred_proj_kernel<<<(rows + kPpRows - 1) / kPpRows, 256, smem, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_rnnt_lattice(const AlignArgs& a, cudaStream_t stream, char* err) {
  CUtensorMap tm;
  if (!make_tmap_bf16(&tm, a.w_out, static_cast<uint64_t>(a.V) + 1, a.Hj, a.Hj, kBN, err)) return cudaErrorInvalidValue;
  const size_t smem = lattice_smem(a.Hj, a.V);
  static DeviceOnce attr_once;
  if (attr_once.pending()) {
    const cudaError_t e = cudaFuncSetAttribute(rnnt_lattice_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_once.set();
  }
  const int tiles = ((a.T_max + kTileT - 1) / kTileT) * ((a.U_max + 1 + kTileU - 1) / kTileU);
  rnnt_lattice_kernel<<<a.B * tiles, kLatThreads, smem, stream>>>(tm, a);
  return cudaGetLastError();
}

cudaError_t launch_rnnt_align_dp(const AlignArgs& a, cudaStream_t stream) {
  static DeviceOnce attr_once;
  if (attr_once.pending()) {
    const cudaError_t e = cudaFuncSetAttribute(rnnt_align_dp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_once.set();
  }
  rnnt_align_dp_kernel<<<a.B, 256, align_dp_smem(a.U_max), stream>>>(a);
  return cudaGetLastError();
}

}  // namespace rs
