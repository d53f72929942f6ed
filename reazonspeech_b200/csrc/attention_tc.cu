// Relative-position local attention with a global token (N5) on the Hopper tensor cores (wgmma).
//
// NeMo RelPositionMultiHeadAttentionLongformer (parts/submodules/multi_head_attention.py, reached through
// model.transcribe at pkg/nemo-asr/src/transcribe.py:48-53; semantics restated in
// oracle/nemo_restated.py::local_attention_core).
//
// One CTA = 128 query rows of one (utterance, head): two consumer warpgroups of 64 rows each and one producer warp.
// With a band of +-w (w <= 128) those rows see the 384 keys [q0-128, q0+256), walked in six blocks of 64 keys:
//
//   TMA    Q' [128 x 128] (q + pos_bias_u, folded into the QKV projection's bias at pack time) and the head's positional
//          table P [n_rel_pad x 128] (linear_pos(pos_emb), packed at load) -> shared memory, 128-byte swizzle, K-major
//   wgmma  BD[64 x n_rel_pad] = Q' P^T per warpgroup, 32 columns at a time (the relative-position term; + the constant
//          (pos_bias_v - pos_bias_u) . p[c] it equals (q + pos_bias_v) . p[c]) -> (acc + bias[c]) / sqrt(dk) * log2 e as
//          IEEE half, row-major in shared memory.  It never leaves the SM.
//   TMA    K [64 x 128] and V^T [128 x 64] blocks through a three-stage ring laid over the positional table (dead once
//          the BD product has retired); the QKV GEMM's epilogue writes V transposed (RS_EPI_QKV_VT)
//   per key block and warpgroup:
//     wgmma  S[64 x 64] = Q' K^T, accumulators in registers
//     t = S / sqrt(dk) + BD[i, j-i+w] (the rel_shift: row i reads its BD row at an offset that depends on i) with the band /
//         padding mask; running row maximum and sum (online softmax, log2 domain), O rescaled when the maximum moves
//     wgmma  O[64 x 128] += P V with P = exp2(t - m) as bf16 taken straight from the S accumulator registers (the
//            accumulator fragment of S is the A fragment of the next product)
//   epilogue  O + p_global * v_0, divided by the row sum -> bf16, staged per warp and stored in whole rows
//
// Rows of the global token itself are overwritten afterwards by global_row_attention_tc_kernel (full attention, no
// positional term).  Shared memory: 32 KB Q' + 96 KB positional table / K, V^T ring + 74 KB BD.
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"

namespace rs {

namespace {

constexpr int TQ = 128;                 // query rows per CTA
constexpr int TDK = 128;                // head dim
constexpr int KB = 64;                  // keys per block
constexpr int kBlocks = 6;              // key window = 384 keys
constexpr int kSlab = TQ * 128;         // bytes of one [128 rows x 64 bf16] swizzled slab
constexpr int kAtcThreads = 32 * 9;     // warps 0..7: two consumer warpgroups; warp 8: TMA producer
constexpr int kKvStages = 3;
constexpr uint32_t kKvStageBytes = 2 * KB * 128 + TDK * 128;   // K block as two k-slabs of 64 rows + V^T block of 128 rows
constexpr uint32_t kOffQ = 0;                       // 2 slabs
constexpr uint32_t kOffKV = 2 * kSlab;              // positional table (2 k-slabs x n_rel_pad rows), then the K / V^T ring
constexpr uint32_t kOffBD = kOffKV + kKvStages * kKvStageBytes;   // BD as IEEE half [128][kBdPitch]; a warp's rows stage its output at the end
constexpr int kBdPitch = 296;                       // halves per BD row
constexpr int kNrelPadMax = 288;                    // 2 * 128 + 1 relative offsets rounded up to 32
constexpr uint32_t kOffBar = kOffBD + TQ * kBdPitch * 2;   // 8 mbarriers | k_0 [128] bf16 (+64) | u.k_0 (+320) | q'.k_0 [128] (+512) | v_0 [128] (+1024)
constexpr uint32_t kAtcSmem = kOffBar + 1536 + 1024;       // + alignment slack
constexpr int kOutPitch = 136;                      // bf16 per staged output row (272 B: conflict-free fragment writes)
static_assert(2 * kNrelPadMax * 128 <= kKvStages * kKvStageBytes && kOutPitch <= kBdPitch && kAtcSmem <= 227 * 1024, "shared memory layout");

struct AtcDev {
  const __nv_bfloat16* qk;      // [M, ld_qk]: q' at column h*128, k at column d + h*128
  const __nv_bfloat16* vt;      // [d, ld_vt]: V^T, column = global frame index
  const float* bd_bias;         // [H, n_rel_pad]: (pos_bias_v - pos_bias_u) . p[h][c]
  const float* bias_u;          // [H, 128]
  __nv_bfloat16* out;           // [M, d]
  const int32_t* enc_len;
  int T_max, H, w_left, w_right, n_global, n_rel_pad, ld_qk, ld_vt;
};

__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// byte offset of the 16-byte chunk `chunk` (0..7) of row `row` inside a [rows x 64 bf16] 128B-swizzled slab
__device__ __forceinline__ uint32_t sw128(int row, int chunk) {
  return static_cast<uint32_t>((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

__global__ void __launch_bounds__(kAtcThreads, 1)
local_attention_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                          const __grid_constant__ CUtensorMap tm_vt, const __grid_constant__ CUtensorMap tm_pos, const AtcDev p) {
  extern __shared__ uint8_t atc_raw[];
  const uint32_t base = (smem_u32(atc_raw) + 1023u) & ~1023u;
  uint8_t* gen = atc_raw + (base - smem_u32(atc_raw));          // generic pointer to the aligned base
  const uint32_t bar_qk = base + kOffBar, bar_drained = bar_qk + 8;
  auto full_bar = [&](int s) { return bar_qk + 16u + 8u * s; };
  auto empty_bar = [&](int s) { return bar_qk + 40u + 8u * s; };
  __nv_bfloat16* s_k0 = reinterpret_cast<__nv_bfloat16*>(gen + kOffBar + 64);   // [128] global key
  float* s_uk = reinterpret_cast<float*>(gen + kOffBar + 320);
  float* s_sg = reinterpret_cast<float*>(gen + kOffBar + 512);                  // [128] raw q'.k_0
  float* s_v0 = reinterpret_cast<float*>(gen + kOffBar + 1024);                 // [128] V row of frame 0

  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * TQ;
  const int len = p.enc_len[b];
  const int d = p.H * TDK;
  const int warp = warp_id_uniform(), lane = lane_id();
  const size_t row0 = static_cast<size_t>(b) * p.T_max;
  __nv_bfloat16* obase = p.out + row0 * d + h * TDK;

  if (q0 >= len) {                                   // fully padded tile: defined zeros
    for (int id = threadIdx.x; id < TQ * 16; id += blockDim.x) {
      const int r = id >> 4, c = (id & 15) * 8;
      if (q0 + r < p.T_max) *reinterpret_cast<uint4*>(obase + static_cast<size_t>(q0 + r) * d + c) = make_uint4(0, 0, 0, 0);
    }
    return;
  }

  // key blocks (64 keys each) that hold at least one key an in-range query of this tile may attend to
  const int j_base = q0 - 128;
  const int q_hi = min(q0 + TQ, len) - 1;                                    // last valid query row of the tile
  const int key_lo = max(0, q0 - p.w_left), key_hi = min(len - 1, q_hi + p.w_right);
  const int blk_lo = max((key_lo - j_base) >> 6, 0), blk_hi = min((key_hi - j_base) >> 6, kBlocks - 1);   // inclusive
  const uint32_t pos_slab = static_cast<uint32_t>(p.n_rel_pad) * 128u;          // bytes of one k-slab of the positional table

  if (threadIdx.x == 256) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_vt);
    tma_prefetch_desc(&tm_pos);
    mbar_init(bar_qk, 1); mbar_init(bar_drained, 8);
    for (int s = 0; s < kKvStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
    fence_barrier_init();
    // Q' and the head's positional table: two k-slabs of n_rel_pad rows, each fetched as two boxes of n_rel_pad / 2 rows
    mbar_arrive_expect_tx(bar_qk, static_cast<uint32_t>(2 * kSlab + 2 * pos_slab));
    for (int kb = 0; kb < 2; ++kb) {
      tma_load_2d(base + kOffQ + kb * kSlab, &tm_q, h * TDK + kb * 64, static_cast<int>(row0) + q0, bar_qk);
      for (int hh = 0; hh < 2; ++hh)
        tma_load_2d(base + kOffKV + kb * pos_slab + hh * (pos_slab / 2), &tm_pos, kb * 64, h * p.n_rel_pad + hh * (p.n_rel_pad / 2), bar_qk);
    }
  }
  __syncthreads();

  if (warp == 8) {
    // ---- producer: K / V^T blocks over the positional table once both warpgroups' BD products have retired
    if (lane == 0) {
      mbar_wait(bar_drained, 0);
      int s = 0; uint32_t phase = 0;
      for (int blk = blk_lo; blk <= blk_hi; ++blk) {
        mbar_wait(empty_bar(s), phase ^ 1u);
        mbar_arrive_expect_tx(full_bar(s), kKvStageBytes);
        const uint32_t st = base + kOffKV + s * kKvStageBytes;
        const int key0 = static_cast<int>(row0) + j_base + blk * KB;
        for (int kb = 0; kb < 2; ++kb) tma_load_2d(st + kb * (KB * 128), &tm_k, d + h * TDK + kb * 64, key0, full_bar(s));
        tma_load_2d(st + 2 * KB * 128, &tm_vt, key0, h * TDK, full_bar(s));
        if (++s == kKvStages) { s = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ---- consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile; a lane holds rows r0 and r1 = r0 + 8 of its warp's 16
  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const int rbase = wg * 64 + (warp & 3) * 16;
  const int r0 = rbase + g, r1 = r0 + 8;
  const int i0 = q0 + r0, i1 = q0 + r1;
  const bool ok0 = i0 < len, ok1 = i1 < len;
  const float scale2 = rsqrtf(static_cast<float>(TDK)) * 1.4426950408889634f;       // 1/sqrt(dk) * log2(e)
  __half* s_bd = reinterpret_cast<__half*>(gen + kOffBD);

  // global token: score of its key against each row, without bias_u and without a positional term:
  // (q' - u) . k_0 = q'.k_0 (per row, two threads each) - u.k_0 (one scalar per CTA, by warp 0)
  float sg0 = -INFINITY, sg1 = -INFINITY;
  if (p.n_global > 0) {
    const int tid = threadIdx.x;                                                 // 0..255
    if (tid < 16) *reinterpret_cast<uint4*>(s_k0 + tid * 8) = __ldg(reinterpret_cast<const uint4*>(p.qk + row0 * p.ld_qk + d + h * TDK) + tid);
    if (tid >= 128) s_v0[tid - 128] = __bfloat162float(p.vt[static_cast<size_t>(h * TDK + (tid - 128)) * p.ld_vt + row0]);
    named_bar_sync(1, 256);
    if (warp == 0) {
      float uk = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) uk = fmaf(__ldg(p.bias_u + h * TDK + lane * 4 + e), __bfloat162float(s_k0[lane * 4 + e]), uk);
      uk = warp_sum(uk);
      if (lane == 0) *s_uk = uk;
    }
    mbar_wait(bar_qk, 0);                                                        // Q' has landed
    {
      const int r = tid >> 1, hf = tid & 1;                                      // row, 64-column half
      float acc0 = 0.f, acc1 = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 qv = *reinterpret_cast<const uint4*>(gen + kOffQ + hf * kSlab + sw128(r, c));
        const uint4 kv = *reinterpret_cast<const uint4*>(s_k0 + hf * 64 + c * 8);
        const uint32_t qw[4] = {qv.x, qv.y, qv.z, qv.w}, kw[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 q2 = unpack_bf16x2(qw[e]), k2 = unpack_bf16x2(kw[e]);
          acc0 = fmaf(q2.x, k2.x, acc0); acc1 = fmaf(q2.y, k2.y, acc1);
        }
      }
      float acc = acc0 + acc1;
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      if (hf == 0) s_sg[r] = acc;
    }
    named_bar_sync(1, 256);
    sg0 = (s_sg[r0] - *s_uk) * scale2;
    sg1 = (s_sg[r1] - *s_uk) * scale2;
  } else {
    mbar_wait(bar_qk, 0);
  }

  const uint32_t q_addr = base + kOffQ + wg * (64 * 128);       // the warpgroup's 64 rows inside each k-slab of Q'
  // ---- the positional product: BD[r][c] = ((q' . p[c]) + bias[c]) / sqrt(dk) * log2 e as IEEE half, row-major
#pragma unroll 1
  for (int ch = 0; ch < (p.n_rel_pad >> 5); ++ch) {
    float acc[16];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 2; ++kb) {
      const uint64_t da = wgmma_desc_k_sw128(q_addr + kb * kSlab);
      const uint64_t db = wgmma_desc_k_sw128(base + kOffKV + kb * pos_slab + ch * 4096);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_bf16_ss_n32(acc, da + 2u * k, db + 2u * k, (kb | k) != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = ch * 32 + 8 * j + 2 * t;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bd_bias + h * p.n_rel_pad + col));
      *reinterpret_cast<__half2*>(s_bd + r0 * kBdPitch + col) = __floats2half2_rn((acc[4 * j] + bb.x) * scale2, (acc[4 * j + 1] + bb.y) * scale2);
      *reinterpret_cast<__half2*>(s_bd + r1 * kBdPitch + col) = __floats2half2_rn((acc[4 * j + 2] + bb.x) * scale2, (acc[4 * j + 3] + bb.y) * scale2);
    }
  }
  __syncwarp();                                        // a warp reads back only the BD rows it wrote
  if (lane == 0) mbar_arrive(bar_drained);             // the ring may overwrite the positional table

  // keys the warpgroup's in-range rows may attend to
  const int wrow_lo = q0 + wg * 64;
  const bool wg_valid = wrow_lo < len;
  const int wkey_lo = max(0, wrow_lo - p.w_left), wkey_hi = min(len - 1, min(wrow_lo + 64, len) - 1 + p.w_right);

  float o[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) o[e] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;      // running maxima (log2 domain) and this lane's partial row sums
  const __half* bd0 = s_bd + r0 * kBdPitch + p.w_left - i0;      // BD column of key j for row i: j - i + w_left
  const __half* bd1 = s_bd + r1 * kBdPitch + p.w_left - i1;
  int s = 0; uint32_t phase = 0;
#pragma unroll 1
  for (int blk = blk_lo; blk <= blk_hi; ++blk) {
    mbar_wait(full_bar(s), phase);
    const int jlo = j_base + blk * KB;
    if (wg_valid && jlo + KB - 1 >= wkey_lo && jlo <= wkey_hi) {          // warpgroup-uniform
      const uint32_t st = base + kOffKV + s * kKvStageBytes;
      float sc[32];
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        const uint64_t da = wgmma_desc_k_sw128(q_addr + kb * kSlab);
        const uint64_t db = wgmma_desc_k_sw128(st + kb * (KB * 128));
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_bf16_ss_n64(sc, da + 2u * k, db + 2u * k, (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // t = S * scale2 + BD (pre-scaled), masked to the band (-w_left <= j - i <= w_right) and to 0 <= j < len
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int ja = jlo + 8 * j + 2 * t + q;
          const bool in = ja >= 0 && ja < len;
          const bool a0 = in && ok0 && ja - i0 >= -p.w_left && ja - i0 <= p.w_right;
          const bool a1 = in && ok1 && ja - i1 >= -p.w_left && ja - i1 <= p.w_right;
          const float t0 = a0 ? fmaf(sc[4 * j + q], scale2, __half2float(bd0[ja])) : -INFINITY;
          const float t1 = a1 ? fmaf(sc[4 * j + 2 + q], scale2, __half2float(bd1[ja])) : -INFINITY;
          sc[4 * j + q] = t0; sc[4 * j + 2 + q] = t1;
          mx0 = fmaxf(mx0, t0); mx1 = fmaxf(mx1, t1);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);
      const float c0 = m0 == -INFINITY ? 0.f : ex2f(m0 - n0), c1 = m1 == -INFINITY ? 0.f : ex2f(m1 - n1);
      const float ref0 = n0 == -INFINITY ? 0.f : n0, ref1 = n1 == -INFINITY ? 0.f : n1;
      m0 = n0; m1 = n1;
      l0 *= c0; l1 *= c1;
#pragma unroll
      for (int j = 0; j < 16; ++j) { o[4 * j] *= c0; o[4 * j + 1] *= c0; o[4 * j + 2] *= c1; o[4 * j + 3] *= c1; }
      // p = exp2(t - m) as bf16 (row sums of the rounded values), handed to the P.V product as its A fragments
      uint32_t pa[4][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t w0 = pack_bf16x2(ex2f(sc[4 * j] - ref0), ex2f(sc[4 * j + 1] - ref0));
        const uint32_t w1 = pack_bf16x2(ex2f(sc[4 * j + 2] - ref1), ex2f(sc[4 * j + 3] - ref1));
        const float2 b0 = unpack_bf16x2(w0), b1 = unpack_bf16x2(w1);
        l0 += b0.x + b0.y; l1 += b1.x + b1.y;
        pa[j >> 1][(j & 1) * 2] = w0; pa[j >> 1][(j & 1) * 2 + 1] = w1;
      }
      wgmma_fence();
      const uint64_t dv = wgmma_desc_k_sw128(st + 2 * KB * 128);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_bf16_rs_n128(o, pa[kk], dv + 2u * kk, 1u);
      wgmma_commit();
      wgmma_wait<0>();
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar(s));
    if (++s == kKvStages) { s = 0; phase ^= 1u; }
  }

  // ---- epilogue: O + p_global * v_0, divided by the row sum -> bf16
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  float pg0 = 0.f, pg1 = 0.f;
  if (p.n_global > 0) {
    const float f0 = fmaxf(m0, sg0), f1 = fmaxf(m1, sg1);
    const float c0 = m0 == -INFINITY ? 0.f : ex2f(m0 - f0), c1 = m1 == -INFINITY ? 0.f : ex2f(m1 - f1);
    pg0 = ok0 ? ex2f(sg0 - f0) : 0.f; pg1 = ok1 ? ex2f(sg1 - f1) : 0.f;
    l0 = l0 * c0 + pg0; l1 = l1 * c1 + pg1;
#pragma unroll
    for (int j = 0; j < 16; ++j) { o[4 * j] *= c0; o[4 * j + 1] *= c0; o[4 * j + 2] *= c1; o[4 * j + 3] *= c1; }
  }
  const float inv0 = (ok0 && l0 > 0.f) ? 1.0f / l0 : 0.f, inv1 = (ok1 && l1 > 0.f) ? 1.0f / l1 : 0.f;
  __syncwarp();                                        // the warp's BD rows are dead: they stage its 16 output rows
  __nv_bfloat16* stage = reinterpret_cast<__nv_bfloat16*>(s_bd + rbase * kBdPitch);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = 8 * j + 2 * t;
    const float v0a = p.n_global > 0 ? s_v0[col] : 0.f, v0b = p.n_global > 0 ? s_v0[col + 1] : 0.f;
    *reinterpret_cast<uint32_t*>(stage + g * kOutPitch + col) = pack_bf16x2((o[4 * j] + pg0 * v0a) * inv0, (o[4 * j + 1] + pg0 * v0b) * inv0);
    *reinterpret_cast<uint32_t*>(stage + (g + 8) * kOutPitch + col) = pack_bf16x2((o[4 * j + 2] + pg1 * v0a) * inv1, (o[4 * j + 3] + pg1 * v0b) * inv1);
  }
  __syncwarp();
#pragma unroll
  for (int it = 0; it < 8; ++it) {                      // 2 rows x 256 B per instruction
    const int rr = it * 2 + (lane >> 4), cc = (lane & 15) * 8;
    const int row = q0 + rbase + rr;
    const uint4 a = *reinterpret_cast<const uint4*>(stage + rr * kOutPitch + cc);
    if (row < p.T_max) *reinterpret_cast<uint4*>(obase + static_cast<size_t>(row) * d + cc) = a;
  }
}

// Row(s) of the global token(s): full attention softmax_j((q_g / sqrt(dk)) . k_j) v_j, no positional terms.
// On the layouts of the tensor-core path: the query row
// holds q + pos_bias_u (subtracted again here) and V is read from its transposed copy (keys contiguous).
// grid (H, B), 256 threads.
__global__ void __launch_bounds__(256)
global_row_attention_tc_kernel(const AtcDev p) {
  extern __shared__ __align__(16) float gs[];        // [T_pad] scores | [8] reduction scratch | [128] q
  const int h = blockIdx.x, b = blockIdx.y;
  const int len = p.enc_len[b];
  if (len <= 0) return;
  const int d = p.H * TDK;
  const size_t row0 = static_cast<size_t>(b) * p.T_max;
  const __nv_bfloat16* qrow = p.qk + row0 * p.ld_qk + h * TDK;
  const __nv_bfloat16* kbase = qrow + d;
  const float scale = rsqrtf(static_cast<float>(TDK));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int t_pad = ((p.T_max > 1024 ? p.T_max : 1024) + 7) & ~7;
  float* red = gs + t_pad;
  float* sq = red + 8;
  if (tid < TDK) sq[tid] = (__bfloat162float(qrow[tid]) - p.bias_u[h * TDK + tid]) * scale;
  __syncthreads();
  float mx = -INFINITY;
  for (int j = tid; j < len; j += 256) {
    const uint4* kr = reinterpret_cast<const uint4*>(kbase + static_cast<size_t>(j) * p.ld_qk);
    uint4 kk[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) kk[i] = __ldg(kr + i);
    float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float4 qa = *reinterpret_cast<const float4*>(sq + 8 * i), qb = *reinterpret_cast<const float4*>(sq + 8 * i + 4);
      d0 = fmaf(bf16_lo(kk[i].x), qa.x, d0); d1 = fmaf(bf16_hi(kk[i].x), qa.y, d1);
      d2 = fmaf(bf16_lo(kk[i].y), qa.z, d2); d3 = fmaf(bf16_hi(kk[i].y), qa.w, d3);
      d0 = fmaf(bf16_lo(kk[i].z), qb.x, d0); d1 = fmaf(bf16_hi(kk[i].z), qb.y, d1);
      d2 = fmaf(bf16_lo(kk[i].w), qb.z, d2); d3 = fmaf(bf16_hi(kk[i].w), qb.w, d3);
    }
    const float v = (d0 + d1) + (d2 + d3);
    gs[j] = v;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3])), fmaxf(fmaxf(red[4], red[5]), fmaxf(red[6], red[7])));
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j < len; j += 256) { const float e = __expf(gs[j] - mx); gs[j] = e; sum += e; }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  const float inv = 1.0f / (((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7])));
  // out[dim] = sum_j p_j V^T[dim][j]: thread = (dim, one of two key segments); it walks its V^T row eight keys (16 bytes)
  // at a time with four loads in flight (the last, partial group of eight goes key by key: what follows the utterance in
  // V^T is not this kernel's to read).
  __syncthreads();
  const __nv_bfloat16* vt = p.vt + static_cast<size_t>(h * TDK) * p.ld_vt + row0;
  const int len8 = ((row0 & 7) == 0) ? (len & ~7) : 0;
  const int dim = tid & 127, seg = tid >> 7;
  const int n8 = len8 >> 3;                                  // whole groups of eight keys
  const int g_lo = seg == 0 ? 0 : (n8 + 1) / 2, g_hi = seg == 0 ? (n8 + 1) / 2 : n8;
  const __nv_bfloat16* vr = vt + static_cast<size_t>(dim) * p.ld_vt;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  auto dot8 = [&](const uint4 raw, int j, float& acc) {
    const float4 p0 = *reinterpret_cast<const float4*>(gs + j), p1 = *reinterpret_cast<const float4*>(gs + j + 4);
    acc = fmaf(p0.x, bf16_lo(raw.x), acc); acc = fmaf(p0.y, bf16_hi(raw.x), acc);
    acc = fmaf(p0.z, bf16_lo(raw.y), acc); acc = fmaf(p0.w, bf16_hi(raw.y), acc);
    acc = fmaf(p1.x, bf16_lo(raw.z), acc); acc = fmaf(p1.y, bf16_hi(raw.z), acc);
    acc = fmaf(p1.z, bf16_lo(raw.w), acc); acc = fmaf(p1.w, bf16_hi(raw.w), acc);
  };
  int g = g_lo;
  for (; g + 4 <= g_hi; g += 4) {
    const uint4 r0 = __ldg(reinterpret_cast<const uint4*>(vr) + g), r1 = __ldg(reinterpret_cast<const uint4*>(vr) + g + 1);
    const uint4 r2 = __ldg(reinterpret_cast<const uint4*>(vr) + g + 2), r3 = __ldg(reinterpret_cast<const uint4*>(vr) + g + 3);
    dot8(r0, 8 * g, a0); dot8(r1, 8 * g + 8, a1); dot8(r2, 8 * g + 16, a2); dot8(r3, 8 * g + 24, a3);
  }
  for (; g < g_hi; ++g) dot8(__ldg(reinterpret_cast<const uint4*>(vr) + g), 8 * g, a0);
  if (seg == 1) for (int j = len8; j < len; ++j) a1 = fmaf(gs[j], __bfloat162float(vr[j]), a1);
  const float part = (a0 + a1) + (a2 + a3);
  __syncthreads();                                   // everyone is done reading the probabilities
  if (seg == 1) gs[dim] = part;
  __syncthreads();
  if (seg == 0) p.out[row0 * d + h * TDK + dim] = __float2bfloat16_rn((part + gs[dim]) * inv);
}

}  // namespace

bool attention_tc_supported(const AttnArgs& a) {
  return a.dk == TDK && a.w_left >= 0 && a.w_right >= 0 && a.w_left <= 128 && a.w_right <= 128 && (a.w_left & 7) == 0 && a.n_global >= 0 &&
         a.n_global <= 1 && a.vt != nullptr && (a.T_max & 7) == 0 && a.n_rel_pad >= a.w_left + a.w_right + 1 && a.n_rel_pad % 32 == 0 &&
         a.n_rel_pad <= kNrelPadMax;
}

cudaError_t launch_attention_tc(const AttnArgs& a, cudaStream_t stream) {
  if (!attention_tc_supported(a) || a.pos == nullptr || a.bd_bias == nullptr || (a.ld_vt & 7)) return cudaErrorInvalidValue;
  const int d = a.H * TDK;
  const int64_t M = static_cast<int64_t>(a.B) * a.T_max;
  AtcDev p;
  p.qk = static_cast<const __nv_bfloat16*>(a.qkv); p.vt = static_cast<const __nv_bfloat16*>(a.vt);
  p.bd_bias = a.bd_bias; p.bias_u = a.bias_u; p.out = static_cast<__nv_bfloat16*>(a.out);
  p.enc_len = a.enc_len; p.T_max = a.T_max; p.H = a.H; p.w_left = a.w_left; p.w_right = a.w_right;
  p.n_global = a.n_global; p.n_rel_pad = a.n_rel_pad; p.ld_qk = 3 * d; p.ld_vt = a.ld_vt;
  CUtensorMap tm_q, tm_k, tm_vt, tm_pos;
  char err[256];
  // positional table [H * n_rel_pad, 128] bf16, fetched in boxes of n_rel_pad / 2 rows (<= 144; a TMA box holds at most 256)
  if (!make_tmap_bf16(&tm_pos, a.pos, static_cast<uint64_t>(a.H) * a.n_rel_pad, TDK, TDK, static_cast<uint32_t>(a.n_rel_pad / 2), err)) return cudaErrorInvalidValue;
  if (!make_tmap_bf16(&tm_q, p.qk, static_cast<uint64_t>(M), static_cast<uint64_t>(2 * d), static_cast<uint64_t>(p.ld_qk), 128, err)) return cudaErrorInvalidValue;
  if (!make_tmap_bf16(&tm_k, p.qk, static_cast<uint64_t>(M), static_cast<uint64_t>(2 * d), static_cast<uint64_t>(p.ld_qk), KB, err)) return cudaErrorInvalidValue;
  if (!make_tmap_bf16(&tm_vt, p.vt, static_cast<uint64_t>(d), static_cast<uint64_t>(M), static_cast<uint64_t>(p.ld_vt), 128, err)) return cudaErrorInvalidValue;
  static DeviceOnce attr_once;
  if (attr_once.pending()) {
    cudaError_t e = cudaFuncSetAttribute(local_attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kAtcSmem));
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(global_row_attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return e;
    attr_once.set();
  }
  const dim3 grid((a.T_max + TQ - 1) / TQ, a.H, a.B);
  local_attention_tc_kernel<<<grid, kAtcThreads, kAtcSmem, stream>>>(tm_q, tm_k, tm_vt, tm_pos, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  if (a.n_global > 0) {
    const size_t gsmem = (static_cast<size_t>(((a.T_max > 1024 ? a.T_max : 1024) + 7) & ~7) + 8 + TDK) * sizeof(float);
    if (gsmem > 200 * 1024) return cudaErrorInvalidValue;
    global_row_attention_tc_kernel<<<dim3(a.H, a.B), 256, gsmem, stream>>>(p);
    e = cudaGetLastError();
  }
  return e;
}

}  // namespace rs
