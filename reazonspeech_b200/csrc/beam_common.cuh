// Device pieces shared by the transducer beam searches: ALSD (decode_alsd.cu) and MAES (decode_maes.cu).
#pragma once
#include <cfloat>
#include <cuda_bf16.h>

#include "common.cuh"

namespace rs {

// x -> three bf16 values with hi + mid + lo == x to 24 mantissa bits
__device__ __forceinline__ void split3(float x, __nv_bfloat16& hi, __nv_bfloat16& mid, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  const float r1 = x - __bfloat162float(hi);
  mid = __float2bfloat16_rn(r1);
  lo = __float2bfloat16_rn(r1 - __bfloat162float(mid));
}

__device__ __forceinline__ double logaddexp(double a, double b) {
  const double hi = a > b ? a : b, lo = a > b ? b : a;
  return hi + log1p(exp(lo - hi));
}

// One joint row x of NC = V + 1 logits (blank last), by a block of 256 threads: the log-sum-exp lse, log p(blank), and the m
// largest of the first n_cls classes as log-probabilities with their indices (ties -> lower class index).  ALSD ranks the
// non-blank classes (n_cls = V), MAES all of them (n_cls = V + 1).  lse_out / blank_out may be null; m may be 0.
__device__ __forceinline__ void beam_row_reduce(const float* __restrict__ x, int NC, int n_cls, int m, float* lse_out, float* blank_out,
                                                float* top_lp, int* top_tok) {
  __shared__ float s_red[8];
  __shared__ float s_val[8];
  __shared__ int s_idx[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float mx = -FLT_MAX;
  for (int j = tid; j < NC; j += 256) mx = fmaxf(mx, x[j]);
  mx = warp_max(mx);
  if (lane == 0) s_red[warp] = mx;
  __syncthreads();
  mx = s_red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_red[w]);
  __syncthreads();
  float se = 0.f;
  for (int j = tid; j < NC; j += 256) se += expf(x[j] - mx);
  se = warp_sum(se);
  if (lane == 0) s_red[warp] = se;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += s_red[w];
  const float lse = mx + logf(tot);
  if (tid == 0) {
    if (lse_out) *lse_out = lse;
    if (blank_out) *blank_out = x[NC - 1] - lse;
  }
  // top-m: m rounds of (max, lowest index), each round excluding what was taken before
  float prev_v = FLT_MAX;
  int prev_i = -1;
  for (int round = 0; round < m; ++round) {
    float bv = -FLT_MAX;
    int bi = 0x7fffffff;
    for (int j = tid; j < n_cls; j += 256) {
      const float v = x[j];
      const bool after = v < prev_v || (v == prev_v && j > prev_i);        // strictly after the previous pick in (value desc, index asc) order
      if (after && (v > bv || (v == bv && j < bi))) { bv = v; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    __syncthreads();
    if (lane == 0) { s_val[warp] = bv; s_idx[warp] = bi; }
    __syncthreads();
    bv = s_val[0]; bi = s_idx[0];
#pragma unroll
    for (int w = 1; w < 8; ++w)
      if (s_val[w] > bv || (s_val[w] == bv && s_idx[w] < bi)) { bv = s_val[w]; bi = s_idx[w]; }
    if (tid == 0) {
      top_lp[round] = bv - lse;
      top_tok[round] = bi;
    }
    prev_v = bv; prev_i = bi;
  }
}

}  // namespace rs
