// HBM-bound row kernels of the Conformer layer: LayerNorm (N7 / pre-norms) and the middle of
// ConformerConvolution (mask -> depthwise k=9 -> BatchNorm(eval, folded) -> Swish) (N6).
// Warp-shuffle reductions, 128-bit / 32-bit coalesced accesses; no tensor cores on purpose.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace rs {

// ------------------------------------------------------------------------------ LayerNorm
// One warp per row of d = 128*NV fp32 values held in registers (two-pass mean / variance).
// Optional second LayerNorm chained on the result (norm_out of layer i feeding
// norm_feed_forward1 of layer i+1) so the residual stream is read once.
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ g1, const float* __restrict__ b1,
                 float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16,
                 const float* __restrict__ g2, const float* __restrict__ b2, int rows, float eps) {
  // Persistent: a warp walks rows (stride = warps in the grid) with the NEXT row's loads already in flight while
  // the current one is reduced and stored -- short-lived one-row warps left HBM at ~40 % (profiles/r01_v2_other_ncu.md).
  constexpr int D = 128 * NV;
  const int lane = lane_id();
  const int wstride = gridDim.x * (blockDim.x >> 5);
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  float4 v[NV], nx[NV];
  {
    const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * D);
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = xr[lane + 32 * i];
  }

  auto normalize = [&](const float* __restrict__ g, const float* __restrict__ b) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) * (1.0f / D);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, dd = v[i].w - mean;
      ss += (a * a + bb * bb) + (c * c + dd * dd);
    }
    const float rstd = rsqrtf(warp_sum(ss) * (1.0f / D) + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + lane + 32 * i);
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b) + lane + 32 * i);
      v[i].x = (v[i].x - mean) * rstd * gg.x + bb.x;
      v[i].y = (v[i].y - mean) * rstd * gg.y + bb.y;
      v[i].z = (v[i].z - mean) * rstd * gg.z + bb.z;
      v[i].w = (v[i].w - mean) * rstd * gg.w + bb.w;
    }
  };

  for (; row < rows; row += wstride) {
    const int nrow = row + wstride;
    if (nrow < rows) {                                         // warp-uniform
      const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(nrow) * D);
#pragma unroll
      for (int i = 0; i < NV; ++i) nx[i] = xr[lane + 32 * i];
    }
    normalize(g1, b1);
    if (out_f32 != nullptr) {
      float4* o = reinterpret_cast<float4*>(out_f32 + static_cast<size_t>(row) * D);
#pragma unroll
      for (int i = 0; i < NV; ++i) o[lane + 32 * i] = v[i];
    }
    if (g2 != nullptr) normalize(g2, b2);
    if (out_bf16 != nullptr) {
      uint2* o = reinterpret_cast<uint2*>(out_bf16 + static_cast<size_t>(row) * D);
#pragma unroll
      for (int i = 0; i < NV; ++i) o[lane + 32 * i] = make_uint2(pack_bf16x2(v[i].x, v[i].y), pack_bf16x2(v[i].z, v[i].w));
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = nx[i];
  }
}

cudaError_t launch_layernorm(const float* x, const float* gamma, const float* beta, float* out_f32, void* out_bf16,
                             const float* gamma2, const float* beta2, int rows, int d, float eps, cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  const int wpb = 8;
  int num_sms = 0, dev = 0;                                    // per call: engines on different devices share this code
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || num_sms <= 0) num_sms = 132;
  const int need = (rows + wpb - 1) / wpb;
  const int cap = num_sms * 2;                                 // 2 resident CTAs per SM (16 warps x 2 rows in flight)
  auto* ob = static_cast<__nv_bfloat16*>(out_bf16);
  const dim3 grid(need < cap ? need : cap), block(32 * wpb);
  switch (d) {
    case 256: layernorm_kernel<2><<<grid, block, 0, stream>>>(x, gamma, beta, out_f32, ob, gamma2, beta2, rows, eps); break;
    case 512: layernorm_kernel<4><<<grid, block, 0, stream>>>(x, gamma, beta, out_f32, ob, gamma2, beta2, rows, eps); break;
    case 1024: layernorm_kernel<8><<<grid, block, 0, stream>>>(x, gamma, beta, out_f32, ob, gamma2, beta2, rows, eps); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------ conv module middle
// u: GLU output, bf16 [B, T_max, d].  Frames t >= len[b] read as zero (masked_fill before the
// depthwise conv); t < 0 is the conv's own zero padding.  BatchNorm(eval) is folded at pack time:
// w'[j][c] = w[c][j] * gamma/sqrt(var+eps),  shift[c] = (bias - mean) * gamma/sqrt(var+eps) + beta.
template <int KW, int TT>
__global__ void __launch_bounds__(256)
conv_dw_kernel(const __nv_bfloat16* __restrict__ u, __nv_bfloat16* __restrict__ out, const float* __restrict__ w,
               const float* __restrict__ shift, const int32_t* __restrict__ len, int T_max, int d) {
  // Four channels per thread (8-byte accesses), TT output frames per thread.  All TT + KW - 1 input rows of the
  // thread are requested before the first one is used (one round trip to L2 / HBM instead of one per few frames:
  // the earlier four-rows-at-a-time version sat at ~1.4 TB/s); they stay packed (bf16) in registers and are
  // unpacked into the KW-row sliding window as it advances.
  constexpr int PAD = (KW - 1) / 2;
  constexpr int ROWS = TT + KW - 1;
  const int b = blockIdx.z;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (c >= d) return;
  const int t0 = blockIdx.y * TT;
  const int n = len[b];
  const __nv_bfloat16* base = u + (static_cast<size_t>(b) * T_max) * d + c;
  uint2 raw[ROWS];
#pragma unroll
  for (int j = 0; j < ROWS; ++j) {
    const int t = t0 - PAD + j;
    raw[j] = (t >= 0 && t < n) ? __ldg(reinterpret_cast<const uint2*>(base + static_cast<size_t>(t) * d)) : make_uint2(0u, 0u);
  }
  float4 wt[KW];
#pragma unroll
  for (int j = 0; j < KW; ++j) wt[j] = __ldg(reinterpret_cast<const float4*>(w + static_cast<size_t>(j) * d + c));
  const float4 sh = __ldg(reinterpret_cast<const float4*>(shift + c));
  auto unpack = [](uint2 v) { return make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y)); };
  float4 win[KW];
#pragma unroll
  for (int j = 0; j < KW - 1; ++j) win[j + 1] = unpack(raw[j]);
#pragma unroll
  for (int q = 0; q < TT; ++q) {
#pragma unroll
    for (int j = 0; j < KW - 1; ++j) win[j] = win[j + 1];
    win[KW - 1] = unpack(raw[q + KW - 1]);
    float4 a = sh;
#pragma unroll
    for (int j = 0; j < KW; ++j) {
      a.x = fmaf(win[j].x, wt[j].x, a.x); a.y = fmaf(win[j].y, wt[j].y, a.y);
      a.z = fmaf(win[j].z, wt[j].z, a.z); a.w = fmaf(win[j].w, wt[j].w, a.w);
    }
    if (t0 + q < T_max)
      *reinterpret_cast<uint2*>(out + (static_cast<size_t>(b) * T_max + t0 + q) * d + c) =
          make_uint2(pack_bf16x2(swishf_fast(a.x), swishf_fast(a.y)), pack_bf16x2(swishf_fast(a.z), swishf_fast(a.w)));
  }
}

cudaError_t launch_conv_dw(const void* u, void* out, const float* w, const float* shift, const int32_t* enc_len,
                           int B, int T_max, int d, int k, cudaStream_t stream) {
  if (k != 9 || (d & 3)) return cudaErrorInvalidValue;
  constexpr int TT = 8;
  const int threads = d / 4 < 256 ? d / 4 : 256;
  const dim3 block(threads), grid((d / 4 + threads - 1) / threads, (T_max + TT - 1) / TT, B);
  conv_dw_kernel<9, TT><<<grid, block, 0, stream>>>(static_cast<const __nv_bfloat16*>(u), static_cast<__nv_bfloat16*>(out),
            w, shift, enc_len, T_max, d);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------ utilities
__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t n) {
  int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i + 3 < n) {
    const float4 v = *reinterpret_cast<const float4*>(in + i);
    *reinterpret_cast<uint2*>(out + i) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  } else {
    for (; i < n; ++i) out[i] = __float2bfloat16_rn(in[i]);
  }
}
cudaError_t launch_f32_to_bf16(const float* in, void* out, int64_t n, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const int threads = 256;
  const int64_t blocks = (n / 4 + threads) / threads;
  f32_to_bf16_kernel<<<static_cast<unsigned>(blocks), threads, 0, stream>>>(in, static_cast<__nv_bfloat16*>(out), n);
  return cudaGetLastError();
}

// Zero rows t >= len[b] of a padded fp32 [B, T_max, d] tensor (final encoder output hygiene).
__global__ void zero_pad_rows_kernel(float* __restrict__ x, const int32_t* __restrict__ len, int T_max, int d) {
  const int b = blockIdx.y, t = blockIdx.x;
  if (t < len[b]) return;
  float4* r = reinterpret_cast<float4*>(x + (static_cast<size_t>(b) * T_max + t) * d);
  for (int i = threadIdx.x; i < d / 4; i += blockDim.x) r[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}
cudaError_t launch_zero_pad_rows(float* x, const int32_t* len, int B, int T_max, int d, cudaStream_t stream) {
  zero_pad_rows_kernel<<<dim3(T_max, B), 128, 0, stream>>>(x, len, T_max, d);
  return cudaGetLastError();
}

}  // namespace rs
