// ConvSubsampling (dw_striding, x8) direct-convolution parts (N2).  NeMo reference module:
// parts/submodules/subsampling.py ConvSubsampling (reached via model.transcribe,
// pkg/nemo-asr/src/transcribe.py:48-53).  The 1x1 convs and the output Linear run on the
// wgmma GEMM over channels-last activations; this file holds the HBM-bound 3x3 convs.
//
// Kernel A fuses the per-feature normalisation of the log-mel features (statistics from logmel.cu), conv.0
// (1->C, 3x3, s2, p1) + ReLU + conv.2 (depthwise 3x3, s2, p1): the
// [B, T1, 40, C] intermediate (1 GB at 32 x 30 s in bf16) never reaches HBM.  One thread per
// channel; the mel patch of the tile sits in shared memory and is read as a warp broadcast.
// Every stage treats frames at or beyond the utterance's length at that stage as zero, which is
// what batch=1 execution sees as conv zero-padding (padding invariance, SURVEY.md finding 4).
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace rs {

// floor((n - 1) / 2) + 1 as NeMo's calc_length computes it: 0 frames stay 0 (C division would truncate -1/2 to 0 and give 1)
__host__ __device__ __forceinline__ int conv_len(int n) { return n > 0 ? (n - 1) / 2 + 1 : 0; }

constexpr int kSubTT = 4;     // t2 rows per CTA
constexpr int kMelOff = 4;    // smem column of mel bin 0 (bin -1 sits at column 3) so bins 4k..4k+3 are one aligned LDS.128

// One thread per channel.  For output (t2, f2) the depthwise 3x3 needs conv.0 at t1 = 2*t2-1..2*t2+1 and
// f1 = 2*f2-1..2*f2+1, i.e. mel rows 4*t2-3..4*t2+3 (7 rows) and mel bins 4*f2-3..4*f2+3.  Sliding along f2
// the 7 x 4 new mel values of a step are fetched with seven 128-bit broadcast loads and kept in registers
// together with the previous step's last three columns, and conv.0 at f1 = 2*f2-1 is carried over from
// the previous step: per output 7 LDS.128 + 63 FMA instead of 54 scalar shared loads.
// LDC: the shared-memory row pitch as a compile-time constant (0: run-time).  With it the 7 row loads of a step are one base
// register + immediates; the run-time pitch cost an IMAD / LEA pair per load (30 of the 140 instructions of a step).
template <int LDC>
__global__ void __launch_bounds__(256)
sub_conv0_dw1_kernel(const float* __restrict__ mel, const int32_t* __restrict__ mel_len, const float* __restrict__ mel_stats,
                     int F_max, int n_mels, int C,
                     const float* __restrict__ w0, const float* __restrict__ b0, const float* __restrict__ wd,
                     const float* __restrict__ bd, __nv_bfloat16* __restrict__ out, int T2, int F1, int F2) {
  extern __shared__ __align__(16) float s_mel[];         // [(4*TT+3)][ld], column kMelOff + bin
  const int b = blockIdx.y;
  const int t2_0 = blockIdx.x * kSubTT;
  const int len0 = mel_len[b];
  const int len1 = conv_len(len0);
  const int len2 = conv_len(len1);
  const int rows = 4 * kSubTT + 3;
  const int ld = LDC > 0 ? LDC : ((n_mels + kMelOff + 4 + 3) / 4) * 4;   // bins -4 .. n_mels+3 addressable, multiple of 4 floats
  const int t0_base = 4 * t2_0 - 3;                      // first mel row needed: 2*(2*t2_0-1)-1
  // The log-mel kernel leaves the features un-normalised next to their per-utterance statistics (logmel.cu): NeMo's
  // per-feature normalisation (x - mean) / (std + eps) and its zero tail (frames >= len read as 0, which is also the
  // convolution's zero padding at batch = 1) are applied here, while the patch is staged.
  const float* st = mel_stats != nullptr ? mel_stats + static_cast<size_t>(b) * n_mels * 2 : nullptr;   // nullptr: already normalised (rs_encode)
  for (int i = threadIdx.x; i < rows * ld; i += blockDim.x) {
    const int r = i / ld, bin = i % ld - kMelOff;
    const int t0 = t0_base + r;
    float v = 0.f;
    if (t0 >= 0 && t0 < len0 && t0 < F_max && bin >= 0 && bin < n_mels) {
      v = mel[(static_cast<size_t>(b) * F_max + t0) * n_mels + bin];
      if (st != nullptr) v = (v - __ldg(st + 2 * bin)) * __ldg(st + 2 * bin + 1);
    }
    s_mel[i] = v;
  }
  __syncthreads();

  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float k0[9], kd[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) { k0[j] = __ldg(w0 + c * 9 + j); kd[j] = __ldg(wd + c * 9 + j); }
    const float bias0 = __ldg(b0 + c), biasd = __ldg(bd + c);
    for (int tt = 0; tt < kSubTT; ++tt) {
      const int t2 = t2_0 + tt;
      if (t2 >= T2) break;
      __nv_bfloat16* orow = out + ((static_cast<size_t>(b) * T2 + t2) * F2) * C + c;
      if (t2 >= len2) {                                   // padded frame: defined value, never read as valid
        for (int f2 = 0; f2 < F2; ++f2) orow[static_cast<size_t>(f2) * C] = __float2bfloat16_rn(0.f);
        continue;
      }
      // validity of the three conv.0 rows t1 = 2*t2-1+dt (dw zero padding / frames beyond the utterance)
      bool tv[3];
#pragma unroll
      for (int dt = 0; dt < 3; ++dt) { const int t1 = 2 * t2 - 1 + dt; tv[dt] = t1 >= 0 && t1 < len1; }
      const float* base = s_mel + (4 * tt) * ld + kMelOff;   // mel row 4*t2-3 of this t2, bin 0
      float m[7][7];                                       // mel[row 4*t2-3+i][bin 4*f2-3+j]
#pragma unroll
      for (int i = 0; i < 7; ++i) {                        // f2 = 0: bins -3..-1 are zero padding
        m[i][0] = m[i][1] = m[i][2] = 0.f;
        m[i][3] = 0.f;
      }
      float left[3] = {0.f, 0.f, 0.f};                    // conv.0 at f1 = 2*f2-1 (carried from the previous step)
      // interior frames (all three conv.0 rows exist, F1 == 2 * F2) take a path without the per-element validity selects
      auto run = [&](auto all_valid) {
        constexpr bool kAll = decltype(all_valid)::value;
#pragma unroll 1
        for (int f2 = 0; f2 < F2; ++f2) {
#pragma unroll
          for (int i = 0; i < 7; ++i) {
            const float4 q = *reinterpret_cast<const float4*>(base + i * ld + 4 * f2);   // bins 4*f2 .. 4*f2+3
            m[i][3] = q.x; m[i][4] = q.y; m[i][5] = q.z; m[i][6] = q.w;
          }
          // conv.0 at f1 = 2*f2 (bins 4f2-1..4f2+1 -> m cols 2..4) and f1 = 2*f2+1 (bins 4f2+1..4f2+3 -> m cols 4..6)
          float mid[3], right[3];
#pragma unroll
          for (int dt = 0; dt < 3; ++dt) {
            float a0 = bias0, a1 = bias0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
              for (int j = 0; j < 3; ++j) {
                a0 = fmaf(m[2 * dt + i][2 + j], k0[i * 3 + j], a0);
                a1 = fmaf(m[2 * dt + i][4 + j], k0[i * 3 + j], a1);
              }
            mid[dt] = (kAll || (tv[dt] && 2 * f2 < F1)) ? fmaxf(a0, 0.f) : 0.f;
            right[dt] = (kAll || (tv[dt] && 2 * f2 + 1 < F1)) ? fmaxf(a1, 0.f) : 0.f;
          }
          float a = biasd;
#pragma unroll
          for (int dt = 0; dt < 3; ++dt) {
            a = fmaf(left[dt], kd[dt * 3 + 0], a);
            a = fmaf(mid[dt], kd[dt * 3 + 1], a);
            a = fmaf(right[dt], kd[dt * 3 + 2], a);
            left[dt] = right[dt];
          }
          orow[static_cast<size_t>(f2) * C] = __float2bfloat16_rn(a);
#pragma unroll
          for (int i = 0; i < 7; ++i) { m[i][2] = m[i][6]; }  // bin 4*f2+3 becomes bin 4*(f2+1)-1 (bin -1 of the first step is the zero set above)
        }
      };
      if (tv[0] && tv[1] && tv[2] && F1 == 2 * F2) run(std::true_type{});
      else run(std::false_type{});
    }
  }
}

cudaError_t launch_sub_conv0_dw1(const SubsampleArgs& a, cudaStream_t stream) {
  const int ld = ((a.n_mels + kMelOff + 4 + 3) / 4) * 4;
  const size_t smem = static_cast<size_t>(4 * kSubTT + 3) * ld * sizeof(float);
  const dim3 grid((a.T2 + kSubTT - 1) / kSubTT, a.B);
  if (ld == 88)                                            // 80 mel bins: every shipped configuration
    sub_conv0_dw1_kernel<88><<<grid, 256, smem, stream>>>(a.mel, a.mel_len, a.mel_stats, a.F_max, a.n_mels, a.C, a.w0, a.b0, a.wd1, a.bd1,
                                                         static_cast<__nv_bfloat16*>(a.out1), a.T2, a.F1, a.F2);
  else
    sub_conv0_dw1_kernel<0><<<grid, 256, smem, stream>>>(a.mel, a.mel_len, a.mel_stats, a.F_max, a.n_mels, a.C, a.w0, a.b0, a.wd1, a.bd1,
                                                        static_cast<__nv_bfloat16*>(a.out1), a.T2, a.F1, a.F2);
  return cudaGetLastError();
}

// Depthwise 3x3 s2 p1 on channels-last bf16 [B, Tin, Fin, C] -> [B, Tout, Fout, C].
// The valid input length of utterance b is conv_len applied `len_shift` times to mel_len[b].
// One thread = eight channels of one output frame, ALL Fout frequency bins: the 72 tap weights are fetched once per
// thread instead of once per output (the one-output-per-thread version issued as many weight loads as FMAs and ran at
// a sixth of the HBM rate), and the input column shared by neighbouring bins (stride 2, kernel 3) is reused from registers.
constexpr int kDwThreads = 128;
__global__ void __launch_bounds__(kDwThreads)
sub_dw_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, const float* __restrict__ w,
              const float* __restrict__ bias, const int32_t* __restrict__ mel_len, int len_shift, int Tin, int Fin,
              int Tout, int Fout, int C) {
  const int b = blockIdx.z;
  int lin = mel_len[b];
  for (int i = 0; i < len_shift; ++i) lin = conv_len(lin);
  const int lout = conv_len(lin);
  const int c8 = C / 8;
  const int t = blockIdx.y * (kDwThreads / c8) + threadIdx.x / c8;   // a block covers kDwThreads / c8 whole frames
  const int c = (threadIdx.x % c8) * 8;
  if (t >= Tout) return;
  __nv_bfloat16* orow = out + ((static_cast<size_t>(b) * Tout + t) * Fout) * C + c;
  if (t >= lout) {
    for (int f = 0; f < Fout; ++f) *reinterpret_cast<uint4*>(orow + static_cast<size_t>(f) * C) = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  float wt[9][8], bs[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    bs[k] = __ldg(bias + c + k);
#pragma unroll
    for (int q = 0; q < 9; ++q) wt[q][k] = __ldg(w + (c + k) * 9 + q);
  }
  // input rows 2t-1, 2t, 2t+1 (absent rows read as zero)
  const __nv_bfloat16* rowp[3];
  bool rok[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int ti = 2 * t - 1 + i;
    rok[i] = ti >= 0 && ti < lin && ti < Tin;
    rowp[i] = in + ((static_cast<size_t>(b) * Tin + (rok[i] ? ti : 0)) * Fin) * C + c;
  }
  auto load_col = [&](int fi, float (&col)[3][8]) {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (rok[i] && fi >= 0 && fi < Fin) v = __ldg(reinterpret_cast<const uint4*>(rowp[i] + static_cast<size_t>(fi) * C));
      const uint32_t vw[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) { col[i][2 * k] = bf16_lo(vw[k]); col[i][2 * k + 1] = bf16_hi(vw[k]); }
    }
  };
  float left[3][8], mid[3][8], right[3][8];
  load_col(-1, left);
  for (int f = 0; f < Fout; ++f) {
    load_col(2 * f, mid);
    load_col(2 * f + 1, right);
    float a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float s = bs[k];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        s = fmaf(left[i][k], wt[i * 3 + 0][k], s);
        s = fmaf(mid[i][k], wt[i * 3 + 1][k], s);
        s = fmaf(right[i][k], wt[i * 3 + 2][k], s);
      }
      a[k] = s;
    }
    *reinterpret_cast<uint4*>(orow + static_cast<size_t>(f) * C) =
        make_uint4(pack_bf16x2(a[0], a[1]), pack_bf16x2(a[2], a[3]), pack_bf16x2(a[4], a[5]), pack_bf16x2(a[6], a[7]));
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < 8; ++k) left[i][k] = right[i][k];
  }
}

cudaError_t launch_sub_dw(const void* in, void* out, const float* w, const float* b, const int32_t* mel_len, int len_shift,
                          int B, int Tin, int Fin, int Tout, int Fout, int C, cudaStream_t stream) {
  const int c8 = C / 8;
  if (C % 8 || c8 > kDwThreads || kDwThreads % c8) return cudaErrorInvalidValue;
  const int frames_per_block = kDwThreads / c8;
  const dim3 grid(1, (Tout + frames_per_block - 1) / frames_per_block, B);
  sub_dw_kernel<<<grid, kDwThreads, 0, stream>>>(static_cast<const __nv_bfloat16*>(in), static_cast<__nv_bfloat16*>(out), w, b,
                                                 mel_len, len_shift, Tin, Fin, Tout, Fout, C);
  return cudaGetLastError();
}

}  // namespace rs
