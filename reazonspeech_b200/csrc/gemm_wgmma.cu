// Persistent, warp-specialised bf16 GEMM for sm_90a:  out = epi(A[M,K] * W[N,K]^T)
//
//   warpgroup 0     TMA producer   one thread: cp.async.bulk.tensor 2-D tiles (128B swizzle) -> smem ring; the warpgroup
//                                  hands most of its registers to the consumers (setmaxnreg)
//   warpgroups 1,2  consumers      each owns 64 rows of the 128 x BN tile: wgmma.mma_async m64nBNk16 straight from the ring,
//                                  fp32 accumulators in registers, then the fused epilogue (bias / activation / GLU /
//                                  V^T) in registers, written as 64-row subtiles into swizzled shared buffers from which
//                                  one thread issues TMA stores (the residual: a TMA f32 add into out, done in L2).  The
//                                  stores drain while the warpgroup runs the next tile's main loop; the tile's bias slice
//                                  arrives by cp.async during that loop.  Rows past M are clipped by the tensor maps.
//
// Two instances of the one kernel body:
//   BN = 256  128 fp32 accumulators per consumer thread (the producer's registers moved over with setmaxnreg); a CTA
//             pulls 48 KB from L2 per 4.2 MFLOP k-block (85 FLOP/B, against 64 for a 128 x 128 tile).
//   BN = 64   for launches whose 256-wide tiling would not give every SM a tile or would leave part of its last W tile
//             empty (the ALSD search's products, single-clip encoder passes, N = 640): more, smaller tiles.
// Both run the same k16 steps in the same k order with fp32 accumulation and the same epilogue operations, so a row's
// result does not depend on which instance computed it.
//
// Covers every dense contraction of the FastConformer encoder (SURVEY.md App. A.3): FFN W1/W2,
// fused QKV, attention out-proj, conv pointwise 1/2, the subsampling 1x1 convs and out-linear,
// and the joint's encoder projection.  Replaces the cuBLAS fp32 GEMMs NeMo dispatches under
// model.transcribe (pkg/nemo-asr/src/transcribe.py:48-53).
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../include/rs_engine.h"
#include "common.cuh"
#include "kernels.h"

namespace rs {

constexpr int BM = 128;
constexpr int BK = 64;                 // 64 bf16 = 128 B = one swizzle atom row
constexpr int kConsumerWarps = 8;      // two warpgroups
constexpr int kGemmThreads = 128 + 32 * kConsumerWarps;
constexpr int kABytes = BM * BK * 2;   // 16 KiB
// Epilogue subtile of one consumer warpgroup: its 64 rows x 64 B (32 bf16 / f16 or 16 f32 columns, 64 B swizzle), or for
// V^T 32 head dims x 64 frames (128 B swizzle).  Three buffers per warpgroup: one is written while the stores of the other
// two drain.
constexpr int kEpiBufs = 3, kEpiBufBytes = 4096;
constexpr int kBiasBytes = 256 * 4;    // the tile's bias slice, one copy per warpgroup
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K registers

struct GemmDev {
  const float* bias;
  int M, N, K;
  int epilogue;
  float alpha;
  int split;            // RS_EPI_QKV_VT
};
template <int BN>
struct GemmCfg {
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiBytes = 2 * (kEpiBufs * kEpiBufBytes + kBiasBytes);
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/ + kEpiBytes;
  static constexpr int kStages = (227 * 1024 - kFixedBytes) / kStageBytes;   // 4 (BN = 256), 8 (BN = 64)
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(2 * 8 * kStages <= 256, "barrier area");
  static_assert(kStageBytes % 1024 == 0, "epilogue buffers need the 1024 B alignment of the 128 B swizzle");
};

// Byte offset of 16-byte group `chunk` of row `row` in a 64 B-pitch buffer with the tensor map's 64 B swizzle
// (address bits [4,6) ^= bits [7,9)): the eight rows a stmatrix matrix or a half-warp's f32 stores touch land in distinct banks.
__device__ __forceinline__ uint32_t sw64(int row, int chunk) { return static_cast<uint32_t>(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4)); }

template <int BN, int EG>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                    const __grid_constant__ CUtensorMap tm_out, const __grid_constant__ CUtensorMap tm_out2, const GemmDev p) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled operand tiles need 1024 B alignment.
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t epi_base = smem_base + Cfg::kStages * Cfg::kStageBytes;   // 2 x 3 subtile buffers, then 2 bias slices
  const uint32_t bar_base = epi_base + Cfg::kEpiBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };
  auto smem_a = [&](int s) { return smem_base + s * Cfg::kStageBytes; };
  auto smem_b = [&](int s) { return smem_base + s * Cfg::kStageBytes + kABytes; };
  auto smem_gen = [&](uint32_t addr) { return smem_raw + (addr - smem_u32(smem_raw)); };

  const int warp = warp_id_uniform();
  const int lane = lane_id();
  const int num_m = (p.M + BM - 1) / BM;
  const int num_n = (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_k = p.K / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    tma_prefetch_desc(&tm_out);
    if constexpr (EG == 1) tma_prefetch_desc(&tm_out2);
    for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          mbar_arrive_expect_tx(full_bar(stage), Cfg::kStageBytes);
          tma_load_2d(smem_a(stage), &tm_a, kb * BK, m0, full_bar(stage));
          tma_load_2d(smem_b(stage), &tm_b, kb * BK, n0, full_bar(stage));
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<kConsumerRegs>();
    const int cw = warp - 4;                                   // consumer warp 0..7
    const int wg = cw >> 2, wq = cw & 3;                       // warpgroup, warp within it
    const int rows0 = wg * 64;                                 // the warpgroup's rows of the tile
    const int tw = threadIdx.x & 127;                          // thread within the warpgroup; 0 issues its TMA stores
    const uint32_t buf0 = epi_base + wg * kEpiBufs * kEpiBufBytes;
    float* bias_s = reinterpret_cast<float*>(smem_gen(epi_base + 2 * kEpiBufs * kEpiBufBytes + wg * kBiasBytes));
    const int g = lane >> 2, t = lane & 3;
    const int mi = lane >> 3, mr = lane & 7;                   // the stmatrix matrix and row this lane addresses
    int nbuf = 0;                                              // the buffer the next subtile is written into
    auto buf = [&]() { return buf0 + nbuf * kEpiBufBytes; };
    // Hand the written buffer to one TMA store (or f32 add).  Once the barrier is passed, every store but the last has
    // finished reading shared memory, so the buffer after this one is free for the next subtile.
    auto flush = [&](const CUtensorMap* map, int c0, int c1, bool reduce) {
      fence_proxy_async();
      if (tw == 0) bulk_wait_read<kEpiBufs - 2>();
      named_bar_sync(1 + wg, 128);
      if (tw == 0) {
        if (reduce) tma_reduce_add_2d(map, buf(), c0, c1);
        else tma_store_2d(map, buf(), c0, c1);
        bulk_commit();
      }
      nbuf = nbuf == kEpiBufs - 1 ? 0 : nbuf + 1;
    };

    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
      // The tile's bias slice lands during the main loop.  The previous epilogue's last barrier ordered its reads before this.
      if (4 * tw < min(BN, p.N - n0)) {
        if (p.bias != nullptr) cp_async16(bias_s + 4 * tw, p.bias + n0 + 4 * tw);
        else *reinterpret_cast<float4*>(bias_s + 4 * tw) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      float d[BN / 2];
      int prev = -1;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint64_t da = wgmma_desc_k_sw128(smem_a(stage) + rows0 * 128);
        const uint64_t db = wgmma_desc_k_sw128(smem_b(stage));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          if constexpr (BN == 256) wgmma_bf16_ss_n256(d, da + 2u * k, db + 2u * k, (kb | k) != 0 ? 1u : 0u);
          else wgmma_bf16_ss_n64(d, da + 2u * k, db + 2u * k, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                                       // the previous k-block's MMAs have retired: its slot is reusable
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      cp_async_wait_all();
      named_bar_sync(1 + wg, 128);                             // every thread's share of the bias slice has landed

      // ---- epilogue: 32-column chunks of the warpgroup's 64 rows, in registers, then through the buffers to TMA
      const int row_g = m0 + rows0;
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        const int col0 = n0 + c * 32;
        if (col0 < p.N) {                                      // warpgroup-uniform
          // v[j][h][x]: row 16 wq + g + 8h of the warpgroup, column 32c + 8j + 2t + x of the tile, bias added
          float v[4][2][2];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 b = *reinterpret_cast<const float2*>(bias_s + 32 * c + 8 * j + 2 * t);
#pragma unroll
            for (int h = 0; h < 2; ++h) { v[j][h][0] = d[16 * c + 4 * j + 2 * h] + b.x; v[j][h][1] = d[16 * c + 4 * j + 2 * h + 1] + b.y; }
          }
          const int epi = EG == 1 ? RS_EPI_QKV_VT : p.epilogue;
          if (EG == 1 && col0 >= p.split) {
            // V columns -> out2[col - split][row]: each 8 x 8 block stored transposed; buffer row = head dim (64 frames,
            // 128 B, 128 B swizzle), this warp's 16 frames are its 16-byte groups 2 wq and 2 wq + 1.
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const int dim = 8 * (2 * q + (mi >> 1)) + mr;
              stmatrix_x4_trans(buf() + dim * 128 + (((2 * wq + (mi & 1)) ^ mr) << 4),
                                pack_bf16x2(v[2 * q][0][0], v[2 * q][0][1]), pack_bf16x2(v[2 * q][1][0], v[2 * q][1][1]),
                                pack_bf16x2(v[2 * q + 1][0][0], v[2 * q + 1][0][1]), pack_bf16x2(v[2 * q + 1][1][0], v[2 * q + 1][1][1]));
            }
            flush(&tm_out2, row_g, col0 - p.split, false);
          } else if (epi == RS_EPI_BIAS_GLU_BF16) {
            // columns [0,16) of the chunk are values, [16,32) the matching gates (weights interleaved at pack time); two
            // chunks make one 32-column output subtile
            uint32_t r[2][2];
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
              for (int h = 0; h < 2; ++h)
                r[j][h] = pack_bf16x2(v[j][h][0] * sigmoidf_fast(v[j + 2][h][0]), v[j][h][1] * sigmoidf_fast(v[j + 2][h][1]));
            stmatrix_x4(buf() + sw64(16 * wq + 8 * (mi & 1) + mr, 2 * (c & 1) + (mi >> 1)), r[0][0], r[0][1], r[1][0], r[1][1]);
            if ((c & 1) || col0 + 32 >= p.N) flush(&tm_out, (col0 & ~63) / 2, row_g, false);
          } else if (epi == RS_EPI_BIAS_F32 || epi == RS_EPI_RESID_F32) {
            // alpha (acc + bias) as two 16-column subtiles.  Lanes with bit 1 of g set store their column pairs in the other
            // order, so that each half-warp's 8-byte stores cover all 32 banks.
            const bool swp = (g >> 1) & 1;
#pragma unroll
            for (int s = 0; s < 2; ++s) {
#pragma unroll
              for (int k = 0; k < 2; ++k) {
                const int jl = k ^ static_cast<int>(swp);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int row = 16 * wq + g + 8 * h;
                  const float a0 = jl ? v[2 * s + 1][h][0] : v[2 * s][h][0], a1 = jl ? v[2 * s + 1][h][1] : v[2 * s][h][1];
                  *reinterpret_cast<float2*>(smem_gen(buf() + sw64(row, 2 * jl + (t >> 1)) + 8 * (t & 1))) =
                      make_float2(a0 * p.alpha, a1 * p.alpha);
                }
              }
              flush(&tm_out, col0 + 16 * s, row_g, epi == RS_EPI_RESID_F32);
            }
          } else {
            // bf16 / f16: q | k columns of RS_EPI_QKV_VT, RS_EPI_BIAS_BF16 / RELU / SWISH / F16
            uint32_t r[4][2];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float x0 = v[j][h][0], x1 = v[j][h][1];
                if (epi == RS_EPI_BIAS_RELU_BF16) { x0 = fmaxf(x0, 0.0f); x1 = fmaxf(x1, 0.0f); }
                else if (epi == RS_EPI_BIAS_SWISH_BF16) { x0 = swishf_fast(x0); x1 = swishf_fast(x1); }
                r[j][h] = epi == RS_EPI_BIAS_F16 ? pack_f16x2(x0, x1) : pack_bf16x2(x0, x1);
              }
#pragma unroll
            for (int q = 0; q < 2; ++q)
              stmatrix_x4(buf() + sw64(16 * wq + 8 * (mi & 1) + mr, 2 * q + (mi >> 1)),
                          r[2 * q][0], r[2 * q][1], r[2 * q + 1][0], r[2 * q + 1][1]);
            flush(&tm_out, col0, row_g, false);
          }
        }
      }
    }
    if (tw == 0) bulk_wait<0>();
  }
}

// ---------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D map over a row-major [rows, cols] array (row pitch ld elements of esize bytes) with a box_rows x box_cols box.
static bool make_tmap_2d(CUtensorMap* m, CUtensorMapDataType dtype, int esize, const void* ptr, uint64_t rows, uint64_t cols,
                         uint64_t ld, uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle, char* err) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) { snprintf(err, 256, "cuTensorMapEncodeTiled entry point unavailable"); return false; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * esize};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, dtype, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(err, 256, "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu", (int)r, (unsigned long long)rows, (unsigned long long)cols); return false; }
  return true;
}

bool make_tmap_bf16(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, char* err) {
  return make_tmap_2d(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, rows, cols, ld, BK, box_rows, CU_TENSOR_MAP_SWIZZLE_128B, err);
}

inline int epilogue_group(int epilogue) { return epilogue == RS_EPI_QKV_VT ? 1 : 0; }

template <int BN, int EG>
static cudaError_t launch_bn_eg(const GemmArgs& g, int num_sms, cudaStream_t stream, char* err) {
  using Cfg = GemmCfg<BN>;
  static DeviceOnce attr_once;
  if (attr_once.pending()) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_tn_kernel<BN, EG>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) { snprintf(err, 256, "cudaFuncSetAttribute(smem=%d): %s", Cfg::kSmemBytes, cudaGetErrorString(e)); return e; }
    attr_once.set();
  }
  CUtensorMap tm_a, tm_b, tm_out, tm_out2;
  if (!make_tmap_bf16(&tm_a, g.a, g.M, g.K, g.K, BM, err)) return cudaErrorInvalidValue;
  if (!make_tmap_bf16(&tm_b, g.w, g.N, g.K, g.K, BN, err)) return cudaErrorInvalidValue;
  // Output: 64-row subtiles of 64 B (16 f32 or 32 two-byte columns); the GLU writes N / 2 columns.
  const bool f32 = g.epilogue == RS_EPI_RESID_F32 || g.epilogue == RS_EPI_BIAS_F32;
  const int ldo = g.epilogue == RS_EPI_BIAS_GLU_BF16 ? g.N / 2 : g.N;
  const CUtensorMapDataType dt = f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                     : g.epilogue == RS_EPI_BIAS_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (!make_tmap_2d(&tm_out, dt, f32 ? 4 : 2, g.out, g.M, ldo, ldo, f32 ? 16 : 32, 64, CU_TENSOR_MAP_SWIZZLE_64B, err)) return cudaErrorInvalidValue;
  // V^T: [N - split head dims, M frames] with row pitch ld2, 32 x 64 boxes; frames >= M are outside the map and untouched.
  if (EG == 1 && !make_tmap_2d(&tm_out2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, g.out2, g.N - g.split, g.M, g.ld2, 64, 32,
                               CU_TENSOR_MAP_SWIZZLE_128B, err))
    return cudaErrorInvalidValue;
  if (EG == 0) tm_out2 = tm_out;                             // not read
  GemmDev p{g.bias, g.M, g.N, g.K, g.epilogue, g.alpha, g.split};
  const int tiles = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN);
  const int grid = tiles < num_sms ? tiles : num_sms;
  gemm_bf16_tn_kernel<BN, EG><<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(tm_a, tm_b, tm_out, tm_out2, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) snprintf(err, 256, "gemm launch (M=%d N=%d K=%d BN=%d): %s", g.M, g.N, g.K, BN, cudaGetErrorString(e));
  return e;
}

template <int BN>
static cudaError_t launch_bn(const GemmArgs& g, int num_sms, cudaStream_t stream, char* err) {
  switch (epilogue_group(g.epilogue)) {
    case 1: return launch_bn_eg<BN, 1>(g, num_sms, stream, err);
    default: return launch_bn_eg<BN, 0>(g, num_sms, stream, err);
  }
}

cudaError_t launch_gemm(const GemmArgs& g, int num_sms, cudaStream_t stream, char* err) {
  if (g.M <= 0 || g.N <= 0 || g.K <= 0 || g.K % BK != 0 || g.N % 32 != 0) {
    snprintf(err, 256, "gemm shape unsupported: M=%d N=%d K=%d (need K%%64==0, N%%32==0)", g.M, g.N, g.K);
    return cudaErrorInvalidValue;
  }
  if ((reinterpret_cast<uintptr_t>(g.a) | reinterpret_cast<uintptr_t>(g.w) | reinterpret_cast<uintptr_t>(g.out) |
       reinterpret_cast<uintptr_t>(g.bias) | reinterpret_cast<uintptr_t>(g.out2)) & 15u) {
    snprintf(err, 256, "gemm operands, bias and outputs must be 16-byte aligned");
    return cudaErrorInvalidValue;
  }
  if (g.epilogue == RS_EPI_RESID_F32 && g.resid == nullptr) { snprintf(err, 256, "gemm: residual epilogue without resid"); return cudaErrorInvalidValue; }
  if (g.epilogue == RS_EPI_QKV_VT && (g.out2 == nullptr || g.split % 32 || g.ld2 % 8 || g.M % 8 || g.ld2 < g.M)) {
    snprintf(err, 256, "gemm: RS_EPI_QKV_VT needs out2, split %% 32 == 0, ld2 %% 8 == 0, M %% 8 == 0, ld2 >= M");
    return cudaErrorInvalidValue;
  }
  // The residual epilogue adds into out in place (a TMA reduction); a separate resid is copied to out first.
  if (g.epilogue == RS_EPI_RESID_F32 && g.resid != g.out) {
    cudaError_t e = cudaMemcpyAsync(g.out, g.resid, static_cast<size_t>(g.M) * g.N * sizeof(float), cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) { snprintf(err, 256, "gemm: residual copy: %s", cudaGetErrorString(e)); return e; }
  }
  // 256-wide tiles when N fills them and they give every SM a tile, else 64-wide ones on more SMs.  The two instances
  // compute every element alike, so the choice (which depends on M) cannot make a row's result depend on the batch it
  // sits in (tests/test_gpu_gemm_cluster.py).
  if (g.N % 256 == 0 && ((g.M + BM - 1) / BM) * (g.N / 256) >= num_sms) return launch_bn<256>(g, num_sms, stream, err);
  return launch_bn<64>(g, num_sms, stream, err);
}

}  // namespace rs
