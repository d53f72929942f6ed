// Persistent, warp-specialised bf16 GEMM for sm_90a:  out = epi(A[M,K] * W[N,K]^T)
//
//   warpgroup 0     TMA producer   one thread: cp.async.bulk.tensor 2-D tiles (128B swizzle) -> smem ring; the warpgroup
//                                  hands most of its registers to the consumers (setmaxnreg)
//   warpgroups 1,2  consumers      each owns 64 rows of the 128 x BN tile: wgmma.mma_async m64nBNk16 straight from the ring,
//                                  fp32 accumulators in registers, then the fused epilogue (bias / activation / GLU /
//                                  residual) staged per warp through shared memory so that global stores cover whole lines;
//                                  the producer keeps filling the ring with the next tile's operands meanwhile
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
constexpr int kStageLd = 40;           // floats per staged row (160 B: 16 B-aligned; the fragment's float2 writes are conflict-free)
constexpr int kStageBytesPerWarp = 16 * kStageLd * 4;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K registers

struct GemmDev {
  const float* bias;
  const float* resid;
  void* out;
  int M, N, K;
  int epilogue;
  float alpha;
  int ldo;              // output (and residual) row stride in elements
  void* out2; int split, ld2;    // RS_EPI_QKV_VT
};
template <int BN>
struct GemmCfg {
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/ + kConsumerWarps * kStageBytesPerWarp;
  static constexpr int kStages = (227 * 1024 - kFixedBytes) / kStageBytes;   // 4 (BN = 256), 8 (BN = 64)
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(2 * 8 * kStages <= 256, "barrier area");
};

// Fused epilogue of one 16-row x 32-column chunk (one consumer warp) whose biased fp32 values sit in the warp's staging
// buffer: activation / GLU / residual, conversion, store.  The accumulator fragment gives a lane two columns of two rows;
// storing that directly would write 8- or 4-byte pieces of 16 different lines per instruction, so the chunk is re-read
// from the staging buffer in an ownership where one instruction covers whole rows of the chunk.
// EG: epilogue group compiled into a kernel instance -- 0: the common epilogues, 1: RS_EPI_QKV_VT.
template <int EG>
__device__ __forceinline__ void epilogue_store(const GemmDev& p, const float* stage, int tile_row0, int lane, int col0) {
  int epi = p.epilogue;
  if constexpr (EG == 1) {
    if (col0 < p.split) {
      epi = RS_EPI_BIAS_BF16;                                  // q | k columns: plain row-major bf16
    } else {
      // V columns: out2[col - split][row] = bf16(v).  Lane = head dim; its 16 frames are 32 contiguous bytes of out2.
      uint32_t w[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) w[r] = pack_bf16x2(stage[(2 * r) * kStageLd + lane], stage[(2 * r + 1) * kStageLd + lane]);
      __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(p.out2) + static_cast<size_t>(col0 - p.split + lane) * p.ld2 + tile_row0;
      // M is a multiple of 8 (checked at launch): frames beyond it belong to another row range of the same buffer
      if (tile_row0 < p.M) *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
      if (tile_row0 + 8 < p.M) *reinterpret_cast<uint4*>(dst + 8) = make_uint4(w[4], w[5], w[6], w[7]);
      return;
    }
  }
  switch (epi) {
    case RS_EPI_BIAS_F16:
    case RS_EPI_BIAS_BF16:
    case RS_EPI_BIAS_RELU_BF16:
    case RS_EPI_BIAS_SWISH_BF16: {
#pragma unroll
      for (int i = 0; i < 2; ++i) {                            // 8 rows x 64 B per instruction
        const int rl = i * 8 + (lane >> 2), c8 = (lane & 3) * 8;
        const int row = tile_row0 + rl;
        const float4 a = *reinterpret_cast<const float4*>(stage + rl * kStageLd + c8), b = *reinterpret_cast<const float4*>(stage + rl * kStageLd + c8 + 4);
        float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        if (epi == RS_EPI_BIAS_RELU_BF16) {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.0f);
        } else if (epi == RS_EPI_BIAS_SWISH_BF16) {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = swishf_fast(v[j]);
        }
        const uint4 o = epi == RS_EPI_BIAS_F16
                            ? make_uint4(pack_f16x2(v[0], v[1]), pack_f16x2(v[2], v[3]), pack_f16x2(v[4], v[5]), pack_f16x2(v[6], v[7]))
                            : make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
        if (row < p.M)       // __half and __nv_bfloat16 are both two bytes: one address computation
          *reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + static_cast<size_t>(row) * p.ldo + col0 + c8) = o;
      }
      break;
    }
    case RS_EPI_BIAS_GLU_BF16: {
      // columns [0,16) of the chunk are values, [16,32) the matching gates (weights interleaved at pack time)
      const int rl = lane >> 1, c8 = (lane & 1) * 8;           // 16 rows x 32 B in one instruction
      const int row = tile_row0 + rl;
      float g[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = stage[rl * kStageLd + c8 + j] * sigmoidf_fast(stage[rl * kStageLd + 16 + c8 + j]);
      if (row < p.M)
        *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.out) + static_cast<size_t>(row) * p.ldo + col0 / 2 + c8) =
            make_uint4(pack_bf16x2(g[0], g[1]), pack_bf16x2(g[2], g[3]), pack_bf16x2(g[4], g[5]), pack_bf16x2(g[6], g[7]));
      break;
    }
    default: {  // RS_EPI_RESID_F32 / RS_EPI_BIAS_F32
      const bool add = p.epilogue == RS_EPI_RESID_F32;
#pragma unroll
      for (int i = 0; i < 4; ++i) {                            // 4 rows x 128 B per instruction
        const int rl = i * 4 + (lane >> 3), cw = (lane & 7) * 4;
        const int row = tile_row0 + rl;
        if (row < p.M) {
          const size_t off = static_cast<size_t>(row) * p.ldo + col0 + cw;
          float4 a = *reinterpret_cast<const float4*>(stage + rl * kStageLd + cw);
          a.x *= p.alpha; a.y *= p.alpha; a.z *= p.alpha; a.w *= p.alpha;
          if (add) {                                           // out may be resid (in place): each element is read and written by this lane only
            const float4 r = *reinterpret_cast<const float4*>(p.resid + off);
            a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w;
          }
          *reinterpret_cast<float4*>(static_cast<float*>(p.out) + off) = a;
        }
      }
      break;
    }
  }
}

template <int BN, int EG>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, const GemmDev p) {
  using Cfg = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled operand tiles need 1024 B alignment.
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + Cfg::kStages * Cfg::kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };
  uint8_t* stage_gen = smem_raw + ((bar_base + 256u) - smem_u32(smem_raw));   // generic pointer to the staging area
  auto smem_a = [&](int s) { return smem_base + s * Cfg::kStageBytes; };
  auto smem_b = [&](int s) { return smem_base + s * Cfg::kStageBytes + kABytes; };

  const int warp = warp_id_uniform();
  const int lane = lane_id();
  const int num_m = (p.M + BM - 1) / BM;
  const int num_n = (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_k = p.K / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
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
    const int rows0 = (cw >> 2) * 64;                          // the warpgroup's rows of the tile
    float* stage_f = reinterpret_cast<float*>(stage_gen + cw * kStageBytesPerWarp);
    const int g = lane >> 2, t = lane & 3;
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
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
      // ---- epilogue: 32-column chunks of the warp's 16 rows
      const int tile_row0 = m0 + rows0 + (cw & 3) * 16;
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        const int col0 = n0 + c * 32;
        if (col0 < p.N && tile_row0 < p.M) {                   // warp-uniform
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int col = 8 * j + 2 * t;
            const float2 b = p.bias != nullptr ? __ldg(reinterpret_cast<const float2*>(p.bias + col0 + col)) : make_float2(0.f, 0.f);
            *reinterpret_cast<float2*>(stage_f + g * kStageLd + col) = make_float2(d[c * 16 + j * 4] + b.x, d[c * 16 + j * 4 + 1] + b.y);
            *reinterpret_cast<float2*>(stage_f + (g + 8) * kStageLd + col) = make_float2(d[c * 16 + j * 4 + 2] + b.x, d[c * 16 + j * 4 + 3] + b.y);
          }
          __syncwarp();
          epilogue_store<EG>(p, stage_f, tile_row0, lane, col0);
          __syncwarp();                                        // staging buffer reusable
        }
      }
    }
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

bool make_tmap_bf16(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, char* err) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) { snprintf(err, 256, "cuTensorMapEncodeTiled entry point unavailable"); return false; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { snprintf(err, 256, "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu", (int)r, (unsigned long long)rows, (unsigned long long)cols); return false; }
  return true;
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
  CUtensorMap tm_a, tm_b;
  const int ldo = g.epilogue == RS_EPI_BIAS_GLU_BF16 ? g.N / 2 : g.N;
  if (!make_tmap_bf16(&tm_a, g.a, g.M, g.K, g.K, BM, err)) return cudaErrorInvalidValue;
  if (!make_tmap_bf16(&tm_b, g.w, g.N, g.K, g.K, BN, err)) return cudaErrorInvalidValue;
  GemmDev p{g.bias, g.resid, g.out, g.M, g.N, g.K, g.epilogue, g.alpha, ldo, g.out2, g.split, g.ld2};
  const int tiles = ((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN);
  const int grid = tiles < num_sms ? tiles : num_sms;
  gemm_bf16_tn_kernel<BN, EG><<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(tm_a, tm_b, p);
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
  if ((reinterpret_cast<uintptr_t>(g.a) | reinterpret_cast<uintptr_t>(g.w) | reinterpret_cast<uintptr_t>(g.out)) & 15u) {
    snprintf(err, 256, "gemm operands must be 16-byte aligned");
    return cudaErrorInvalidValue;
  }
  if (g.epilogue == RS_EPI_RESID_F32 && g.resid == nullptr) { snprintf(err, 256, "gemm: residual epilogue without resid"); return cudaErrorInvalidValue; }
  if (g.epilogue == RS_EPI_QKV_VT && (g.out2 == nullptr || g.split % 32 || g.ld2 % 8 || g.M % 8 || g.ld2 < g.M)) {
    snprintf(err, 256, "gemm: RS_EPI_QKV_VT needs out2, split %% 32 == 0, ld2 %% 8 == 0, M %% 8 == 0, ld2 >= M");
    return cudaErrorInvalidValue;
  }
  // 256-wide tiles when N fills them and they give every SM a tile, else 64-wide ones on more SMs.  The two instances
  // compute every element alike, so the choice (which depends on M) cannot make a row's result depend on the batch it
  // sits in (tests/test_gpu_gemm_cluster.py).
  if (g.N % 256 == 0 && ((g.M + BM - 1) / BM) * (g.N / 256) >= num_sms) return launch_bn<256>(g, num_sms, stream, err);
  return launch_bn<64>(g, num_sms, stream, err);
}

}  // namespace rs
