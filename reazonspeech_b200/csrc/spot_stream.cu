// Streaming keyword spotting: the recursion of spot.cu resumed chunk by chunk from a per-(stream, keyword) record, and the
// streaming hit policy (semantics: reazonspeech_b200/keywords.py, "Streaming").
//
//   spot_gather_kernel            copies row b's joint.enc rows [dec_begin, dec_end) into a compact [B][C][Hj] block, so that
//                                 rnnt_lattice_kernel<true> runs unchanged on (row, keyword) pairs with enc_len = dec_end -
//                                 dec_begin (every lattice cell depends only on its own enc_proj and pred_proj rows)
//   rnnt_spot_resume_dp_kernel    rnnt_spot_dp_kernel's wavefront (one warp per pair, lane u - 1 owns row u) started from the
//                                 record's carried column (delta, start frame, lp_blank of the last decoded frame) and stored
//                                 back at the end.  Instead of predecessor bytes it keeps a forward traceback: each row holds
//                                 the token frames and lp_emit of the path to its current cell (a blank keeps the row's list,
//                                 an emission copies row u - 1's list from the previous diagonal and appends (t, lp_emit)),
//                                 double-buffered by diagonal parity in shared memory.  Every candidate end frame is appended
//                                 to the pair's pending ring.
//   rnnt_spot_resume_pick_kernel  one CTA (one warp) per pair: sigma, the natural cut's fixpoint, the forced cut, the greedy over
//                                 the decided prefix of the ring, the barrier, and the ring's compaction.  Decided hits go to
//                                 one device list through an atomic counter; the host sorts them.
//
// The record layout (SpotRecord in kernels.h): header int32[8] = frames seen, barrier + 1, forced cuts, ring head, ring size |
// column: delta f32[U_max], start i32[U_max], lp_blank f32[U_max] | lists: frames i32[U_max][U_max], lp f32[U_max][U_max] |
// ring: ring_cap entries of (e i32, E f32, S i32, frames i32[U_max], lp f32[U_max]).  An all-zero record has seen no frame.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace rs {

namespace {

constexpr int kDpWarps = 4;         // pairs per CTA of the DP
constexpr int kDpBatch = 16;        // anti-diagonals whose lattice loads are issued together, as in rnnt_spot_dp_kernel

__device__ __forceinline__ float mean_lp(float E, int e, int s) { return __fdiv_rn(E, static_cast<float>(e - s + 1)); }

struct Rec {
  int32_t* hdr; float* v; int32_t* st; float* lb; int32_t* lf; float* ll; uint8_t* ring;
  __device__ Rec(const SpotStreamArgs& s, int slot, int k) {
    const SpotRecord L = spot_record(s.U_max, s.ring_cap);
    uint8_t* r = s.records + (static_cast<size_t>(slot) * s.n_kw + k) * L.total;
    hdr = reinterpret_cast<int32_t*>(r);
    v = reinterpret_cast<float*>(r + L.column);
    st = reinterpret_cast<int32_t*>(v + s.U_max);
    lb = reinterpret_cast<float*>(st + s.U_max);
    lf = reinterpret_cast<int32_t*>(r + L.lists);
    ll = reinterpret_cast<float*>(lf + s.U_max * s.U_max);
    ring = r + L.ring;
  }
  __device__ uint8_t* entry(const SpotStreamArgs& s, int i) const { return ring + static_cast<size_t>(i) * spot_entry_bytes(s.U_max); }
};

__global__ void __launch_bounds__(128) spot_gather_kernel(const float* encp, int T_max, int Hj, const SpotStreamArgs s, float* out) {
  const int b = blockIdx.y, c = blockIdx.x;
  const int b0 = s.dec_begin[b], n = s.dec_end[b] - b0;
  if (c == 0 && threadIdx.x == 0) s.len[b] = n;
  if (c >= n) return;
  const float4* src = reinterpret_cast<const float4*>(encp + (static_cast<size_t>(b) * T_max + b0 + c) * Hj);
  float4* dst = reinterpret_cast<float4*>(out + (static_cast<size_t>(b) * s.C + c) * Hj);
  for (int i = threadIdx.x; i < Hj / 4; i += blockDim.x) dst[i] = src[i];
}

// Dynamic shared memory per warp: frames i32[2][U_max][U_max + 1] | lp f32[2][U_max][U_max + 1] (parity, row, token).
__global__ void __launch_bounds__(32 * kDpWarps) rnnt_spot_resume_dp_kernel(const AlignArgs a, const SpotStreamArgs s) {
  extern __shared__ __align__(16) uint8_t s_dp[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, p = blockIdx.x * kDpWarps + warp;
  if (p >= s.B * s.n_kw) return;                                       // warp-uniform
  const int k = p % s.n_kw, b = p / s.n_kw, UM = s.U_max, LP = UM + 1, U1 = a.U_max + 1;
  const int T = a.enc_len[b], U = a.label_len[k];
  const size_t plane = static_cast<size_t>(UM) * LP;
  int32_t* lf = reinterpret_cast<int32_t*>(s_dp) + warp * 4 * plane;  // [2][UM][LP]
  float* ll = reinterpret_cast<float*>(lf + 2 * plane);                // [2][UM][LP]
  const Rec R(s, s.slot[b], k);
  const int F0 = R.hdr[0];
  const int u = lane + 1;
  const bool row = u <= U;
  float v = 0.f, lb_prev = 0.f;                                        // delta[t][u] and lp_blank[t][u] of this lane's last cell
  int st = 0;                                                          // the frame of token 1 on the path to it
  if (row) {
    v = R.v[lane]; st = R.st[lane]; lb_prev = R.lb[lane];
    const int par = (lane + 1) & 1;                                    // read at this row's first diagonal d = lane as parity d - 1
    for (int i = 0; i < u; ++i) {
      lf[par * plane + lane * LP + i] = R.lf[lane * UM + i];
      ll[par * plane + lane * LP + i] = R.ll[lane * UM + i];
    }
  }
  __syncwarp();
  int head = R.hdr[3], size = R.hdr[4];
  const float* lpb = a.lp_blank + static_cast<size_t>(p) * a.T_max * U1;
  const float* lpe = a.lp_emit + static_cast<size_t>(p) * a.T_max * U1;
  const int b0 = s.dec_begin[b];
  for (int d0 = 0; d0 < T + U - 1; d0 += kDpBatch) {
    float lb[kDpBatch], le[kDpBatch];
#pragma unroll
    for (int i = 0; i < kDpBatch; ++i) {
      const int t = d0 + i - lane;
      const bool on = row && t >= 0 && t < T;
      lb[i] = on ? lpb[static_cast<size_t>(t) * U1 + u] : 0.f;
      le[i] = on ? lpe[static_cast<size_t>(t) * U1 + u - 1] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < kDpBatch; ++i) {
      const int t = d0 + i - lane, cur = (d0 + i) & 1, prv = cur ^ 1;
      const float dv = __shfl_up_sync(0xffffffffu, v, 1);              // lane - 1 holds (t, u - 1), one diagonal back
      const int ds = __shfl_up_sync(0xffffffffu, st, 1);
      if (row && t >= 0 && t < T) {
        const int tg = F0 + t;                                         // the stream's frame
        const float ve = (lane == 0 ? 0.f : dv) + le[i];
        const float vb = tg > 0 ? v + lb_prev : -INFINITY;
        const bool ch = tg == 0 || ve > vb;                            // an exact tie goes to the blank predecessor
        st = ch ? (lane == 0 ? tg : ds) : st;
        v = ch ? ve : vb;
        int32_t* dst_f = lf + cur * plane + lane * LP;
        float* dst_l = ll + cur * plane + lane * LP;
        if (ch) {                                                      // row u - 1's list at (t, u - 1), then this token
          for (int j = 0; j < lane; ++j) { dst_f[j] = lf[prv * plane + (lane - 1) * LP + j]; dst_l[j] = ll[prv * plane + (lane - 1) * LP + j]; }
          dst_f[lane] = tg; dst_l[lane] = le[i];
        } else {                                                       // this row's own list at (t - 1, u)
          for (int j = 0; j < u; ++j) { dst_f[j] = lf[prv * plane + lane * LP + j]; dst_l[j] = ll[prv * plane + lane * LP + j]; }
        }
        lb_prev = lb[i];
        if (u == U) {
          const float E = v + lb[i];
          if (s.E_out) {
            const size_t o = static_cast<size_t>(p) * s.T_out + b0 + t;
            s.E_out[o] = E; s.S_out[o] = st;
          }
          if (mean_lp(E, tg, st) >= s.threshold && size < s.ring_cap) {
            uint8_t* en = R.entry(s, (head + size) % s.ring_cap);
            int32_t* ei = reinterpret_cast<int32_t*>(en);
            ei[0] = tg; reinterpret_cast<float*>(ei)[1] = E; ei[2] = st;
            int32_t* ef = ei + 3;
            float* el = reinterpret_cast<float*>(ef + UM);
            for (int j = 0; j < UM; ++j) { ef[j] = j < U ? dst_f[j] : -1; el[j] = j < U ? dst_l[j] : NAN; }
            ++size;
          }
        }
      }
      __syncwarp();
    }
  }
  if (row) {
    R.v[lane] = v; R.st[lane] = st; R.lb[lane] = lb_prev;
    if (T > 0) {
      const int par = (T - 1 + lane) & 1;                              // the diagonal of this row's last cell
      for (int i = 0; i < u; ++i) { R.lf[lane * UM + i] = lf[par * plane + lane * LP + i]; R.ll[lane * UM + i] = ll[par * plane + lane * LP + i]; }
    }
  }
  if (lane == U - 1) { R.hdr[0] = F0 + max(T, 0); R.hdr[4] = size; }   // the lane that appended to the ring
}

// One warp per pair.  Dynamic shared memory: e i32[ring_cap] | S i32[ring_cap] | m f32[ring_cap] | alive i32[ring_cap].
__global__ void __launch_bounds__(32) rnnt_spot_resume_pick_kernel(const SpotStreamArgs s) {
  extern __shared__ __align__(16) int s_pk[];
  const int p = blockIdx.x, lane = threadIdx.x, k = p % s.n_kw, b = p / s.n_kw, cap = s.ring_cap;
  int* se = s_pk;
  int* sS = se + cap;
  float* sm = reinterpret_cast<float*>(sS + cap);
  int* alive = reinterpret_cast<int*>(sm + cap);
  const int U = s.label_len[k];
  const Rec R(s, s.slot[b], k);
  const int F = R.hdr[0], head = R.hdr[3], size = R.hdr[4], barrier = R.hdr[1] - 1;
  int sigma = INT_MAX;                                                 // min over u of start[t][u] at the last frame t
  for (int u = lane; u < U; u += 32) sigma = min(sigma, R.st[u]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sigma = min(sigma, __shfl_xor_sync(0xffffffffu, sigma, o));
  if (s.sigma_out && lane == 0) s.sigma_out[p] = F > 0 ? sigma : -1;
  if (F == 0) return;                                                  // no frame seen: nothing pending
  for (int i = lane; i < size; i += 32) {
    const int32_t* ei = reinterpret_cast<const int32_t*>(R.entry(s, (head + i) % cap));
    se[i] = ei[0]; sS[i] = ei[2];
    sm[i] = mean_lp(reinterpret_cast<const float*>(ei)[1], ei[0], ei[2]);
  }
  __syncwarp();
  int L = INT_MAX, cut = INT_MAX;
  if (lane == 0) {
    const int t = F - 1;
    if (!s.last[b]) {
      L = sigma;                                                       // L <- min(L, min{S(e) : pending e >= L}) to a fixpoint
      for (;;) {
        int nl = L;
        for (int i = size - 1; i >= 0 && se[i] >= L; --i) nl = min(nl, sS[i]);
        if (nl == L) break;
        L = nl;
      }
    }
    cut = L;
    for (int i = 0; i < size; ++i)                                     // the forced cut: a pending candidate has waited D frames
      if (se[i] >= L && t - se[i] >= s.delay) { cut = t + 1 - s.delay; break; }
  }
  L = __shfl_sync(0xffffffffu, L, 0);
  cut = __shfl_sync(0xffffffffu, cut, 0);
  int nd = 0;                                                          // the decided prefix: e < cut
  for (int i = lane; i < size; i += 32) {
    const bool dec = se[i] < cut;
    alive[i] = dec && sS[i] > barrier;                                 // a span reaching back over a reported hit is dropped
    nd += dec;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nd += __shfl_xor_sync(0xffffffffu, nd, o);
  __syncwarp();
  int top = barrier;
  for (;;) {
    float bm = -INFINITY;
    int bi = -1;
    for (int i = lane; i < nd; i += 32)
      if (alive[i] && (bi < 0 || sm[i] > bm)) { bm = sm[i]; bi = i; }   // ascending i: the smaller e wins a tie in a lane
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, bm, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || om > bm || (om == bm && oi < bi))) { bm = om; bi = oi; }
    }
    if (bi < 0) break;                                                 // warp-uniform
    const int hs = sS[bi], he = se[bi];
    if (lane == 0) {
      const int h = atomicAdd(s.n_hits, 1);
      if (h < s.hit_cap) {
        const int32_t* ei = reinterpret_cast<const int32_t*>(R.entry(s, (head + bi) % cap));
        int32_t* mt = s.hit_meta + static_cast<size_t>(h) * kSpotHitInts;
        mt[0] = b; mt[1] = k; mt[2] = hs; mt[3] = he; mt[4] = he >= L;
        s.hit_val[2 * static_cast<size_t>(h)] = reinterpret_cast<const float*>(ei)[1];
        s.hit_val[2 * static_cast<size_t>(h) + 1] = bm;
        for (int j = 0; j < s.U_max; ++j) {
          s.hit_frames[static_cast<size_t>(h) * s.U_max + j] = ei[3 + j];
          s.hit_lp[static_cast<size_t>(h) * s.U_max + j] = reinterpret_cast<const float*>(ei)[3 + s.U_max + j];
        }
      }
    }
    top = max(top, he);
    for (int i = lane; i < nd; i += 32)
      if (sS[i] <= he && se[i] >= hs) alive[i] = 0;                    // intersects the hit (the hit itself included)
    __syncwarp();
  }
  if (lane == 0) {
    R.hdr[1] = top + 1;
    R.hdr[2] += cut > L;
    R.hdr[3] = (head + nd) % cap;
    R.hdr[4] = size - nd;
  }
}

size_t dp_smem(int U_max) { return static_cast<size_t>(kDpWarps) * 4 * U_max * (U_max + 1) * 4; }

}  // namespace

size_t spot_pick_stream_smem(int ring_cap) { return static_cast<size_t>(16) * ring_cap; }

cudaError_t launch_spot_gather(const float* encp, int T_max, int Hj, const SpotStreamArgs& s, float* out, cudaStream_t stream) {
  spot_gather_kernel<<<dim3(s.C, s.B), 128, 0, stream>>>(encp, T_max, Hj, s, out);
  return cudaGetLastError();
}

cudaError_t launch_rnnt_spot_resume_dp(const AlignArgs& a, const SpotStreamArgs& s, cudaStream_t stream) {
  static DeviceOnce attr_once;
  if (attr_once.pending()) {
    const cudaError_t e = cudaFuncSetAttribute(rnnt_spot_resume_dp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_once.set();
  }
  const int pairs = s.B * s.n_kw;
  rnnt_spot_resume_dp_kernel<<<(pairs + kDpWarps - 1) / kDpWarps, 32 * kDpWarps, dp_smem(s.U_max), stream>>>(a, s);
  return cudaGetLastError();
}

cudaError_t launch_rnnt_spot_resume_pick(const SpotStreamArgs& s, cudaStream_t stream) {
  static DeviceOnce attr_once;
  if (attr_once.pending()) {
    const cudaError_t e = cudaFuncSetAttribute(rnnt_spot_resume_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_once.set();
  }
  rnnt_spot_resume_pick_kernel<<<s.B * s.n_kw, 32, spot_pick_stream_smem(s.ring_cap), stream>>>(s);
  return cudaGetLastError();
}

}  // namespace rs
