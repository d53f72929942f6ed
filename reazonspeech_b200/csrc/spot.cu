// Keyword spotting on the RNN-T lattice of every (recording, keyword) pair (semantics: reazonspeech_b200/keywords.py).
//
//   rnnt_spot_dp_kernel     the segment recursion of align.cu's rnnt_segment_dp_kernel with the score of every end frame
//                           kept: one warp per pair, lane u - 1 owns row u (U <= 32), an anti-diagonal wavefront in which
//                           each lane receives (delta, start frame) of the cell below it through __shfl_up_sync.  Writes
//                           E(e), S(e) and the predecessor byte of every cell (the choice array of the forced alignment).
//   rnnt_spot_pick_kernel   one CTA per pair: the hit policy (repeatedly the candidate with the largest m(e), the smaller e
//                           on a tie; every candidate whose span intersects it is dropped), then the backtrace of every hit
//                           from (e, U) through the choice bytes.
//
// The lattice comes from rnnt_lattice_kernel<true> (align.cu), the predictor from the teacher-forced align kernels.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace rs {

namespace {

constexpr int kSpotWarps = 4;       // pairs per CTA of the DP
constexpr int kSpotBatch = 16;      // anti-diagonals whose lattice loads are issued together (they do not depend on delta)
constexpr int kPickThreads = 256;

// Pair p is valid when its recording has enc_len in [0, T_max] and its keyword label_len in [1, U_max] with every label in
// [0, V); the frames [0, T) of a valid pair are the segment ends it can have (none when T = 0).  -> T, or -1 when invalid.
__device__ __forceinline__ int pair_frames(const AlignArgs& a, int r, int k, int lane) {
  const int T = a.enc_len[r], U = a.label_len[k];
  bool bad = T < 0 || T > a.T_max || U < 1 || U > a.U_max;
  if (!bad && lane < U) {
    const int y = a.labels[static_cast<size_t>(k) * a.U_max + lane];
    bad = y < 0 || y >= a.V;
  }
  return __any_sync(0xffffffffu, bad) ? -1 : T;
}

// m(e) = E(e) / (e - S(e) + 1), rounded to nearest whatever the build's division flags
__device__ __forceinline__ float mean_lp(float E, int e, int s) { return __fdiv_rn(E, static_cast<float>(e - s + 1)); }

__global__ void __launch_bounds__(32 * kSpotWarps) rnnt_spot_dp_kernel(const AlignArgs a, const SpotArgs sp) {
  const int lane = threadIdx.x & 31, p = blockIdx.x * kSpotWarps + (threadIdx.x >> 5);
  if (p >= sp.n_rec * a.B) return;                                    // warp-uniform
  const int k = p % a.B, r = p / a.B, U1 = a.U_max + 1;
  const int T = pair_frames(a, r, k, lane), U = a.label_len[k];
  float* E = sp.E + static_cast<size_t>(p) * a.T_max;
  int32_t* S = sp.S + static_cast<size_t>(p) * a.T_max;
  for (int t = max(T, 0) + lane; t < a.T_max; t += 32) { E[t] = NAN; S[t] = -1; }   // no segment ends there
  if (T <= 0) return;
  const size_t base = static_cast<size_t>(p) * a.T_max * U1;
  const float* lpb = a.lp_blank + base;
  const float* lpe = a.lp_emit + base;
  uint8_t* choice = a.choice + base;
  const int u = lane + 1;
  const bool row = u <= U;
  float v = 0.f, lb_prev = 0.f;                                      // delta[t][u] and lp_blank[t - 1][u] of this lane's cell
  int st = 0;                                                        // the frame of token 1 on the path to it
  for (int d0 = 0; d0 < T + U - 1; d0 += kSpotBatch) {
    float lb[kSpotBatch], le[kSpotBatch];
#pragma unroll
    for (int i = 0; i < kSpotBatch; ++i) {
      const int t = d0 + i - lane;
      const bool on = row && t >= 0 && t < T;
      lb[i] = on ? lpb[static_cast<size_t>(t) * U1 + u] : 0.f;      // the blank leaving (t, u): used at t + 1, and by E at u = U
      le[i] = on ? lpe[static_cast<size_t>(t) * U1 + u - 1] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < kSpotBatch; ++i) {
      const int t = d0 + i - lane;
      const float dv = __shfl_up_sync(0xffffffffu, v, 1);            // lane - 1 holds (t, u - 1), one diagonal back
      const int ds = __shfl_up_sync(0xffffffffu, st, 1);
      if (row && t >= 0 && t < T) {
        const float ve = (lane == 0 ? 0.f : dv) + le[i];             // row 0 is free at every frame: token 1 may start at t
        const float vb = t > 0 ? v + lb_prev : -INFINITY;
        const bool ch = t == 0 || ve > vb;                           // an exact tie goes to the blank predecessor
        choice[static_cast<size_t>(t) * U1 + u] = ch ? 1 : 0;
        st = ch ? (lane == 0 ? t : ds) : st;
        v = ch ? ve : vb;
        if (u == U) { E[t] = v + lb[i]; S[t] = st; }
      }
      lb_prev = lb[i];
    }
  }
}

// Dynamic shared memory: the hits' spans [max_hits][2] | the warps' best (m, e) [8][2] | one bit per frame: still a candidate.
__global__ void __launch_bounds__(kPickThreads) rnnt_spot_pick_kernel(const AlignArgs a, const SpotArgs sp) {
  extern __shared__ __align__(16) int s_pick[];
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, H = sp.max_hits;
  const int k = p % a.B, r = p / a.B, U1 = a.U_max + 1;
  int* s_span = s_pick;
  float* s_m = reinterpret_cast<float*>(s_span + 2 * H);
  int* s_e = s_pick + 2 * H + kPickThreads / 32;
  uint32_t* s_alive = reinterpret_cast<uint32_t*>(s_e + kPickThreads / 32);
  const int T = pair_frames(a, r, k, lane), U = a.label_len[k];
  if (T <= 0) {
    if (tid == 0) sp.count[p] = 0;
    return;
  }
  const float* E = sp.E + static_cast<size_t>(p) * a.T_max;
  const int32_t* S = sp.S + static_cast<size_t>(p) * a.T_max;
  const int W = (T + 31) / 32;
  for (int w = warp; w < W; w += kPickThreads / 32) {
    const int e = 32 * w + lane;
    const bool cand = e < T && mean_lp(E[e], e, S[e]) >= sp.threshold;
    const uint32_t bits = __ballot_sync(0xffffffffu, cand);
    if (lane == 0) s_alive[w] = bits;
  }
  __syncthreads();
  int n = 0, hs = 0, he = -1;                                        // the last hit's span (none yet: nothing intersects it)
  while (n < H) {
    float bm = -INFINITY;
    int be = INT_MAX;
    for (int w = warp; w < W; w += kPickThreads / 32) {
      const uint32_t bits = s_alive[w];
      if (bits == 0) continue;                                       // warp-uniform
      const int e = 32 * w + lane;
      bool alive = (bits >> lane) & 1u;
      if (alive) {
        const int s = S[e];
        if (s <= he && e >= hs) {
          alive = false;                                             // intersects the last hit (the hit itself included)
        } else {
          const float m = mean_lp(E[e], e, s);
          if (m > bm || (m == bm && e < be)) { bm = m; be = e; }
        }
      }
      const uint32_t keep = __ballot_sync(0xffffffffu, alive);
      if (lane == 0) s_alive[w] = keep;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, bm, o);
      const int oe = __shfl_xor_sync(0xffffffffu, be, o);
      if (om > bm || (om == bm && oe < be)) { bm = om; be = oe; }
    }
    if (lane == 0) { s_m[warp] = bm; s_e[warp] = be; }
    __syncthreads();
    bm = s_m[0]; be = s_e[0];
    for (int i = 1; i < kPickThreads / 32; ++i)
      if (s_m[i] > bm || (s_m[i] == bm && s_e[i] < be)) { bm = s_m[i]; be = s_e[i]; }
    __syncthreads();                                                 // s_m / s_e are rewritten by the next round
    if (be == INT_MAX) break;                                        // no candidate left (block-uniform)
    hs = S[be]; he = be;
    if (tid == 0) {
      const size_t h = static_cast<size_t>(p) * H + n;
      sp.span[2 * h] = hs; sp.span[2 * h + 1] = he;
      sp.score[h] = E[be]; sp.conf[h] = bm;
      s_span[2 * n] = hs; s_span[2 * n + 1] = he;
    }
    ++n;
  }
  if (tid == 0) sp.count[p] = n;
  __syncthreads();
  const float* lpe = a.lp_emit + static_cast<size_t>(p) * a.T_max * U1;
  const uint8_t* choice = a.choice + static_cast<size_t>(p) * a.T_max * U1;
  for (int h = tid; h < n; h += kPickThreads) {                      // one thread per hit backtraces it from (e, U)
    const size_t o = (static_cast<size_t>(p) * H + h) * a.U_max;
    int32_t* frames = sp.frames + o;
    float* token_lp = sp.token_lp + o;
    for (int i = U; i < a.U_max; ++i) { frames[i] = -1; token_lp[i] = NAN; }
    int t = s_span[2 * h + 1], u = U;
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

size_t pick_smem(int T_max, int max_hits) {
  return (static_cast<size_t>(2) * max_hits + 2 * (kPickThreads / 32) + (static_cast<size_t>(T_max) + 31) / 32) * 4;
}

}  // namespace

bool spot_pick_fits(int T_max, int max_hits) { return pick_smem(T_max, max_hits) <= 227 * 1024; }

cudaError_t launch_rnnt_spot_dp(const AlignArgs& a, const SpotArgs& sp, cudaStream_t stream) {
  const int pairs = sp.n_rec * a.B;
  rnnt_spot_dp_kernel<<<(pairs + kSpotWarps - 1) / kSpotWarps, 32 * kSpotWarps, 0, stream>>>(a, sp);
  return cudaGetLastError();
}

cudaError_t launch_rnnt_spot_pick(const AlignArgs& a, const SpotArgs& sp, cudaStream_t stream) {
  static DeviceOnce attr_once;
  if (attr_once.pending()) {
    const cudaError_t e = cudaFuncSetAttribute(rnnt_spot_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_once.set();
  }
  rnnt_spot_pick_kernel<<<sp.n_rec * a.B, kPickThreads, pick_smem(a.T_max, sp.max_hits), stream>>>(a, sp);
  return cudaGetLastError();
}

}  // namespace rs
