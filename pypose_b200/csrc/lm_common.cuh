// lm_common.cuh — shared by lm.cu and pcg.cu: launch geometry and the deterministic fp64 last-block reduction.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "lm_math.cuh"
#include "b200pose.h"   // every definition is checked against the generated declaration

namespace b200pose {

#define B200_EXPORT extern "C" __attribute__((visibility("default")))
constexpr int kLmThreads = 128;
constexpr int kMaxSums = 4;

static inline int lm_sms() {
  static thread_local int dev_cached = -1, sms = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev != dev_cached) { cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); dev_cached = dev; }
  return sms;
}

// Block-reduce NS doubles per thread, store the CTA partial, and let the last CTA produce the totals.
// workspace layout (doubles): [0 .. NS) totals | [7] ticket (as unsigned) | [8 ..) partials[grid][NS]
template <int NS>
__device__ __forceinline__ bool reduce_sums(double (&v)[NS], double* ws) {
  __shared__ double sh[kLmThreads / 32][NS];
  __shared__ bool is_last;
#pragma unroll
  for (int k = 0; k < NS; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < NS; ++k) sh[warp][k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0) {
    double* part = ws + 8 + (size_t)blockIdx.x * NS;
#pragma unroll
    for (int k = 0; k < NS; ++k) {
      double t = 0;
      for (int w = 0; w < kLmThreads / 32; ++w) t += sh[w][k];
      part[k] = t;
    }
    __threadfence();
    unsigned* ticket = reinterpret_cast<unsigned*>(ws + 7);
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    // Fixed-order fold by the whole CTA: thread-strided partial sums with the loads of kFold CTAs' partials issued before
    // the first add, then the shuffle tree and a fixed-order sum of the warp results.  (The one-warp, one-load-at-a-time loop
    // this replaces walked grid/32 dependent L2 round trips.)
    constexpr int kFold = 4;
    double t[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) t[k] = 0;
    unsigned b = threadIdx.x;
    for (; b + (kFold - 1) * kLmThreads < gridDim.x; b += kFold * kLmThreads) {
      double x[kFold][NS];
#pragma unroll
      for (int u = 0; u < kFold; ++u)
#pragma unroll
        for (int k = 0; k < NS; ++k) x[u][k] = __ldcg(ws + 8 + (size_t)(b + u * kLmThreads) * NS + k);
#pragma unroll
      for (int u = 0; u < kFold; ++u)
#pragma unroll
        for (int k = 0; k < NS; ++k) t[k] += x[u][k];
    }
    for (; b < gridDim.x; b += kLmThreads)
#pragma unroll
      for (int k = 0; k < NS; ++k) t[k] += __ldcg(ws + 8 + (size_t)b * NS + k);
#pragma unroll
    for (int k = 0; k < NS; ++k)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t[k] += __shfl_xor_sync(0xffffffffu, t[k], o);
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < NS; ++k) sh[warp][k] = t[k];
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
      for (int k = 0; k < NS; ++k) {
        double tot = 0;
        for (int w = 0; w < kLmThreads / 32; ++w) tot += sh[w][k];
        ws[k] = tot;
      }
      *reinterpret_cast<unsigned*>(ws + 7) = 0u;   // re-arm the ticket for the next launch
      return true;                                 // thread 0 of the last CTA: totals are in ws[0..NS)
    }
  }
  return false;
}

// (n, 6) work vectors of the PCG entry points are accessed as 8-byte (float) / 16-byte (double) pairs
constexpr int kMisaligned = 716;                      // cudaErrorMisalignedAddress
template <typename T, typename... P> static inline bool pairs_aligned(const P*... ptrs) {
  const uintptr_t bits = (0 | ... | reinterpret_cast<uintptr_t>(ptrs));
  return (bits & (2 * sizeof(T) - 1)) == 0;
}

template <typename T> __device__ __forceinline__ Elem<T> load_se3(const T* p) { return load_elem<SE3g, T>(p); }

static inline unsigned lm_grid(long long work_items, int per_block) {
  long long need = (work_items + per_block - 1) / per_block;
  long long cap = (long long)lm_sms() * 8;
  if (need < 1) need = 1;
  return (unsigned)(need < cap ? need : cap);
}

}  // namespace b200pose

namespace b200pose {

// Scatter-add K values per lane to dst (already offset by the lane's key) with as few atomics as the key layout allows:
// lanes holding the same key are found with match.any; if every such group is a contiguous lane range (keys sorted, the
// usual case for observations grouped by camera) a segmented shuffle reduction leaves the group's sum in its first lane,
// which issues the K atomics.  Any other layout falls back to per-lane atomics.  Must be called by all 32 lanes.
template <typename T, int K>
__device__ __forceinline__ void seg_atomic_add(T* dst, long long key, T (&v)[K], bool active) {
  const int lane = threadIdx.x & 31;
  const unsigned peers = __match_any_sync(0xffffffffu, active ? key : (long long)(-1 - lane));
  const int lo = __ffs(peers) - 1, hi = 31 - __clz(peers);
  const bool contig = __popc(peers) == hi - lo + 1;
  if (__all_sync(0xffffffffu, contig)) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const bool take = lane + o <= hi;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const T other = __shfl_down_sync(0xffffffffu, v[k], o);
        if (take) v[k] += other;
      }
    }
    if (active && lane == lo)
#pragma unroll
      for (int k = 0; k < K; ++k) atomicAdd(dst + k, v[k]);
  } else if (active) {
#pragma unroll
    for (int k = 0; k < K; ++k) atomicAdd(dst + k, v[k]);
  }
}

}  // namespace b200pose

namespace b200pose {

// Rows of one observation rebuilt from 16 B: Y4[k] = (y = T_c p, sqrt(rho')) and the camera quaternion (gathered, the
// observations are grouped by camera so a warp mostly shares it).  jc0/jc1 = d r / d xi_c (2x6), jp0/jp1 = d r / d p (2x3).
template <typename T> struct ObsRows { T jc0[6], jc1[6], jp0[3], jp1[3]; };
template <typename T>
__device__ __forceinline__ void obs_rows(const T* __restrict__ Y4, const T* __restrict__ poses, long long k, long long c,
                                         ObsRows<T>& R) {
  const T yx = Y4[k * 4], yy = Y4[k * 4 + 1], yz = Y4[k * 4 + 2], sw = Y4[k * 4 + 3];
  Elem<T> Tc;
  Tc.q.v = mk(__ldg(poses + c * 7 + 3), __ldg(poses + c * 7 + 4), __ldg(poses + c * 7 + 5));
  Tc.q.w = __ldg(poses + c * 7 + 6);
  const V3<T> y = mk(yx, yy, yz);
  reproj_rows(y, R.jc0, R.jc1);
  reproj_point_rows(Tc, y, R.jp0, R.jp1);
#pragma unroll
  for (int a = 0; a < 6; ++a) { R.jc0[a] *= sw; R.jc1[a] *= sw; }
#pragma unroll
  for (int a = 0; a < 3; ++a) { R.jp0[a] *= sw; R.jp1[a] *= sw; }
}

}  // namespace b200pose

namespace b200pose {
// ba.cu: y[c] -= sum over camera c's rows of Jc^T Jp (Hp^-1) t, one writer per camera (deterministic)
template <typename CT>
int ba_wv_seg_launch(const CT* Y4, const CT* poses, const int* pidx, const int* cseg, int S, int tpi, const CT* Hpinv,
                     const CT* t, CT* y, CT* part, const double* cg, long long C, cudaStream_t st);
}  // namespace b200pose
