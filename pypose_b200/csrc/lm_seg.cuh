// lm_seg.cuh — per-camera work items with one writer per camera (ba.cu, bal.cu): observations grouped by camera,
// item (camera c, sub-range s of S), fixed-order item reduction and the fold of the S partials in s order.
#pragma once
#include "lm_common.cuh"

namespace b200pose {

// fixed-order reduction of NV values over the TPI threads of an item; the result is valid in the item's first thread
template <typename T, int NV, int TPI>
__device__ __forceinline__ void item_reduce(T (&v)[NV], T (*sh)[NV]) {
#pragma unroll
  for (int k = 0; k < NV; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  if (TPI > 32) {                                   // one item per CTA: fold the warp partials in warp order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();                                // previous item's readers are done with sh
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < NV; ++k) sh[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        T t = sh[0][k];
        for (int w = 1; w < TPI / 32; ++w) t += sh[w][k];
        v[k] = t;
      }
  }
}

struct ItemRange { long long c; int b, e; };
__device__ __forceinline__ ItemRange item_range(long long it, int S, const int* __restrict__ cseg) {
  ItemRange r;
  r.c = it / S;
  const int s = (int)(it - r.c * S);
  const long long b = cseg[r.c], len = (long long)cseg[r.c + 1] - b;
  r.b = (int)(b + len * s / S);
  r.e = (int)(b + len * (s + 1) / S);
  return r;
}

// dst (+)= sum_s part[(c, s)] in s order; the first WA values go to A (stride WA), the remaining WB to B (stride WB)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) cam_fold_kernel(const T* __restrict__ part, int S, int WA, int WB,
                                                               T* __restrict__ A, T* __restrict__ B, int add,
                                                               const double* cg, long long C) {
  if (cg && cg[5] != 0.0) return;
  const int NV = WA + WB;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < C * NV; i += (long long)gridDim.x * kLmThreads) {
    const long long c = i / NV;
    const int v = (int)(i - c * NV);
    T t = T(0);
    for (int s = 0; s < S; ++s) t += part[(c * S + s) * NV + v];
    T* d = v < WA ? A + c * WA + v : B + c * WB + (v - WA);
    *d = add ? *d + t : t;
  }
}

static inline unsigned item_grid(long long items, int tpi) {
  const int ipb = kLmThreads / tpi;
  return lm_grid(items, ipb);
}

}  // namespace b200pose
