// knn.cu — batched exact brute-force k-nearest-neighbour search, point-to-point ICP and the radius mask of the
// point-cloud filters (C-ABI: include/b200pose.h, section "point clouds").  DESIGN.md §3.4, §3.5.
//
// k-NN: one thread owns Q queries and keeps each query's top-k list (distance, index) in registers, sorted, with fully
// unrolled insertion.  The CTA stages tiles of kTile target points in shared memory with coalesced loads of the
// contiguous (N2, D) rows (D = 3: padded to 4-wide points, one 16-byte broadcast load per target and thread for fp32) and
// every staged point is compared with all Q queries of the thread.  Distances come from coordinate differences in the data
// dtype; ord 2 compares squared distances and takes the root of the k outputs only.  Targets are visited in increasing
// index order and a candidate must be strictly better to enter a list, so equal distances keep the lower index first.
// When B * N1 is too small to fill the GPU, the N2 range is split over CTAs and a merge kernel combines the per-split
// lists in split order (same tie rule): deterministic, no atomics.
//
// ICP: one iteration is two launches.  (a) k = 1 matching of A * source against target, A applied on the fly, and per-CTA
// fp64 partial sums of the matched pairs; (b) one CTA per batch element reduces its partials in a fixed order, solves the
// Kabsch step in fp64 (icp_math.cuh) and composes A <- T A; the last CTA evaluates the ReduceToBason rule over the batch
// and sets the done flag that turns later enqueued iterations into no-ops.
//
// ICP backward: the recording variant stores each iteration's matches, A and sums (a trace); the backward walks the
// iterations in reverse with fp64 cotangents, per-batch fixed-order sums, and a sorted segmented sum for the targets.
#include <cuda_runtime.h>
#include <math_constants.h>
#include <initializer_list>
#include <cub/device/device_radix_sort.cuh>
#include "icp_math.cuh"

#define B200_EXPORT extern "C" __attribute__((visibility("default")))

namespace b200pose {
namespace {

constexpr int kKnnThreads = 256;
constexpr int kTile = 256;                 // target points per shared-memory round
constexpr int kMaxD = 16;
constexpr int kUpdThreads = 128;
constexpr int kSums = 17;                  // sum s(3), sum t(3), sum t s^T (9), sum dist, count

template <typename T> struct alignas(4 * sizeof(T)) Pt4 { T x, y, z, w; };

template <typename T> __device__ __forceinline__ T pos_inf();
template <> __device__ __forceinline__ float pos_inf<float>() { return CUDART_INF_F; }
template <> __device__ __forceinline__ double pos_inf<double>() { return CUDART_INF; }

template <bool LARGEST, typename T> __device__ __forceinline__ bool better(T a, T b) { return LARGEST ? a > b : a < b; }

// ord: 1, 2 (squared), 0 = inf
template <int ORD, typename T> __device__ __forceinline__ T dist3(T ax, T ay, T az, const Pt4<T>& p) {
  const T dx = ax - p.x, dy = ay - p.y, dz = az - p.z;
  if (ORD == 2) return fma(dz, dz, fma(dy, dy, dx * dx));
  if (ORD == 1) return fabs(dx) + fabs(dy) + fabs(dz);
  return fmax(fabs(dx), fmax(fabs(dy), fabs(dz)));
}
// ord inf starts from the first coordinate rather than 0: fmax(0, NaN) would be 0, so a NaN point would be at distance 0
template <int ORD, typename T> __device__ __forceinline__ T distn(const T (&q)[kMaxD], const T* p, int D) {
  T acc = ORD == 0 ? fabs(q[0] - p[0]) : T(0);
#pragma unroll
  for (int d = ORD == 0 ? 1 : 0; d < kMaxD; ++d)
    if (d < D) {
      const T t = q[d] - p[d];
      acc = ORD == 2 ? fma(t, t, acc) : ORD == 1 ? acc + fabs(t) : fmax(acc, fabs(t));
    }
  return acc;
}

// sorted insertion of (d, j) into a register-resident list; strictly better only (ties keep the earlier entry)
template <int K, bool LARGEST, typename T>
__device__ __forceinline__ void topk_insert(T (&v)[K], int (&id)[K], T d, int j) {
  if (better<LARGEST>(d, v[K - 1])) {
#pragma unroll
    for (int i = K - 1; i > 0; --i) {
      if (better<LARGEST>(d, v[i - 1])) { v[i] = v[i - 1]; id[i] = id[i - 1]; }
      else if (better<LARGEST>(d, v[i])) { v[i] = d; id[i] = j; }
    }
    if (better<LARGEST>(d, v[0])) { v[0] = d; id[0] = j; }
  }
}

// Shared-memory tile of target points: D == 3 as padded 4-wide points, otherwise D-strided rows.
template <typename T, int DV> struct Tile;
template <typename T> struct Tile<T, 3> { Pt4<T> p[kTile]; };
template <typename T> struct Tile<T, kMaxD> { T p[kTile * kMaxD]; };

template <typename T, int DV, int NT>
__device__ __forceinline__ void stage_tile(Tile<T, DV>& tl, const T* __restrict__ P, int j0, int n, int D) {
  const T* src = P + (long long)j0 * D;
  for (int e = threadIdx.x; e < n * D; e += NT) {
    const T v = src[e];
    if (DV == 3) {
      const int pt = e / 3, c = e - 3 * pt;
      reinterpret_cast<T*>(&tl.p[pt])[c] = v;
    } else {
      reinterpret_cast<T*>(tl.p)[e] = v;
    }
  }
}

// ord inf: fmax drops a NaN operand, so a point with a NaN coordinate would get a finite distance from the others.  Such a
// point is made NaN in every coordinate instead, which gives it a NaN distance (as ord 1 and 2 do by arithmetic): it never
// enters a list.  x: the point's first coordinate, n: its coordinate count.
template <typename T> __device__ __forceinline__ void nan_spread(T* x, int n) {
  bool bad = false;
  for (int d = 0; d < n; ++d) bad = bad || isnan(x[d]);
  if (bad)
    for (int d = 0; d < n; ++d) x[d] = pos_inf<T>() - pos_inf<T>();
}
template <typename T, int DV, int NT> __device__ __forceinline__ void nan_spread_tile(Tile<T, DV>& tl, int n, int D) {
  for (int pt = threadIdx.x; pt < n; pt += NT)
    nan_spread(reinterpret_cast<T*>(tl.p) + pt * (DV == 3 ? 4 : D), DV == 3 ? 3 : D);
}

// Q queries of this thread against targets [jb, je): the CTA's core loop.  q: query coordinates (D == 3: q[r][0..2]).
// NANS: make NaN targets NaN in every coordinate for ord inf (k-NN; ICP and the radius mask take finite coordinates only).
template <typename T, int DV, int K, int ORD, bool LARGEST, int Q, int NT, bool NANS>
__device__ __forceinline__ void scan_targets(Tile<T, DV>& tl, const T* __restrict__ P, int jb, int je, int D,
                                             const T (&q)[Q][kMaxD], T (&v)[Q][K], int (&id)[Q][K]) {
  for (int j0 = jb; j0 < je; j0 += kTile) {
    const int n = min(kTile, je - j0);
    __syncthreads();
    stage_tile<T, DV, NT>(tl, P, j0, n, D);
    __syncthreads();
    if (NANS && ORD == 0) {
      nan_spread_tile<T, DV, NT>(tl, n, D);
      __syncthreads();
    }
#pragma unroll 4
    for (int jj = 0; jj < n; ++jj) {
      if (DV == 3) {
        const Pt4<T> p = reinterpret_cast<const Tile<T, 3>&>(tl).p[jj];
#pragma unroll
        for (int r = 0; r < Q; ++r) topk_insert<K, LARGEST>(v[r], id[r], dist3<ORD>(q[r][0], q[r][1], q[r][2], p), j0 + jj);
      } else {
        const T* p = reinterpret_cast<const T*>(tl.p) + jj * D;
#pragma unroll
        for (int r = 0; r < Q; ++r) topk_insert<K, LARGEST>(v[r], id[r], distn<ORD>(q[r], p, D), j0 + jj);
      }
    }
  }
}

// an empty slot of a `largest` list holds -inf, whose root would be NaN: it stays -inf
template <int ORD, bool LARGEST, typename T> __device__ __forceinline__ T finish_dist(T d) {
  return ORD == 2 && (!LARGEST || d >= T(0)) ? sqrt(d) : d;
}

// grid: nqb query blocks x S splits x B batch elements (flattened in x).  S == 1 writes the results, otherwise the
// per-split lists (all K entries, ord-2 values still squared) go to pv / pi at ((b S + s) N1 + i) K.
template <typename T, int DV, int K, int ORD, bool LARGEST, int Q>
__global__ void __launch_bounds__(kKnnThreads) knn_kernel(const T* __restrict__ ref, long long rbs, const T* __restrict__ nbr,
                                                          long long nbs, int N1, int N2, int D, int kout, int nqb, int S,
                                                          int chunk, T* __restrict__ vals, long long* __restrict__ idx,
                                                          T* __restrict__ pv, int* __restrict__ pi) {
  __shared__ Tile<T, DV> tl;
  const int qb = blockIdx.x % nqb, rest = blockIdx.x / nqb, s = rest % S, b = rest / S;
  const T* R = ref + (long long)b * rbs;
  const T* P = nbr + (long long)b * nbs;
  T q[Q][kMaxD];
  T v[Q][K];
  int id[Q][K];
#pragma unroll
  for (int r = 0; r < Q; ++r) {
    const int i = min((qb * Q + r) * kKnnThreads + (int)threadIdx.x, N1 - 1);
#pragma unroll
    for (int d = 0; d < kMaxD; ++d) q[r][d] = (DV == 3 ? d < 3 : d < D) ? R[(long long)i * D + d] : T(0);
    if (ORD == 0) {                                // as nan_spread (unrolled: q stays in registers)
      bool bad = false;
#pragma unroll
      for (int d = 0; d < kMaxD; ++d) bad = bad || ((DV == 3 ? d < 3 : d < D) && isnan(q[r][d]));
      if (bad)
#pragma unroll
        for (int d = 0; d < kMaxD; ++d) q[r][d] = pos_inf<T>() - pos_inf<T>();
    }
#pragma unroll
    for (int c = 0; c < K; ++c) { v[r][c] = LARGEST ? -pos_inf<T>() : pos_inf<T>(); id[r][c] = -1; }
  }
  const int jb = s * chunk, je = min(N2, jb + chunk);
  scan_targets<T, DV, K, ORD, LARGEST, Q, kKnnThreads, true>(tl, P, jb, je, D, q, v, id);
#pragma unroll
  for (int r = 0; r < Q; ++r) {
    const int i = (qb * Q + r) * kKnnThreads + (int)threadIdx.x;
    if (i >= N1) continue;
    if (S == 1) {
      const long long o = ((long long)b * N1 + i) * kout;
#pragma unroll
      for (int c = 0; c < K; ++c)
        if (c < kout) { vals[o + c] = finish_dist<ORD, LARGEST>(v[r][c]); idx[o + c] = id[r][c]; }
    } else {
      const long long o = (((long long)b * S + s) * N1 + i) * K;
#pragma unroll
      for (int c = 0; c < K; ++c) { pv[o + c] = v[r][c]; pi[o + c] = id[r][c]; }
    }
  }
}

// one thread per (b, i): the S per-split lists, inserted in split order (= index order), give the exact top-k
template <typename T, int K, int ORD, bool LARGEST>
__global__ void __launch_bounds__(kKnnThreads) knn_merge_kernel(const T* __restrict__ pv, const int* __restrict__ pi, int S,
                                                                long long BN1, int N1, int kout, T* __restrict__ vals,
                                                                long long* __restrict__ idx) {
  const long long g = (long long)blockIdx.x * kKnnThreads + threadIdx.x;
  if (g >= BN1) return;
  const long long b = g / N1, i = g - b * N1;
  T v[K];
  int id[K];
#pragma unroll
  for (int c = 0; c < K; ++c) { v[c] = LARGEST ? -pos_inf<T>() : pos_inf<T>(); id[c] = -1; }
  for (int s = 0; s < S; ++s) {
    const long long o = ((b * S + s) * N1 + i) * K;
#pragma unroll
    for (int c = 0; c < K; ++c) topk_insert<K, LARGEST>(v, id, pv[o + c], pi[o + c]);
  }
#pragma unroll
  for (int c = 0; c < K; ++c)
    if (c < kout) { vals[g * kout + c] = finish_dist<ORD, LARGEST>(v[c]); idx[g * kout + c] = id[c]; }
}

int sm_count() {
  static int cache[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!cache[dev]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cache[dev] = n > 0 ? n : 132;
  }
  return cache[dev];
}

int kbucket(int k) { return k <= 1 ? 1 : k <= 4 ? 4 : k <= 8 ? 8 : k <= 16 ? 16 : 32; }
int queries_per_thread(int D, int K) { return D != 3 ? 1 : K == 1 ? 4 : K == 4 ? 2 : 1; }

// Split of the N2 range: enough CTAs for ~4 per SM, each split at least 2048 targets, at most 64 splits.
struct KnnPlan { int nqb, S, chunk, K; };
KnnPlan knn_plan(long long B, long long N1, long long N2, int D, int k) {
  KnnPlan p;
  p.K = kbucket(k);
  const long long per = (long long)kKnnThreads * queries_per_thread(D, p.K);
  p.nqb = (int)((N1 + per - 1) / per);
  const long long base = B * p.nqb, want = 4LL * sm_count();
  long long S = 1;
  if (base > 0 && base < want) {
    S = (want + base - 1) / base;
    S = min(S, (N2 + 2047) / 2048);
    S = max(1LL, min(S, 64LL));
  }
  long long chunk = (N2 + S - 1) / S;
  chunk = (chunk + kTile - 1) / kTile * kTile;
  p.chunk = (int)max(chunk, (long long)kTile);
  p.S = (int)((N2 + p.chunk - 1) / p.chunk);
  if (p.S < 1) p.S = 1;
  return p;
}

long long knn_ws_bytes(const KnnPlan& p, long long B, long long N1, int elem) {
  if (p.S <= 1) return 0;
  const long long n = (long long)p.S * B * N1 * p.K;
  return (n * elem + 255) / 256 * 256 + n * 4;
}

template <typename T> struct KnnArgs {
  const T* ref; long long rbs; const T* nbr; long long nbs; T* vals; long long* idx; void* ws;
  long long B, N1, N2; int D, k, ord, largest;
};

template <typename T, int DV, int K, int ORD, bool LARGEST>
int launch_knn(const KnnArgs<T>& a, cudaStream_t st) {
  const KnnPlan p = knn_plan(a.B, a.N1, a.N2, a.D, a.k);
  T* pv = nullptr;
  int* pi = nullptr;
  if (p.S > 1) {
    const long long n = (long long)p.S * a.B * a.N1 * K;
    pv = reinterpret_cast<T*>(a.ws);
    pi = reinterpret_cast<int*>(reinterpret_cast<char*>(a.ws) + (n * (long long)sizeof(T) + 255) / 256 * 256);
  }
  const long long grid = (long long)p.nqb * p.S * a.B;
  constexpr int Q = DV != 3 ? 1 : K == 1 ? 4 : K == 4 ? 2 : 1;
  knn_kernel<T, DV, K, ORD, LARGEST, Q><<<(unsigned)grid, kKnnThreads, 0, st>>>(
      a.ref, a.rbs, a.nbr, a.nbs, (int)a.N1, (int)a.N2, a.D, a.k, p.nqb, p.S, p.chunk, a.vals, a.idx, pv, pi);
  if (p.S > 1) {
    const long long BN1 = a.B * a.N1;
    knn_merge_kernel<T, K, ORD, LARGEST><<<(unsigned)((BN1 + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, st>>>(
        pv, pi, p.S, BN1, (int)a.N1, a.k, a.vals, a.idx);
  }
  return (int)cudaGetLastError();
}

template <typename T, int DV, int K, int ORD> int knn_l(const KnnArgs<T>& a, cudaStream_t s) {
  return a.largest ? launch_knn<T, DV, K, ORD, true>(a, s) : launch_knn<T, DV, K, ORD, false>(a, s);
}
template <typename T, int DV, int K> int knn_o(const KnnArgs<T>& a, cudaStream_t s) {
  return a.ord == 1 ? knn_l<T, DV, K, 1>(a, s) : a.ord == 2 ? knn_l<T, DV, K, 2>(a, s) : knn_l<T, DV, K, 0>(a, s);
}
template <typename T, int DV> int knn_k(const KnnArgs<T>& a, cudaStream_t s) {
  switch (kbucket(a.k)) {
    case 1: return knn_o<T, DV, 1>(a, s);
    case 4: return knn_o<T, DV, 4>(a, s);
    case 8: return knn_o<T, DV, 8>(a, s);
    case 16: return knn_o<T, DV, 16>(a, s);
    default: return knn_o<T, DV, 32>(a, s);
  }
}
// Every pointer the kernels dereference must be device (or managed) memory: a host pointer that reached this far (a CPU
// tensor passed through the C-ABI) is refused here instead of faulting inside a kernel.
bool device_ptrs(std::initializer_list<const void*> ps) {
  for (const void* p : ps) {
    if (!p) continue;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) return false;
  }
  return true;
}

template <typename T> int knn_run(const KnnArgs<T>& a, cudaStream_t s) {
  if (a.B <= 0 || a.N1 <= 0) return 0;
  if (!a.ref || !a.nbr || !a.vals || !a.idx || !device_ptrs({a.ref, a.nbr, a.vals, a.idx, a.ws})) return (int)cudaErrorInvalidValue;
  if (a.k < 1 || a.k > 32 || a.k > a.N2 || a.D < 1 || a.D > kMaxD || (a.ord != 0 && a.ord != 1 && a.ord != 2))
    return (int)cudaErrorInvalidValue;
  if (a.N1 > 0x7fffffffLL || a.N2 > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  return a.D == 3 ? knn_k<T, 3>(a, s) : knn_k<T, kMaxD>(a, s);
}

// ----------------------------------------------------------------------------------------------------------------------
// Radius mask (nbr_filter / knn_filter): count the points within `thr` of every point, itself included, and keep it when
// the count reaches `need`.  Same layout as the k-NN search (Q queries per thread, 256-point tiles in shared memory);
// ord 2 compares squared distances against the host-computed threshold (DESIGN.md §3.5).  After each tile the CTA stops
// when every live query already has its count: the mask does not depend on how many tiles were visited.
// ----------------------------------------------------------------------------------------------------------------------
template <typename T, int DV, int ORD, int Q>
__global__ void __launch_bounds__(kKnnThreads) radius_mask_kernel(const T* __restrict__ P, int N, int D, T thr, int need,
                                                                  unsigned char* __restrict__ mask) {
  __shared__ Tile<T, DV> tl;
  T q[Q][kMaxD];
  int cnt[Q];
  bool live[Q];
#pragma unroll
  for (int r = 0; r < Q; ++r) {
    const int i0 = (blockIdx.x * Q + r) * kKnnThreads + (int)threadIdx.x;
    const int i = min(i0, N - 1);
    live[r] = i0 < N;
    cnt[r] = 0;
#pragma unroll
    for (int d = 0; d < kMaxD; ++d) q[r][d] = (DV == 3 ? d < 3 : d < D) ? P[(long long)i * D + d] : T(0);
  }
  for (int j0 = 0; j0 < N; j0 += kTile) {
    const int n = min(kTile, N - j0);
    __syncthreads();
    stage_tile<T, DV, kKnnThreads>(tl, P, j0, n, D);
    __syncthreads();
#pragma unroll 4
    for (int jj = 0; jj < n; ++jj) {
      if (DV == 3) {
        const Pt4<T> p = reinterpret_cast<const Tile<T, 3>&>(tl).p[jj];
#pragma unroll
        for (int r = 0; r < Q; ++r) cnt[r] += dist3<ORD>(q[r][0], q[r][1], q[r][2], p) <= thr;
      } else {
        const T* p = reinterpret_cast<const T*>(tl.p) + jj * D;
#pragma unroll
        for (int r = 0; r < Q; ++r) cnt[r] += distn<ORD>(q[r], p, D) <= thr;
      }
    }
    bool done = true;
#pragma unroll
    for (int r = 0; r < Q; ++r) done = done && (!live[r] || cnt[r] >= need);
    if (__syncthreads_and(done)) break;
  }
#pragma unroll
  for (int r = 0; r < Q; ++r) {
    const int i = (blockIdx.x * Q + r) * kKnnThreads + (int)threadIdx.x;
    if (i < N) mask[i] = cnt[r] >= need;
  }
}

__global__ void fill_bytes_kernel(unsigned char* __restrict__ out, long long n, unsigned char v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = v;
}

// One query per thread when four per thread would leave SMs idle (fewer than 2 CTAs per SM).
bool radius_small(long long N) { return (N + 4LL * kKnnThreads - 1) / (4LL * kKnnThreads) < 2LL * sm_count(); }

template <typename T, int DV, int ORD> void launch_radius(const T* P, int N, int D, T thr, int need, unsigned char* mask,
                                                          cudaStream_t s) {
  if (DV == 3 && !radius_small(N)) {
    radius_mask_kernel<T, DV, ORD, 4><<<(unsigned)((N + 4 * kKnnThreads - 1) / (4 * kKnnThreads)), kKnnThreads, 0, s>>>(
        P, N, D, thr, need, mask);
  } else {
    radius_mask_kernel<T, DV, ORD, 1><<<(unsigned)((N + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, s>>>(
        P, N, D, thr, need, mask);
  }
}

template <typename T, int DV> void radius_o(const T* P, int N, int D, T thr, int ord, int need, unsigned char* mask,
                                            cudaStream_t s) {
  if (ord == 2) launch_radius<T, DV, 2>(P, N, D, thr, need, mask, s);
  else if (ord == 1) launch_radius<T, DV, 1>(P, N, D, thr, need, mask, s);
  else launch_radius<T, DV, 0>(P, N, D, thr, need, mask, s);
}

template <typename T>
int radius_run(const T* P, long long N, int D, double thr, int ord, long long need, unsigned char* mask, cudaStream_t s) {
  if (N <= 0) return 0;
  if (!P || !mask || !device_ptrs({P, mask})) return (int)cudaErrorInvalidValue;
  if (D < 1 || D > kMaxD || (ord != 0 && ord != 1 && ord != 2) || N > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  if (need <= 0) {
    fill_bytes_kernel<<<(unsigned)min((N + 255) / 256, 4096LL), 256, 0, s>>>(mask, N, 1);
    return (int)cudaGetLastError();
  }
  const int nd = (int)min(need, N + 1);       // a count never exceeds N
  if (D == 3) radius_o<T, 3>(P, (int)N, D, (T)thr, ord, nd, mask, s);
  else radius_o<T, kMaxD>(P, (int)N, D, (T)thr, ord, nd, mask, s);
  return (int)cudaGetLastError();
}

// ----------------------------------------------------------------------------------------------------------------------
// ICP
// ----------------------------------------------------------------------------------------------------------------------
// workspace: [st: 8 doubles | ticket: 8 doubles | A: B x 12 doubles | partials: B x nx x 17 doubles]
// st: [0] steps, [1] patience count, [2] continual (0 = done)
constexpr int kStWords = 8;
constexpr int kIcpBig = 256 * 4;           // source points per CTA: 256 threads x 4 queries
constexpr int kIcpSmall = 128;             // 128 threads x 1 query, when the big CTAs would not fill the GPU

// trace of the recording variant, one block per enqueued iteration: [A before the step (12), sums (17)] x B in fp64, then
// the match of every source point (B x Ns int32).  An iteration skipped after the done flag leaves its block unwritten.
constexpr int kRecD = 12 + kSums;
long long icp_rec_ad_bytes(long long B) { return (B * kRecD * 8 + 255) / 256 * 256; }
long long icp_rec_block(long long B, long long Ns) { return icp_rec_ad_bytes(B) + (B * Ns * 4 + 255) / 256 * 256; }

bool icp_small(long long B, long long Ns) { return B * ((Ns + kIcpBig - 1) / kIcpBig) < 2LL * sm_count(); }
long long icp_nx(long long B, long long Ns) {
  const long long per = icp_small(B, Ns) ? kIcpSmall : kIcpBig;
  return (Ns + per - 1) / per;
}

__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  return x;
}

// fixed-order block reduction of NS values; the totals end up in red[0][*] (visible after the final __syncthreads)
template <int NT, int NS = kSums> __device__ __forceinline__ void block_sums(double (&acc)[NS], double (*red)[NS]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NS; ++k) acc[k] = warp_sum(acc[k]);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < NS; ++k) red[w][k] = acc[k];
  __syncthreads();
  if (threadIdx.x < NS) {
    double s = 0.0;
    for (int i = 0; i < NT / 32; ++i) s += red[i][threadIdx.x];
    red[0][threadIdx.x] = s;          // row 0 is only read again by this thread before the barrier below
  }
  __syncthreads();
}

// (a): k = 1 matching of A source against target and the per-CTA fp64 sums.  grid: nx x B (flattened).
// REC: also store the match of every source point in rec (B x Ns).
template <typename T, int ORD, int Q, int NT, bool REC>
__global__ void __launch_bounds__(NT) icp_match_kernel(const T* __restrict__ src, long long sbs, const T* __restrict__ tgt,
                                                       long long tbs, int Ns, int Nt, const double* __restrict__ A,
                                                       const double* st, double* __restrict__ part, int nx, int decide,
                                                       int* __restrict__ rec) {
  if (decide && st[2] == 0.0) return;
  __shared__ Tile<T, 3> tl;
  __shared__ double red[NT / 32][kSums];
  const int x = blockIdx.x % nx, b = blockIdx.x / nx;
  const T* S = src + (long long)b * sbs;
  const T* P = tgt + (long long)b * tbs;
  T Ra[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) Ra[k] = (T)A[b * 12 + k];
  T q[Q][kMaxD];
  T v[Q][1];
  int id[Q][1];
#pragma unroll
  for (int r = 0; r < Q; ++r) {
    const int i = min((x * Q + r) * NT + (int)threadIdx.x, Ns - 1);
    const T px = S[(long long)i * 3], py = S[(long long)i * 3 + 1], pz = S[(long long)i * 3 + 2];
#pragma unroll
    for (int c = 0; c < 3; ++c) q[r][c] = fma(Ra[4 * c], px, fma(Ra[4 * c + 1], py, fma(Ra[4 * c + 2], pz, Ra[4 * c + 3])));
#pragma unroll
    for (int d = 3; d < kMaxD; ++d) q[r][d] = T(0);
    v[r][0] = pos_inf<T>();
    id[r][0] = 0;
  }
  scan_targets<T, 3, 1, ORD, false, Q, NT, false>(tl, P, 0, Nt, 3, q, v, id);
  const double c0x = (double)P[0], c0y = (double)P[1], c0z = (double)P[2];
  double acc[kSums];
#pragma unroll
  for (int k = 0; k < kSums; ++k) acc[k] = 0.0;
#pragma unroll
  for (int r = 0; r < Q; ++r) {
    const int i = (x * Q + r) * NT + (int)threadIdx.x;
    if (i >= Ns) continue;
    const long long j = id[r][0];
    if (REC) rec[(long long)b * Ns + i] = (int)j;
    const double s[3] = {(double)q[r][0] - c0x, (double)q[r][1] - c0y, (double)q[r][2] - c0z};
    const double t[3] = {(double)P[j * 3] - c0x, (double)P[j * 3 + 1] - c0y, (double)P[j * 3 + 2] - c0z};
#pragma unroll
    for (int c = 0; c < 3; ++c) { acc[c] += s[c]; acc[3 + c] += t[c]; }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[6 + 3 * a + c] += t[a] * s[c];
    acc[15] += (double)finish_dist<ORD, false>(v[r][0]);
    acc[16] += 1.0;
  }
  block_sums<NT>(acc, red);
  if (threadIdx.x < kSums) part[((long long)b * nx + x) * kSums + threadIdx.x] = red[0][threadIdx.x];
}

__device__ __forceinline__ void icp_publish(const double* st, double* host_out, double seq) {
  volatile double* o = host_out;
  o[0] = st[0]; o[1] = st[1]; o[2] = st[2];
  __threadfence_system();
  o[kStWords - 1] = seq;
}

// (b): per batch element: fixed-order reduction, Kabsch, A <- T A, mean distance, SE3 output; the last CTA decides.
template <typename T>
__global__ void __launch_bounds__(kUpdThreads) icp_update_kernel(const T* __restrict__ tgt, long long tbs, double* A,
                                                                 const double* __restrict__ part, int nx, double* st,
                                                                 unsigned* ticket, T* last, T* err, T* out, int B,
                                                                 int decide, R2bCtl ctl, double eps, double* host_out,
                                                                 double seq, int publish, double* rec) {
  if (decide && st[2] == 0.0) {
    if (publish && host_out && blockIdx.x == 0 && threadIdx.x == 0) icp_publish(st, host_out, seq);
    return;
  }
  __shared__ double red[kUpdThreads / 32][kSums];
  __shared__ bool is_last;
  const int b = blockIdx.x;
  double acc[kSums];
#pragma unroll
  for (int k = 0; k < kSums; ++k) acc[k] = 0.0;
  for (int x = threadIdx.x; x < nx; x += kUpdThreads)
#pragma unroll
    for (int k = 0; k < kSums; ++k) acc[k] += part[((long long)b * nx + x) * kSums + k];
  block_sums<kUpdThreads>(acc, red);
  if (threadIdx.x == 0) {
    const T* P = tgt + (long long)b * tbs;
    const double c0[3] = {(double)P[0], (double)P[1], (double)P[2]};
    double Ab[12], q[4];
    for (int k = 0; k < 12; ++k) Ab[k] = A[b * 12 + k];
    if (rec) {                                     // trace: A before the step and the sums it is solved from
      for (int k = 0; k < 12; ++k) rec[b * kRecD + k] = Ab[k];
      for (int k = 0; k < kSums; ++k) rec[b * kRecD + 12 + k] = red[0][k];
    }
    icp_step(red[0], c0, eps, Ab);
    for (int k = 0; k < 12; ++k) A[b * 12 + k] = Ab[k];
    err[b] = (T)(red[0][15] / red[0][16]);
    icp_mat2quat(Ab, q);
    T* o = out + (long long)b * 7;
    o[0] = (T)Ab[3]; o[1] = (T)Ab[7]; o[2] = (T)Ab[11];
    o[3] = (T)q[0]; o[4] = (T)q[1]; o[5] = (T)q[2]; o[6] = (T)q[3];
  }
  if (!decide) return;
  __threadfence();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  bool below = true, flat = true;
  for (int bb = threadIdx.x; bb < B; bb += kUpdThreads) {
    bool bt, fl;
    icp_r2b_flags<T>(__ldcg(err + bb), last[bb], ctl, bt, fl);
    below = below && bt;
    flat = flat && fl;
  }
  below = __syncthreads_and(below);
  flat = __syncthreads_and(flat);
  for (int bb = threadIdx.x; bb < B; bb += kUpdThreads) last[bb] = __ldcg(err + bb);
  if (threadIdx.x == 0) {
    icp_r2b_update(st, below, flat, ctl);
    *ticket = 0u;
    if (publish && host_out) icp_publish(st, host_out, seq);
  }
}

template <typename T>
__global__ void icp_init_kernel(const T* __restrict__ init, long long ibs, double* A, double* st, unsigned* ticket, T* last,
                                T* out, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) { st[0] = 0.0; st[1] = 0.0; st[2] = 1.0; *ticket = 0u; }
  if (b >= B) return;
  double a[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  if (init) {
    const T* p = init + (long long)b * ibs;
    const double q[4] = {(double)p[3], (double)p[4], (double)p[5], (double)p[6]};
    icp_quat2mat(q, a);
    a[3] = (double)p[0]; a[7] = (double)p[1]; a[11] = (double)p[2];
  }
  for (int k = 0; k < 12; ++k) A[b * 12 + k] = a[k];
  last[b] = pos_inf<T>();
  double q[4];                                     // the result if no iteration runs
  icp_mat2quat(a, q);
  T* o = out + (long long)b * 7;
  o[0] = (T)a[3]; o[1] = (T)a[7]; o[2] = (T)a[11];
  o[3] = (T)q[0]; o[4] = (T)q[1]; o[5] = (T)q[2]; o[6] = (T)q[3];
}

template <typename T, int ORD, bool REC>
void launch_match_r(const T* src, long long sbs, const T* tgt, long long tbs, long long B, long long Ns, long long Nt,
                    const double* A, const double* st, double* part, int nx, int decide, int* rec, cudaStream_t s) {
  const unsigned grid = (unsigned)(B * nx);
  if (icp_small(B, Ns))
    icp_match_kernel<T, ORD, 1, kIcpSmall, REC><<<grid, kIcpSmall, 0, s>>>(src, sbs, tgt, tbs, (int)Ns, (int)Nt, A, st, part,
                                                                          nx, decide, rec);
  else
    icp_match_kernel<T, ORD, 4, 256, REC><<<grid, 256, 0, s>>>(src, sbs, tgt, tbs, (int)Ns, (int)Nt, A, st, part, nx, decide,
                                                              rec);
}
template <typename T, int ORD>
void launch_match(const T* src, long long sbs, const T* tgt, long long tbs, long long B, long long Ns, long long Nt,
                  const double* A, const double* st, double* part, int nx, int decide, int* rec, cudaStream_t s) {
  if (rec) launch_match_r<T, ORD, true>(src, sbs, tgt, tbs, B, Ns, Nt, A, st, part, nx, decide, rec, s);
  else launch_match_r<T, ORD, false>(src, sbs, tgt, tbs, B, Ns, Nt, A, st, part, nx, decide, nullptr, s);
}

int wait_seq(double* host_out, long long seq, cudaStream_t s) {
  volatile double* flag = host_out + (kStWords - 1);
  for (long long spin = 0;; ++spin) {
    if (*flag == (double)seq) return 0;
    if ((spin & 0xffff) == 0xffff) {           // has the stream died or finished without publishing?
      const cudaError_t e = cudaStreamQuery(s);
      if (e == cudaSuccess) return *flag == (double)seq ? 0 : (int)cudaErrorUnknown;
      if (e != cudaErrorNotReady) return (int)e;
    }
  }
}

template <typename T>
int icp_run(const T* src, long long sbs, const T* tgt, long long tbs, const T* init, long long ibs, T* out, T* err, T* last,
            void* ws, long long B, long long Ns, long long Nt, int ord, long long first, long long iters, int decide,
            long long max_steps, long long patience, double decreasing, double tol, double* host_out, long long seq,
            void* trace, cudaStream_t s) {
  if (B <= 0) return 0;
  if (!src || !tgt || !out || !err || !last || !ws || !device_ptrs({src, tgt, init, out, err, last, ws, trace}))
    return (int)cudaErrorInvalidValue;
  if (Ns <= 0 || Nt <= 0 || Ns > 0x7fffffffLL || Nt > 0x7fffffffLL || (ord != 0 && ord != 1 && ord != 2))
    return (int)cudaErrorInvalidValue;
  double* st = reinterpret_cast<double*>(ws);
  unsigned* ticket = reinterpret_cast<unsigned*>(st + kStWords);
  double* A = st + 2 * kStWords;
  double* part = A + B * 12;
  const int nx = (int)icp_nx(B, Ns);
  const double eps = sizeof(T) == 4 ? 1e-6 : 1e-12;
  const R2bCtl ctl{max_steps, patience, decreasing, tol};
  if (host_out) reinterpret_cast<volatile double*>(host_out)[kStWords - 1] = -1.0;
  if (first) icp_init_kernel<T><<<(unsigned)((B + 127) / 128), 128, 0, s>>>(init, ibs, A, st, ticket, last, out, (int)B);
  for (long long it = 0; it < iters; ++it) {
    char* blk = trace ? reinterpret_cast<char*>(trace) + it * icp_rec_block(B, Ns) : nullptr;
    double* rec_ad = reinterpret_cast<double*>(blk);
    int* rec_idx = blk ? reinterpret_cast<int*>(blk + icp_rec_ad_bytes(B)) : nullptr;
    if (ord == 2) launch_match<T, 2>(src, sbs, tgt, tbs, B, Ns, Nt, A, st, part, nx, decide, rec_idx, s);
    else if (ord == 1) launch_match<T, 1>(src, sbs, tgt, tbs, B, Ns, Nt, A, st, part, nx, decide, rec_idx, s);
    else launch_match<T, 0>(src, sbs, tgt, tbs, B, Ns, Nt, A, st, part, nx, decide, rec_idx, s);
    icp_update_kernel<T><<<(unsigned)B, kUpdThreads, 0, s>>>(tgt, tbs, A, part, nx, st, ticket, last, err, out, (int)B, decide,
                                                             ctl, eps, host_out, (double)seq, it == iters - 1, rec_ad);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  if (!host_out || iters <= 0) return 0;
  return wait_seq(host_out, seq, s);
}


// ----------------------------------------------------------------------------------------------------------------------
// ICP backward (DESIGN.md §3.4, "Gradients").  Per batch element b and point i, in fp64: G = the cotangent of the current
// moved point p_k = A_k s, GS = the source's cotangent through the closing svdtf(source, p_K), C = a point's contribution
// to its matched target in the current iteration, GT = the target cotangent.  Workspace, each part 256-byte aligned:
// G, GS, C (B Ns 3) | GT (TB Nt 3) | coef (B x 32) | part (B nx 15) | gi (B x 7) | keys[2], vals[2] (B Ns u32) | CUB.
// ----------------------------------------------------------------------------------------------------------------------
constexpr int kBwdThreads = 256, kBwdPer = 4;   // per-CTA sums over 1024 points
constexpr int kCoef = 32;
long long icp_bwd_nx(long long Ns) { return (Ns + kBwdThreads * kBwdPer - 1) / (kBwdThreads * kBwdPer); }
long long al256(long long n) { return (n + 255) / 256 * 256; }
int key_bits(long long n) {
  int b = 1;
  while (b < 32 && (1LL << b) < n) ++b;
  return b;
}
size_t icp_sort_bytes(long long n, int bits) {
  size_t tb = 0;
  cub::DoubleBuffer<unsigned> k(nullptr, nullptr), v(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, tb, k, v, (int)n, 0, bits);
  return tb;
}
struct IcpBwdWs {
  double *G, *GS, *C, *GT, *coef, *part, *gi;
  unsigned *keys[2], *vals[2];
  void* tmp;
  size_t tmp_bytes;
  long long bytes;
};
IcpBwdWs icp_bwd_layout(char* base, long long B, long long Ns, long long Nt, long long TB) {
  IcpBwdWs w;
  const long long BN = B * Ns;
  long long o = 0;
  auto take = [&](long long n) { char* p = base ? base + o : nullptr; o += al256(n); return p; };
  w.G = (double*)take(BN * 24); w.GS = (double*)take(BN * 24); w.C = (double*)take(BN * 24);
  w.GT = (double*)take(TB * Nt * 24); w.coef = (double*)take(B * kCoef * 8);
  w.part = (double*)take(B * icp_bwd_nx(Ns) * 15 * 8); w.gi = (double*)take(B * 7 * 8);
  for (int k = 0; k < 2; ++k) { w.keys[k] = (unsigned*)take(BN * 4); w.vals[k] = (unsigned*)take(BN * 4); }
  w.tmp_bytes = icp_sort_bytes(BN, key_bits(TB * Nt));
  w.tmp = take((long long)w.tmp_bytes);
  w.bytes = o;
  return w;
}

template <typename T> __device__ __forceinline__ void ld3(const T* p, double x[3]) {
  x[0] = (double)p[0]; x[1] = (double)p[1]; x[2] = (double)p[2];
}
__device__ __forceinline__ void aff(const double* A, const double s[3], double p[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = fma(A[4 * c], s[0], fma(A[4 * c + 1], s[1], fma(A[4 * c + 2], s[2], A[4 * c + 3])));
}
__device__ __forceinline__ void rot(const double* A, const double d[3], double e[3]) {   // rotation part of a 3x4 A
#pragma unroll
  for (int c = 0; c < 3; ++c) e[c] = A[4 * c] * d[0] + A[4 * c + 1] * d[1] + A[4 * c + 2] * d[2];
}
__device__ __forceinline__ void mv(const double* M, const double x[3], bool tr, double y[3]) {   // y (+)= M x or M^T x
#pragma unroll
  for (int r = 0; r < 3; ++r)
    y[r] += tr ? M[r] * x[0] + M[3 + r] * x[1] + M[6 + r] * x[2] : M[3 * r] * x[0] + M[3 * r + 1] * x[1] + M[3 * r + 2] * x[2];
}

// Per-CTA sums, grid nx x B.  FINAL: over d = s - s_0 and e = R_A d (A = A_K): sum d, sum e, sum e d^T (15).
// Otherwise: sum g [A s; 1]^T (12, 3x4 row major), g = G.  A: 12 doubles per batch element, `as` apart.
template <typename T, bool FINAL>
__global__ void __launch_bounds__(kBwdThreads) icp_bwd_sums_kernel(const T* __restrict__ src, long long sbs, int Ns,
                                                                   const double* __restrict__ A, int as,
                                                                   const double* __restrict__ G, double* __restrict__ part,
                                                                   int nx) {
  constexpr int NS = FINAL ? 15 : 12;
  __shared__ double red[kBwdThreads / 32][NS];
  const int x = blockIdx.x % nx, b = blockIdx.x / nx;
  const T* S = src + (long long)b * sbs;
  double a[12], cs[3], acc[NS];
#pragma unroll
  for (int k = 0; k < 12; ++k) a[k] = A[(long long)b * as + k];
  ld3(S, cs);
#pragma unroll
  for (int k = 0; k < NS; ++k) acc[k] = 0.0;
#pragma unroll
  for (int r = 0; r < kBwdPer; ++r) {
    const int i = (x * kBwdPer + r) * kBwdThreads + (int)threadIdx.x;
    if (i >= Ns) continue;
    double s[3], p[3];
    ld3(S + (long long)i * 3, s);
    if (FINAL) {
      const double d[3] = {s[0] - cs[0], s[1] - cs[1], s[2] - cs[2]};
      rot(a, d, p);
#pragma unroll
      for (int c = 0; c < 3; ++c) { acc[c] += d[c]; acc[3 + c] += p[c]; }
#pragma unroll
      for (int r2 = 0; r2 < 3; ++r2)
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[6 + 3 * r2 + c] += p[r2] * d[c];
    } else {
      aff(a, s, p);
      const double* g = G + ((long long)b * Ns + i) * 3;
#pragma unroll
      for (int r2 = 0; r2 < 3; ++r2) {
        const double gr = g[r2];
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[4 * r2 + c] += gr * p[c];
        acc[4 * r2 + 3] += gr;
      }
    }
  }
  block_sums<kBwdThreads, NS>(acc, red);
  if (threadIdx.x < NS) part[((long long)b * nx + x) * NS + threadIdx.x] = red[0][threadIdx.x];
}

// One CTA per batch element: the partials in a fixed order, then thread 0 solves the per-batch adjoint.
// MODE 0: closing svdtf -> coef = [GH 9, md 3, me 3, dms 3, dmt 3]; 1: iteration (rec: its trace) -> coef = [R 9, GH 9,
// ms 3, mt 3, dms 3, dmt 3]; 2: init -> gi = [sum g, sum p x g, 0].
template <typename T, int MODE>
__global__ void __launch_bounds__(kUpdThreads) icp_bwd_batch_kernel(const double* __restrict__ part, int nx,
                                                                    const T* __restrict__ src, long long sbs,
                                                                    const T* __restrict__ tgt, long long tbs, int Ns,
                                                                    const double* __restrict__ rec,
                                                                    const T* __restrict__ gout, double eps,
                                                                    double* __restrict__ coef, double* __restrict__ gi) {
  constexpr int NS = MODE == 0 ? 15 : 12;
  __shared__ double red[kUpdThreads / 32][NS];
  const int b = blockIdx.x;
  double acc[NS];
#pragma unroll
  for (int k = 0; k < NS; ++k) acc[k] = 0.0;
  for (int x = threadIdx.x; x < nx; x += kUpdThreads)
#pragma unroll
    for (int k = 0; k < NS; ++k) acc[k] += part[((long long)b * nx + x) * NS + k];
  block_sums<kUpdThreads, NS>(acc, red);
  if (threadIdx.x != 0) return;
  const double* P = red[0];
  double* c = coef + (long long)b * kCoef;
  if (MODE == 0) {
    double cs[3], g[7], GH[3][3];
    ld3(src + (long long)b * sbs, cs);
    for (int k = 0; k < 7; ++k) g[k] = (double)gout[(long long)b * 7 + k];
    icp_final_adj(P, cs, (double)Ns, eps, g, GH, c + 9, c + 12, c + 15, c + 18);
    for (int k = 0; k < 9; ++k) c[k] = GH[k / 3][k % 3];
  } else if (MODE == 1) {
    double c0[3], R[3][3], GH[3][3];
    ld3(tgt + (long long)b * tbs, c0);
    icp_iter_adj(rec + (long long)b * kRecD + 12, c0, eps, P, R, GH, c + 18, c + 21, c + 24, c + 27);
    for (int k = 0; k < 9; ++k) { c[k] = R[k / 3][k % 3]; c[9 + k] = GH[k / 3][k % 3]; }
  } else {
    double* o = gi + (long long)b * 7;
    o[0] = P[3]; o[1] = P[7]; o[2] = P[11];
    o[3] = P[9] - P[6]; o[4] = P[2] - P[8]; o[5] = P[4] - P[1]; o[6] = 0.0;
  }
}

// closing svdtf, one thread per (b, i): G = GH (d - md) + dmt (cotangent of p_K), GS = GH^T (e - me) + dms
template <typename T>
__global__ void icp_bwd_final_pts_kernel(const T* __restrict__ src, long long sbs, int Ns, long long BN,
                                         const double* __restrict__ A, const double* __restrict__ coef,
                                         double* __restrict__ G, double* __restrict__ GS) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= BN) return;
  const long long b = g / Ns, i = g - b * Ns;
  const T* S = src + b * sbs;
  double cs[3], s[3], e[3];
  ld3(S, cs);
  ld3(S + i * 3, s);
  const double d[3] = {s[0] - cs[0], s[1] - cs[1], s[2] - cs[2]};
  rot(A + b * 12, d, e);
  const double* c = coef + b * kCoef;
  const double x[3] = {d[0] - c[9], d[1] - c[10], d[2] - c[11]}, y[3] = {e[0] - c[12], e[1] - c[13], e[2] - c[14]};
  double gp[3] = {c[18], c[19], c[20]}, gs[3] = {c[15], c[16], c[17]};
  mv(c, x, false, gp);
  mv(c, y, true, gs);
  for (int k = 0; k < 3; ++k) { G[g * 3 + k] = gp[k]; GS[g * 3 + k] = gs[k]; }
}

// one iteration, one thread per (b, i): p = A_{k-1} s, y its match; G <- R^T G + GH^T (y - mt) + dms, C = GH (p - ms) + dmt,
// and the sort pair (target row, b Ns + i) when the target gradient is wanted.
template <typename T>
__global__ void icp_bwd_iter_pts_kernel(const T* __restrict__ src, long long sbs, const T* __restrict__ tgt, long long tbs,
                                        int Ns, int Nt, long long BN, const double* __restrict__ rec,
                                        const int* __restrict__ idx, const double* __restrict__ coef, double* __restrict__ G,
                                        double* __restrict__ C, unsigned* __restrict__ keys, unsigned* __restrict__ vals) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= BN) return;
  const long long b = g / Ns, i = g - b * Ns;
  const double* c = coef + b * kCoef;
  const int m = idx[g];
  double s[3], p[3], y[3];
  ld3(src + b * sbs + i * 3, s);
  aff(rec + b * kRecD, s, p);
  ld3(tgt + b * tbs + (long long)m * 3, y);
  const double gk[3] = {G[g * 3], G[g * 3 + 1], G[g * 3 + 2]};
  const double ym[3] = {y[0] - c[21], y[1] - c[22], y[2] - c[23]}, pm[3] = {p[0] - c[18], p[1] - c[19], p[2] - c[20]};
  double gn[3] = {c[24], c[25], c[26]}, ct[3] = {c[27], c[28], c[29]};
  mv(c, gk, true, gn);
  mv(c + 9, ym, true, gn);
  mv(c + 9, pm, false, ct);
  for (int k = 0; k < 3; ++k) { G[g * 3 + k] = gn[k]; C[g * 3 + k] = ct[k]; }
  if (keys) { keys[g] = (unsigned)((tbs ? b : 0) * Nt + m); vals[g] = (unsigned)g; }
}

// segmented sum over the (target row, point) pairs sorted by row, points in increasing order: the first entry of each
// row adds the row's contributions to GT in that order.  No atomics: the result does not depend on scheduling.
__global__ void icp_bwd_scatter_kernel(const unsigned* __restrict__ keys, const unsigned* __restrict__ vals, long long n,
                                       const double* __restrict__ C, double* __restrict__ GT) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const unsigned k = keys[p];
  if (p > 0 && keys[p - 1] == k) return;
  double a0 = 0.0, a1 = 0.0, a2 = 0.0;
  for (long long q = p; q < n && keys[q] == k; ++q) {
    const double* ct = C + (long long)vals[q] * 3;
    a0 += ct[0]; a1 += ct[1]; a2 += ct[2];
  }
  GT[(long long)k * 3] += a0; GT[(long long)k * 3 + 1] += a1; GT[(long long)k * 3 + 2] += a2;
}

// source gradient: GS + R_0^T G (G when there is no init), summed over b in order for a broadcast source
template <typename T>
__global__ void icp_bwd_src_kernel(const double* __restrict__ G, const double* __restrict__ GS, const double* __restrict__ A0,
                                   int as, int has_init, long long B, int Ns, int bcast, T* __restrict__ out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (bcast ? 1 : B) * Ns) return;
  const long long b0 = bcast ? 0 : g / Ns, i = g - b0 * Ns, b1 = bcast ? B : b0 + 1;
  double acc[3] = {0.0, 0.0, 0.0};
  for (long long b = b0; b < b1; ++b) {
    const long long e = (b * Ns + i) * 3;
    const double gk[3] = {G[e], G[e + 1], G[e + 2]};
    double r[3] = {GS[e], GS[e + 1], GS[e + 2]};
    if (has_init) {
      const double* a = A0 + b * as;
      for (int c = 0; c < 3; ++c) r[c] += a[c] * gk[0] + a[4 + c] * gk[1] + a[8 + c] * gk[2];
    } else {
      for (int c = 0; c < 3; ++c) r[c] += gk[c];
    }
    for (int c = 0; c < 3; ++c) acc[c] += r[c];
  }
  for (int c = 0; c < 3; ++c) out[g * 3 + c] = (T)acc[c];
}

// rows of w doubles -> T, summed over the B rows in order when `sum` (a broadcast operand)
template <typename T>
__global__ void icp_bwd_out_kernel(const double* __restrict__ x, long long rows, int w, int sum, T* __restrict__ out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (sum ? w : rows * w)) return;
  double a = 0.0;
  if (sum)
    for (long long r = 0; r < rows; ++r) a += x[r * w + g];
  else
    a = x[g];
  out[g] = (T)a;
}

unsigned blocks(long long n, int nt) { return (unsigned)((n + nt - 1) / nt); }

template <typename T>
int icp_bwd_run(const T* src, long long sbs, const T* tgt, long long tbs, const T* init, long long ibs, const void* fwd_ws,
                const long long* trace_host, long long K, const T* gout, T* gsrc, T* gtgt, T* ginit, void* ws, long long B,
                long long Ns, long long Nt, cudaStream_t s) {
  if (B <= 0) return 0;
  if (!src || !tgt || !fwd_ws || !gout || !ws || (K > 0 && !trace_host) || K < 0 || (ginit && !init) ||
      !device_ptrs({src, tgt, init, fwd_ws, gout, gsrc, gtgt, ginit, ws}))
    return (int)cudaErrorInvalidValue;
  for (long long k = 0; k < K; ++k)
    if (!trace_host[k] || !device_ptrs({reinterpret_cast<const void*>(trace_host[k])})) return (int)cudaErrorInvalidValue;
  const long long TB = tbs ? B : 1, BN = B * Ns;
  if (Ns <= 0 || Nt <= 0 || BN > 0x7fffffffLL || TB * Nt > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  const IcpBwdWs w = icp_bwd_layout(reinterpret_cast<char*>(ws), B, Ns, Nt, TB);
  const double* AK = reinterpret_cast<const double*>(fwd_ws) + 2 * kStWords;
  auto rec = [&](long long k) { return reinterpret_cast<const double*>(trace_host[k]); };   // iteration k + 1
  const int nx = (int)icp_bwd_nx(Ns);
  const double eps = sizeof(T) == 4 ? 1e-6 : 1e-12;
  const unsigned gb = (unsigned)(B * nx), pb = blocks(BN, 256);
  icp_bwd_sums_kernel<T, true><<<gb, kBwdThreads, 0, s>>>(src, sbs, (int)Ns, AK, 12, nullptr, w.part, nx);
  icp_bwd_batch_kernel<T, 0><<<(unsigned)B, kUpdThreads, 0, s>>>(w.part, nx, src, sbs, tgt, tbs, (int)Ns, nullptr, gout, eps,
                                                                  w.coef, nullptr);
  icp_bwd_final_pts_kernel<T><<<pb, 256, 0, s>>>(src, sbs, (int)Ns, BN, AK, w.coef, w.G, w.GS);
  if (gtgt) cudaMemsetAsync(w.GT, 0, TB * Nt * 24, s);
  const int bits = key_bits(TB * Nt);
  for (long long k = K; k >= 1; --k) {           // iteration k: p_{k-1} -> p_k, trace rec(k - 1); A_k from the next one
    const double* r = rec(k - 1);
    const double* Ak = k < K ? rec(k) : AK;
    const int* idx = reinterpret_cast<const int*>(reinterpret_cast<const char*>(r) + icp_rec_ad_bytes(B));
    icp_bwd_sums_kernel<T, false><<<gb, kBwdThreads, 0, s>>>(src, sbs, (int)Ns, Ak, k < K ? kRecD : 12, w.G, w.part, nx);
    icp_bwd_batch_kernel<T, 1><<<(unsigned)B, kUpdThreads, 0, s>>>(w.part, nx, src, sbs, tgt, tbs, (int)Ns, r, nullptr, eps,
                                                                    w.coef, nullptr);
    icp_bwd_iter_pts_kernel<T><<<pb, 256, 0, s>>>(src, sbs, tgt, tbs, (int)Ns, (int)Nt, BN, r, idx, w.coef, w.G, w.C,
                                                  gtgt ? w.keys[0] : nullptr, w.vals[0]);
    if (gtgt) {
      cub::DoubleBuffer<unsigned> kb(w.keys[0], w.keys[1]), vb(w.vals[0], w.vals[1]);
      size_t tb = w.tmp_bytes;
      const cudaError_t e = cub::DeviceRadixSort::SortPairs(w.tmp, tb, kb, vb, (int)BN, 0, bits, s);
      if (e != cudaSuccess) return (int)e;
      icp_bwd_scatter_kernel<<<pb, 256, 0, s>>>(kb.Current(), vb.Current(), BN, w.C, w.GT);
    }
  }
  const double* A0 = K > 0 ? rec(0) : AK;
  const int a0s = K > 0 ? kRecD : 12;
  if (ginit) {                                     // p_0 = init (.) source: the Act gradient of init
    icp_bwd_sums_kernel<T, false><<<gb, kBwdThreads, 0, s>>>(src, sbs, (int)Ns, A0, a0s, w.G, w.part, nx);
    icp_bwd_batch_kernel<T, 2><<<(unsigned)B, kUpdThreads, 0, s>>>(w.part, nx, src, sbs, tgt, tbs, (int)Ns, nullptr, nullptr,
                                                                    eps, w.coef, w.gi);
    const int bc = ibs == 0 && B > 1;
    icp_bwd_out_kernel<T><<<blocks(bc ? 7 : B * 7, 256), 256, 0, s>>>(w.gi, B, 7, bc, ginit);
  }
  if (gsrc) {
    const int bc = sbs == 0 && B > 1;
    icp_bwd_src_kernel<T><<<blocks((bc ? 1 : B) * Ns, 256), 256, 0, s>>>(w.G, w.GS, A0, a0s, init != nullptr, B, (int)Ns, bc,
                                                                         gsrc);
  }
  if (gtgt) icp_bwd_out_kernel<T><<<blocks(TB * Nt * 3, 256), 256, 0, s>>>(w.GT, TB * Nt * 3, 1, 0, gtgt);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace b200pose

using namespace b200pose;

B200_EXPORT long long b200_knn_workspace_bytes(long long B, long long N1, long long N2, long long D, long long k,
                                               long long elem_size) {
  if (B <= 0 || N1 <= 0 || N2 <= 0 || k < 1) return 0;
  return knn_ws_bytes(knn_plan(B, N1, N2, (int)D, (int)k), B, N1, (int)elem_size);
}

B200_EXPORT long long b200_icp_workspace_bytes(long long B, long long Ns) {
  if (B <= 0 || Ns <= 0) return 2 * kStWords * 8;
  return (2 * kStWords + B * 12 + B * icp_nx(B, Ns) * kSums) * 8;
}

B200_EXPORT long long b200_icp_trace_bytes(long long B, long long Ns, long long iters) {
  if (B <= 0 || Ns <= 0 || iters <= 0) return 0;
  return iters * icp_rec_block(B, Ns);
}

B200_EXPORT long long b200_icp_bwd_workspace_bytes(long long B, long long Ns, long long Nt, long long tgt_batches) {
  if (B <= 0 || Ns <= 0 || Nt <= 0) return 0;
  return icp_bwd_layout(nullptr, B, Ns, Nt, tgt_batches > 1 ? B : 1).bytes;
}

#define B200_KNN_ENTRIES(CT, SFX)                                                                                          \
  B200_EXPORT int b200_knn_##SFX(const CT* ref, long long ref_bstride, const CT* nbr, long long nbr_bstride, CT* values,    \
                                 long long* indices, void* ws, long long B, long long N1, long long N2, int D, int k,      \
                                 int ord, int largest, void* stream) {                                                     \
    KnnArgs<CT> a{ref, ref_bstride, nbr, nbr_bstride, values, indices, ws, B, N1, N2, D, k, ord, largest};                 \
    return knn_run<CT>(a, (cudaStream_t)stream);                                                                           \
  }                                                                                                                        \
  B200_EXPORT int b200_radius_mask_##SFX(const CT* pts, long long N, int D, double thr, int ord, long long need,           \
                                         unsigned char* mask_out, void* stream) {                                          \
    return radius_run<CT>(pts, N, D, thr, ord, need, mask_out, (cudaStream_t)stream);                                      \
  }                                                                                                                        \
  B200_EXPORT int b200_icp_##SFX(const CT* src, long long src_bstride, const CT* tgt, long long tgt_bstride,               \
                                 const CT* init, long long init_bstride, CT* out, CT* err, CT* last, void* ws, long long B, \
                                 long long Ns, long long Nt, int ord, long long first, long long iters, int decide,        \
                                 long long max_steps, long long patience, double decreasing, double tol,                   \
                                 double* host_out, long long seq, void* stream) {                                          \
    return icp_run<CT>(src, src_bstride, tgt, tgt_bstride, init, init_bstride, out, err, last, ws, B, Ns, Nt, ord, first,  \
                       iters, decide, max_steps, patience, decreasing, tol, host_out, seq, nullptr, (cudaStream_t)stream); \
  }                                                                                                                        \
  B200_EXPORT int b200_icp_rec_##SFX(const CT* src, long long src_bstride, const CT* tgt, long long tgt_bstride,           \
                                     const CT* init, long long init_bstride, CT* out, CT* err, CT* last, void* ws,         \
                                     long long B, long long Ns, long long Nt, int ord, long long first, long long iters,   \
                                     int decide, long long max_steps, long long patience, double decreasing, double tol,   \
                                     double* host_out, long long seq, void* trace, void* stream) {                         \
    if (!trace && B > 0 && iters > 0) return (int)cudaErrorInvalidValue;                                                   \
    return icp_run<CT>(src, src_bstride, tgt, tgt_bstride, init, init_bstride, out, err, last, ws, B, Ns, Nt, ord, first,  \
                       iters, decide, max_steps, patience, decreasing, tol, host_out, seq, trace, (cudaStream_t)stream);   \
  }                                                                                                                        \
  B200_EXPORT int b200_icp_bwd_##SFX(const CT* src, long long src_bstride, const CT* tgt, long long tgt_bstride,           \
                                     const CT* init, long long init_bstride, const void* fwd_ws,                           \
                                     const long long* trace_host, long long K, const CT* grad_out, CT* grad_src,           \
                                     CT* grad_tgt, CT* grad_init, void* ws, long long B, long long Ns, long long Nt,       \
                                     void* stream) {                                                                       \
    return icp_bwd_run<CT>(src, src_bstride, tgt, tgt_bstride, init, init_bstride, fwd_ws, trace_host, K, grad_out,        \
                           grad_src, grad_tgt, grad_init, ws, B, Ns, Nt, (cudaStream_t)stream);                            \
  }

B200_KNN_ENTRIES(float, f32)
B200_KNN_ENTRIES(double, f64)
