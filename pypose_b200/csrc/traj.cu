// traj.cu — trajectory metrics pp.metric.ape / rpe (C-ABI: include/b200pose.h, section "trajectory metrics").
// DESIGN.md §3.6.  Per-element math in traj_math.cuh; everything is fp64, poses are widened on load.
//
//   b200_traj_match       one thread per short stamp: binary search in the long stamps (tr_match), both arrays checked
//                         for order in the same pass, then the matches compacted in increasing short index
//   b200_traj_pairs_dist  the path walk of pairs_by_dist in one CTA (warps 1..7 compute the next chunk of segment
//                         lengths into shared memory while lane 0 of warp 0 does the dependent adds), then for all=True
//                         one thread per pose searches its partner in the accumulated distances (tr_pair)
//   b200_traj_err         one thread per pair: gather, align by a Sim3 read from device memory, error
//   b200_traj_stats       Max/Min/Mean/RMSE/SSE/STD from fixed-order per-CTA partials folded by the last CTA, STD in a
//                         second pass around the mean; the median is an exact radix select on the bit patterns of |e|
// No entry point reads anything back to the host.
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <initializer_list>
#include "traj_math.cuh"

#define B200_EXPORT extern "C" __attribute__((visibility("default")))

namespace b200pose {
namespace {

constexpr int kTrThreads = 256;
constexpr int kWalkChunk = 2048;           // segment lengths per shared-memory buffer (two buffers: 32 KB)
constexpr int kStatMaxGrid = 1024;
constexpr int kStatPerCta = 8 * kTrThreads;

struct TrState {
  unsigned int ticket, pad;
  double sum_abs, sum_sq, mx, mn, mean, m2;
  unsigned long long prefix;
  long long k;
  unsigned long long hist[256];
};

long long align256(long long b) { return (b + 255) / 256 * 256; }

size_t scan_temp_bytes(long long n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, (int)n);
  return b;
}

// workspace: state | stat partials | A[n] i64 | F[n] i32 | P[n] i32 | D[n] f64 | CUB temporary storage
struct TrWs {
  TrState* st;
  double* part;
  long long* A;
  int *F, *P;
  double* D;
  void* tmp;
  size_t tmp_bytes;
};

long long tr_ws_layout(long long n, char* base, TrWs* w) {
  long long off = 0;
  auto take = [&](long long bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  char* st = take(sizeof(TrState));
  char* part = take(kStatMaxGrid * 4 * sizeof(double));
  char* a = take(n * 8); char* f = take(n * 4); char* p = take(n * 4); char* d = take(n * 8);
  const size_t tb = scan_temp_bytes(n);
  char* tmp = take((long long)tb);
  if (w) {
    w->st = reinterpret_cast<TrState*>(st); w->part = reinterpret_cast<double*>(part);
    w->A = reinterpret_cast<long long*>(a); w->F = reinterpret_cast<int*>(f); w->P = reinterpret_cast<int*>(p);
    w->D = reinterpret_cast<double*>(d); w->tmp = tmp; w->tmp_bytes = tb;
  }
  return off;
}

bool tr_device_ptrs(std::initializer_list<const void*> ps) {
  for (const void* p : ps) {
    if (!p) continue;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) return false;
  }
  return true;
}

unsigned grid_of(long long n) { return (unsigned)((n + kTrThreads - 1) / kTrThreads); }

// ---------------------------------------------------------------- association
__global__ void traj_match_kernel(const double* __restrict__ S, long long ns, const double* __restrict__ L, long long nl,
                                  double off, double diff, long long* __restrict__ A, int* __restrict__ F,
                                  unsigned long long* __restrict__ info) {
  const long long t = (long long)blockIdx.x * kTrThreads + threadIdx.x;
  if (t < ns) {
    const double s = S[t];
    if (isnan(s) || (t + 1 < ns && s > S[t + 1])) atomicOr(info + 1, 1ull);
    double d;
    A[t] = tr_match(L, nl, s, off, d);
    F[t] = d < diff;
  }
  if (t < nl) {
    const double l = L[t];
    if (isnan(l) || (t + 1 < nl && l > L[t + 1])) atomicOr(info + 2, 1ull);
  }
}

// out_a[P[i]] = i, out_b[P[i]] = A[i] where F[i]; *count = number of flagged
__global__ void traj_scatter_kernel(const int* __restrict__ F, const int* __restrict__ P, const long long* __restrict__ A,
                                    long long n, long long* __restrict__ out_a, long long* __restrict__ out_b,
                                    long long* __restrict__ count) {
  const long long i = (long long)blockIdx.x * kTrThreads + threadIdx.x;
  if (i >= n) return;
  const int f = F[i], p = P[i];
  if (f) { out_a[p] = i; out_b[p] = A[i]; }
  if (i == n - 1) *count = (long long)p + f;
}

cudaError_t compact(const TrWs& w, long long n, long long* out_a, long long* out_b, long long* count, cudaStream_t s) {
  size_t tb = w.tmp_bytes;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.F, w.P, (int)n, s);
  if (e != cudaSuccess) return e;
  traj_scatter_kernel<<<grid_of(n), kTrThreads, 0, s>>>(w.F, w.P, w.A, n, out_a, out_b, count);
  return cudaGetLastError();
}

// ---------------------------------------------------------------- path walk and distance pairs
template <typename T>
__device__ __forceinline__ V3<double> tr_trans(const T* P, long long rs, long long cs, const long long* idx, long long k,
                                               const double* S) {
  return tr_align(S, tr_load(P + idx[k] * rs, cs)).t;
}

// lengths of segments c0 .. c0 + kWalkChunk - 1 (segment k joins poses k and k + 1) by threads t0, t0 + nt, ...
template <typename T>
__device__ __forceinline__ void walk_fill(double* buf, long long c0, int t0, int nt, const T* P, long long rs, long long cs,
                                          const long long* idx, long long n, const double* S) {
  for (int j = t0; j < kWalkChunk; j += nt) {
    const long long k = c0 + j;
    if (k < n - 1) {
      const V3<double> a = tr_trans(P, rs, cs, idx, k, S), b = tr_trans(P, rs, cs, idx, k + 1, S);
      buf[j] = tr_norm3(a.x - b.x, a.y - b.y, a.z - b.z);
    }
  }
}

// all: D[0] = 0, D[k + 1] = D[k] + l_k (the reference's cat(0, cumsum));
// else: the greedy walk cur += l_{i-1} (0 at i = 0), record i and reset when cur >= delta; list of *count indices
template <typename T>
__global__ void __launch_bounds__(kTrThreads) traj_walk_kernel(const T* __restrict__ P, long long rs, long long cs,
                                                                const long long* __restrict__ idx, long long n,
                                                                const double* __restrict__ S, double delta, int all,
                                                                double* __restrict__ D, long long* __restrict__ list,
                                                                long long* __restrict__ count) {
  __shared__ double buf[2][kWalkChunk];
  const int tid = threadIdx.x;
  const long long nseg = n - 1;
  const long long nchunks = (nseg + kWalkChunk - 1) / kWalkChunk;
  double acc = 0.0;
  long long cnt = 0;
  if (tid == 0) {
    if (all) D[0] = 0.0;
    else if (acc >= delta) { list[cnt++] = 0; }     // i = 0 adds ||t_0 - t_0|| = 0
  }
  if (nchunks > 0) walk_fill(buf[0], 0, tid, kTrThreads, P, rs, cs, idx, n, S);
  __syncthreads();
  for (long long c = 0; c < nchunks; ++c) {
    if (tid >= 32) {
      if (c + 1 < nchunks) walk_fill(buf[(c + 1) & 1], (c + 1) * kWalkChunk, tid - 32, kTrThreads - 32, P, rs, cs, idx, n, S);
    } else if (tid == 0) {
      const double* b = buf[c & 1];
      const long long c0 = c * kWalkChunk;
      const int m = (int)min((long long)kWalkChunk, nseg - c0);
      if (all) {
        for (int j = 0; j < m; ++j) { acc = tr_add(acc, b[j]); D[c0 + j + 1] = acc; }
      } else {
        for (int j = 0; j < m; ++j) {        // branch-free: the store lands on the next free slot, kept when hit
          acc = tr_add(acc, b[j]);
          const bool hit = acc >= delta;
          list[cnt] = c0 + j + 1;
          cnt += hit;
          acc = hit ? 0.0 : acc;
        }
      }
    }
    __syncthreads();
  }
  if (tid == 0 && !all) *count = cnt;
}

__global__ void traj_pair_kernel(const double* __restrict__ D, long long n, double delta, double tol, long long* __restrict__ A,
                                 int* __restrict__ F) {
  const long long i = (long long)blockIdx.x * kTrThreads + threadIdx.x;
  if (i >= n) return;
  if (i == n - 1) { F[i] = 0; A[i] = 0; return; }
  double h;
  A[i] = tr_pair(D, n, i, delta, h);
  F[i] = !(h > tol);
}

// ---------------------------------------------------------------- errors
template <typename T>
__global__ void traj_err_kernel(const T* __restrict__ rp, long long rrs, long long rcs, const T* __restrict__ ep,
                                long long ers, long long ecs, const long long* __restrict__ ra,
                                const long long* __restrict__ rb, const long long* __restrict__ ea,
                                const long long* __restrict__ eb, const double* __restrict__ S, long long M, int etype,
                                double* __restrict__ err) {
  const long long k = (long long)blockIdx.x * kTrThreads + threadIdx.x;
  if (k >= M) return;
  const Elem<double> r0 = tr_load(rp + ra[k] * rrs, rcs);
  const Elem<double> e0 = tr_align(S, tr_load(ep + ea[k] * ers, ecs));
  if (!rb) { err[k] = tr_ape(r0, e0, etype); return; }
  const Elem<double> r1 = tr_load(rp + rb[k] * rrs, rcs);
  const Elem<double> e1 = tr_align(S, tr_load(ep + eb[k] * ers, ecs));
  err[k] = tr_rpe(r0, r1, e0, e1, etype);
}

// ---------------------------------------------------------------- statistics
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || b != b) ? a + b : fmax(a, b); }
__device__ __forceinline__ double nan_min(double a, double b) { return (a != a || b != b) ? a + b : fmin(a, b); }

// fixed-order reduction of v over the CTA (result in thread 0); op: 0 sum, 1 max, 2 min
__device__ __forceinline__ double cta_reduce(double v, int op, double* sh) {
  for (int o = 16; o > 0; o >>= 1) {
    const double u = __shfl_down_sync(0xffffffffu, v, o);
    v = op == 0 ? v + u : op == 1 ? nan_max(v, u) : nan_min(v, u);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int j = 1; j < kTrThreads / 32; ++j) v = op == 0 ? v + sh[j] : op == 1 ? nan_max(v, sh[j]) : nan_min(v, sh[j]);
  return v;
}

// pass 1: sum |e|, sum e^2, max |e|, min |e|; pass 2 (second = 1): sum (|e| - mean)^2.  The last CTA folds the partials
// in CTA order.
__global__ void __launch_bounds__(kTrThreads) traj_stats_kernel(const double* __restrict__ e, long long M, int second,
                                                                 TrState* st, double* part) {
  __shared__ double sh[kTrThreads / 32];
  __shared__ bool last;
  double a = 0.0, q = 0.0, mx = -INFINITY, mn = INFINITY;
  const double mean = second ? st->mean : 0.0;
  for (long long i = (long long)blockIdx.x * kTrThreads + threadIdx.x; i < M; i += (long long)gridDim.x * kTrThreads) {
    const double v = fabs(e[i]);
    if (second) { const double d = v - mean; q = fma(d, d, q); }
    else { a += v; q = fma(v, v, q); mx = nan_max(mx, v); mn = nan_min(mn, v); }
  }
  q = cta_reduce(q, 0, sh);
  if (!second) { a = cta_reduce(a, 0, sh); mx = cta_reduce(mx, 1, sh); mn = cta_reduce(mn, 2, sh); }
  if (threadIdx.x == 0) {
    double* p = part + 4 * blockIdx.x;
    p[0] = q; p[1] = a; p[2] = mx; p[3] = mn;
    __threadfence();
    last = atomicAdd(&st->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double Q = 0.0, A = 0.0, MX = -INFINITY, MN = INFINITY;
  for (unsigned b = 0; b < gridDim.x; ++b) {
    const double* p = part + 4 * b;
    Q += __ldcg(p);
    if (!second) { A += __ldcg(p + 1); MX = nan_max(MX, __ldcg(p + 2)); MN = nan_min(MN, __ldcg(p + 3)); }
  }
  if (second) {
    st->m2 = Q;
  } else {
    st->sum_sq = Q; st->sum_abs = A; st->mx = MX; st->mn = MN; st->mean = A / (double)M;
  }
  st->ticket = 0;
}

// one digit of the radix select: histogram of the 8 bits at `shift` over the |e| whose higher bits equal the prefix
__global__ void __launch_bounds__(kTrThreads) traj_hist_kernel(const double* __restrict__ e, long long M, int shift,
                                                                unsigned long long hi_mask, TrState* st) {
  __shared__ unsigned int h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const unsigned long long prefix = st->prefix;
  for (long long i = (long long)blockIdx.x * kTrThreads + threadIdx.x; i < M; i += (long long)gridDim.x * kTrThreads) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(fabs(e[i]));
    if ((b & hi_mask) == prefix) atomicAdd(&h[(b >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&st->hist[threadIdx.x], (unsigned long long)h[threadIdx.x]);
}

// pick the digit holding rank k, narrow the prefix, clear the histogram
__global__ void traj_select_kernel(int shift, long long k0, TrState* st) {
  if (threadIdx.x != 0) return;
  long long k = shift == 56 ? k0 : st->k;
  unsigned long long cum = 0;
  int d = 255;
  for (int j = 0; j < 256; ++j) {
    const unsigned long long c = st->hist[j];
    if ((unsigned long long)k < cum + c) { d = j; break; }
    cum += c;
  }
  st->k = k - (long long)cum;
  st->prefix |= (unsigned long long)d << shift;
  for (int j = 0; j < 256; ++j) st->hist[j] = 0;
}

// out = [Max, Min, Mean, Median, RMSE, SSE, STD]
__global__ void traj_final_kernel(const TrState* st, long long M, double* out) {
  if (threadIdx.x != 0) return;
  const double m = (double)M;
  out[0] = st->mx; out[1] = st->mn; out[2] = st->mean;
  out[3] = __longlong_as_double((long long)st->prefix);
  out[4] = sqrt(st->sum_sq / m); out[5] = st->sum_sq;
  out[6] = sqrt(st->m2 / (m - 1.0));
}

// ---------------------------------------------------------------- entry points
int match_run(const double* S, long long ns, const double* L, long long nl, double off, double diff, void* ws,
              long long* idx_short, long long* idx_long, long long* info, cudaStream_t s) {
  if (ns <= 0 || nl <= 0 || ns > 0x7fffffffLL || nl > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  if (!S || !L || !ws || !idx_short || !idx_long || !info || !tr_device_ptrs({S, L, ws, idx_short, idx_long, info}))
    return (int)cudaErrorInvalidValue;
  TrWs w;
  tr_ws_layout(ns, reinterpret_cast<char*>(ws), &w);
  cudaError_t e = cudaMemsetAsync(info, 0, 3 * sizeof(long long), s);
  if (e != cudaSuccess) return (int)e;
  traj_match_kernel<<<grid_of(ns > nl ? ns : nl), kTrThreads, 0, s>>>(S, ns, L, nl, off, diff, w.A, w.F,
                                                                      reinterpret_cast<unsigned long long*>(info));
  return (int)compact(w, ns, idx_short, idx_long, info, s);
}

template <typename T>
int pairs_run(const T* P, long long rs, long long cs, const long long* idx, long long n, const double* Sim, double delta,
              double tol, int all, void* ws, long long* src, long long* tgt, long long* count, cudaStream_t s) {
  if (n <= 0 || n > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  if (!P || !idx || !ws || !src || !count || (all && !tgt) || !tr_device_ptrs({P, idx, Sim, ws, src, tgt, count}))
    return (int)cudaErrorInvalidValue;
  TrWs w;
  tr_ws_layout(n, reinterpret_cast<char*>(ws), &w);
  traj_walk_kernel<T><<<1, kTrThreads, 0, s>>>(P, rs, cs, idx, n, Sim, delta, all, w.D, src, count);
  if (!all) return (int)cudaGetLastError();
  traj_pair_kernel<<<grid_of(n), kTrThreads, 0, s>>>(w.D, n, delta, tol, w.A, w.F);
  return (int)compact(w, n, src, tgt, count, s);
}

template <typename T>
int err_run(const T* rp, long long rrs, long long rcs, const T* ep, long long ers, long long ecs, const long long* ra,
            const long long* rb, const long long* ea, const long long* eb, const double* Sim, long long M, int etype,
            double* err, cudaStream_t s) {
  if (M <= 0) return 0;
  if (!rp || !ep || !ra || !ea || !err || (!rb) != (!eb) || etype < kTrTranslation || etype > kTrDegree ||
      !tr_device_ptrs({rp, ep, ra, rb, ea, eb, Sim, err}))
    return (int)cudaErrorInvalidValue;
  traj_err_kernel<T><<<grid_of(M), kTrThreads, 0, s>>>(rp, rrs, rcs, ep, ers, ecs, ra, rb, ea, eb, Sim, M, etype, err);
  return (int)cudaGetLastError();
}

int stats_run(const double* e, long long M, int mask, void* ws, double* out, cudaStream_t s) {
  if (M <= 0) return (int)cudaErrorInvalidValue;
  if (!e || !ws || !out || !tr_device_ptrs({e, ws, out})) return (int)cudaErrorInvalidValue;
  TrWs w;
  tr_ws_layout(0, reinterpret_cast<char*>(ws), &w);
  cudaError_t err = cudaMemsetAsync(w.st, 0, sizeof(TrState), s);
  if (err != cudaSuccess) return (int)err;
  const long long g = (M + kStatPerCta - 1) / kStatPerCta;
  const unsigned grid = (unsigned)(g < kStatMaxGrid ? g : kStatMaxGrid);
  traj_stats_kernel<<<grid, kTrThreads, 0, s>>>(e, M, 0, w.st, w.part);
  if (mask & (1 << 6)) traj_stats_kernel<<<grid, kTrThreads, 0, s>>>(e, M, 1, w.st, w.part);
  if (mask & (1 << 3)) {
    unsigned long long hi = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
      traj_hist_kernel<<<grid, kTrThreads, 0, s>>>(e, M, shift, hi, w.st);
      traj_select_kernel<<<1, 32, 0, s>>>(shift, (M - 1) / 2, w.st);
      hi |= 255ull << shift;
    }
  }
  traj_final_kernel<<<1, 32, 0, s>>>(w.st, M, out);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace b200pose

using namespace b200pose;

B200_EXPORT long long b200_traj_workspace_bytes(long long n) {
  if (n < 0 || n > 0x7fffffffLL) return 0;
  return tr_ws_layout(n, nullptr, nullptr);
}

B200_EXPORT int b200_traj_match(const double* s_short, long long n_short, const double* s_long, long long n_long,
                                double offset, double diff, void* ws, long long* idx_short, long long* idx_long,
                                long long* info, void* stream) {
  return match_run(s_short, n_short, s_long, n_long, offset, diff, ws, idx_short, idx_long, info, (cudaStream_t)stream);
}

B200_EXPORT int b200_traj_stats(const double* err, long long M, int mask, void* ws, double* out, void* stream) {
  return stats_run(err, M, mask, ws, out, (cudaStream_t)stream);
}

#define B200_TRAJ_ENTRIES(CT, SFX)                                                                                         \
  B200_EXPORT int b200_traj_pairs_dist_##SFX(const CT* pose, long long row_stride, long long col_stride,                  \
                                             const long long* idx, long long n, const double* sim3, double delta,         \
                                             double tol, int all, void* ws, long long* src, long long* tgt,               \
                                             long long* count, void* stream) {                                            \
    return pairs_run<CT>(pose, row_stride, col_stride, idx, n, sim3, delta, tol, all, ws, src, tgt, count,                \
                         (cudaStream_t)stream);                                                                           \
  }                                                                                                                        \
  B200_EXPORT int b200_traj_err_##SFX(const CT* rpose, long long r_row_stride, long long r_col_stride, const CT* epose,    \
                                      long long e_row_stride, long long e_col_stride, const long long* r_a,               \
                                      const long long* r_b, const long long* e_a, const long long* e_b,                   \
                                      const double* sim3, long long M, int etype, double* err, void* stream) {            \
    return err_run<CT>(rpose, r_row_stride, r_col_stride, epose, e_row_stride, e_col_stride, r_a, r_b, e_a, e_b, sim3,   \
                       M, etype, err, (cudaStream_t)stream);                                                              \
  }

B200_TRAJ_ENTRIES(float, f32)
B200_TRAJ_ENTRIES(double, f64)
