// pcg_vec.cuh — the vector side of the block-Jacobi PCG (pcg.cu, bal.cu): the device-resident state,
// the point-block solves and the CG vector kernels, generic in the block width W of the unknowns (6: SE3 tangents,
// 9: a BAL camera).
#pragma once
#include "lm_common.cuh"
#include "bal_math.cuh"

namespace b200pose {

// state (16 doubles).  DONE: 0 running, 1 converged (|r| <= tol |b|), 2 breakdown (p.Ap <= 0), 3 stagnated (no new minimum of
// |r| for PATIENCE = max(100, unknowns) iterations), 4 maxiter.  BEST / SINCE / SAVE guard the solve against finite-precision CG: when the
// tolerance is below what the arithmetic can reach (fp32, ill-conditioned Schur complements) the iterate degrades after
// its best point, so the iterate with the smallest recursive residual is kept in xbest and returned unless the solve
// converged (then the last iterate IS the best one, i.e. attainable tolerances behave exactly like solver.py:312-340).
enum { CG_RZ0 = 0, CG_RZ1 = 1, CG_PQ = 2, CG_RR = 3, CG_STOP2 = 4, CG_DONE = 5, CG_ITERS = 6, CG_MAXIT = 7,
       CG_BEST = 8, CG_SINCE = 9, CG_SAVE = 10, CG_PATIENCE = 11, CG_STATE = 16 };
constexpr double kCgPatience = 100.0;

// after an update produced |r|^2 = rr: bookkeeping of the best iterate and the stop decision (one thread)
__device__ __forceinline__ void cg_after_update(double* cg, double rr, double it) {
  if (rr < cg[CG_BEST]) { cg[CG_BEST] = rr; cg[CG_SINCE] = 0.0; cg[CG_SAVE] = 1.0; }
  else { cg[CG_SINCE] += 1.0; cg[CG_SAVE] = 0.0; }
  if (!(rr > cg[CG_STOP2])) cg[CG_DONE] = 1.0;
  else if (it >= cg[CG_MAXIT]) cg[CG_DONE] = 4.0;
  else if (cg[CG_SINCE] >= cg[CG_PATIENCE]) cg[CG_DONE] = 3.0;
}

// (n, 6) vectors are read and written as three 8-byte (float) / 16-byte (double) pairs: a node's six values start at a
// multiple of 24 / 48 bytes, so the arrays only have to be 8- / 16-byte aligned (checked at the entry points).  Scalar
// accesses cost one LSU wavefront per touched line and instruction — 36 per warp and vector instead of 18 (the PCG
// kernels are LSU-bound, not DRAM-bound).
template <typename T> struct Pair6;
template <> struct Pair6<float> { using type = float2; };
template <> struct Pair6<double> { using type = double2; };
template <typename T> __device__ __forceinline__ void ld6(const T* p, long long i, T (&v)[6]) {
  using P = typename Pair6<T>::type;
  const P* q = reinterpret_cast<const P*>(p + i * 6);
#pragma unroll
  for (int k = 0; k < 3; ++k) { const P t = q[k]; v[2 * k] = t.x; v[2 * k + 1] = t.y; }
}
template <typename T> __device__ __forceinline__ void st6(T* p, long long i, const T (&v)[6]) {
  using P = typename Pair6<T>::type;
  P* q = reinterpret_cast<P*>(p + i * 6);
#pragma unroll
  for (int k = 0; k < 3; ++k) { P t; t.x = v[2 * k]; t.y = v[2 * k + 1]; q[k] = t; }
}
template <typename T> __device__ __forceinline__ void sym6_mv_packed(const T* a21, const T (&x)[6], T (&y)[6]) {
  T A[6][6];
  sym6_unpack(a21, A);
  sym6_mv(A, x, y);
}
// block rows of W unknowns: (n, 6) rows as pairs (above); (n, 9) rows start at multiples of 36 / 72 bytes and are read
// value by value
template <int W> constexpr int packed_words() { return W * (W + 1) / 2; }
template <typename T, int W> __device__ __forceinline__ void ldw(const T* p, long long i, T (&v)[W]) {
  if constexpr (W == 6) {
    ld6(p, i, v);
  } else {
#pragma unroll
    for (int k = 0; k < W; ++k) v[k] = p[i * W + k];
  }
}
template <typename T, int W> __device__ __forceinline__ void stw(T* p, long long i, const T (&v)[W]) {
  if constexpr (W == 6) {
    st6(p, i, v);
  } else {
#pragma unroll
    for (int k = 0; k < W; ++k) p[i * W + k] = v[k];
  }
}
template <typename T, int W> __device__ __forceinline__ void symw_mv_packed(const T* a, const T (&x)[W], T (&y)[W]) {
  if constexpr (W == 6) sym6_mv_packed(a, x, y);
  else symn_mv_packed<T, W>(a, x, y);
}
// q = D p with D none (0), diagonal (n,W) (1) or packed symmetric blocks (n,W(W+1)/2) (2)
template <typename T, int W>
__device__ __forceinline__ void apply_D(const T* D, int dmode, long long i, const T (&p)[W], T (&q)[W]) {
  if (dmode == 2) {
    symw_mv_packed<T, W>(D + i * packed_words<W>(), p, q);
  } else {
#pragma unroll
    for (int k = 0; k < W; ++k) q[k] = dmode == 1 ? D[i * W + k] * p[k] : T(0);
  }
}

template <typename T>
__global__ void __launch_bounds__(kLmThreads) pt3_damp_inv_kernel(const T* __restrict__ H, T scale, T dmin, T dmax,
                                                                   T* __restrict__ Hinv, long long n) {
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T A[3][3], Ai[3][3];
    sym3_unpack(H + i * 6, A);
#pragma unroll
    for (int k = 0; k < 3; ++k) { const T d = A[k][k]; A[k][k] = (d < dmin ? dmin : (d > dmax ? dmax : d)) * scale; }
    spd_inverse<T, 3>(A, Ai);
    T* o = Hinv + i * 6;
    o[0] = Ai[0][0]; o[1] = Ai[0][1]; o[2] = Ai[0][2]; o[3] = Ai[1][1]; o[4] = Ai[1][2]; o[5] = Ai[2][2];
  }
}
// out = alpha * A t for packed 3x3 blocks
template <typename T>
__global__ void __launch_bounds__(kLmThreads) pt3_apply_kernel(const T* __restrict__ A6, const T* __restrict__ t, T alpha,
                                                                T* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T A[3][3];
    sym3_unpack(A6 + i * 6, A);
    const T a = t[i * 3], b = t[i * 3 + 1], c = t[i * 3 + 2];
#pragma unroll
    for (int k = 0; k < 3; ++k) out[i * 3 + k] = alpha * (A[k][0] * a + A[k][1] * b + A[k][2] * c);
  }
}

// ---- CG vector kernels -------------------------------------------------------------------------------------------
// W: unknowns per block row (6: pose tangents, the default; 9: BAL cameras, bal.cu).
template <typename T, int W = 6>
__global__ void __launch_bounds__(kLmThreads) cg_init_kernel(const T* __restrict__ Minv, const T* __restrict__ b, T sign,
                                             const T* __restrict__ D, int dmode, T* __restrict__ x,
                                             T* __restrict__ r, T* __restrict__ p, T* __restrict__ q,
                                             double* cg, double* ws, double tol, double maxiter, long long n) {
  constexpr int NP = packed_words<W>();
  double acc[2] = {0.0, 0.0};
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T rv[W], z[W], qv[W], zero[W];
#pragma unroll
    for (int k = 0; k < W; ++k) zero[k] = T(0);
    ldw<T, W>(b, i, rv);
#pragma unroll
    for (int k = 0; k < W; ++k) rv[k] *= sign;
    symw_mv_packed<T, W>(Minv + i * NP, rv, z);
    apply_D<T, W>(D, dmode, i, z, qv);
    stw<T, W>(x, i, zero); stw<T, W>(r, i, rv); stw<T, W>(p, i, z); stw<T, W>(q, i, qv);
#pragma unroll
    for (int k = 0; k < W; ++k) { acc[0] += (double)rv[k] * (double)z[k]; acc[1] += (double)rv[k] * (double)rv[k]; }
  }
  if (reduce_sums<2>(acc, ws)) {
    const double rz = ws[0], rr = ws[1];
    cg[CG_RZ0] = rz; cg[CG_RZ1] = 0.0; cg[CG_PQ] = 0.0; cg[CG_RR] = rr; cg[CG_STOP2] = tol * tol * rr;
    cg[CG_ITERS] = 0.0; cg[CG_MAXIT] = maxiter;
    cg[CG_BEST] = rr; cg[CG_SINCE] = 0.0; cg[CG_SAVE] = 1.0;       // x = 0 is the first best
    // exact CG ends within (number of unknowns) iterations: no new minimum of |r| for that long is stagnation, not a plateau
    cg[CG_PATIENCE] = fmax(kCgPatience, (double)W * (double)n);
    cg[CG_DONE] = (!(rr > tol * tol * rr) || maxiter <= 0.0) ? 1.0 : 0.0;      // |r| <= tol |b| (also NaN) -> nothing to do
  }
}
template <typename T, int W = 6>
__global__ void __launch_bounds__(kLmThreads) cg_dot_kernel(const T* __restrict__ p, const T* __restrict__ q, double* cg, double* ws,
                                            long long n) {
  if (cg[CG_DONE] != 0.0) return;
  double acc[1] = {0.0};
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
#pragma unroll
    for (int k = 0; k < W; ++k) acc[0] += (double)p[i * W + k] * (double)q[i * W + k];
  }
  if (reduce_sums<1>(acc, ws)) cg[CG_PQ] = ws[0];
}
template <typename T, int W = 6>
__global__ void __launch_bounds__(kLmThreads) cg_update_kernel(const T* __restrict__ Minv, const T* __restrict__ p,
                                               const T* __restrict__ q, T* __restrict__ x, T* __restrict__ r,
                                               T* __restrict__ z, T* __restrict__ xbest, double* cg, double* ws, int par,
                                               long long n) {
  constexpr int NP = packed_words<W>();
  if (cg[CG_DONE] != 0.0) return;
  const bool save = cg[CG_SAVE] != 0.0;      // the iterate entering this update is the best so far: keep a copy
  const double pq = cg[CG_PQ];
  if (!(pq > 0.0)) {                       // breakdown (operator not positive definite along p): stop with the current x
    if (blockIdx.x == 0 && threadIdx.x == 0) cg[CG_DONE] = 2.0;
    return;
  }
  const T alpha = (T)(cg[par] / pq);
  double acc[2] = {0.0, 0.0};
  // The NP-word preconditioner blocks of a warp's 32 consecutive nodes are contiguous (2688 bytes for fp32 6x6 blocks):
  // the warp copies them with NP coalesced loads into shared memory (one wavefront each) and every lane reads its block
  // from there (stride NP words, odd: conflict-free) — read per lane straight from global memory, each of the NP load
  // instructions touched NP lines.
  __shared__ T sM[kLmThreads / 32][32 * NP];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long base = (long long)blockIdx.x * kLmThreads + warp * 32; base < n; base += (long long)gridDim.x * kLmThreads) {
    const long long i = base + lane;
    const int words = (int)(n - base < 32 ? n - base : 32) * NP;
    __syncwarp();
    for (int w = lane; w < words; w += 32) sM[warp][w] = Minv[base * NP + w];
    __syncwarp();
    if (i >= n) continue;
    T pv[W], qv[W], xv[W], rv[W], zv[W];
    ldw<T, W>(p, i, pv); ldw<T, W>(q, i, qv); ldw<T, W>(x, i, xv); ldw<T, W>(r, i, rv);
    if (save) stw<T, W>(xbest, i, xv);
#pragma unroll
    for (int k = 0; k < W; ++k) { xv[k] += alpha * pv[k]; rv[k] -= alpha * qv[k]; }
    symw_mv_packed<T, W>(&sM[warp][lane * NP], rv, zv);
    stw<T, W>(x, i, xv); stw<T, W>(r, i, rv); stw<T, W>(z, i, zv);
#pragma unroll
    for (int k = 0; k < W; ++k) { acc[0] += (double)rv[k] * (double)zv[k]; acc[1] += (double)rv[k] * (double)rv[k]; }
  }
  if (reduce_sums<2>(acc, ws)) {       // thread 0 of the last CTA: every CTA has read the state it needs by now
    cg[par ^ 1] = ws[0];
    cg[CG_RR] = ws[1];
    const double it = cg[CG_ITERS] + 1.0;
    cg[CG_ITERS] = it;
    cg_after_update(cg, ws[1], it);
  }
}
template <typename T, int W = 6>
__global__ void __launch_bounds__(kLmThreads) cg_dir_kernel(const T* __restrict__ z, const T* __restrict__ D, int dmode, T* __restrict__ p,
                                            T* __restrict__ q, const double* cg, int par, long long n) {
  if (cg[CG_DONE] != 0.0) return;
  const T beta = (T)(cg[par ^ 1] / cg[par]);
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T pv[W], zv[W], qv[W];
    ldw<T, W>(p, i, pv); ldw<T, W>(z, i, zv);
#pragma unroll
    for (int k = 0; k < W; ++k) pv[k] = zv[k] + beta * pv[k];
    apply_D<T, W>(D, dmode, i, pv, qv);
    stw<T, W>(p, i, pv); stw<T, W>(q, i, qv);
  }
}

// x <- xbest unless the solve converged or the last iterate is the best one (see the state enum)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) cg_finish_kernel(T* __restrict__ x, const T* __restrict__ xbest,
                                                                const double* cg, long long n6) {
  if (cg[CG_DONE] == 1.0 || cg[CG_SAVE] != 0.0) return;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n6; i += (long long)gridDim.x * kLmThreads)
    x[i] = xbest[i];
}

// dot + update + dir of one iteration in ONE single-CTA launch, for systems small enough that a grid is only latency
// (bundle adjustment: a few thousand cameras; the three separate kernels cost ~28 us at 1e3 rows, this one ~8 us).
// Fixed-order block reductions (warp shuffles, then warp 0 over the 32 warp partials): deterministic.
constexpr long long kVecSmallRows = 4096;
template <int NS, int THREADS> __device__ __forceinline__ void block_sums(double (&v)[NS], double (*sh)[NS], double (&out)[NS]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NS; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < NS; ++k) sh[warp][k] = v[k];
  __syncthreads();
  if (warp == 0) {
    double t[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) {
      t[k] = lane < THREADS / 32 ? sh[lane][k] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t[k] += __shfl_xor_sync(0xffffffffu, t[k], o);
    }
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < NS; ++k) sh[0][k] = t[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NS; ++k) out[k] = sh[0][k];
  __syncthreads();
}
template <typename T, int THREADS, int W = 6>
__global__ void __launch_bounds__(THREADS) cg_vec_small_kernel(const T* __restrict__ Minv, const T* __restrict__ D, int dmode,
                                                  T* __restrict__ x, T* __restrict__ r, T* __restrict__ z,
                                                  T* __restrict__ p, T* __restrict__ q, T* __restrict__ xbest, double* cg,
                                                  int par, long long n) {
  constexpr int NP = packed_words<W>();
  __shared__ double sh[32][2];
  __shared__ double done_sh;
  if (cg[CG_DONE] != 0.0) return;
  const double rz_old = cg[par], it = cg[CG_ITERS] + 1.0;
  const bool save = cg[CG_SAVE] != 0.0;
  double a1[2] = {0.0, 0.0}, s1[2];
  for (long long i = threadIdx.x; i < n; i += THREADS)
#pragma unroll
    for (int k = 0; k < W; ++k) a1[0] += (double)p[i * W + k] * (double)q[i * W + k];
  block_sums<2, THREADS>(a1, sh, s1);
  const double pq = s1[0];
  if (!(pq > 0.0)) {                       // breakdown: stop with the current x
    if (threadIdx.x == 0) cg[CG_DONE] = 2.0;
    return;
  }
  const T alpha = (T)(rz_old / pq);
  double a2[2] = {0.0, 0.0}, s2[2];
  for (long long i = threadIdx.x; i < n; i += THREADS) {
    T pv[W], qv[W], xv[W], rv[W], zv[W];
    ldw<T, W>(p, i, pv); ldw<T, W>(q, i, qv); ldw<T, W>(x, i, xv); ldw<T, W>(r, i, rv);
    if (save) stw<T, W>(xbest, i, xv);
#pragma unroll
    for (int k = 0; k < W; ++k) { xv[k] += alpha * pv[k]; rv[k] -= alpha * qv[k]; }
    symw_mv_packed<T, W>(Minv + i * NP, rv, zv);
    stw<T, W>(x, i, xv); stw<T, W>(r, i, rv); stw<T, W>(z, i, zv);
#pragma unroll
    for (int k = 0; k < W; ++k) { a2[0] += (double)rv[k] * (double)zv[k]; a2[1] += (double)rv[k] * (double)rv[k]; }
  }
  block_sums<2, THREADS>(a2, sh, s2);
  if (threadIdx.x == 0) {
    cg[CG_PQ] = pq; cg[par ^ 1] = s2[0]; cg[CG_RR] = s2[1]; cg[CG_ITERS] = it;
    cg_after_update(cg, s2[1], it);
    done_sh = cg[CG_DONE];
  }
  __syncthreads();
  if (done_sh != 0.0) return;
  const T beta = (T)(s2[0] / rz_old);
  for (long long i = threadIdx.x; i < n; i += THREADS) {     // the same thread wrote z[i] above
    T pv[W], zv[W], qv[W];
    ldw<T, W>(p, i, pv); ldw<T, W>(z, i, zv);
#pragma unroll
    for (int k = 0; k < W; ++k) pv[k] = zv[k] + beta * pv[k];
    apply_D<T, W>(D, dmode, i, pv, qv);
    stw<T, W>(p, i, pv); stw<T, W>(q, i, qv);
  }
}

template <typename T>
static void launch_cg_vec_small(const T* Minv, const T* D, int dmode, T* x, T* r, T* z, T* p, T* q, T* xbest, double* cg,
                                int par, long long n, cudaStream_t st) {
  const int th = n <= 2048 ? 256 : (n <= 3072 ? 512 : 1024);     // measured: 256 beats 1024 at 1e3 rows
  if (th == 256) cg_vec_small_kernel<T, 256><<<1, 256, 0, st>>>(Minv, D, dmode, x, r, z, p, q, xbest, cg, par, n);
  else if (th == 512) cg_vec_small_kernel<T, 512><<<1, 512, 0, st>>>(Minv, D, dmode, x, r, z, p, q, xbest, cg, par, n);
  else cg_vec_small_kernel<T, 1024><<<1, 1024, 0, st>>>(Minv, D, dmode, x, r, z, p, q, xbest, cg, par, n);
}

}  // namespace b200pose
