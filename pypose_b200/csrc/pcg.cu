// pcg.cu — device-resident block-Jacobi preconditioned conjugate gradients for the block-sparse LM routes
// (C-ABI: include/b200pose.h, section LM; reference algorithm: pypose/optim/solver.py:276-340 PCG/CG, and the
// `bae` PCG the sparse branch delegates to, solver.py:343-363 / optimizer.py:629-643).
//
// The vectors are (n,6) block rows (one SE3 tangent per pose / camera).  Every scalar of the iteration (r.z, p.Ap,
// |r|^2, the stop threshold, the iteration counter and the "done" flag) lives in a small fp64 state array on the
// device, so a whole chunk of iterations is enqueued by ONE host call without any synchronisation; once the flag is
// set all remaining kernels of the chunk return immediately.  Per iteration: operator kernel(s) + 3 vector kernels
//   dot     pq = p.q
//   update  alpha = rz/pq; x += alpha p; r -= alpha q; z = Minv r; rz' = r.z; rr = r.r; converged / maxiter -> done
//   dir     beta = rz'/rz; p = z + beta p; q = D p          (D: the block-diagonal part of the operator)
// Reductions are the deterministic last-block fp64 folds of lm_common.cuh.
#include "lm_common.cuh"
#include "comm.cuh"

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
// q = D p with D none (0), diagonal (n,6) (1) or packed symmetric blocks (n,21) (2)
template <typename T> __device__ __forceinline__ void apply_D(const T* D, int dmode, long long i, const T (&p)[6], T (&q)[6]) {
  if (dmode == 2) {
    sym6_mv_packed(D + i * 21, p, q);
  } else {
#pragma unroll
    for (int k = 0; k < 6; ++k) q[k] = dmode == 1 ? D[i * 6 + k] * p[k] : T(0);
  }
}

// diag <- clamp(diag, dmin, dmax) * scale (optimizer.py:657 + cumulative :666); optional outputs: the damped block,
// the amount added to the diagonal, the inverse of the damped block.
template <typename T>
__global__ void __launch_bounds__(kLmThreads) blk6_damp_inv_kernel(const T* __restrict__ H, T scale, T dmin, T dmax,
                                                                    T* __restrict__ Hd, T* __restrict__ extra,
                                                                    T* __restrict__ Minv, long long n) {
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T A[6][6], Ai[6][6];
    sym6_unpack(H + i * 21, A);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const T d = A[k][k];
      const T c = (d < dmin ? dmin : (d > dmax ? dmax : d)) * scale;
      if (extra) extra[i * 6 + k] = c - d;
      A[k][k] = c;
    }
    if (Hd) sym6_pack(A, Hd + i * 21);
    if (Minv) { spd_inverse<T, 6>(A, Ai); sym6_pack(Ai, Minv + i * 21); }
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
template <typename T>
__global__ void __launch_bounds__(kLmThreads) cg_init_kernel(const T* __restrict__ Minv, const T* __restrict__ b, T sign,
                                                              const T* __restrict__ D, int dmode, T* __restrict__ x,
                                                              T* __restrict__ r, T* __restrict__ p, T* __restrict__ q,
                                                              double* cg, double* ws, double tol, double maxiter,
                                                              long long n) {
  double acc[2] = {0.0, 0.0};
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T rv[6], z[6], qv[6], zero[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
    ld6(b, i, rv);
#pragma unroll
    for (int k = 0; k < 6; ++k) rv[k] *= sign;
    sym6_mv_packed(Minv + i * 21, rv, z);
    apply_D(D, dmode, i, z, qv);
    st6(x, i, zero); st6(r, i, rv); st6(p, i, z); st6(q, i, qv);
#pragma unroll
    for (int k = 0; k < 6; ++k) { acc[0] += (double)rv[k] * (double)z[k]; acc[1] += (double)rv[k] * (double)rv[k]; }
  }
  if (reduce_sums<2>(acc, ws)) {
    const double rz = ws[0], rr = ws[1];
    cg[CG_RZ0] = rz; cg[CG_RZ1] = 0.0; cg[CG_PQ] = 0.0; cg[CG_RR] = rr; cg[CG_STOP2] = tol * tol * rr;
    cg[CG_ITERS] = 0.0; cg[CG_MAXIT] = maxiter;
    cg[CG_BEST] = rr; cg[CG_SINCE] = 0.0; cg[CG_SAVE] = 1.0;       // x = 0 is the first best
    // exact CG ends within (number of unknowns) iterations: no new minimum of |r| for that long is stagnation, not a plateau
    cg[CG_PATIENCE] = fmax(kCgPatience, 6.0 * (double)n);
    cg[CG_DONE] = (!(rr > tol * tol * rr) || maxiter <= 0.0) ? 1.0 : 0.0;      // |r| <= tol |b| (also NaN) -> nothing to do
  }
}
template <typename T>
__global__ void __launch_bounds__(kLmThreads) cg_dot_kernel(const T* __restrict__ p, const T* __restrict__ q, double* cg,
                                                             double* ws, long long n) {
  if (cg[CG_DONE] != 0.0) return;
  double acc[1] = {0.0};
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
#pragma unroll
    for (int k = 0; k < 6; ++k) acc[0] += (double)p[i * 6 + k] * (double)q[i * 6 + k];
  }
  if (reduce_sums<1>(acc, ws)) cg[CG_PQ] = ws[0];
}
template <typename T>
__global__ void __launch_bounds__(kLmThreads) cg_update_kernel(const T* __restrict__ Minv, const T* __restrict__ p,
                                                                const T* __restrict__ q, T* __restrict__ x,
                                                                T* __restrict__ r, T* __restrict__ z,
                                                                T* __restrict__ xbest, double* cg,
                                                                double* ws, int par, long long n) {
  if (cg[CG_DONE] != 0.0) return;
  const bool save = cg[CG_SAVE] != 0.0;      // the iterate entering this update is the best so far: keep a copy
  const double pq = cg[CG_PQ];
  if (!(pq > 0.0)) {                       // breakdown (operator not positive definite along p): stop with the current x
    if (blockIdx.x == 0 && threadIdx.x == 0) cg[CG_DONE] = 2.0;
    return;
  }
  const T alpha = (T)(cg[par] / pq);
  double acc[2] = {0.0, 0.0};
  // The 21-word preconditioner blocks of a warp's 32 consecutive nodes are 2688 contiguous bytes: the warp copies them
  // with 21 coalesced loads into shared memory (one wavefront each) and every lane reads its block from there (stride 21
  // words: conflict-free) — read per lane straight from global memory, each of the 21 load instructions touched 21 lines.
  __shared__ T sM[kLmThreads / 32][32 * 21];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long base = (long long)blockIdx.x * kLmThreads + warp * 32; base < n; base += (long long)gridDim.x * kLmThreads) {
    const long long i = base + lane;
    const int words = (int)(n - base < 32 ? n - base : 32) * 21;
    __syncwarp();
    for (int w = lane; w < words; w += 32) sM[warp][w] = Minv[base * 21 + w];
    __syncwarp();
    if (i >= n) continue;
    T pv[6], qv[6], xv[6], rv[6], zv[6];
    ld6(p, i, pv); ld6(q, i, qv); ld6(x, i, xv); ld6(r, i, rv);
    if (save) st6(xbest, i, xv);
#pragma unroll
    for (int k = 0; k < 6; ++k) { xv[k] += alpha * pv[k]; rv[k] -= alpha * qv[k]; }
    sym6_mv_packed(&sM[warp][lane * 21], rv, zv);
    st6(x, i, xv); st6(r, i, rv); st6(z, i, zv);
#pragma unroll
    for (int k = 0; k < 6; ++k) { acc[0] += (double)rv[k] * (double)zv[k]; acc[1] += (double)rv[k] * (double)rv[k]; }
  }
  if (reduce_sums<2>(acc, ws)) {       // thread 0 of the last CTA: every CTA has read the state it needs by now
    cg[par ^ 1] = ws[0];
    cg[CG_RR] = ws[1];
    const double it = cg[CG_ITERS] + 1.0;
    cg[CG_ITERS] = it;
    cg_after_update(cg, ws[1], it);
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
template <typename T>
__global__ void __launch_bounds__(kLmThreads) cg_dir_kernel(const T* __restrict__ z, const T* __restrict__ D, int dmode,
                                                             T* __restrict__ p, T* __restrict__ q, const double* cg, int par,
                                                             long long n) {
  if (cg[CG_DONE] != 0.0) return;
  const T beta = (T)(cg[par ^ 1] / cg[par]);
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T pv[6], zv[6], qv[6];
    ld6(p, i, pv); ld6(z, i, zv);
#pragma unroll
    for (int k = 0; k < 6; ++k) pv[k] = zv[k] + beta * pv[k];
    apply_D(D, dmode, i, pv, qv);
    st6(p, i, pv); st6(q, i, qv);
  }
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
template <typename T, int THREADS>
__global__ void __launch_bounds__(THREADS) cg_vec_small_kernel(const T* __restrict__ Minv, const T* __restrict__ D, int dmode,
                                                                    T* __restrict__ x, T* __restrict__ r, T* __restrict__ z,
                                                                    T* __restrict__ p, T* __restrict__ q,
                                                                    T* __restrict__ xbest, double* cg, int par,
                                                                    long long n) {
  __shared__ double sh[32][2];
  __shared__ double done_sh;
  if (cg[CG_DONE] != 0.0) return;
  const double rz_old = cg[par], it = cg[CG_ITERS] + 1.0;
  const bool save = cg[CG_SAVE] != 0.0;
  double a1[2] = {0.0, 0.0}, s1[2];
  for (long long i = threadIdx.x; i < n; i += THREADS)
#pragma unroll
    for (int k = 0; k < 6; ++k) a1[0] += (double)p[i * 6 + k] * (double)q[i * 6 + k];
  block_sums<2, THREADS>(a1, sh, s1);
  const double pq = s1[0];
  if (!(pq > 0.0)) {                       // breakdown: stop with the current x
    if (threadIdx.x == 0) cg[CG_DONE] = 2.0;
    return;
  }
  const T alpha = (T)(rz_old / pq);
  double a2[2] = {0.0, 0.0}, s2[2];
  for (long long i = threadIdx.x; i < n; i += THREADS) {
    T pv[6], qv[6], xv[6], rv[6], zv[6];
    ld6(p, i, pv); ld6(q, i, qv); ld6(x, i, xv); ld6(r, i, rv);
    if (save) st6(xbest, i, xv);
#pragma unroll
    for (int k = 0; k < 6; ++k) { xv[k] += alpha * pv[k]; rv[k] -= alpha * qv[k]; }
    sym6_mv_packed(Minv + i * 21, rv, zv);
    st6(x, i, xv); st6(r, i, rv); st6(z, i, zv);
#pragma unroll
    for (int k = 0; k < 6; ++k) { a2[0] += (double)rv[k] * (double)zv[k]; a2[1] += (double)rv[k] * (double)rv[k]; }
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
    T pv[6], zv[6], qv[6];
    ld6(p, i, pv); ld6(z, i, zv);
#pragma unroll
    for (int k = 0; k < 6; ++k) pv[k] = zv[k] + beta * pv[k];
    apply_D(D, dmode, i, pv, qv);
    st6(p, i, pv); st6(q, i, qv);
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

// ---- operators (ObsRows / obs_rows: lm_common.cuh) -----------------------------------------------------------------
// pose graph: q += H p edge by edge (lm.cu lm_pgo_spmv_kernel), skipped once the CG has finished
template <typename T>
__global__ void __launch_bounds__(kLmThreads) pcg_pgo_spmv_kernel(const T* __restrict__ M, const int* __restrict__ ei,
                                                                   const int* __restrict__ ej, const T* __restrict__ x,
                                                                   T* __restrict__ y, const double* cg, long long E) {
  if (cg[CG_DONE] != 0.0) return;
  for (long long e = (long long)blockIdx.x * kLmThreads + threadIdx.x; e < E; e += (long long)gridDim.x * kLmThreads) {
    const long long i = ei[e], j = ej[e];
    T d[6], v[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) d[k] = __ldg(x + i * 6 + k) - __ldg(x + j * 6 + k);
    sym6_mv_packed(M + e * 21, d, v);
#pragma unroll
    for (int k = 0; k < 6; ++k) { atomicAdd(y + i * 6 + k, v[k]); atomicAdd(y + j * 6 + k, -v[k]); }
  }
}
// u[j] = alpha * Hp^-1_j (t0[j] + sum_{k in obs(j)} Jp_k^T Jc_k x[c_k])   — W^T x by GATHER over a point-ordered copy
// of the per-observation data (Y4p, cidx_p; pptr = offsets per point), so there are no atomics, no zero-fill of
// a (P,3) buffer, the result is deterministic, and the 3x3 point-block inverse is applied while the sum is in registers.
// With t0 = gp, alpha = -1 and x = dc this is the back-substitution dp = -Hpp^-1 (gp + W^T dc).
// LPP lanes cooperate on one point (a point has ~2-20 observations; one thread per point was latency-bound on the
// dependent padj -> cidx/Y4 -> pose/x gathers: 28 us at 1e6 observations, this form: see DESIGN.md).
constexpr int kLanesPerPoint = 8;
template <typename T>
__global__ void __launch_bounds__(kLmThreads) pcg_ba_wtx_gather_kernel(const T* __restrict__ Y4p, const T* __restrict__ poses,
                                                                        const int* __restrict__ cidx_p,
                                                                        const int* __restrict__ pptr, const T* __restrict__ Hpinv,
                                                                        const T* __restrict__ x, const T* __restrict__ t0, T alpha,
                                                                        T* __restrict__ u, const double* cg, long long P) {
  if (cg && cg[CG_DONE] != 0.0) return;
  constexpr int LPP = kLanesPerPoint, PPB = kLmThreads / LPP;           // points per CTA and sweep
  const int sub = threadIdx.x % LPP;
  // warp-uniform trip count (the shuffles below need all 32 lanes): iterate over groups of PPB points
  const long long groups = (P + PPB - 1) / PPB;
  for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
    const long long j = g * PPB + threadIdx.x / LPP;
    T t[3] = {T(0), T(0), T(0)};
    if (j < P) {
      const int lo = pptr[j], hi = pptr[j + 1];
      for (int s = lo + sub; s < hi; s += LPP) {        // Y4p / cidx_p are stored in point order: coalesced
        const long long c = cidx_p[s];
        ObsRows<T> R;
        obs_rows(Y4p, poses, s, c, R);
        T v0 = T(0), v1 = T(0);
#pragma unroll
        for (int a = 0; a < 6; ++a) { const T xa = __ldg(x + c * 6 + a); v0 += R.jc0[a] * xa; v1 += R.jc1[a] * xa; }
#pragma unroll
        for (int a = 0; a < 3; ++a) t[a] += R.jp0[a] * v0 + R.jp1[a] * v1;
      }
    }
#pragma unroll
    for (int o = LPP / 2; o > 0; o >>= 1)
#pragma unroll
      for (int a = 0; a < 3; ++a) t[a] += __shfl_xor_sync(0xffffffffu, t[a], o);      // stays inside the LPP-lane group
    if (j < P && sub == 0) {
      if (t0) { t[0] += t0[j * 3]; t[1] += t0[j * 3 + 1]; t[2] += t0[j * 3 + 2]; }
      T A[3][3];
      sym3_unpack(Hpinv + j * 6, A);
#pragma unroll
      for (int a = 0; a < 3; ++a) u[j * 3 + a] = alpha * (A[a][0] * t[0] + A[a][1] * t[1] + A[a][2] * t[2]);
    }
  }
}
// ws[0] = sum_k (J_k d)^T (2 r_k + J_k d) with J_k d = Jc x_c + Jp x_p    (strategy.py:143 'predicted')
template <typename T>
__global__ void __launch_bounds__(kLmThreads) ba_predicted_kernel(const T* __restrict__ Y4, const T* __restrict__ poses,
                                                                   const T* __restrict__ rs, const int* __restrict__ cidx,
                                                                   const int* __restrict__ pidx, const T* __restrict__ xc,
                                                                   const T* __restrict__ xp, double* ws, long long m) {
  double acc[1] = {0.0};
  for (long long k = (long long)blockIdx.x * kLmThreads + threadIdx.x; k < m; k += (long long)gridDim.x * kLmThreads) {
    const long long c = cidx[k], j = pidx[k];
    ObsRows<T> R;
    obs_rows(Y4, poses, k, c, R);
    T d0 = T(0), d1 = T(0);
#pragma unroll
    for (int a = 0; a < 6; ++a) { const T v = __ldg(xc + c * 6 + a); d0 += R.jc0[a] * v; d1 += R.jc1[a] * v; }
#pragma unroll
    for (int a = 0; a < 3; ++a) { const T v = __ldg(xp + j * 3 + a); d0 += R.jp0[a] * v; d1 += R.jp1[a] * v; }
    acc[0] += (double)(d0 * (T(2) * rs[k * 2] + d0) + d1 * (T(2) * rs[k * 2 + 1] + d1));
  }
  reduce_sums<1>(acc, ws);
}
// ws[0] = D^T H D + 2 D^T g for the pose graph: sum over edges of d^T M_e d (d = D_i - D_j) plus the linear term
template <typename T>
__global__ void __launch_bounds__(kLmThreads) pgo_predicted_kernel(const T* __restrict__ M, const int* __restrict__ ei,
                                                                    const int* __restrict__ ej, const T* __restrict__ D,
                                                                    const T* __restrict__ g, double* ws, long long E,
                                                                    long long n) {
  double acc[1] = {0.0};
  const long long tid = (long long)blockIdx.x * kLmThreads + threadIdx.x, nth = (long long)gridDim.x * kLmThreads;
  for (long long e = tid; e < E; e += nth) {
    const long long i = ei[e], j = ej[e];
    T d[6], v[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) d[k] = __ldg(D + i * 6 + k) - __ldg(D + j * 6 + k);
    sym6_mv_packed(M + e * 21, d, v);
    T s = T(0);
#pragma unroll
    for (int k = 0; k < 6; ++k) s += d[k] * v[k];
    acc[0] += (double)s;
  }
  for (long long i = tid; i < n; i += nth) {
    T s = T(0);
#pragma unroll
    for (int k = 0; k < 6; ++k) s += D[i * 6 + k] * g[i * 6 + k];
    acc[0] += 2.0 * (double)s;
  }
  reduce_sums<1>(acc, ws);
}

// ws[0] = sum_e d^T M0_e d + 2 d^T u0_e, d = D_j - D_i: the same quantity from per-edge blocks (used when M0 / u0 differ
// from the blocks of the solve, i.e. with information-matrix weights)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) pgo_predicted_edge_kernel(const T* __restrict__ M0, const T* __restrict__ u0,
                                                                         const int* __restrict__ ei, const int* __restrict__ ej,
                                                                         const T* __restrict__ D, double* ws, long long E) {
  double acc[1] = {0.0};
  for (long long e = (long long)blockIdx.x * kLmThreads + threadIdx.x; e < E; e += (long long)gridDim.x * kLmThreads) {
    const long long i = ei[e], j = ej[e];
    T d[6], v[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) d[k] = __ldg(D + j * 6 + k) - __ldg(D + i * 6 + k);
    sym6_mv_packed(M0 + e * 21, d, v);
    T s = T(0);
#pragma unroll
    for (int k = 0; k < 6; ++k) s += d[k] * (v[k] + T(2) * u0[e * 6 + k]);
    acc[0] += (double)s;
  }
  reduce_sums<1>(acc, ws);
}

// used by pcg2.cu (node-ordered two-kernel iteration): x = 0, r = -b, z = M^-1 r (stored through the `p` slot), state reset
template <typename T>
void pcg_launch_init(const T* Minv, const T* b, T* x, T* r, T* z, T* q, double* cg, double* ws, double tol, double maxiter,
                     long long n, cudaStream_t st) {
  cg_init_kernel<T><<<lm_grid(n, kLmThreads), kLmThreads, 0, st>>>(Minv, b, (T)-1, (const T*)nullptr, 0, x, r, z, q, cg, ws, tol,
                                                                  maxiter, n);
}
template <typename T>
void pcg_launch_update(const T* Minv, const T* p, const T* q, T* x, T* r, T* z, T* xbest, double* cg, double* ws, int par,
                       long long n, cudaStream_t st) {
  cg_update_kernel<T><<<lm_grid(n, kLmThreads), kLmThreads, 0, st>>>(Minv, p, q, x, r, z, xbest, cg, ws, par, n);
}
template void pcg_launch_init<float>(const float*, const float*, float*, float*, float*, float*, double*, double*, double, double,
                                     long long, cudaStream_t);
template void pcg_launch_init<double>(const double*, const double*, double*, double*, double*, double*, double*, double*, double,
                                      double, long long, cudaStream_t);
template void pcg_launch_update<float>(const float*, const float*, const float*, float*, float*, float*, float*, double*, double*,
                                       int, long long, cudaStream_t);
template void pcg_launch_update<double>(const double*, const double*, const double*, double*, double*, double*, double*, double*,
                                        double*, int, long long, cudaStream_t);

}  // namespace b200pose

using namespace b200pose;

#define LM_LAUNCH(kern, work, st, ...) kern<<<lm_grid(work, kLmThreads), kLmThreads, 0, (cudaStream_t)(st)>>>(__VA_ARGS__)

// One chunk of PCG iterations for the pose graph on per-edge blocks (A = M, ia/ib = ei/ej, E edges): the operator walks the
// edges and scatter-adds.  Single GPU uses pcg2.cu (node-ordered gathers) by default; this is the multi-GPU operator (every
// rank holds a shard of the edges and the partial products are all-reduced on the device) and the A/B baseline.
// Multi-GPU: edges / observations are sharded, the CG vectors are replicated.  Every operator product is a partial sum that
// is all-reduced ON THE DEVICE (comm.cu: scatter to slice owners, reduce in rank order, broadcast) between the operator
// and the vector kernels of the iteration — no host in the loop, no collective library call.  The block-diagonal part
// D p of the operator is added by rank 0 only (dmode 0 elsewhere) so that the reduction counts it once.
struct PcgComm {
  bool on;
  Peers P;
  long long stage, result;
  unsigned long long epoch;       // epochs epoch+1, epoch+2, ... are consumed, one per all-reduce, in enqueue order
  unsigned* tickets;
};
static PcgComm make_pcg_comm(const unsigned long long* bases, int rank, int world, long long stage, long long result,
                             long long epoch, unsigned* tickets) {
  PcgComm c;
  c.on = bases != nullptr && world > 1;
  for (int r = 0; r < kMaxRanks; ++r) c.P.base[r] = (c.on && r < world) ? reinterpret_cast<char*>(bases[r]) : nullptr;
  c.P.rank = rank; c.P.world = world;
  c.stage = stage; c.result = result; c.epoch = (unsigned long long)epoch; c.tickets = tickets;
  return c;
}
constexpr int kPcgChannel = 6;

template <typename CT>
static int pgo_pcg_run(const CT* A, const int* ia, const int* ib, long long E, const CT* Minv, const CT* extra, const CT* g,
                       CT* x, CT* r, CT* z, CT* p, CT* q, CT* xbest, double* cg, double* ws, double tol, long long maxiter,
                       long long first_iter, long long iters, long long n, cudaStream_t stream, PcgComm cm) {
  if (n <= 0) return 0;
  const int dmode = (!cm.on || cm.P.rank == 0) ? 1 : 0;
  if (first_iter == 0)
    LM_LAUNCH(cg_init_kernel<CT>, n, stream, Minv, g, (CT)-1, extra, dmode, x, r, p, q, cg, ws, tol, (double)maxiter, n);
  for (long long it = first_iter; it < first_iter + iters; ++it) {
    const int par = (int)(it & 1);
    if (E > 0) LM_LAUNCH(pcg_pgo_spmv_kernel<CT>, E, stream, A, ia, ib, p, q, cg, E);
    if (cm.on)
      comm_allreduce_launch<CT>(q, q, n * 6, cm.P, cm.stage, cm.result, kPcgChannel, ++cm.epoch, cm.tickets, cg, stream);
    if (n <= kVecSmallRows) {
      launch_cg_vec_small<CT>(Minv, extra, dmode, x, r, z, p, q, xbest, cg, par, n, stream);
      continue;
    }
    LM_LAUNCH(cg_dot_kernel<CT>, n, stream, p, q, cg, ws, n);
    LM_LAUNCH(cg_update_kernel<CT>, n, stream, Minv, p, q, x, r, z, xbest, cg, ws, par, n);
    LM_LAUNCH(cg_dir_kernel<CT>, n, stream, z, extra, dmode, p, q, cg, par, n);
  }
  return (int)cudaGetLastError();
}
template <typename CT>
static int ba_pcg_run(const CT* Y4, const CT* poses, const int* pidx, const int* cseg, long long split, long long tpi,
                      long long m, const CT* Y4p, const int* cidx_p, const int* pptr, const CT* Hc, const CT* Hpinv,
                      const CT* Minv, const CT* bneg, CT* x, CT* r, CT* z, CT* p, CT* q, CT* t, CT* part, CT* xbest,
                      double* cg, double* ws, double tol, long long maxiter,
                      long long P, long long first_iter, long long iters, long long n, cudaStream_t stream, PcgComm cm) {
  if (n <= 0) return 0;
  const int dmode = (!cm.on || cm.P.rank == 0) ? 2 : 0;
  if (first_iter == 0)
    LM_LAUNCH(cg_init_kernel<CT>, n, stream, Minv, bneg, (CT)-1, Hc, dmode, x, r, p, q, cg, ws, tol, (double)maxiter, n);
  for (long long it = first_iter; it < first_iter + iters; ++it) {
    const int par = (int)(it & 1);
    if (cm.on || m > 0) {         // a rank without observations still takes part in both all-reduces
      // t = Hpp^-1 W^T p: Hpp^-1 is replicated and linear, so the partial sums over this rank's observations are reduced
      LM_LAUNCH(pcg_ba_wtx_gather_kernel<CT>, P * kLanesPerPoint, stream, Y4p, poses, cidx_p, pptr, Hpinv, p,
                (const CT*)nullptr, (CT)1, t, cg, P);
      if (cm.on)
        comm_allreduce_launch<CT>(t, t, P * 3, cm.P, cm.stage, cm.result, kPcgChannel, ++cm.epoch, cm.tickets, cg, stream);
      ba_wv_seg_launch<CT>(Y4, poses, pidx, cseg, (int)split, (int)tpi, (const CT*)nullptr, t, q, part, cg, n, stream);
      if (cm.on)
        comm_allreduce_launch<CT>(q, q, n * 6, cm.P, cm.stage, cm.result, kPcgChannel, ++cm.epoch, cm.tickets, cg, stream);
    }
    if (n <= kVecSmallRows) {
      launch_cg_vec_small<CT>(Minv, Hc, dmode, x, r, z, p, q, xbest, cg, par, n, stream);
      continue;
    }
    LM_LAUNCH(cg_dot_kernel<CT>, n, stream, p, q, cg, ws, n);
    LM_LAUNCH(cg_update_kernel<CT>, n, stream, Minv, p, q, x, r, z, xbest, cg, ws, par, n);
    LM_LAUNCH(cg_dir_kernel<CT>, n, stream, z, Hc, dmode, p, q, cg, par, n);
  }
  return (int)cudaGetLastError();
}

#define PCG_ABI(SFX, CT)                                                                                              \
  B200_EXPORT int b200_lm_blk6_damp_inv_##SFX(const CT* H, double scale, double dmin, double dmax, CT* Hd, CT* extra, \
                                              CT* Minv, long long n, void* stream) {                                  \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH(blk6_damp_inv_kernel<CT>, n, stream, H, (CT)scale, (CT)dmin, (CT)dmax, Hd, extra, Minv, n);             \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pt3_damp_inv_##SFX(const CT* H, double scale, double dmin, double dmax, CT* Hinv,           \
                                             long long n, void* stream) {                                             \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH(pt3_damp_inv_kernel<CT>, n, stream, H, (CT)scale, (CT)dmin, (CT)dmax, Hinv, n);                         \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pt3_apply_##SFX(const CT* A6, const CT* t, double alpha, CT* out, long long n,              \
                                          void* stream) {                                                             \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH(pt3_apply_kernel<CT>, n, stream, A6, t, (CT)alpha, out, n);                                             \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pgo_pcg_##SFX(const CT* M, const int* ei, const int* ej, long long E, const CT* Minv,       \
                                        const CT* extra, const CT* g, CT* x, CT* r, CT* z, CT* p, CT* q, CT* xbest,   \
                                        double* cg, double* ws, double tol, long long maxiter, long long first_iter,  \
                                        long long iters, const unsigned long long* bases, int rank, int world,        \
                                        long long stage, long long result, long long epoch, unsigned* tickets,        \
                                        long long n, void* stream) {                                                  \
    if (!pairs_aligned<CT>(g, x, r, z, p, q, xbest)) return kMisaligned;                                              \
    return pgo_pcg_run<CT>(M, ei, ej, E, Minv, extra, g, x, r, z, p, q, xbest, cg, ws, tol, maxiter, first_iter,      \
                           iters, n, (cudaStream_t)stream,                                                            \
                           make_pcg_comm(bases, rank, world, stage, result, epoch, tickets));                         \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_cg_finish_##SFX(CT* x, const CT* xbest, const double* cg, long long n, void* stream) {      \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH(cg_finish_kernel<CT>, n * 6, stream, x, xbest, cg, n * 6);                                              \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pgo_predicted_##SFX(const CT* M, const int* ei, const int* ej, long long E, const CT* D,    \
                                              const CT* g, double* ws, long long n, void* stream) {                   \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH(pgo_predicted_kernel<CT>, (E > n ? E : n), stream, M, ei, ej, D, g, ws, E, n);                          \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pgo_predicted_edge_##SFX(const CT* M0, const CT* u0, const int* ei, const int* ej,          \
                                                   const CT* D, double* ws, long long E, void* stream) {              \
    if (E <= 0) return 0;                                                                                             \
    LM_LAUNCH(pgo_predicted_edge_kernel<CT>, E, stream, M0, u0, ei, ej, D, ws, E);                                    \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_ba_wtx_gather_##SFX(const CT* Y4p, const CT* poses, const int* cidx_p, const int* pptr,     \
                                              const CT* Hpinv, const CT* x, const CT* t0, double alpha, CT* u,        \
                                              long long P, void* stream) {                                            \
    if (P <= 0) return 0;                                                                                             \
    LM_LAUNCH(pcg_ba_wtx_gather_kernel<CT>, P * kLanesPerPoint, stream, Y4p, poses, cidx_p, pptr, Hpinv, x, t0,       \
              (CT)alpha, u, (const double*)nullptr, P);                                                                             \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_ba_pcg_##SFX(const CT* Y4, const CT* poses, const int* pidx, const int* cseg,               \
                                       long long split, long long tpi, long long m,                                   \
                                       const CT* Y4p, const int* cidx_p, const int* pptr, const CT* Hc,               \
                                       const CT* Hpinv, const CT* Minv, const CT* bneg, CT* x, CT* r, CT* z, CT* p,   \
                                       CT* q, CT* t, CT* part, CT* xbest, double* cg, double* ws, double tol,         \
                                       long long maxiter, long long P, long long first_iter, long long iters,         \
                                       const unsigned long long* bases, int rank, int world, long long stage,         \
                                       long long result, long long epoch, unsigned* tickets, long long n,             \
                                       void* stream) {                                                                \
    if (!pairs_aligned<CT>(bneg, x, r, z, p, q, xbest)) return kMisaligned;                                           \
    return ba_pcg_run<CT>(Y4, poses, pidx, cseg, split, tpi, m, Y4p, cidx_p, pptr, Hc, Hpinv, Minv, bneg, x, r, z, p, \
                          q, t, part, xbest, cg, ws, tol, maxiter, P, first_iter, iters, n, (cudaStream_t)stream,     \
                          make_pcg_comm(bases, rank, world, stage, result, epoch, tickets));                          \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_ba_predicted_##SFX(const CT* Y4, const CT* poses, const CT* rs, const int* cidx,            \
                                             const int* pidx, const CT* xc, const CT* xp, double* ws, long long m,    \
                                             void* stream) {                                                          \
    if (m <= 0) return 0;                                                                                             \
    LM_LAUNCH(ba_predicted_kernel<CT>, m, stream, Y4, poses, rs, cidx, pidx, xc, xp, ws, m);                          \
    return (int)cudaGetLastError();                                                                                   \
  }

PCG_ABI(f32, float)
PCG_ABI(f64, double)
