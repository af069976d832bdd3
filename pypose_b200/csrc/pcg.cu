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
#include "pcg_vec.cuh"

namespace b200pose {


// diag <- clamp(diag, dmin, dmax) * scale (optimizer.py:657 + cumulative :666); optional outputs: the damped block,
// the amount added to the diagonal, the inverse of the damped block.  W = 6: SE3 blocks; W = 7: Sim3 pose-graph blocks;
// W = 3: SO3 pose-graph blocks.
template <int W, typename T> __device__ __forceinline__ void blkw_unpack(const T* a, T (&A)[W][W]) {
  if constexpr (W == 6) sym6_unpack(a, A);
  else symn_unpack<T, W>(a, A);
}
template <int W, typename T> __device__ __forceinline__ void blkw_pack(const T (&A)[W][W], T* a) {
  if constexpr (W == 6) sym6_pack(A, a);
  else symn_pack<T, W>(A, a);
}
template <typename T, int W>
__global__ void __launch_bounds__(kLmThreads) blkw_damp_inv_kernel(const T* __restrict__ H, T scale, T dmin, T dmax,
                                                                    T* __restrict__ Hd, T* __restrict__ extra,
                                                                    T* __restrict__ Minv, long long n) {
  constexpr int NP = packed_words<W>();
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T A[W][W], Ai[W][W];
    blkw_unpack<W>(H + i * NP, A);
#pragma unroll
    for (int k = 0; k < W; ++k) {
      const T d = A[k][k];
      const T c = (d < dmin ? dmin : (d > dmax ? dmax : d)) * scale;
      if (extra) extra[i * W + k] = c - d;
      A[k][k] = c;
    }
    if (Hd) blkw_pack<W>(A, Hd + i * NP);
    if (Minv) { spd_inverse<T, W>(A, Ai); blkw_pack<W>(Ai, Minv + i * NP); }
  }
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
template <typename T, int W>
void pcg_launch_init(const T* Minv, const T* b, T* x, T* r, T* z, T* q, double* cg, double* ws, double tol, double maxiter,
                     long long n, cudaStream_t st) {
  cg_init_kernel<T, W><<<lm_grid(n, kLmThreads), kLmThreads, 0, st>>>(Minv, b, (T)-1, (const T*)nullptr, 0, x, r, z, q, cg, ws,
                                                                     tol, maxiter, n);
}
template <typename T, int W>
void pcg_launch_update(const T* Minv, const T* p, const T* q, T* x, T* r, T* z, T* xbest, double* cg, double* ws, int par,
                       long long n, cudaStream_t st) {
  cg_update_kernel<T, W><<<lm_grid(n, kLmThreads), kLmThreads, 0, st>>>(Minv, p, q, x, r, z, xbest, cg, ws, par, n);
}
#define PCG_LAUNCH_INST(T, W)                                                                                        \
  template void pcg_launch_init<T, W>(const T*, const T*, T*, T*, T*, T*, double*, double*, double, double, long long,     \
                                      cudaStream_t);                                                                  \
  template void pcg_launch_update<T, W>(const T*, const T*, const T*, T*, T*, T*, T*, double*, double*, int, long long,   \
                                        cudaStream_t);
PCG_LAUNCH_INST(float, 6)
PCG_LAUNCH_INST(double, 6)
PCG_LAUNCH_INST(float, 7)
PCG_LAUNCH_INST(double, 7)
PCG_LAUNCH_INST(float, 3)
PCG_LAUNCH_INST(double, 3)

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
    LM_LAUNCH((blkw_damp_inv_kernel<CT, 6>), n, stream, H, (CT)scale, (CT)dmin, (CT)dmax, Hd, extra, Minv, n);        \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_sim3pgo_damp_inv_##SFX(const CT* H, double scale, double dmin, double dmax, CT* Hd,         \
                                                 CT* extra, CT* Minv, long long n, void* stream) {                    \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH((blkw_damp_inv_kernel<CT, 7>), n, stream, H, (CT)scale, (CT)dmin, (CT)dmax, Hd, extra, Minv, n);        \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_sim3pgo_cg_finish_##SFX(CT* x, const CT* xbest, const double* cg, long long n,              \
                                                  void* stream) {                                                     \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH(cg_finish_kernel<CT>, n * 7, stream, x, xbest, cg, n * 7);                                              \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_so3pgo_damp_inv_##SFX(const CT* H, double scale, double dmin, double dmax, CT* Hd,          \
                                                CT* extra, CT* Minv, long long n, void* stream) {                     \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH((blkw_damp_inv_kernel<CT, 3>), n, stream, H, (CT)scale, (CT)dmin, (CT)dmax, Hd, extra, Minv, n);        \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_so3pgo_cg_finish_##SFX(CT* x, const CT* xbest, const double* cg, long long n,               \
                                                 void* stream) {                                                      \
    if (n <= 0) return 0;                                                                                             \
    LM_LAUNCH(cg_finish_kernel<CT>, n * 3, stream, x, xbest, cg, n * 3);                                              \
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
