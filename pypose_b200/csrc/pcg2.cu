// pcg2.cu — pose-graph / pose-pair PCG without atomics, two kernels per iteration (C-ABI: include/b200pose.h, section LM).
//
// The per-edge scatter route (`lm_pgo_scatter`, `pcg_pgo_spmv`) is throttled by global fp32 atomics and needs four kernels
// per CG iteration.  This file replaces that route on one GPU:
//
//  * the per-edge blocks are produced directly in NODE order by the linearisation kernels: every edge (i, j) owns one slot
//    in i's list and one in j's (epos_i / epos_j), each slot holds the 21 numbers of M_e padded to 24 (96 B, 16-byte
//    aligned -> six 128-bit loads) and the signed u_e; block sums and H products are then GATHERS with one writer per
//    node: no atomics, bit-reproducible;
//  * the direction update p = z + beta p is folded into the operator kernel (a neighbour's p is rebuilt from z and the
//    previous p, both L2-resident), together with the p.Ap reduction:
//        A:  p' = z + beta p;  q = (H + D) p';  p'.q            (gather over node-ordered blocks)
//        B:  alpha;  x += alpha p';  r -= alpha q;  z = M^-1 r;  r.z, r.r;  stop / best-iterate bookkeeping
//    i.e. 2 launches per iteration instead of 4, same arithmetic as optim/solver.py:312-340 with M = block-Jacobi.
#include "lm_common.cuh"

namespace b200pose {

enum { CG2_RZ0 = 0, CG2_RZ1 = 1, CG2_PQ = 2, CG2_DONE = 5 };       // same slots as pcg.cu
constexpr int kBlk = 24;                                            // floats per node-ordered block (21 used)
constexpr int kLanes = 4;                                           // lanes cooperating on one node

template <typename T> __device__ __forceinline__ void ld_block24(const T* __restrict__ p, T (&A)[6][6]) {
  T a[24];
  if (sizeof(T) == 4) {
    const float4* v = reinterpret_cast<const float4*>(p);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float4 t = __ldg(v + k);
      a[4 * k] = t.x; a[4 * k + 1] = t.y; a[4 * k + 2] = t.z; a[4 * k + 3] = t.w;
    }
  } else {
    const double2* v = reinterpret_cast<const double2*>(p);
#pragma unroll
    for (int k = 0; k < 12; ++k) {
      const double2 t = __ldg(v + k);
      a[2 * k] = t.x; a[2 * k + 1] = t.y;
    }
  }
  sym6_unpack(a, A);
}
template <typename T> struct Pair6g;
template <> struct Pair6g<float> { using type = float2; };
template <> struct Pair6g<double> { using type = double2; };
// gather of one node's six values as three 8- / 16-byte pairs (see pcg.cu ld6): half the LSU wavefronts of scalar loads
template <typename T> __device__ __forceinline__ void ld6g(const T* __restrict__ p, long long i, T (&v)[6]) {
  using P = typename Pair6g<T>::type;
  const P* q = reinterpret_cast<const P*>(p + i * 6);
#pragma unroll
  for (int k = 0; k < 3; ++k) { const P t = __ldg(q + k); v[2 * k] = t.x; v[2 * k + 1] = t.y; }
}

// Hd[n] (21) = sum of the node's blocks, g[n] (6) = sum of its signed u   (diagonal of J^T J and J^T R, optimizer.py:642-643,668)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) pgo2_node_sums_kernel(const T* __restrict__ Mn, const T* __restrict__ un,
                                                                     const int* __restrict__ nptr, T* __restrict__ Hd,
                                                                     T* __restrict__ g, long long N) {
  constexpr int L = kLanes, NPB = kLmThreads / L;
  const int sub = threadIdx.x % L;
  const long long groups = (N + NPB - 1) / NPB;
  for (long long grp = blockIdx.x; grp < groups; grp += gridDim.x) {
    const long long n = grp * NPB + threadIdx.x / L;
    T a[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) a[k] = T(0);
    if (n < N)
      for (int s = nptr[n] + sub; s < nptr[n + 1]; s += L) {
#pragma unroll
        for (int k = 0; k < 21; ++k) a[k] += Mn[(long long)s * kBlk + k];
#pragma unroll
        for (int k = 0; k < 6; ++k) a[21 + k] += un[(long long)s * 6 + k];
      }
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < 27; ++k) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    if (n < N && sub == 0) {
#pragma unroll
      for (int k = 0; k < 21; ++k) Hd[n * 21 + k] = a[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) g[n * 6 + k] = a[21 + k];
    }
  }
}

// Kernel A.  mode 0: CG iteration (p' = z + beta p_old, q = (H + extra) p', p_new <- p', ws/cg[PQ] = p'.q)
//            mode 1: predicted reduction of a finished solve: ws[0] = x^T H x + 2 x^T g   (z := x, g2 := g, nothing written)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) pgo2_operator_kernel(const T* __restrict__ Mn, const int* __restrict__ nother,
                                                                    const int* __restrict__ nptr, const T* __restrict__ extra,
                                                                    const T* __restrict__ z, const T* __restrict__ p_old,
                                                                    T* __restrict__ p_new, T* __restrict__ q,
                                                                    const T* __restrict__ g2, double* cg, double* ws, int mode,
                                                                    int first, int par_prev, long long N) {
  if (mode == 0 && cg[CG2_DONE] != 0.0) return;
  constexpr int L = kLanes, NPB = kLmThreads / L;
  const int sub = threadIdx.x % L;
  const T beta = (mode == 1 || first) ? T(0) : (T)(cg[par_prev ^ 1] / cg[par_prev]);
  const long long groups = (N + NPB - 1) / NPB;
  double acc[1] = {0.0};
  for (long long grp = blockIdx.x; grp < groups; grp += gridDim.x) {
    const long long n = grp * NPB + threadIdx.x / L;
    T v[6] = {T(0), T(0), T(0), T(0), T(0), T(0)}, pn[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
    if (n < N) {
      ld6g(z, n, pn);
      if (beta != T(0)) {
        T po[6];
        ld6g(p_old, n, po);
#pragma unroll
        for (int k = 0; k < 6; ++k) pn[k] += beta * po[k];
      }
      for (int s = nptr[n] + sub; s < nptr[n + 1]; s += L) {
        const long long o = nother[s];
        T d[6], w[6], A[6][6];
        ld6g(z, o, d);
        if (beta != T(0)) {
          T po[6];
          ld6g(p_old, o, po);
#pragma unroll
          for (int k = 0; k < 6; ++k) d[k] += beta * po[k];
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) d[k] = pn[k] - d[k];
        ld_block24(Mn + (long long)s * kBlk, A);
        sym6_mv(A, d, w);
#pragma unroll
        for (int k = 0; k < 6; ++k) v[k] += w[k];
      }
    }
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < 6; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (n < N && sub == 0) {
      T dot = T(0);
      if (mode == 0) {
#pragma unroll
        for (int k = 0; k < 6; ++k) { v[k] += extra[n * 6 + k] * pn[k]; dot += pn[k] * v[k]; }
#pragma unroll
        for (int k = 0; k < 6; ++k) { p_new[n * 6 + k] = pn[k]; q[n * 6 + k] = v[k]; }
      } else {
#pragma unroll
        for (int k = 0; k < 6; ++k) dot += pn[k] * (v[k] + T(2) * g2[n * 6 + k]);
      }
      acc[0] += (double)dot;
    }
  }
  if (reduce_sums<1>(acc, ws) && mode == 0) cg[CG2_PQ] = ws[0];
}

// declared in pcg.cu (same translation-unit-independent kernels): init, update and finish of the CG vectors
template <typename T>
void pcg_launch_init(const T* Minv, const T* b, T* x, T* r, T* p, T* q, double* cg, double* ws, double tol, double maxiter,
                     long long n, cudaStream_t st);
template <typename T>
void pcg_launch_update(const T* Minv, const T* p, const T* q, T* x, T* r, T* z, T* xbest, double* cg, double* ws, int par,
                       long long n, cudaStream_t st);

}  // namespace b200pose

using namespace b200pose;

#define PCG2_ABI(SFX, CT)                                                                                             \
  B200_EXPORT int b200_lm_pgo2_node_sums_##SFX(const CT* Mn, const CT* un, const int* nptr, CT* Hd, CT* g,            \
                                               long long N, void* stream) {                                           \
    if (N <= 0) return 0;                                                                                             \
    pgo2_node_sums_kernel<CT><<<lm_grid(N * kLanes, kLmThreads), kLmThreads, 0, (cudaStream_t)stream>>>(Mn, un, nptr, \
                                                                                                        Hd, g, N);    \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pgo2_pcg_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* Minv,            \
                                         const CT* extra, const CT* g, CT* x, CT* r, CT* z, CT* p0, CT* p1, CT* q,    \
                                         CT* xbest, double* cg, double* ws, double tol, long long maxiter,            \
                                         long long first_iter, long long iters, long long n, void* stream) {          \
    if (n <= 0) return 0;                                                                                             \
    if (!pairs_aligned<CT>(g, x, r, z, p0, p1, q, xbest)) return kMisaligned;                                         \
    cudaStream_t st = (cudaStream_t)stream;                                                                           \
    const unsigned grid = lm_grid(n * kLanes, kLmThreads);                                                            \
    if (first_iter == 0) pcg_launch_init<CT>(Minv, g, x, r, z, q, cg, ws, tol, (double)maxiter, n, st);               \
    for (long long it = first_iter; it < first_iter + iters; ++it) {                                                  \
      CT* pn = (it & 1) ? p1 : p0;                                                                                    \
      const CT* po = (it & 1) ? p0 : p1;                                                                              \
      pgo2_operator_kernel<CT><<<grid, kLmThreads, 0, st>>>(Mn, nother, nptr, extra, z, po, pn, q, (const CT*)nullptr,\
                                                            cg, ws, 0, it == 0 ? 1 : 0, (int)((it - 1) & 1), n);      \
      pcg_launch_update<CT>(Minv, pn, q, x, r, z, xbest, cg, ws, (int)(it & 1), n, st);                               \
    }                                                                                                                 \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pgo2_predicted_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* x,         \
                                               const CT* g, double* ws, long long n, void* stream) {                  \
    if (n <= 0) return 0;                                                                                             \
    if (!pairs_aligned<CT>(x)) return kMisaligned;                                                                    \
    pgo2_operator_kernel<CT><<<lm_grid(n * kLanes, kLmThreads), kLmThreads, 0, (cudaStream_t)stream>>>(               \
        Mn, nother, nptr, (const CT*)nullptr, x, (const CT*)nullptr, (CT*)nullptr, (CT*)nullptr, g, (double*)nullptr, \
        ws, 1, 1, 0, n);                                                                                              \
    return (int)cudaGetLastError();                                                                                   \
  }

PCG2_ABI(f32, float)
PCG2_ABI(f64, double)
