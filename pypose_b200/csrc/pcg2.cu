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
// The kernels are templated on the block width W: 6 for SE3 nodes, 7 for Sim3 nodes (sim3pgo.cu; 28-word slots), 3 for
// SO3 nodes (so3pgo.cu; 8-word slots).
#include "lm_common.cuh"
#include "sim3pgo_math.cuh"

namespace b200pose {

enum { CG2_RZ0 = 0, CG2_RZ1 = 1, CG2_PQ = 2, CG2_DONE = 5 };       // same slots as pcg.cu
constexpr int kLanes = 4;                                           // lanes cooperating on one node
// node-ordered slot of W unknowns: W = 6 (SE3): 21 words padded to 24 (96 / 192 B, six 16-byte loads in fp32);
// W = 7 (Sim3, sim3pgo.cu): 28 words, unpadded (112 / 224 B); W = 3 (SO3, so3pgo.cu): 6 words padded to 8 (32 / 64 B)
template <int W> struct Slot;
template <> struct Slot<6> { static constexpr int words = 24, packed = 21; };
template <> struct Slot<7> { static constexpr int words = 28, packed = 28; };
template <> struct Slot<3> { static constexpr int words = 8, packed = 6; };

template <typename T, int NW> __device__ __forceinline__ void ld_slot(const T* __restrict__ p, T (&a)[NW]) {
  if (sizeof(T) == 4) {
    const float4* v = reinterpret_cast<const float4*>(p);
#pragma unroll
    for (int k = 0; k < NW / 4; ++k) {
      const float4 t = __ldg(v + k);
      a[4 * k] = t.x; a[4 * k + 1] = t.y; a[4 * k + 2] = t.z; a[4 * k + 3] = t.w;
    }
  } else {
    const double2* v = reinterpret_cast<const double2*>(p);
#pragma unroll
    for (int k = 0; k < NW / 2; ++k) {
      const double2 t = __ldg(v + k);
      a[2 * k] = t.x; a[2 * k + 1] = t.y;
    }
  }
}
// w = M d for the block in one slot (W = 6 unpacks to 6x6 first; a 7x7 fp64 copy would cost 98 registers)
template <typename T, int W> __device__ __forceinline__ void slot_mv(const T* __restrict__ p, const T (&d)[W], T (&w)[W]) {
  T a[Slot<W>::words];
  ld_slot<T, Slot<W>::words>(p, a);
  if constexpr (W == 6) {
    T A[6][6];
    sym6_unpack(a, A);
    sym6_mv(A, d, w);
  } else {
    symn_mv_packed<T, W>(a, d, w);
  }
}
template <typename T> struct Pair6g;
template <> struct Pair6g<float> { using type = float2; };
template <> struct Pair6g<double> { using type = double2; };
// gather of one node's six values as three 8- / 16-byte pairs (see pcg.cu ld6): half the LSU wavefronts of scalar loads;
// a node's seven (or three) values are not pair-aligned and are read value by value
template <typename T, int W> __device__ __forceinline__ void ldwg(const T* __restrict__ p, long long i, T (&v)[W]) {
  if constexpr (W == 6) {
    using P = typename Pair6g<T>::type;
    const P* q = reinterpret_cast<const P*>(p + i * 6);
#pragma unroll
    for (int k = 0; k < 3; ++k) { const P t = __ldg(q + k); v[2 * k] = t.x; v[2 * k + 1] = t.y; }
  } else {
#pragma unroll
    for (int k = 0; k < W; ++k) v[k] = __ldg(p + i * W + k);
  }
}

// Hd[n] = sum of the node's blocks (packed W x W), g[n] (W) = sum of its signed u   (diagonal of J^T J and J^T R,
// optimizer.py:642-643,668)
template <typename T, int W>
__global__ void __launch_bounds__(kLmThreads) pgo2_node_sums_kernel(const T* __restrict__ Mn, const T* __restrict__ un,
                                                                     const int* __restrict__ nptr, T* __restrict__ Hd,
                                                                     T* __restrict__ g, long long N) {
  constexpr int L = kLanes, NPB = kLmThreads / L, PW = Slot<W>::packed, NS = PW + W;
  const int sub = threadIdx.x % L;
  const long long groups = (N + NPB - 1) / NPB;
  for (long long grp = blockIdx.x; grp < groups; grp += gridDim.x) {
    const long long n = grp * NPB + threadIdx.x / L;
    T a[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) a[k] = T(0);
    if (n < N)
      for (int s = nptr[n] + sub; s < nptr[n + 1]; s += L) {
#pragma unroll
        for (int k = 0; k < PW; ++k) a[k] += Mn[(long long)s * Slot<W>::words + k];
#pragma unroll
        for (int k = 0; k < W; ++k) a[PW + k] += un[(long long)s * W + k];
      }
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < NS; ++k) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    if (n < N && sub == 0) {
#pragma unroll
      for (int k = 0; k < PW; ++k) Hd[n * PW + k] = a[k];
#pragma unroll
      for (int k = 0; k < W; ++k) g[n * W + k] = a[PW + k];
    }
  }
}

// Kernel A.  mode 0: CG iteration (p' = z + beta p_old, q = (H + extra) p', p_new <- p', ws/cg[PQ] = p'.q)
//            mode 1: predicted reduction of a finished solve: ws[0] = x^T H x + 2 x^T g   (z := x, g2 := g, nothing written)
template <typename T, int W>
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
    T v[W], pn[W];
#pragma unroll
    for (int k = 0; k < W; ++k) { v[k] = T(0); pn[k] = T(0); }
    if (n < N) {
      ldwg<T, W>(z, n, pn);
      if (beta != T(0)) {
        T po[W];
        ldwg<T, W>(p_old, n, po);
#pragma unroll
        for (int k = 0; k < W; ++k) pn[k] += beta * po[k];
      }
      for (int s = nptr[n] + sub; s < nptr[n + 1]; s += L) {
        const long long o = nother[s];
        T d[W], w[W];
        ldwg<T, W>(z, o, d);
        if (beta != T(0)) {
          T po[W];
          ldwg<T, W>(p_old, o, po);
#pragma unroll
          for (int k = 0; k < W; ++k) d[k] += beta * po[k];
        }
#pragma unroll
        for (int k = 0; k < W; ++k) d[k] = pn[k] - d[k];
        slot_mv<T, W>(Mn + (long long)s * Slot<W>::words, d, w);
#pragma unroll
        for (int k = 0; k < W; ++k) v[k] += w[k];
      }
    }
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < W; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (n < N && sub == 0) {
      T dot = T(0);
      if (mode == 0) {
#pragma unroll
        for (int k = 0; k < W; ++k) { v[k] += extra[n * W + k] * pn[k]; dot += pn[k] * v[k]; }
#pragma unroll
        for (int k = 0; k < W; ++k) { p_new[n * W + k] = pn[k]; q[n * W + k] = v[k]; }
      } else {
#pragma unroll
        for (int k = 0; k < W; ++k) dot += pn[k] * (v[k] + T(2) * g2[n * W + k]);
      }
      acc[0] += (double)dot;
    }
  }
  if (reduce_sums<1>(acc, ws) && mode == 0) cg[CG2_PQ] = ws[0];
}

// declared in pcg.cu (same translation-unit-independent kernels): init, update and finish of the CG vectors
template <typename T, int W>
void pcg_launch_init(const T* Minv, const T* b, T* x, T* r, T* p, T* q, double* cg, double* ws, double tol, double maxiter,
                     long long n, cudaStream_t st);
template <typename T, int W>
void pcg_launch_update(const T* Minv, const T* p, const T* q, T* x, T* r, T* z, T* xbest, double* cg, double* ws, int par,
                       long long n, cudaStream_t st);

template <typename CT, int W>
static int pgo2_node_sums_launch(const CT* Mn, const CT* un, const int* nptr, CT* Hd, CT* g, long long N, cudaStream_t st) {
  if (N <= 0) return 0;
  pgo2_node_sums_kernel<CT, W><<<lm_grid(N * kLanes, kLmThreads), kLmThreads, 0, st>>>(Mn, un, nptr, Hd, g, N);
  return (int)cudaGetLastError();
}
template <typename CT, int W>
static int pgo2_pcg_run(const CT* Mn, const int* nother, const int* nptr, const CT* Minv, const CT* extra, const CT* g, CT* x,
                        CT* r, CT* z, CT* p0, CT* p1, CT* q, CT* xbest, double* cg, double* ws, double tol, long long maxiter,
                        long long first_iter, long long iters, long long n, cudaStream_t st) {
  if (n <= 0) return 0;
  const unsigned grid = lm_grid(n * kLanes, kLmThreads);
  if (first_iter == 0) pcg_launch_init<CT, W>(Minv, g, x, r, z, q, cg, ws, tol, (double)maxiter, n, st);
  for (long long it = first_iter; it < first_iter + iters; ++it) {
    CT* pn = (it & 1) ? p1 : p0;
    const CT* po = (it & 1) ? p0 : p1;
    pgo2_operator_kernel<CT, W><<<grid, kLmThreads, 0, st>>>(Mn, nother, nptr, extra, z, po, pn, q, (const CT*)nullptr, cg, ws,
                                                             0, it == 0 ? 1 : 0, (int)((it - 1) & 1), n);
    pcg_launch_update<CT, W>(Minv, pn, q, x, r, z, xbest, cg, ws, (int)(it & 1), n, st);
  }
  return (int)cudaGetLastError();
}
template <typename CT, int W>
static int pgo2_predicted_launch(const CT* Mn, const int* nother, const int* nptr, const CT* x, const CT* g, double* ws,
                                 long long n, cudaStream_t st) {
  if (n <= 0) return 0;
  pgo2_operator_kernel<CT, W><<<lm_grid(n * kLanes, kLmThreads), kLmThreads, 0, st>>>(
      Mn, nother, nptr, (const CT*)nullptr, x, (const CT*)nullptr, (CT*)nullptr, (CT*)nullptr, g, (double*)nullptr, ws, 1, 1, 0,
      n);
  return (int)cudaGetLastError();
}

}  // namespace b200pose

using namespace b200pose;

// W = 6: SE3 pose graphs and pose pairs (vectors accessed as pairs, so they must be pair-aligned); W = 7: Sim3 pose graphs;
// W = 3: SO3 pose graphs
#define PCG2_ABI(SFX, CT)                                                                                             \
  B200_EXPORT int b200_lm_pgo2_node_sums_##SFX(const CT* Mn, const CT* un, const int* nptr, CT* Hd, CT* g,            \
                                               long long N, void* stream) {                                           \
    return pgo2_node_sums_launch<CT, 6>(Mn, un, nptr, Hd, g, N, (cudaStream_t)stream);                                \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pgo2_pcg_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* Minv,            \
                                         const CT* extra, const CT* g, CT* x, CT* r, CT* z, CT* p0, CT* p1, CT* q,    \
                                         CT* xbest, double* cg, double* ws, double tol, long long maxiter,            \
                                         long long first_iter, long long iters, long long n, void* stream) {          \
    if (n <= 0) return 0;                                                                                             \
    if (!pairs_aligned<CT>(g, x, r, z, p0, p1, q, xbest)) return kMisaligned;                                         \
    return pgo2_pcg_run<CT, 6>(Mn, nother, nptr, Minv, extra, g, x, r, z, p0, p1, q, xbest, cg, ws, tol, maxiter,     \
                               first_iter, iters, n, (cudaStream_t)stream);                                           \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_pgo2_predicted_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* x,         \
                                               const CT* g, double* ws, long long n, void* stream) {                  \
    if (n <= 0) return 0;                                                                                             \
    if (!pairs_aligned<CT>(x)) return kMisaligned;                                                                    \
    return pgo2_predicted_launch<CT, 6>(Mn, nother, nptr, x, g, ws, n, (cudaStream_t)stream);                         \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_sim3pgo_node_sums_##SFX(const CT* Mn, const CT* un, const int* nptr, CT* Hd, CT* g,         \
                                                  long long N, void* stream) {                                        \
    return pgo2_node_sums_launch<CT, 7>(Mn, un, nptr, Hd, g, N, (cudaStream_t)stream);                                \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_sim3pgo_pcg_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* Minv,         \
                                            const CT* extra, const CT* g, CT* x, CT* r, CT* z, CT* p0, CT* p1, CT* q, \
                                            CT* xbest, double* cg, double* ws, double tol, long long maxiter,         \
                                            long long first_iter, long long iters, long long n, void* stream) {       \
    return pgo2_pcg_run<CT, 7>(Mn, nother, nptr, Minv, extra, g, x, r, z, p0, p1, q, xbest, cg, ws, tol, maxiter,     \
                               first_iter, iters, n, (cudaStream_t)stream);                                           \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_sim3pgo_predicted_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* x,      \
                                                  const CT* g, double* ws, long long n, void* stream) {               \
    return pgo2_predicted_launch<CT, 7>(Mn, nother, nptr, x, g, ws, n, (cudaStream_t)stream);                         \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_so3pgo_node_sums_##SFX(const CT* Mn, const CT* un, const int* nptr, CT* Hd, CT* g,          \
                                                 long long N, void* stream) {                                         \
    return pgo2_node_sums_launch<CT, 3>(Mn, un, nptr, Hd, g, N, (cudaStream_t)stream);                                \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_so3pgo_pcg_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* Minv,          \
                                           const CT* extra, const CT* g, CT* x, CT* r, CT* z, CT* p0, CT* p1, CT* q,  \
                                           CT* xbest, double* cg, double* ws, double tol, long long maxiter,          \
                                           long long first_iter, long long iters, long long n, void* stream) {        \
    return pgo2_pcg_run<CT, 3>(Mn, nother, nptr, Minv, extra, g, x, r, z, p0, p1, q, xbest, cg, ws, tol, maxiter,     \
                               first_iter, iters, n, (cudaStream_t)stream);                                           \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_so3pgo_predicted_##SFX(const CT* Mn, const int* nother, const int* nptr, const CT* x,       \
                                                 const CT* g, double* ws, long long n, void* stream) {                \
    return pgo2_predicted_launch<CT, 3>(Mn, nother, nptr, x, g, ws, n, (cudaStream_t)stream);                         \
  }

PCG2_ABI(f32, float)
PCG2_ABI(f64, double)
