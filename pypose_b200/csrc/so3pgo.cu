// so3pgo.cu — linearisation and loss of the SO3 pose graph (rotation averaging) in node order (C-ABI: include/b200pose.h,
// section LM).
//
// The SO3 counterpart of sim3pgo.cu: every edge (i, j) writes its block M_e (3x3 packed, 6 words, plus 2 zero words of
// padding: 8-word slots of 32 B in fp32 and 64 B in fp64, so slots stay 16-byte aligned) and its signed u_e into one slot
// of each endpoint's adjacency list (epos_i / epos_j).  Block sums, the CG operator and the predicted reduction are the
// gathers of pcg2.cu at block width 3; the per-edge math is so3pgo_math.cuh.
#include "lm_common.cuh"
#include "so3pgo_math.cuh"

namespace b200pose {

constexpr int kSo3Slot = 8;                       // words per node-ordered slot (pcg2.cu Slot<3>)

template <typename T>
__device__ __forceinline__ void load_so3_edge(const T* __restrict__ nodes, const T* __restrict__ Z, long long e, long long i,
                                              long long j, Elem<T>& A, Elem<T>& B, Elem<T>& Ze) {
  T a[4], b[4], z[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { a[k] = __ldg(nodes + i * 4 + k); b[k] = __ldg(nodes + j * 4 + k); z[k] = Z[e * 4 + k]; }
  A = load_elem<SO3g, T>(a); B = load_elem<SO3g, T>(b); Ze = load_elem<SO3g, T>(z);
}

template <typename T>
__global__ void __launch_bounds__(kLmThreads) so3pgo_linearize_kernel(const T* __restrict__ nodes, const T* __restrict__ Z,
                                                                       const int* __restrict__ ei, const int* __restrict__ ej,
                                                                       const int* __restrict__ epos_i,
                                                                       const int* __restrict__ epos_j, T* __restrict__ Mn,
                                                                       T* __restrict__ un, double* ws, int rk, T rdelta,
                                                                       long long E) {
  double acc[1] = {0.0};
  for (long long e = (long long)blockIdx.x * kLmThreads + threadIdx.x; e < E; e += (long long)gridDim.x * kLmThreads) {
    Elem<T> A, B, Ze;
    load_so3_edge(nodes, Z, e, ei[e], ej[e], A, B, Ze);
    Tang<T> r;
    T M[kSo3Packed], u[kSo3];
    so3pgo_linearize(A, B, Ze, r, M, u);
    T rho, w;
    robust_eval(rk, rdelta, tang3_sqnorm(r), rho, w);
    if (rk) sys3_scale(M, u, w);
    const long long si = epos_i[e], sj = epos_j[e];
#pragma unroll
    for (int k = 0; k < kSo3Slot; ++k) {
      const T v = k < kSo3Packed ? M[k] : T(0);
      Mn[si * kSo3Slot + k] = v; Mn[sj * kSo3Slot + k] = v;
    }
#pragma unroll
    for (int k = 0; k < kSo3; ++k) { un[si * kSo3 + k] = -u[k]; un[sj * kSo3 + k] = u[k]; }
    acc[0] += (double)rho;
  }
  reduce_sums<1>(acc, ws);
}

template <typename T>
__global__ void __launch_bounds__(kLmThreads) so3pgo_loss_kernel(const T* __restrict__ nodes, const T* __restrict__ Z,
                                                                  const int* __restrict__ ei, const int* __restrict__ ej,
                                                                  double* ws, int rk, T rdelta, long long E) {
  double acc[1] = {0.0};
  for (long long e = (long long)blockIdx.x * kLmThreads + threadIdx.x; e < E; e += (long long)gridDim.x * kLmThreads) {
    Elem<T> A, B, Ze, S;
    load_so3_edge(nodes, Z, e, ei[e], ej[e], A, B, Ze);
    T rho, w;
    robust_eval(rk, rdelta, tang3_sqnorm(so3pgo_residual(A, B, Ze, S)), rho, w);
    acc[0] += (double)rho;
  }
  reduce_sums<1>(acc, ws);
}

}  // namespace b200pose

using namespace b200pose;

#define SO3PGO_ABI(SFX, CT)                                                                                           \
  B200_EXPORT int b200_lm_so3pgo_linearize_##SFX(const CT* nodes, const CT* Z, const int* ei, const int* ej,           \
                                                 const int* epos_i, const int* epos_j, CT* Mn, CT* un, double* ws,    \
                                                 int robust, double delta, long long E, void* stream) {               \
    if (E <= 0) return 0;                                                                                             \
    so3pgo_linearize_kernel<CT><<<lm_grid(E, kLmThreads), kLmThreads, 0, (cudaStream_t)stream>>>(                     \
        nodes, Z, ei, ej, epos_i, epos_j, Mn, un, ws, robust, (CT)delta, E);                                          \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_so3pgo_loss_##SFX(const CT* nodes, const CT* Z, const int* ei, const int* ej, double* ws,   \
                                            int robust, double delta, long long E, void* stream) {                    \
    if (E <= 0) return 0;                                                                                             \
    so3pgo_loss_kernel<CT><<<lm_grid(E, kLmThreads), kLmThreads, 0, (cudaStream_t)stream>>>(nodes, Z, ei, ej, ws,     \
                                                                                            robust, (CT)delta, E);    \
    return (int)cudaGetLastError();                                                                                   \
  }

SO3PGO_ABI(f32, float)
SO3PGO_ABI(f64, double)
