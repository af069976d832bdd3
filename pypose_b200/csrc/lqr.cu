// lqr.cu — batched LQR for affine dynamics x' = A_t x + B_t u + c1_t and its KKT adjoint (C-ABI: include/b200pose.h,
// section "LQR").  DESIGN.md §3.7.  One warp per problem, n = ns + nc <= 32; the per-problem math is lqr_math.cuh.  Each
// warp keeps Q_t + F^T V F, F_t = [A_t B_t], V, the Cholesky factor of Quu and [K_t | k_t] in its slab of dynamic shared
// memory; [K_t | k_t] for every step (and d_tau in the adjoint) go to the workspace, because the rollout runs forwards
// in time after the recursion ran backwards.  No entry point reads anything back to the host.
#include <cuda_runtime.h>
#include "lqr_math.cuh"

#define B200_EXPORT extern "C" __attribute__((visibility("default")))

namespace b200pose {
namespace {

constexpr int kLqrSmemBudget = 48 * 1024;   // per CTA, so no opt-in attribute is needed (a slab is <= 34 KB: n = 32, fp64)

template <class T>
int warps_per_cta(int ns, int nc) {
  const int per = lqr_smem_elems(ns, nc) * (int)sizeof(T);
  const int w = kLqrSmemBudget / per;
  return w < 1 ? 1 : (w > 8 ? 8 : w);
}

template <class T>
__global__ void lqr_fwd_kernel(LqrProb<T> P, long long nb, T* ws, T* x, T* u, T* cost, T* xtr, int* status) {
  extern __shared__ __align__(16) unsigned char lqr_sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long b = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (b >= nb) return;
  const int ne = lqr_smem_elems(P.ns, P.nc);
  LqrSmem<T> s = lqr_carve(reinterpret_cast<T*>(lqr_sm) + warp * ne, P.ns, P.nc);
  const long long kw = (long long)P.nc * (P.ns + 1);
  const int st = lqr_solve(P, b, s, ws + b * P.steps * kw, x, u, cost, xtr, LqrLane{lane, 32});
  if (lane == 0) status[b] = st;
}

template <class T>
__global__ void lqr_bwd_kernel(LqrProb<T> P, long long nb, T* ws, const T* x, const T* u, const T* gx, const T* gu,
                               const T* gc, LqrGrad<T> G) {
  extern __shared__ __align__(16) unsigned char lqr_sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long b = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (b >= nb) return;
  const int ne = lqr_smem_elems(P.ns, P.nc);
  LqrSmem<T> s = lqr_carve(reinterpret_cast<T*>(lqr_sm) + warp * ne, P.ns, P.nc);
  const long long per = (long long)P.nc * (P.ns + 1) + P.ns + P.nc;
  lqr_adjoint(P, b, s, ws + b * P.steps * per, x, u, gx, gu, gc, G, LqrLane{lane, 32});
}

template <class T>
LqrProb<T> make_prob(const T* Q, long long Qb, long long Qt, const T* p, long long pb, long long pt, const T* A, long long Ab,
                     long long At, const T* B, long long Bb, long long Bt, const T* c1, long long cb, long long ct,
                     const T* x0, const T* u0, long long ub, long long ut, int T_, int ns, int nc) {
  return LqrProb<T>{{Q, Qb, Qt}, {p, pb, pt}, {A, Ab, At}, {B, Bb, Bt}, {c1, cb, ct}, {u0, ub, ut}, x0, T_, ns, nc};
}

bool valid(long long nb, int T_, int ns, int nc) { return nb >= 0 && T_ >= 1 && ns >= 1 && nc >= 1 && ns + nc <= 32; }

template <class T>
int fwd_run(const LqrProb<T>& P, long long nb, void* ws, T* x, T* u, T* cost, T* xtr, int* status, cudaStream_t s) {
  if (!valid(nb, P.steps, P.ns, P.nc)) return (int)cudaErrorInvalidValue;
  if (nb == 0) return 0;
  const int w = warps_per_cta<T>(P.ns, P.nc);
  const size_t sm = (size_t)w * lqr_smem_elems(P.ns, P.nc) * sizeof(T);
  lqr_fwd_kernel<T><<<(unsigned)((nb + w - 1) / w), 32 * w, sm, s>>>(P, nb, (T*)ws, x, u, cost, xtr, status);
  return (int)cudaGetLastError();
}

template <class T>
int bwd_run(const LqrProb<T>& P, long long nb, void* ws, const T* x, const T* u, const T* gx, const T* gu, const T* gc,
            const LqrGrad<T>& G, cudaStream_t s) {
  if (!valid(nb, P.steps, P.ns, P.nc)) return (int)cudaErrorInvalidValue;
  if (nb == 0) return 0;
  const int w = warps_per_cta<T>(P.ns, P.nc);
  const size_t sm = (size_t)w * lqr_smem_elems(P.ns, P.nc) * sizeof(T);
  lqr_bwd_kernel<T><<<(unsigned)((nb + w - 1) / w), 32 * w, sm, s>>>(P, nb, (T*)ws, x, u, gx, gu, gc, G);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace b200pose

using namespace b200pose;

#define B200_LQR_OPERANDS(CT)                                                                                               \
  const CT *Q, long long Q_bs, long long Q_ts, const CT *p, long long p_bs, long long p_ts, const CT *A, long long A_bs,   \
      long long A_ts, const CT *B, long long B_bs, long long B_ts, const CT *c1, long long c1_bs, long long c1_ts,          \
      const CT *x_init, const CT *u_traj, long long u_bs, long long u_ts
#define B200_LQR_PROB(CT) \
  make_prob<CT>(Q, Q_bs, Q_ts, p, p_bs, p_ts, A, A_bs, A_ts, B, B_bs, B_ts, c1, c1_bs, c1_ts, x_init, u_traj, u_bs, u_ts, T, ns, nc)

#define B200_LQR_ENTRIES(CT, SFX)                                                                                          \
  B200_EXPORT int b200_lqr_affine_##SFX(B200_LQR_OPERANDS(CT), CT* x, CT* u, CT* cost, CT* x_traj, int* status, void* ws, \
                                        long long nb, int T, int ns, int nc, void* stream) {                              \
    return fwd_run<CT>(B200_LQR_PROB(CT), nb, ws, x, u, cost, x_traj, status, (cudaStream_t)stream);                      \
  }                                                                                                                       \
  B200_EXPORT int b200_lqr_affine_bwd_##SFX(B200_LQR_OPERANDS(CT), const CT* x, const CT* u, const CT* gx, const CT* gu,  \
                                            const CT* gcost, CT* gQ, int gQ_tv, CT* gp, int gp_tv, CT* gA, int gA_tv,     \
                                            CT* gB, int gB_tv, CT* gc1, int gc1_tv, CT* gx_init, void* ws, long long nb,  \
                                            int T, int ns, int nc, void* stream) {                                        \
    const LqrGrad<CT> G{gQ, gp, gA, gB, gc1, gx_init, gQ_tv, gp_tv, gA_tv, gB_tv, gc1_tv};                               \
    return bwd_run<CT>(B200_LQR_PROB(CT), nb, ws, x, u, gx, gu, gcost, G, (cudaStream_t)stream);                          \
  }

B200_LQR_ENTRIES(float, f32)
B200_LQR_ENTRIES(double, f64)
