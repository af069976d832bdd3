// lmdrive.cu — native driver of one LM trial for the block-sparse pose families (C-ABI: b200_lm_pgo2_step).
//
// Driven from Python, the pose-graph step spends about as long in ~15 Python-level launches around the PCG loop, plus two
// blocking reads, as in its kernels.  The reference's counterpart is Python too
// (optimizer.py:629-680 + the external bae PCG), but here the per-trial sequence is fixed, so it is enqueued from C++ by
// calling the library's own entry points back to back, and the two things the host must learn — "has
// the CG finished?" and "was the trial accepted?" — arrive through mapped pinned memory that small kernels publish into.
#include <string.h>
#include <type_traits>
#include "lm_common.cuh"
#include "b200pose.h"

namespace b200pose {

// copy n doubles to mapped pinned host memory, then the sequence number (one thread)
__global__ void publish_kernel(const double* __restrict__ src, int n, double* host, double seq) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  volatile double* o = host;
  for (int k = 0; k < n; ++k) o[k] = src[k];
  __threadfence_system();
  o[n] = seq;
}
// optimizer.py:662-680 for this trial: cur loss from the linearisation slot, trial loss, predicted reduction
__global__ void pgo_decide_kernel(const double* ws_lin, const double* ws_loss, const double* ws_pred, LmCtl ctl, double* st,
                                  double* host, double seq) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  lm_decide(ctl, ws_lin[0], ws_loss[0], ws_pred[0], 0.0, st);
  volatile double* o = host;
  for (int k = 0; k <= ST_FAILED; ++k) o[k] = st[k];
  __threadfence_system();
  o[ST_SIZE - 1] = seq;
}
template <typename T>
__global__ void __launch_bounds__(kLmThreads) commit_kernel(const double* __restrict__ st, const T* __restrict__ src,
                                                             T* __restrict__ dst, long long count) {
  if (st[ST_STATUS] != 1.0) return;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < count; i += (long long)gridDim.x * kLmThreads)
    dst[i] = src[i];
}

static int spin_until(volatile double* flag, double seq, cudaStream_t s) {
  for (long long spin = 0;; ++spin) {
    if (*flag == seq) return 0;
    if ((spin & 0xffff) == 0xffff) {
      cudaError_t e = cudaStreamQuery(s);
      if (e == cudaSuccess) return *flag == seq ? 0 : (int)cudaErrorUnknown;
      if (e != cudaErrorNotReady) return (int)e;
    }
  }
}

#define B200_TRY(call) do { int rc_ = (call); if (rc_ != 0) return rc_; } while (0)

template <typename CT> struct Api;
#define B200_API(SFX, CT)                                                                                             \
  template <> struct Api<CT> {                                                                                        \
    static constexpr auto linearize = b200_lm_pgo_linearize_n_##SFX;                                                  \
    static constexpr auto accum2 = b200_lm_reproj2_accum_n_##SFX;                                                     \
    static constexpr auto node_sums = b200_lm_pgo2_node_sums_##SFX;                                                   \
    static constexpr auto damp_inv = b200_lm_blk6_damp_inv_##SFX;                                                     \
    static constexpr auto pcg = b200_lm_pgo2_pcg_##SFX;                                                               \
    static constexpr auto finish = b200_lm_cg_finish_##SFX;                                                           \
    static constexpr auto predicted = b200_lm_pgo2_predicted_##SFX;                                                   \
    static constexpr auto exp = b200_se3_exp_fwd_##SFX;                                                               \
    static constexpr auto mul = b200_SE3_mul_fwd_##SFX;                                                               \
    static constexpr auto loss = b200_lm_pgo_loss_##SFX;                                                              \
    static constexpr auto loss1 = b200_lm_reproj2_loss_##SFX;                                                         \
  };
B200_API(f32, float)
B200_API(f64, double)
// families 2 (Sim3 pose graph) and 3 (SO3 pose graph): the same sequence at block widths 7 and 3 (entry points of the
// same signatures)
#define B200_LIE_PGO_API(NAME, PFX, GRP, ALG, SFX, CT)                                                                \
  template <> struct NAME<CT> {                                                                                       \
    static constexpr auto linearize = b200_lm_##PFX##_linearize_##SFX;                                                \
    static constexpr auto node_sums = b200_lm_##PFX##_node_sums_##SFX;                                                \
    static constexpr auto damp_inv = b200_lm_##PFX##_damp_inv_##SFX;                                                  \
    static constexpr auto pcg = b200_lm_##PFX##_pcg_##SFX;                                                            \
    static constexpr auto finish = b200_lm_##PFX##_cg_finish_##SFX;                                                   \
    static constexpr auto predicted = b200_lm_##PFX##_predicted_##SFX;                                                \
    static constexpr auto exp = b200_##ALG##_exp_fwd_##SFX;                                                           \
    static constexpr auto mul = b200_##GRP##_mul_fwd_##SFX;                                                           \
    static constexpr auto loss = b200_lm_##PFX##_loss_##SFX;                                                          \
  };
template <typename CT> struct Sim3Api;
template <typename CT> struct So3Api;
B200_LIE_PGO_API(Sim3Api, sim3pgo, Sim3, sim3, f32, float)
B200_LIE_PGO_API(Sim3Api, sim3pgo, Sim3, sim3, f64, double)
B200_LIE_PGO_API(So3Api, so3pgo, SO3, so3, f32, float)
B200_LIE_PGO_API(So3Api, so3pgo, SO3, so3, f64, double)

// the entry points and widths of the family being run: W unknowns per node, parameter width D
template <typename CT> struct PgoFns {
  template <class F> using Fn = std::remove_cv_t<F>;
  Fn<decltype(Api<CT>::linearize)> linearize;             // families 0, 2 and 3 (family 1: Api::accum2)
  Fn<decltype(Api<CT>::node_sums)> node_sums;
  Fn<decltype(Api<CT>::damp_inv)> damp_inv;
  Fn<decltype(Api<CT>::pcg)> pcg;
  Fn<decltype(Api<CT>::finish)> finish;
  Fn<decltype(Api<CT>::predicted)> predicted;
  Fn<decltype(Api<CT>::exp)> exp;
  Fn<decltype(Api<CT>::mul)> mul;
  Fn<decltype(Api<CT>::loss)> loss;                       // families 0, 2 and 3 (family 1: Api::loss1)
  long long W, D;
};
template <typename CT, class F> static PgoFns<CT> pgo_fns(long long W, long long D) {
  return {F::linearize, F::node_sums, F::damp_inv, F::pcg, F::finish, F::predicted, F::exp, F::mul, F::loss, W, D};
}

static LmCtl ctl_from(const double* c) {
  LmCtl k;
  k.last = c[0]; k.cached = c[1] != 0.0; k.damping = c[2]; k.pg_down = c[3]; k.reject_count = c[4]; k.reject_limit = c[5];
  k.kind = (int)c[6]; k.high = c[7]; k.low = c[8]; k.up = c[9]; k.self_down = c[10]; k.factor = c[11]; k.smin = c[12];
  k.smax = c[13];
  return k;
}

template <typename CT> static int pgo_step(b200_pgo_step_args* a, void* stream) {
  using A = Api<CT>;
  cudaStream_t s = (cudaStream_t)stream;
  const long long N = a->N, E = a->E;
  const PgoFns<CT> f = a->family == 2   ? pgo_fns<CT, Sim3Api<CT>>(7, 8)
                       : a->family == 3 ? pgo_fns<CT, So3Api<CT>>(3, 4)
                                        : pgo_fns<CT, A>(6, 7);
  const bool reproj2 = a->family == 1;
  CT* nodes = (CT*)a->nodes;
  CT *Mn = (CT*)a->Mn, *un = (CT*)a->un, *Hd = (CT*)a->Hd, *g = (CT*)a->g, *extra = (CT*)a->extra, *Minv = (CT*)a->Minv;
  CT *x = (CT*)a->x, *r = (CT*)a->r, *z = (CT*)a->z, *p0 = (CT*)a->p0, *p1 = (CT*)a->p1, *q = (CT*)a->q, *xbest = (CT*)a->xbest;
  CT *X7 = (CT*)a->X7, *Pt = (CT*)a->Pt;
  volatile double* host = a->host;
  if (!a->retry) {                                       // linearise at the current parameters (kept across rejected trials)
    if (reproj2)
      B200_TRY(A::accum2(nodes, (const CT*)a->pts, (const CT*)a->pix, a->pseg, a->pa, a->pb, a->intr, a->epos_i, a->epos_j, Mn, un,
                         a->ws3, a->robust, a->delta, E, stream));
    else
      B200_TRY(f.linearize(nodes, (const CT*)a->Z, a->ei, a->ej, a->epos_i, a->epos_j, Mn, un, a->ws3, a->robust, a->delta, E, stream));
    B200_TRY(f.node_sums(Mn, un, a->nptr, Hd, g, N, stream));
  }
  B200_TRY(f.damp_inv(Hd, a->scale, a->dmin, a->dmax, (CT*)nullptr, extra, Minv, N, stream));
  // PCG: chunks of iterations without host involvement; after each chunk a one-thread kernel publishes the CG state
  const long long maxiter = a->maxiter > 0 ? a->maxiter : 10 * f.W * N;
  long long it = 0;
  double cgseq = host[32];
  for (;;) {
    long long n = (it == 0 && a->hint > 0) ? a->hint : 8;
    if (n > maxiter - it) n = maxiter - it;
    if (n < 1) n = 1;
    B200_TRY(f.pcg(Mn, a->nother, a->nptr, Minv, extra, g, x, r, z, p0, p1, q, xbest, a->cg, a->ws0, a->tol, maxiter, it, n, N,
                   stream));
    it += n;
    cgseq += 1.0;
    publish_kernel<<<1, 32, 0, s>>>(a->cg, 16, a->host + 16, cgseq);
    B200_TRY((int)cudaGetLastError());
    B200_TRY(spin_until(host + 32, cgseq, s));
    if (host[16 + 5] != 0.0 || it >= maxiter) break;      // done flag of the CG state
  }
  a->iters_out = (long long)host[16 + 6];
  B200_TRY(f.finish(x, xbest, a->cg, N, stream));
  B200_TRY(f.predicted(Mn, a->nother, a->nptr, x, g, a->ws2, N, stream));
  B200_TRY(f.exp(x, X7, N, stream));                     // retraction P' = Exp(D) P  (lietensor.py:442-444)
  B200_TRY(f.mul(X7, nodes, Pt, N, stream));
  if (reproj2) B200_TRY(A::loss1(Pt, (const CT*)a->pts, (const CT*)a->pix, a->pseg, a->pa, a->pb, a->intr, a->ws1, a->robust, a->delta, E, stream));
  else B200_TRY(f.loss(Pt, (const CT*)a->Z, a->ei, a->ej, a->ws1, a->robust, a->delta, E, stream));
  host[ST_SIZE - 1] = -1.0;
  pgo_decide_kernel<<<1, 32, 0, s>>>(a->ws3, a->ws1, a->ws2, ctl_from(a->ctl), a->st, a->host, (double)a->seq);
  commit_kernel<CT><<<lm_grid(N * f.D, kLmThreads), kLmThreads, 0, s>>>(a->st, Pt, nodes, N * f.D);
  B200_TRY((int)cudaGetLastError());
  return spin_until(host + (ST_SIZE - 1), (double)a->seq, s);
}

// ---- bundle adjustment ---------------------------------------------------------------------------------------------
template <typename CT> struct BaApi;
#define B200_BA_API(SFX, CT)                                                                                          \
  template <> struct BaApi<CT> {                                                                                      \
    static constexpr auto linearize = b200_lm_ba_linearize_seg_##SFX;                                                 \
    static constexpr auto point_blocks = b200_lm_ba_point_blocks_##SFX;                                               \
    static constexpr auto damp_inv = b200_lm_blk6_damp_inv_##SFX;                                                     \
    static constexpr auto pt3_inv = b200_lm_pt3_damp_inv_##SFX;                                                       \
    static constexpr auto schur = b200_lm_ba_schur_diag_seg_##SFX;                                                    \
    static constexpr auto wv = b200_lm_ba_wv_seg_##SFX;                                                               \
    static constexpr auto pcg = b200_lm_ba_pcg_##SFX;                                                                 \
    static constexpr auto finish = b200_lm_cg_finish_##SFX;                                                           \
    static constexpr auto wtx = b200_lm_ba_wtx_gather_##SFX;                                                          \
    static constexpr auto predicted = b200_lm_ba_predicted_##SFX;                                                     \
    static constexpr auto exp = b200_se3_exp_fwd_##SFX;                                                               \
    static constexpr auto mul = b200_SE3_mul_fwd_##SFX;                                                               \
    static constexpr auto loss = b200_lm_ba_loss_##SFX;                                                               \
  };
B200_BA_API(f32, float)
B200_BA_API(f64, double)

template <typename T>
__global__ void __launch_bounds__(kLmThreads) add_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ o,
                                                          long long n) {
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads)
    o[i] = a[i] + b[i];
}
template <typename T>
__global__ void __launch_bounds__(kLmThreads) commit2_kernel(const double* __restrict__ st, const T* __restrict__ s0,
                                                              T* __restrict__ d0, long long n0, const T* __restrict__ s1,
                                                              T* __restrict__ d1, long long n1) {
  if (st[ST_STATUS] != 1.0) return;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n0 + n1; i += (long long)gridDim.x * kLmThreads) {
    if (i < n0) d0[i] = s0[i];
    else d1[i - n0] = s1[i - n0];
  }
}

template <typename CT> static int ba_step(b200_ba_step_args* a, void* stream) {
  using A = BaApi<CT>;
  cudaStream_t s = (cudaStream_t)stream;
  const long long C = a->C, P = a->P, m = a->m;
  CT *poses = (CT*)a->poses, *points = (CT*)a->points;
  const CT* pix = (const CT*)a->pix;
  CT *Y4 = (CT*)a->Y4, *Y4p = (CT*)a->Y4p, *rs = (CT*)a->rs, *Hcc = (CT*)a->Hcc, *gc = (CT*)a->gc, *Hpp = (CT*)a->Hpp;
  CT *gp = (CT*)a->gp, *part = (CT*)a->part, *Hc = (CT*)a->Hc, *Hpinv = (CT*)a->Hpinv, *Minv = (CT*)a->Minv, *Sd = (CT*)a->Sd;
  CT *bneg = (CT*)a->bneg, *x = (CT*)a->x, *r = (CT*)a->r, *z = (CT*)a->z, *p = (CT*)a->p, *q = (CT*)a->q, *t = (CT*)a->t;
  CT *xbest = (CT*)a->xbest, *xp = (CT*)a->xp, *X7 = (CT*)a->X7, *Tn = (CT*)a->Tn, *pn = (CT*)a->pn;
  volatile double* host = a->host;
  if (!a->retry) {
    B200_TRY(A::linearize(poses, points, pix, a->pidx, a->cseg, a->split, a->tpi, Y4, a->ppos, Y4p, rs, Hcc, gc, part, a->ws3,
                          a->robust, a->delta, C, stream));
    B200_TRY(A::point_blocks(Y4p, (const CT*)a->pix_p, poses, a->cidx_p, a->pptr, Hpp, gp, P, stream));
  }
  B200_TRY(A::damp_inv(Hcc, a->scale, a->dmin, a->dmax, Hc, (CT*)nullptr, (CT*)nullptr, C, stream));
  B200_TRY(A::pt3_inv(Hpp, a->scale, a->dmin, a->dmax, Hpinv, P, stream));
  B200_TRY((int)cudaMemcpyAsync(Sd, Hc, sizeof(CT) * 21 * C, cudaMemcpyDeviceToDevice, s));
  B200_TRY(A::schur(Y4, poses, a->pidx, a->cseg, a->split, a->tpi, Hpinv, Sd, part, C, stream));
  B200_TRY(A::damp_inv(Sd, 1.0, -3.0e38, 3.0e38, (CT*)nullptr, (CT*)nullptr, Minv, C, stream));
  B200_TRY((int)cudaMemcpyAsync(bneg, gc, sizeof(CT) * 6 * C, cudaMemcpyDeviceToDevice, s));      // -(rhs) = gc - W Hpp^-1 gp
  B200_TRY(A::wv(Y4, poses, a->pidx, a->cseg, a->split, a->tpi, Hpinv, gp, bneg, part, C, stream));
  const long long maxiter = a->maxiter > 0 ? a->maxiter : 10 * 6 * C;
  long long it = 0;
  double cgseq = host[32];
  for (;;) {
    long long n = (it == 0 && a->hint > 0) ? a->hint : 8;
    if (n > maxiter - it) n = maxiter - it;
    if (n < 1) n = 1;
    B200_TRY(A::pcg(Y4, poses, a->pidx, a->cseg, a->split, a->tpi, m, Y4p, a->cidx_p, a->pptr, Hc, Hpinv, Minv, bneg, x, r, z, p, q,
                    t, part, xbest, a->cg, a->ws0, a->tol, maxiter, P, it, n, (const unsigned long long*)nullptr, 0, 1, 0, 0, 0,
                    (unsigned*)nullptr, C, stream));
    it += n;
    cgseq += 1.0;
    publish_kernel<<<1, 32, 0, s>>>(a->cg, 16, a->host + 16, cgseq);
    B200_TRY((int)cudaGetLastError());
    B200_TRY(spin_until(host + 32, cgseq, s));
    if (host[16 + 5] != 0.0 || it >= maxiter) break;
  }
  a->iters_out = (long long)host[16 + 6];
  B200_TRY(A::finish(x, xbest, a->cg, C, stream));
  B200_TRY(A::wtx(Y4p, poses, a->cidx_p, a->pptr, Hpinv, x, gp, -1.0, xp, P, stream));            // dp = -Hpp^-1 (gp + W^T dc)
  B200_TRY(A::predicted(Y4, poses, rs, a->cidx, a->pidx, x, xp, a->ws2, m, stream));
  B200_TRY(A::exp(x, X7, C, stream));
  B200_TRY(A::mul(X7, poses, Tn, C, stream));
  add_kernel<CT><<<lm_grid(P * 3, kLmThreads), kLmThreads, 0, s>>>(points, xp, pn, P * 3);
  B200_TRY(A::loss(Tn, pn, pix, a->cidx, a->pidx, a->ws1, a->robust, a->delta, m, stream));
  host[ST_SIZE - 1] = -1.0;
  pgo_decide_kernel<<<1, 32, 0, s>>>(a->ws3, a->ws1, a->ws2, ctl_from(a->ctl), a->st, a->host, (double)a->seq);
  commit2_kernel<CT><<<lm_grid(C * 7 + P * 3, kLmThreads), kLmThreads, 0, s>>>(a->st, Tn, poses, C * 7, pn, points, P * 3);
  B200_TRY((int)cudaGetLastError());
  return spin_until(host + (ST_SIZE - 1), (double)a->seq, s);
}

}  // namespace b200pose

B200_EXPORT int b200_lm_ba_step(b200_ba_step_args* args, void* stream) {
  if (!args || args->C <= 0) return 0;
  return args->is64 ? b200pose::ba_step<double>(args, stream) : b200pose::ba_step<float>(args, stream);
}
B200_EXPORT long long b200_ba_step_args_size(void) { return (long long)sizeof(b200_ba_step_args); }

B200_EXPORT int b200_lm_pgo2_step(b200_pgo_step_args* args, void* stream) {
  if (!args || args->N <= 0) return 0;
  if (args->family < 0 || args->family > 3) return (int)cudaErrorInvalidValue;
  return args->is64 ? b200pose::pgo_step<double>(args, stream) : b200pose::pgo_step<float>(args, stream);
}
B200_EXPORT long long b200_pgo_step_args_size(void) { return (long long)sizeof(b200_pgo_step_args); }
