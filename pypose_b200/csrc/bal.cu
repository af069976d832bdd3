// bal.cu — bundle adjustment of BAL problems (per-camera f, k1, k2 optimised with poses and points) without atomics
// (C-ABI: include/b200pose.h, section LM).
//
// The camera-side structure of ba.cu at block width 9 (unknowns [xi | f, k1, k2] per camera, bal_math.cuh): every sum
// has ONE writer and a fixed order — per-camera work items (lm_seg.cuh) reduced by a fixed shuffle tree and folded in
// item order, point blocks and W^T x by gather over a point-ordered copy of the per-observation data.  Per observation
// the linearisation keeps 16 B (Y4 = y = T_c p and sqrt(rho')) in camera order and in point order plus the scaled
// residual; every later kernel rebuilds the 2x9 / 2x3 Jacobian rows from Y4, the camera's rotation and its intrinsics.
//
// Reference semantics: the J^T J / J^T R sums of optimizer.py:645-656 for the three-parameter model of
// examples/module/ba/bundle_adjustment.py (`Reproj(K, C, P)`), retraction lietensor.py:442-444 (poses) and plain
// addition (intrinsics, points).
#include "lm_common.cuh"
#include "lm_seg.cuh"
#include "pcg_vec.cuh"

namespace b200pose {

template <typename T> struct CamK { Q4<T> q; T f, k1, k2; };
template <typename T> __device__ __forceinline__ CamK<T> load_camk(const T* __restrict__ poses, const T* __restrict__ intr,
                                                                    long long c) {
  CamK<T> k;
  k.q.v = mk(__ldg(poses + c * 7 + 3), __ldg(poses + c * 7 + 4), __ldg(poses + c * 7 + 5));
  k.q.w = __ldg(poses + c * 7 + 6);
  k.f = __ldg(intr + c * 3); k.k1 = __ldg(intr + c * 3 + 1); k.k2 = __ldg(intr + c * 3 + 2);
  return k;
}
template <typename T> __device__ __forceinline__ V3<T> y4_point(const T* __restrict__ Y4, long long k, T& sw) {
  const long long k4 = k * 4;
  sw = Y4[k4 + 3];
  return mk(Y4[k4], Y4[k4 + 1], Y4[k4 + 2]);
}

// Linearisation: per observation y = T_c p_j, residual, robust scale; stores Y4 (camera order), Y4p (point order) and the
// scaled residual; per item the 45 + 9 camera sums.  ws[0] = sum rho(|r|^2).
constexpr int kBalCamSums = kBalCamPacked + kBalCam;
template <typename T, int TPI>
__global__ void __launch_bounds__(kLmThreads) bal_linearize_seg_kernel(
    const T* __restrict__ poses, const T* __restrict__ intr, const T* __restrict__ points, const T* __restrict__ pix,
    const int* __restrict__ pidx, const int* __restrict__ cseg, int S, T* __restrict__ Y4, const int* __restrict__ ppos,
    T* __restrict__ Y4p, T* __restrict__ rs, T* __restrict__ Hcc, T* __restrict__ gc, T* __restrict__ part, double* ws,
    int rk, T rdelta, long long C) {
  constexpr int IPB = kLmThreads / TPI;
  __shared__ T sh[TPI > 32 ? TPI / 32 : 1][kBalCamSums];
  const int sub = threadIdx.x % TPI;
  const long long items = C * S, rounds = (items + IPB - 1) / IPB;
  double acc[1] = {0.0};
  for (long long rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const long long it = rd * IPB + threadIdx.x / TPI;
    T cam[kBalCamSums];
#pragma unroll
    for (int a = 0; a < kBalCamSums; ++a) cam[a] = T(0);
    ItemRange r = {0, 0, 0};
    if (it < items) {
      r = item_range(it, S, cseg);
      T pr[7];
#pragma unroll
      for (int q = 0; q < 7; ++q) pr[q] = __ldg(poses + r.c * 7 + q);
      const Elem<T> Tc = load_se3(pr);
      const T f = __ldg(intr + r.c * 3), k1 = __ldg(intr + r.c * 3 + 1), k2 = __ldg(intr + r.c * 3 + 2);
      for (int k = r.b + sub; k < r.e; k += TPI) {
        const long long j = pidx[k];
        const V3<T> p = mk(__ldg(points + j * 3), __ldg(points + j * 3 + 1), __ldg(points + j * 3 + 2));
        T rx, ry;
        V3<T> y;
        bal_residual(Tc, p, f, k1, k2, pix[(long long)k * 2], pix[(long long)k * 2 + 1], rx, ry, y);
        T rho, w;
        robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
        const T sw = rk ? m_sqrt(w) : T(1);
        rx *= sw; ry *= sw;
        BalRows<T> R;
        bal_rows(y, Tc.q, f, k1, k2, sw, R);
        const long long k4 = (long long)k * 4;
        Y4[k4] = y.x; Y4[k4 + 1] = y.y; Y4[k4 + 2] = y.z; Y4[k4 + 3] = sw;
        if (Y4p) {
          const long long s4 = (long long)ppos[k] * 4;
          Y4p[s4] = y.x; Y4p[s4 + 1] = y.y; Y4p[s4 + 2] = y.z; Y4p[s4 + 3] = sw;
        }
        rs[(long long)k * 2] = rx; rs[(long long)k * 2 + 1] = ry;
#pragma unroll
        for (int a = 0; a < kBalCam; ++a) cam[kBalCamPacked + a] += R.jc0[a] * rx + R.jc1[a] * ry;
        sym9_add_rows(cam, R.jc0, R.jc1);
        acc[0] += (double)rho;
      }
    }
    item_reduce<T, kBalCamSums, TPI>(cam, sh);
    if (it < items && sub == 0) {
      if (S == 1) {
#pragma unroll
        for (int a = 0; a < kBalCamPacked; ++a) Hcc[r.c * kBalCamPacked + a] = cam[a];
#pragma unroll
        for (int a = 0; a < kBalCam; ++a) gc[r.c * kBalCam + a] = cam[kBalCamPacked + a];
      } else {
#pragma unroll
        for (int a = 0; a < kBalCamSums; ++a) part[it * kBalCamSums + a] = cam[a];
      }
    }
  }
  reduce_sums<1>(acc, ws);
}

// Point blocks Hpp (6) and gp (3) by gather over the point-ordered rows: LPP lanes per point, fixed shuffle tree.
constexpr int kBalLanesPerPoint = 8;
template <typename T>
__global__ void __launch_bounds__(kLmThreads) bal_point_blocks_kernel(const T* __restrict__ Y4p, const T* __restrict__ pix_p,
                                                                       const T* __restrict__ poses, const T* __restrict__ intr,
                                                                       const int* __restrict__ cidx_p,
                                                                       const int* __restrict__ pptr, T* __restrict__ Hpp,
                                                                       T* __restrict__ gp, long long P) {
  constexpr int LPP = kBalLanesPerPoint, PPB = kLmThreads / LPP;
  const int sub = threadIdx.x % LPP;
  const long long groups = (P + PPB - 1) / PPB;
  for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
    const long long j = g * PPB + threadIdx.x / LPP;
    T a[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) a[k] = T(0);
    if (j < P)
      for (int s = pptr[j] + sub; s < pptr[j + 1]; s += LPP) {
        const CamK<T> K = load_camk(poses, intr, cidx_p[s]);
        T sw;
        const V3<T> y = y4_point(Y4p, s, sw);
        BalRows<T> R;
        bal_rows(y, K.q, K.f, K.k1, K.k2, sw, R);
        T rx, ry;
        bal_residual_y(y, K.f, K.k1, K.k2, pix_p[(long long)s * 2], pix_p[(long long)s * 2 + 1], rx, ry);
        rx *= sw; ry *= sw;
        int t = 0;
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          a[6 + u] += R.jp0[u] * rx + R.jp1[u] * ry;
#pragma unroll
          for (int v = u; v < 3; ++v) a[t++] += R.jp0[u] * R.jp0[v] + R.jp1[u] * R.jp1[v];
        }
      }
#pragma unroll
    for (int o = LPP / 2; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < 9; ++k) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    if (j < P && sub == 0) {
#pragma unroll
      for (int k = 0; k < 6; ++k) Hpp[j * 6 + k] = a[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) gp[j * 3 + k] = a[6 + k];
    }
  }
}

// y[c] -= sum_{k in c} Jc_k^T Jp_k (Hp^-1) t[j_k]      (W Hpp^-1 t of the reduced camera system; one writer per camera)
template <typename T, int TPI>
__global__ void __launch_bounds__(kLmThreads) bal_wv_seg_kernel(const T* __restrict__ Y4, const T* __restrict__ poses,
                                                                 const T* __restrict__ intr, const int* __restrict__ pidx,
                                                                 const int* __restrict__ cseg, int S,
                                                                 const T* __restrict__ Hpinv, const T* __restrict__ t,
                                                                 T* __restrict__ y, T* __restrict__ part, const double* cg,
                                                                 long long C) {
  if (cg && cg[CG_DONE] != 0.0) return;
  constexpr int IPB = kLmThreads / TPI;
  __shared__ T sh[TPI > 32 ? TPI / 32 : 1][kBalCam];
  const int sub = threadIdx.x % TPI;
  const long long items = C * S, rounds = (items + IPB - 1) / IPB;
  for (long long rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const long long it = rd * IPB + threadIdx.x / TPI;
    T out[kBalCam];
#pragma unroll
    for (int a = 0; a < kBalCam; ++a) out[a] = T(0);
    ItemRange r = {0, 0, 0};
    if (it < items) {
      r = item_range(it, S, cseg);
      const CamK<T> K = load_camk(poses, intr, r.c);
      for (int k = r.b + sub; k < r.e; k += TPI) {
        const long long j = pidx[k];
        const T t0 = __ldg(t + j * 3), t1 = __ldg(t + j * 3 + 1), t2 = __ldg(t + j * 3 + 2);
        T v[3] = {t0, t1, t2};
        if (Hpinv) {
          T A[3][3], h[6];
#pragma unroll
          for (int a = 0; a < 6; ++a) h[a] = __ldg(Hpinv + j * 6 + a);
          sym3_unpack(h, A);
#pragma unroll
          for (int a = 0; a < 3; ++a) v[a] = A[a][0] * t0 + A[a][1] * t1 + A[a][2] * t2;
        }
        T sw;
        const V3<T> yv = y4_point(Y4, k, sw);
        BalRows<T> R;
        bal_rows(yv, K.q, K.f, K.k1, K.k2, sw, R);
        T u0 = T(0), u1 = T(0);
#pragma unroll
        for (int a = 0; a < 3; ++a) { u0 += R.jp0[a] * v[a]; u1 += R.jp1[a] * v[a]; }
#pragma unroll
        for (int a = 0; a < kBalCam; ++a) out[a] -= R.jc0[a] * u0 + R.jc1[a] * u1;
      }
    }
    item_reduce<T, kBalCam, TPI>(out, sh);
    if (it < items && sub == 0) {
      if (S == 1) {
#pragma unroll
        for (int a = 0; a < kBalCam; ++a) y[r.c * kBalCam + a] += out[a];
      } else {
#pragma unroll
        for (int a = 0; a < kBalCam; ++a) part[it * kBalCam + a] = out[a];
      }
    }
  }
}

// Sd[c] -= sum_k (Jc^T Jp) Hp^-1 (Jp^T Jc)   (diagonal blocks of the Schur complement; Sd pre-set to the damped Hcc)
template <typename T, int TPI>
__global__ void __launch_bounds__(kLmThreads) bal_schur_diag_seg_kernel(const T* __restrict__ Y4, const T* __restrict__ poses,
                                                                         const T* __restrict__ intr,
                                                                         const int* __restrict__ pidx,
                                                                         const int* __restrict__ cseg, int S,
                                                                         const T* __restrict__ Hpinv, T* __restrict__ Sd,
                                                                         T* __restrict__ part, long long C) {
  constexpr int IPB = kLmThreads / TPI;
  __shared__ T sh[TPI > 32 ? TPI / 32 : 1][kBalCamPacked];
  const int sub = threadIdx.x % TPI;
  const long long items = C * S, rounds = (items + IPB - 1) / IPB;
  for (long long rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const long long it = rd * IPB + threadIdx.x / TPI;
    T out[kBalCamPacked];
#pragma unroll
    for (int a = 0; a < kBalCamPacked; ++a) out[a] = T(0);
    ItemRange r = {0, 0, 0};
    if (it < items) {
      r = item_range(it, S, cseg);
      const CamK<T> K = load_camk(poses, intr, r.c);
      for (int k = r.b + sub; k < r.e; k += TPI) {
        const long long j = pidx[k];
        T A[3][3], h[6];
#pragma unroll
        for (int a = 0; a < 6; ++a) h[a] = __ldg(Hpinv + j * 6 + a);
        sym3_unpack(h, A);
        T sw;
        const V3<T> yv = y4_point(Y4, k, sw);
        BalRows<T> R;
        bal_rows(yv, K.q, K.f, K.k1, K.k2, sw, R);
        // G = Jp Hp^-1 Jp^T (2x2), then T_k = Jc^T G Jc
        T B0[3], B1[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          B0[a] = R.jp0[0] * A[0][a] + R.jp0[1] * A[1][a] + R.jp0[2] * A[2][a];
          B1[a] = R.jp1[0] * A[0][a] + R.jp1[1] * A[1][a] + R.jp1[2] * A[2][a];
        }
        const T g00 = B0[0] * R.jp0[0] + B0[1] * R.jp0[1] + B0[2] * R.jp0[2];
        const T g01 = B0[0] * R.jp1[0] + B0[1] * R.jp1[1] + B0[2] * R.jp1[2];
        const T g11 = B1[0] * R.jp1[0] + B1[1] * R.jp1[1] + B1[2] * R.jp1[2];
        int qq = 0;
#pragma unroll
        for (int a = 0; a < kBalCam; ++a) {
          const T l0 = R.jc0[a] * g00 + R.jc1[a] * g01, l1 = R.jc0[a] * g01 + R.jc1[a] * g11;
#pragma unroll
          for (int b = a; b < kBalCam; ++b) out[qq++] -= l0 * R.jc0[b] + l1 * R.jc1[b];
        }
      }
    }
    item_reduce<T, kBalCamPacked, TPI>(out, sh);
    if (it < items && sub == 0) {
      if (S == 1) {
#pragma unroll
        for (int a = 0; a < kBalCamPacked; ++a) Sd[r.c * kBalCamPacked + a] += out[a];
      } else {
#pragma unroll
        for (int a = 0; a < kBalCamPacked; ++a) part[it * kBalCamPacked + a] = out[a];
      }
    }
  }
}

// u[j] = alpha * Hp^-1_j (t0[j] + sum_{k in obs(j)} Jp_k^T Jc_k x[c_k])   — W^T x by gather over the point-ordered rows
template <typename T>
__global__ void __launch_bounds__(kLmThreads) bal_wtx_gather_kernel(const T* __restrict__ Y4p, const T* __restrict__ poses,
                                                                     const T* __restrict__ intr,
                                                                     const int* __restrict__ cidx_p,
                                                                     const int* __restrict__ pptr, const T* __restrict__ Hpinv,
                                                                     const T* __restrict__ x, const T* __restrict__ t0,
                                                                     T alpha, T* __restrict__ u, const double* cg,
                                                                     long long P) {
  if (cg && cg[CG_DONE] != 0.0) return;
  constexpr int LPP = kBalLanesPerPoint, PPB = kLmThreads / LPP;
  const int sub = threadIdx.x % LPP;
  const long long groups = (P + PPB - 1) / PPB;       // warp-uniform trip count (the shuffles need all 32 lanes)
  for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
    const long long j = g * PPB + threadIdx.x / LPP;
    T t[3] = {T(0), T(0), T(0)};
    if (j < P) {
      const int lo = pptr[j], hi = pptr[j + 1];
      for (int s = lo + sub; s < hi; s += LPP) {
        const long long c = cidx_p[s];
        const CamK<T> K = load_camk(poses, intr, c);
        T sw;
        const V3<T> y = y4_point(Y4p, s, sw);
        BalRows<T> R;
        bal_rows(y, K.q, K.f, K.k1, K.k2, sw, R);
        T v0 = T(0), v1 = T(0);
#pragma unroll
        for (int a = 0; a < kBalCam; ++a) {
          const T xa = __ldg(x + c * kBalCam + a);
          v0 += R.jc0[a] * xa; v1 += R.jc1[a] * xa;
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) t[a] += R.jp0[a] * v0 + R.jp1[a] * v1;
      }
    }
#pragma unroll
    for (int o = LPP / 2; o > 0; o >>= 1)
#pragma unroll
      for (int a = 0; a < 3; ++a) t[a] += __shfl_xor_sync(0xffffffffu, t[a], o);
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
__global__ void __launch_bounds__(kLmThreads) bal_predicted_kernel(const T* __restrict__ Y4, const T* __restrict__ poses,
                                                                    const T* __restrict__ intr, const T* __restrict__ rs,
                                                                    const int* __restrict__ cidx, const int* __restrict__ pidx,
                                                                    const T* __restrict__ xc, const T* __restrict__ xp,
                                                                    double* ws, long long m) {
  double acc[1] = {0.0};
  for (long long k = (long long)blockIdx.x * kLmThreads + threadIdx.x; k < m; k += (long long)gridDim.x * kLmThreads) {
    const long long c = cidx[k], j = pidx[k];
    const CamK<T> K = load_camk(poses, intr, c);
    T sw;
    const V3<T> y = y4_point(Y4, k, sw);
    BalRows<T> R;
    bal_rows(y, K.q, K.f, K.k1, K.k2, sw, R);
    T d0 = T(0), d1 = T(0);
#pragma unroll
    for (int a = 0; a < kBalCam; ++a) { const T v = __ldg(xc + c * kBalCam + a); d0 += R.jc0[a] * v; d1 += R.jc1[a] * v; }
#pragma unroll
    for (int a = 0; a < 3; ++a) { const T v = __ldg(xp + j * 3 + a); d0 += R.jp0[a] * v; d1 += R.jp1[a] * v; }
    acc[0] += (double)(d0 * (T(2) * rs[k * 2] + d0) + d1 * (T(2) * rs[k * 2 + 1] + d1));
  }
  reduce_sums<1>(acc, ws);
}

// ws[0] = sum_k rho(|r_k|^2) at the given parameters (the loss of RobustModel, optimizer.py:118-125)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) bal_loss_kernel(const T* __restrict__ poses, const T* __restrict__ intr,
                                                               const T* __restrict__ points, const T* __restrict__ pix,
                                                               const int* __restrict__ cidx, const int* __restrict__ pidx,
                                                               double* ws, int rk, T rdelta, long long m) {
  double acc[1] = {0.0};
  for (long long k = (long long)blockIdx.x * kLmThreads + threadIdx.x; k < m; k += (long long)gridDim.x * kLmThreads) {
    const long long c = cidx[k], j = pidx[k];
    T pr[7];
#pragma unroll
    for (int q = 0; q < 7; ++q) pr[q] = __ldg(poses + c * 7 + q);
    const Elem<T> Tc = load_se3(pr);
    const V3<T> p = mk(__ldg(points + j * 3), __ldg(points + j * 3 + 1), __ldg(points + j * 3 + 2));
    T rx, ry;
    V3<T> y;
    bal_residual(Tc, p, __ldg(intr + c * 3), __ldg(intr + c * 3 + 1), __ldg(intr + c * 3 + 2), pix[k * 2], pix[k * 2 + 1],
                 rx, ry, y);
    T rho, w;
    robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
    acc[0] += (double)rho;
  }
  reduce_sums<1>(acc, ws);
}

// trial parameters: T' = Exp(xi) T, K' = K + dK (cameras), p' = p + dp (points)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) bal_retract_kernel(const T* __restrict__ poses, const T* __restrict__ intr,
                                                                  const T* __restrict__ points, const T* __restrict__ xc,
                                                                  const T* __restrict__ xp, T* __restrict__ poses_t,
                                                                  T* __restrict__ intr_t, T* __restrict__ points_t,
                                                                  long long C, long long P) {
  const long long n = C > P ? C : P;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    if (i < C) {
      T D[6];
#pragma unroll
      for (int a = 0; a < 6; ++a) D[a] = xc[i * kBalCam + a];
      T pr[7];
#pragma unroll
      for (int q = 0; q < 7; ++q) pr[q] = poses[i * 7 + q];
      store_elem<SE3g, T>(poses_t + i * 7, se3_retract(D, load_se3(pr)));
#pragma unroll
      for (int a = 0; a < 3; ++a) intr_t[i * 3 + a] = intr[i * 3 + a] + xc[i * kBalCam + 6 + a];
    }
    if (i < P) {
#pragma unroll
      for (int a = 0; a < 3; ++a) points_t[i * 3 + a] = points[i * 3 + a] + xp[i * 3 + a];
    }
  }
}

// diag <- clamp(diag, dmin, dmax) * scale of packed 9x9 camera blocks; optional outputs: the damped block, its inverse
template <typename T>
__global__ void __launch_bounds__(kLmThreads) blk9_damp_inv_kernel(const T* __restrict__ H, T scale, T dmin, T dmax,
                                                                    T* __restrict__ Hd, T* __restrict__ Minv, long long n) {
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T A[9][9], Ai[9][9];
    symn_unpack<T, 9>(H + i * kBalCamPacked, A);
    blk9_damp(A, scale, dmin, dmax);
    if (Hd) symn_pack<T, 9>(A, Hd + i * kBalCamPacked);
    if (Minv) { spd_inverse<T, 9>(A, Ai); symn_pack<T, 9>(Ai, Minv + i * kBalCamPacked); }
  }
}

// ---- reduced-camera PCG: the pcg_vec.cuh kernels at block width 9 --------------------------------------------------
template <typename T>
static void launch_cg9_vec_small(const T* Minv, const T* D, int dmode, T* x, T* r, T* z, T* p, T* q, T* xbest, double* cg,
                                 int par, long long n, cudaStream_t st) {
  // at most 512 threads: 1024 would cap a thread at 64 registers, below what a 9-wide fp64 row needs (spills)
  if (n <= 2048) cg_vec_small_kernel<T, 256, kBalCam><<<1, 256, 0, st>>>(Minv, D, dmode, x, r, z, p, q, xbest, cg, par, n);
  else cg_vec_small_kernel<T, 512, kBalCam><<<1, 512, 0, st>>>(Minv, D, dmode, x, r, z, p, q, xbest, cg, par, n);
}

template <typename CT>
static int bal_wv_seg_launch(const CT* Y4, const CT* poses, const CT* intr, const int* pidx, const int* cseg, int S,
                             int tpi, const CT* Hpinv, const CT* t, CT* y, CT* part, const double* cg, long long C,
                             cudaStream_t st) {
  const unsigned grid = item_grid(C * S, tpi);
  if (tpi == 32)
    bal_wv_seg_kernel<CT, 32><<<grid, kLmThreads, 0, st>>>(Y4, poses, intr, pidx, cseg, S, Hpinv, t, y, part, cg, C);
  else
    bal_wv_seg_kernel<CT, 128><<<grid, kLmThreads, 0, st>>>(Y4, poses, intr, pidx, cseg, S, Hpinv, t, y, part, cg, C);
  if (S > 1)
    cam_fold_kernel<CT><<<lm_grid(C * kBalCam, kLmThreads), kLmThreads, 0, st>>>(part, S, kBalCam, 0, y, (CT*)nullptr, 1,
                                                                                   cg, C);
  return (int)cudaGetLastError();
}

#define BAL_LAUNCH(kern, work, st, ...) kern<<<lm_grid(work, kLmThreads), kLmThreads, 0, (cudaStream_t)(st)>>>(__VA_ARGS__)

// Iterations [first_iter, first_iter + iters) of the reduced-camera PCG: q = Hc p - W Hpp^-1 W^T p, then the vector
// kernels of pcg_vec.cuh at width 9 (one single-CTA kernel up to kVecSmallRows cameras).
template <typename CT>
static int bal_pcg_run(const CT* Y4, const CT* poses, const CT* intr, const int* pidx, const int* cseg, long long split,
                       long long tpi, long long m, const CT* Y4p, const int* cidx_p, const int* pptr, const CT* Hc,
                       const CT* Hpinv, const CT* Minv, const CT* bneg, CT* x, CT* r, CT* z, CT* p, CT* q, CT* t, CT* part,
                       CT* xbest, double* cg, double* ws, double tol, long long maxiter, long long P, long long first_iter,
                       long long iters, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  const unsigned vg = lm_grid(n, kLmThreads);
  if (first_iter == 0)
    cg_init_kernel<CT, kBalCam><<<vg, kLmThreads, 0, stream>>>(Minv, bneg, (CT)-1, Hc, 2, x, r, p, q, cg, ws, tol,
                                                                (double)maxiter, n);
  for (long long it = first_iter; it < first_iter + iters; ++it) {
    const int par = (int)(it & 1);
    if (m > 0) {
      BAL_LAUNCH(bal_wtx_gather_kernel<CT>, P * kBalLanesPerPoint, stream, Y4p, poses, intr, cidx_p, pptr, Hpinv, p,
                 (const CT*)nullptr, (CT)1, t, cg, P);
      bal_wv_seg_launch<CT>(Y4, poses, intr, pidx, cseg, (int)split, (int)tpi, (const CT*)nullptr, t, q, part, cg, n, stream);
    }
    if (n <= kVecSmallRows) {
      launch_cg9_vec_small<CT>(Minv, Hc, 2, x, r, z, p, q, xbest, cg, par, n, stream);
      continue;
    }
    cg_dot_kernel<CT, kBalCam><<<vg, kLmThreads, 0, stream>>>(p, q, cg, ws, n);
    cg_update_kernel<CT, kBalCam><<<vg, kLmThreads, 0, stream>>>(Minv, p, q, x, r, z, xbest, cg, ws, par, n);
    cg_dir_kernel<CT, kBalCam><<<vg, kLmThreads, 0, stream>>>(z, Hc, 2, p, q, cg, par, n);
  }
  return (int)cudaGetLastError();
}

}  // namespace b200pose

using namespace b200pose;

#define BAL_ABI(SFX, CT)                                                                                              \
  B200_EXPORT int b200_lm_bal_linearize_seg_##SFX(const CT* poses, const CT* intr, const CT* points, const CT* pix,   \
                                                  const int* pidx, const int* cseg, long long split, long long tpi,   \
                                                  CT* Y4, const int* ppos, CT* Y4p, CT* rs, CT* Hcc, CT* gc,          \
                                                  CT* part, double* ws, int robust, double delta, long long C,        \
                                                  void* stream) {                                                     \
    if (C <= 0) return 0;                                                                                             \
    cudaStream_t st = (cudaStream_t)stream;                                                                           \
    const int S = (int)split;                                                                                         \
    const unsigned grid = item_grid(C * S, (int)tpi);                                                                 \
    if (tpi == 32)                                                                                                    \
      bal_linearize_seg_kernel<CT, 32><<<grid, kLmThreads, 0, st>>>(poses, intr, points, pix, pidx, cseg, S, Y4,      \
                                                                    ppos, Y4p, rs, Hcc, gc, part, ws, robust,         \
                                                                    (CT)delta, C);                                    \
    else                                                                                                              \
      bal_linearize_seg_kernel<CT, 128><<<grid, kLmThreads, 0, st>>>(poses, intr, points, pix, pidx, cseg, S, Y4,     \
                                                                     ppos, Y4p, rs, Hcc, gc, part, ws, robust,        \
                                                                     (CT)delta, C);                                   \
    if (S > 1)                                                                                                        \
      cam_fold_kernel<CT><<<lm_grid(C * kBalCamSums, kLmThreads), kLmThreads, 0, st>>>(                               \
          part, S, kBalCamPacked, kBalCam, Hcc, gc, 0, (const double*)nullptr, C);                                    \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_point_blocks_##SFX(const CT* Y4p, const CT* pix_p, const CT* poses, const CT* intr,     \
                                                 const int* cidx_p, const int* pptr, CT* Hpp, CT* gp, long long P,    \
                                                 void* stream) {                                                      \
    if (P <= 0) return 0;                                                                                             \
    BAL_LAUNCH(bal_point_blocks_kernel<CT>, P * kBalLanesPerPoint, stream, Y4p, pix_p, poses, intr, cidx_p, pptr,     \
               Hpp, gp, P);                                                                                           \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_wv_seg_##SFX(const CT* Y4, const CT* poses, const CT* intr, const int* pidx,            \
                                           const int* cseg, long long split, long long tpi, const CT* Hpinv,          \
                                           const CT* t, CT* y, CT* part, long long C, void* stream) {                 \
    if (C <= 0) return 0;                                                                                             \
    return bal_wv_seg_launch<CT>(Y4, poses, intr, pidx, cseg, (int)split, (int)tpi, Hpinv, t, y, part,                \
                                 (const double*)nullptr, C, (cudaStream_t)stream);                                    \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_schur_diag_seg_##SFX(const CT* Y4, const CT* poses, const CT* intr, const int* pidx,    \
                                                   const int* cseg, long long split, long long tpi, const CT* Hpinv,  \
                                                   CT* Sd, CT* part, long long C, void* stream) {                     \
    if (C <= 0) return 0;                                                                                             \
    cudaStream_t st = (cudaStream_t)stream;                                                                           \
    const int S = (int)split;                                                                                         \
    const unsigned grid = item_grid(C * S, (int)tpi);                                                                 \
    if (tpi == 32)                                                                                                    \
      bal_schur_diag_seg_kernel<CT, 32><<<grid, kLmThreads, 0, st>>>(Y4, poses, intr, pidx, cseg, S, Hpinv, Sd,       \
                                                                     part, C);                                        \
    else                                                                                                              \
      bal_schur_diag_seg_kernel<CT, 128><<<grid, kLmThreads, 0, st>>>(Y4, poses, intr, pidx, cseg, S, Hpinv, Sd,      \
                                                                      part, C);                                       \
    if (S > 1)                                                                                                        \
      cam_fold_kernel<CT><<<lm_grid(C * kBalCamPacked, kLmThreads), kLmThreads, 0, st>>>(                             \
          part, S, kBalCamPacked, 0, Sd, (CT*)nullptr, 1, (const double*)nullptr, C);                                 \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_wtx_gather_##SFX(const CT* Y4p, const CT* poses, const CT* intr, const int* cidx_p,     \
                                               const int* pptr, const CT* Hpinv, const CT* x, const CT* t0,           \
                                               double alpha, CT* u, long long P, void* stream) {                      \
    if (P <= 0) return 0;                                                                                             \
    BAL_LAUNCH(bal_wtx_gather_kernel<CT>, P * kBalLanesPerPoint, stream, Y4p, poses, intr, cidx_p, pptr, Hpinv, x,    \
               t0, (CT)alpha, u, (const double*)nullptr, P);                                                          \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_damp_inv_##SFX(const CT* H, double scale, double dmin, double dmax, CT* Hd, CT* Minv,   \
                                             long long n, void* stream) {                                             \
    if (n <= 0) return 0;                                                                                             \
    BAL_LAUNCH(blk9_damp_inv_kernel<CT>, n, stream, H, (CT)scale, (CT)dmin, (CT)dmax, Hd, Minv, n);                   \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_pcg_##SFX(const CT* Y4, const CT* poses, const CT* intr, const int* pidx,               \
                                        const int* cseg, long long split, long long tpi, long long m, const CT* Y4p,  \
                                        const int* cidx_p, const int* pptr, const CT* Hc, const CT* Hpinv,            \
                                        const CT* Minv, const CT* bneg, CT* x, CT* r, CT* z, CT* p, CT* q, CT* t,     \
                                        CT* part, CT* xbest, double* cg, double* ws, double tol, long long maxiter,    \
                                        long long P, long long first_iter, long long iters, long long n,              \
                                        void* stream) {                                                               \
    return bal_pcg_run<CT>(Y4, poses, intr, pidx, cseg, split, tpi, m, Y4p, cidx_p, pptr, Hc, Hpinv, Minv, bneg, x,   \
                           r, z, p, q, t, part, xbest, cg, ws, tol, maxiter, P, first_iter, iters, n,                 \
                           (cudaStream_t)stream);                                                                     \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_cg_finish_##SFX(CT* x, const CT* xbest, const double* cg, long long n, void* stream) {  \
    if (n <= 0) return 0;                                                                                             \
    BAL_LAUNCH(cg_finish_kernel<CT>, n * kBalCam, stream, x, xbest, cg, n * kBalCam);                                 \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_predicted_##SFX(const CT* Y4, const CT* poses, const CT* intr, const CT* rs,            \
                                              const int* cidx, const int* pidx, const CT* xc, const CT* xp,           \
                                              double* ws, long long m, void* stream) {                                \
    if (m <= 0) return 0;                                                                                             \
    BAL_LAUNCH(bal_predicted_kernel<CT>, m, stream, Y4, poses, intr, rs, cidx, pidx, xc, xp, ws, m);                  \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_loss_##SFX(const CT* poses, const CT* intr, const CT* points, const CT* pix,            \
                                         const int* cidx, const int* pidx, double* ws, int robust, double delta,      \
                                         long long m, void* stream) {                                                 \
    if (m <= 0) return 0;                                                                                             \
    BAL_LAUNCH(bal_loss_kernel<CT>, m, stream, poses, intr, points, pix, cidx, pidx, ws, robust, (CT)delta, m);       \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_bal_retract_##SFX(const CT* poses, const CT* intr, const CT* points, const CT* xc,          \
                                            const CT* xp, CT* poses_t, CT* intr_t, CT* points_t, long long C,         \
                                            long long P, void* stream) {                                              \
    const long long n = C > P ? C : P;                                                                                \
    if (n <= 0) return 0;                                                                                             \
    BAL_LAUNCH(bal_retract_kernel<CT>, n, stream, poses, intr, points, xc, xp, poses_t, intr_t, points_t, C, P);      \
    return (int)cudaGetLastError();                                                                                   \
  }

BAL_ABI(f32, float)
BAL_ABI(f64, double)
