// ba.cu — bundle adjustment without atomics: bit-reproducible block sums (C-ABI: include/b200pose.h, section LM).
//
// Scatter-added with warp-aggregated atomics, the camera-side sums of the BA route (Hcc / gc / the Schur diagonal / every
// W v product) depend on the order in which warps reach the atomic unit.  On an ill-conditioned fp32 system that noise
// seeds a chaotic CG (different outcomes from run to run of the same seeded problem).  Here every sum has ONE writer and a fixed order:
//
//  * observations are grouped by camera once (optim/structured.py BAProblem), cseg[c] .. cseg[c+1] are camera c's rows;
//  * a work item is (camera c, sub-range s of S): TPI threads (one warp, or one 128-thread CTA) stride over the item's
//    rows, reduce with a fixed shuffle tree (+ a fixed-order fold of the 4 warp partials), and ONE thread writes the
//    result — directly when S == 1, to a partial slot (c, s) otherwise, folded in s order by cam_fold_kernel;
//  * the point side is a gather over the point-ordered copy (Y4p / cidx_p / pix_p, offsets pptr) with 8 lanes per point.
//
// Reference semantics: these are the J^T J / J^T R sums of optimizer.py:645-656 (sparse counterpart: bae
// autograd.graph.jacobian + J.mT @ J, optimizer.py:637-642) for the two-parameter reprojection model README.md:163-198.
#include "lm_common.cuh"

namespace b200pose {

// fixed-order reduction of NV values over the TPI threads of an item; the result is valid in the item's first thread
template <typename T, int NV, int TPI>
__device__ __forceinline__ void item_reduce(T (&v)[NV], T (*sh)[NV]) {
#pragma unroll
  for (int k = 0; k < NV; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  if (TPI > 32) {                                   // one item per CTA: fold the warp partials in warp order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();                                // previous item's readers are done with sh
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < NV; ++k) sh[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        T t = sh[0][k];
        for (int w = 1; w < TPI / 32; ++w) t += sh[w][k];
        v[k] = t;
      }
  }
}

// rows of one observation from y (camera frame), the robust scale and the camera quaternion (held by the item)
template <typename T>
__device__ __forceinline__ void rows_from_y(const V3<T>& y, T sw, const Q4<T>& q, ObsRows<T>& R) {
  Elem<T> Tc;
  Tc.q = q;
  reproj_rows(y, R.jc0, R.jc1);
  reproj_point_rows(Tc, y, R.jp0, R.jp1);
#pragma unroll
  for (int a = 0; a < 6; ++a) { R.jc0[a] *= sw; R.jc1[a] *= sw; }
#pragma unroll
  for (int a = 0; a < 3; ++a) { R.jp0[a] *= sw; R.jp1[a] *= sw; }
}

struct ItemRange { long long c; int b, e; };
__device__ __forceinline__ ItemRange item_range(long long it, int S, const int* __restrict__ cseg) {
  ItemRange r;
  r.c = it / S;
  const int s = (int)(it - r.c * S);
  const long long b = cseg[r.c], len = (long long)cseg[r.c + 1] - b;
  r.b = (int)(b + len * s / S);
  r.e = (int)(b + len * (s + 1) / S);
  return r;
}

// Linearisation: per observation y = T_c p_j, residual, robust scale; stores Y4 (camera order), Y4p (point order) and the
// scaled residual; per item the 21 + 6 camera sums.  sums: ws[0] = sum rho(|r|^2).
template <typename T, int TPI>
__global__ void __launch_bounds__(kLmThreads) ba_linearize_seg_kernel(
    const T* __restrict__ poses, const T* __restrict__ points, const T* __restrict__ pix, const int* __restrict__ pidx,
    const int* __restrict__ cseg, int S, T* __restrict__ Y4, const int* __restrict__ ppos, T* __restrict__ Y4p,
    T* __restrict__ rs, T* __restrict__ Hcc, T* __restrict__ gc, T* __restrict__ part, double* ws, int rk, T rdelta,
    long long C) {
  constexpr int IPB = kLmThreads / TPI;
  __shared__ T sh[TPI > 32 ? TPI / 32 : 1][27];
  const int sub = threadIdx.x % TPI;
  const long long items = C * S, rounds = (items + IPB - 1) / IPB;
  double acc[1] = {0.0};
  for (long long rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const long long it = rd * IPB + threadIdx.x / TPI;
    T cam[27];
#pragma unroll
    for (int a = 0; a < 27; ++a) cam[a] = T(0);
    ItemRange r = {0, 0, 0};
    if (it < items) {
      r = item_range(it, S, cseg);
      T pr[7];
#pragma unroll
      for (int q = 0; q < 7; ++q) pr[q] = __ldg(poses + r.c * 7 + q);
      const Elem<T> Tc = load_se3(pr);
      for (int k = r.b + sub; k < r.e; k += TPI) {
        const long long j = pidx[k];
        const V3<T> p = mk(__ldg(points + j * 3), __ldg(points + j * 3 + 1), __ldg(points + j * 3 + 2));
        T rx, ry;
        V3<T> y;
        reproj_residual(Tc, p, pix[(long long)k * 2], pix[(long long)k * 2 + 1], rx, ry, y);
        T rho, w;
        robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
        const T sw = rk ? m_sqrt(w) : T(1);
        rx *= sw; ry *= sw;
        T j0[6], j1[6];
        reproj_rows(y, j0, j1);
#pragma unroll
        for (int a = 0; a < 6; ++a) { j0[a] *= sw; j1[a] *= sw; }
        const long long k4 = (long long)k * 4;
        Y4[k4] = y.x; Y4[k4 + 1] = y.y; Y4[k4 + 2] = y.z; Y4[k4 + 3] = sw;
        if (Y4p) {
          const long long s4 = (long long)ppos[k] * 4;
          Y4p[s4] = y.x; Y4p[s4 + 1] = y.y; Y4p[s4 + 2] = y.z; Y4p[s4 + 3] = sw;
        }
        rs[(long long)k * 2] = rx; rs[(long long)k * 2 + 1] = ry;
        int q = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          cam[21 + a] += j0[a] * rx + j1[a] * ry;
#pragma unroll
          for (int b = a; b < 6; ++b) cam[q++] += j0[a] * j0[b] + j1[a] * j1[b];
        }
        acc[0] += (double)rho;
      }
    }
    item_reduce<T, 27, TPI>(cam, sh);
    if (it < items && sub == 0) {
      if (S == 1) {
#pragma unroll
        for (int a = 0; a < 21; ++a) Hcc[r.c * 21 + a] = cam[a];
#pragma unroll
        for (int a = 0; a < 6; ++a) gc[r.c * 6 + a] = cam[21 + a];
      } else {
#pragma unroll
        for (int a = 0; a < 27; ++a) part[it * 27 + a] = cam[a];
      }
    }
  }
  reduce_sums<1>(acc, ws);
}

// dst (+)= sum_s part[(c, s)] in s order; the first WA values go to A (stride WA), the remaining WB to B (stride WB)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) cam_fold_kernel(const T* __restrict__ part, int S, int WA, int WB,
                                                               T* __restrict__ A, T* __restrict__ B, int add,
                                                               const double* cg, long long C) {
  if (cg && cg[5] != 0.0) return;
  const int NV = WA + WB;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < C * NV; i += (long long)gridDim.x * kLmThreads) {
    const long long c = i / NV;
    const int v = (int)(i - c * NV);
    T t = T(0);
    for (int s = 0; s < S; ++s) t += part[(c * S + s) * NV + v];
    T* d = v < WA ? A + c * WA + v : B + c * WB + (v - WA);
    *d = add ? *d + t : t;
  }
}

// Point blocks Hpp (6) and gp (3) by gather over the point-ordered rows: LPP lanes per point, fixed shuffle tree.
constexpr int kBaLanesPerPoint = 8;
template <typename T>
__global__ void __launch_bounds__(kLmThreads) ba_point_blocks_kernel(const T* __restrict__ Y4p, const T* __restrict__ pix_p,
                                                                      const T* __restrict__ poses,
                                                                      const int* __restrict__ cidx_p,
                                                                      const int* __restrict__ pptr, T* __restrict__ Hpp,
                                                                      T* __restrict__ gp, long long P) {
  constexpr int LPP = kBaLanesPerPoint, PPB = kLmThreads / LPP;
  const int sub = threadIdx.x % LPP;
  const long long groups = (P + PPB - 1) / PPB;
  for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
    const long long j = g * PPB + threadIdx.x / LPP;
    T a[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) a[k] = T(0);
    if (j < P)
      for (int s = pptr[j] + sub; s < pptr[j + 1]; s += LPP) {
        const long long c = cidx_p[s];
        const long long s4 = (long long)s * 4;
        const V3<T> y = mk(Y4p[s4], Y4p[s4 + 1], Y4p[s4 + 2]);
        const T sw = Y4p[s4 + 3];
        Q4<T> q;
        q.v = mk(__ldg(poses + c * 7 + 3), __ldg(poses + c * 7 + 4), __ldg(poses + c * 7 + 5));
        q.w = __ldg(poses + c * 7 + 6);
        ObsRows<T> R;
        rows_from_y(y, sw, q, R);
        const T iz = m_rcp(y.z);
        const T rx = (-y.x * iz - pix_p[(long long)s * 2]) * sw, ry = (-y.y * iz - pix_p[(long long)s * 2 + 1]) * sw;
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
__global__ void __launch_bounds__(kLmThreads) ba_wv_seg_kernel(const T* __restrict__ Y4, const T* __restrict__ poses,
                                                                const int* __restrict__ pidx, const int* __restrict__ cseg,
                                                                int S, const T* __restrict__ Hpinv, const T* __restrict__ t,
                                                                T* __restrict__ y, T* __restrict__ part, const double* cg,
                                                                long long C) {
  if (cg && cg[5] != 0.0) return;
  constexpr int IPB = kLmThreads / TPI;
  __shared__ T sh[TPI > 32 ? TPI / 32 : 1][6];
  const int sub = threadIdx.x % TPI;
  const long long items = C * S, rounds = (items + IPB - 1) / IPB;
  for (long long rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const long long it = rd * IPB + threadIdx.x / TPI;
    T out[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
    ItemRange r = {0, 0, 0};
    if (it < items) {
      r = item_range(it, S, cseg);
      Q4<T> q;
      q.v = mk(__ldg(poses + r.c * 7 + 3), __ldg(poses + r.c * 7 + 4), __ldg(poses + r.c * 7 + 5));
      q.w = __ldg(poses + r.c * 7 + 6);
      for (int k = r.b + sub; k < r.e; k += TPI) {
        const long long j = pidx[k], k4 = (long long)k * 4;
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
        ObsRows<T> R;
        rows_from_y(mk(Y4[k4], Y4[k4 + 1], Y4[k4 + 2]), Y4[k4 + 3], q, R);
        T u0 = T(0), u1 = T(0);
#pragma unroll
        for (int a = 0; a < 3; ++a) { u0 += R.jp0[a] * v[a]; u1 += R.jp1[a] * v[a]; }
#pragma unroll
        for (int a = 0; a < 6; ++a) out[a] -= R.jc0[a] * u0 + R.jc1[a] * u1;
      }
    }
    item_reduce<T, 6, TPI>(out, sh);
    if (it < items && sub == 0) {
      if (S == 1) {
#pragma unroll
        for (int a = 0; a < 6; ++a) y[r.c * 6 + a] += out[a];
      } else {
#pragma unroll
        for (int a = 0; a < 6; ++a) part[it * 6 + a] = out[a];
      }
    }
  }
}

// Sd[c] -= sum_k (Jc^T Jp) Hp^-1 (Jp^T Jc)   (diagonal blocks of the Schur complement; Sd pre-set to the damped Hcc)
template <typename T, int TPI>
__global__ void __launch_bounds__(kLmThreads) ba_schur_diag_seg_kernel(const T* __restrict__ Y4, const T* __restrict__ poses,
                                                                        const int* __restrict__ pidx,
                                                                        const int* __restrict__ cseg, int S,
                                                                        const T* __restrict__ Hpinv, T* __restrict__ Sd,
                                                                        T* __restrict__ part, long long C) {
  constexpr int IPB = kLmThreads / TPI;
  __shared__ T sh[TPI > 32 ? TPI / 32 : 1][21];
  const int sub = threadIdx.x % TPI;
  const long long items = C * S, rounds = (items + IPB - 1) / IPB;
  for (long long rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const long long it = rd * IPB + threadIdx.x / TPI;
    T out[21];
#pragma unroll
    for (int a = 0; a < 21; ++a) out[a] = T(0);
    ItemRange r = {0, 0, 0};
    if (it < items) {
      r = item_range(it, S, cseg);
      Q4<T> q;
      q.v = mk(__ldg(poses + r.c * 7 + 3), __ldg(poses + r.c * 7 + 4), __ldg(poses + r.c * 7 + 5));
      q.w = __ldg(poses + r.c * 7 + 6);
      for (int k = r.b + sub; k < r.e; k += TPI) {
        const long long j = pidx[k], k4 = (long long)k * 4;
        T A[3][3], h[6];
#pragma unroll
        for (int a = 0; a < 6; ++a) h[a] = __ldg(Hpinv + j * 6 + a);
        sym3_unpack(h, A);
        ObsRows<T> R;
        rows_from_y(mk(Y4[k4], Y4[k4 + 1], Y4[k4 + 2]), Y4[k4 + 3], q, R);
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
        for (int a = 0; a < 6; ++a) {
          const T l0 = R.jc0[a] * g00 + R.jc1[a] * g01, l1 = R.jc0[a] * g01 + R.jc1[a] * g11;
#pragma unroll
          for (int b = a; b < 6; ++b) out[qq++] -= l0 * R.jc0[b] + l1 * R.jc1[b];
        }
      }
    }
    item_reduce<T, 21, TPI>(out, sh);
    if (it < items && sub == 0) {
      if (S == 1) {
#pragma unroll
        for (int a = 0; a < 21; ++a) Sd[r.c * 21 + a] += out[a];
      } else {
#pragma unroll
        for (int a = 0; a < 21; ++a) part[it * 21 + a] = out[a];
      }
    }
  }
}

static inline unsigned item_grid(long long items, int tpi) {
  const int ipb = kLmThreads / tpi;
  return lm_grid(items, ipb);
}

template <typename CT>
int ba_wv_seg_launch(const CT* Y4, const CT* poses, const int* pidx, const int* cseg, int S, int tpi, const CT* Hpinv,
                     const CT* t, CT* y, CT* part, const double* cg, long long C, cudaStream_t st) {
  const unsigned grid = item_grid(C * S, tpi);
  if (tpi == 32) ba_wv_seg_kernel<CT, 32><<<grid, kLmThreads, 0, st>>>(Y4, poses, pidx, cseg, S, Hpinv, t, y, part, cg, C);
  else ba_wv_seg_kernel<CT, 128><<<grid, kLmThreads, 0, st>>>(Y4, poses, pidx, cseg, S, Hpinv, t, y, part, cg, C);
  if (S > 1) cam_fold_kernel<CT><<<lm_grid(C * 6, kLmThreads), kLmThreads, 0, st>>>(part, S, 6, 0, y, (CT*)nullptr, 1, cg, C);
  return (int)cudaGetLastError();
}
template int ba_wv_seg_launch<float>(const float*, const float*, const int*, const int*, int, int, const float*, const float*,
                                     float*, float*, const double*, long long, cudaStream_t);
template int ba_wv_seg_launch<double>(const double*, const double*, const int*, const int*, int, int, const double*,
                                      const double*, double*, double*, const double*, long long, cudaStream_t);

}  // namespace b200pose

using namespace b200pose;

#define BA_SEG_ABI(SFX, CT)                                                                                           \
  B200_EXPORT int b200_lm_ba_linearize_seg_##SFX(const CT* poses, const CT* points, const CT* pix, const int* pidx,   \
                                                 const int* cseg, long long split, long long tpi, CT* Y4,             \
                                                 const int* ppos, CT* Y4p, CT* rs, CT* Hcc, CT* gc, CT* part,         \
                                                 double* ws, int robust, double delta, long long C, void* stream) {   \
    if (C <= 0) return 0;                                                                                             \
    cudaStream_t st = (cudaStream_t)stream;                                                                           \
    const int S = (int)split;                                                                                         \
    const unsigned grid = item_grid(C * S, (int)tpi);                                                                 \
    if (tpi == 32)                                                                                                    \
      ba_linearize_seg_kernel<CT, 32><<<grid, kLmThreads, 0, st>>>(poses, points, pix, pidx, cseg, S, Y4, ppos, Y4p,  \
                                                                   rs, Hcc, gc, part, ws, robust, (CT)delta, C);      \
    else                                                                                                              \
      ba_linearize_seg_kernel<CT, 128><<<grid, kLmThreads, 0, st>>>(poses, points, pix, pidx, cseg, S, Y4, ppos, Y4p, \
                                                                    rs, Hcc, gc, part, ws, robust, (CT)delta, C);     \
    if (S > 1)                                                                                                        \
      cam_fold_kernel<CT><<<lm_grid(C * 27, kLmThreads), kLmThreads, 0, st>>>(part, S, 21, 6, Hcc, gc, 0,             \
                                                                               (const double*)nullptr, C);            \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_ba_point_blocks_##SFX(const CT* Y4p, const CT* pix_p, const CT* poses, const int* cidx_p,   \
                                                const int* pptr, CT* Hpp, CT* gp, long long P, void* stream) {        \
    if (P <= 0) return 0;                                                                                             \
    ba_point_blocks_kernel<CT><<<lm_grid(P * kBaLanesPerPoint, kLmThreads), kLmThreads, 0, (cudaStream_t)stream>>>(   \
        Y4p, pix_p, poses, cidx_p, pptr, Hpp, gp, P);                                                                 \
    return (int)cudaGetLastError();                                                                                   \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_ba_wv_seg_##SFX(const CT* Y4, const CT* poses, const int* pidx, const int* cseg,            \
                                          long long split, long long tpi, const CT* Hpinv, const CT* t, CT* y,        \
                                          CT* part, long long C, void* stream) {                                      \
    if (C <= 0) return 0;                                                                                             \
    return ba_wv_seg_launch<CT>(Y4, poses, pidx, cseg, (int)split, (int)tpi, Hpinv, t, y, part,                       \
                                (const double*)nullptr, C, (cudaStream_t)stream);                                     \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_ba_schur_diag_seg_##SFX(const CT* Y4, const CT* poses, const int* pidx, const int* cseg,    \
                                                  long long split, long long tpi, const CT* Hpinv, CT* Sd, CT* part,  \
                                                  long long C, void* stream) {                                        \
    if (C <= 0) return 0;                                                                                             \
    cudaStream_t st = (cudaStream_t)stream;                                                                           \
    const int S = (int)split;                                                                                         \
    const unsigned grid = item_grid(C * S, (int)tpi);                                                                 \
    if (tpi == 32)                                                                                                    \
      ba_schur_diag_seg_kernel<CT, 32><<<grid, kLmThreads, 0, st>>>(Y4, poses, pidx, cseg, S, Hpinv, Sd, part, C);    \
    else                                                                                                              \
      ba_schur_diag_seg_kernel<CT, 128><<<grid, kLmThreads, 0, st>>>(Y4, poses, pidx, cseg, S, Hpinv, Sd, part, C);   \
    if (S > 1)                                                                                                        \
      cam_fold_kernel<CT><<<lm_grid(C * 21, kLmThreads), kLmThreads, 0, st>>>(part, S, 21, 0, Sd, (CT*)nullptr, 1,    \
                                                                               (const double*)nullptr, C);            \
    return (int)cudaGetLastError();                                                                                   \
  }

BA_SEG_ABI(f32, float)
BA_SEG_ABI(f64, double)
