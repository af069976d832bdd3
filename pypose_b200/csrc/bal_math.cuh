// bal_math.cuh — per-observation math of the BAL camera model (host+device, see lie_math.cuh).
//
// BAL ("Bundle Adjustment in the Large") residual of the reference's examples/module/ba/bundle_adjustment.py `Reproj`:
//   y = T_c p_j,   n = -y[:2] / y[2],   rho = |n|^2,   d = 1 + k1 rho + k2 rho^2,   r = f d n - z
// with per-camera intrinsics K = (f, k1, k2).  The unknowns of one camera are [xi (6) | f, k1, k2] (xi: left SE3
// perturbation, the LieTensor `add_` retraction), of one point dp (3).  Jacobian rows:
//   dr/df = d n,   dr/dk1 = f rho n,   dr/dk2 = f rho^2 n,
//   dr/dn = f (d I + 2 (k1 + 2 k2 rho) n n^T),   dn/dy = [[-1/y2, 0, y0/y2^2], [0, -1/y2, y1/y2^2]],
//   dy/dxi = [I, -y^],   dy/dp = R(T_c).
// Symmetric NxN blocks are packed as their row-major upper triangle (N = 9: 45 words, N = 3: 6 words).
#pragma once
#include "lm_math.cuh"

namespace b200pose {

constexpr int kBalCam = 9;                        // unknowns per camera
constexpr int kBalCamPacked = 45;                 // packed upper triangle of a 9x9 block

template <typename T> struct BalRows { T jc0[9], jc1[9], jp0[3], jp1[3]; };

// residual r = f d n - z and the camera-frame point y
template <typename T>
LM_HD void bal_residual(const Elem<T>& Tc, const V3<T>& p, T f, T k1, T k2, T zx, T zy, T& rx, T& ry, V3<T>& y) {
  y = g_act<SE3g, T>(Tc, p);
  const T iz = m_rcp(y.z);
  const T n0 = -y.x * iz, n1 = -y.y * iz;
  const T rho = n0 * n0 + n1 * n1;
  const T d = T(1) + k1 * rho + k2 * rho * rho;
  rx = f * d * n0 - zx;
  ry = f * d * n1 - zy;
}

// residual from a stored y (the trial-free recomputation of the gather kernels)
template <typename T> LM_HD void bal_residual_y(const V3<T>& y, T f, T k1, T k2, T zx, T zy, T& rx, T& ry) {
  const T iz = m_rcp(y.z);
  const T n0 = -y.x * iz, n1 = -y.y * iz;
  const T rho = n0 * n0 + n1 * n1;
  const T d = T(1) + k1 * rho + k2 * rho * rho;
  rx = f * d * n0 - zx;
  ry = f * d * n1 - zy;
}

// the 2x9 camera rows and the 2x3 point rows of one observation from y = T_c p, the camera rotation and intrinsics,
// all scaled by sw (sqrt of the robust weight, FastTriggs)
template <typename T> LM_HD void bal_rows(const V3<T>& y, const Q4<T>& q, T f, T k1, T k2, T sw, BalRows<T>& R) {
  const T iz = m_rcp(y.z), iz2 = iz * iz;
  const T n0 = -y.x * iz, n1 = -y.y * iz;
  const T rho = n0 * n0 + n1 * n1;
  const T d = T(1) + k1 * rho + k2 * rho * rho;
  // A = dr/dn = f (d I + e n n^T), e = 2 (k1 + 2 k2 rho)
  const T e = T(2) * (k1 + T(2) * k2 * rho);
  const T a00 = f * (d + e * n0 * n0), a01 = f * e * n0 * n1, a11 = f * (d + e * n1 * n1);
  // B = dn/dy
  const T b0 = -iz, c0 = y.x * iz2, c1 = y.y * iz2;
  // G = A B (2x3): rows of dr/dy
  const V3<T> g0 = mk(a00 * b0, a01 * b0, a00 * c0 + a01 * c1);
  const V3<T> g1 = mk(a01 * b0, a11 * b0, a01 * c0 + a11 * c1);
  // camera pose columns: g [I, -y^] = [g, y x g]
  const V3<T> h0 = cross(y, g0), h1 = cross(y, g1);
  R.jc0[0] = g0.x; R.jc0[1] = g0.y; R.jc0[2] = g0.z; R.jc0[3] = h0.x; R.jc0[4] = h0.y; R.jc0[5] = h0.z;
  R.jc1[0] = g1.x; R.jc1[1] = g1.y; R.jc1[2] = g1.z; R.jc1[3] = h1.x; R.jc1[4] = h1.y; R.jc1[5] = h1.z;
  // intrinsics columns
  const T fr = f * rho, fr2 = fr * rho;
  R.jc0[6] = d * n0; R.jc0[7] = fr * n0; R.jc0[8] = fr2 * n0;
  R.jc1[6] = d * n1; R.jc1[7] = fr * n1; R.jc1[8] = fr2 * n1;
  // point columns: g R = R^T g
  const V3<T> p0 = qrot_t(q, g0), p1 = qrot_t(q, g1);
  R.jp0[0] = p0.x; R.jp0[1] = p0.y; R.jp0[2] = p0.z;
  R.jp1[0] = p1.x; R.jp1[1] = p1.y; R.jp1[2] = p1.z;
#pragma unroll
  for (int a = 0; a < 9; ++a) { R.jc0[a] *= sw; R.jc1[a] *= sw; }
#pragma unroll
  for (int a = 0; a < 3; ++a) { R.jp0[a] *= sw; R.jp1[a] *= sw; }
}

// ---- packed symmetric NxN blocks (row-major upper triangle, N (N+1) / 2 words) ----
template <typename T, int N> LM_HD void symn_unpack(const T* a, T (&A)[N][N]) {
  int q = 0;
#pragma unroll
  for (int p = 0; p < N; ++p)
#pragma unroll
    for (int c = p; c < N; ++c) { A[p][c] = a[q]; A[c][p] = a[q]; ++q; }
}
template <typename T, int N> LM_HD void symn_pack(const T (&A)[N][N], T* a) {
  int q = 0;
#pragma unroll
  for (int p = 0; p < N; ++p)
#pragma unroll
    for (int c = p; c < N; ++c) a[q++] = A[p][c];
}
// position of diagonal entry k inside a packed upper triangle of an NxN block
LM_HD constexpr int symn_diag(int N, int k) { return k * N - k * (k - 1) / 2; }
// y = A x straight from the packed words, row by row (an unpacked 9x9 copy costs 81 registers)
template <typename T, int N> LM_HD void symn_mv_packed(const T* a, const T (&x)[N], T (&y)[N]) {
#pragma unroll
  for (int p = 0; p < N; ++p) {
    T v = T(0);
#pragma unroll
    for (int c = 0; c < N; ++c) v += a[c < p ? symn_diag(N, c) + (p - c) : symn_diag(N, p) + (c - p)] * x[c];
    y[p] = v;
  }
}
// accumulate the outer products of two rows into a packed 9x9 block: H += j0 j0^T + j1 j1^T
template <typename T> LM_HD void sym9_add_rows(T* H, const T (&j0)[9], const T (&j1)[9]) {
  int q = 0;
#pragma unroll
  for (int a = 0; a < 9; ++a)
#pragma unroll
    for (int b = a; b < 9; ++b) H[q++] += j0[a] * j0[b] + j1[a] * j1[b];
}

// diag <- clamp(diag, dmin, dmax) * scale of an unpacked 9x9 block (optimizer.py:657 + cumulative :666)
template <typename T> LM_HD void blk9_damp(T (&A)[9][9], T scale, T dmin, T dmax) {
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const T d = A[k][k];
    A[k][k] = (d < dmin ? dmin : (d > dmax ? dmax : d)) * scale;
  }
}

}  // namespace b200pose
