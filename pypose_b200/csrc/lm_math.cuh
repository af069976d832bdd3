// lm_math.cuh — per-block math of the Levenberg-Marquardt inner loop (host+device, see lie_math.cuh).
//
// Reference semantics (pypose/optim/optimizer.py:645-680, dense branch), specialised to the block
// structure the reference's dense Jacobian actually has (SURVEY.md §3.3, §8a "analytic Jacobians"):
//   * PoseInv  r = Log(P X):        dr/dP = Jl^-1(r)                      (6x6 per pose)
//   * Reproj   r = pi(T p) - z:     dr/dT = dpi/dy [I, -y^], y = T p      (2x6 per observation)
// with left perturbations and K = 6 tangent columns (the 7th dense column is identically zero and only
// produces D[6] = 0 in the reference).
#pragma once
#include "lie_math.cuh"

namespace b200pose {

template <typename T> struct M3 { T m[3][3]; };

template <typename T> LM_HD M3<T> m3_skew(const V3<T>& v) {
  M3<T> a;
  a.m[0][0] = T(0); a.m[0][1] = -v.z; a.m[0][2] = v.y;
  a.m[1][0] = v.z;  a.m[1][1] = T(0); a.m[1][2] = -v.x;
  a.m[2][0] = -v.y; a.m[2][1] = v.x;  a.m[2][2] = T(0);
  return a;
}
template <typename T> LM_HD M3<T> m3_mul(const M3<T>& a, const M3<T>& b) {
  M3<T> c;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) c.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
  return c;
}
template <typename T> LM_HD M3<T> m3_t(const M3<T>& a) {
  M3<T> c;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) c.m[i][j] = a.m[j][i];
  return c;
}

// Ji = Jl^-1(phi) and B = -Ji Q Ji of se3_Jl_inv (operation.py:68-75) as explicit 3x3 blocks.
template <typename T> LM_HD void se3_jlinv_blocks(const Tang<T>& x, M3<T>& Ji, M3<T>& B) {
  const RotCoef<T> r = rot_coef(x.phi);
  const T c = jlinv_coef(x.phi);
  T a2, a3;
  q_coef(r, a2, a3);
  const T a1 = r.c2;
  const M3<T> P = m3_skew(x.phi), Tm = m3_skew(x.tau);
  const M3<T> PP = m3_mul(P, P);
  const M3<T> PT = m3_mul(P, Tm);       // TP = PT^T
  const M3<T> PTP = m3_mul(PT, P);
  const M3<T> PPT = m3_mul(P, PT);      // TPP = -PPT^T
  const M3<T> PTPP = m3_mul(PTP, P);    // PPTP = PTPP^T
  M3<T> Q;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      Ji.m[i][j] = (i == j ? T(1) : T(0)) - T(0.5) * P.m[i][j] + c * PP.m[i][j];
      Q.m[i][j] = T(0.5) * Tm.m[i][j] + a1 * (PT.m[i][j] + PT.m[j][i] + PTP.m[i][j]) +
                  a2 * (PPT.m[i][j] - PPT.m[j][i] - T(3) * PTP.m[i][j]) + a3 * (PTPP.m[i][j] + PTPP.m[j][i]);
    }
  const M3<T> JQJ = m3_mul(m3_mul(Ji, Q), Ji);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) B.m[i][j] = -JQJ.m[i][j];
}

// One 6x6 normal-equation block, symmetric, full storage in registers.
template <typename T> struct Sys6 {
  T A[6][6];   // J^T J (only j >= i is maintained)
  T g[6];      // J^T r
};
template <typename T> LM_HD void sys6_zero(Sys6<T>& s) {
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    s.g[i] = T(0);
#pragma unroll
    for (int j = 0; j < 6; ++j) s.A[i][j] = T(0);
  }
}
// rank-1 update with one Jacobian row j (1x6) and residual component r
template <typename T> LM_HD void sys6_add_row(Sys6<T>& s, const T (&j)[6], T r) {
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    s.g[a] += j[a] * r;
#pragma unroll
    for (int b = a; b < 6; ++b) s.A[a][b] += j[a] * j[b];
  }
}

// LM damping + Cholesky solve of one block (optimizer.py:657, 666, 668; solver.py:213-216):
//   diag <- clamp(diag, dmin, dmax) * scale      (scale = prod (1 + damping_k) over the trials so far)
//   D = A^-1 (-g);   predicted = (J D)^T (2 R + J D) = D^T A0 D + 2 D^T g   with A0 the undamped J^T J
// Returns false if the factorisation hit a non-positive pivot.
template <typename T> LM_HD bool sys6_damped_solve(const Sys6<T>& s, T scale, T dmin, T dmax, T (&D)[6], T& predicted) {
  T L[6][6];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    T djj = s.A[j][j];
    djj = djj < dmin ? dmin : (djj > dmax ? dmax : djj);
    T sum = djj * scale;
#pragma unroll
    for (int k = 0; k < j; ++k) sum -= L[j][k] * L[j][k];
    ok = ok && (sum > T(0));
    const T inv = m_rsqrt(sum);
    L[j][j] = sum * inv;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      T v = s.A[j][i];
#pragma unroll
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      L[i][j] = v * inv;
    }
  }
  T y[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {       // L y = -g
    T v = -s.g[i];
#pragma unroll
    for (int k = 0; k < i; ++k) v -= L[i][k] * y[k];
    y[i] = v * m_rcp(L[i][i]);
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {      // L^T D = y
    T v = y[i];
#pragma unroll
    for (int k = i + 1; k < 6; ++k) v -= L[k][i] * D[k];
    D[i] = v * m_rcp(L[i][i]);
  }
  T q = T(0), lin = T(0);
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    lin += D[a] * s.g[a];
    T row = T(0);
#pragma unroll
    for (int b = 0; b < 6; ++b) row += (b >= a ? s.A[a][b] : s.A[b][a]) * D[b];
    q += D[a] * row;
  }
  predicted = q + T(2) * lin;
  return ok;
}

// ---------------------------------------------------------------- robust kernels (optim/kernel.py) + FastTriggs
// rho(x) on x = |r|^2 and its derivative w = rho'(x).  FastTriggs (optim/corrector.py:73-95) scales the
// residual and its Jacobian rows by sqrt(w), i.e. J^T J and J^T r by w; the loss is sum rho(x) (optimizer.py:118-125).
// kind: 0 none, 1 Huber, 2 PseudoHuber, 3 Cauchy, 4 SoftLOne, 5 Arctan, 6 Scale
template <typename T> LM_HD void robust_eval(int kind, T delta, T x, T& rho, T& w) {
  const T d2 = delta * delta;
  switch (kind) {
    case 1: {                                   // kernel.py:5-45
      const T root = m_sqrt(x);
      const bool in = root < delta;
      rho = in ? x : T(2) * delta * root - d2;
      w = in ? T(1) : delta / root;
    } break;
    case 2: {                                   // kernel.py:48-86
      const T q = m_sqrt(x / d2 + T(1));
      rho = T(2) * d2 * (q - T(1));
      w = T(1) / q;
    } break;
    case 3: {                                   // kernel.py:89-126
      const T q = x / d2 + T(1);
      rho = d2 * m_log(q);
      w = T(1) / q;
    } break;
    case 4: {                                   // kernel.py:129-168
      const T q = m_sqrt(T(1) / d2 + x);
      rho = T(2) * (delta * q - T(1));
      w = delta / q;
    } break;
    case 5: {                                   // kernel.py:171-207
      const T q = x / d2;
      rho = d2 * m_atan(q);
      w = T(1) / (T(1) + q * q);
    } break;
    case 6: rho = delta * x; w = delta; break;  // kernel.py:258-297
    default: rho = x; w = T(1);
  }
}
template <typename T> LM_HD void sys6_scale(Sys6<T>& s, T w) {
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    s.g[a] *= w;
#pragma unroll
    for (int b = a; b < 6; ++b) s.A[a][b] *= w;
  }
}

// ---------------------------------------------------------------- PoseInv: r = Log(P X)
template <typename T> LM_HD Tang<T> poseinv_residual(const Elem<T>& P, const Elem<T>& X) {
  return g_log<SE3g, T>(g_mul<SE3g, T>(P, X));
}
template <typename T> LM_HD void poseinv_linearize(const Elem<T>& P, const Elem<T>& X, Tang<T>& r, Sys6<T>& s) {
  r = poseinv_residual(P, X);
  M3<T> Ji, B;
  se3_jlinv_blocks(r, Ji, B);
  // J = [[Ji, B], [0, Ji]]; rows 0-2: [Ji_i, B_i], rows 3-5: [0, Ji_i]
  sys6_zero(s);
  const T rr[6] = {r.tau.x, r.tau.y, r.tau.z, r.phi.x, r.phi.y, r.phi.z};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const T top[6] = {Ji.m[i][0], Ji.m[i][1], Ji.m[i][2], B.m[i][0], B.m[i][1], B.m[i][2]};
    const T bot[6] = {T(0), T(0), T(0), Ji.m[i][0], Ji.m[i][1], Ji.m[i][2]};
    sys6_add_row(s, top, rr[i]);
    sys6_add_row(s, bot, rr[i + 3]);
  }
}
template <typename T> LM_HD T tang6_sqnorm(const Tang<T>& r) { return dot(r.tau, r.tau) + dot(r.phi, r.phi); }

// retraction of the optimizers: P <- Exp(D) P   (lietensor.py:442-444)
template <typename T> LM_HD Elem<T> se3_retract(const T (&D)[6], const Elem<T>& P) {
  Tang<T> d; d.tau = mk(D[0], D[1], D[2]); d.phi = mk(D[3], D[4], D[5]); d.sigma = T(0);
  return g_mul<SE3g, T>(g_exp<SE3g, T>(d), P);
}

// ---------------------------------------------------------------- PGO edge: r = Log(Z^-1 A^-1 B)
// (examples/module/pgo/pgo.py:15-25).  With S = Z^-1 A^-1:  dr/dB = Jl^-1(r) Adj(S) =: J,  dr/dA = -J
// (left perturbations; SURVEY.md §8a), so the edge contributes M = J^T J to H_ii, H_jj and -M to H_ij, H_ji.
template <typename T> LM_HD Tang<T> pgo_residual(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Elem<T>& S) {
  S = g_mul<SE3g, T>(g_inv<SE3g, T>(Z), g_inv<SE3g, T>(A));
  return g_log<SE3g, T>(g_mul<SE3g, T>(S, B));
}
// rows of J = dr/dB (6x6) for one edge
template <typename T> LM_HD void pgo_jacobian(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Tang<T>& r, T (&J)[6][6]) {
  Elem<T> S;
  r = pgo_residual(A, B, Z, S);
  M3<T> Ji, Bm;
  se3_jlinv_blocks(r, Ji, Bm);
  // R(S) as a matrix, and t^ R
  M3<T> R;
  {
    const V3<T> c0 = qrot(S.q, mk(T(1), T(0), T(0))), c1 = qrot(S.q, mk(T(0), T(1), T(0))), c2 = qrot(S.q, mk(T(0), T(0), T(1)));
    R.m[0][0] = c0.x; R.m[1][0] = c0.y; R.m[2][0] = c0.z;
    R.m[0][1] = c1.x; R.m[1][1] = c1.y; R.m[2][1] = c1.z;
    R.m[0][2] = c2.x; R.m[1][2] = c2.y; R.m[2][2] = c2.z;
  }
  const M3<T> tR = m3_mul(m3_skew(S.t), R);
  // J = [[Ji, Bm],[0, Ji]] [[R, tR],[0, R]] = [[Ji R, Ji tR + Bm R],[0, Ji R]]
  const M3<T> JR = m3_mul(Ji, R);
  const M3<T> JtR = m3_mul(Ji, tR), BR = m3_mul(Bm, R);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      J[i][c] = JR.m[i][c];
      J[i][3 + c] = JtR.m[i][c] + BR.m[i][c];
      J[3 + i][c] = T(0);
      J[3 + i][3 + c] = JR.m[i][c];
    }
}
template <typename T> LM_HD void pgo_linearize(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Tang<T>& r, Sys6<T>& s) {
  T J[6][6];
  pgo_jacobian(A, B, Z, r, J);
  sys6_zero(s);
  const T rr[6] = {r.tau.x, r.tau.y, r.tau.z, r.phi.x, r.phi.y, r.phi.z};
#pragma unroll
  for (int i = 0; i < 6; ++i) sys6_add_row(s, J[i], rr[i]);
}
// with a per-edge information matrix W (6x6, row-major): sw.A = J^T W J, sw.g = J^T W r (optimizer.py:654-656 with
// `weight`), next to the unweighted s0 (the TrustRegion quality uses J and R without the weight, strategy.py:143)
template <typename T>
LM_HD void pgo_linearize_w(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, const T* W, Tang<T>& r, Sys6<T>& sw, Sys6<T>& s0) {
  T J[6][6];
  pgo_jacobian(A, B, Z, r, J);
  sys6_zero(s0);
  const T rr[6] = {r.tau.x, r.tau.y, r.tau.z, r.phi.x, r.phi.y, r.phi.z};
#pragma unroll
  for (int i = 0; i < 6; ++i) sys6_add_row(s0, J[i], rr[i]);
  T WJ[6][6], Wr[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    T a = T(0);
#pragma unroll
    for (int k = 0; k < 6; ++k) a += W[i * 6 + k] * rr[k];
    Wr[i] = a;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      T v = T(0);
#pragma unroll
      for (int k = 0; k < 6; ++k) v += W[i * 6 + k] * J[k][c];
      WJ[i][c] = v;
    }
  }
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    T g = T(0);
#pragma unroll
    for (int k = 0; k < 6; ++k) g += J[k][a] * Wr[k];
    sw.g[a] = g;
#pragma unroll
    for (int b = 0; b < 6; ++b) {
      T v = T(0);
#pragma unroll
      for (int k = 0; k < 6; ++k) v += J[k][a] * WJ[k][b];
      sw.A[a][b] = v;
    }
  }
}

// ---------------------------------------------------------------- Reprojection: r = pi(T p) - z, pi(y) = -y[:2]/y[2]
// (README.md:170-178 `project`; the Jacobian of T p w.r.t. T is [I, -y^], operation.py:225-227)
template <typename T> LM_HD void reproj_residual(const Elem<T>& Tc, const V3<T>& p, T zx, T zy, T& rx, T& ry, V3<T>& y) {
  y = g_act<SE3g, T>(Tc, p);
  const T iz = m_rcp(y.z);
  rx = -y.x * iz - zx;
  ry = -y.y * iz - zy;
}
template <typename T> LM_HD void reproj_rows(const V3<T>& y, T (&j0)[6], T (&j1)[6]) {
  const T iz = m_rcp(y.z), iz2 = iz * iz;
  // dpi/dy = [[-1/z, 0, x/z^2], [0, -1/z, y/z^2]];  d y / d xi = [I, -y^]
  const T a0 = -iz, c0 = y.x * iz2, c1 = y.y * iz2;
  // -y^ = [[0, z, -y], [-z, 0, x], [y, -x, 0]]
  j0[0] = a0; j0[1] = T(0); j0[2] = c0;
  j0[3] = c0 * y.y;              // a0*0 + 0*(-z) + c0*y
  j0[4] = a0 * y.z - c0 * y.x;   // a0*z + c0*(-x)
  j0[5] = -a0 * y.y;             // a0*(-y)
  j1[0] = T(0); j1[1] = a0; j1[2] = c1;
  j1[3] = -a0 * y.z + c1 * y.y;  // a0*(-z) + c1*y
  j1[4] = -c1 * y.x;             // c1*(-x)
  j1[5] = a0 * y.x;              // a0*x
}

// d pi / d p = d pi/dy R(T)  (2x3): Jacobian of the projection w.r.t. a world point (SE3_Act.backward gp = g @ R,
// operation.py:560-568)
template <typename T> LM_HD void reproj_point_rows(const Elem<T>& Tc, const V3<T>& y, T (&p0)[3], T (&p1)[3]) {
  const T iz = m_rcp(y.z), iz2 = iz * iz;
  const T a0 = -iz, c0 = y.x * iz2, c1 = y.y * iz2;
  // rows of dpi/dy: [a0, 0, c0], [0, a0, c1];  row @ R = R^T row
  const V3<T> r0 = qrot_t(Tc.q, mk(a0, T(0), c0)), r1 = qrot_t(Tc.q, mk(T(0), a0, c1));
  p0[0] = r0.x; p0[1] = r0.y; p0[2] = r0.z;
  p1[0] = r1.x; p1[1] = r1.y; p1[2] = r1.z;
}

// ---- packed symmetric blocks: 6x6 as 21 (row-major upper triangle), 3x3 as 6 ----
template <typename T> LM_HD void sym6_unpack(const T* a, T (&A)[6][6]) {
  int q = 0;
#pragma unroll
  for (int p = 0; p < 6; ++p)
#pragma unroll
    for (int c = p; c < 6; ++c) { A[p][c] = a[q]; A[c][p] = a[q]; ++q; }
}
template <typename T> LM_HD void sym6_pack(const T (&A)[6][6], T* a) {
  int q = 0;
#pragma unroll
  for (int p = 0; p < 6; ++p)
#pragma unroll
    for (int c = p; c < 6; ++c) a[q++] = A[p][c];
}
template <typename T> LM_HD void sym6_mv(const T (&A)[6][6], const T (&x)[6], T (&y)[6]) {
#pragma unroll
  for (int p = 0; p < 6; ++p) {
    T v = T(0);
#pragma unroll
    for (int c = 0; c < 6; ++c) v += A[p][c] * x[c];
    y[p] = v;
  }
}
// A^-1 of a symmetric positive definite NxN block through its Cholesky factor: A = L L^T, A^-1 = L^-T L^-1.
// Non-positive pivots (only reachable with a numerically singular block) are replaced by a tiny positive number.
template <typename T, int N> LM_HD void spd_inverse(const T (&A)[N][N], T (&Ai)[N][N]) {
  T L[N][N], R[N][N];      // R = L^-1 (lower)
#pragma unroll
  for (int j = 0; j < N; ++j) {
    T s = A[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
    s = s > T(0) ? s : T(1e-30);
    const T inv = m_rsqrt(s);
    L[j][j] = s * inv;
    R[j][j] = inv;
#pragma unroll
    for (int i = j + 1; i < N; ++i) {
      T v = A[j][i];
#pragma unroll
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      L[i][j] = v * inv;
    }
  }
#pragma unroll
  for (int j = 0; j < N; ++j)
#pragma unroll
    for (int i = j + 1; i < N; ++i) {
      T v = T(0);
#pragma unroll
      for (int k = j; k < i; ++k) v += L[i][k] * R[k][j];
      R[i][j] = -v * R[i][i];
    }
#pragma unroll
  for (int a = 0; a < N; ++a)
#pragma unroll
    for (int b = a; b < N; ++b) {
      T v = T(0);
#pragma unroll
      for (int k = b; k < N; ++k) v += R[k][a] * R[k][b];
      Ai[a][b] = v; Ai[b][a] = v;
    }
}
template <typename T> LM_HD void sym3_unpack(const T* a, T (&A)[3][3]) {
  A[0][0] = a[0]; A[0][1] = A[1][0] = a[1]; A[0][2] = A[2][0] = a[2];
  A[1][1] = a[3]; A[1][2] = A[2][1] = a[4]; A[2][2] = a[5];
}



// ---------------------------------------------------------------- J^T J accumulator
// Acc6<T>: the running 6x6 system of a thread (21 + 6 scalar FMAs per Jacobian row; sm_90 has no packed fp32 FMA).
template <typename T> struct Acc6 {
  Sys6<T> s;
  LM_HD void zero() { sys6_zero(s); }
  LM_HD void add_row(const T (&j)[6], T r) { sys6_add_row(s, j, r); }
  LM_HD Sys6<T> finish() const { return s; }
};

// ---------------------------------------------------------------- two-pose reprojection (lm.cu lm_reproj2_*)
// r = proj(T_b^-1 T_a p) - z with proj(y) = (fx y.x/y.z + sk y.y/y.z + cx, fy y.y/y.z + cy); see lm.cu for the citations
template <typename T> struct Intr { T fx, sk, cx, fy, cy; };

template <typename T> LM_HD void reproj2_point(const Elem<T>& Ta, const Elem<T>& Tb, const V3<T>& p, V3<T>& w, V3<T>& y) {
  w = g_act<SE3g, T>(Ta, p);
  y = qrot_t(Tb.q, w - Tb.t);
}
template <typename T> LM_HD void reproj2_residual(const Intr<T>& K, const V3<T>& y, T zx, T zy, T& rx, T& ry) {
  const T iz = m_rcp(y.z);
  rx = (K.fx * y.x + K.sk * y.y) * iz + K.cx - zx;
  ry = K.fy * y.y * iz + K.cy - zy;
}
// rows of J = d r / d xi_a (2x6); d r / d xi_b = -J.  d proj / d y rotated to the world frame, then [e, w x e]
template <typename T>
LM_HD void reproj2_rows(const Intr<T>& K, const Elem<T>& Tb, const V3<T>& w, const V3<T>& y, T (&j0)[6], T (&j1)[6]) {
  const T iz = m_rcp(y.z), iz2 = iz * iz;
  const V3<T> e0 = qrot(Tb.q, mk(K.fx * iz, K.sk * iz, -(K.fx * y.x + K.sk * y.y) * iz2));
  const V3<T> e1 = qrot(Tb.q, mk(T(0), K.fy * iz, -K.fy * y.y * iz2));
  const V3<T> c0 = cross(w, e0), c1 = cross(w, e1);
  j0[0] = e0.x; j0[1] = e0.y; j0[2] = e0.z; j0[3] = c0.x; j0[4] = c0.y; j0[5] = c0.z;
  j1[0] = e1.x; j1[1] = e1.y; j1[2] = e1.z; j1[3] = c1.x; j1[4] = c1.y; j1[5] = c1.z;
}


// ---------------------------------------------------------------- LM accept / reject decision + damping strategies
// IEEE double operations exactly as Python evaluates them: no fused multiply-adds on the device
#ifdef __CUDA_ARCH__
LM_HD double lm_ddiv(double a, double b) { return __ddiv_rn(a, b); }
LM_HD double lm_dsub(double a, double b) { return __dsub_rn(a, b); }
LM_HD double lm_dmul(double a, double b) { return __dmul_rn(a, b); }
#else
LM_HD double lm_ddiv(double a, double b) { return a / b; }
LM_HD double lm_dsub(double a, double b) { return a - b; }
LM_HD double lm_dmul(double a, double b) { return a * b; }
#endif
LM_HD double lm_fmax(double a, double b) { return a > b ? a : (b == b ? b : a); }     // Python max(a, b) for non-NaN input
LM_HD double lm_fmin(double a, double b) { return a < b ? a : (b == b ? b : a); }

// control block of one trial (filled from the host's `ctl` array, passed by value)
struct LmCtl {
  double last;          // loss the trial has to beat (the cached loss of the previous step), if `cached`
  double damping;       // pg['damping'] used for this trial
  double pg_down;       // pg['down']  (Adaptive: its constant factor; TrustRegion: the shrinking state)
  double reject_count;  // rejected trials so far in this step
  double reject_limit;  // LM(reject=...)
  double high, low, up, self_down, factor, smin, smax;
  int cached;           // 0: first step ever -> last = current loss of this linearisation
  int kind;             // 0 Constant, 1 Adaptive, 2 TrustRegion
};

enum { ST_STATUS = 0, ST_LOSS = 1, ST_LAST = 2, ST_DAMPING = 3, ST_RADIUS = 4, ST_DOWN = 5, ST_REJECT = 6, ST_CUR = 7,
       ST_TRIAL = 8, ST_PRED = 9, ST_FAILED = 10, ST_SIZE = 16 };

// optimizer.py:662-680 for one trial: strategy.update, then accept (status 1) / reject (0) / solver failure (2).
// Plain IEEE double operations in the order Python evaluates them (no fused multiply-adds).
LM_HD void lm_decide(const LmCtl& c, double cur, double trial, double predicted, double failed,
                                          double* st) {
  const double last = c.cached ? c.last : cur;
  double damping = c.damping, down = c.pg_down, radius = lm_ddiv(1.0, c.damping);
  st[ST_CUR] = cur; st[ST_TRIAL] = trial; st[ST_PRED] = predicted; st[ST_FAILED] = failed; st[ST_LAST] = last;
  if (failed > 0.0) {                      // solver.py:214-215 -> optimizer.py:669-671: break, nothing changes
    st[ST_STATUS] = 2.0; st[ST_LOSS] = last; st[ST_DAMPING] = damping; st[ST_RADIUS] = radius; st[ST_DOWN] = down;
    st[ST_REJECT] = c.reject_count;
    return;
  }
  if (c.kind != 0) {
    const double quality = lm_ddiv(lm_dsub(last, trial), -predicted);      // strategy.py:143 / 260
    if (c.kind == 1) {                                                         // Adaptive, strategy.py:134-151
      if (quality > c.high) damping = lm_dmul(damping, down);
      else if (quality > c.low) { }
      else damping = lm_dmul(damping, c.up);
      damping = lm_fmax(c.smin, lm_fmin(damping, c.smax));
    } else {                                                                   // TrustRegion, strategy.py:248-274
      if (quality > c.high) { radius = lm_dmul(c.up, radius); down = c.self_down; }
      else if (quality > c.low) { down = c.self_down; }
      else { radius = lm_dmul(radius, down); down = lm_dmul(down, c.factor); }
      down = lm_fmax(c.smin, lm_fmin(down, c.smax));
      radius = lm_fmax(c.smin, lm_fmin(radius, c.smax));
      damping = lm_ddiv(1.0, radius);
    }
  }
  const bool reject = (last < trial) && (c.reject_count < c.reject_limit);     // optimizer.py:675
  st[ST_STATUS] = reject ? 0.0 : 1.0;
  st[ST_LOSS] = reject ? last : trial;
  st[ST_REJECT] = reject ? c.reject_count + 1.0 : c.reject_count;
  st[ST_DAMPING] = damping; st[ST_RADIUS] = radius; st[ST_DOWN] = down;
}


}  // namespace b200pose
