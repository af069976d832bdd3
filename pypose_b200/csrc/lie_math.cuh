// lie_math.cuh — register-resident Lie group math for SO3 / SE3 / RxSO3 / Sim3.
//
// Everything here works on one group element held in registers; the kernels in
// lie_kernels.cuh are thin HBM<->smem<->register shells around these functions.
// The functions are __host__ __device__ so that the same source can be compiled
// by g++ in a *test-only* harness (tests/hostmath) to triage fp32 numerics
// without a GPU; the shipped package never runs them on the host.
//
// Behavioural spec: pypose/lietensor/operation.py of the reference (cited per
// function as op.py:LINE).  Formulas are re-derived in cross-product form (no
// 3x3 / 6x6 temporaries) and use wide Taylor windows where the reference's
// closed forms cancel catastrophically in fp32 (SURVEY.md §8c): parity is
// judged against the reference evaluated in fp64.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define LM_HD __host__ __device__ __forceinline__
#else
#define LM_HD inline
#endif

namespace b200pose {

// ----------------------------------------------------------------------------
// scalar helpers
// ----------------------------------------------------------------------------
template <typename T> struct num;
template <> struct num<float> {
  static constexpr float eps = 1.1920928955078125e-07f;  // torch.finfo(float32).eps
  static constexpr float small2 = 0.25f;    // theta^2 below which coefficient series are used
  static constexpr float tiny2 = 1e-6f;     // theta^2 below which sim3 Ws uses the theta->0 limit
  static constexpr float sig_small = 0.05f; // |sigma| below which sigma-series are used
};
template <> struct num<double> {
  static constexpr double eps = 2.220446049250313e-16;
  static constexpr double small2 = 1e-2;
  static constexpr double tiny2 = 1e-14;
  static constexpr double sig_small = 1e-3;
};

LM_HD float m_sqrt(float x) { return sqrtf(x); }
LM_HD double m_sqrt(double x) { return sqrt(x); }
LM_HD float m_abs(float x) { return fabsf(x); }
LM_HD double m_abs(double x) { return fabs(x); }
LM_HD float m_atan(float x) { return atanf(x); }
LM_HD double m_atan(double x) { return atan(x); }
LM_HD float m_exp(float x) { return expf(x); }
LM_HD double m_exp(double x) { return exp(x); }
LM_HD float m_expm1(float x) { return expm1f(x); }
LM_HD double m_expm1(double x) { return expm1(x); }
LM_HD float m_log(float x) { return logf(x); }
LM_HD double m_log(double x) { return log(x); }
LM_HD void m_sincos(float x, float& s, float& c) {
#if defined(__CUDA_ARCH__)
  sincosf(x, &s, &c);
#else
  s = sinf(x); c = cosf(x);
#endif
}
LM_HD void m_sincos(double x, double& s, double& c) {
#if defined(__CUDA_ARCH__)
  sincos(x, &s, &c);
#else
  s = sin(x); c = cos(x);
#endif
}

// Reciprocal and reciprocal square root.  fp32 on the device: one MUFU approximation + one Newton step
// (~1 ulp, 3-4 instructions, no branches) instead of the IEEE division / sqrt sequences whose
// denormal fix-up paths cost ~10 extra instructions and a divergent branch each.
// x = 0 yields inf/NaN exactly like 1/x would; callers select those lanes away.
LM_HD float m_rcp(float x) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return fmaf(r, fmaf(-x, r, 1.0f), r);
#else
  return 1.0f / x;
#endif
}
LM_HD double m_rcp(double x) { return 1.0 / x; }
LM_HD float m_rsqrt(float x) {
#if defined(__CUDA_ARCH__)
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return fmaf(0.5f * y, fmaf(-x * y, y, 1.0f), y);
#else
  return 1.0f / sqrtf(x);
#endif
}
LM_HD double m_rsqrt(double x) { return 1.0 / sqrt(x); }

// pm(x): sign with pm(0) = +1 (reference basics/ops.py:26)
template <typename T> LM_HD T pm(T x) { return x < T(0) ? T(-1) : T(1); }

// ----------------------------------------------------------------------------
// 3-vectors
// ----------------------------------------------------------------------------
template <typename T> struct V3 { T x, y, z; };

template <typename T> LM_HD V3<T> mk(T x, T y, T z) { V3<T> r; r.x = x; r.y = y; r.z = z; return r; }
template <typename T> LM_HD V3<T> ld3(const T* p) { return mk(p[0], p[1], p[2]); }
template <typename T> LM_HD void st3(T* p, const V3<T>& v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
template <typename T> LM_HD V3<T> operator+(const V3<T>& a, const V3<T>& b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
template <typename T> LM_HD V3<T> operator-(const V3<T>& a, const V3<T>& b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
template <typename T> LM_HD V3<T> operator-(const V3<T>& a) { return mk(-a.x, -a.y, -a.z); }
template <typename T> LM_HD V3<T> operator*(T s, const V3<T>& a) { return mk(s * a.x, s * a.y, s * a.z); }
template <typename T> LM_HD T dot(const V3<T>& a, const V3<T>& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> LM_HD V3<T> cross(const V3<T>& a, const V3<T>& b) {
  return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
// a + s*b
template <typename T> LM_HD V3<T> axpy(T s, const V3<T>& b, const V3<T>& a) { return mk(a.x + s * b.x, a.y + s * b.y, a.z + s * b.z); }

// unit-quaternion [v, w]
template <typename T> struct Q4 { V3<T> v; T w; };
template <typename T> LM_HD Q4<T> ldq(const T* p) { Q4<T> q; q.v = ld3(p); q.w = p[3]; return q; }
template <typename T> LM_HD void stq(T* p, const Q4<T>& q) { st3(p, q.v); p[3] = q.w; }

// R(q) p  (op.py:520-525: uv = 2 (v x p); p' = p + w uv + v x uv)
template <typename T> LM_HD V3<T> qrot(const Q4<T>& q, const V3<T>& p) {
  V3<T> uv = cross(q.v, p);
  uv = uv + uv;
  return p + q.w * uv + cross(q.v, uv);
}
// R(q)^T p = rotation by the conjugate
template <typename T> LM_HD V3<T> qrot_t(const Q4<T>& q, const V3<T>& p) {
  V3<T> uv = cross(p, q.v);  // (-v) x p
  uv = uv + uv;
  return p + q.w * uv + cross(uv, q.v);
}
// quaternion product (op.py:833-837)
template <typename T> LM_HD Q4<T> qmul(const Q4<T>& a, const Q4<T>& b) {
  Q4<T> z;
  z.v = a.w * b.v + b.w * a.v + cross(a.v, b.v);
  z.w = a.w * b.w - dot(a.v, b.v);
  return z;
}
template <typename T> LM_HD Q4<T> qconj(const Q4<T>& a) { Q4<T> z; z.v = -a.v; z.w = a.w; return z; }

// ----------------------------------------------------------------------------
// coefficient functions of theta (x = theta^2)
// ----------------------------------------------------------------------------
// All so3/se3 coefficients derived from one sincos of theta/2.
template <typename T> struct RotCoef {
  T theta2, theta;
  T sh, ch;     // sin(theta/2), cos(theta/2)
  T imag;       // sin(theta/2)/theta             (op.py:343-357)
  T c1;         // (1-cos theta)/theta^2          (op.py:14-15)
  T c2;         // (theta - sin theta)/theta^3    (op.py:17-19)
  bool small;
};

template <typename T> LM_HD RotCoef<T> rot_coef(const V3<T>& phi) {
  RotCoef<T> r;
  T x = dot(phi, phi);
  r.theta2 = x;
  r.small = x < num<T>::small2;
  const T inv = m_rsqrt(x);          // 1/theta (inf at 0: only used through selects)
  r.theta = (x > T(1e-30)) ? x * inv : T(0);   // theta < 1e-15 behaves as 0 (cos(theta/2) == 1)
  m_sincos(T(0.5) * r.theta, r.sh, r.ch);
  // both evaluations are computed and selected (FSEL): warps almost always hold both kinds of lanes,
  // so a branch would execute both sides anyway plus the divergence bookkeeping.
  // series in x; remainder < 1e-10 (fp32 window) / 1e-22 (fp64 window)
  const T imag_s = T(0.5) + x * (T(-1.0 / 48) + x * (T(1.0 / 3840) + x * (T(-1.0 / 645120) + x * T(1.0 / 185794560))));
  const T c2_s = T(1.0 / 6) + x * (T(-1.0 / 120) + x * (T(1.0 / 5040) + x * (T(-1.0 / 362880) + x * T(1.0 / 39916800))));
  const T imag_c = r.sh * inv;
  const T c2_c = (r.theta - T(2) * r.sh * r.ch) * inv * inv * inv;     // theta - sin(theta) = theta - 2 sh ch
  r.imag = r.small ? imag_s : imag_c;
  r.c2 = r.small ? c2_s : c2_c;
  r.c1 = T(2) * r.imag * r.imag;  // (1-cos)/theta^2 = 2 sin^2(theta/2)/theta^2, no cancellation
  return r;
}

// coefficient of K^2 in Jl^{-1}: (1 - (theta/2) cot(theta/2)) / theta^2   (op.py:23-32)
// `half_cot` = (theta/2) * cos(theta/2)/sin(theta/2) supplied by the caller when x is not small.
template <typename T> LM_HD T jlinv_series(T x) {
  return T(1.0 / 12) + x * (T(1.0 / 720) + x * (T(1.0 / 30240) + x * (T(1.0 / 1209600) + x * (T(1.0 / 47900160) + x * T(691.0 / 1307674368000.0)))));
}
template <typename T> LM_HD T jlinv_coef(const V3<T>& phi) {
  T x = dot(phi, phi);
  const bool small = x < num<T>::small2;
  T th = x * m_rsqrt(x), s, c;          // NaN at x = 0 is selected away below
  m_sincos(T(0.5) * th, s, c);
  const T closed = (T(1) - T(0.5) * th * c * m_rcp(s)) * m_rcp(x);
  return small ? jlinv_series(x) : closed;
}

// extra coefficients of Q(tau, phi) (op.py:37-58): a1 = c2, a2, a3
template <typename T> LM_HD void q_coef(const RotCoef<T>& r, T& a2, T& a3) {
  const T x = r.theta2;
  const T a2_s = T(1.0 / 24) + x * (T(-1.0 / 720) + x * (T(1.0 / 40320) + x * (T(-1.0 / 3628800) + x * T(1.0 / 479001600))));
  const T a3_s = T(1.0 / 120) + x * (T(-2.0 / 5040) + x * (T(3.0 / 362880) + x * (T(-4.0 / 39916800) + x * T(5.0 / 6227020800.0))));
  const T th = r.theta;
  const T st = T(2) * r.sh * r.ch;               // sin(theta)
  const T one_m_cos = T(2) * r.sh * r.sh;        // 1 - cos(theta)
  const T ix2 = m_rcp(T(2) * x * x);
  const T a2_c = (x - T(2) * one_m_cos) * ix2;                          // (th^2 + 2cos - 2)/(2 th^4)
  const T a3_c = (T(3) * (th - st) - th * one_m_cos) * ix2 * m_rcp(th); // (2th - 3sin + th cos)/(2 th^5)
  a2 = r.small ? a2_s : a2_c;
  a3 = r.small ? a3_s : a3_c;
}

// ----------------------------------------------------------------------------
// so3 <-> SO3
// ----------------------------------------------------------------------------
template <typename T> LM_HD Q4<T> so3_exp(const V3<T>& phi, const RotCoef<T>& r) {
  Q4<T> q; q.v = r.imag * phi; q.w = r.ch; return q;
}

// SO3 Log with the reference's three branches (op.py:308-324); also returns the Jl^{-1} K^2
// coefficient computed from the quaternion itself: cot(theta/2) = w/|v| exactly on the
// principal branch, so no sincos is needed.
template <typename T> LM_HD V3<T> so3_log(const Q4<T>& q, T& jinv_c) {
  const T eps = num<T>::eps;
  const T PI = T(3.14159265358979323846);
  const T n2 = dot(q.v, q.v);
  const T inv_n = m_rsqrt(n2);
  const T n = n2 * inv_n;                // NaN at n2 = 0: that lane takes the third branch below
  const T w = q.w;
  // branch 1 (op.py:320): |v| > eps and |w| > eps
  const T half = m_atan(n * m_rcp(w));   // theta/2 in (-pi/2, pi/2)
  const T x = T(4) * half * half;
  const T f1 = T(2) * half * inv_n;
  const T c1 = (x < num<T>::small2) ? jlinv_series(x) : (T(1) - half * w * inv_n) * m_rcp(x);
  // branch 2 (op.py:321): |w| <= eps -> theta = +-pi
  const T f2 = pm(w) * PI * inv_n;
  const T c2 = T(1) / (PI * PI);
  // branch 3 (op.py:322): |v| <= eps -> series in |v|/w
  const T iw = m_rcp(w);
  const T f3 = T(2) * (iw - n2 * iw * iw * iw * T(1.0 / 3));
  const bool vbig = n2 > eps * eps, wbig = m_abs(w) > eps;
  const T factor = vbig ? (wbig ? f1 : f2) : f3;
  jinv_c = vbig ? (wbig ? c1 : c2) : T(1.0 / 12);
  return factor * q.v;
}

// Jl(phi) u = u + c1 phi x u + c2 phi x (phi x u)           (op.py:7-20)
template <typename T> LM_HD V3<T> jl_apply(const RotCoef<T>& r, const V3<T>& phi, const V3<T>& u) {
  V3<T> a = cross(phi, u);
  return u + r.c1 * a + r.c2 * cross(phi, a);
}
// Jl(phi)^T u  (row-vector product u @ Jl)
template <typename T> LM_HD V3<T> jl_apply_t(const RotCoef<T>& r, const V3<T>& phi, const V3<T>& u) {
  V3<T> a = cross(phi, u);
  return u - r.c1 * a + r.c2 * cross(phi, a);
}
// Jl^{-1}(phi) u = u - 1/2 phi x u + c phi x (phi x u)      (op.py:23-32)
template <typename T> LM_HD V3<T> jlinv_apply(T c, const V3<T>& phi, const V3<T>& u) {
  V3<T> a = cross(phi, u);
  return u - T(0.5) * a + c * cross(phi, a);
}
template <typename T> LM_HD V3<T> jlinv_apply_t(T c, const V3<T>& phi, const V3<T>& u) {
  V3<T> a = cross(phi, u);
  return u + T(0.5) * a + c * cross(phi, a);
}

// Q(tau,phi) g and Q^T g in cross-product form (op.py:37-58).
// Q = 1/2 T + a1 (PT + TP + PTP) + a2 (PPT + TPP - 3 PTP) + a3 (PTPP + PPTP),  P = phi^, T = tau^
template <typename T, bool TRANSPOSE>
LM_HD V3<T> q_apply(const RotCoef<T>& r, const V3<T>& tau, const V3<T>& phi, const V3<T>& g) {
  T a1 = r.c2, a2, a3;
  q_coef(r, a2, a3);
  V3<T> u1 = cross(phi, g);      // P g
  V3<T> u2 = cross(phi, u1);     // PP g
  V3<T> w0 = cross(tau, g);      // T g
  V3<T> w1 = cross(tau, u1);     // TP g
  V3<T> w2 = cross(tau, u2);     // TPP g
  V3<T> p0 = cross(phi, w0);     // PT g
  V3<T> p1 = cross(phi, w1);     // PTP g
  V3<T> p2 = cross(phi, w2);     // PTPP g
  V3<T> pp0 = cross(phi, p0);    // PPT g
  V3<T> pp1 = cross(phi, p1);    // PPTP g
  V3<T> out;
  if (!TRANSPOSE) {
    out = T(0.5) * w0 + a1 * (p0 + w1 + p1) + a2 * (pp0 + w2 - T(3) * p1) + a3 * (p2 + pp1);
  } else {
    // transposes: (PT)^T = TP, (PTP)^T = -PTP, (PPT)^T = -TPP, (PTPP)^T = PPTP
    out = T(-0.5) * w0 + a1 * (w1 + p0 - p1) + a2 * (T(3) * p1 - w2 - pp0) + a3 * (pp1 + p2);
  }
  return out;
}

// ----------------------------------------------------------------------------
// sim3 translation map Ws = A K + B K^2 + C I  (op.py:85-129) and its inverse
// ----------------------------------------------------------------------------
template <typename T> struct WsCoef { T A, B, C; T theta2; };

template <typename T> LM_HD WsCoef<T> ws_coef(const V3<T>& phi, T sigma) {
  WsCoef<T> o;
  T x = dot(phi, phi);
  o.theta2 = x;
  T em1 = m_expm1(sigma);          // s - 1 without cancellation
  T s = em1 + T(1);
  bool sig_small = m_abs(sigma) < num<T>::sig_small;
  // C = (e^sigma - 1)/sigma
  o.C = (m_abs(sigma) > num<T>::eps) ? em1 * m_rcp(sigma) : T(1);
  if (x < num<T>::tiny2) {
    // theta -> 0 limits: A = ((sigma-1)s+1)/sigma^2, B = (s(sigma^2/2 - sigma + 1) - 1)/sigma^3.
    // A multiplies K (|K| = theta) and B multiplies K^2, so first-order accuracy is enough.
    if (sig_small) {
      o.A = T(0.5) + sigma * (T(1.0 / 3) + sigma * (T(1.0 / 8) + sigma * (T(1.0 / 30) + sigma * T(1.0 / 144))));
      o.B = T(1.0 / 6) + sigma * (T(1.0 / 8) + sigma * (T(1.0 / 20) + sigma * T(1.0 / 72)));
    } else {
      T s2 = sigma * sigma;
      const T is2 = m_rcp(s2);
      o.A = ((sigma - T(1)) * s + T(1)) * is2;
      o.B = (s * (T(0.5) * s2 - sigma + T(1)) - T(1)) * is2 * m_rcp(sigma);
    }
    return o;
  }
  T th = m_sqrt(x), sh, ch;
  m_sincos(T(0.5) * th, sh, ch);
  T st = T(2) * sh * ch;            // sin(theta)
  T omc = T(2) * sh * sh;           // 1 - cos(theta)
  T ct = T(1) - omc;                // cos(theta)
  T a = s * st;
  T bm1 = em1 * ct - omc;           // s cos(theta) - 1, cancellation-free
  const T ic = m_rcp(x + sigma * sigma);
  o.A = (a * sigma - bm1 * th) * ic * m_rcp(th);
  o.B = (o.C - (bm1 * sigma + a * th) * ic) * m_rcp(x);
  return o;
}
template <typename T> LM_HD V3<T> ws_apply(const WsCoef<T>& k, const V3<T>& phi, const V3<T>& u) {
  V3<T> a = cross(phi, u);
  return k.C * u + k.A * a + k.B * cross(phi, a);
}
// Ws^{-1} = alpha I + beta K + gamma K^2 (polynomial inverse using K^3 = -theta^2 K); the reference
// calls a numeric 3x3 .inverse() (op.py:473)
template <typename T> LM_HD V3<T> ws_inv_apply(const WsCoef<T>& k, const V3<T>& phi, const V3<T>& u) {
  T D = k.C - k.theta2 * k.B;
  T idet = m_rcp(D * D + k.theta2 * k.A * k.A);
  T alpha = m_rcp(k.C);
  T beta = -k.A * idet;
  T gamma = alpha * (k.A * k.A - k.B * D) * idet;
  V3<T> a = cross(phi, u);
  return alpha * u + beta * a + gamma * cross(phi, a);
}

// ----------------------------------------------------------------------------
// group structs: every group implements the same static interface on raw register rows
//   D   : data width of the group element          K : manifold (tangent) width
// ----------------------------------------------------------------------------
struct SO3g { static constexpr int D = 4, K = 3; };
struct SE3g { static constexpr int D = 7, K = 6; };
struct RxSO3g { static constexpr int D = 5, K = 4; };
struct Sim3g { static constexpr int D = 8, K = 7; };

// unpacked element: translation, rotation, scale (unused members are identity)
template <typename T> struct Elem { V3<T> t; Q4<T> q; T s; };
// unpacked tangent: tau, phi, sigma
template <typename T> struct Tang { V3<T> tau; V3<T> phi; T sigma; };

template <class G, typename T> LM_HD Elem<T> load_elem(const T* p) {
  Elem<T> e; e.t = mk(T(0), T(0), T(0)); e.s = T(1);
  if (G::D == 4) { e.q = ldq(p); }
  else if (G::D == 7) { e.t = ld3(p); e.q = ldq(p + 3); }
  else if (G::D == 5) { e.q = ldq(p); e.s = p[4]; }
  else { e.t = ld3(p); e.q = ldq(p + 3); e.s = p[7]; }
  return e;
}
template <class G, typename T> LM_HD void store_elem(T* p, const Elem<T>& e) {
  if (G::D == 4) { stq(p, e.q); }
  else if (G::D == 7) { st3(p, e.t); stq(p + 3, e.q); }
  else if (G::D == 5) { stq(p, e.q); p[4] = e.s; }
  else { st3(p, e.t); stq(p + 3, e.q); p[7] = e.s; }
}
template <class G, typename T> LM_HD Tang<T> load_tang(const T* p) {
  Tang<T> a; a.tau = mk(T(0), T(0), T(0)); a.sigma = T(0);
  if (G::K == 3) { a.phi = ld3(p); }
  else if (G::K == 6) { a.tau = ld3(p); a.phi = ld3(p + 3); }
  else if (G::K == 4) { a.phi = ld3(p); a.sigma = p[3]; }
  else { a.tau = ld3(p); a.phi = ld3(p + 3); a.sigma = p[6]; }
  return a;
}
template <class G, typename T> LM_HD void store_tang(T* p, const Tang<T>& a) {
  if (G::K == 3) { st3(p, a.phi); }
  else if (G::K == 6) { st3(p, a.tau); st3(p + 3, a.phi); }
  else if (G::K == 4) { st3(p, a.phi); p[3] = a.sigma; }
  else { st3(p, a.tau); st3(p + 3, a.phi); p[6] = a.sigma; }
}
// tangent gradient written into a D-wide group-gradient row: [grad_K, 0]
template <class G, typename T> LM_HD void store_tang_pad(T* p, const Tang<T>& a) {
  store_tang<G, T>(p, a);
  p[G::D - 1] = T(0);
}
template <class G> struct has_t { static constexpr bool v = (G::D == 7 || G::D == 8); };
template <class G> struct has_s { static constexpr bool v = (G::D == 5 || G::D == 8); };

// ---------------------------------------------------------------- Exp / Log
// Exp (op.py:340-357 so3, 398-405 se3, 444-451 rxso3, 492-500 sim3)
template <class G, typename T> LM_HD Elem<T> g_exp(const Tang<T>& a) {
  Elem<T> e; e.t = mk(T(0), T(0), T(0)); e.s = T(1);
  RotCoef<T> r = rot_coef(a.phi);
  e.q = so3_exp(a.phi, r);
  if (G::D == 7) e.t = jl_apply(r, a.phi, a.tau);
  if (has_s<G>::v) e.s = m_exp(a.sigma);
  if (G::D == 8) { WsCoef<T> k = ws_coef(a.phi, a.sigma); e.t = ws_apply(k, a.phi, a.tau); }
  return e;
}
// Log (op.py:304-324 SO3, 373-382 SE3, 421-428 RxSO3, 467-476 Sim3)
template <class G, typename T> LM_HD Tang<T> g_log(const Elem<T>& e) {
  Tang<T> a; a.tau = mk(T(0), T(0), T(0)); a.sigma = T(0);
  T c;
  a.phi = so3_log(e.q, c);
  if (G::D == 7) a.tau = jlinv_apply(c, a.phi, e.t);
  if (has_s<G>::v) a.sigma = m_log(e.s);
  if (G::D == 8) { WsCoef<T> k = ws_coef(a.phi, a.sigma); a.tau = ws_inv_apply(k, a.phi, e.t); }
  return a;
}

// ---------------------------------------------------------------- little adjoint products
// y = ad(x)^T g  (row-vector product g @ ad(x)); ad per op.py:34-35 (so3), 77-83 (se3), 142-145 (rxso3), 147-156 (sim3)
template <class G, typename T> LM_HD Tang<T> ad_t_apply(const Tang<T>& x, const Tang<T>& g) {
  Tang<T> y; y.tau = mk(T(0), T(0), T(0)); y.sigma = T(0);
  if (G::K == 3 || G::K == 4) { y.phi = cross(g.phi, x.phi); }           // K^T g = -phi x g
  else if (G::K == 6) { y.tau = cross(g.tau, x.phi); y.phi = cross(g.tau, x.tau) + cross(g.phi, x.phi); }
  else {
    y.tau = cross(g.tau, x.phi) + x.sigma * g.tau;
    y.phi = cross(g.tau, x.tau) + cross(g.phi, x.phi);
    y.sigma = -dot(x.tau, g.tau);
  }
  return y;
}
// y = ad(x) p
template <class G, typename T> LM_HD Tang<T> ad_apply(const Tang<T>& x, const Tang<T>& p) {
  Tang<T> y; y.tau = mk(T(0), T(0), T(0)); y.sigma = T(0);
  if (G::K == 3 || G::K == 4) { y.phi = cross(x.phi, p.phi); }
  else if (G::K == 6) { y.tau = cross(x.phi, p.tau) + cross(x.tau, p.phi); y.phi = cross(x.phi, p.phi); }
  else {
    y.tau = cross(x.phi, p.tau) + x.sigma * p.tau + cross(x.tau, p.phi) - p.sigma * x.tau;
    y.phi = cross(x.phi, p.phi);
  }
  return y;
}
template <typename T> LM_HD Tang<T> t_axpy(T s, const Tang<T>& b, const Tang<T>& a) {
  Tang<T> y; y.tau = axpy(s, b.tau, a.tau); y.phi = axpy(s, b.phi, a.phi); y.sigma = a.sigma + s * b.sigma; return y;
}

// ---------------------------------------------------------------- left Jacobians as operators
// g @ Jl(x)  (Exp backward: op.py:365-370, 413-418, 459-464, 508-513)
template <class G, typename T> LM_HD Tang<T> jl_t_apply(const Tang<T>& x, const Tang<T>& g) {
  Tang<T> y; y.tau = mk(T(0), T(0), T(0)); y.sigma = T(0);
  if (G::K == 7) {
    // truncated series of the reference (op.py:159-164): I + X/2 + X^2/6 + X^3/24 + X^4/120 + X^5/720
    Tang<T> v = g; y = g;
    const T cf[5] = {T(0.5), T(1.0 / 6), T(1.0 / 24), T(1.0 / 120), T(1.0 / 720)};
#pragma unroll
    for (int k = 0; k < 5; ++k) { v = ad_t_apply<G, T>(x, v); y = t_axpy(cf[k], v, y); }
    return y;
  }
  RotCoef<T> r = rot_coef(x.phi);
  if (G::K == 3) { y.phi = jl_apply_t(r, x.phi, g.phi); }
  else if (G::K == 4) { y.phi = jl_apply_t(r, x.phi, g.phi); y.sigma = g.sigma; }   // blockdiag(Jl,1) op.py:132-135
  else {  // se3: [[J,Q],[0,J]] (op.py:61-65): g @ Jl = [J^T gt, Q^T gt + J^T gr]
    y.tau = jl_apply_t(r, x.phi, g.tau);
    y.phi = q_apply<T, true>(r, x.tau, x.phi, g.tau) + jl_apply_t(r, x.phi, g.phi);
  }
  return y;
}
// g @ Jl^{-1}(x)  (Log backward: op.py:331-337, 389-395, 435-441, 483-489)
template <class G, typename T> LM_HD Tang<T> jlinv_t_apply(const Tang<T>& x, const Tang<T>& g) {
  Tang<T> y; y.tau = mk(T(0), T(0), T(0)); y.sigma = T(0);
  if (G::K == 7) {
    // op.py:167-172: I - X/2 + X^2/12 - X^4/720
    Tang<T> v1 = ad_t_apply<G, T>(x, g);
    Tang<T> v2 = ad_t_apply<G, T>(x, v1);
    Tang<T> v3 = ad_t_apply<G, T>(x, v2);
    Tang<T> v4 = ad_t_apply<G, T>(x, v3);
    y = t_axpy(T(-0.5), v1, g); y = t_axpy(T(1.0 / 12), v2, y); y = t_axpy(T(-1.0 / 720), v4, y);
    return y;
  }
  T c = jlinv_coef(x.phi);
  if (G::K == 3) { y.phi = jlinv_apply_t(c, x.phi, g.phi); }
  else if (G::K == 4) { y.phi = jlinv_apply_t(c, x.phi, g.phi); y.sigma = g.sigma; }
  else {  // se3 (op.py:68-75): [[Ji, -Ji Q Ji],[0,Ji]]: g @ = [h, Ji^T (gr - Q^T h)], h = Ji^T gt
    RotCoef<T> r = rot_coef(x.phi);
    V3<T> h = jlinv_apply_t(c, x.phi, g.tau);
    y.tau = h;
    y.phi = jlinv_apply_t(c, x.phi, g.phi - q_apply<T, true>(r, x.tau, x.phi, h));
  }
  return y;
}
// Jl^{-1}(x) p  (Jinvp: lietensor.py:257-264, 422-429, 556-563, 700-707)
template <class G, typename T> LM_HD Tang<T> jlinv_apply_g(const Tang<T>& x, const Tang<T>& p) {
  Tang<T> y; y.tau = mk(T(0), T(0), T(0)); y.sigma = T(0);
  if (G::K == 7) {
    Tang<T> v1 = ad_apply<G, T>(x, p);
    Tang<T> v2 = ad_apply<G, T>(x, v1);
    Tang<T> v3 = ad_apply<G, T>(x, v2);
    Tang<T> v4 = ad_apply<G, T>(x, v3);
    y = t_axpy(T(-0.5), v1, p); y = t_axpy(T(1.0 / 12), v2, y); y = t_axpy(T(-1.0 / 720), v4, y);
    return y;
  }
  T c = jlinv_coef(x.phi);
  if (G::K == 3) { y.phi = jlinv_apply(c, x.phi, p.phi); }
  else if (G::K == 4) { y.phi = jlinv_apply(c, x.phi, p.phi); y.sigma = p.sigma; }
  else {
    RotCoef<T> r = rot_coef(x.phi);
    V3<T> h = jlinv_apply(c, x.phi, p.phi);
    y.phi = h;
    y.tau = jlinv_apply(c, x.phi, p.tau - q_apply<T, false>(r, x.tau, x.phi, h));
  }
  return y;
}

// ---------------------------------------------------------------- group ops
// Inv (op.py:930-936, 952-960, 976-984, 1000-1008)
template <class G, typename T> LM_HD Elem<T> g_inv(const Elem<T>& X) {
  Elem<T> Y; Y.q = qconj(X.q); Y.s = T(1); Y.t = mk(T(0), T(0), T(0));
  if (has_s<G>::v) Y.s = m_rcp(X.s);
  if (has_t<G>::v) { V3<T> r = qrot(Y.q, X.t); Y.t = -(Y.s * r); }
  return Y;
}
// Mul (op.py:829-837, 855-862, 880-887, 905-912)
template <class G, typename T> LM_HD Elem<T> g_mul(const Elem<T>& X, const Elem<T>& Y) {
  Elem<T> Z; Z.q = qmul(X.q, Y.q); Z.s = X.s * Y.s; Z.t = mk(T(0), T(0), T(0));
  if (has_t<G>::v) Z.t = X.t + X.s * qrot(X.q, Y.t);
  return Z;
}
// Act on a 3-vector (op.py:516-525, 545-551, 571-577, 597-603)
template <class G, typename T> LM_HD V3<T> g_act(const Elem<T>& X, const V3<T>& p) {
  V3<T> o = qrot(X.q, p);
  if (has_s<G>::v) o = X.s * o;
  if (has_t<G>::v) o = o + X.t;
  return o;
}
// Adj(X) a  (op.py:175-179, 202-210, 237-240, 268-276)
template <class G, typename T> LM_HD Tang<T> g_adj(const Elem<T>& X, const Tang<T>& a) {
  Tang<T> y; y.tau = mk(T(0), T(0), T(0)); y.sigma = a.sigma;
  y.phi = qrot(X.q, a.phi);
  if (G::K == 6) y.tau = qrot(X.q, a.tau) + cross(X.t, y.phi);
  if (G::K == 7) y.tau = X.s * qrot(X.q, a.tau) + cross(X.t, y.phi) - a.sigma * X.t;
  return y;
}
// g @ Adj(X) = Adj(X)^T g
template <class G, typename T> LM_HD Tang<T> g_adj_t(const Elem<T>& X, const Tang<T>& g) {
  Tang<T> y; y.tau = mk(T(0), T(0), T(0)); y.sigma = g.sigma;
  if (G::K == 3 || G::K == 4) { y.phi = qrot_t(X.q, g.phi); }
  else {
    V3<T> rt = qrot_t(X.q, g.tau);
    y.tau = (G::K == 7) ? X.s * rt : rt;
    y.phi = qrot_t(X.q, g.phi - cross(X.t, g.tau));
    if (G::K == 7) y.sigma = g.sigma - dot(X.t, g.tau);
  }
  return y;
}
template <typename T> LM_HD Tang<T> t_neg(const Tang<T>& a) { Tang<T> y; y.tau = -a.tau; y.phi = -a.phi; y.sigma = -a.sigma; return y; }

}  // namespace b200pose
