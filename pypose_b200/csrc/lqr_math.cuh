// lqr_math.cuh — per-problem math of the affine LQR route (csrc/lqr.cu, DESIGN.md §3.7), compiled for the device and for
// the host (tests/lqr_host.cpp).  One problem is solved by a group of `stride` lanes; every loop runs `for (i = lane; i <
// N; i += stride)`, so the device runs it with one warp (stride 32) and the host with one lane (0, 1).  The lanes of a
// problem share the scratch `LqrSmem` (shared memory on the device).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define LQR_HD __host__ __device__ __forceinline__
#else
#define LQR_HD inline
#endif

namespace b200pose {

// an operand read at (problem b, step t) with element strides; a NULL pointer reads as zeros
template <class T>
struct LqrOp {
  const T* p;
  long long sb, st;
  LQR_HD const T* at(long long b, int t) const { return p + b * sb + (long long)t * st; }
};

template <class T>
struct LqrProb {
  LqrOp<T> Q, p, A, B, c1, u0;   // (n,n), (n), (ns,ns), (ns,nc), (ns) or NULL, (nc) or NULL per problem and step
  const T* x0;                   // (nb, ns)
  int steps, ns, nc;
};

// gradient outputs, per problem (nb, T or 1, ...) contiguous; tv = 0: summed over the steps
template <class T>
struct LqrGrad {
  T *Q, *p, *A, *B, *c1, *x0;
  int Qtv, ptv, Atv, Btv, c1tv;
};

struct LqrLane {
  int lane, stride;
  LQR_HD void sync() const {
#ifdef __CUDA_ARCH__
    __syncwarp();
#endif
  }
  LQR_HD double sum(double v) const {
#ifdef __CUDA_ARCH__
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
    return v;
  }
};

LQR_HD float lqr_sqrt(float x) { return sqrtf(x); }
LQR_HD double lqr_sqrt(double x) { return sqrt(x); }

template <class T>
struct LqrSmem {
  T *Qt, *H, *F, *V, *L, *K, *q, *v, *tau, *w, *e, *lam, *dlam;
};

// elements of T per problem, rounded up to even so that every problem's slab stays 8-byte aligned (all accesses are scalar)
LQR_HD int lqr_smem_elems(int ns, int nc) {
  const int n = ns + nc;
  const int e = n * n + 2 * n * ns + ns * ns + nc * nc + nc * (ns + 1) + 4 * n + 3 * ns;
  return (e + 1) & ~1;
}

template <class T>
LQR_HD LqrSmem<T> lqr_carve(T* s, int ns, int nc) {
  const int n = ns + nc;
  LqrSmem<T> m;
  m.Qt = s; s += n * n;
  m.H = s; s += n * ns;
  m.F = s; s += ns * n;
  m.V = s; s += ns * ns;
  m.L = s; s += nc * nc;
  m.K = s; s += nc * (ns + 1);
  m.q = s; s += n;
  m.tau = s; s += n;
  m.w = s; s += n;
  m.e = s; s += n;
  m.v = s; s += ns;
  m.lam = s; s += ns;
  m.dlam = s;
  return m;
}

// F = [A_t B_t]  (ns, n)
template <class T>
LQR_HD void lqr_load_F(const LqrProb<T>& P, long long b, int t, T* F, LqrLane l) {
  const int ns = P.ns, nc = P.nc, n = ns + nc;
  const T* A = P.A.at(b, t);
  const T* B = P.B.at(b, t);
  for (int i = l.lane; i < ns * n; i += l.stride) {
    const int r = i / n, c = i % n;
    F[i] = c < ns ? A[r * ns + c] : B[r * nc + c - ns];
  }
}

// y = Q_t tau + p_t  (n)
template <class T>
LQR_HD void lqr_Qtau_p(const LqrProb<T>& P, long long b, int t, const T* tau, T* y, LqrLane l) {
  const int n = P.ns + P.nc;
  const T* Q = P.Q.at(b, t);
  const T* p = P.p.at(b, t);
  for (int i = l.lane; i < n; i += l.stride) {
    T s = 0;
    for (int j = 0; j < n; ++j) s += Q[i * n + j] * tau[j];
    y[i] = s + p[i];
  }
}

// One step of the backward (Riccati) recursion, in the reference's order (pypose/module/lqr.py:330-353):
//   Qt = Q_t + (F^T V) F  (when quad),  q = q + F^T v  (when lin; q holds the step's own linear term on entry),
//   L = chol(Quu),  [K | k] = -Quu^{-1} [Qux | qu],
//   V = Qxx + Qxu K + K^T Qux + (K^T Quu) K,  v = qx + Qxu k + K^T qu + (K^T Quu) k.
// F holds F_t when quad or lin.  Writes [K | k] (nc, ns+1) to Kout.  Returns false when Quu is not positive definite;
// the decision is the same on every lane.
template <class T>
LQR_HD bool lqr_riccati_step(const LqrProb<T>& P, long long b, int t, bool quad, bool lin, LqrSmem<T>& s, T* Kout,
                             LqrLane l) {
  const int ns = P.ns, nc = P.nc, n = ns + nc, kw = ns + 1;
  if (lin)
    for (int i = l.lane; i < n; i += l.stride) {
      T a = 0;
      for (int m = 0; m < ns; ++m) a += s.F[m * n + i] * s.v[m];
      s.q[i] += a;
    }
  if (quad) {
    for (int idx = l.lane; idx < n * ns; idx += l.stride) {
      const int i = idx / ns, k = idx % ns;
      T a = 0;
      for (int m = 0; m < ns; ++m) a += s.F[m * n + i] * s.V[m * ns + k];
      s.H[idx] = a;
    }
    l.sync();
  }
  const T* Q = P.Q.at(b, t);
  for (int idx = l.lane; idx < n * n; idx += l.stride) {
    const int i = idx / n, j = idx % n;
    T a = Q[idx];
    if (quad) {
      T h = 0;
      for (int k = 0; k < ns; ++k) h += s.H[i * ns + k] * s.F[k * n + j];
      a += h;
    }
    s.Qt[idx] = a;
  }
  l.sync();
  // Cholesky of Quu (lower, dpotf2's column order: diagonal, then the column below it scaled by 1 / L_cc)
  const T* Quu = s.Qt + ns * n + ns;
  for (int c = 0; c < nc; ++c) {
    T d = Quu[c * n + c];
    for (int k = 0; k < c; ++k) d -= s.L[c * nc + k] * s.L[c * nc + k];
    if (!(d > T(0))) return false;
    const T ljj = lqr_sqrt(d), r = T(1) / ljj;
    for (int rr = c + 1 + l.lane; rr < nc; rr += l.stride) {
      T a = Quu[rr * n + c];
      for (int k = 0; k < c; ++k) a -= s.L[rr * nc + k] * s.L[c * nc + k];
      s.L[rr * nc + c] = a * r;
    }
    if (l.lane == 0) s.L[c * nc + c] = ljj;
    l.sync();
  }
  // one lane per right-hand side: the ns columns of Qux, then qu
  for (int j = l.lane; j <= ns; j += l.stride) {
    T* y = s.K + j;
    for (int r = 0; r < nc; ++r) {
      T a = j < ns ? s.Qt[(ns + r) * n + j] : s.q[ns + r];
      for (int k = 0; k < r; ++k) a -= s.L[r * nc + k] * y[k * kw];
      y[r * kw] = a / s.L[r * nc + r];
    }
    for (int r = nc - 1; r >= 0; --r) {
      T a = y[r * kw];
      for (int k = r + 1; k < nc; ++k) a -= s.L[k * nc + r] * y[k * kw];
      y[r * kw] = a / s.L[r * nc + r];
    }
    for (int r = 0; r < nc; ++r) y[r * kw] = -y[r * kw];
  }
  l.sync();
  // W = K^T Quu (ns, nc), kept in H
  for (int idx = l.lane; idx < ns * nc; idx += l.stride) {
    const int i = idx / nc, c = idx % nc;
    T a = 0;
    for (int d = 0; d < nc; ++d) a += s.K[d * kw + i] * Quu[d * n + c];
    s.H[idx] = a;
  }
  l.sync();
  for (int idx = l.lane; idx < ns * ns + ns; idx += l.stride) {
    const bool vec = idx >= ns * ns;
    const int i = vec ? idx - ns * ns : idx / ns, j = vec ? ns : idx % ns;   // column ns of K is k
    T a1 = 0, a2 = 0, a3 = 0;
    for (int c = 0; c < nc; ++c) {
      a1 += s.Qt[i * n + ns + c] * s.K[c * kw + j];
      a2 += s.K[c * kw + i] * (vec ? s.q[ns + c] : s.Qt[(ns + c) * n + j]);
      a3 += s.H[i * nc + c] * s.K[c * kw + j];
    }
    const T r = ((vec ? s.q[i] : s.Qt[i * n + j]) + a1 + a2) + a3;
    if (vec) s.v[i] = r; else s.V[idx] = r;
  }
  for (int idx = l.lane; idx < nc * kw; idx += l.stride) Kout[idx] = s.K[idx];
  l.sync();
  return true;
}

// x_next = A_t x + B_t u (+ c1_t), with x = xu[0:ns], u = xu[ns:n] (u == NULL: B_t 0 is added)
template <class T>
LQR_HD void lqr_step_state(const LqrProb<T>& P, long long b, int t, const T* x, const T* u, T* out, LqrLane l) {
  const int ns = P.ns, nc = P.nc;
  const T* A = P.A.at(b, t);
  const T* B = P.B.at(b, t);
  const T* c1 = P.c1.p ? P.c1.at(b, t) : nullptr;
  for (int i = l.lane; i < ns; i += l.stride) {
    T a = 0, bb = 0;
    for (int j = 0; j < ns; ++j) a += A[i * ns + j] * x[j];
    for (int c = 0; c < nc; ++c) bb += B[i * nc + c] * (u ? u[c] : T(0));
    T y = a + bb;
    if (c1) y += c1[i];
    out[i] = y;
  }
}

// The forward solve of one problem b: the rollout of u_traj (runsys), the backward recursion on p_bar = Q tau* + p and
// the rollout du = K dx + k with the cost (pypose/module/lqr.py:310-380).  ws: T * nc * (ns+1) elements for [K_t | k_t].
// Returns 1 when a Quu is not positive definite (the outputs of b are then incomplete).
template <class T>
LQR_HD int lqr_solve(const LqrProb<T>& P, long long b, LqrSmem<T> s, T* ws, T* x, T* u, T* cost, T* xtr, LqrLane l) {
  const int ns = P.ns, nc = P.nc, n = ns + nc, TT = P.steps, kw = nc * (ns + 1);
  const T* x0 = P.x0 + b * ns;
  T* xb = x + b * (TT + 1) * ns;
  T* ub = u + b * TT * nc;
  T* xt = xtr + b * TT * ns;
  for (int i = l.lane; i < ns; i += l.stride) s.tau[i] = xt[i] = x0[i];
  l.sync();
  for (int t = 0; t + 1 < TT; ++t) {
    lqr_step_state(P, b, t, s.tau, P.u0.p ? P.u0.at(b, t) : nullptr, s.w, l);
    l.sync();
    for (int i = l.lane; i < ns; i += l.stride) s.tau[i] = xt[(t + 1) * ns + i] = s.w[i];
    l.sync();
  }
  for (int t = TT - 1; t >= 0; --t) {
    const T* u0 = P.u0.p ? P.u0.at(b, t) : nullptr;
    for (int i = l.lane; i < n; i += l.stride) s.tau[i] = i < ns ? xt[t * ns + i] : (u0 ? u0[i - ns] : T(0));
    const bool chain = t < TT - 1;
    if (chain) lqr_load_F(P, b, t, s.F, l);
    l.sync();
    lqr_Qtau_p(P, b, t, s.tau, s.q, l);
    l.sync();
    if (!lqr_riccati_step(P, b, t, chain, chain, s, ws + (long long)t * kw, l)) return 1;
  }
  double c = 0;
  for (int i = l.lane; i < ns; i += l.stride) s.tau[i] = xb[i] = x0[i];
  l.sync();
  for (int t = 0; t < TT; ++t) {
    const T* K = ws + (long long)t * kw;
    const T* u0 = P.u0.p ? P.u0.at(b, t) : nullptr;
    for (int i = l.lane; i < ns; i += l.stride) s.w[i] = s.tau[i] - xt[t * ns + i];
    l.sync();
    for (int r = l.lane; r < nc; r += l.stride) {
      T a = 0;
      for (int j = 0; j < ns; ++j) a += K[r * (ns + 1) + j] * s.w[j];
      const T du = a + K[r * (ns + 1) + ns];
      s.tau[ns + r] = ub[t * nc + r] = du + (u0 ? u0[r] : T(0));
    }
    l.sync();
    const T* Q = P.Q.at(b, t);
    const T* p = P.p.at(b, t);
    double quad = 0, lin = 0;
    for (int j = l.lane; j < n; j += l.stride) {
      double a = 0;
      for (int i = 0; i < n; ++i) a += (double)s.tau[i] * (double)Q[i * n + j];
      quad += a * (double)s.tau[j];
      lin += (double)s.tau[j] * (double)p[j];
    }
    c += 0.5 * l.sum(quad) + l.sum(lin);
    lqr_step_state(P, b, t, s.tau, s.tau + ns, s.w, l);
    l.sync();
    for (int i = l.lane; i < ns; i += l.stride) s.tau[i] = xb[(t + 1) * ns + i] = s.w[i];
    l.sync();
  }
  if (l.lane == 0) cost[b] = (T)c;
  return 0;
}

template <class T>
LQR_HD void lqr_put(T* g, int tv, long long per, long long b, int TT, int t, int idx, T val) {
  T* base = g + b * (tv ? TT : 1) * per;
  if (tv) base[t * per + idx] = val;
  else base[idx] = t == TT - 1 ? val : base[idx] + val;
}

// The KKT adjoint of one problem b at its solution (x, u), for the cotangents gx (T+1, ns), gu (T, nc), gc (1); any of
// them NULL reads as 0.  One more LQR solve with the same Q_t, F_t, the linear term -g_tau (g_tau = [gx_t; gu_t] +
// gc (Q_t tau_t + p_t)) and the terminal term -gx_T from a zero initial state gives d_tau; then, backwards, the duals
// lam (of the solution) and dlam (of the adjoint) and the gradients
//   dQ_t = -sym(d_tau tau^T) + gc tau tau^T / 2,  dp_t = -d_tau + gc tau,  dF_t = -(lam_{t+1} d_tau^T + dlam_{t+1} tau^T),
//   dc1_t = -dlam_{t+1},  dx_init = -dlam_0.
// ws: T * (nc * (ns+1) + n) elements.
template <class T>
LQR_HD void lqr_adjoint(const LqrProb<T>& P, long long b, LqrSmem<T> s, T* ws, const T* x, const T* u, const T* gx,
                        const T* gu, const T* gc, LqrGrad<T> G, LqrLane l) {
  const int ns = P.ns, nc = P.nc, n = ns + nc, TT = P.steps, kw = nc * (ns + 1);
  const T* xb = x + b * (TT + 1) * ns;
  const T* ub = u + b * TT * nc;
  const T* gxb = gx ? gx + b * (TT + 1) * ns : nullptr;
  const T* gub = gu ? gu + b * TT * nc : nullptr;
  const T g0 = gc ? gc[b] : T(0);
  T* D = ws + (long long)TT * kw;
  auto tau_at = [&](int t) {
    for (int i = l.lane; i < n; i += l.stride) s.tau[i] = i < ns ? xb[t * ns + i] : ub[t * nc + i - ns];
  };
  auto gtau = [&](int t, int i) { return (i < ns ? (gxb ? gxb[t * ns + i] : T(0)) : (gub ? gub[t * nc + i - ns] : T(0))); };
  for (int i = l.lane; i < ns; i += l.stride) s.v[i] = gxb ? -gxb[TT * ns + i] : T(0);
  for (int t = TT - 1; t >= 0; --t) {
    tau_at(t);
    lqr_load_F(P, b, t, s.F, l);
    l.sync();
    lqr_Qtau_p(P, b, t, s.tau, s.w, l);
    for (int i = l.lane; i < n; i += l.stride) s.q[i] = -(gtau(t, i) + g0 * s.w[i]);
    l.sync();
    lqr_riccati_step(P, b, t, t < TT - 1, true, s, ws + (long long)t * kw, l);
  }
  for (int i = l.lane; i < ns; i += l.stride) s.tau[i] = T(0);
  l.sync();
  for (int t = 0; t < TT; ++t) {
    const T* K = ws + (long long)t * kw;
    for (int r = l.lane; r < nc; r += l.stride) {
      T a = 0;
      for (int j = 0; j < ns; ++j) a += K[r * (ns + 1) + j] * s.tau[j];
      s.tau[ns + r] = a + K[r * (ns + 1) + ns];
    }
    l.sync();
    for (int i = l.lane; i < n; i += l.stride) D[(long long)t * n + i] = s.tau[i];
    lqr_step_state<T>(LqrProb<T>{P.Q, P.p, P.A, P.B, LqrOp<T>{nullptr, 0, 0}, P.u0, P.x0, P.steps, P.ns, P.nc}, b, t, s.tau,
                      s.tau + ns, s.w, l);
    l.sync();
    for (int i = l.lane; i < ns; i += l.stride) s.tau[i] = s.w[i];
    l.sync();
  }
  for (int i = l.lane; i < ns; i += l.stride) {
    s.lam[i] = T(0);
    s.dlam[i] = gxb ? -gxb[TT * ns + i] : T(0);
  }
  for (int t = TT - 1; t >= 0; --t) {
    tau_at(t);
    for (int i = l.lane; i < n; i += l.stride) s.e[i] = D[(long long)t * n + i];   // d_tau
    lqr_load_F(P, b, t, s.F, l);
    l.sync();
    lqr_Qtau_p(P, b, t, s.tau, s.q, l);
    for (int idx = l.lane; idx < ns * n; idx += l.stride) {
      const int i = idx / n, j = idx % n;
      const T val = -(s.lam[i] * s.e[j] + s.dlam[i] * s.tau[j]);
      if (j < ns) lqr_put(G.A, G.Atv, (long long)ns * ns, b, TT, t, i * ns + j, val);
      else lqr_put(G.B, G.Btv, (long long)ns * nc, b, TT, t, i * nc + j - ns, val);
    }
    for (int idx = l.lane; idx < n * n; idx += l.stride) {
      const int i = idx / n, j = idx % n;
      const T val = T(-0.5) * (s.e[i] * s.tau[j] + s.tau[i] * s.e[j]) + T(0.5) * g0 * s.tau[i] * s.tau[j];
      lqr_put(G.Q, G.Qtv, (long long)n * n, b, TT, t, idx, val);
    }
    for (int i = l.lane; i < n; i += l.stride) lqr_put(G.p, G.ptv, (long long)n, b, TT, t, i, -s.e[i] + g0 * s.tau[i]);
    if (G.c1)
      for (int i = l.lane; i < ns; i += l.stride) lqr_put(G.c1, G.c1tv, (long long)ns, b, TT, t, i, -s.dlam[i]);
    l.sync();
    const T* Q = P.Q.at(b, t);
    for (int i = l.lane; i < ns; i += l.stride) {
      T fl = 0, fd = 0, qd = 0;
      for (int m = 0; m < ns; ++m) {
        fl += s.F[m * n + i] * s.lam[m];
        fd += s.F[m * n + i] * s.dlam[m];
      }
      for (int j = 0; j < n; ++j) qd += Q[i * n + j] * s.e[j];
      s.H[i] = s.q[i] + fl;
      s.H[ns + i] = qd + fd - (gtau(t, i) + g0 * s.q[i]);
    }
    l.sync();
    for (int i = l.lane; i < ns; i += l.stride) {
      s.lam[i] = s.H[i];
      s.dlam[i] = s.H[ns + i];
    }
    l.sync();
  }
  for (int i = l.lane; i < ns; i += l.stride) G.x0[b * ns + i] = -s.dlam[i];
}

}  // namespace b200pose
