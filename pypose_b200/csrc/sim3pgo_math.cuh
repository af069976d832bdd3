// sim3pgo_math.cuh — per-edge math of the Sim3 pose graph (host+device, see lie_math.cuh).
//
// Residual of the reference's examples/module/pgo `PoseGraph` on Sim3 nodes: r_e = Log(Z_e^-1 A^-1 B) in R^7 = [tau phi sigma],
// A = nodes[i], B = nodes[j].  With S = Z^-1 A^-1 the reference's autograd Jacobian with respect to B (left perturbation,
// 7 tangent columns) is
//   J = sim3_Jl_inv(r) Adj(S),   J_A = -J,
// where sim3_Jl_inv is the reference's TRUNCATED series I - X/2 + X^2/12 - X^4/720 of X = ad(r) (operation.py:167-172),
// not the exact inverse left Jacobian: at large residuals the two differ, and the route follows the reference.  The 8th
// column of the reference's dense Jacobian is identically zero (its step component is 0), so 7 unknowns per node give the
// same step.  An edge contributes M = J^T J to both diagonal blocks and u = J^T r with the endpoint's sign, as on SE3.
// Symmetric 7x7 blocks are packed as their row-major upper triangle (28 words).
#pragma once
#include "bal_math.cuh"

namespace b200pose {

constexpr int kSim3 = 7;                          // unknowns per node
constexpr int kSim3Packed = 28;                   // packed upper triangle of a 7x7 block

template <typename T> LM_HD Tang<T> sim3pgo_residual(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Elem<T>& S) {
  S = g_mul<Sim3g, T>(g_inv<Sim3g, T>(Z), g_inv<Sim3g, T>(A));
  return g_log<Sim3g, T>(g_mul<Sim3g, T>(S, B));
}
template <typename T> LM_HD T tang7_sqnorm(const Tang<T>& r) { return dot(r.tau, r.tau) + dot(r.phi, r.phi) + r.sigma * r.sigma; }

// J = dr/dB (7x7), column by column: J e_k = Jl^-1(r) (Adj(S) e_k)
template <typename T>
LM_HD void sim3pgo_jacobian(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Tang<T>& r, T (&J)[7][7]) {
  Elem<T> S;
  r = sim3pgo_residual(A, B, Z, S);
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    T e[7], c[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) e[i] = i == k ? T(1) : T(0);
    store_tang<Sim3g, T>(c, jlinv_apply_g<Sim3g, T>(r, g_adj<Sim3g, T>(S, load_tang<Sim3g, T>(e))));
#pragma unroll
    for (int i = 0; i < 7; ++i) J[i][k] = c[i];
  }
}

// M = J^T J (packed, 28) and u = J^T r of one edge
template <typename T>
LM_HD void sim3pgo_linearize(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Tang<T>& r, T (&M)[28], T (&u)[7]) {
  T J[7][7], rr[7];
  sim3pgo_jacobian(A, B, Z, r, J);
  store_tang<Sim3g, T>(rr, r);
  int q = 0;
#pragma unroll
  for (int a = 0; a < 7; ++a) {
    T g = T(0);
#pragma unroll
    for (int k = 0; k < 7; ++k) g += J[k][a] * rr[k];
    u[a] = g;
#pragma unroll
    for (int b = a; b < 7; ++b) {
      T v = T(0);
#pragma unroll
      for (int k = 0; k < 7; ++k) v += J[k][a] * J[k][b];
      M[q++] = v;
    }
  }
}
// robust weighting of one edge's blocks (FastTriggs, as sys6_scale)
template <typename T> LM_HD void sys7_scale(T (&M)[28], T (&u)[7], T w) {
#pragma unroll
  for (int k = 0; k < 28; ++k) M[k] *= w;
#pragma unroll
  for (int k = 0; k < 7; ++k) u[k] *= w;
}

}  // namespace b200pose
