// so3pgo_math.cuh — per-edge math of the SO3 pose graph (rotation averaging; host+device, see lie_math.cuh).
//
// Residual of the reference's examples/module/pgo `PoseGraph` on SO3 nodes: r_e = Log(Z_e^-1 A^-1 B) in R^3,
// A = nodes[i], B = nodes[j].  With S = Z^-1 A^-1 the reference's autograd Jacobian with respect to B (left perturbation,
// 3 tangent columns) is
//   J = Jl^-1(r) Adj(S) = Jl^-1(r) R(S),   J_A = -J,
// where Jl^-1(r) = I - K/2 + c2 K^2, K = [r]x, is the reference's so3_Jl_inv (operation.py:23-32; c2 = 1/12 at theta <= eps,
// which jlinv_coef's series gives to rounding).  The reference's dense Jacobian has 4 columns per SO3 node and the 4th is
// identically zero (SO3_Log.backward pads the gradient with a zero), so 3 unknowns per node give the same step.  An edge
// contributes M = J^T J to both diagonal blocks and u = J^T r with the endpoint's sign, as on SE3.  Symmetric 3x3 blocks
// are packed as their row-major upper triangle (6 words).
#pragma once
#include "bal_math.cuh"

namespace b200pose {

constexpr int kSo3 = 3;                           // unknowns per node
constexpr int kSo3Packed = 6;                     // packed upper triangle of a 3x3 block

template <typename T> LM_HD Tang<T> so3pgo_residual(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Elem<T>& S) {
  S = g_mul<SO3g, T>(g_inv<SO3g, T>(Z), g_inv<SO3g, T>(A));
  return g_log<SO3g, T>(g_mul<SO3g, T>(S, B));
}
template <typename T> LM_HD T tang3_sqnorm(const Tang<T>& r) { return dot(r.phi, r.phi); }

// J = dr/dB (3x3), column by column: J e_k = Jl^-1(r) (Adj(S) e_k)
template <typename T>
LM_HD void so3pgo_jacobian(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Tang<T>& r, T (&J)[3][3]) {
  Elem<T> S;
  r = so3pgo_residual(A, B, Z, S);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    T e[3], c[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) e[i] = i == k ? T(1) : T(0);
    store_tang<SO3g, T>(c, jlinv_apply_g<SO3g, T>(r, g_adj<SO3g, T>(S, load_tang<SO3g, T>(e))));
#pragma unroll
    for (int i = 0; i < 3; ++i) J[i][k] = c[i];
  }
}

// M = J^T J (packed, 6) and u = J^T r of one edge
template <typename T>
LM_HD void so3pgo_linearize(const Elem<T>& A, const Elem<T>& B, const Elem<T>& Z, Tang<T>& r, T (&M)[6], T (&u)[3]) {
  T J[3][3], rr[3];
  so3pgo_jacobian(A, B, Z, r, J);
  store_tang<SO3g, T>(rr, r);
  int q = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    T g = T(0);
#pragma unroll
    for (int k = 0; k < 3; ++k) g += J[k][a] * rr[k];
    u[a] = g;
#pragma unroll
    for (int b = a; b < 3; ++b) {
      T v = T(0);
#pragma unroll
      for (int k = 0; k < 3; ++k) v += J[k][a] * J[k][b];
      M[q++] = v;
    }
  }
}
// robust weighting of one edge's blocks (FastTriggs, as sys7_scale)
template <typename T> LM_HD void sys3_scale(T (&M)[6], T (&u)[3], T w) {
#pragma unroll
  for (int k = 0; k < 6; ++k) M[k] *= w;
#pragma unroll
  for (int k = 0; k < 3; ++k) u[k] *= w;
}

}  // namespace b200pose
