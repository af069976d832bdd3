// TEST-ONLY: host build of csrc/bal_math.cuh for tests/test_bal.py (compiled by the test into a temporary directory
// with -ffp-contract=off): Jacobian rows, packed 9x9 blocks and the damped 9x9 inverse, in fp64.
#include "bal_math.cuh"

using namespace b200pose;

extern "C" {

// per observation: y (3) = T_c p (given), camera rows (2,9) and point rows (2,3); q (4) the camera quaternion,
// K (3) = (f, k1, k2), sw the robust scale
void bal_host_rows(const double* y, const double* q, const double* K, double sw, double* jc, double* jp, long long m) {
  for (long long k = 0; k < m; ++k) {
    Q4<double> qq;
    qq.v = mk(q[k * 4], q[k * 4 + 1], q[k * 4 + 2]);
    qq.w = q[k * 4 + 3];
    BalRows<double> R;
    bal_rows(mk(y[k * 3], y[k * 3 + 1], y[k * 3 + 2]), qq, K[k * 3], K[k * 3 + 1], K[k * 3 + 2], sw, R);
    for (int a = 0; a < 9; ++a) { jc[k * 18 + a] = R.jc0[a]; jc[k * 18 + 9 + a] = R.jc1[a]; }
    for (int a = 0; a < 3; ++a) { jp[k * 6 + a] = R.jp0[a]; jp[k * 6 + 3 + a] = R.jp1[a]; }
  }
}

// H (45) = sum_k jc0 jc0^T + jc1 jc1^T over m pairs of rows jc (m,2,9)
void bal_host_sum_rows(const double* jc, double* H, long long m) {
  for (int a = 0; a < 45; ++a) H[a] = 0.0;
  for (long long k = 0; k < m; ++k) {
    double j0[9], j1[9];
    for (int a = 0; a < 9; ++a) { j0[a] = jc[k * 18 + a]; j1[a] = jc[k * 18 + 9 + a]; }
    sym9_add_rows(H, j0, j1);
  }
}

// y = A x for a packed block A (45) and the inverse of clamp(diag, dmin, dmax) * scale, packed
void bal_host_block(const double* H, const double* x, double scale, double dmin, double dmax, double* y, double* Hinv) {
  double xv[9], yv[9];
  for (int a = 0; a < 9; ++a) xv[a] = x[a];
  symn_mv_packed<double, 9>(H, xv, yv);
  for (int a = 0; a < 9; ++a) y[a] = yv[a];
  double A[9][9], Ai[9][9];
  symn_unpack<double, 9>(H, A);
  blk9_damp(A, scale, dmin, dmax);
  spd_inverse<double, 9>(A, Ai);
  symn_pack<double, 9>(Ai, Hinv);
}

}  // extern "C"
