// icp_math.cuh — per-batch math of point-to-point ICP (host+device, see lie_math.cuh): the Kabsch rotation of a 3x3
// cross-covariance with a defined answer when it is rank-deficient, SE3 helpers, and the ReduceToBason stop rule.
//
// Kabsch rule (DESIGN.md §3.4), for H = sum (t - mt)(s - ms)^T = U diag(s1 >= s2 >= s3) V^T, all in fp64:
//   s1 == 0                : R = I
//   s2 <= eps s1 (rank 1)  : the smallest rotation taking v1 to u1
//   s3 <= eps s1 (rank 2)  : u3 = u1 x u2, v3 = v1 x v2, R = U V^T (det R = +1)
//   otherwise              : R = U V^T, negated as a whole when |det R + 1| < 1e-6 (pypose/function/geometry.py svdtf)
// Every case is invariant to the joint sign of (u_i, v_i), so R does not depend on how the SVD picks signs.
#pragma once
#include "lie_math.cuh"

namespace b200pose {

constexpr int kIcpSweeps = 40;

// One-sided (Hestenes) Jacobi SVD of a 3x3 matrix: on return W = M V has orthogonal columns w_i = s_i u_i, V is
// orthonormal, columns sorted by decreasing s_i.  Working on M rather than M^T M keeps small singular values accurate
// to eps * s1, which the rank tests need.
LM_HD void icp_svd3(const double M[3][3], double W[3][3], double s[3], double V[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { W[i][j] = M[i][j]; V[i][j] = i == j ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < kIcpSweeps; ++sweep) {
    bool rotated = false;
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double a = 0.0, b = 0.0, g = 0.0;
      for (int i = 0; i < 3; ++i) { a += W[i][p] * W[i][p]; b += W[i][q] * W[i][q]; g += W[i][p] * W[i][q]; }
      if (g == 0.0 || fabs(g) <= 1e-15 * sqrt(a * b)) continue;
      rotated = true;
      const double z = (b - a) / (2.0 * g);
      const double t = (z >= 0.0 ? 1.0 : -1.0) / (fabs(z) + sqrt(1.0 + z * z));
      const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
      for (int i = 0; i < 3; ++i) {
        const double wp = W[i][p], wq = W[i][q];
        W[i][p] = c * wp - sn * wq; W[i][q] = sn * wp + c * wq;
        const double vp = V[i][p], vq = V[i][q];
        V[i][p] = c * vp - sn * vq; V[i][q] = sn * vp + c * vq;
      }
    }
    if (!rotated) break;
  }
  for (int j = 0; j < 3; ++j) s[j] = sqrt(W[0][j] * W[0][j] + W[1][j] * W[1][j] + W[2][j] * W[2][j]);
  for (int a = 0; a < 2; ++a)                      // selection sort, decreasing; ties keep the column order
    for (int b = a + 1; b < 3; ++b)
      if (s[b] > s[a]) {
        double tmp = s[a]; s[a] = s[b]; s[b] = tmp;
        for (int i = 0; i < 3; ++i) {
          tmp = W[i][a]; W[i][a] = W[i][b]; W[i][b] = tmp;
          tmp = V[i][a]; V[i][a] = V[i][b]; V[i][b] = tmp;
        }
      }
}

LM_HD void icp_cross(const double a[3], const double b[3], double c[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
LM_HD void icp_unit(double a[3]) {
  const double n = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  if (n > 0.0) { a[0] /= n; a[1] /= n; a[2] /= n; }
}

// Rotation of the Kabsch step for the cross-covariance H (target x source); eps: relative rank threshold.
LM_HD void icp_kabsch(const double H[3][3], double eps, double R[3][3]) {
  double W[3][3], s[3], V[3][3];
  icp_svd3(H, W, s, V);
  double u[3][3], v[3][3];                         // u[i], v[i]: i-th singular vectors
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) { u[i][k] = s[i] > 0.0 ? W[k][i] / s[i] : 0.0; v[i][k] = V[k][i]; }
  if (!(s[0] > 0.0)) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[i][j] = i == j ? 1.0 : 0.0;
    return;
  }
  if (s[1] <= eps * s[0]) {                        // rank 1: Rodrigues rotation v1 -> u1 about v1 x u1
    double a[3];
    icp_cross(v[0], u[0], a);
    const double c = v[0][0] * u[0][0] + v[0][1] * u[0][1] + v[0][2] * u[0][2];
    if (1.0 + c > 1e-12) {
      const double f = 1.0 / (1.0 + c);
      R[0][0] = c + f * a[0] * a[0];  R[0][1] = -a[2] + f * a[0] * a[1]; R[0][2] = a[1] + f * a[0] * a[2];
      R[1][0] = a[2] + f * a[1] * a[0]; R[1][1] = c + f * a[1] * a[1];  R[1][2] = -a[0] + f * a[1] * a[2];
      R[2][0] = -a[1] + f * a[2] * a[0]; R[2][1] = a[0] + f * a[2] * a[1]; R[2][2] = c + f * a[2] * a[2];
    } else {                                       // v1 = -u1: half turn about an axis normal to v1
      int m = 0;
      for (int k = 1; k < 3; ++k)
        if (fabs(v[0][k]) < fabs(v[0][m])) m = k;
      double e[3] = {0.0, 0.0, 0.0}, n[3];
      e[m] = 1.0;
      icp_cross(v[0], e, n);
      icp_unit(n);
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = 2.0 * n[i] * n[j] - (i == j ? 1.0 : 0.0);
    }
    return;
  }
  const bool rank2 = s[2] <= eps * s[0];
  if (rank2) {                                     // complete both bases as right-handed frames
    double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
    for (int k = 0; k < 3; ++k) u[1][k] -= d * u[0][k];
    icp_unit(u[1]);
    d = v[0][0] * v[1][0] + v[0][1] * v[1][1] + v[0][2] * v[1][2];
    for (int k = 0; k < 3; ++k) v[1][k] -= d * v[0][k];
    icp_unit(v[1]);
    icp_cross(u[0], u[1], u[2]);
    icp_cross(v[0], v[1], v[2]);
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i][j] = u[0][i] * v[0][j] + u[1][i] * v[1][j] + u[2][i] * v[2][j];
  if (!rank2) {
    const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0]) +
                       R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
    if (fabs(det + 1.0) < 1e-6)
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = -R[i][j];
  }
}

// A = [R | t] row-major 3x4 <-> SE3 [t, qx qy qz qw].
LM_HD void icp_quat2mat(const double q[4], double A[12]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  A[0] = w * w + x * x - y * y - z * z; A[1] = 2 * (x * y - w * z); A[2] = 2 * (x * z + w * y);
  A[4] = 2 * (x * y + w * z); A[5] = w * w - x * x + y * y - z * z; A[6] = 2 * (y * z - w * x);
  A[8] = 2 * (x * z - w * y); A[9] = 2 * (y * z + w * x); A[10] = w * w - x * x - y * y + z * z;
}
LM_HD void icp_mat2quat(const double A[12], double q[4]) {   // Shepperd: branch on the largest of trace, diagonal
  const double r00 = A[0], r11 = A[5], r22 = A[10], tr = r00 + r11 + r22;
  double x, y, z, w;
  if (tr >= r00 && tr >= r11 && tr >= r22) {
    const double s = 2.0 * sqrt(1.0 + tr);
    w = 0.25 * s; x = (A[9] - A[6]) / s; y = (A[2] - A[8]) / s; z = (A[4] - A[1]) / s;
  } else if (r00 >= r11 && r00 >= r22) {
    const double s = 2.0 * sqrt(1.0 + r00 - r11 - r22);
    w = (A[9] - A[6]) / s; x = 0.25 * s; y = (A[1] + A[4]) / s; z = (A[2] + A[8]) / s;
  } else if (r11 >= r22) {
    const double s = 2.0 * sqrt(1.0 + r11 - r00 - r22);
    w = (A[2] - A[8]) / s; x = (A[1] + A[4]) / s; y = 0.25 * s; z = (A[6] + A[9]) / s;
  } else {
    const double s = 2.0 * sqrt(1.0 + r22 - r00 - r11);
    w = (A[4] - A[1]) / s; x = (A[2] + A[8]) / s; y = (A[6] + A[9]) / s; z = 0.25 * s;
  }
  const double sg = w < 0.0 ? -1.0 : 1.0, n = sg / sqrt(x * x + y * y + z * z + w * w);
  q[0] = x * n; q[1] = y * n; q[2] = z * n; q[3] = w * n;
}

// One Kabsch step from the sums of a batch element (points shifted by c0 before summing):
// S = [sum s(3), sum t(3), sum t s^T (9, row-major), sum dist, count].  A <- [R | t] A.
LM_HD void icp_step(const double S[17], const double c0[3], double eps, double A[12]) {
  const double n = S[16];
  if (!(n > 0.0)) return;
  double ms[3], mt[3], H[3][3], R[3][3], t[3];
  for (int i = 0; i < 3; ++i) { ms[i] = S[i] / n; mt[i] = S[3 + i] / n; }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) H[i][j] = S[6 + 3 * i + j] - S[3 + i] * ms[j];
  icp_kabsch(H, eps, R);
  for (int i = 0; i < 3; ++i)
    t[i] = (mt[i] + c0[i]) - (R[i][0] * (ms[0] + c0[0]) + R[i][1] * (ms[1] + c0[1]) + R[i][2] * (ms[2] + c0[2]));
  double B[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 4; ++j) B[4 * i + j] = R[i][0] * A[j] + R[i][1] * A[4 + j] + R[i][2] * A[8 + j];
    B[4 * i + 3] += t[i];
  }
  for (int k = 0; k < 12; ++k) A[k] = B[k];
}

// ReduceToBason.step (pypose/utils/stepper.py) over a batch of losses, in the loss dtype T.  st: [steps, patience count,
// continual]; last: previous losses (+inf after reset).  Returns the new `continual`.
struct R2bCtl { long long max_steps, patience; double decreasing, tol; };
template <typename T> LM_HD void icp_r2b_flags(T loss, T last, const R2bCtl& c, bool& below_tol, bool& flat) {
  below_tol = loss < (T)c.tol;
  const T rel = (T)(last - loss) / loss;           // 0/0 = NaN compares false: the patience count resets
  flat = rel < (T)c.decreasing;
}
LM_HD void icp_r2b_update(double st[3], bool all_below_tol, bool all_flat, const R2bCtl& c) {
  st[0] += 1.0;
  if (all_below_tol) st[2] = 0.0;
  if (st[0] >= (double)c.max_steps) st[2] = 0.0;
  st[1] = all_flat ? st[1] + 1.0 : 0.0;
  if (st[1] >= (double)c.patience) st[2] = 0.0;
}

}  // namespace b200pose
