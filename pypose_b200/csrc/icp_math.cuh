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

// ---------------------------------------------------------------------------------------------------------------------
// Backward of ICP (DESIGN.md §3.4, "Gradients").  All fp64.  Only the part of a rotation cotangent G_R that is tangent to
// SO(3) at R reaches H through the Kabsch step, so quaternion derivatives are taken along SO(3): for the right
// perturbation R exp(th^), dq = q (x) [th/2, 0] and the cotangent g_q maps to g_th = (w g_v + g_v x v - g_w v) / 2, which
// is the rotation cotangent G_R = R (g_th / 2)^.
// ---------------------------------------------------------------------------------------------------------------------

// The quaternion [x y z w] that the reference's mat2SE3 gives for a rotation R (pypose/lietensor/convert.py mat2SO3):
// its branch is chosen by R22 < 1e-5, then R00 > R11 (or R00 < -R11 when R22 >= 1e-5), and w keeps the sign of its
// branch formula, so w < 0 is possible outside the trace branch.  icp_mat2quat returns the same rotation with w >= 0.
LM_HD void icp_mat2quat_ref(const double R[3][3], double q[4]) {
  double t, x, y, z, w;
  if (R[2][2] < 1e-5) {
    if (R[0][0] > R[1][1]) {
      t = 1.0 + R[0][0] - R[1][1] - R[2][2];
      w = R[2][1] - R[1][2]; x = t; y = R[1][0] + R[0][1]; z = R[0][2] + R[2][0];
    } else {
      t = 1.0 - R[0][0] + R[1][1] - R[2][2];
      w = R[0][2] - R[2][0]; x = R[1][0] + R[0][1]; y = t; z = R[2][1] + R[1][2];
    }
  } else if (R[0][0] < -R[1][1]) {
    t = 1.0 - R[0][0] - R[1][1] + R[2][2];
    w = R[1][0] - R[0][1]; x = R[0][2] + R[2][0]; y = R[2][1] + R[1][2]; z = t;
  } else {
    t = 1.0 + R[0][0] + R[1][1] + R[2][2];
    w = t; x = R[2][1] - R[1][2]; y = R[0][2] - R[2][0]; z = R[1][0] - R[0][1];
  }
  const double f = 0.5 / sqrt(t);
  q[0] = x * f; q[1] = y * f; q[2] = z * f; q[3] = w * f;
}

// G_R (accumulated) += R (g_th / 2)^ for the cotangent g (4) of the quaternion q (4) of R.
LM_HD void icp_quat_adj(const double R[3][3], const double q[4], const double g[4], double GR[3][3]) {
  const double v[3] = {q[0], q[1], q[2]}, gv[3] = {g[0], g[1], g[2]};
  double c[3], o[3];
  icp_cross(gv, v, c);
  for (int a = 0; a < 3; ++a) o[a] = 0.25 * (q[3] * gv[a] + c[a] - g[3] * v[a]);
  const double K[3][3] = {{0.0, -o[2], o[1]}, {o[2], 0.0, -o[0]}, {-o[1], o[0], 0.0}};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) GR[i][j] += R[i][0] * K[0][j] + R[i][1] * K[1][j] + R[i][2] * K[2][j];
}

// Adjoint of icp_kabsch: the cotangent GH of H for the cotangent GR of R, with the forward's rank rule.
//   full rank : GH = U Y V^T, Y_ij = (M_ij - M_ji) / (s_i + s_j), M = U^T (sg GR) V, sg = -1 where R was negated
//   rank 2    : the same with the right-handed frames of the forward and s_3 replaced by u3^T H v3 (= det U det V s_3,
//               the special-orthogonal Procrustes derivative)
//   rank <= 1 : GH = 0
// Y is invariant to the joint sign of (u_i, v_i), and finite for repeated singular values.
LM_HD void icp_kabsch_adj(const double H[3][3], double eps, const double GR[3][3], double GH[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) GH[i][j] = 0.0;
  double W[3][3], s[3], V[3][3];
  icp_svd3(H, W, s, V);
  if (!(s[0] > 0.0) || s[1] <= eps * s[0]) return;
  double u[3][3], v[3][3];
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) { u[i][k] = s[i] > 0.0 ? W[k][i] / s[i] : 0.0; v[i][k] = V[k][i]; }
  double sg = 1.0;
  if (s[2] <= eps * s[0]) {                        // rank 2: the forward's right-handed completion
    double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
    for (int k = 0; k < 3; ++k) u[1][k] -= d * u[0][k];
    icp_unit(u[1]);
    d = v[0][0] * v[1][0] + v[0][1] * v[1][1] + v[0][2] * v[1][2];
    for (int k = 0; k < 3; ++k) v[1][k] -= d * v[0][k];
    icp_unit(v[1]);
    icp_cross(u[0], u[1], u[2]);
    icp_cross(v[0], v[1], v[2]);
    double s3 = 0.0;
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) s3 += u[2][a] * H[a][b] * v[2][b];
    s[2] = s3;
  } else {
    double R[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[i][j] = u[0][i] * v[0][j] + u[1][i] * v[1][j] + u[2][i] * v[2][j];
    const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0]) +
                       R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
    if (fabs(det + 1.0) < 1e-6) sg = -1.0;
  }
  double M[3][3], Y[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double m = 0.0;
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) m += u[i][a] * GR[a][b] * v[j][b];
      M[i][j] = sg * m;
    }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Y[i][j] = i == j ? 0.0 : (M[i][j] - M[j][i]) / (s[i] + s[j]);
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      double g = 0.0;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) g += u[i][a] * Y[i][j] * v[j][b];
      GH[a][b] = g;
    }
}

// Shared tail of both Kabsch adjoints: t = mt - R ms with the cotangents GR (rotation, accumulated) and gt (translation).
// Out: GH, and the cotangents of the two centroids divided by n (what every matched point receives).
LM_HD void icp_svdtf_adj(const double H[3][3], double eps, const double R[3][3], const double ms[3], double n,
                         const double gt[3], double GR[3][3], double GH[3][3], double dms[3], double dmt[3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) GR[i][j] -= gt[i] * ms[j];
  icp_kabsch_adj(H, eps, GR, GH);
  for (int i = 0; i < 3; ++i) {
    dmt[i] = gt[i] / n;
    dms[i] = -(R[0][i] * gt[0] + R[1][i] * gt[1] + R[2][i] * gt[2]) / n;
  }
}

// Backward of one ICP iteration of one batch element.  S, c0: the recorded sums and shift of icp_step; P (3x4, row
// major): sum over the points of g [p; 1]^T, g the cotangent of the iteration's output point p.  The reference applies
// the step with SE3 Act, whose backward gives the 7-vector of T the gradient [sum g, sum p x g, 0]; that flows through
// the reference's quaternion (icp_mat2quat_ref) into R and t = mt - R ms.
// Out: R, GH, the absolute centroids ms (moved points), mt (matched targets), and dms, dmt as icp_svdtf_adj.
LM_HD void icp_iter_adj(const double S[17], const double c0[3], double eps, const double P[12], double R[3][3],
                        double GH[3][3], double ms[3], double mt[3], double dms[3], double dmt[3]) {
  const double n = S[16];
  double H[3][3], GR[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  if (!(n > 0.0)) {                                // the step was skipped: identity, nothing flows into the sums
    for (int i = 0; i < 3; ++i) {
      ms[i] = mt[i] = dms[i] = dmt[i] = 0.0;
      for (int j = 0; j < 3; ++j) { R[i][j] = i == j ? 1.0 : 0.0; GH[i][j] = 0.0; }
    }
    return;
  }
  double msr[3];
  for (int i = 0; i < 3; ++i) { msr[i] = S[i] / n; ms[i] = msr[i] + c0[i]; mt[i] = S[3 + i] / n + c0[i]; }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) H[i][j] = S[6 + 3 * i + j] - S[3 + i] * msr[j];
  icp_kabsch(H, eps, R);
  const double gt[3] = {P[3], P[7], P[11]};
  const double g[4] = {P[9] - P[6], P[2] - P[8], P[4] - P[1], 0.0};     // sum p x g, and 0 for w
  double q[4];
  icp_mat2quat_ref(R, q);
  icp_quat_adj(R, q, g, GR);
  icp_svdtf_adj(H, eps, R, ms, n, gt, GR, GH, dms, dmt);
}

// Backward of the closing svdtf(source, p_K) of one batch element, with the quaternion this project returns.
// F: sum d (3), sum e (3), sum e d^T (9, row major) over the points, d = s - cs, e = p_K - cp; n: point count;
// gout: the cotangent [t, q] of the returned 7-vector.  Out: GH, the centroids md = mean d, me = mean e, dms, dmt.
LM_HD void icp_final_adj(const double F[15], const double cs[3], double n, double eps, const double gout[7],
                         double GH[3][3], double md[3], double me[3], double dms[3], double dmt[3]) {
  double H[3][3], R[3][3], GR[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, A[12], q[4], ms[3];
  for (int i = 0; i < 3; ++i) { md[i] = F[i] / n; me[i] = F[3 + i] / n; ms[i] = md[i] + cs[i]; }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) H[i][j] = F[6 + 3 * i + j] - F[3 + i] * md[j];
  icp_kabsch(H, eps, R);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) A[4 * i + j] = R[i][j];
    A[4 * i + 3] = 0.0;
  }
  icp_mat2quat(A, q);
  icp_quat_adj(R, q, gout + 3, GR);
  icp_svdtf_adj(H, eps, R, ms, n, gout, GR, GH, dms, dmt);
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
