// traj_math.cuh — per-element math of the trajectory metrics pp.metric.ape / rpe (host+device, see lie_math.cuh):
// timestamp association, segment lengths of the path, and the pose errors.  All arithmetic is fp64.  DESIGN.md §3.6.
//
// Association (matching_time_indices, pypose/metric/ape_rpe.py:107-139): for a short stamp s and the long stamps l_j
// shifted by `off`, the reference takes argmin_j |fl(s - fl(l_j + off))| (lowest j on ties) and keeps it when the
// distance is < diff.  fl(l_j + off) is non-decreasing in j and fl(s - x) is non-increasing in x with the sign of
// s - x, so the distance falls up to the first j with l_j' >= s and rises from there: the minimum is at that j or the
// one before it.  Equal distances can repeat to the left of the one before it (duplicate stamps, or stamps that round
// to the same difference), so the lowest index is found by a second binary search over that run.
//
// Segment lengths: ||a - b|| = sqrt(fma(z, z, fma(y, y, x * x))), correctly rounded at each step, the rounding of
// torch's fp64 3-vector norm on the CPU.
#pragma once
#include "lie_math.cuh"

namespace b200pose {

LM_HD double tr_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
LM_HD double tr_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}
LM_HD double tr_sqrt(double a) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(a);
#else
  return sqrt(a);
#endif
}
LM_HD double tr_add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
LM_HD double tr_sub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}

// ||v|| with the rounding of torch.linalg.norm(v, dim=-1) on a (.., 3) fp64 tensor
LM_HD double tr_norm3(double x, double y, double z) { return tr_sqrt(tr_fma(z, z, tr_fma(y, y, tr_mul(x, x)))); }

// ---------------------------------------------------------------- association
// distance of short stamp s to long stamp l shifted by off
LM_HD double tr_tdist(double s, double l, double off) { return fabs(tr_sub(s, tr_add(l, off))); }

// index in [0, n) of the long stamp nearest to s (lowest on ties), and its distance
LM_HD long long tr_match(const double* L, long long n, double s, double off, double& dist) {
  long long lo = 0, hi = n;                  // first j with fl(L_j + off) >= s
  while (lo < hi) {
    const long long mid = lo + (hi - lo) / 2;
    if (tr_add(L[mid], off) >= s) hi = mid; else lo = mid + 1;
  }
  const long long p = lo;
  if (p == 0) { dist = tr_tdist(s, L[0], off); return 0; }
  const double dl = tr_tdist(s, L[p - 1], off);
  if (p < n) {
    const double dr = tr_tdist(s, L[p], off);
    if (dr < dl) { dist = dr; return p; }
  }
  // distances are non-increasing on [0, p): the first j with d_j <= dl starts the run of equal minima
  lo = 0; hi = p - 1;
  while (lo < hi) {
    const long long mid = lo + (hi - lo) / 2;
    if (tr_tdist(s, L[mid], off) <= dl) hi = mid; else lo = mid + 1;
  }
  dist = dl;
  return lo;
}

// ---------------------------------------------------------------- distance pairs (pairs_by_dist, all=True)
// |fl(fl(D_j - D_i) - delta)|
LM_HD double tr_pdist(const double* D, long long i, long long j, double delta) {
  return fabs(tr_sub(tr_sub(D[j], D[i]), delta));
}

// argmin over j in (i, n) of |fl(fl(D_j - D_i) - delta)| (lowest on ties) for non-decreasing D, and the minimum
LM_HD long long tr_pair(const double* D, long long n, long long i, double delta, double& h) {
  long long lo = i + 1, hi = n;              // first j with fl(D_j - D_i) >= delta
  while (lo < hi) {
    const long long mid = lo + (hi - lo) / 2;
    if (tr_sub(D[mid], D[i]) >= delta) hi = mid; else lo = mid + 1;
  }
  const long long p = lo;
  if (p == i + 1) { h = tr_pdist(D, i, p, delta); return p; }
  const double hl = tr_pdist(D, i, p - 1, delta);
  if (p < n) {
    const double hr = tr_pdist(D, i, p, delta);
    if (hr < hl) { h = hr; return p; }
  }
  lo = i + 1; hi = p - 1;
  while (lo < hi) {
    const long long mid = lo + (hi - lo) / 2;
    if (tr_pdist(D, i, mid, delta) <= hl) hi = mid; else lo = mid + 1;
  }
  h = hl;
  return lo;
}

// ---------------------------------------------------------------- poses
// SE3 row [t, q] read through a row of any strides, widened to fp64
template <typename T> LM_HD Elem<double> tr_load(const T* p, long long cs) {
  Elem<double> e;
  e.t = mk((double)p[0], (double)p[cs], (double)p[2 * cs]);
  e.q.v = mk((double)p[3 * cs], (double)p[4 * cs], (double)p[5 * cs]);
  e.q.w = (double)p[6 * cs];
  e.s = 1.0;
  return e;
}

// Sim3 [t, q, s] (fp64, contiguous) @ Sim3(pose, 1), keeping [t, q] (StampedSE3.align, ape_rpe.py:58-66); S NULL: pose
LM_HD Elem<double> tr_align(const double* S, const Elem<double>& X) {
  if (!S) return X;
  Elem<double> A = load_elem<Sim3g, double>(S);
  Elem<double> Y = g_mul<Sim3g, double>(A, X);
  Y.s = 1.0;
  return Y;
}

// error types, in the order of the Python `etype` names
enum TrajEtype { kTrTranslation = 0, kTrRotation = 1, kTrPose = 2, kTrRadian = 3, kTrDegree = 4 };

// columns of R(E), built as matrix() does: R e_j = Act(E, e_j) without the translation
LM_HD void tr_rotmat(const Q4<double>& q, double R[3][3]) {
  for (int j = 0; j < 3; ++j) {
    const V3<double> c = qrot(q, mk(j == 0 ? 1.0 : 0.0, j == 1 ? 1.0 : 0.0, j == 2 ? 1.0 : 0.0));
    R[0][j] = c.x; R[1][j] = c.y; R[2][j] = c.z;
  }
}

// mat2SO3(R, check=False) (pypose/lietensor/convert.py:97-145): Shepperd's method with the reference's branch rule
LM_HD Q4<double> tr_mat2q(const double R[3][3]) {
  double m[3][3];                                  // rmat_t = R^T
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) m[a][b] = R[b][a];
  const bool d2 = m[2][2] < 1e-5, d0_d1 = m[0][0] > m[1][1], d0_nd1 = m[0][0] < -m[1][1];
  double t, w, x, y, z;                            // q in wxyz order before the division
  if (d2 && d0_d1) {
    t = 1 + m[0][0] - m[1][1] - m[2][2];
    w = m[1][2] - m[2][1]; x = t; y = m[0][1] + m[1][0]; z = m[2][0] + m[0][2];
  } else if (d2) {
    t = 1 - m[0][0] + m[1][1] - m[2][2];
    w = m[2][0] - m[0][2]; x = m[0][1] + m[1][0]; y = t; z = m[1][2] + m[2][1];
  } else if (d0_nd1) {
    t = 1 - m[0][0] - m[1][1] + m[2][2];
    w = m[0][1] - m[1][0]; x = m[2][0] + m[0][2]; y = m[1][2] + m[2][1]; z = t;
  } else {
    t = 1 + m[0][0] + m[1][1] + m[2][2];
    w = t; x = m[1][2] - m[2][1]; y = m[2][0] - m[0][2]; z = m[0][1] - m[1][0];
  }
  const double d = 2 * sqrt(t);
  Q4<double> q;
  q.v = mk(x / d, y / d, z / d);
  q.w = w / d;
  return q;
}

// error of E for the given type; `ape_t` is the APE translation difference t_e' - t_r (used by kTrTranslation only
// when `ape` is set, RPE uses t(E))
LM_HD double tr_error(const Elem<double>& E, int etype, bool ape, const V3<double>& ape_t) {
  if (etype == kTrTranslation) {
    const V3<double> v = ape ? ape_t : E.t;
    return tr_norm3(v.x, v.y, v.z);
  }
  double R[3][3];
  tr_rotmat(E.q, R);
  if (etype == kTrRotation || etype == kTrPose) {
    double acc = 0.0;
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) {
        const double v = R[a][b] - (a == b ? 1.0 : 0.0);
        acc = tr_fma(v, v, acc);
      }
    if (etype == kTrPose) {
      acc = tr_fma(E.t.x, E.t.x, acc);
      acc = tr_fma(E.t.y, E.t.y, acc);
      acc = tr_fma(E.t.z, E.t.z, acc);
    }
    return tr_sqrt(acc);
  }
  double jc;
  const V3<double> phi = so3_log(tr_mat2q(R), jc);
  const double r = tr_norm3(phi.x, phi.y, phi.z);
  return etype == kTrDegree ? r * 57.295779513082320876798154814105170332405472466564321549160243861 : r;
}

// APE of one associated pair: translation ||t_e' - t_r||, otherwise the error of E = e'^-1 r
LM_HD double tr_ape(const Elem<double>& r, const Elem<double>& e_aligned, int etype) {
  if (etype == kTrTranslation) return tr_error(r, etype, true, e_aligned.t - r.t);
  const Elem<double> E = g_mul<SE3g, double>(g_inv<SE3g, double>(e_aligned), r);
  return tr_error(E, etype, false, E.t);
}

// RPE of one pair (a, b): E = (r_a^-1 r_b)^-1 (e_a'^-1 e_b')
LM_HD double tr_rpe(const Elem<double>& ra, const Elem<double>& rb, const Elem<double>& ea, const Elem<double>& eb,
                    int etype) {
  const Elem<double> R = g_mul<SE3g, double>(g_inv<SE3g, double>(ra), rb);
  const Elem<double> Q = g_mul<SE3g, double>(g_inv<SE3g, double>(ea), eb);
  const Elem<double> E = g_mul<SE3g, double>(g_inv<SE3g, double>(R), Q);
  return tr_error(E, etype, false, E.t);
}

}  // namespace b200pose
