// TEST-ONLY: host build of csrc/traj_math.cuh for tests/test_metric.py (compiled by the test into a temporary directory).
#include "traj_math.cuh"

using namespace b200pose;

extern "C" {

// segment lengths l_k = ||t_k - t_{k+1}|| and D = cat(0, sequential cumsum(l)) of (n, 3) translations
void metric_host_path(const double* t, long long n, double* l, double* D) {
  D[0] = 0.0;
  for (long long k = 0; k + 1 < n; ++k) {
    const double* a = t + 3 * k;
    const double* b = a + 3;
    l[k] = tr_norm3(a[0] - b[0], a[1] - b[1], a[2] - b[2]);
    D[k + 1] = D[k] + l[k];
  }
}

// association of every short stamp: long index and whether it is kept
void metric_host_match(const double* S, long long ns, const double* L, long long nl, double off, double diff,
                       long long* j, unsigned char* keep) {
  for (long long i = 0; i < ns; ++i) {
    double d;
    j[i] = tr_match(L, nl, S[i], off, d);
    keep[i] = d < diff;
  }
}

// distance pairs (all = True) of an accumulated path D
void metric_host_pairs(const double* D, long long n, double delta, double tol, long long* j, unsigned char* keep) {
  for (long long i = 0; i + 1 < n; ++i) {
    double h;
    j[i] = tr_pair(D, n, i, delta, h);
    keep[i] = !(h > tol);
  }
}

// per-pair errors of aligned poses (S: Sim3 or NULL); rb / eb NULL for APE
void metric_host_err(const double* r, const double* rb, const double* e, const double* eb, const double* S, long long M,
                     int etype, double* err) {
  for (long long k = 0; k < M; ++k) {
    const Elem<double> r0 = tr_load(r + 7 * k, 1), e0 = tr_align(S, tr_load(e + 7 * k, 1));
    if (!rb) { err[k] = tr_ape(r0, e0, etype); continue; }
    err[k] = tr_rpe(r0, tr_load(rb + 7 * k, 1), e0, tr_align(S, tr_load(eb + 7 * k, 1)), etype);
  }
}

}
