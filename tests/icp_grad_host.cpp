// TEST-ONLY: host build of the ICP backward math of csrc/icp_math.cuh for tests/test_icp_grad.py (compiled by the test
// into a temporary directory).
#include "icp_math.cuh"

using namespace b200pose;

extern "C" {

void icp_host_kabsch_adj(const double* H, double eps, const double* GR, double* GH, long long n) {
  for (long long i = 0; i < n; ++i) {
    double h[3][3], g[3][3], o[3][3];
    for (int a = 0; a < 9; ++a) { h[a / 3][a % 3] = H[9 * i + a]; g[a / 3][a % 3] = GR[9 * i + a]; }
    icp_kabsch_adj(h, eps, g, o);
    for (int a = 0; a < 9; ++a) GH[9 * i + a] = o[a / 3][a % 3];
  }
}

void icp_host_quat_ref(const double* R, double* q, long long n) {
  for (long long i = 0; i < n; ++i) {
    double r[3][3];
    for (int a = 0; a < 9; ++a) r[a / 3][a % 3] = R[9 * i + a];
    icp_mat2quat_ref(r, q + 4 * i);
  }
}

// out (30 per element): R 9, GH 9, ms 3, mt 3, dms 3, dmt 3
void icp_host_iter_adj(const double* S, const double* c0, double eps, const double* P, double* out, long long n) {
  for (long long i = 0; i < n; ++i) {
    double R[3][3], GH[3][3];
    double* o = out + 30 * i;
    icp_iter_adj(S + 17 * i, c0 + 3 * i, eps, P + 12 * i, R, GH, o + 18, o + 21, o + 24, o + 27);
    for (int a = 0; a < 9; ++a) { o[a] = R[a / 3][a % 3]; o[9 + a] = GH[a / 3][a % 3]; }
  }
}

// out (21 per element): GH 9, md 3, me 3, dms 3, dmt 3
void icp_host_final_adj(const double* F, const double* cs, double npts, double eps, const double* gout, double* out,
                        long long n) {
  for (long long i = 0; i < n; ++i) {
    double GH[3][3];
    double* o = out + 21 * i;
    icp_final_adj(F + 15 * i, cs + 3 * i, npts, eps, gout + 7 * i, GH, o + 9, o + 12, o + 15, o + 18);
    for (int a = 0; a < 9; ++a) o[a] = GH[a / 3][a % 3];
  }
}

}

extern "C" void icp_grad_host_kabsch(const double* H, double eps, double* R) {
  double h[3][3], r[3][3];
  for (int a = 0; a < 9; ++a) h[a / 3][a % 3] = H[a];
  icp_kabsch(h, eps, r);
  for (int a = 0; a < 9; ++a) R[a] = r[a / 3][a % 3];
}
