// TEST-ONLY: host build of csrc/icp_math.cuh for tests/test_icp.py (compiled by the test into a temporary directory).
#include "icp_math.cuh"

using namespace b200pose;

extern "C" {

void icp_host_kabsch(const double* H, double eps, double* R, long long n) {
  for (long long i = 0; i < n; ++i) {
    double h[3][3], r[3][3];
    for (int a = 0; a < 9; ++a) h[a / 3][a % 3] = H[9 * i + a];
    icp_kabsch(h, eps, r);
    for (int a = 0; a < 9; ++a) R[9 * i + a] = r[a / 3][a % 3];
  }
}

// one ReduceToBason step on a batch of losses in fp32 (is64 = 0) or fp64; st = [steps, patience count, continual]
void icp_host_r2b(int is64, const void* loss, void* last, long long n, double* st, long long max_steps, long long patience,
                  double decreasing, double tol) {
  const R2bCtl c{max_steps, patience, decreasing, tol};
  bool below = true, flat = true;
  for (long long i = 0; i < n; ++i) {
    bool b, f;
    if (is64) icp_r2b_flags<double>(((const double*)loss)[i], ((double*)last)[i], c, b, f);
    else icp_r2b_flags<float>(((const float*)loss)[i], ((float*)last)[i], c, b, f);
    below = below && b;
    flat = flat && f;
  }
  for (long long i = 0; i < n; ++i) {
    if (is64) ((double*)last)[i] = ((const double*)loss)[i];
    else ((float*)last)[i] = ((const float*)loss)[i];
  }
  icp_r2b_update(st, below, flat, c);
}

}
