// TEST-ONLY: host build of csrc/so3pgo_math.cuh for tests/test_so3pgo.py (compiled by the test into a temporary directory
// with -ffp-contract=off): residual, Jacobian and packed blocks of SO3 pose-graph edges, in fp64.
#include "so3pgo_math.cuh"

using namespace b200pose;

extern "C" {

// per edge e: A, B, Z (4 each) -> r (3), J (3,3) row-major, M (6) packed J^T J, u (3) = J^T r
void so3pgo_host_edges(const double* A, const double* B, const double* Z, double* r, double* J, double* M, double* u,
                       long long E) {
  for (long long e = 0; e < E; ++e) {
    const Elem<double> a = load_elem<SO3g, double>(A + e * 4), b = load_elem<SO3g, double>(B + e * 4),
                       z = load_elem<SO3g, double>(Z + e * 4);
    Tang<double> rt;
    double Jm[3][3], Mp[6], up[3];
    so3pgo_jacobian(a, b, z, rt, Jm);
    so3pgo_linearize(a, b, z, rt, Mp, up);
    store_tang<SO3g, double>(r + e * 3, rt);
    for (int i = 0; i < 3; ++i)
      for (int k = 0; k < 3; ++k) J[e * 9 + i * 3 + k] = Jm[i][k];
    for (int k = 0; k < 6; ++k) M[e * 6 + k] = Mp[k];
    for (int k = 0; k < 3; ++k) u[e * 3 + k] = up[k];
  }
}

}  // extern "C"
