// TEST-ONLY: host build of csrc/sim3pgo_math.cuh for tests/test_sim3pgo.py (compiled by the test into a temporary directory
// with -ffp-contract=off): residual, Jacobian and packed blocks of Sim3 pose-graph edges, in fp64.
#include "sim3pgo_math.cuh"

using namespace b200pose;

extern "C" {

// per edge e: A, B, Z (8 each) -> r (7), J (7,7) row-major, M (28) packed J^T J, u (7) = J^T r
void sim3pgo_host_edges(const double* A, const double* B, const double* Z, double* r, double* J, double* M, double* u,
                        long long E) {
  for (long long e = 0; e < E; ++e) {
    const Elem<double> a = load_elem<Sim3g, double>(A + e * 8), b = load_elem<Sim3g, double>(B + e * 8),
                       z = load_elem<Sim3g, double>(Z + e * 8);
    Tang<double> rt;
    double Jm[7][7], Mp[28], up[7];
    sim3pgo_jacobian(a, b, z, rt, Jm);
    sim3pgo_linearize(a, b, z, rt, Mp, up);
    store_tang<Sim3g, double>(r + e * 7, rt);
    for (int i = 0; i < 7; ++i)
      for (int k = 0; k < 7; ++k) J[e * 49 + i * 7 + k] = Jm[i][k];
    for (int k = 0; k < 28; ++k) M[e * 28 + k] = Mp[k];
    for (int k = 0; k < 7; ++k) u[e * 7 + k] = up[k];
  }
}

}  // extern "C"
