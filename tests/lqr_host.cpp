// TEST-ONLY: host build of csrc/lqr_math.cuh for tests/test_lqr.py (compiled by the test into a temporary directory).
// Runs the device's per-problem code with one lane (lane 0, stride 1) on full-size operands (nb, T, ...), fp64 or fp32.
#include <vector>
#include "lqr_math.cuh"

using namespace b200pose;

template <class R>
static LqrProb<R> prob(const R* Q, const R* p, const R* A, const R* B, const R* c1, const R* x0, const R* u0, int T, int ns,
                       int nc) {
  const long long n = ns + nc;
  return LqrProb<R>{{Q, T * n * n, n * n}, {p, T * n, n}, {A, T * ns * ns, ns * ns}, {B, T * ns * nc, ns * nc},
                    {c1, T * ns, ns}, {u0, T * nc, nc}, x0, T, ns, nc};
}

template <class R>
static int solve(const R* Q, const R* p, const R* A, const R* B, const R* c1, const R* x0, const R* u0, long long nb, int T,
                 int ns, int nc, R* x, R* u, R* cost, R* xtr, int* status) {
  const LqrProb<R> P = prob(Q, p, A, B, c1, x0, u0, T, ns, nc);
  std::vector<R> sm(lqr_smem_elems(ns, nc)), ws((size_t)T * nc * (ns + 1));
  for (long long b = 0; b < nb; ++b)
    status[b] = lqr_solve(P, b, lqr_carve(sm.data(), ns, nc), ws.data(), x, u, cost, xtr, LqrLane{0, 1});
  return 0;
}

extern "C" {

// the per-warp shared-memory slab of csrc/lqr.cu, in elements (tests/test_lqr_paths_gpu.py mirrors the launch shape)
int lqr_host_smem_elems(int ns, int nc) { return lqr_smem_elems(ns, nc); }

int lqr_host_solve(const double* Q, const double* p, const double* A, const double* B, const double* c1, const double* x0,
                   const double* u0, long long nb, int T, int ns, int nc, double* x, double* u, double* cost,
                   double* xtr, int* status) {
  return solve(Q, p, A, B, c1, x0, u0, nb, T, ns, nc, x, u, cost, xtr, status);
}

int lqr_host_solve_f32(const float* Q, const float* p, const float* A, const float* B, const float* c1, const float* x0,
                       const float* u0, long long nb, int T, int ns, int nc, float* x, float* u, float* cost, float* xtr,
                       int* status) {
  return solve(Q, p, A, B, c1, x0, u0, nb, T, ns, nc, x, u, cost, xtr, status);
}

// gradients per problem and step (tv = 1 everywhere)
int lqr_host_adjoint(const double* Q, const double* p, const double* A, const double* B, const double* c1,
                     const double* x0, long long nb, int T, int ns, int nc, const double* x, const double* u,
                     const double* gx, const double* gu, const double* gc, double* gQ, double* gp, double* gA,
                     double* gB, double* gc1, double* gx0) {
  const LqrProb<double> P = prob<double>(Q, p, A, B, c1, x0, nullptr, T, ns, nc);
  const LqrGrad<double> G{gQ, gp, gA, gB, gc1, gx0, 1, 1, 1, 1, 1};
  std::vector<double> sm(lqr_smem_elems(ns, nc)), ws((size_t)T * (nc * (ns + 1) + ns + nc));
  for (long long b = 0; b < nb; ++b) lqr_adjoint(P, b, lqr_carve(sm.data(), ns, nc), ws.data(), x, u, gx, gu, gc, G, LqrLane{0, 1});
  return 0;
}
}
