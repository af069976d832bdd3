// TEST-ONLY: host build of csrc/bsr_math.cuh for tests/test_sparse.py (compiled by the test into a temporary directory
// with -ffp-contract=off, so it reproduces the device's fma order bit for bit).
#include "bsr_math.cuh"

using namespace b200pose;

template <typename T>
static void numeric(const T* L, long long lsb, long long ls0, long long ls1, const T* R, long long rsb, long long rs0,
                    long long rs1, const unsigned long long* tri, const long long* ptr, long long nout, int dx, int dy,
                    int dz, T* out) {
  const BsrOperand lo{lsb, ls0, ls1}, ro{rsb, rs0, rs1};
  for (long long g = 0; g < nout; ++g)
    for (int x = 0; x < dx; ++x)
      for (int y = 0; y < dy; ++y)
        out[(g * dx + x) * dy + y] = bsr_elem(L, lo, R, ro, tri, ptr[g], ptr[g + 1], x, y, dz);
}

extern "C" {

// out (nout, dx, dy): block g sums L[l] (x, z) R[r] (z, y) over the triples (l << 32) | r of tri[ptr[g] .. ptr[g + 1])
void sparse_host_numeric_f64(const double* L, long long lsb, long long ls0, long long ls1, const double* R, long long rsb,
                             long long rs0, long long rs1, const unsigned long long* tri, const long long* ptr,
                             long long nout, int dx, int dy, int dz, double* out) {
  numeric(L, lsb, ls0, ls1, R, rsb, rs0, rs1, tri, ptr, nout, dx, dy, dz, out);
}

void sparse_host_numeric_f32(const float* L, long long lsb, long long ls0, long long ls1, const float* R, long long rsb,
                             long long rs0, long long rs1, const unsigned long long* tri, const long long* ptr,
                             long long nout, int dx, int dy, int dz, float* out) {
  numeric(L, lsb, ls0, ls1, R, rsb, rs0, rs1, tri, ptr, nout, dx, dy, dz, out);
}

}
