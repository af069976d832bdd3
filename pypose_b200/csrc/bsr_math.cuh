// bsr_math.cuh — per-element accumulation of the block-sparse products pp.bsr_bsc_matmul (host+device, see
// lie_math.cuh).  DESIGN.md §3.8.
//
// Every output block of the forward product and of both gradients is a sum of small dense products over a segment of
// block triples:  out[x][y] = sum_t sum_z L_t[x][z] * R_t[z][y].  A triple is packed as (l << 32) | r, the indices of
// its left and right blocks in their values arrays; a block is addressed through three element strides (block, x, z)
// on the left and (block, z, y) on the right, so transposed views (A.mT, B^T in dA, A^T in dB) cost nothing.
//
//   forward  C[c]  = sum A[a] B[b]        L = A,  R = B      triples (a, b) of the segment of c, k ascending
//   dA       dA[a] = sum dC[c] B[b]^T     L = dC, R = B^T    triples (c, b) of a, j ascending
//   dB       dB[b] = sum A[a]^T dC[c]     L = A^T, R = dC    triples (a, c) of b, i ascending
//
// Each element keeps one accumulator in the values' dtype and runs acc = fma(l, r, acc) over the triples in segment
// order, then z ascending.  The order is fixed, so results are bit-identical from run to run, and a host build with
// -ffp-contract=off (tests/sparse_host.cpp) reproduces the device bit for bit.
#pragma once
#include "lie_math.cuh"

namespace b200pose {

LM_HD float bsr_fma(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
  return __fmaf_rn(a, b, c);
#else
  return fmaf(a, b, c);
#endif
}
LM_HD double bsr_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}

struct BsrOperand {          // a values array (nnz, d0, d1) read through element strides
  long long sb, s0, s1;      // block, first index, second index
};

// element (x, y) of the sum over triples t0 .. t1 - 1; L is read as (block, x, z) and R as (block, z, y)
template <typename T>
LM_HD T bsr_elem(const T* L, BsrOperand lo, const T* R, BsrOperand ro, const unsigned long long* tri, long long t0,
                 long long t1, int x, int y, int nz) {
  T acc = T(0);
  for (long long t = t0; t < t1; ++t) {
    const unsigned long long p = tri[t];
    const T* l = L + (long long)(p >> 32) * lo.sb + x * lo.s0;
    const T* r = R + (long long)(p & 0xffffffffull) * ro.sb + y * ro.s1;
    for (int z = 0; z < nz; ++z) acc = bsr_fma(l[z * lo.s1], r[z * ro.s0], acc);
  }
  return acc;
}

}  // namespace b200pose
