// lm_tc.cu — tensor-core variant of the per-camera J^T J accumulation, kept as the EVIDENCE run that BASELINE.json's
// north_star asks for ("tensor cores used only where J^T J over a dense residual block is genuinely a large contraction —
// each choice evidenced ... tensor-pipe % for the J^T J path").  It is NOT on the production path: the scalar kernel
// is (DESIGN.md §3.3).
//
// Contraction: per camera c with m observations, V = [J | r] is (2m x 7); H = J^T J, g = J^T r and the loss r^T r are the
// 7x7 Gram matrix V^T V.  K = 2m can be thousands, but M = N = 7: the smallest warp-level tile of the tensor pipe is
// m16n8k8 (TF32), i.e. at most 7*7 / (16*8) = 38 % of every MMA is useful, and wgmma's minimum M of 64 would waste
// > 90 % (different cameras have different J, so a block-diagonal batch cannot share one MMA).
//
// Layout: one CTA (4 warps) per camera; each lane builds the two rows of its observation in registers, the warp stages
// its 64 x 8 tile in shared memory, and eight k-steps feed mma.sync.m16n8k8 with A = V^T (rows 8..15 zero) and B = V — the
// same registers serve both operands.  3xTF32 (hi*hi + hi*lo + lo*hi) keeps fp32-level accuracy.
#include "lm_common.cuh"

namespace b200pose {

__device__ __forceinline__ unsigned f2tf32(float x) {
  unsigned r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], unsigned a0, unsigned a2, unsigned b0, unsigned b1) {
  // rows 8..15 of A are zero: a1 = a3 = 0
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
}

constexpr int kTcThreads = 128;

__global__ void __launch_bounds__(kTcThreads) lm_reproj_accum_tc_kernel(const float* __restrict__ poses,
                                                                         const float* __restrict__ pts,
                                                                         const float* __restrict__ pix,
                                                                         const int* __restrict__ seg, float* __restrict__ H,
                                                                         float* __restrict__ g, double* ws, int ncam) {
  __shared__ float tile[kTcThreads / 32][64][9];          // per warp: 64 residual rows x 8 columns (+1 pad: conflict-free)
  __shared__ float red[kTcThreads / 32][8][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gid = lane >> 2, tig = lane & 3;
  double acc[1] = {0.0};
  for (int c = blockIdx.x; c < ncam; c += gridDim.x) {
    float pr[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) pr[k] = poses[(long long)c * 7 + k];
    const Elem<float> Tc = load_se3(pr);
    const int b = seg[c], e = seg[c + 1];
    float cfrag[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = b + warp * 32; k0 < e; k0 += kTcThreads) {          // warp-uniform trip count
      const int k = k0 + lane;
      float v0[8], v1[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) { v0[q] = 0.f; v1[q] = 0.f; }
      if (k < e) {
        const long long kk = k;
        float rx, ry;
        V3<float> y;
        reproj_residual(Tc, mk(pts[kk * 3], pts[kk * 3 + 1], pts[kk * 3 + 2]), pix[kk * 2], pix[kk * 2 + 1], rx, ry, y);
        float j0[6], j1[6];
        reproj_rows(y, j0, j1);
#pragma unroll
        for (int q = 0; q < 6; ++q) { v0[q] = j0[q]; v1[q] = j1[q]; }
        v0[6] = rx; v1[6] = ry;
      }
      __syncwarp();
#pragma unroll
      for (int q = 0; q < 8; ++q) { tile[warp][2 * lane][q] = v0[q]; tile[warp][2 * lane + 1][q] = v1[q]; }
      __syncwarp();
#pragma unroll
      for (int s = 0; s < 8; ++s) {                                    // 8 k-steps of 8 residual rows
        const float x0 = tile[warp][s * 8 + tig][gid], x1 = tile[warp][s * 8 + tig + 4][gid];
        const unsigned h0 = f2tf32(x0), h1 = f2tf32(x1);
        const unsigned l0 = f2tf32(x0 - __uint_as_float(h0)), l1 = f2tf32(x1 - __uint_as_float(h1));
        mma_tf32(cfrag, h0, h1, h0, h1);
        mma_tf32(cfrag, h0, h1, l0, l1);
        mma_tf32(cfrag, l0, l1, h0, h1);
      }
    }
    // C rows 0..7 live in c[0], c[1] of each lane: (row gid, cols 2 tig, 2 tig + 1); fold the four warps in warp order
    red[warp][gid][2 * tig] = cfrag[0];
    red[warp][gid][2 * tig + 1] = cfrag[1];
    __syncthreads();
    if (threadIdx.x < 64) {
      const int r = threadIdx.x >> 3, q = threadIdx.x & 7;
      float t = red[0][r][q];
      for (int w = 1; w < kTcThreads / 32; ++w) t += red[w][r][q];
      red[0][r][q] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int a = 0; a < 6; ++a) {
        g[(long long)c * 6 + a] = red[0][a][6];
        for (int bb = a; bb < 6; ++bb) H[(long long)c * 21 + t++] = red[0][a][bb];
      }
      acc[0] += (double)red[0][6][6];
    }
    __syncthreads();
  }
  reduce_sums<1>(acc, ws);
}

}  // namespace b200pose

using namespace b200pose;

B200_EXPORT int b200_lm_reproj_accum_tc_f32(const float* poses, const float* pts, const float* pix, const int* seg, float* H,
                                            float* g, double* ws, long long ncam, void* stream) {
  if (ncam <= 0) return 0;
  static_assert(kTcThreads == kLmThreads, "reduce_sums assumes kLmThreads threads per CTA");
  lm_reproj_accum_tc_kernel<<<lm_grid(ncam, 1), kTcThreads, 0, (cudaStream_t)stream>>>(poses, pts, pix, seg, H, g, ws,
                                                                                      (int)ncam);
  return (int)cudaGetLastError();
}
