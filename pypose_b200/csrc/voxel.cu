// voxel.cu — voxel down-sampling of one point cloud (C-ABI: include/b200pose.h, section "point clouds").  DESIGN.md §3.5.
//
// Two entry points with one host read between them (the number of voxels M, which sizes the output):
//   b200_voxel_sort: integer voxel coordinates -> key groups of <= 64 bits -> stable LSD radix sort of the row indices,
//     one group at a time (CUB DeviceRadixSort) -> segment heads -> segment ids (CUB inclusive scan), segment starts,
//     the voxel id of every point at its original index, and M;
//   b200_voxel_reduce: per voxel, either the centroid (sum of the member rows in increasing original index, starting
//     from 0, divided by the member count, all in the data dtype) or the row of one member picked by a given uniform.
// The voxel coordinate of a point is trunc((p_d - min_d) / v_d) with a separate subtract and divide, as the reference
// computes it; the host plans the key layout from the coordinate ranges (pypose_b200/function/geometry.py).
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <initializer_list>

#define B200_EXPORT extern "C" __attribute__((visibility("default")))

namespace b200pose {
namespace {

constexpr int kVoxMaxDim = 16;
constexpr int kVoxThreads = 256;

// Key layout of every voxel dimension: its minimum and size in the data dtype, the lowest integer coordinate, the key
// group it belongs to and its shift inside that group's key.
struct VoxPlan {
  double mn[kVoxMaxDim], v[kVoxMaxDim];
  long long lo[kVoxMaxDim];
  int group[kVoxMaxDim], shift[kVoxMaxDim];
  int vdim;
};

template <typename T> __device__ __forceinline__ long long vox_coord(const T* __restrict__ row, const VoxPlan& pl, int d) {
  const T a = row[d] - (T)pl.mn[d];
  return (long long)(a / (T)pl.v[d]);
}

template <typename T> __device__ __forceinline__ unsigned long long vox_key(const T* __restrict__ row, const VoxPlan& pl, int g) {
  unsigned long long k = 0;
  for (int d = 0; d < pl.vdim; ++d)
    if (pl.group[d] == g) k |= (unsigned long long)(vox_coord(row, pl, d) - pl.lo[d]) << pl.shift[d];
  return k;
}

// key of group g for sorted position i (row perm[i]; perm == NULL: the identity)
template <typename T>
__global__ void voxel_key_kernel(const T* __restrict__ P, int N, int D, VoxPlan pl, int g, const int* __restrict__ perm,
                                 unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const int i = blockIdx.x * kVoxThreads + threadIdx.x;
  if (i >= N) return;
  const int row = perm ? perm[i] : i;
  keys[i] = vox_key(P + (long long)row * D, pl, g);
  vals[i] = row;
}

// head[i] = 1 where sorted row i starts a voxel.  keys: the sorted keys when there is one group, else NULL (all groups
// are recomputed for the two neighbouring rows).
template <typename T>
__global__ void voxel_head_kernel(const T* __restrict__ P, int N, int D, VoxPlan pl, int ngroups,
                                  const unsigned long long* __restrict__ keys, const int* __restrict__ perm,
                                  int* __restrict__ head) {
  const int i = blockIdx.x * kVoxThreads + threadIdx.x;
  if (i >= N) return;
  int h = i == 0;
  if (i > 0) {
    if (keys) {
      h = keys[i] != keys[i - 1];
    } else {
      const T* a = P + (long long)perm[i] * D;
      const T* b = P + (long long)perm[i - 1] * D;
      for (int g = 0; g < ngroups && !h; ++g) h = vox_key(a, pl, g) != vox_key(b, pl, g);
    }
  }
  head[i] = h;
}

// seg = inclusive scan of the heads: start[seg - 1] = i at every head, start[M] = N, M, and vid[perm[i]] = seg - 1
__global__ void voxel_seg_kernel(const int* __restrict__ perm, const int* __restrict__ head, const int* __restrict__ seg,
                                 int N, int* __restrict__ start, long long* __restrict__ vid, long long* __restrict__ M) {
  const int i = blockIdx.x * kVoxThreads + threadIdx.x;
  if (i >= N) return;
  const int s = seg[i] - 1;
  if (head[i]) start[s] = i;
  if (i == N - 1) { start[s + 1] = N; *M = s + 1; }
  vid[perm[i]] = s;
}

// one thread per (voxel, column): sequential sum of the members in sorted order (= increasing original index), the
// count accumulated the same way in the data dtype, then the division
template <typename T>
__global__ void voxel_centroid_kernel(const T* __restrict__ P, int D, const int* __restrict__ perm,
                                      const int* __restrict__ start, long long M, T* __restrict__ out, T* __restrict__ cnt) {
  const long long t = (long long)blockIdx.x * kVoxThreads + threadIdx.x;
  if (t >= M * D) return;
  const long long m = t / D;
  const int c = (int)(t - m * D);
  const int b = start[m], e = start[m + 1];
  T acc = T(0), n = T(0);
  for (int i = b; i < e; ++i) {
    acc += P[(long long)perm[i] * D + c];
    n += T(1);
  }
  out[t] = acc / n;
  if (c == 0 && cnt) cnt[m] = n;
}

// one thread per voxel: member min(floor(u count), count - 1) in sorted order
__global__ void voxel_pick_kernel(const int* __restrict__ perm, const int* __restrict__ start, long long M,
                                  const double* __restrict__ u, long long* __restrict__ sel) {
  const long long m = (long long)blockIdx.x * kVoxThreads + threadIdx.x;
  if (m >= M) return;
  const int b = start[m], n = start[m + 1] - b;
  const long long r = min((long long)floor(u[m] * (double)n), (long long)n - 1);
  sel[m] = perm[b + r];
}

bool vox_device_ptrs(std::initializer_list<const void*> ps) {
  for (const void* p : ps) {
    if (!p) continue;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) return false;
  }
  return true;
}

long long align256(long long b) { return (b + 255) / 256 * 256; }

size_t cub_temp_bytes(int N) {
  size_t sort = 0, scan = 0;
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, sort, k, v, N, 0, 64);
  cub::DeviceScan::InclusiveSum(nullptr, scan, (const int*)nullptr, (int*)nullptr, N);
  return sort > scan ? sort : scan;
}

// workspace: keys[2][N] u64 | perm[2][N] | head[N] | seg[N] | start[N + 1] | CUB temporary storage (each 256-aligned)
struct VoxWs {
  unsigned long long* keys[2];
  int *perm[2], *head, *seg, *start;
  void* tmp;
  size_t tmp_bytes;
};

long long vox_ws_layout(long long N, char* base, VoxWs* w) {
  long long off = 0;
  auto take = [&](long long bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  char* k0 = take(N * 8); char* k1 = take(N * 8);
  char* p0 = take(N * 4); char* p1 = take(N * 4);
  char* h = take(N * 4); char* s = take(N * 4); char* st = take((N + 1) * 4);
  const size_t tb = cub_temp_bytes((int)N);
  char* tmp = take((long long)tb);
  if (w) {
    w->keys[0] = reinterpret_cast<unsigned long long*>(k0); w->keys[1] = reinterpret_cast<unsigned long long*>(k1);
    w->perm[0] = reinterpret_cast<int*>(p0); w->perm[1] = reinterpret_cast<int*>(p1);
    w->head = reinterpret_cast<int*>(h); w->seg = reinterpret_cast<int*>(s); w->start = reinterpret_cast<int*>(st);
    w->tmp = tmp; w->tmp_bytes = tb;
  }
  return off;
}

template <typename T>
int voxel_sort_run(const T* P, long long N, int D, int vdim, const double* bounds_host, const long long* plan_host,
                   int ngroups, void* ws, long long* vid, long long* M, cudaStream_t s) {
  if (N <= 0) return 0;
  if (!P || !ws || !vid || !M || !bounds_host || !plan_host || !vox_device_ptrs({P, ws, vid, M}))
    return (int)cudaErrorInvalidValue;
  if (N > 0x7fffffffLL || vdim < 1 || vdim > kVoxMaxDim || vdim > D || ngroups < 1 || ngroups > vdim)
    return (int)cudaErrorInvalidValue;
  VoxPlan pl;
  pl.vdim = vdim;
  for (int d = 0; d < vdim; ++d) {
    pl.mn[d] = bounds_host[2 * d];
    pl.v[d] = bounds_host[2 * d + 1];
    pl.lo[d] = plan_host[3 * d];
    pl.group[d] = (int)plan_host[3 * d + 1];
    pl.shift[d] = (int)plan_host[3 * d + 2];
    if (pl.group[d] < 0 || pl.group[d] >= ngroups || pl.shift[d] < 0 || pl.shift[d] > 63) return (int)cudaErrorInvalidValue;
  }
  const long long* gbits = plan_host + 3 * vdim;
  VoxWs w;
  vox_ws_layout(N, reinterpret_cast<char*>(ws), &w);
  const int n = (int)N;
  const unsigned grid = (unsigned)((N + kVoxThreads - 1) / kVoxThreads);
  cub::DoubleBuffer<unsigned long long> kb(w.keys[0], w.keys[1]);
  cub::DoubleBuffer<int> pb(w.perm[0], w.perm[1]);
  // least significant group first; stability keeps equal keys in the order of the previous pass (= index order)
  for (int g = ngroups - 1; g >= 0; --g) {
    const int bits = (int)gbits[g];
    if (bits < 0 || bits > 64) return (int)cudaErrorInvalidValue;
    const bool first = g == ngroups - 1;
    voxel_key_kernel<T><<<grid, kVoxThreads, 0, s>>>(P, n, D, pl, g, first ? nullptr : pb.Current(), kb.Current(), pb.Current());
    if (bits == 0) continue;
    size_t tb = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, pb, n, 0, bits, s);
    if (tb > w.tmp_bytes) return (int)cudaErrorInvalidValue;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(w.tmp, tb, kb, pb, n, 0, bits, s);
    if (e != cudaSuccess) return (int)e;
  }
  voxel_head_kernel<T><<<grid, kVoxThreads, 0, s>>>(P, n, D, pl, ngroups, ngroups == 1 ? kb.Current() : nullptr,
                                                    pb.Current(), w.head);
  size_t tb = w.tmp_bytes;
  cudaError_t e = cub::DeviceScan::InclusiveSum(w.tmp, tb, w.head, w.seg, n, s);
  if (e != cudaSuccess) return (int)e;
  voxel_seg_kernel<<<grid, kVoxThreads, 0, s>>>(pb.Current(), w.head, w.seg, n, w.start, vid, M);
  // the reduce step reads the sorted rows from perm[0]
  if (pb.Current() != w.perm[0]) {
    e = cudaMemcpyAsync(w.perm[0], pb.Current(), N * sizeof(int), cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaGetLastError();
}

template <typename T>
int voxel_reduce_run(const T* P, long long N, int D, void* ws, long long M, const double* u, T* out, T* cnt,
                     long long* sel, cudaStream_t s) {
  if (N <= 0 || M <= 0) return 0;
  if (!P || !ws || (!u && !out) || (u && !sel) || !vox_device_ptrs({P, ws, u, out, cnt, sel}))
    return (int)cudaErrorInvalidValue;
  if (N > 0x7fffffffLL || M > N || D < 1) return (int)cudaErrorInvalidValue;
  VoxWs w;
  vox_ws_layout(N, reinterpret_cast<char*>(ws), &w);
  if (u) {
    voxel_pick_kernel<<<(unsigned)((M + kVoxThreads - 1) / kVoxThreads), kVoxThreads, 0, s>>>(w.perm[0], w.start, M, u, sel);
  } else {
    const long long t = M * D;
    voxel_centroid_kernel<T><<<(unsigned)((t + kVoxThreads - 1) / kVoxThreads), kVoxThreads, 0, s>>>(P, D, w.perm[0], w.start,
                                                                                                   M, out, cnt);
  }
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace b200pose

using namespace b200pose;

B200_EXPORT long long b200_voxel_workspace_bytes(long long N) {
  if (N <= 0 || N > 0x7fffffffLL) return 0;
  return vox_ws_layout(N, nullptr, nullptr);
}

#define B200_VOXEL_ENTRIES(CT, SFX)                                                                                         \
  B200_EXPORT int b200_voxel_sort_##SFX(const CT* pts, long long N, int D, int vdim, const double* bounds_host,            \
                                        const long long* plan_host, int ngroups, void* ws, long long* vid, long long* M,  \
                                        void* stream) {                                                                    \
    return voxel_sort_run<CT>(pts, N, D, vdim, bounds_host, plan_host, ngroups, ws, vid, M, (cudaStream_t)stream);        \
  }                                                                                                                        \
  B200_EXPORT int b200_voxel_reduce_##SFX(const CT* pts, long long N, int D, void* ws, long long M, const double* u,       \
                                          CT* out, CT* count, long long* sel, void* stream) {                             \
    return voxel_reduce_run<CT>(pts, N, D, ws, M, u, out, count, sel, (cudaStream_t)stream);                               \
  }

B200_VOXEL_ENTRIES(float, f32)
B200_VOXEL_ENTRIES(double, f64)
