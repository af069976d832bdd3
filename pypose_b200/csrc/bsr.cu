// bsr.cu — block-sparse products pp.bsr_bsc_matmul: C = A B with A in BSR and B in BSC, and the gradients of both
// values arrays (C-ABI: include/b200pose.h, section "block-sparse products").  DESIGN.md §3.8.  The per-element
// accumulation is bsr_math.cuh.
//
//   b200_bsr_count    checks both index structures (pointer arrays, ranges, strictly increasing indices within each
//                     compressed row / column), transposes B's pattern to row lists (stable radix sort of B's entries on
//                     their row), and counts the block products of every A entry, |B_k| for its column k; an inclusive
//                     scan gives the triple offsets.  info = [triples, invalid]: the first host read.
//   b200_bsr_expand   one thread per triple (a, b) in A-entry order: key i * sp + j.  A stable radix sort on the key gives
//                     (i, j, k) order; an exclusive scan over key changes numbers the output block of every triple.
//                     nnz(C) is written to device memory: the second host read.
//   b200_bsr_numeric  crow (binary search of i * sp in the sorted keys), col and each output block's triple segment, then
//                     one thread per output element walks its segment (bsr_elem).
//   b200_bsr_grad     dA groups the triples by a, dB by b (stable radix sorts, so both are deterministic), then the same
//                     element kernel.  No host reads.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "bsr_math.cuh"

#define B200_EXPORT extern "C" __attribute__((visibility("default")))

namespace b200pose {
namespace {

constexpr int kBsThreads = 256;
constexpr unsigned kBsMaxGrid = 1u << 20;

long long align256(long long b) { return (b + 255) / 256 * 256; }

unsigned grid_of(long long n) {
  const long long g = (n + kBsThreads - 1) / kBsThreads;
  return (unsigned)(g < 1 ? 1 : g < kBsMaxGrid ? g : kBsMaxGrid);
}

int bits_of(unsigned long long v) {        // bits to represent v (at least 1)
  int b = 1;
  while (b < 64 && (v >> b)) ++b;
  return b;
}

#define BS_LOOP(i, n) for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (n); \
                           i += (long long)gridDim.x * blockDim.x)

// first index in [0, n) with a[idx] > v, or n
template <typename K, typename V>
__device__ __forceinline__ long long upper_bound(const K* a, long long n, V v) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] > (K)v) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// first index in [0, n) with a[idx] >= v, or n
template <typename K, typename V>
__device__ __forceinline__ long long lower_bound(const K* a, long long n, V v) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < (K)v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ---------------------------------------------------------------- workspaces
size_t sort_u32_u32_bytes(long long n) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, (int)n);
  return b;
}
size_t sort_u64_u64_bytes(long long n) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n);
  return b;
}
size_t sort_u32_u64_bytes(long long n) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr,
                                  (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n);
  return b;
}
size_t scan_i64_bytes(long long n) {
  size_t b = 0;
  cub::DeviceScan::InclusiveSum(nullptr, b, (const long long*)nullptr, (long long*)nullptr, (int)n);
  return b;
}
size_t scan_i32_bytes(long long n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, (int)n);
  return b;
}
size_t max_sz(size_t a, size_t b) { return a > b ? a : b; }

struct Carve {
  char* base;
  long long off = 0;
  template <typename P>
  P* take(long long count) {
    P* p = base ? reinterpret_cast<P*>(base + off) : nullptr;
    off += align256(count * (long long)sizeof(P));
    return p;
  }
};

// count (stage 0): the pattern of A and of B^T, kept for b200_bsr_expand
struct CountWs {
  unsigned* bad;
  int* arow;                 // (nnzA) block row of every A entry
  unsigned* acol;            // (nnzA) its block column, clamped into range
  int* bcol;                 // (nnzB) block column of every B entry
  unsigned *brow, *brow_s;   // (nnzB) its block row, clamped; sorted
  int *biota, *bt_b;         // (nnzB) 0..nnzB-1; B entries sorted by row (stable: by column within a row)
  long long* bt_ptr;         // (sn + 1) row pointers of B^T
  long long *cnt, *off;      // (nnzA) products per A entry, their inclusive scan
  void* tmp;
  size_t tmp_bytes;
};

long long count_layout(long long sn, long long nnzA, long long nnzB, char* base, CountWs* w) {
  Carve c{base};
  CountWs x;
  x.bad = c.take<unsigned>(1);
  x.arow = c.take<int>(nnzA); x.acol = c.take<unsigned>(nnzA);
  x.bcol = c.take<int>(nnzB); x.brow = c.take<unsigned>(nnzB); x.brow_s = c.take<unsigned>(nnzB);
  x.biota = c.take<int>(nnzB); x.bt_b = c.take<int>(nnzB);
  x.bt_ptr = c.take<long long>(sn + 1);
  x.cnt = c.take<long long>(nnzA); x.off = c.take<long long>(nnzA);
  x.tmp_bytes = max_sz(sort_u32_u32_bytes(nnzB), scan_i64_bytes(nnzA));
  x.tmp = c.take<char>((long long)x.tmp_bytes);
  if (w) *w = x;
  return c.off;
}

// expand (stage 1): the triples' keys; the sorted keys and the segment pointers are read by b200_bsr_numeric
struct ExpandWs {
  unsigned long long *key, *key_s, *val;   // (T)
  int* flag;                               // (T) 1 where the next key differs
  long long* segptr;                       // (T + 1) first triple of every output block
  void* tmp;
  size_t tmp_bytes;
};

long long expand_layout(long long T, char* base, ExpandWs* w) {
  Carve c{base};
  ExpandWs x;
  x.key = c.take<unsigned long long>(T); x.key_s = c.take<unsigned long long>(T);
  x.val = c.take<unsigned long long>(T);
  x.flag = c.take<int>(T);
  x.segptr = c.take<long long>(T + 1);
  x.tmp_bytes = max_sz(sort_u64_u64_bytes(T), scan_i32_bytes(T));
  x.tmp = c.take<char>((long long)x.tmp_bytes);
  if (w) *w = x;
  return c.off;
}

// grad (stage 2): triples regrouped by a or by b
struct GradWs {
  unsigned *key, *key_s;                   // (T)
  unsigned long long *val, *val_s;         // (T)
  long long* ptr;                          // (max(nnzA, nnzB) + 1)
  void* tmp;
  size_t tmp_bytes;
};

long long grad_layout(long long nnzA, long long nnzB, long long T, char* base, GradWs* w) {
  Carve c{base};
  GradWs x;
  x.key = c.take<unsigned>(T); x.key_s = c.take<unsigned>(T);
  x.val = c.take<unsigned long long>(T); x.val_s = c.take<unsigned long long>(T);
  x.ptr = c.take<long long>((nnzA > nnzB ? nnzA : nnzB) + 1);
  x.tmp_bytes = sort_u32_u64_bytes(T);
  x.tmp = c.take<char>((long long)x.tmp_bytes);
  if (w) *w = x;
  return c.off;
}

// ---------------------------------------------------------------- count
// ptr (n + 1): ptr[0] = 0, ptr[n] = nnz, non-decreasing
__global__ void bsr_check_ptr_kernel(const long long* __restrict__ ptr, long long n, long long nnz, unsigned* bad) {
  BS_LOOP(i, n + 1) {
    const long long v = ptr[i];
    if ((i == 0 && v != 0) || (i == n && v != nnz) || (i < n && v > ptr[i + 1])) atomicOr(bad, 1u);
  }
}

// every entry e of a compressed structure: its segment (row of BSR / column of BSC), its index clamped into [0, lim),
// and whether the index is in range and strictly below the next one of its segment
__global__ void bsr_entries_kernel(const long long* __restrict__ ptr, long long n, const long long* __restrict__ idx,
                                   long long nnz, long long lim, int* __restrict__ seg, unsigned* __restrict__ key,
                                   int* __restrict__ iota, unsigned* bad) {
  BS_LOOP(e, nnz) {
    long long s = upper_bound(ptr, n + 1, e) - 1;
    s = s < 0 ? 0 : s >= n ? n - 1 : s;
    const long long v = idx[e];
    bool ok = v >= 0 && v < lim;
    const long long end = ptr[s + 1];
    if (e + 1 < end && e + 1 < nnz && !(v < idx[e + 1])) ok = false;
    if (!ok) atomicOr(bad, 1u);
    seg[e] = (int)s;
    key[e] = (unsigned)(v < 0 ? 0 : v >= lim ? lim - 1 : v);
    if (iota) iota[e] = (int)e;
  }
}

__global__ void bsr_lower_bound_kernel(const unsigned* __restrict__ keys, long long n, long long m,
                                       long long* __restrict__ ptr) {
  BS_LOOP(g, m + 1) ptr[g] = lower_bound(keys, n, g);
}

__global__ void bsr_products_kernel(const unsigned* __restrict__ acol, long long nnzA, const long long* __restrict__ bt_ptr,
                                    long long* __restrict__ cnt) {
  BS_LOOP(a, nnzA) {
    const unsigned k = acol[a];
    cnt[a] = bt_ptr[k + 1] - bt_ptr[k];
  }
}

__global__ void bsr_info_kernel(const long long* __restrict__ off, long long nnzA, const unsigned* bad, long long* info) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    info[0] = nnzA > 0 ? off[nnzA - 1] : 0;
    info[1] = *bad ? 1 : 0;
  }
}

int count_run(const long long* a_crow, const long long* a_col, long long sm, long long nnzA, const long long* b_ccol,
              const long long* b_row, long long sp, long long nnzB, long long sn, void* ws, long long* info,
              cudaStream_t s) {
  // block rows, columns and entries are stored as 32-bit indices
  if (sm < 1 || sn < 1 || sp < 1 || nnzA < 0 || nnzB < 0 || nnzA > 0x7fffffffLL || nnzB > 0x7fffffffLL ||
      sm > 0x7fffffffLL || sn > 0x7fffffffLL || sp > 0x7fffffffLL || !a_crow || !b_ccol || !ws || !info ||
      (nnzA && !a_col) || (nnzB && !b_row))
    return (int)cudaErrorInvalidValue;
  CountWs w;
  count_layout(sn, nnzA, nnzB, reinterpret_cast<char*>(ws), &w);
  cudaError_t e = cudaMemsetAsync(w.bad, 0, sizeof(unsigned), s);
  if (e != cudaSuccess) return (int)e;
  bsr_check_ptr_kernel<<<grid_of(sm + 1), kBsThreads, 0, s>>>(a_crow, sm, nnzA, w.bad);
  bsr_check_ptr_kernel<<<grid_of(sp + 1), kBsThreads, 0, s>>>(b_ccol, sp, nnzB, w.bad);
  if (nnzA) bsr_entries_kernel<<<grid_of(nnzA), kBsThreads, 0, s>>>(a_crow, sm, a_col, nnzA, sn, w.arow, w.acol,
                                                                     nullptr, w.bad);
  if (nnzB) {
    bsr_entries_kernel<<<grid_of(nnzB), kBsThreads, 0, s>>>(b_ccol, sp, b_row, nnzB, sn, w.bcol, w.brow, w.biota, w.bad);
    size_t tb = w.tmp_bytes;
    e = cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.brow, w.brow_s, w.biota, w.bt_b, (int)nnzB, 0,
                                        bits_of((unsigned long long)(sn - 1)), s);
    if (e != cudaSuccess) return (int)e;
  }
  bsr_lower_bound_kernel<<<grid_of(sn + 1), kBsThreads, 0, s>>>(w.brow_s, nnzB, sn, w.bt_ptr);
  if (nnzA) {
    bsr_products_kernel<<<grid_of(nnzA), kBsThreads, 0, s>>>(w.acol, nnzA, w.bt_ptr, w.cnt);
    size_t tb = w.tmp_bytes;
    e = cub::DeviceScan::InclusiveSum(w.tmp, tb, w.cnt, w.off, (int)nnzA, s);
    if (e != cudaSuccess) return (int)e;
  }
  bsr_info_kernel<<<1, 32, 0, s>>>(w.off, nnzA, w.bad, info);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- expand
// triple t of A entry a = first a with off[a] > t; the (t - start)-th entry of B^T's row col[a]
__global__ void bsr_expand_kernel(const long long* __restrict__ off, long long nnzA, const int* __restrict__ arow,
                                  const unsigned* __restrict__ acol, const long long* __restrict__ bt_ptr,
                                  const int* __restrict__ bt_b, const int* __restrict__ bcol, long long sp, long long T,
                                  unsigned long long* __restrict__ key, unsigned long long* __restrict__ val) {
  BS_LOOP(t, T) {
    const long long a = upper_bound(off, nnzA, t);
    const long long start = a > 0 ? off[a - 1] : 0;
    const int b = bt_b[bt_ptr[acol[a]] + (t - start)];
    key[t] = (unsigned long long)arow[a] * (unsigned long long)sp + (unsigned long long)bcol[b];
    val[t] = ((unsigned long long)a << 32) | (unsigned)b;
  }
}

__global__ void bsr_flag_kernel(const unsigned long long* __restrict__ key, long long T, int* __restrict__ flag) {
  BS_LOOP(t, T) flag[t] = t + 1 < T && key[t + 1] != key[t];
}

__global__ void bsr_nnz_kernel(const int* __restrict__ seg, long long T, long long* __restrict__ nnz) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *nnz = (long long)seg[T - 1] + 1;
}

int expand_run(const long long* a_col, long long nnzA, long long sm, long long sp, long long sn, long long nnzB,
               void* ws_count, long long T, void* ws, unsigned long long* tri, int* seg, long long* nnz, cudaStream_t s) {
  if (T < 1 || T > 0x7fffffffLL || nnzA < 1 || nnzB < 1 || sm < 1 || sp < 1 || sm > 0x7fffffffLL ||
      sp > 0x7fffffffLL || !a_col || !ws_count || !ws || !tri || !seg || !nnz)
    return (int)cudaErrorInvalidValue;
  CountWs c;
  count_layout(sn, nnzA, nnzB, reinterpret_cast<char*>(ws_count), &c);
  ExpandWs w;
  expand_layout(T, reinterpret_cast<char*>(ws), &w);
  bsr_expand_kernel<<<grid_of(T), kBsThreads, 0, s>>>(c.off, nnzA, c.arow, c.acol, c.bt_ptr, c.bt_b, c.bcol, sp, T,
                                                       w.key, w.val);
  size_t tb = w.tmp_bytes;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.key, w.key_s, w.val, tri, (int)T, 0,
                                                  bits_of((unsigned long long)sm * (unsigned long long)sp - 1), s);
  if (e != cudaSuccess) return (int)e;
  bsr_flag_kernel<<<grid_of(T), kBsThreads, 0, s>>>(w.key_s, T, w.flag);
  tb = w.tmp_bytes;
  e = cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.flag, seg, (int)T, s);     // seg[t] = output block of triple t
  if (e != cudaSuccess) return (int)e;
  bsr_nnz_kernel<<<1, 32, 0, s>>>(seg, T, nnz);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- numeric
// col and the first triple of every output block; crow[i] = output blocks with a key below i * sp
__global__ void bsr_segments_kernel(const unsigned long long* __restrict__ key_s, const int* __restrict__ flag,
                                    const int* __restrict__ seg, long long T, long long sp, long long nnz,
                                    long long* __restrict__ segptr, long long* __restrict__ col) {
  BS_LOOP(t, T) {
    if (t == 0 || flag[t - 1]) {
      segptr[seg[t]] = t;
      col[seg[t]] = (long long)(key_s[t] % (unsigned long long)sp);
    }
    if (t == T - 1) segptr[nnz] = T;
  }
}

__global__ void bsr_crow_kernel(const unsigned long long* __restrict__ key_s, const int* __restrict__ seg, long long T,
                                long long sm, long long sp, long long nnz, long long* __restrict__ crow) {
  BS_LOOP(i, sm + 1) {
    const long long p = lower_bound(key_s, T, (unsigned long long)i * (unsigned long long)sp);
    crow[i] = p < T ? (long long)seg[p] : nnz;
  }
}

// out (nout, dx, dy) contiguous; output block g sums the triples ptr[g] .. ptr[g + 1] - 1
template <typename T>
__global__ void __launch_bounds__(kBsThreads) bsr_numeric_kernel(const T* __restrict__ L, BsrOperand lo,
                                                                 const T* __restrict__ R, BsrOperand ro,
                                                                 const unsigned long long* __restrict__ tri,
                                                                 const long long* __restrict__ ptr, long long nout,
                                                                 int dx, int dy, int dz, T* __restrict__ out) {
  const long long per = (long long)dx * dy;
  BS_LOOP(e, nout * per) {
    const long long g = e / per;
    const int r = (int)(e - g * per), x = r / dy, y = r - x * dy;
    out[e] = bsr_elem(L, lo, R, ro, tri, ptr[g], ptr[g + 1], x, y, dz);
  }
}

template <typename T>
int numeric_run(const T* A, BsrOperand ao, const T* B, BsrOperand bo, int dm, int dn, int dp, long long sm, long long sp,
                long long T_, void* ws, const unsigned long long* tri, const int* seg, long long nnz, long long* crow,
                long long* col, T* C, cudaStream_t s) {
  if (T_ < 1 || T_ > 0x7fffffffLL || nnz < 1 || nnz > T_ || dm < 1 || dn < 1 || dp < 1 || sm < 1 || sp < 1 || !A ||
      !B || !ws || !tri || !seg || !crow || !col || !C)
    return (int)cudaErrorInvalidValue;
  ExpandWs w;
  expand_layout(T_, reinterpret_cast<char*>(ws), &w);
  bsr_segments_kernel<<<grid_of(T_), kBsThreads, 0, s>>>(w.key_s, w.flag, seg, T_, sp, nnz, w.segptr, col);
  bsr_crow_kernel<<<grid_of(sm + 1), kBsThreads, 0, s>>>(w.key_s, seg, T_, sm, sp, nnz, crow);
  bsr_numeric_kernel<T><<<grid_of(nnz * dm * dp), kBsThreads, 0, s>>>(A, ao, B, bo, tri, w.segptr, nnz, dm, dp, dn, C);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- gradients
// by_a: key a, value (c << 32) | b; else key b, value (a << 32) | c
__global__ void bsr_regroup_kernel(const unsigned long long* __restrict__ tri, const int* __restrict__ seg, long long T,
                                   int by_a, unsigned* __restrict__ key, unsigned long long* __restrict__ val) {
  BS_LOOP(t, T) {
    const unsigned long long p = tri[t];
    const unsigned a = (unsigned)(p >> 32), b = (unsigned)(p & 0xffffffffull), c = (unsigned)seg[t];
    key[t] = by_a ? a : b;
    val[t] = by_a ? ((unsigned long long)c << 32) | b : ((unsigned long long)a << 32) | c;
  }
}

template <typename T>
int grad_run(const T* A, BsrOperand ao, const T* B, BsrOperand bo, const T* dC, int dm, int dn, int dp,
             const unsigned long long* tri, const int* seg, long long T_, long long nnzA, long long nnzB, void* ws, T* dA,
             T* dB, cudaStream_t s) {
  if (T_ < 1 || T_ > 0x7fffffffLL || nnzA < 1 || nnzB < 1 || dm < 1 || dn < 1 || dp < 1 || !A || !B || !dC || !tri ||
      !seg || !ws)
    return (int)cudaErrorInvalidValue;
  GradWs w;
  grad_layout(nnzA, nnzB, T_, reinterpret_cast<char*>(ws), &w);
  const BsrOperand co{(long long)dm * dp, dp, 1};
  for (int by_a = 1; by_a >= 0; --by_a) {
    T* out = by_a ? dA : dB;
    if (!out) continue;
    const long long n = by_a ? nnzA : nnzB;
    bsr_regroup_kernel<<<grid_of(T_), kBsThreads, 0, s>>>(tri, seg, T_, by_a, w.key, w.val);
    size_t tb = w.tmp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.key, w.key_s, w.val, w.val_s, (int)T_, 0,
                                                    bits_of((unsigned long long)(n - 1)), s);
    if (e != cudaSuccess) return (int)e;
    bsr_lower_bound_kernel<<<grid_of(n + 1), kBsThreads, 0, s>>>(w.key_s, T_, n, w.ptr);
    if (by_a)       // dA[a] (dm, dn) = sum dC[c] (dm, dp) B[b]^T (dp, dn)
      bsr_numeric_kernel<T><<<grid_of(n * dm * dn), kBsThreads, 0, s>>>(dC, co, B, BsrOperand{bo.sb, bo.s1, bo.s0},
                                                                        w.val_s, w.ptr, n, dm, dn, dp, out);
    else            // dB[b] (dn, dp) = sum A[a]^T (dn, dm) dC[c] (dm, dp)
      bsr_numeric_kernel<T><<<grid_of(n * dn * dp), kBsThreads, 0, s>>>(A, BsrOperand{ao.sb, ao.s1, ao.s0}, dC, co,
                                                                        w.val_s, w.ptr, n, dn, dp, dm, out);
  }
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace b200pose

using namespace b200pose;

B200_EXPORT long long b200_bsr_workspace_bytes(int stage, long long sn, long long nnzA, long long nnzB, long long T) {
  if (sn < 0 || nnzA < 0 || nnzB < 0 || T < 0 || sn > 0x7fffffffLL || nnzA > 0x7fffffffLL || nnzB > 0x7fffffffLL ||
      T > 0x7fffffffLL)
    return 0;
  if (stage == 0) return count_layout(sn, nnzA, nnzB, nullptr, nullptr);
  if (stage == 1) return expand_layout(T, nullptr, nullptr);
  if (stage == 2) return grad_layout(nnzA, nnzB, T, nullptr, nullptr);
  return 0;
}

B200_EXPORT int b200_bsr_count(const long long* a_crow, const long long* a_col, long long sm, long long nnzA,
                               const long long* b_ccol, const long long* b_row, long long sp, long long nnzB, long long sn,
                               void* ws, long long* info, void* stream) {
  return count_run(a_crow, a_col, sm, nnzA, b_ccol, b_row, sp, nnzB, sn, ws, info, (cudaStream_t)stream);
}

B200_EXPORT int b200_bsr_expand(const long long* a_col, long long nnzA, long long sm, long long sp, long long sn,
                                long long nnzB, void* ws_count, long long T, void* ws, unsigned long long* tri, int* seg,
                                long long* nnz, void* stream) {
  return expand_run(a_col, nnzA, sm, sp, sn, nnzB, ws_count, T, ws, tri, seg, nnz, (cudaStream_t)stream);
}

#define B200_BSR_ENTRIES(CT, SFX)                                                                                          \
  B200_EXPORT int b200_bsr_numeric_##SFX(const CT* A, long long a_sb, long long a_s0, long long a_s1, const CT* B,       \
                                         long long b_sb, long long b_s0, long long b_s1, int dm, int dn, int dp,         \
                                         long long sm, long long sp, long long T, void* ws,                              \
                                         const unsigned long long* tri, const int* seg, long long nnz, long long* crow,  \
                                         long long* col, CT* C, void* stream) {                                           \
    return numeric_run<CT>(A, BsrOperand{a_sb, a_s0, a_s1}, B, BsrOperand{b_sb, b_s0, b_s1}, dm, dn, dp, sm, sp, T, ws,  \
                           tri, seg, nnz, crow, col, C, (cudaStream_t)stream);                                            \
  }                                                                                                                        \
  B200_EXPORT int b200_bsr_grad_##SFX(const CT* A, long long a_sb, long long a_s0, long long a_s1, const CT* B,          \
                                      long long b_sb, long long b_s0, long long b_s1, const CT* dC, int dm, int dn,      \
                                      int dp, const unsigned long long* tri, const int* seg, long long T,                \
                                      long long nnzA, long long nnzB, void* ws, CT* dA, CT* dB, void* stream) {          \
    return grad_run<CT>(A, BsrOperand{a_sb, a_s0, a_s1}, B, BsrOperand{b_sb, b_s0, b_s1}, dC, dm, dn, dp, tri, seg, T,   \
                        nnzA, nnzB, ws, dA, dB, (cudaStream_t)stream);                                                    \
  }

B200_BSR_ENTRIES(float, f32)
B200_BSR_ENTRIES(double, f64)
