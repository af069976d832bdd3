// scan.cu — single-pass group-product scans (cumprod / cummul) and the fused IMU preintegration.
//
// Reference: pypose/basics/ops.py:29-58 (`cumops_`: ceil(log2 L)+1 full passes of index_select + a ~37-op
// group multiply + index_copy_), pypose/module/imu_preintegrator.py:314-384 (`integrate`).
//
// Layout: (B, L, d) row-major, scan along L.  One CTA owns one sequence and walks it tile by tile, carrying
// the running prefix in registers/shared memory, so every element is read once and written once (the
// reference moves 2 d (log2 L + 1) words per element).  Inside a tile each thread scans CH consecutive
// elements in registers, thread totals are scanned with order-preserving warp shuffles, warp totals through
// shared memory.  The group operation is not commutative: every combine keeps (earlier, later) order.
#include <cuda_runtime.h>
#include <stdlib.h>
#include <stdint.h>
#include "lie_math.cuh"
#include "b200pose.h"   // every definition is checked against the generated declaration
#include "imu_cov_math.cuh"
#include "tma.cuh"

namespace b200pose {

#define B200_EXPORT extern "C" __attribute__((visibility("default")))
constexpr int kScanThreads = 128;

template <typename T> __device__ __forceinline__ T shfl_up(T v, int o) { return __shfl_up_sync(0xffffffffu, v, o); }
template <typename T> __device__ __forceinline__ T shfl_idx(T v, int l) { return __shfl_sync(0xffffffffu, v, l); }

template <typename T> __device__ __forceinline__ Elem<T> elem_shfl_up(const Elem<T>& e, int o) {
  Elem<T> r;
  r.t = mk(shfl_up(e.t.x, o), shfl_up(e.t.y, o), shfl_up(e.t.z, o));
  r.q.v = mk(shfl_up(e.q.v.x, o), shfl_up(e.q.v.y, o), shfl_up(e.q.v.z, o));
  r.q.w = shfl_up(e.q.w, o);
  r.s = shfl_up(e.s, o);
  return r;
}
template <typename T> __device__ __forceinline__ Elem<T> elem_identity() {
  Elem<T> e; e.t = mk(T(0), T(0), T(0)); e.q.v = mk(T(0), T(0), T(0)); e.q.w = T(1); e.s = T(1); return e;
}
// combine(earlier, later): y_i = y_{i-1} * x_i (right) or x_i * y_{i-1} (left)   (basics/ops.py:41-58)
template <class G, typename T, bool LEFT> __device__ __forceinline__ Elem<T> combine(const Elem<T>& a, const Elem<T>& b) {
  return LEFT ? g_mul<G, T>(b, a) : g_mul<G, T>(a, b);
}

// Block-wide exclusive scan of one Elem per thread (thread order = sequence order).
// Returns the exclusive prefix for this thread (identity for thread 0) and the block total via `total`.
template <class G, typename T, bool LEFT>
__device__ __forceinline__ Elem<T> block_exclusive(const Elem<T>& mine, Elem<T>& total, T* sh /* [warps+1][8] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kScanThreads / 32;
  Elem<T> inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Elem<T> up = elem_shfl_up(inc, o);
    if (lane >= o) inc = combine<G, T, LEFT>(up, inc);
  }
  Elem<T> excl = elem_shfl_up(inc, 1);
  if (lane == 0) excl = elem_identity<T>();
  if (lane == 31) store_elem<Sim3g, T>(sh + warp * 8, inc);      // widest layout holds every group
  __syncthreads();
  Elem<T> wpre = elem_identity<T>();
  Elem<T> tot = elem_identity<T>();
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    Elem<T> e = load_elem<Sim3g, T>(sh + w * 8);
    if (w < warp) wpre = combine<G, T, LEFT>(wpre, e);
    tot = combine<G, T, LEFT>(tot, e);
  }
  __syncthreads();
  total = tot;
  return combine<G, T, LEFT>(wpre, excl);
}

// ------------------------------------------------------------------------------------------------
// generic group cumprod
// ------------------------------------------------------------------------------------------------
// Tile staging.  A thread owns CH consecutive rows (CH * D words); read straight from global memory, every load
// instruction of a warp touches 32 different 128-byte lines, so the LSU wavefront count, not the bytes, sets the time.  The tile therefore goes through shared memory:
// coalesced 16-byte (or 4/8-byte, when the tile is not 16-byte aligned) global accesses, and each thread's CH * D words sit
// at stride CH * D + 1 words — odd, so the per-thread reads and writes are bank-conflict free.
template <typename T, int D, int CH> struct TileSmem {
  static constexpr int PER = CH * D;                       // words owned by one thread
  static constexpr int STRIDE = PER + 1;
  static constexpr int WORDS = kScanThreads * STRIDE;
};
template <typename T, int D, int CH>
__device__ __forceinline__ void tile_load(const T* __restrict__ src, int words, T* __restrict__ sm) {
  constexpr int PER = TileSmem<T, D, CH>::PER, EV = 16 / (int)sizeof(T);
  constexpr int NV = PER / EV;                               // 16-byte vectors per thread in a full tile (= 2 D)
  static_assert(PER % EV == 0, "a thread's rows are a whole number of 16-byte vectors");
  if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    const float4* v4 = reinterpret_cast<const float4*>(src);
    if (words == kScanThreads * PER) {                       // full tile: every load in flight before the first store
      float4 x[NV];
#pragma unroll
      for (int j = 0; j < NV; ++j) x[j] = v4[threadIdx.x + j * kScanThreads];
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const T* e = reinterpret_cast<const T*>(&x[j]);
        const int v = threadIdx.x + j * kScanThreads;             // a vector never straddles two threads' words
        T* d = sm + v * EV + v / NV;
#pragma unroll
        for (int k = 0; k < EV; ++k) d[k] = e[k];
      }
    } else {
      const int nv = words / EV;
#pragma unroll 4
      for (int v = threadIdx.x; v < nv; v += kScanThreads) {
        const float4 x = v4[v];
        const T* e = reinterpret_cast<const T*>(&x);
#pragma unroll
        for (int k = 0; k < EV; ++k) {
          const int w = v * EV + k;
          sm[w + w / PER] = e[k];
        }
      }
      for (int w = nv * EV + threadIdx.x; w < words; w += kScanThreads) sm[w + w / PER] = src[w];
    }
  } else {
#pragma unroll 8
    for (int w = threadIdx.x; w < words; w += kScanThreads) sm[w + w / PER] = src[w];
  }
  __syncthreads();
}
template <typename T, int D, int CH>
__device__ __forceinline__ void tile_store(T* __restrict__ dst, int words, const T* __restrict__ sm) {
  constexpr int PER = TileSmem<T, D, CH>::PER, EV = 16 / (int)sizeof(T);
  constexpr int NV = PER / EV;
  __syncthreads();
  if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0 && words == kScanThreads * PER) {
    float4* v4 = reinterpret_cast<float4*>(dst);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int v = threadIdx.x + j * kScanThreads;
      const T* d = sm + v * EV + v / NV;
      float4 x;
      T* e = reinterpret_cast<T*>(&x);
#pragma unroll
      for (int k = 0; k < EV; ++k) e[k] = d[k];
      v4[v] = x;
    }
  } else if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    const int nv = words / EV;
    float4* v4 = reinterpret_cast<float4*>(dst);
#pragma unroll 4
    for (int v = threadIdx.x; v < nv; v += kScanThreads) {
      float4 x;
      T* e = reinterpret_cast<T*>(&x);
#pragma unroll
      for (int k = 0; k < EV; ++k) {
        const int w = v * EV + k;
        e[k] = sm[w + w / PER];
      }
      v4[v] = x;
    }
    for (int w = nv * EV + threadIdx.x; w < words; w += kScanThreads) dst[w] = sm[w + w / PER];
  } else {
#pragma unroll 8
    for (int w = threadIdx.x; w < words; w += kScanThreads) dst[w] = sm[w + w / PER];
  }
}

template <class G, typename T, bool LEFT, int CH>
__global__ void __launch_bounds__(kScanThreads) cumprod_kernel(const T* __restrict__ in, T* __restrict__ out, long long L) {
  using TS = TileSmem<T, G::D, CH>;
  __shared__ T sh[(kScanThreads / 32) * 8];
  __shared__ __align__(16) T tile[TS::WORDS];
  const T* src = in + (long long)blockIdx.x * L * G::D;
  T* dst = out + (long long)blockIdx.x * L * G::D;
  Elem<T> carry = elem_identity<T>();
  constexpr long long TILE = (long long)kScanThreads * CH;
  const int first = threadIdx.x * CH;
  T* mine = tile + threadIdx.x * TS::STRIDE;
  for (long long base = 0; base < L; base += TILE) {
    const int rows = (int)(L - base < TILE ? L - base : TILE);
    tile_load<T, G::D, CH>(src + base * G::D, rows * G::D, tile);        // coalesced; see TileSmem
    Elem<T> loc[CH];
    Elem<T> run = elem_identity<T>();
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (first + c < rows) {
        T row[G::D];
#pragma unroll
        for (int k = 0; k < G::D; ++k) row[k] = mine[c * G::D + k];
        run = combine<G, T, LEFT>(run, load_elem<G, T>(row));
      }
      loc[c] = run;
    }
    Elem<T> total;
    Elem<T> pre = combine<G, T, LEFT>(carry, block_exclusive<G, T, LEFT>(run, total, sh));
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (first + c < rows) {
        T row[G::D];
        store_elem<G, T>(row, combine<G, T, LEFT>(pre, loc[c]));
#pragma unroll
        for (int k = 0; k < G::D; ++k) mine[c * G::D + k] = row[k];
      }
    }
    tile_store<T, G::D, CH>(dst + base * G::D, rows * G::D, tile);
    __syncthreads();                      // the next tile overwrites the staging buffer
    carry = combine<G, T, LEFT>(carry, total);
  }
}

// ------------------------------------------------------------------------------------------------
// The same scan with the TIME AXIS split over CTAs, for few long sequences ((B = 1, L = 1e6) ran on ONE SM with
// cumprod_kernel).  Reduce-then-scan in three launches, deterministic, no flags:
//   1. every tile (kScanThreads x CH rows) multiplies its rows together              -> aggregate of the tile
//   2. one CTA per sequence scans the tile aggregates (exclusive)                     -> prefix entering each tile
//   3. every tile scans its rows again starting from that prefix and stores them
// The rows are read twice, the second time mostly from L2 (a 28 MB sequence stays resident in the H100's 50 MB L2).  A
// single pass with decoupled look-back was slower: with only ~1000 tiles, all resident at once, every tile had to walk back over hundreds of unfinished predecessors — the look-back chain, not the bandwidth, set the
// time.  Workspace (caller-owned, no initialisation needed): aggregates (tiles x 8) and prefixes (tiles x 8).
// ------------------------------------------------------------------------------------------------
// tile aggregates / prefixes live in 8-number slots (the widest group layout) of a 16-byte aligned workspace: moved as
// 16-byte vectors (2 for float, 4 for double) instead of 8 scalars
template <typename T> __device__ __forceinline__ Elem<T> load_agg(const T* __restrict__ p) {
  constexpr int EV = 16 / (int)sizeof(T);
  __align__(16) T v[8];
#pragma unroll
  for (int i = 0; i < 8 / EV; ++i) reinterpret_cast<float4*>(v)[i] = reinterpret_cast<const float4*>(p)[i];
  return load_elem<Sim3g, T>(v);
}
template <typename T> __device__ __forceinline__ void store_agg(T* __restrict__ p, const Elem<T>& e) {
  constexpr int EV = 16 / (int)sizeof(T);
  __align__(16) T v[8];
  store_elem<Sim3g, T>(v, e);
#pragma unroll
  for (int i = 0; i < 8 / EV; ++i) reinterpret_cast<float4*>(p)[i] = reinterpret_cast<const float4*>(v)[i];
}

template <class G, typename T, bool LEFT, int CH>
__global__ void __launch_bounds__(kScanThreads) cumprod_tile_reduce_kernel(const T* __restrict__ in, long long L, int nt,
                                                                            T* __restrict__ agg) {
  using TS = TileSmem<T, G::D, CH>;
  __shared__ T sh[(kScanThreads / 32) * 8];
  __shared__ __align__(16) T tile[TS::WORDS];
  const long long gid = blockIdx.x;
  const long long b = gid / nt;
  const int t = (int)(gid - b * nt);
  constexpr long long TILE = (long long)kScanThreads * CH;
  const long long row0 = (long long)t * TILE;
  const int rows = (int)(L - row0 < TILE ? L - row0 : TILE);
  tile_load<T, G::D, CH>(in + (b * L + row0) * G::D, rows * G::D, tile);
  const int first = threadIdx.x * CH;
  const T* mine = tile + threadIdx.x * TS::STRIDE;
  Elem<T> run = elem_identity<T>();
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (first + c < rows) {
      T row[G::D];
#pragma unroll
      for (int k = 0; k < G::D; ++k) row[k] = mine[c * G::D + k];
      run = combine<G, T, LEFT>(run, load_elem<G, T>(row));
    }
  }
  Elem<T> total;
  block_exclusive<G, T, LEFT>(run, total, sh);
  if (threadIdx.x == 0) store_agg(agg + gid * 8, total);
}
// exclusive scan of the nt tile aggregates of one sequence: one CTA of kPrefixThreads per sequence, one aggregate per
// thread and round (carry across rounds), two levels of warp-shuffle scans (a 128-thread version needs 8 rounds of a block
// scan for the 977 tiles of L = 1e6).
constexpr int kPrefixThreads = 1024;
template <class G, typename T, bool LEFT>
__global__ void __launch_bounds__(kPrefixThreads) cumprod_tile_prefix_kernel(const T* __restrict__ agg, T* __restrict__ pre, int nt) {
  constexpr int NW = kPrefixThreads / 32;
  __shared__ T sh_tot[NW * 8];
  __shared__ T sh_pre[(NW + 1) * 8];
  const long long b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Elem<T> carry = elem_identity<T>();
  for (int base = 0; base < nt; base += kPrefixThreads) {
    const int t = base + threadIdx.x;
    Elem<T> inc = t < nt ? load_agg(agg + (b * nt + t) * 8) : elem_identity<T>();
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      Elem<T> up = elem_shfl_up(inc, o);
      if (lane >= o) inc = combine<G, T, LEFT>(up, inc);
    }
    Elem<T> excl = elem_shfl_up(inc, 1);
    if (lane == 0) excl = elem_identity<T>();
    if (lane == 31) store_elem<Sim3g, T>(sh_tot + warp * 8, inc);
    __syncthreads();
    if (warp == 0) {                                   // scan of the NW (= 32) warp totals by one warp
      Elem<T> w = load_elem<Sim3g, T>(sh_tot + lane * 8);
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        Elem<T> up = elem_shfl_up(w, o);
        if (lane >= o) w = combine<G, T, LEFT>(up, w);
      }
      Elem<T> wex = elem_shfl_up(w, 1);
      if (lane == 0) wex = elem_identity<T>();
      store_elem<Sim3g, T>(sh_pre + lane * 8, wex);
      if (lane == 31) store_elem<Sim3g, T>(sh_pre + NW * 8, w);
    }
    __syncthreads();
    const Elem<T> wpre = load_elem<Sim3g, T>(sh_pre + warp * 8);
    const Elem<T> total = load_elem<Sim3g, T>(sh_pre + NW * 8);
    if (t < nt) store_agg(pre + (b * nt + t) * 8, combine<G, T, LEFT>(carry, combine<G, T, LEFT>(wpre, excl)));
    carry = combine<G, T, LEFT>(carry, total);
    __syncthreads();                                   // sh_tot / sh_pre are rewritten by the next round
  }
}
template <class G, typename T, bool LEFT, int CH>
__global__ void __launch_bounds__(kScanThreads) cumprod_tile_apply_kernel(const T* __restrict__ in, T* __restrict__ out,
                                                                           long long L, int nt, const T* __restrict__ pre) {
  using TS = TileSmem<T, G::D, CH>;
  __shared__ T sh[(kScanThreads / 32) * 8];
  __shared__ __align__(16) T tile[TS::WORDS];
  const long long gid = blockIdx.x;
  const long long b = gid / nt;
  const int t = (int)(gid - b * nt);
  constexpr long long TILE = (long long)kScanThreads * CH;
  const long long row0 = (long long)t * TILE;
  const int rows = (int)(L - row0 < TILE ? L - row0 : TILE);
  const Elem<T> tile_pfx = load_agg(pre + gid * 8);
  tile_load<T, G::D, CH>(in + (b * L + row0) * G::D, rows * G::D, tile);
  const int first = threadIdx.x * CH;
  T* mine = tile + threadIdx.x * TS::STRIDE;
  Elem<T> loc[CH];
  Elem<T> run = elem_identity<T>();
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (first + c < rows) {
      T row[G::D];
#pragma unroll
      for (int k = 0; k < G::D; ++k) row[k] = mine[c * G::D + k];
      run = combine<G, T, LEFT>(run, load_elem<G, T>(row));
    }
    loc[c] = run;
  }
  Elem<T> total;
  const Elem<T> pre_thread = block_exclusive<G, T, LEFT>(run, total, sh);
  const Elem<T> pfx = combine<G, T, LEFT>(tile_pfx, pre_thread);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (first + c < rows) {
      T row[G::D];
      store_elem<G, T>(row, combine<G, T, LEFT>(pfx, loc[c]));
#pragma unroll
      for (int k = 0; k < G::D; ++k) mine[c * G::D + k] = row[k];      // own words only: no hazard with other threads
    }
  }
  tile_store<T, G::D, CH>(out + (b * L + row0) * G::D, rows * G::D, tile);
}

template <typename T> constexpr int scan_ch() { return sizeof(T) == 8 ? 4 : 8; }
static inline long long scan_tiles(long long L, int elem) { return (L + (long long)kScanThreads * (elem == 8 ? 4 : 8) - 1) / ((long long)kScanThreads * (elem == 8 ? 4 : 8)); }

template <class G, typename T>
int launch_cumprod(const T* in, T* out, long long B, long long L, int left, cudaStream_t s) {
  if (B <= 0 || L <= 0) return 0;
  constexpr int CH = scan_ch<T>();
  if (left) cumprod_kernel<G, T, true, CH><<<(unsigned)B, kScanThreads, 0, s>>>(in, out, L);
  else cumprod_kernel<G, T, false, CH><<<(unsigned)B, kScanThreads, 0, s>>>(in, out, L);
  return (int)cudaGetLastError();
}
// time-split variant; ws: b200_scan_workspace_bytes(B, L, sizeof(T)) bytes (no initialisation needed)
template <class G, typename T>
int launch_cumprod_lb(const T* in, T* out, long long B, long long L, int left, void* ws, cudaStream_t s) {
  if (B <= 0 || L <= 0) return 0;
  constexpr int CH = scan_ch<T>();
  const long long nt = scan_tiles(L, (int)sizeof(T)), tiles = B * nt;
  T* agg = reinterpret_cast<T*>(ws);
  T* pre = agg + tiles * 8;
  if (left) {
    cumprod_tile_reduce_kernel<G, T, true, CH><<<(unsigned)tiles, kScanThreads, 0, s>>>(in, L, (int)nt, agg);
    cumprod_tile_prefix_kernel<G, T, true><<<(unsigned)B, kPrefixThreads, 0, s>>>(agg, pre, (int)nt);
    cumprod_tile_apply_kernel<G, T, true, CH><<<(unsigned)tiles, kScanThreads, 0, s>>>(in, out, L, (int)nt, pre);
  } else {
    cumprod_tile_reduce_kernel<G, T, false, CH><<<(unsigned)tiles, kScanThreads, 0, s>>>(in, L, (int)nt, agg);
    cumprod_tile_prefix_kernel<G, T, false><<<(unsigned)B, kPrefixThreads, 0, s>>>(agg, pre, (int)nt);
    cumprod_tile_apply_kernel<G, T, false, CH><<<(unsigned)tiles, kScanThreads, 0, s>>>(in, out, L, (int)nt, pre);
  }
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// IMU preintegration (imu_preintegrator.py:314-384), one kernel:
//   dr_k = Exp(gyro_k dt_k);  R_k = dr_1 ... dr_k (R_0 = I)                       -> Dr (= incre_r[:,1:]), w = dr
//   a_k  = acc_k - (init_rot R_k)^-1 g      (or acc_k - rot_k^-1 g when `rot` is given)   [uses R_k = after sample k]
//   dv_k = R_{k-1} a_k dt_k;   Dv_k = sum_{j<=k} dv_j                                      [rotates with R before k]
//   dp_k = Dv_{k-1} dt_k + R_{k-1} a_k dt_k^2 / 2;  Dp_k = sum dp_j;   Dt_k = sum dt_j
// The (v, p, t) recurrences form an associative scan with combine((v1,p1,t1),(v2,p2,t2)) = (v1+v2, p1+p2+v1 t2, t1+t2).
// ------------------------------------------------------------------------------------------------
template <typename T> struct Vpt { V3<T> v, p; T t; };
template <typename T> __device__ __forceinline__ Vpt<T> vpt_identity() {
  Vpt<T> e; e.v = mk(T(0), T(0), T(0)); e.p = e.v; e.t = T(0); return e;
}
template <typename T> __device__ __forceinline__ Vpt<T> vpt_combine(const Vpt<T>& a, const Vpt<T>& b) {
  Vpt<T> r; r.v = a.v + b.v; r.p = a.p + b.p + b.t * a.v; r.t = a.t + b.t; return r;
}
template <typename T> __device__ __forceinline__ Vpt<T> vpt_shfl_up(const Vpt<T>& e, int o) {
  Vpt<T> r;
  r.v = mk(shfl_up(e.v.x, o), shfl_up(e.v.y, o), shfl_up(e.v.z, o));
  r.p = mk(shfl_up(e.p.x, o), shfl_up(e.p.y, o), shfl_up(e.p.z, o));
  r.t = shfl_up(e.t, o);
  return r;
}
template <typename T>
__device__ __forceinline__ Vpt<T> vpt_block_exclusive(const Vpt<T>& mine, Vpt<T>& total, T* sh /* [warps][8] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kScanThreads / 32;
  Vpt<T> inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Vpt<T> up = vpt_shfl_up(inc, o);
    if (lane >= o) inc = vpt_combine(up, inc);
  }
  Vpt<T> excl = vpt_shfl_up(inc, 1);
  if (lane == 0) excl = vpt_identity<T>();
  if (lane == 31) { st3(sh + warp * 8, inc.v); st3(sh + warp * 8 + 3, inc.p); sh[warp * 8 + 6] = inc.t; }
  __syncthreads();
  Vpt<T> wpre = vpt_identity<T>(), tot = vpt_identity<T>();
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    Vpt<T> e; e.v = ld3(sh + w * 8); e.p = ld3(sh + w * 8 + 3); e.t = sh[w * 8 + 6];
    if (w < warp) wpre = vpt_combine(wpre, e);
    tot = vpt_combine(tot, e);
  }
  __syncthreads();
  total = tot;
  return vpt_combine(wpre, excl);
}

// Exp of one gyro increment.  |gyro dt| is ~1e-3 rad for any real IMU, far inside the window where the coefficient series
// are exact to rounding (theta^2 < small2: remainder < 1e-20), so when every active lane of the warp is inside it the
// double-precision sincos — the bulk of the general path's instructions — is not
// executed at all; any lane outside takes the general path for the whole warp (same values as so3_exp(phi, rot_coef(phi))
// to rounding).
template <typename T> __device__ __forceinline__ Q4<T> so3_exp_imu(const V3<T>& phi) {
  const T x = dot(phi, phi);
  if (__all_sync(__activemask(), x < num<T>::small2)) {
    const T imag = T(0.5) + x * (T(-1.0 / 48) + x * (T(1.0 / 3840) + x * (T(-1.0 / 645120) + x * T(1.0 / 185794560))));
    const T ch = T(1) + x * (T(-1.0 / 8) + x * (T(1.0 / 384) + x * (T(-1.0 / 46080) + x * (T(1.0 / 10321920) +
                 x * (T(-1.0 / 3715891200.0) + x * T(1.0 / 1961990553600.0))))));
    Q4<T> q; q.v = imag * phi; q.w = ch; return q;
  }
  return so3_exp(phi, rot_coef(phi));
}

template <typename T, int CH>
__global__ void __launch_bounds__(kScanThreads) imu_integrate_kernel(
    const T* __restrict__ dt, const T* __restrict__ gyro, const T* __restrict__ acc, const T* __restrict__ rot,
    const T* __restrict__ init_rot, long long init_stride, T gx, T gy, T gz, T* __restrict__ a_out, T* __restrict__ Dp,
    T* __restrict__ Dv, T* __restrict__ Dr, T* __restrict__ Dt, T* __restrict__ w_out, const T* __restrict__ init_pos,
    const T* __restrict__ init_vel, long long pv_stride, T* __restrict__ rot_o, T* __restrict__ vel_o,
    T* __restrict__ pos_o, long long F) {
  __shared__ T sh[(kScanThreads / 32) * 8];
  const long long b = blockIdx.x;
  dt += b * F; gyro += b * F * 3; acc += b * F * 3;
  if (rot) rot += b * F * 4;
  // every output is optional: the integrate outputs (imu_preintegrator.py:383-384) and/or the predicted
  // states rot = R0 Dr, vel = v0 + R0 Dv, pos = p0 + R0 Dp + v0 Dt (imu_preintegrator.py:422-426)
  if (a_out) { a_out += b * F * 3; Dp += b * F * 3; Dv += b * F * 3; Dr += b * F * 4; Dt += b * F; w_out += b * F * 4; }
  if (rot_o) { rot_o += b * F * 4; vel_o += b * F * 3; pos_o += b * F * 3; }
  const V3<T> grav = mk(gx, gy, gz);
  Elem<T> R0 = elem_identity<T>();
  if (init_rot) R0.q = ldq(init_rot + b * init_stride);
  V3<T> p0 = mk(T(0), T(0), T(0)), v0 = p0;
  if (init_pos) p0 = ld3(init_pos + b * pv_stride);
  if (init_vel) v0 = ld3(init_vel + b * pv_stride);
  Elem<T> carryR = elem_identity<T>();
  Vpt<T> carry = vpt_identity<T>();
  constexpr long long TILE = (long long)kScanThreads * CH;
  for (long long base = 0; base < F; base += TILE) {
    const long long first = base + (long long)threadIdx.x * CH;
    // ---- rotation part: dr_k and the thread-local running product
    Elem<T> loc[CH];
    T dts[CH];
    Elem<T> run = elem_identity<T>();
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      dts[c] = T(0);
      if (first + c < F) {
        const long long k = first + c;
        dts[c] = dt[k];
        const V3<T> phi = dts[c] * mk(gyro[k * 3], gyro[k * 3 + 1], gyro[k * 3 + 2]);
        Elem<T> dr = elem_identity<T>();
        dr.q = so3_exp_imu(phi);
        if (a_out) stq(w_out + k * 4, dr.q);        // written here so that the increments need not stay in registers
        run = g_mul<SO3g, T>(run, dr);
      }
      loc[c] = run;
    }
    Elem<T> totR;
    const Elem<T> preR = g_mul<SO3g, T>(carryR, block_exclusive<SO3g, T, false>(run, totR, sh));
    // ---- translation part: a_k, dv_k, dp_k, thread-local (v, p, t) scan
    Vpt<T> vloc[CH];
    Vpt<T> vrun = vpt_identity<T>();
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (first + c < F) {
        const long long k = first + c;
        const Elem<T> Rafter = g_mul<SO3g, T>(preR, loc[c]);                            // R_k
        const Elem<T> Rbefore = c == 0 ? preR : g_mul<SO3g, T>(preR, loc[c - 1]);       // R_{k-1}
        Q4<T> qg;                                                                        // rotation used for gravity
        if (rot) qg = ldq(rot + k * 4);
        else qg = qmul(R0.q, Rafter.q);
        const V3<T> ak = mk(acc[k * 3], acc[k * 3 + 1], acc[k * 3 + 2]) - qrot_t(qg, grav);
        const V3<T> Ra = qrot(Rbefore.q, ak);
        Vpt<T> e; e.v = dts[c] * Ra; e.p = (T(0.5) * dts[c] * dts[c]) * Ra; e.t = dts[c];
        vrun = vpt_combine(vrun, e);
        if (a_out) {
          st3(a_out + k * 3, ak);
          stq(Dr + k * 4, Rafter.q);
        }
        if (rot_o) stq(rot_o + k * 4, qmul(R0.q, Rafter.q));
      }
      vloc[c] = vrun;
    }
    Vpt<T> totV;
    const Vpt<T> preV = vpt_combine(carry, vpt_block_exclusive(vrun, totV, sh));
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (first + c < F) {
        const long long k = first + c;
        const Vpt<T> y = vpt_combine(preV, vloc[c]);
        if (a_out) {
          st3(Dv + k * 3, y.v);
          st3(Dp + k * 3, y.p);
          Dt[k] = y.t;
        }
        if (rot_o) {
          st3(vel_o + k * 3, v0 + qrot(R0.q, y.v));
          st3(pos_o + k * 3, p0 + qrot(R0.q, y.p) + y.t * v0);
        }
      }
    }
    carryR = g_mul<SO3g, T>(carryR, totR);
    carry = vpt_combine(carry, totV);
  }
}

// ------------------------------------------------------------------------------------------------
// IMU covariance propagation (imu_preintegrator.py:428-465) without materialising (B, F+1, 9, 9):
//   cov = sum_{k=0..F} L_k B_k L_k^T,  L_k = A_k A_{k+1} ... A_{F-1},  B_0 = init_cov, B_{j+1} = N_j (noise of sample j)
// exactly the reference's `cumprod(A.flip).flip` ordering, with
//   A_j = [[Rk^T,0,0],[M1, I, 0],[M1 dt/2, dt I, I]],  M1 = -Rij a^ dt;   N_j = (Bg Cg Bg^T + Ba Ca Ba^T)/dt,
//   Bg = [Jr(dr) dt; 0; 0],  Ba = [0; Rij dt; Rij dt^2/2].
// Products of such A keep the shape  L = [[X,0,0],[Y,I,0],[Z,tau I,I]]  (X,Y,Z 3x3, tau = sum of dt), so a 9x9 matrix
// is 28 numbers and one step A_j L costs two 3x3 products; the noise term needs only the first block column:
//   L Bg = [X;Y;Z] Jr dt,   L Ba = [0; R dt; (tau + dt/2) R dt]
//   L N L^T = [X;Y;Z] Q [X;Y;Z]^T + [[0,0,0],[0,K,sK],[0,sK,s^2 K]],  Q = Jr diag(cg dt) Jr^T, K = R diag(ca dt) R^T, s = tau+dt/2.
// Everything lives in registers (the first version kept dense 9x9 matrices in local memory: 17.7 ms for 1e3 x 1e4
// samples; this form: see DESIGN.md §3.2).  Three passes over chunks of the time axis:
//   1. P_c = product of the A_j of chunk c                        (one thread per (trajectory, chunk))
//   2. S_c = P_c S_{c+1}: suffix products over chunks              (one thread per trajectory, NC steps)
//   3. T_c = sum_{j in c} L_{j+1} N_j L_{j+1}^T walking the chunk backwards from L = S_{c+1} (symmetric, 45 numbers);
//      cov = sum_c T_c + L_0 init L_0^T                            (81 threads per trajectory)
// ------------------------------------------------------------------------------------------------
// CovL, covl_* and quat_matrix: imu_cov_math.cuh (host + device, checked on the CPU by tests/test_hostmath.py)
constexpr int kCovThreads = 64;

template <typename T>
__global__ void __launch_bounds__(kCovThreads) imu_cov_chunk_prod_kernel(const T* Rk, const T* Rij, const T* a, const T* dt, T* P,
                                                                        long long F, long long chunk, long long NC,
                                                                        long long total) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= total) return;
  const long long b = id / NC, c = id % NC;
  Rk += b * F * 4; Rij += b * F * 4; a += b * F * 3; dt += b * F;
  CovL<T> L;
  covl_identity(L);
  const long long lo = c * chunk, hi = (lo + chunk < F) ? lo + chunk : F;
  // the loads of step j-1 are issued before the arithmetic of step j (each thread walks its own stream: the only
  // latency hiding inside a thread is this one-step software pipeline)
  Q4<T> qk = ldq(Rk + (hi - 1) * 4), qi = ldq(Rij + (hi - 1) * 4);
  V3<T> av = ld3(a + (hi - 1) * 3);
  T d = dt[hi - 1];
  for (long long j = hi - 1; j >= lo; --j) {
    const long long jn = j > lo ? j - 1 : j;
    const Q4<T> qk_n = ldq(Rk + jn * 4), qi_n = ldq(Rij + jn * 4);
    const V3<T> av_n = ld3(a + jn * 3);
    const T d_n = dt[jn];
    T R[3][3];
    quat_matrix(qi, R);
    covl_apply_A(L, qk, R, av, d);
    qk = qk_n; qi = qi_n; av = av_n; d = d_n;
  }
  covl_store(L, P + id * kCovL);
}
// S[c] = P_c P_{c+1} ... P_{NC-1};  S[NC] = I     (S: (B, NC+1, 28)).  One warp per trajectory: tiles of 32 chunks from
// the right, order-preserving suffix scan by shuffles (the product is associative, not commutative), carry = S of the
// tile to the right.
template <typename T> __device__ __forceinline__ CovL<T> covl_shfl_down(const CovL<T>& v, int o) {
  CovL<T> r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      r.X[i][j] = __shfl_down_sync(0xffffffffu, v.X[i][j], o);
      r.Y[i][j] = __shfl_down_sync(0xffffffffu, v.Y[i][j], o);
      r.Z[i][j] = __shfl_down_sync(0xffffffffu, v.Z[i][j], o);
    }
  r.tau = __shfl_down_sync(0xffffffffu, v.tau, o);
  return r;
}
template <typename T> __device__ __forceinline__ CovL<T> covl_bcast0(const CovL<T>& v) {
  CovL<T> r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      r.X[i][j] = __shfl_sync(0xffffffffu, v.X[i][j], 0);
      r.Y[i][j] = __shfl_sync(0xffffffffu, v.Y[i][j], 0);
      r.Z[i][j] = __shfl_sync(0xffffffffu, v.Z[i][j], 0);
    }
  r.tau = __shfl_sync(0xffffffffu, v.tau, 0);
  return r;
}
template <typename T> __global__ void __launch_bounds__(128) imu_cov_suffix_kernel(const T* P, T* S, long long NC, long long B) {
  const long long b = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;                                    // whole warps leave together
  const int lane = threadIdx.x & 31;
  CovL<T> carry, v, o, nx;
  covl_identity(carry);
  if (lane == 0) covl_store(carry, S + (b * (NC + 1) + NC) * kCovL);
  for (long long base = ((NC - 1) / 32) * 32; base >= 0; base -= 32) {
    const long long c = base + lane;
    if (c < NC) covl_load(v, P + (b * NC + c) * kCovL); else covl_identity(v);
#pragma unroll 1
    for (int off = 1; off < 32; off <<= 1) {
      o = covl_shfl_down(v, off);
      if (lane + off < 32) { covl_mul(v, o, nx); v = nx; }
    }
    covl_mul(v, carry, nx);
    if (c < NC) covl_store(nx, S + (b * (NC + 1) + c) * kCovL);
    carry = covl_bcast0(nx);
  }
}
template <typename T>
__global__ void __launch_bounds__(kCovThreads) imu_cov_accum_kernel(const T* Rk, const T* Rij, const T* a, const T* dt,
                                                                   const T* gcov, const T* acov, long long cov_stride_b,
                                                                   long long cov_stride_f, const T* S, T* Tc, long long F,
                                                                   long long chunk, long long NC, long long total) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= total) return;
  const long long b = id / NC, c = id % NC;
  Rk += b * F * 4; Rij += b * F * 4; a += b * F * 3; dt += b * F;
  gcov += b * cov_stride_b; acov += b * cov_stride_b;
  CovL<T> L;
  covl_load(L, S + (b * (NC + 1) + c + 1) * kCovL);
  T Tm[kCovT];
#pragma unroll
  for (int i = 0; i < kCovT; ++i) Tm[i] = T(0);
  const long long lo = c * chunk, hi = (lo + chunk < F) ? lo + chunk : F;
  for (long long j = hi - 1; j >= lo; --j) {
    const Q4<T> qk = ldq(Rk + j * 4);
    T R[3][3];
    quat_matrix(ldq(Rij + j * 4), R);
    const T d = dt[j];
    covl_accum_noise(L, qk, R, d, gcov + j * cov_stride_f, acov + j * cov_stride_f, Tm);   // uses L_{j+1}
    covl_apply_A(L, qk, R, ld3(a + j * 3), d);                                              // L_j = A_j L_{j+1}
  }
#pragma unroll
  for (int i = 0; i < kCovT; ++i) Tc[id * kCovT + i] = Tm[i];
}
// cov[b] = sum_c T_c + S_0 init_cov S_0^T: one CTA of 81 threads per trajectory, thread e owns entry (e/9, e%9)
template <typename T>
__global__ void __launch_bounds__(96) imu_cov_finish_kernel(const T* S, const T* Tc, const T* init_cov, long long init_stride,
                                                           T* cov, long long NC) {
  const long long b = blockIdx.x;
  __shared__ T L0[81], C0[81], tmp[81];
  const int e = threadIdx.x;
  if (e < 81) {
    const T* s = S + b * (NC + 1) * kCovL;
    const int r = e / 9, c = e % 9, br = r / 3, bc = c / 3, rr = r % 3, cc = c % 3;
    T v = T(0);
    if (bc == 0) v = s[br * 9 + rr * 3 + cc];                         // X, Y, Z
    else if (br == bc) v = rr == cc ? T(1) : T(0);                    // identity blocks
    else if (br == 2 && bc == 1) v = rr == cc ? s[27] : T(0);         // tau I
    L0[e] = v;
    C0[e] = init_cov[b * init_stride + e];
  }
  __syncthreads();
  if (e < 81) {
    const int i = e / 9, jj = e % 9;
    T v = T(0);
    for (int k = 0; k < 9; ++k) v += L0[i * 9 + k] * C0[k * 9 + jj];
    tmp[e] = v;
  }
  __syncthreads();
  if (e < 81) {
    const int i = e / 9, jj = e % 9;
    T v = T(0);
    for (int k = 0; k < 9; ++k) v += tmp[i * 9 + k] * L0[jj * 9 + k];
    const int q = i <= jj ? tri9(i, jj) : tri9(jj, i);
    const T* t = Tc + b * NC * kCovT + q;
    for (long long c = 0; c < NC; ++c) v += t[c * kCovT];
    cov[b * 81 + e] = v;
  }
}

}  // namespace b200pose

using namespace b200pose;

#define SCAN_ABI(GRP, G)                                                                                               \
  B200_EXPORT int b200_##GRP##_cumprod_lb_f32(const float* in, float* out, long long B, long long L, int left, void* ws, void* s) { \
    return launch_cumprod_lb<G, float>(in, out, B, L, left, ws, (cudaStream_t)s);                                      \
  }                                                                                                                    \
  B200_EXPORT int b200_##GRP##_cumprod_lb_f64(const double* in, double* out, long long B, long long L, int left, void* ws, void* s) { \
    return launch_cumprod_lb<G, double>(in, out, B, L, left, ws, (cudaStream_t)s);                                     \
  }                                                                                                                    \
  B200_EXPORT int b200_##GRP##_cumprod_f32(const float* in, float* out, long long B, long long L, int left, void* s) { \
    return launch_cumprod<G, float>(in, out, B, L, left, (cudaStream_t)s);                                             \
  }                                                                                                                    \
  B200_EXPORT int b200_##GRP##_cumprod_f64(const double* in, double* out, long long B, long long L, int left, void* s) { \
    return launch_cumprod<G, double>(in, out, B, L, left, (cudaStream_t)s);                                            \
  }
SCAN_ABI(SO3, SO3g)
SCAN_ABI(SE3, SE3g)
SCAN_ABI(RxSO3, RxSO3g)
SCAN_ABI(Sim3, Sim3g)

// ------------------------------------------------------------------------------------------------
// Predict-only integration with the samples STAGED through shared memory by 1-D TMA bulk copies (tma.cuh).
// imu_integrate_kernel needs ~124 registers -> 16 warps per SM, and it waits on the tile's own loads plus LSU back-pressure
// from 3-word strided stores — the next tile cannot start loading before this one has been scanned.  Here thread 0 queues the bulk loads of tile i+2 while the CTA scans tile i
// out of shared memory, and the results leave through one bulk store per output array, so the LSU only sees shared memory.
// Same arithmetic, same order of operations as imu_integrate_kernel (results are bit-identical).
// Preconditions (checked by the launcher, which otherwise uses imu_integrate_kernel): no per-sample `rot`, no integrate
// outputs, 16-byte aligned arrays and F * sizeof(T) a multiple of 16.
// ------------------------------------------------------------------------------------------------
template <typename T, int CH> struct ImuTma {
  static constexpr int TILE = kScanThreads * CH;
  static constexpr int S = 2;                                   // input stages
  static constexpr int IN_WORDS = TILE * 7, OUT_WORDS = TILE * 10;
  static constexpr int BYTES = (S * IN_WORDS + OUT_WORDS) * (int)sizeof(T) + 8 * S;
};
template <typename T, int CH>
__global__ void __launch_bounds__(kScanThreads) imu_predict_tma_kernel(
    const T* __restrict__ dt, const T* __restrict__ gyro, const T* __restrict__ acc, const T* __restrict__ init_rot,
    long long init_stride, T gx, T gy, T gz, const T* __restrict__ init_pos, const T* __restrict__ init_vel,
    long long pv_stride, T* __restrict__ rot_o, T* __restrict__ vel_o, T* __restrict__ pos_o, long long F) {
  using L = ImuTma<T, CH>;
  constexpr int TILE = L::TILE, S = L::S;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ T sh[(kScanThreads / 32) * 8];
  T* s_in = reinterpret_cast<T*>(smem_raw);
  T* s_out = s_in + S * L::IN_WORDS;
  uint64_t* full = reinterpret_cast<uint64_t*>(s_out + L::OUT_WORDS);
  const long long b = blockIdx.x;
  dt += b * F; gyro += b * F * 3; acc += b * F * 3;
  rot_o += b * F * 4; vel_o += b * F * 3; pos_o += b * F * 3;
  const int tid = threadIdx.x;
  if (tid == 0) {
#pragma unroll
    for (int q = 0; q < S; ++q) mbar_init(&full[q], 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int ntiles = (int)((F + TILE - 1) / TILE);
  auto issue_load = [&](int t, int q) {                         // thread 0 only
    const long long base = (long long)t * TILE;
    const uint32_t cnt = (uint32_t)(F - base < TILE ? F - base : TILE);
    T* dst = s_in + q * L::IN_WORDS;
    mbar_expect_tx(&full[q], cnt * 7u * (uint32_t)sizeof(T));
    bulk_g2s(dst, dt + base, cnt * (uint32_t)sizeof(T), &full[q]);
    bulk_g2s(dst + TILE, gyro + base * 3, cnt * 3u * (uint32_t)sizeof(T), &full[q]);
    bulk_g2s(dst + 4 * TILE, acc + base * 3, cnt * 3u * (uint32_t)sizeof(T), &full[q]);
  };
  if (tid == 0)
    for (int t = 0; t < ntiles && t < S; ++t) issue_load(t, t);

  const V3<T> grav = mk(gx, gy, gz);
  Elem<T> R0 = elem_identity<T>();
  if (init_rot) R0.q = ldq(init_rot + b * init_stride);
  V3<T> p0 = mk(T(0), T(0), T(0)), v0 = p0;
  if (init_pos) p0 = ld3(init_pos + b * pv_stride);
  if (init_vel) v0 = ld3(init_vel + b * pv_stride);
  Elem<T> carryR = elem_identity<T>();
  Vpt<T> carry = vpt_identity<T>();
  T* o_rot = s_out;
  T* o_vel = s_out + 4 * TILE;
  T* o_pos = s_out + 7 * TILE;
  int q = 0;
  uint32_t parity = 0;
  for (int i = 0; i < ntiles; ++i) {
    const long long base = (long long)i * TILE;
    const int cnt = (int)(F - base < TILE ? F - base : TILE);
    const T* i_dt = s_in + q * L::IN_WORDS;
    const T* i_gy = i_dt + TILE;
    const T* i_ac = i_dt + 4 * TILE;
    const int first = tid * CH;
    mbar_wait(&full[q], parity);
    if (tid == 0) bulk_wait_read<0>();     // the store of tile i-1 has left s_out (ordered for the CTA by the scan's barrier)
    Elem<T> loc[CH];
    T dts[CH];
    Elem<T> run = elem_identity<T>();
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      dts[c] = T(0);
      if (first + c < cnt) {
        const int k = first + c;
        dts[c] = i_dt[k];
        const V3<T> phi = dts[c] * mk(i_gy[k * 3], i_gy[k * 3 + 1], i_gy[k * 3 + 2]);
        Elem<T> dr = elem_identity<T>();
        dr.q = so3_exp_imu(phi);
        run = g_mul<SO3g, T>(run, dr);
      }
      loc[c] = run;
    }
    Elem<T> totR;
    const Elem<T> preR = g_mul<SO3g, T>(carryR, block_exclusive<SO3g, T, false>(run, totR, sh));
    Vpt<T> vloc[CH];
    Vpt<T> vrun = vpt_identity<T>();
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (first + c < cnt) {
        const int k = first + c;
        const Elem<T> Rafter = g_mul<SO3g, T>(preR, loc[c]);
        const Elem<T> Rbefore = c == 0 ? preR : g_mul<SO3g, T>(preR, loc[c - 1]);
        const Q4<T> qg = qmul(R0.q, Rafter.q);
        const V3<T> ak = mk(i_ac[k * 3], i_ac[k * 3 + 1], i_ac[k * 3 + 2]) - qrot_t(qg, grav);
        const V3<T> Ra = qrot(Rbefore.q, ak);
        Vpt<T> e; e.v = dts[c] * Ra; e.p = (T(0.5) * dts[c] * dts[c]) * Ra; e.t = dts[c];
        vrun = vpt_combine(vrun, e);
        stq(o_rot + k * 4, qmul(R0.q, Rafter.q));
      }
      vloc[c] = vrun;
    }
    Vpt<T> totV;
    const Vpt<T> preV = vpt_combine(carry, vpt_block_exclusive(vrun, totV, sh));
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (first + c < cnt) {
        const int k = first + c;
        const Vpt<T> y = vpt_combine(preV, vloc[c]);
        st3(o_vel + k * 3, v0 + qrot(R0.q, y.v));
        st3(o_pos + k * 3, p0 + qrot(R0.q, y.p) + y.t * v0);
      }
    }
    carryR = g_mul<SO3g, T>(carryR, totR);
    carry = vpt_combine(carry, totV);
    fence_async_smem();
    __syncthreads();                       // s_out complete, stage q read by everyone
    if (tid == 0) {
      bulk_s2g(rot_o + base * 4, o_rot, (uint32_t)cnt * 4u * (uint32_t)sizeof(T));
      bulk_s2g(vel_o + base * 3, o_vel, (uint32_t)cnt * 3u * (uint32_t)sizeof(T));
      bulk_s2g(pos_o + base * 3, o_pos, (uint32_t)cnt * 3u * (uint32_t)sizeof(T));
      bulk_commit();
      if (i + S < ntiles) issue_load(i + S, q);
    }
    if (++q == S) { q = 0; parity ^= 1; }
  }
  if (tid == 0) bulk_wait_all();
}
// opt-in for > 48 KB of dynamic shared memory, once per device and instantiation
constexpr int kMaxDevices = 64;
template <typename T, int CH> static int imu_tma_prepare() {
  static bool done[kMaxDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) return (int)cudaErrorInvalidDevice;
  if (done[dev]) return 0;
  cudaError_t e = cudaFuncSetAttribute(imu_predict_tma_kernel<T, CH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       ImuTma<T, CH>::BYTES);
  if (e == cudaSuccess) done[dev] = true;
  return (int)e;
}
template <typename T, int CH>
static int imu_tma_launch(const T* dt, const T* gyro, const T* acc, const T* init_rot, long long init_stride, const T* g,
                          const T* init_pos, const T* init_vel, long long pv_stride, T* rot_out, T* vel_out, T* pos_out,
                          long long B, long long F, cudaStream_t s) {
  int rc = imu_tma_prepare<T, CH>();
  if (rc) return rc;
  imu_predict_tma_kernel<T, CH><<<(unsigned)B, kScanThreads, ImuTma<T, CH>::BYTES, s>>>(
      dt, gyro, acc, init_rot, init_stride, g[0], g[1], g[2], init_pos, init_vel, pv_stride, rot_out, vel_out, pos_out, F);
  return (int)cudaGetLastError();
}

// Samples per thread (CH) trades scan overhead (amortised over CH) against coalescing (a thread's CH consecutive
// samples make every warp access CH-strided).  tools/ab_imu.py compares the choices at 1e3 x 1e4 samples;
// B200POSE_IMU_CH overrides for A/B runs.
template <typename T, int CH>
static void imu_launch(const T* dt, const T* gyro, const T* acc, const T* rot, const T* init_rot, long long init_stride,
                       const T* g, T* a, T* Dp, T* Dv, T* Dr, T* Dt, T* w, const T* init_pos, const T* init_vel,
                       long long pv_stride, T* rot_out, T* vel_out, T* pos_out, long long B, long long F, cudaStream_t s) {
  imu_integrate_kernel<T, CH><<<(unsigned)B, kScanThreads, 0, s>>>(dt, gyro, acc, rot, init_rot, init_stride, g[0], g[1], g[2],
                                                                   a, Dp, Dv, Dr, Dt, w, init_pos, init_vel, pv_stride,
                                                                   rot_out, vel_out, pos_out, F);
}
// B200POSE_IMU_TMA / b200_imu_tma_mode: 1 (default) predict-only calls take imu_predict_tma_kernel when they can, 0 never
static int g_imu_tma = -1;
static int imu_tma_mode() {
  if (g_imu_tma < 0) {
    const char* v = getenv("B200POSE_IMU_TMA");
    g_imu_tma = v && *v ? atoi(v) : 1;
  }
  return g_imu_tma;
}
B200_EXPORT int b200_imu_tma_mode(int mode) {
  const int prev = imu_tma_mode();
  if (mode >= 0) g_imu_tma = mode;
  return prev;
}
#define IMU_ABI(SFX, CT, CH_PREDICT, CH_FULL)                                                                          \
  B200_EXPORT int b200_imu_integrate_##SFX(const CT* dt, const CT* gyro, const CT* acc, const CT* rot,                 \
                                           const CT* init_rot, long long init_stride, const CT* gravity3_host, CT* a,  \
                                           CT* Dp, CT* Dv, CT* Dr, CT* Dt, CT* w, const CT* init_pos,                  \
                                           const CT* init_vel, long long pv_stride, CT* rot_out, CT* vel_out,          \
                                           CT* pos_out, long long B, long long F, void* s) {                           \
    if (B <= 0 || F <= 0) return 0;                                                                                    \
    static const int ch_env = getenv("B200POSE_IMU_CH") ? atoi(getenv("B200POSE_IMU_CH")) : 0;                         \
    const int ch = ch_env ? ch_env : (a ? CH_FULL : CH_PREDICT);                                                       \
    const int tma_env = imu_tma_mode();                                                                                \
    const uintptr_t bits = (uintptr_t)dt | (uintptr_t)gyro | (uintptr_t)acc | (uintptr_t)rot_out | (uintptr_t)vel_out | \
                           (uintptr_t)pos_out | (uintptr_t)(F * (long long)sizeof(CT));                                \
    if (tma_env && !a && !rot && rot_out && (bits & 15) == 0) {                                                        \
      auto tgo = ch == 1 ? imu_tma_launch<CT, 1> : (ch == 4 ? imu_tma_launch<CT, 4> : imu_tma_launch<CT, 2>);          \
      return tgo(dt, gyro, acc, init_rot, init_stride, gravity3_host, init_pos, init_vel, pv_stride, rot_out, vel_out, \
                 pos_out, B, F, (cudaStream_t)s);                                                                      \
    }                                                                                                                  \
    auto go = ch == 1 ? imu_launch<CT, 1> : (ch == 4 ? imu_launch<CT, 4> : imu_launch<CT, 2>);                         \
    go(dt, gyro, acc, rot, init_rot, init_stride, gravity3_host, a, Dp, Dv, Dr, Dt, w, init_pos, init_vel, pv_stride,  \
       rot_out, vel_out, pos_out, B, F, (cudaStream_t)s);                                                              \
    return (int)cudaGetLastError();                                                                                    \
  }
IMU_ABI(f32, float, 2, 2)
IMU_ABI(f64, double, 2, 1)

// work: at least B * ((NC + 1) * 28 + NC * (28 + 45)) elements, NC = ceil(F / chunk)  (callers may keep the older,
// larger B * (3 NC + 1) * 81 sizing)
#define IMU_COV_ABI(SFX, CT)                                                                                           \
  B200_EXPORT int b200_imu_cov_##SFX(const CT* Rk, const CT* Rij, const CT* a, const CT* dt, const CT* gyro_cov,       \
                                     const CT* acc_cov, long long cov_stride_b, long long cov_stride_f,                \
                                     const CT* init_cov, long long init_stride, CT* cov, CT* work, long long chunk,    \
                                     long long B, long long F, void* stream) {                                         \
    if (B <= 0 || F <= 0 || chunk <= 0) return 0;                                                                      \
    const long long NC = (F + chunk - 1) / chunk, total = B * NC;                                                      \
    CT* P = work;                                                                                                      \
    CT* S = P + total * kCovL;                                                                                         \
    CT* Tc = S + B * (NC + 1) * kCovL;                                                                                 \
    cudaStream_t st = (cudaStream_t)stream;                                                                            \
    const unsigned gb = (unsigned)((total + kCovThreads - 1) / kCovThreads);                                           \
    imu_cov_chunk_prod_kernel<CT><<<gb, kCovThreads, 0, st>>>(Rk, Rij, a, dt, P, F, chunk, NC, total);                 \
    imu_cov_suffix_kernel<CT><<<(unsigned)((B + 3) / 4), 128, 0, st>>>(P, S, NC, B);                                       \
    imu_cov_accum_kernel<CT><<<gb, kCovThreads, 0, st>>>(Rk, Rij, a, dt, gyro_cov, acc_cov, cov_stride_b,              \
                                                         cov_stride_f, S, Tc, F, chunk, NC, total);                    \
    imu_cov_finish_kernel<CT><<<(unsigned)B, 96, 0, st>>>(S, Tc, init_cov, init_stride, cov, NC);                      \
    return (int)cudaGetLastError();                                                                                    \
  }
IMU_COV_ABI(f32, float)
IMU_COV_ABI(f64, double)

// bytes of the workspace of b200_<G>_cumprod_lb_<T>
B200_EXPORT long long b200_scan_workspace_bytes(long long B, long long L, long long elem_size) {
  const long long tiles = B * b200pose::scan_tiles(L, (int)elem_size);
  return 2 * tiles * 8 * elem_size;
}
