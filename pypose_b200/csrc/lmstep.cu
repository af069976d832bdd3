// lmstep.cu — one Levenberg-Marquardt trial per host call, decided on the device (C-ABI: include/b200pose.h, section LM).
//
// Round 1 drove every trial from Python: three launches, a gather kernel, a blocking read, the damping strategy in
// Python, then the parameter copy — 125 us per step for ~35 us of kernels (VERDICT r1 "What's weak", DESIGN.md §3.3).
// Here ONE C call enqueues the whole trial and the control flow of optimizer.py:659-680 runs on the device:
//
//   reprojection (block-diagonal H):  K1 per camera: linearise + accumulate + damped 6x6 solve + retraction + trial loss over
//                                        the same rows; its last CTA takes the accept / reject decision and updates the
//                                        damping state (Constant / Adaptive / TrustRegion, strategy.py:41-46,134-151,248-274)
//                                     K2 parameters <- trial parameters, if accepted
//   PoseInv (independent poses):      K1 whole trial per pose in registers + decision in its last CTA;  K2 as above
//
// and the 16-double state comes back with one asynchronous copy + one stream synchronisation (the single host read of
// the step).  A rejected trial (rare) is retried by the host with the state it just read: K1 then starts from the stored
// blocks instead of re-linearising.  All scalars the decision needs are arguments of that call — the host stays the owner of
// `param_groups` (users edit the damping between steps), the device computes the update.
#include <stdlib.h>
#include "lm_common.cuh"
#include "comm.cuh"
#include "tma.cuh"

namespace b200pose {

constexpr int kMaxLmDevices = 64;
constexpr int kAccRows = 4;          // rows per lane in flight in the register-fed accumulation loops

// The deciding thread also publishes the state in mapped pinned host memory (zero-copy): the host spins on the sequence
// number instead of paying an asynchronous copy plus a stream synchronisation per trial.
struct HostOut { double* ptr; double seq; };
__device__ __forceinline__ void publish_state(const double* st, const HostOut& h) {
  if (!h.ptr) return;
  volatile double* o = h.ptr;
#pragma unroll
  for (int k = 0; k <= ST_FAILED; ++k) o[k] = st[k];
  __threadfence_system();
  o[ST_SIZE - 1] = h.seq;
}

// The whole reprojection trial of ONE camera in one place (single GPU): accumulate the camera's rows -> 6x6 solve ->
// retraction -> the camera's rows again with the trial pose (second read served by L1 / L2: a camera's rows are a few KB) ->
// trial loss.  Nothing grid-wide separates "solve" from "trial loss" when H is block-diagonal, so K1 and K2 above fuse into
// one launch and the decision runs in its last CTA.  FROM_BLOCKS: a retry starts from the stored blocks instead of the rows.
// sums (ws): [0] current loss, [1] trial loss, [2] predicted reduction, [3] failed pivots
template <typename T, int LPC, bool FROM_BLOCKS>
__global__ void __launch_bounds__(kLmThreads) reproj_trial_kernel(const T* __restrict__ poses, const T* __restrict__ pts,
                                                                   const T* __restrict__ pix, const int* __restrict__ seg,
                                                                   T* __restrict__ H, T* __restrict__ g, T* __restrict__ Pt,
                                                                   double* ws, double* st, LmCtl ctl, HostOut ho, T scale,
                                                                   T dmin, T dmax, int rk, T rdelta, int ncam) {
  const int sub = threadIdx.x % LPC;
  constexpr int cpb = kLmThreads / LPC;
  const int rounds = (ncam + cpb - 1) / cpb;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const int c = rd * cpb + threadIdx.x / LPC;
    const bool valid = c < ncam;
    const int cc = valid ? c : 0;
    T pr[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) pr[k] = poses[(long long)cc * 7 + k];
    const Elem<T> Tc = load_se3(pr);
    const int b = valid ? seg[cc] : 0, e = valid ? seg[cc + 1] : 0;
    Sys6<T> s;
    T loss = T(0);
    if (!FROM_BLOCKS) {
      Acc6<T> ac;
      ac.zero();
      auto accumulate = [&](const V3<T>& p, T zx, T zy) {
        T rx, ry;
        V3<T> y;
        reproj_residual(Tc, p, zx, zy, rx, ry, y);
        T j0[6], j1[6];
        reproj_rows(y, j0, j1);
        T rho, w;
        robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
        if (rk) {
          const T sw = m_sqrt(w);
          rx *= sw; ry *= sw;
#pragma unroll
          for (int a = 0; a < 6; ++a) { j0[a] *= sw; j1[a] *= sw; }
        }
        ac.add_row(j0, rx);
        ac.add_row(j1, ry);
        loss += rho;
      };
      // kAccRows rows per lane in flight: at 96-110 registers only 16-20 warps are resident, so the bytes in flight have
      // to come from the unroll
      int k = b + sub;
      for (; k + (kAccRows - 1) * LPC < e; k += kAccRows * LPC) {
        T v[kAccRows][5];
#pragma unroll
        for (int u = 0; u < kAccRows; ++u) {
          const long long ku = k + u * LPC;
          v[u][0] = pts[ku * 3]; v[u][1] = pts[ku * 3 + 1]; v[u][2] = pts[ku * 3 + 2];
          v[u][3] = pix[ku * 2]; v[u][4] = pix[ku * 2 + 1];
        }
#pragma unroll
        for (int u = 0; u < kAccRows; ++u) accumulate(mk(v[u][0], v[u][1], v[u][2]), v[u][3], v[u][4]);
      }
      for (; k < e; k += LPC) {
        const long long k0 = k;
        accumulate(mk(pts[k0 * 3], pts[k0 * 3 + 1], pts[k0 * 3 + 2]), pix[k0 * 2], pix[k0 * 2 + 1]);
      }
      s = ac.finish();
#pragma unroll
      for (int o = LPC / 2; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          s.g[a] += __shfl_xor_sync(0xffffffffu, s.g[a], o);
#pragma unroll
          for (int bb = a; bb < 6; ++bb) s.A[a][bb] += __shfl_xor_sync(0xffffffffu, s.A[a][bb], o);
        }
        loss += __shfl_xor_sync(0xffffffffu, loss, o);
      }
    } else {
      sys6_zero(s);
      int q = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        s.g[a] = g[(long long)cc * 6 + a];
#pragma unroll
        for (int bb = a; bb < 6; ++bb) s.A[a][bb] = H[(long long)cc * 21 + q++];
      }
    }
    T D[6], pred;
    const bool ok = sys6_damped_solve(s, scale, dmin, dmax, D, pred);
    const Elem<T> Pn = se3_retract(D, Tc);
    if (valid && sub == 0) {
      T o7[7];
      store_elem<SE3g, T>(o7, Pn);
#pragma unroll
      for (int q = 0; q < 7; ++q) Pt[(long long)c * 7 + q] = o7[q];
      if (!FROM_BLOCKS) {
        int q = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          g[(long long)c * 6 + a] = s.g[a];
#pragma unroll
          for (int bb = a; bb < 6; ++bb) H[(long long)c * 21 + q++] = s.A[a][bb];
        }
      }
      acc[0] += (double)loss;
      acc[2] += (double)pred;
      acc[3] += ok ? 0.0 : 1.0;
    }
    // trial loss over the same rows with the trial pose (every lane adds its own partial)
    T tl = T(0);
    {
      auto trial = [&](const T* v) {
        T rx, ry, rho, w;
        V3<T> y;
        reproj_residual(Pn, mk(v[0], v[1], v[2]), v[3], v[4], rx, ry, y);
        robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
        tl += rho;
      };
      // the accumulators are dead here: keep kTrialRows rows per lane in flight (the fused kernel's occupancy is set by
      // the accumulation loop, so the bytes in flight have to come from the unroll)
      constexpr int kTrialRows = 4;
      int k = b + sub;
      for (; k + (kTrialRows - 1) * LPC < e; k += kTrialRows * LPC) {
        T v[kTrialRows][5];
#pragma unroll
        for (int u = 0; u < kTrialRows; ++u) {
          const long long ku = k + u * LPC;
          v[u][0] = pts[ku * 3]; v[u][1] = pts[ku * 3 + 1]; v[u][2] = pts[ku * 3 + 2];
          v[u][3] = pix[ku * 2]; v[u][4] = pix[ku * 2 + 1];
        }
#pragma unroll
        for (int u = 0; u < kTrialRows; ++u) trial(v[u]);
      }
      for (; k < e; k += LPC) {
        const long long k0 = k;
        const T v[5] = {pts[k0 * 3], pts[k0 * 3 + 1], pts[k0 * 3 + 2], pix[k0 * 2], pix[k0 * 2 + 1]};
        trial(v);
      }
    }
    acc[1] += (double)tl;
  }
  if (reduce_sums<4>(acc, ws)) {
    lm_decide(ctl, ws[0], ws[1], ws[2], ws[3], st);
    publish_state(st, ho);
  }
}

// The same trial with the rows STAGED through shared memory by 1-D TMA bulk copies (tma.cuh): one warp per camera, a ring
// of kStages tiles of kStageRows rows per warp, each tile one `cp.async.bulk` of the points and one of the pixels signalled
// by an mbarrier.  The register-fed kernel above keeps (rows in flight per lane) x (resident warps) bytes in flight, and its
// ~96 registers cap the warps.  Here the bytes in flight are the ring
// (kStages x 2.5 KB per warp, ~200 KB per SM), independent of the register count, and the lanes only read shared memory
// (row stride 3 words / 2 words: conflict-free).  Both passes — accumulate, then the trial loss with the solved pose — are
// ONE stream of 2 x tiles through the ring, so the first tiles of the second pass are already in flight while the warp
// reduces and solves; a camera whose rows fit the ring (<= kStages tiles) is read from HBM once.
// Tiles start at a multiple of 4 rows (16-byte alignment of both arrays); rows of the tile outside [seg[c], seg[c+1]) are
// masked.  The one tile that would run past the end of the arrays is copied by the lanes instead.
template <typename T> struct Staged {
  static constexpr int kRows = 128;                               // rows per tile
  static constexpr int kStages = sizeof(T) == 4 ? 4 : 3;
  static constexpr int kWords = kRows * 5;                        // points (3) then pixels (2)
  static constexpr int kWarps = kLmThreads / 32;
  static constexpr int kBytes = kWarps * kStages * (kWords * (int)sizeof(T) + 8);
};
template <typename T, bool FROM_BLOCKS>
__global__ void __launch_bounds__(kLmThreads) reproj_trial_staged_kernel(
    const T* __restrict__ poses, const T* __restrict__ pts, const T* __restrict__ pix, const int* __restrict__ seg,
    T* __restrict__ H, T* __restrict__ g, T* __restrict__ Pt, double* ws, double* st, LmCtl ctl, HostOut ho, T scale, T dmin,
    T dmax, int rk, T rdelta, int ncam, long long rows_total) {
  using L = Staged<T>;
  constexpr int R = L::kRows, S = L::kStages;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  T* ring = reinterpret_cast<T*>(smem_raw) + warp * S * L::kWords;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + L::kWarps * S * L::kWords * sizeof(T)) + warp * S;
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < S; ++q) mbar_init(&full[q], 1);
    fence_mbar_init();
  }
  __syncwarp();
  int sc = 0;                 // next stage to consume == next stage to fill whenever the ring is drained
  uint32_t par = 0;           // phase parity per stage (bit q)
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  const int rounds = (ncam + L::kWarps - 1) / L::kWarps;
  for (int rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const int c = rd * L::kWarps + warp;
    const bool valid = c < ncam;
    const int cc = valid ? c : 0;
    T pr[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) pr[k] = poses[(long long)cc * 7 + k];
    const Elem<T> Tc = load_se3(pr);
    const int b = valid ? seg[cc] : 0, e = valid ? seg[cc + 1] : 0;
    const long long a0 = (long long)(b / 4) * 4;
    const int nt = e > b ? (int)((e - a0 + R - 1) / R) : 0;
    const bool resident = !FROM_BLOCKS && nt <= S;           // second pass straight from the ring
    const int jend = FROM_BLOCKS || resident ? nt : 2 * nt;  // tiles streamed for this camera
    int issued = 0, si = sc;
    auto issue = [&]() {                                      // tile (issued % nt) -> stage si
      const int t = issued >= nt ? issued - nt : issued;
      const long long r0 = a0 + (long long)t * R;
      T* dst = ring + si * L::kWords;
      if (r0 + R <= rows_total) {
        if (lane == 0) {
          mbar_expect_tx(&full[si], (uint32_t)(R * 5 * sizeof(T)));
          bulk_g2s(dst, pts + r0 * 3, (uint32_t)(R * 3 * sizeof(T)), &full[si]);
          bulk_g2s(dst + R * 3, pix + r0 * 2, (uint32_t)(R * 2 * sizeof(T)), &full[si]);
        }
      } else {                                                // the last tile of the arrays: plain copies by the lanes
        const int cnt = (int)(rows_total - r0);
        for (int i = lane; i < cnt * 3; i += 32) dst[i] = pts[r0 * 3 + i];
        for (int i = lane; i < cnt * 2; i += 32) dst[R * 3 + i] = pix[r0 * 2 + i];
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[si]);
      }
      ++issued;
      if (++si == S) si = 0;
    };
    while (issued < jend && issued < S) issue();

    // consume tile t of a pass out of stage q: f(point, pixel) for this lane's rows inside [b, e)
    auto for_rows = [&](int t, int q, auto&& f) {
      const T* sp = ring + q * L::kWords;
      const T* sx = sp + R * 3;
      const long long r0 = a0 + (long long)t * R;
#pragma unroll
      for (int u = 0; u < R / 32; ++u) {
        const int row = lane + 32 * u;
        const long long k = r0 + row;
        if (k >= b && k < e) f(mk(sp[row * 3], sp[row * 3 + 1], sp[row * 3 + 2]), sx[row * 2], sx[row * 2 + 1]);
      }
    };
    auto next_tile = [&](int t, auto&& f) {                   // wait, consume, refill the stage
      mbar_wait(&full[sc], (par >> sc) & 1u);
      par ^= 1u << sc;
      for_rows(t, sc, f);
      __syncwarp();                                           // every lane has read the stage before it is overwritten
      if (issued < jend) issue();
      if (++sc == S) sc = 0;
    };

    Sys6<T> s;
    T loss = T(0);
    const int s_first = sc;
    if (!FROM_BLOCKS) {
      Acc6<T> ac;
      ac.zero();
      auto accumulate = [&](const V3<T>& p, T zx, T zy) {
        T rx, ry;
        V3<T> y;
        reproj_residual(Tc, p, zx, zy, rx, ry, y);
        T j0[6], j1[6];
        reproj_rows(y, j0, j1);
        T rho, w;
        robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
        if (rk) {
          const T sw = m_sqrt(w);
          rx *= sw; ry *= sw;
#pragma unroll
          for (int a = 0; a < 6; ++a) { j0[a] *= sw; j1[a] *= sw; }
        }
        ac.add_row(j0, rx);
        ac.add_row(j1, ry);
        loss += rho;
      };
      for (int t = 0; t < nt; ++t) next_tile(t, accumulate);
      s = ac.finish();
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          s.g[a] += __shfl_xor_sync(0xffffffffu, s.g[a], o);
#pragma unroll
          for (int bb = a; bb < 6; ++bb) s.A[a][bb] += __shfl_xor_sync(0xffffffffu, s.A[a][bb], o);
        }
        loss += __shfl_xor_sync(0xffffffffu, loss, o);
      }
    } else {
      sys6_zero(s);
      int q = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        s.g[a] = g[(long long)cc * 6 + a];
#pragma unroll
        for (int bb = a; bb < 6; ++bb) s.A[a][bb] = H[(long long)cc * 21 + q++];
      }
    }
    T D[6], pred;
    const bool ok = sys6_damped_solve(s, scale, dmin, dmax, D, pred);
    const Elem<T> Pn = se3_retract(D, Tc);
    if (valid && lane == 0) {
      T o7[7];
      store_elem<SE3g, T>(o7, Pn);
#pragma unroll
      for (int q = 0; q < 7; ++q) Pt[(long long)c * 7 + q] = o7[q];
      if (!FROM_BLOCKS) {
        int q = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          g[(long long)c * 6 + a] = s.g[a];
#pragma unroll
          for (int bb = a; bb < 6; ++bb) H[(long long)c * 21 + q++] = s.A[a][bb];
        }
      }
      acc[0] += (double)loss;
      acc[2] += (double)pred;
      acc[3] += ok ? 0.0 : 1.0;
    }
    T tl = T(0);
    auto trial = [&](const V3<T>& p, T zx, T zy) {
      T rx, ry, rho, w;
      V3<T> y;
      reproj_residual(Pn, p, zx, zy, rx, ry, y);
      robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
      tl += rho;
    };
    if (resident) {
      int q = s_first;
      for (int t = 0; t < nt; ++t) {
        for_rows(t, q, trial);
        if (++q == S) q = 0;
      }
      __syncwarp();                                           // the next camera refills these stages
    } else {
      for (int t = 0; t < nt; ++t) next_tile(t, trial);
    }
    acc[1] += (double)tl;
  }
  if (reduce_sums<4>(acc, ws)) {
    lm_decide(ctl, ws[0], ws[1], ws[2], ws[3], st);
    publish_state(st, ho);
  }
}

// K1 of the PoseInv family: the whole trial per pose in registers (lm.cu lm_poseinv_trial_kernel) + the decision
template <typename T>
__global__ void __launch_bounds__(kLmThreads) poseinv_trial_decide_kernel(const T* __restrict__ P, const T* __restrict__ X,
                                                                           T* __restrict__ Pt, double* ws, double* st,
                                                                           LmCtl ctl, HostOut ho, T scale, T dmin, T dmax,
                                                                           int rk, T rdelta, long long n) {
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T p[7], x[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { p[k] = P[i * 7 + k]; x[k] = X[i * 7 + k]; }
    const Elem<T> Pe = load_se3(p), Xe = load_se3(x);
    Tang<T> r;
    Sys6<T> s;
    poseinv_linearize(Pe, Xe, r, s);
    T rho0, w0, rho1, w1;
    robust_eval(rk, rdelta, tang6_sqnorm(r), rho0, w0);
    if (rk) sys6_scale(s, w0);
    T D[6], pred;
    const bool ok = sys6_damped_solve(s, scale, dmin, dmax, D, pred);
    const Elem<T> Pn = se3_retract(D, Pe);
    T o[7];
    store_elem<SE3g, T>(o, Pn);
#pragma unroll
    for (int k = 0; k < 7; ++k) Pt[i * 7 + k] = o[k];
    robust_eval(rk, rdelta, tang6_sqnorm(poseinv_residual(Pn, Xe)), rho1, w1);
    acc[0] += (double)rho0;
    acc[1] += (double)rho1;
    acc[2] += (double)pred;
    acc[3] += ok ? 0.0 : 1.0;
  }
  if (reduce_sums<4>(acc, ws)) {
    lm_decide(ctl, ws[0], ws[1], ws[2], ws[3], st);
    publish_state(st, ho);
  }
}

// K3: parameters <- trial parameters when the decision was "accept" (update_parameter, optimizer.py:135-140)
template <typename T>
__global__ void __launch_bounds__(kLmThreads) lm_commit_kernel(const double* __restrict__ st, const T* __restrict__ src,
                                                                T* __restrict__ dst, long long count) {
  if (st[ST_STATUS] != 1.0) return;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < count; i += (long long)gridDim.x * kLmThreads)
    dst[i] = src[i];
}

// ================================================================================================================
// Multi-GPU trials over NVLink peer memory (comm.cuh): residual-sharded reprojection and pose-sharded PoseInv.
// No collective library call: producers store partial results into the consumer's exchange buffer and publish an epoch.
//
// Reprojection (cameras replicated, observations sharded; SURVEY.md §8e "residuals sharded, one packed reduction of
// [H | g | loss] per iteration, small reduction per trial") as a reduce-scatter / all-gather pair fused into the kernels:
//   K1p  every rank accumulates its observations' 27 sums per camera and stores them into the OWNER of that camera
//        (owner k holds cameras [k q, (k+1) q), q = ceil(C / world));                       signal channel 0
//   K2p  the owner adds the partials of the ranks that hold rows of the camera in rank order, keeps the reduced block for
//        retries, solves, retracts and stores the trial pose into every rank's copy;         signal channel 1
//   K3p  trial loss of the local observations -> scalar to every rank;                      signal channel 2
//   K4p  every rank adds the scalars in rank order (bit-identical decisions), decides, commits.
// Scalars whose producer may run ahead of a slow consumer (current loss, PoseInv sums) are double-buffered by epoch parity.
constexpr int CH_PART = 0, CH_TRIAL = 1, CH_LOSS = 2, CH_POSEINV = 3;

struct PeerRegions { long long part, pt; };     // byte offsets inside the payload: partial blocks, trial poses

// Exchange slots are padded to whole 16-byte vectors: 28 numbers per (source rank, camera) partial block (21 + 6 + pad),
// 8 per trial pose.  Every remote store is a 16-byte store and a thread fences ONCE, after its last store (27 scalar
// stores per camera from one lane with a system-scope fence per camera made the 2-GPU step slower than the 1-GPU step).
constexpr int kPartSlot = 28, kPoseSlot = 8;

// K1p: LPC lanes per camera over the local rows (same loop as reproj_trial_kernel), blocks staged in shared memory, then the
// CTA copies them to the owners with 16-byte stores.
// ALL: every rank receives every rank's blocks (slot [source rank][camera]) — the "gather" form for small problems, see
// reproj_gather_trial_kernel.
template <typename T, int LPC, bool ALL>
__global__ void __launch_bounds__(kLmThreads) reproj_accum_push_kernel(const T* __restrict__ poses, const T* __restrict__ pts,
                                                                        const T* __restrict__ pix, const int* __restrict__ seg,
                                                                        Peers P, PeerRegions R, double* ws,
                                                                        unsigned long long epoch, int rk, T rdelta, int ncam,
                                                                        const int* __restrict__ cams, int nloc) {
  // cams: the nloc cameras this rank holds rows of (with a `present` mask on the receivers), or NULL = all ncam cameras
  constexpr int cpb = kLmThreads / LPC;
  constexpr int NV = kPartSlot * (int)sizeof(T) / 16;
  __shared__ __align__(16) T sP[cpb][kPartSlot];
  __shared__ int sC[cpb];
  const int sub = threadIdx.x % LPC, slot = threadIdx.x / LPC;
  const int nwork = cams ? nloc : ncam;
  const int rounds = (nwork + cpb - 1) / cpb;
  const int q = (ncam + P.world - 1) / P.world;
  double acc[1] = {0.0};
  for (int rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const int idx = rd * cpb + slot;
    const bool valid = idx < nwork;
    const int c = valid ? (cams ? cams[idx] : idx) : -1;
    const int cc = valid ? c : 0;
    T pr[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) pr[k] = poses[(long long)cc * 7 + k];
    const Elem<T> Tc = load_se3(pr);
    const int b = valid ? seg[cc] : 0, e = valid ? seg[cc + 1] : 0;
    Acc6<T> ac;
    ac.zero();
    T loss = T(0);
    auto accumulate = [&](const V3<T>& p, T zx, T zy) {
      T rx, ry;
      V3<T> y;
      reproj_residual(Tc, p, zx, zy, rx, ry, y);
      T j0[6], j1[6];
      reproj_rows(y, j0, j1);
      T rho, w;
      robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
      if (rk) {
        const T sw = m_sqrt(w);
        rx *= sw; ry *= sw;
#pragma unroll
        for (int a = 0; a < 6; ++a) { j0[a] *= sw; j1[a] *= sw; }
      }
      ac.add_row(j0, rx);
      ac.add_row(j1, ry);
      loss += rho;
    };
    int k = b + sub;
    for (; k + (kAccRows - 1) * LPC < e; k += kAccRows * LPC) {
      T v[kAccRows][5];
#pragma unroll
      for (int u = 0; u < kAccRows; ++u) {
        const long long ku = k + u * LPC;
        v[u][0] = pts[ku * 3]; v[u][1] = pts[ku * 3 + 1]; v[u][2] = pts[ku * 3 + 2];
        v[u][3] = pix[ku * 2]; v[u][4] = pix[ku * 2 + 1];
      }
#pragma unroll
      for (int u = 0; u < kAccRows; ++u) accumulate(mk(v[u][0], v[u][1], v[u][2]), v[u][3], v[u][4]);
    }
    for (; k < e; k += LPC) {
      const long long k0 = k;
      accumulate(mk(pts[k0 * 3], pts[k0 * 3 + 1], pts[k0 * 3 + 2]), pix[k0 * 2], pix[k0 * 2 + 1]);
    }
    Sys6<T> s = ac.finish();
#pragma unroll
    for (int o = LPC / 2; o > 0; o >>= 1) {
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        s.g[a] += __shfl_xor_sync(0xffffffffu, s.g[a], o);
#pragma unroll
        for (int bb = a; bb < 6; ++bb) s.A[a][bb] += __shfl_xor_sync(0xffffffffu, s.A[a][bb], o);
      }
      loss += __shfl_xor_sync(0xffffffffu, loss, o);
    }
    if (sub == 0) {
      int t = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int bb = a; bb < 6; ++bb) sP[slot][t++] = s.A[a][bb];
#pragma unroll
      for (int a = 0; a < 6; ++a) sP[slot][21 + a] = s.g[a];
      sP[slot][27] = T(0);
      sC[slot] = c;
      if (valid) acc[0] += (double)loss;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < cpb * NV; j += kLmThreads) {
      const int sl = j / NV, v = j - sl * NV, cj = sC[sl];
      if (cj >= 0) {
        const float4 x = reinterpret_cast<const float4*>(&sP[sl][0])[v];
        if (ALL) {
          const long long off = kDataOffset + R.part + ((long long)P.rank * ncam + cj) * (kPartSlot * (long long)sizeof(T)) + v * 16;
          for (int r = 0; r < P.world; ++r) *reinterpret_cast<float4*>(P.base[r] + off) = x;
        } else {
          const int owner = cj / q;
          char* dst = P.base[owner] + kDataOffset + R.part +
                      ((long long)P.rank * q + (cj - owner * q)) * (kPartSlot * (long long)sizeof(T)) + v * 16;
          *reinterpret_cast<float4*>(dst) = x;
        }
      }
    }
    __syncthreads();                                   // the next round overwrites the staging slots
  }
  __threadfence_system();                              // this thread's remote stores are ordered before the CTA's ticket
  if (reduce_sums<1>(acc, ws)) {           // thread 0 of the last CTA: every CTA's stores are ordered before its ticket
    for (int r = 0; r < P.world; ++r) comm_scalars(P.base[r], CH_PART, P.rank)[(epoch & 1) * 4] = ws[0];
    comm_signal_all(P, CH_PART, epoch);
  }
}

// Gather form, K2g: every rank holds every rank's partial blocks, adds them in rank order per camera (bit-identical on all
// ranks), solves, retracts, keeps the block for retries and the trial pose locally, and goes straight on to the trial loss
// of its local rows — ONE exchange fewer than the owner form (no trial poses travel), at world x the partial-block traffic:
// chosen when world * ncam blocks are a few MB (at 1e4 cameras the owner form's three flag waits dominate the step).  Predicted reduction / failed pivots are counted by the
// camera's owner only, so that the sums over ranks are the totals.
template <typename T, int LPC>
__global__ void __launch_bounds__(kLmThreads) reproj_gather_trial_kernel(
    const T* __restrict__ poses, const T* __restrict__ pts, const T* __restrict__ pix, const int* __restrict__ seg,
    T* __restrict__ H, T* __restrict__ g, Peers P, PeerRegions R, double* ws, unsigned long long epoch0,
    unsigned long long epoch1, int retry, T scale, T dmin, T dmax, int rk, T rdelta, int ncam,
    const unsigned char* __restrict__ present) {
  constexpr int cpb = kLmThreads / LPC;
  constexpr int EV = 16 / (int)sizeof(T), NV = kPartSlot / EV;
  __shared__ __align__(16) T sP[cpb][kPartSlot];
  if (!retry) {
    if (threadIdx.x == 0) comm_wait_all(P, CH_PART, epoch0);
    __syncthreads();
  }
  const T* part = reinterpret_cast<const T*>(P.base[P.rank] + kDataOffset + R.part);
  T* Pt = reinterpret_cast<T*>(P.base[P.rank] + kDataOffset + R.pt);
  const int sub = threadIdx.x % LPC, slot = threadIdx.x / LPC;
  const int rounds = (ncam + cpb - 1) / cpb;
  const int q = (ncam + P.world - 1) / P.world;
  double acc[3] = {0.0, 0.0, 0.0};                      // trial loss (local rows), predicted, failed (owner's cameras)
  for (int rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const int c = rd * cpb + slot;
    const bool valid = c < ncam;
    const int cc = valid ? c : 0;
    if (!retry) {
      // lanes v < NV of the camera's group each add one 16-byte vector of the `world` blocks
      for (int v = sub; v < NV; v += LPC) {
        T a[EV];
#pragma unroll
        for (int kk = 0; kk < EV; ++kk) a[kk] = T(0);
        for (int r = 0; r < P.world; ++r) {
          if (present && !present[(long long)r * ncam + cc]) continue;       // rank r holds no rows of this camera
          const float4 x = reinterpret_cast<const float4*>(part + ((long long)r * ncam + cc) * kPartSlot)[v];
          const T* e = reinterpret_cast<const T*>(&x);
#pragma unroll
          for (int kk = 0; kk < EV; ++kk) a[kk] += e[kk];
        }
#pragma unroll
        for (int kk = 0; kk < EV; ++kk) sP[slot][v * EV + kk] = a[kk];
      }
      __syncwarp();
    }
    Sys6<T> s;
    {
      int t = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        s.g[a] = retry ? g[(long long)cc * 6 + a] : sP[slot][21 + a];
#pragma unroll
        for (int b = a; b < 6; ++b) { s.A[a][b] = retry ? H[(long long)cc * 21 + t] : sP[slot][t]; ++t; }
      }
    }
    T pr[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) pr[k] = poses[(long long)cc * 7 + k];
    T D[6], pred;
    const bool ok = sys6_damped_solve(s, scale, dmin, dmax, D, pred);
    const Elem<T> Pn = se3_retract(D, load_se3(pr));
    if (valid && sub == 0) {
      T o7[7];
      store_elem<SE3g, T>(o7, Pn);
#pragma unroll
      for (int k = 0; k < 7; ++k) Pt[(long long)c * kPoseSlot + k] = o7[k];
      if (!retry) {
        int t = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          g[(long long)c * 6 + a] = s.g[a];
#pragma unroll
          for (int b = a; b < 6; ++b) H[(long long)c * 21 + t++] = s.A[a][b];
        }
      }
      if (c / q == P.rank) {
        acc[1] += (double)pred;
        acc[2] += ok ? 0.0 : 1.0;
      }
    }
    const int b = valid ? seg[cc] : 0, e = valid ? seg[cc + 1] : 0;
    T tl = T(0);
    auto trial = [&](const T* v) {
      T rx, ry, rho, w;
      V3<T> y;
      reproj_residual(Pn, mk(v[0], v[1], v[2]), v[3], v[4], rx, ry, y);
      robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
      tl += rho;
    };
    constexpr int kRows = 4;
    int k = b + sub;
    for (; k + (kRows - 1) * LPC < e; k += kRows * LPC) {
      T v[kRows][5];
#pragma unroll
      for (int u = 0; u < kRows; ++u) {
        const long long ku = k + u * LPC;
        v[u][0] = pts[ku * 3]; v[u][1] = pts[ku * 3 + 1]; v[u][2] = pts[ku * 3 + 2];
        v[u][3] = pix[ku * 2]; v[u][4] = pix[ku * 2 + 1];
      }
#pragma unroll
      for (int u = 0; u < kRows; ++u) trial(v[u]);
    }
    for (; k < e; k += LPC) {
      const long long k0 = k;
      const T v[5] = {pts[k0 * 3], pts[k0 * 3 + 1], pts[k0 * 3 + 2], pix[k0 * 2], pix[k0 * 2 + 1]};
      trial(v);
    }
    acc[0] += (double)tl;
    __syncwarp();                                      // sP[slot] is rewritten by the next round
  }
  if (reduce_sums<3>(acc, ws)) {
    for (int r = 0; r < P.world; ++r) {
      double* sc = comm_scalars(P.base[r], CH_TRIAL, P.rank);
      sc[0] = ws[1]; sc[1] = ws[2];
      comm_scalars(P.base[r], CH_LOSS, P.rank)[0] = ws[0];
    }
    comm_signal_all(P, CH_LOSS, epoch1);
  }
}

template <typename T>
__global__ void __launch_bounds__(kLmThreads) reproj_reduce_solve_push_kernel(const T* __restrict__ poses, T* __restrict__ H,
                                                                               T* __restrict__ g, Peers P, PeerRegions R,
                                                                               double* ws, unsigned long long epoch0,
                                                                               unsigned long long epoch1, int retry, T scale,
                                                                               T dmin, T dmax, int ncam,
                                                                               const unsigned char* __restrict__ present) {
  const int q = (ncam + P.world - 1) / P.world;
  const int c0 = P.rank * q, c1 = min(ncam, c0 + q);
  if (!retry) {
    if (threadIdx.x == 0) comm_wait_all(P, CH_PART, epoch0);
    __syncthreads();
  }
  double acc[2] = {0.0, 0.0};
  const T* part = reinterpret_cast<const T*>(P.base[P.rank] + kDataOffset + R.part);
  constexpr int EV = 16 / (int)sizeof(T), NV = kPartSlot / EV, NVP = kPoseSlot / EV;
  for (int c = c0 + blockIdx.x * kLmThreads + threadIdx.x; c < c1; c += gridDim.x * kLmThreads) {
    Sys6<T> s;
    if (!retry) {
      T v[kPartSlot];
#pragma unroll
      for (int t = 0; t < kPartSlot; ++t) v[t] = T(0);
      for (int r = 0; r < P.world; ++r) {              // rank order: the same sum on every run
        if (present && !present[(long long)r * ncam + c]) continue;            // rank r holds no rows of this camera
        const float4* p4 = reinterpret_cast<const float4*>(part + ((long long)r * q + (c - c0)) * kPartSlot);
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const float4 x = p4[i];
          const T* e = reinterpret_cast<const T*>(&x);
#pragma unroll
          for (int kk = 0; kk < EV; ++kk) v[i * EV + kk] += e[kk];
        }
      }
      int t = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 6; ++b) { s.A[a][b] = v[t]; H[(long long)c * 21 + t] = v[t]; ++t; }
#pragma unroll
      for (int a = 0; a < 6; ++a) { s.g[a] = v[21 + a]; g[(long long)c * 6 + a] = v[21 + a]; }
    } else {
      int t = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        s.g[a] = g[(long long)c * 6 + a];
#pragma unroll
        for (int b = a; b < 6; ++b) s.A[a][b] = H[(long long)c * 21 + t++];
      }
    }
    T D[6], pred;
    const bool ok = sys6_damped_solve(s, scale, dmin, dmax, D, pred);
    T pr[7];
    __align__(16) T o[kPoseSlot];
#pragma unroll
    for (int k = 0; k < 7; ++k) pr[k] = poses[(long long)c * 7 + k];
    T o7[7];
    store_elem<SE3g, T>(o7, se3_retract(D, load_se3(pr)));
#pragma unroll
    for (int k = 0; k < 7; ++k) o[k] = o7[k];
    o[7] = T(0);
    for (int r = 0; r < P.world; ++r) {
      float4* dst = reinterpret_cast<float4*>(P.base[r] + kDataOffset + R.pt + (long long)c * (kPoseSlot * (long long)sizeof(T)));
#pragma unroll
      for (int i = 0; i < NVP; ++i) dst[i] = reinterpret_cast<const float4*>(o)[i];
    }
    acc[0] += (double)pred;
    acc[1] += ok ? 0.0 : 1.0;
  }
  __threadfence_system();                              // once per thread, after its last remote store
  if (reduce_sums<2>(acc, ws)) {
    for (int r = 0; r < P.world; ++r) {
      double* sc = comm_scalars(P.base[r], CH_TRIAL, P.rank);
      sc[0] = ws[0]; sc[1] = ws[1];
    }
    comm_signal_all(P, CH_TRIAL, epoch1);
  }
}

// K3p: trial loss of the local rows with the trial poses every owner pushed; LPC lanes per camera, 4 rows in flight
template <typename T, int LPC>
__global__ void __launch_bounds__(kLmThreads) reproj_loss_push_kernel(const T* __restrict__ pts, const T* __restrict__ pix,
                                                                       const int* __restrict__ seg, Peers P, PeerRegions R,
                                                                       double* ws, unsigned long long epoch1, int rk, T rdelta,
                                                                       int ncam, const int* __restrict__ cams, int nloc) {
  if (threadIdx.x == 0) comm_wait_all(P, CH_TRIAL, epoch1);
  __syncthreads();
  const T* Pt = reinterpret_cast<const T*>(P.base[P.rank] + kDataOffset + R.pt);
  constexpr int cpb = kLmThreads / LPC;
  const int sub = threadIdx.x % LPC, slot = threadIdx.x / LPC;
  const int nwork = cams ? nloc : ncam;
  const int rounds = (nwork + cpb - 1) / cpb;
  double acc[1] = {0.0};
  for (int rd = blockIdx.x; rd < rounds; rd += gridDim.x) {
    const int idx = rd * cpb + slot;
    if (idx >= nwork) continue;
    const int c = cams ? cams[idx] : idx;
    const int b = seg[c], e = seg[c + 1];
    if (b == e) continue;
    T pr[7];
#pragma unroll
    for (int qk = 0; qk < 7; ++qk) pr[qk] = Pt[(long long)c * kPoseSlot + qk];
    const Elem<T> Tc = load_se3(pr);
    T loss = T(0);
    auto trial = [&](const T* v) {
      T rx, ry, rho, w;
      V3<T> y;
      reproj_residual(Tc, mk(v[0], v[1], v[2]), v[3], v[4], rx, ry, y);
      robust_eval(rk, rdelta, rx * rx + ry * ry, rho, w);
      loss += rho;
    };
    constexpr int kRows = 4;
    int k = b + sub;
    for (; k + (kRows - 1) * LPC < e; k += kRows * LPC) {
      T v[kRows][5];
#pragma unroll
      for (int u = 0; u < kRows; ++u) {
        const long long ku = k + u * LPC;
        v[u][0] = pts[ku * 3]; v[u][1] = pts[ku * 3 + 1]; v[u][2] = pts[ku * 3 + 2];
        v[u][3] = pix[ku * 2]; v[u][4] = pix[ku * 2 + 1];
      }
#pragma unroll
      for (int u = 0; u < kRows; ++u) trial(v[u]);
    }
    for (; k < e; k += LPC) {
      const long long k0 = k;
      const T v[5] = {pts[k0 * 3], pts[k0 * 3 + 1], pts[k0 * 3 + 2], pix[k0 * 2], pix[k0 * 2 + 1]};
      trial(v);
    }
    acc[0] += (double)loss;
  }
  if (reduce_sums<1>(acc, ws)) {
    for (int r = 0; r < P.world; ++r) comm_scalars(P.base[r], CH_LOSS, P.rank)[0] = ws[0];
    comm_signal_all(P, CH_LOSS, epoch1);
  }
}
template <typename T>
__global__ void __launch_bounds__(kLmThreads) reproj_decide_commit_kernel(Peers P, PeerRegions R, double* st, LmCtl ctl,
                                                                           HostOut ho, unsigned long long epoch0,
                                                                           unsigned long long epoch1, T* __restrict__ poses,
                                                                           long long count) {
  __shared__ double sh[ST_SIZE];
  if (threadIdx.x == 0) {
    comm_wait_all(P, CH_LOSS, epoch1);
    double cur = 0.0, trial = 0.0, pred = 0.0, failed = 0.0;
    for (int r = 0; r < P.world; ++r) {
      cur += comm_scalars(P.base[P.rank], CH_PART, r)[(epoch0 & 1) * 4];
      pred += comm_scalars(P.base[P.rank], CH_TRIAL, r)[0];
      failed += comm_scalars(P.base[P.rank], CH_TRIAL, r)[1];
      trial += comm_scalars(P.base[P.rank], CH_LOSS, r)[0];
    }
    lm_decide(ctl, cur, trial, pred, failed, sh);
    if (blockIdx.x == 0) {
      for (int k = 0; k < ST_SIZE; ++k) st[k] = k <= ST_FAILED ? sh[k] : 0.0;
      publish_state(sh, ho);
    }
  }
  __syncthreads();
  if (sh[ST_STATUS] != 1.0) return;
  const T* Pt = reinterpret_cast<const T*>(P.base[P.rank] + kDataOffset + R.pt);
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < count; i += (long long)gridDim.x * kLmThreads)
    poses[i] = Pt[(i / 7) * kPoseSlot + i % 7];          // trial poses sit in 8-number slots
}

// PoseInv, poses sharded: the trial kernel of each rank pushes its four sums; decide + commit after one exchange
template <typename T>
__global__ void __launch_bounds__(kLmThreads) poseinv_trial_push_kernel(const T* __restrict__ Pm, const T* __restrict__ X,
                                                                         T* __restrict__ Pt, double* ws, Peers P,
                                                                         unsigned long long epoch, T scale, T dmin, T dmax,
                                                                         int rk, T rdelta, long long n) {
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLmThreads) {
    T p[7], x[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { p[k] = Pm[i * 7 + k]; x[k] = X[i * 7 + k]; }
    const Elem<T> Pe = load_se3(p), Xe = load_se3(x);
    Tang<T> r;
    Sys6<T> s;
    poseinv_linearize(Pe, Xe, r, s);
    T rho0, w0, rho1, w1;
    robust_eval(rk, rdelta, tang6_sqnorm(r), rho0, w0);
    if (rk) sys6_scale(s, w0);
    T D[6], pred;
    const bool ok = sys6_damped_solve(s, scale, dmin, dmax, D, pred);
    const Elem<T> Pn = se3_retract(D, Pe);
    T o[7];
    store_elem<SE3g, T>(o, Pn);
#pragma unroll
    for (int k = 0; k < 7; ++k) Pt[i * 7 + k] = o[k];
    robust_eval(rk, rdelta, tang6_sqnorm(poseinv_residual(Pn, Xe)), rho1, w1);
    acc[0] += (double)rho0;
    acc[1] += (double)rho1;
    acc[2] += (double)pred;
    acc[3] += ok ? 0.0 : 1.0;
  }
  if (reduce_sums<4>(acc, ws)) {
    for (int r = 0; r < P.world; ++r) {
      double* sc = comm_scalars(P.base[r], CH_POSEINV, P.rank) + (epoch & 1) * 4;
      sc[0] = ws[0]; sc[1] = ws[1]; sc[2] = ws[2]; sc[3] = ws[3];
    }
    comm_signal_all(P, CH_POSEINV, epoch);
  }
}
template <typename T>
__global__ void __launch_bounds__(kLmThreads) poseinv_decide_commit_kernel(Peers P, double* st, LmCtl ctl, HostOut ho,
                                                                            unsigned long long epoch,
                                                                            const T* __restrict__ Pt, T* __restrict__ Pm,
                                                                            long long count) {
  __shared__ double sh[ST_SIZE];
  if (threadIdx.x == 0) {
    comm_wait_all(P, CH_POSEINV, epoch);
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    for (int r = 0; r < P.world; ++r) {
      const double* sc = comm_scalars(P.base[P.rank], CH_POSEINV, r) + (epoch & 1) * 4;
      v[0] += sc[0]; v[1] += sc[1]; v[2] += sc[2]; v[3] += sc[3];
    }
    lm_decide(ctl, v[0], v[1], v[2], v[3], sh);
    if (blockIdx.x == 0) {
      for (int k = 0; k < ST_SIZE; ++k) st[k] = k <= ST_FAILED ? sh[k] : 0.0;
      publish_state(sh, ho);
    }
  }
  __syncthreads();
  if (sh[ST_STATUS] != 1.0) return;
  for (long long i = (long long)blockIdx.x * kLmThreads + threadIdx.x; i < count; i += (long long)gridDim.x * kLmThreads)
    Pm[i] = Pt[i];
}

static Peers make_peers(const unsigned long long* bases, int rank, int world) {
  Peers P;
  for (int r = 0; r < kMaxRanks; ++r) P.base[r] = r < world ? reinterpret_cast<char*>(bases[r]) : nullptr;
  P.rank = rank; P.world = world;
  return P;
}

static LmCtl make_ctl(const double* c) {
  LmCtl k;
  k.last = c[0]; k.cached = c[1] != 0.0; k.damping = c[2]; k.pg_down = c[3]; k.reject_count = c[4]; k.reject_limit = c[5];
  k.kind = (int)c[6]; k.high = c[7]; k.low = c[8]; k.up = c[9]; k.self_down = c[10]; k.factor = c[11]; k.smin = c[12];
  k.smax = c[13];
  return k;
}

// host_out is pinned host memory (device-accessible under UVA); the deciding thread writes the state and then `seq` into
// its last slot.  The caller stored a different value there before the launch (see make_host_out).
static HostOut make_host_out(double* host_out, long long seq) {
  HostOut h;
  h.ptr = host_out; h.seq = (double)seq;
  if (host_out) reinterpret_cast<volatile double*>(host_out)[ST_SIZE - 1] = -1.0;
  return h;
}
static int finish_step(double* host_out, long long seq, cudaStream_t s) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  if (!host_out) return 0;
  volatile double* flag = reinterpret_cast<volatile double*>(host_out) + (ST_SIZE - 1);
  for (long long spin = 0;; ++spin) {
    if (*flag == (double)seq) return 0;
    if ((spin & 0xffff) == 0xffff) {            // every ~65k polls: has the stream died or finished without publishing?
      e = cudaStreamQuery(s);
      if (e == cudaSuccess) return *flag == (double)seq ? 0 : (int)cudaErrorUnknown;
      if (e != cudaErrorNotReady) return (int)e;
    }
  }
}

// B200POSE_REPROJ_STAGED: 0 = register-fed kernels only, 1 (default) = TMA-staged kernel for long row lists,
// 2 = TMA-staged kernel always (A/B knob for DESIGN.md §3.3)
static int g_staged_mode = -1;
static int staged_mode() {
  if (g_staged_mode < 0) {
    const char* v = getenv("B200POSE_REPROJ_STAGED");
    g_staged_mode = v && *v ? atoi(v) : 1;
  }
  return g_staged_mode;
}
// lanes per camera of the register-fed kernel: 0 = by row count (32 for long lists, else 8); A/B knob (b200_lm_reproj_lanes)
static int g_reproj_lanes = 0;
template <typename T, int LPC, typename... A>
static void launch_reproj_trial(int retry, long long ncam, cudaStream_t s, const T* poses, const T* pts, const T* pix,
                                const int* seg, T* H, T* g, T* Pt, double* ws, double* st, const LmCtl& k, const HostOut& ho,
                                T scale, T dmin, T dmax, int robust, T delta) {
  const unsigned grid = lm_grid(ncam, kLmThreads / LPC);
  if (!retry)
    reproj_trial_kernel<T, LPC, false><<<grid, kLmThreads, 0, s>>>(poses, pts, pix, seg, H, g, Pt, ws, st, k, ho, scale, dmin,
                                                                   dmax, robust, delta, (int)ncam);
  else
    reproj_trial_kernel<T, LPC, true><<<grid, kLmThreads, 0, s>>>(poses, pts, pix, seg, H, g, Pt, ws, st, k, ho, scale, dmin,
                                                                  dmax, robust, delta, (int)ncam);
}
// dynamic shared memory above 48 KB needs the opt-in attribute, once per device and kernel
template <typename T> static int staged_prepare() {
  if (Staged<T>::kBytes <= 48 * 1024) return 0;
  static bool done[kMaxLmDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  const int slot = dev >= 0 && dev < kMaxLmDevices ? dev : 0;
  if (done[slot] && dev == slot) return 0;
  cudaError_t e = cudaFuncSetAttribute(reproj_trial_staged_kernel<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Staged<T>::kBytes);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(reproj_trial_staged_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             Staged<T>::kBytes);
  if (e == cudaSuccess) done[slot] = true;
  return (int)e;
}

}  // namespace b200pose

using namespace b200pose;

B200_EXPORT int b200_lm_reproj_lanes(int lanes) {
  const int prev = g_reproj_lanes;
  if (lanes == 0 || lanes == 8 || lanes == 16 || lanes == 32) g_reproj_lanes = lanes;
  return prev;
}
B200_EXPORT int b200_lm_reproj_staged_mode(int mode) {
  const int prev = staged_mode();
  if (mode >= 0) g_staged_mode = mode;
  return prev;
}

#define LMSTEP_ABI(SFX, CT)                                                                                           \
  B200_EXPORT int b200_lm_reproj_step_##SFX(CT* poses, const CT* pts, const CT* pix, const int* seg, CT* H, CT* g,    \
                                            CT* P_trial, double* ws0, double* ws1, double* st, double* host_out,      \
                                            long long seq, const double* ctl, int robust, double delta, double scale, \
                                            double dmin, double dmax, int retry, long long rows, long long ncam,      \
                                            void* stream) {                                                           \
    if (ncam <= 0) return 0;                                                                                          \
    cudaStream_t s = (cudaStream_t)stream;                                                                            \
    const LmCtl k = make_ctl(ctl);                                                                                    \
    const HostOut ho = make_host_out(host_out, seq);                                                                  \
    const bool wide = rows >= 384 * ncam;                  /* lanes per camera: 32 for long lists, else 8 */          \
    (void)ws1;                                                                                                        \
    const int staged = staged_mode();                                                                                 \
    if ((staged == 2 || (staged == 1 && wide)) && ((((uintptr_t)pts) | ((uintptr_t)pix)) & 15) == 0) {               \
      int rc = staged_prepare<CT>();                                                                                  \
      if (rc) return rc;                                                                                              \
      const unsigned sgrid = lm_grid(ncam, kLmThreads / 32);                                                          \
      if (!retry)                                                                                                     \
        reproj_trial_staged_kernel<CT, false><<<sgrid, kLmThreads, Staged<CT>::kBytes, s>>>(                          \
            poses, pts, pix, seg, H, g, P_trial, ws0, st, k, ho, (CT)scale, (CT)dmin, (CT)dmax, robust, (CT)delta,    \
            (int)ncam, rows);                                                                                         \
      else                                                                                                            \
        reproj_trial_staged_kernel<CT, true><<<sgrid, kLmThreads, Staged<CT>::kBytes, s>>>(                           \
            poses, pts, pix, seg, H, g, P_trial, ws0, st, k, ho, (CT)scale, (CT)dmin, (CT)dmax, robust, (CT)delta,    \
            (int)ncam, rows);                                                                                         \
    } else {                                                                                                          \
      const int lanes = g_reproj_lanes ? g_reproj_lanes : (wide ? 32 : 8);                                            \
      if (lanes == 32) launch_reproj_trial<CT, 32>(retry, ncam, s, poses, pts, pix, seg, H, g, P_trial, ws0, st, k, ho, \
                                                   (CT)scale, (CT)dmin, (CT)dmax, robust, (CT)delta);                 \
      else if (lanes == 16) launch_reproj_trial<CT, 16>(retry, ncam, s, poses, pts, pix, seg, H, g, P_trial, ws0, st, \
                                                        k, ho, (CT)scale, (CT)dmin, (CT)dmax, robust, (CT)delta);     \
      else launch_reproj_trial<CT, 8>(retry, ncam, s, poses, pts, pix, seg, H, g, P_trial, ws0, st, k, ho, (CT)scale, \
                                      (CT)dmin, (CT)dmax, robust, (CT)delta);                                         \
    }                                                                                                                 \
    lm_commit_kernel<CT><<<lm_grid(ncam * 7, kLmThreads), kLmThreads, 0, s>>>(st, P_trial, poses, ncam * 7);          \
    return finish_step(host_out, seq, s);                                                                             \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_poseinv_step_##SFX(CT* P, const CT* X, CT* P_trial, double* ws, double* st,                 \
                                             double* host_out, long long seq, const double* ctl, int robust,          \
                                             double delta, double scale, double dmin, double dmax, long long n,       \
                                             void* stream) {                                                          \
    if (n <= 0) return 0;                                                                                             \
    cudaStream_t s = (cudaStream_t)stream;                                                                            \
    const LmCtl k = make_ctl(ctl);                                                                                    \
    const HostOut ho = make_host_out(host_out, seq);                                                                  \
    poseinv_trial_decide_kernel<CT><<<lm_grid(n, kLmThreads), kLmThreads, 0, s>>>(                                    \
        P, X, P_trial, ws, st, k, ho, (CT)scale, (CT)dmin, (CT)dmax, robust, (CT)delta, n);                           \
    lm_commit_kernel<CT><<<lm_grid(n * 7, kLmThreads), kLmThreads, 0, s>>>(st, P_trial, P, n * 7);                    \
    return finish_step(host_out, seq, s);                                                                             \
  }

#define LMSTEP_PEER_ABI(SFX, CT)                                                                                      \
  B200_EXPORT int b200_lm_reproj_step_peer_##SFX(CT* poses, const CT* pts, const CT* pix, const int* seg, CT* H,      \
                                                 CT* g, const unsigned long long* bases, int rank, int world,         \
                                                 long long part_off, long long pt_off, long long epoch0,              \
                                                 long long epoch1, double* ws0, double* ws1, double* ws2, double* st, \
                                                 double* host_out, long long seq, const double* ctl, int robust,      \
                                                 double delta, double scale, double dmin, double dmax, int retry,     \
                                                 long long rows, int gather, const unsigned char* present,            \
                                                 const int* cams, long long nloc, long long ncam, void* stream) {     \
    if (ncam <= 0) return 0;                                                                                          \
    cudaStream_t s = (cudaStream_t)stream;                                                                            \
    const LmCtl k = make_ctl(ctl);                                                                                    \
    const HostOut ho = make_host_out(host_out, seq);                                                                  \
    const Peers P = make_peers(bases, rank, world);                                                                   \
    const PeerRegions R = {part_off, pt_off};                                                                         \
    const long long ncw = cams ? nloc : ncam;              /* cameras this rank works on */                           \
    const bool wide = rows >= 384 * ncw;                   /* lanes per camera from the LOCAL rows per local camera */ \
    const unsigned wgrid = lm_grid(ncw, wide ? kLmThreads / 32 : kLmThreads / 8);     /* K1 / K3p: local cameras */    \
    const unsigned agrid = lm_grid(ncam, wide ? kLmThreads / 32 : kLmThreads / 8);    /* K2g: all cameras */           \
    const long long q = (ncam + world - 1) / world;                                                                   \
    const unsigned long long e0 = (unsigned long long)epoch0, e1 = (unsigned long long)epoch1;                        \
    if (!retry) {                                                                                                     \
      if (wide && gather)                                                                                             \
        reproj_accum_push_kernel<CT, 32, true><<<wgrid, kLmThreads, 0, s>>>(poses, pts, pix, seg, P, R, ws0, e0,      \
                                                                            robust, (CT)delta, (int)ncam, cams, (int)nloc);      \
      else if (wide)                                                                                                  \
        reproj_accum_push_kernel<CT, 32, false><<<wgrid, kLmThreads, 0, s>>>(poses, pts, pix, seg, P, R, ws0, e0,     \
                                                                             robust, (CT)delta, (int)ncam, cams, (int)nloc);     \
      else if (gather)                                                                                                \
        reproj_accum_push_kernel<CT, 8, true><<<wgrid, kLmThreads, 0, s>>>(poses, pts, pix, seg, P, R, ws0, e0,       \
                                                                           robust, (CT)delta, (int)ncam, cams, (int)nloc);       \
      else                                                                                                            \
        reproj_accum_push_kernel<CT, 8, false><<<wgrid, kLmThreads, 0, s>>>(poses, pts, pix, seg, P, R, ws0, e0,      \
                                                                            robust, (CT)delta, (int)ncam, cams, (int)nloc);      \
    }                                                                                                                 \
    if (gather) {                                                                                                     \
      if (wide)                                                                                                       \
        reproj_gather_trial_kernel<CT, 32><<<agrid, kLmThreads, 0, s>>>(poses, pts, pix, seg, H, g, P, R, ws1, e0,    \
                                                                        e1, retry, (CT)scale, (CT)dmin, (CT)dmax,     \
                                                                        robust, (CT)delta, (int)ncam, present);       \
      else                                                                                                            \
        reproj_gather_trial_kernel<CT, 8><<<agrid, kLmThreads, 0, s>>>(poses, pts, pix, seg, H, g, P, R, ws1, e0, e1, \
                                                                       retry, (CT)scale, (CT)dmin, (CT)dmax, robust,  \
                                                                       (CT)delta, (int)ncam, present);                \
    } else {                                                                                                          \
      reproj_reduce_solve_push_kernel<CT><<<lm_grid(q, kLmThreads), kLmThreads, 0, s>>>(                              \
          poses, H, g, P, R, ws1, e0, e1, retry, (CT)scale, (CT)dmin, (CT)dmax, (int)ncam, present);                  \
      if (wide)                                                                                                       \
        reproj_loss_push_kernel<CT, 32><<<wgrid, kLmThreads, 0, s>>>(pts, pix, seg, P, R, ws2, e1, robust,            \
                                                                     (CT)delta, (int)ncam, cams, (int)nloc);          \
      else                                                                                                            \
        reproj_loss_push_kernel<CT, 8><<<wgrid, kLmThreads, 0, s>>>(pts, pix, seg, P, R, ws2, e1, robust, (CT)delta,  \
                                                                    (int)ncam, cams, (int)nloc);                      \
    }                                                                                                                 \
    reproj_decide_commit_kernel<CT><<<lm_grid(ncam * 7, kLmThreads), kLmThreads, 0, s>>>(                             \
        P, R, st, k, ho, (unsigned long long)epoch0, (unsigned long long)epoch1, poses, ncam * 7);                    \
    return finish_step(host_out, seq, s);                                                                             \
  }                                                                                                                   \
  B200_EXPORT int b200_lm_poseinv_step_peer_##SFX(CT* P_, const CT* X, CT* P_trial, const unsigned long long* bases,  \
                                                  int rank, int world, long long epoch, double* ws, double* st,       \
                                                  double* host_out, long long seq, const double* ctl, int robust,     \
                                                  double delta, double scale, double dmin, double dmax, long long n,  \
                                                  void* stream) {                                                     \
    cudaStream_t s = (cudaStream_t)stream;                                                                            \
    const LmCtl k = make_ctl(ctl);                                                                                    \
    const HostOut ho = make_host_out(host_out, seq);                                                                  \
    const Peers P = make_peers(bases, rank, world);                                                                   \
    poseinv_trial_push_kernel<CT><<<lm_grid(n > 0 ? n : 1, kLmThreads), kLmThreads, 0, s>>>(                          \
        P_, X, P_trial, ws, P, (unsigned long long)epoch, (CT)scale, (CT)dmin, (CT)dmax, robust, (CT)delta, n);       \
    poseinv_decide_commit_kernel<CT><<<lm_grid(n > 0 ? n * 7 : 1, kLmThreads), kLmThreads, 0, s>>>(                   \
        P, st, k, ho, (unsigned long long)epoch, P_trial, P_, n * 7);                                                 \
    return finish_step(host_out, seq, s);                                                                             \
  }

LMSTEP_ABI(f32, float)
LMSTEP_ABI(f64, double)
LMSTEP_PEER_ABI(f32, float)
LMSTEP_PEER_ABI(f64, double)
