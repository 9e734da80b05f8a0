// Device-resident Gauss-Newton / dogleg loop (stage C shell on the GPU): ImuFactor, marginalisation prior, extrinsic
// PriorFactor, the dense n = 15 (O + 1) + 6 normal equations and the Ceres-1.14 trust-region step all run on the device;
// the host only enqueues kernels and reads the final state back.
//
// Per evaluation of a solve (reference: ceres::Solve at src/imu_processor/Estimator.cc:1989, options :1909-1921):
//
//   asm_ppp    (assemble.cu)  every PivotPointPlaneFactor at the state being evaluated -> O packed 7x7 blocks S_i
//   k_factors  (O + 1 CTAs, beside asm_ppp on a second stream)  everything that depends on the state but not on the lidar
//              features: ImuFactor::Evaluate (include/factor/ImuFactor.h:53-167) -> whitened J^T J (30 x 30), J^T r, cost;
//              MarginalizationFactor::Evaluate (src/factor/MarginalizationFactor.cc:343-392) as Hp dx + bp and its cost;
//              PriorFactor (src/factor/PriorFactor.cc:35-67); the 6 x 18 maps M_i of the lidar blocks
//   k_step     (one CTA, 1024 threads)  judges the candidate (TrustRegionMinimizer), and for an accepted point gathers
//              H = Hp + sum M_i^T S_i M_i + sum J^T J (+ PriorFactor) element-wise, Jacobi-scales it, factors
//              H + mu D^2 with a tiled Cholesky in shared memory and takes the TRADITIONAL_DOGLEG step; writes the
//              candidate and its frame terms (R, t) for the next asm_ppp launch.
//
// Cholesky: the lower triangle lives in shared memory as 8 x 8 tiles (XOR-swizzled so that the fp64 MMA fragment loads
// are bank-conflict free).  Right-looking over 8-column panels: the diagonal tile is factored and inverted by warp 0
// one panel ahead (look-ahead, overlapped with the trailing update), the panel solve X = A L^-T and the trailing update
// C -= X X^T are fp64 tensor-core MMAs (mma.sync m8n8k4, DMMA) - the one piece of the solver that is a genuine GEMM.
// The right-hand side rides along as an extra row, so the forward substitution is free; the back substitution walks the
// tiles in reverse.  n <= 216 (O <= 13) fits one SM (k_step).  O = 14..16 (n <= 261, 33 tile columns, 299 KiB) runs the
// same step body as k_step_x2, a cluster of two CTAs: rank 0 computes, rank 1 lends its shared memory for half of the
// off-diagonal tiles, which rank 0 reaches over DSMEM (OneCta / TwoCta below decide where each tile lives).
#include "solver_dev.cuh"
#include <algorithm>
#include <cooperative_groups.h>

namespace lio {
using namespace hm;
namespace cg = cooperative_groups;

constexpr int kDsThreads = 512;   // 128 registers per thread: the serial diagonal-tile chain lives entirely in one lane's registers
constexpr int kDsWarps = kDsThreads / 32;
constexpr int kFThreads = 256;

struct FPtrs { double *imu, *M, *prior, *ex, *G; };

__device__ __forceinline__ const double *x_pose(const double *x, int k) { return x + 16 * k; }
__device__ __forceinline__ const double *x_sb(const double *x, int k) { return x + 16 * k + 7; }
// upper-triangle (row-major) index of (lo, hi), lo <= hi, in the packed 7 x 7 block of asm_ppp
__device__ __forceinline__ int s_idx(int lo, int hi) { return lo * 7 - lo * (lo - 1) / 2 + (hi - lo); }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum of up to three values over the block; every thread gets the totals.  sred: 3 * 32 + 3 doubles.
__device__ void block_sum3(double &a, double &b, double &c, double *sred) {
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  const int w = warp_id(), l = lane_id(), nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) { sred[w] = a; sred[32 + w] = b; sred[64 + w] = c; }
  __syncthreads();
  if (w == 0) {
    double ta = l < nw ? sred[l] : 0.0, tb = l < nw ? sred[32 + l] : 0.0, tc = l < nw ? sred[64 + l] : 0.0;
    ta = warp_sum(ta); tb = warp_sum(tb); tc = warp_sum(tc);
    if (l == 0) { sred[96] = ta; sred[97] = tb; sred[98] = tc; }
  }
  __syncthreads();
  a = sred[96]; b = sred[97]; c = sred[98];
}

__device__ double block_max(double v, double *sred) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int w = warp_id(), l = lane_id(), nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) sred[w] = v;
  __syncthreads();
  if (w == 0) {
    double t = l < nw ? sred[l] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fmax(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (l == 0) sred[96] = t;
  }
  __syncthreads();
  return sred[96];
}

__device__ void pose_dx_dev(const double *x, const double *x0, double *out) {  // MarginalizationFactor::Evaluate :347-372
  for (int k = 0; k < 3; ++k) out[k] = x[k] - x0[k];
  Q q0(x0[6], x0[3], x0[4], x0[5]), q(x[6], x[3], x[4], x[5]);
  Q dq = inverse(q0) * q;
  Q dn = normalized(dq);
  const double s = dq.w < 0 ? -2.0 : 2.0;
  out[3] = s * dn.x; out[4] = s * dn.y; out[5] = s * dn.z;
}

// =====================================================================================================
// k_factors: one CTA per ImuFactor (+ the frame terms M of the lidar block of frame b + 1), one CTA for the prior
__device__ __forceinline__ long long gtime_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// %globaltimer stamps of the kernels between two k_step launches (dbg[eval][12..15], zeroed with the state upload):
// [12] first k_factors CTA in, [13] last k_factors CTA out, [14] last k_hpart CTA out, [15] asm_ppp tail out (assemble.cu)
__device__ __forceinline__ void stamp_max(DevSolveState *S, int ev, int slot) {
  if (ev < 24) atomicMax(reinterpret_cast<unsigned long long *>(&S->dbg[ev][slot]), (unsigned long long)gtime_ns());
}

__global__ void __launch_bounds__(kFThreads, 2)   // <= 128 registers: a CTA must fit beside an asm_ppp CTA on the same SM
k_factors(DevSolveState *__restrict__ S, const double *__restrict__ Hp, FPtrs F, int eval_index) {
  __shared__ double sA[15 * 31];   // raw [J | r]
  __shared__ double sJ[15 * 31];   // whitened
  __shared__ double sdx[kDsMaxNp];
  __shared__ double sred[kFThreads / 32];
  if (S->sc.done) return;
  const int tid = threadIdx.x, O = S->sc.O, b = blockIdx.x;
  const double *xe = eval_index == 0 ? S->x : S->cand;
  if (b == 0 && tid == 0 && eval_index < 24) S->dbg[eval_index][12] = gtime_ns();
  if (b < O) {
    const bool imu = S->sc.imu_factor && S->pim_valid[b];
    for (int p = tid; p < 15 * 31; p += kFThreads) sA[p] = 0.0;
    __syncthreads();
    if (tid == 0 && imu) {
      double raw[15];
      imu_factor_raw(S->pim[b], x_pose(xe, b), x_sb(xe, b), x_pose(xe, b + 1), x_sb(xe, b + 1), raw, sA, 31);
      for (int a = 0; a < 15; ++a) sA[a * 31 + 30] = raw[a];
    }
    if (tid == 32 && S->sc.point_distance_factor) {
      double R[9], t[3];
      ppp_frame_terms_impl(x_pose(xe, 0), x_pose(xe, b + 1), xe + 16 * (O + 1), R, t, F.M + (size_t)b * kFMStride);
    }
    __syncthreads();
    if (!imu) return;
    const PimData &pim = S->pim[b];
    for (int p = tid; p < 15 * 31; p += kFThreads) {
      const int a = p / 31, c = p - a * 31;
      double s = 0;
      for (int k = a; k < 15; ++k) s += pim.sqrt_info[a][k] * sA[k * 31 + c];
      sJ[p] = s;
    }
    __syncthreads();
    double *out = F.imu + (size_t)b * kFImuStride;
    for (int p = tid; p < 931; p += kFThreads) {
      double s = 0;
      if (p < 900) {
        const int a = p / 30, c = p - a * 30;
#pragma unroll
        for (int k = 0; k < 15; ++k) s += sJ[k * 31 + a] * sJ[k * 31 + c];
      } else if (p < 930) {
        const int a = p - 900;
#pragma unroll
        for (int k = 0; k < 15; ++k) s += sJ[k * 31 + a] * sJ[k * 31 + 30];
      } else {
#pragma unroll
        for (int k = 0; k < 15; ++k) s += sJ[k * 31 + 30] * sJ[k * 31 + 30];
        s *= 0.5;
      }
      out[p] = s;
    }
    __syncthreads();
    if (tid == 0) stamp_max(S, eval_index, 13);
    return;
  }
  // ---- extrinsic PriorFactor CTA (applied only while the extrinsic is free)
  const int np = 15 * O + 6;
  if (b == O) {
    if (tid == 0 && S->sc.prior_factor) {
      double r[6], J[6][6];
      prior_factor_impl(V3(S->sc.ex0_pos), Q(S->sc.ex0_quat[3], S->sc.ex0_quat[0], S->sc.ex0_quat[1], S->sc.ex0_quat[2]), xe + 16 * (O + 1), r, J);
      double c = 0;
      for (int a = 0; a < 6; ++a) {
        double gs = 0;
        for (int k = 0; k < 6; ++k) gs += J[k][a] * r[k];
        F.ex[36 + a] = gs;
        for (int bb = 0; bb < 6; ++bb) { double s = 0; for (int k = 0; k < 6; ++k) s += J[k][a] * J[k][bb]; F.ex[a * 6 + bb] = s; }
        c += 0.5 * r[a] * r[a];
      }
      F.ex[42] = c;
      stamp_max(S, eval_index, 13);
    }
    return;
  }
  // ---- marginalisation prior, slice p of kFPriorCtas: rows r = p, p + kFPriorCtas, ... of Hp dx + bp and their share of the cost
  // (a single CTA needed 11 us for the 156 x 156 matrix-vector product: 20 dependent row passes per warp)
  if (!(S->sc.marginalization_factor && S->sc.prior_valid)) return;
  const int p = b - O - 1;
  if (tid < O) {
    pose_dx_dev(x_pose(xe, tid), S->x0_pose + 7 * tid, sdx + 15 * tid);
    for (int a = 0; a < 9; ++a) sdx[15 * tid + 6 + a] = x_sb(xe, tid)[a] - S->x0_sb[9 * tid + a];
  } else if (tid == O) {
    pose_dx_dev(xe + 16 * (O + 1), S->x0_ex, sdx + 15 * O);
  }
  __syncthreads();
  double part = 0;
  {
    const int w = warp_id(), l = lane_id();
    for (int r = p + kFPriorCtas * w; r < np; r += kFPriorCtas * (kFThreads / 32)) {
      double s = 0;
      for (int c = l; c < np; c += 32) s += Hp[(size_t)r * np + c] * sdx[c];
      s = warp_sum(s);
      if (l == 0) {
        const double bpr = S->bp[r];
        F.prior[r] = s + bpr;
        part += 2.0 * bpr * sdx[r] + sdx[r] * s;
      }
    }
  }
  if (lane_id() == 0) sred[warp_id()] = part;
  __syncthreads();
  if (tid == 0) {
    double tot = 0;
    for (int w = 0; w < kFThreads / 32; ++w) tot += sred[w];
    F.prior[kDsMaxNp + 1 + p] = tot;   // k_hpart adds the slices in order: F.prior[kDsMaxNp] = (c0 + sum) / 2
    stamp_max(S, eval_index, 13);
  }
}

// =====================================================================================================
// tiled Cholesky in shared memory
__device__ __forceinline__ int tile_off(int ib, int jb) { return (ib * (ib + 1) / 2 + jb) * 64; }
__device__ __forceinline__ int swz(int r, int c) { return r * 8 + (c ^ ((r & 2) << 1)); }

// Where tile (ib, jb) of the lower triangle lives: every phase that touches the Cholesky tiles addresses them through one
// of these two maps.  `tiles` is the CTA's own dynamic shared memory.
struct OneCta {   // k_step: all tiles packed row by row in the CTA's own shared memory (rows contiguous)
  static constexpr bool kCluster = false;
  static constexpr int kRowSlices = 7;    // 32-column slices of an Hpart row (n <= 224)
  static constexpr int kLidarLoads = 4;   // staged lidar operands per thread: O * 140 <= 4 * 512
  static constexpr int kBackWarps = 8;    // warps of the back substitution: 8 NB <= 256 rows
  template <class T> __device__ __forceinline__ static T *at(T *tiles, int ib, int jb) { return tiles + tile_off(ib, jb); }
  __device__ __forceinline__ static size_t local_doubles(int NB) { return (size_t)(NB * (NB + 1) / 2) * 64; }
  __device__ __forceinline__ static bool prof_fits(int, int) { return true; }
};

// Address of tile (ib, jb) under the map TP, in a function whose tile base is `tiles`.  A macro, not a call, so that for
// OneCta the expression is exactly the one the one-CTA kernels were written with (going through an inline function
// perturbed their instruction selection).
#define TILE(ib, jb) (TP::kCluster ? TP::at(tiles, ib, jb) : tiles + tile_off(ib, jb))

// k_step_x2 / k_chol_test_x2 (n <= 261, NB <= 33): rank 0 keeps the diagonal tiles (ib, ib) and the first sub-diagonal
// tiles (ib + 1, ib) - every tile the serial chain warp touches - and the remaining tiles of the odd tile rows; rank 1 holds
// the remaining tiles of the even tile rows.  Per CTA at NB = 33: rank 0 33 + 32 + 240 tiles (156 KiB) + the vectors, rank 1
// 256 tiles (128 KiB).  Layout (fixed, independent of NB), in tiles:
//   rank 0: [diagonal ib: 0..32][sub-diagonal (jb + 1, jb): 33..64][odd row ib = 2k + 1, jb <= ib - 2: 65 + k (k - 1) + jb]
//   rank 1: [even row ib = 2k, jb <= ib - 2: (k - 1)^2 + jb]
// Only rank 0's threads read or write tiles, so the CTA barriers that separate its phases order the remote accesses as well
// (the PTX memory model scopes a barrier by the threads that take part, not by where the location lives); rank 1's shared
// memory is live from the cluster barrier at kernel entry to the one at exit.
struct TwoCta {
  static constexpr bool kCluster = true;
  static constexpr int kRowSlices = 9;    // n <= 288
  static constexpr int kLidarLoads = 5;   // O * 140 <= 5 * 512
  static constexpr int kBackWarps = 9;    // 8 NB <= 288 rows
  static constexpr int kMaxNB = 33;
  static constexpr int kLocalTiles = 2 * kMaxNB - 1 + 240, kPeerTiles = 256;
  template <class T> __device__ __forceinline__ static T *at(T *tiles, int ib, int jb) {
    const int d = ib - jb, k = ib >> 1;
    if (d == 0) return tiles + 64 * ib;
    if (d == 1) return tiles + 64 * (kMaxNB + jb);
    if (ib & 1) return tiles + 64 * (2 * kMaxNB - 1 + k * (k - 1) + jb);
    return cg::this_cluster().map_shared_rank(tiles, 1) + 64 * ((k - 1) * (k - 1) + jb);
  }
  __device__ __forceinline__ static size_t local_doubles(int) { return (size_t)kLocalTiles * 64; }
  __device__ __forceinline__ static bool prof_fits(int slot, int cap) { return slot < cap; }
};

__device__ __forceinline__ void dmma884(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// Chain warp: in-place Cholesky of the diagonal tile (lower triangle), then its inverse: on return the tile holds inv(L)
// (lower) and zeros above.  ONE lane factors the 8 x 8 tile entirely in registers: per column the dependent chain is
// rsqrt -> multiply -> fused multiply-add (about 85 cycles), with no shuffle or shared-memory access on it - those go
// through the SM's memory pipe, which the update warps keep saturated (the row-per-lane variant with two shuffles per
// column takes 1.4k cycles alone but 2.6k beside them).  rsqrt(a_kk) = 1 / l_kk stays in registers, so the inverse needs no
// division; lanes 0-7 each solve L x = e_l for one column by right-looking substitution.
__device__ void diag_factor(double *T, int *s_ok) {
  const int l = lane_id();
  double dinv[8];
  if (l == 0) {
    double a[8][8];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c <= r; ++c) a[r][c] = T[swz(r, c)];
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const double d = a[k][k];
      if (!(d > 0.0) || !isfinite(d)) ok = false;
      const double inv = rsqrt(d);
      dinv[k] = inv;
      a[k][k] = d * inv;
#pragma unroll
      for (int i = k + 1; i < 8; ++i) a[i][k] *= inv;
#pragma unroll
      for (int i = k + 1; i < 8; ++i)
#pragma unroll
        for (int j = k + 1; j <= i; ++j) a[i][j] -= a[i][k] * a[j][k];
    }
    if (!ok) *s_ok = 0;
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c <= r; ++c) T[swz(r, c)] = a[r][c];
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) dinv[k] = __shfl_sync(0xffffffffu, dinv[k], 0);
  __syncwarp();
  double x[8], sacc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sacc[i] = (i == l) ? 1.0 : 0.0; x[i] = 0.0; }
  if (l < 8) {  // column l of inv(L)
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      x[k] = sacc[k] * dinv[k];       // zero for k < l
#pragma unroll
      for (int i = k + 1; i < 8; ++i) sacc[i] -= T[swz(i, k)] * x[k];
    }
  }
  __syncwarp();
  if (l < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) T[swz(i, l)] = x[i];
  }
  __syncwarp();
}

// clock64 ordered after a shared-memory value has arrived: a plain clock read right behind __syncthreads() captures the
// barrier's ISSUE time (BAR.SYNC.DEFER_BLOCKING), not its release
// clock64 read that really happens after v is available (v = a shared-memory value loaded behind a barrier): the read is
// control-dependent on v, so neither ptxas nor the issue logic can run it ahead of the load.  (A clock read that merely
// follows the barrier in program order, or "uses" v in a dead move, is issued while the warp still waits: round 2's first
// per-panel profile under-counted every panel by the time spent at the barriers.)
__device__ __forceinline__ long long clock_after(double v) {
  long long t = 0;
  if (__double_as_longlong(v) != 0x7ff8dead00000001LL) asm volatile("mov.u64 %0, %%clock64;" : "=l"(t) : : "memory");
  return t;
}

// Factors the tiled matrix in place (strictly-lower tiles: L; diagonal tiles: inv(L_kk)) and overwrites y (padded to
// 8 NB) with the solution of (L L^T) x = y.  Returns 1 on success; uniform over the CTA (and, since only rank 0 of a
// cluster calls it, over the cluster).  TwoCta: profile slots >= prof_cap are not written.
template <class TP>
__device__ int chol_solve_tiles(double *tiles, int NB, double *y, int *s_ok, long long *prof = nullptr, int prof_cap = 0) {
  const int tid = threadIdx.x, w = warp_id(), l = lane_id();
  const int fr = l >> 2, fq = l & 3;   // fragment row, fragment quad
  if (prof && tid == 0 && TP::prof_fits(4 * NB + 1, prof_cap)) prof[4 * NB + 1] = gtime_ns();
  if (tid == 0) *s_ok = 1;
  __syncthreads();
  // The serial chain (diagonal tiles) runs on the LAST warp: the issue arbiter favours the highest warp id of a
  // scheduler, so the chain is never starved by the seven update warps it shares its scheduler with.
  constexpr int kChainWarp = kDsWarps - 1;
  if (w == kChainWarp) diag_factor(TILE(0, 0), s_ok);
  __syncthreads();
  if (prof && w == kChainWarp && l == 0 && TP::prof_fits(4 * NB + 2, prof_cap)) prof[4 * NB + 2] = gtime_ns();
  for (int kb = 0; kb < NB; ++kb) {
    if (!*s_ok) break;
    const long long tp0 = clock_after(y[0]);
    const double *Li = TILE(kb, kb);   // inv(L_kk)
    const int m = NB - 1 - kb;
    // ---- panel solve: X = A inv(L)^T for the tiles below the diagonal; y_kb = inv(L) y_kb.  The chain warp takes the first
    // tile and at once applies it to the next diagonal tile, so that after the barrier it can start factoring immediately
    // (behind the barrier the same update would queue behind everybody else's shared-memory traffic: 850 cycles measured).
    const double b0 = Li[swz(fr, fq)], b1 = Li[swz(fr, fq + 4)];
    if (w == kChainWarp) {
      if (m > 0) {
        double *A = TILE(kb + 1, kb);
        const double a0 = A[swz(fr, fq)], a1 = A[swz(fr, fq + 4)];
        double d0 = 0.0, d1 = 0.0;
        dmma884(d0, d1, a0, b0);
        dmma884(d0, d1, a1, b1);
        *reinterpret_cast<double2 *>(A + swz(fr, 2 * fq)) = make_double2(d0, d1);
        __syncwarp();
        double *C = TILE(kb + 1, kb + 1);
        const double x0 = A[swz(fr, fq)], x1 = A[swz(fr, fq + 4)];
        double2 c = *reinterpret_cast<double2 *>(C + swz(fr, 2 * fq));
        dmma884(c.x, c.y, -x0, x0);
        dmma884(c.x, c.y, -x1, x1);
        *reinterpret_cast<double2 *>(C + swz(fr, 2 * fq)) = c;
      }
    } else {
      for (int t = 1 + w; t < m; t += kDsWarps - 1) {
        double *A = TILE(kb + 1 + t, kb);
        const double a0 = A[swz(fr, fq)], a1 = A[swz(fr, fq + 4)];
        double d0 = 0.0, d1 = 0.0;
        dmma884(d0, d1, a0, b0);
        dmma884(d0, d1, a1, b1);
        *reinterpret_cast<double2 *>(A + swz(fr, 2 * fq)) = make_double2(d0, d1);
      }
    }
    if (w == 0) {
      double v = 0.0;
      if (l < 8) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v += (k <= l) ? Li[swz(l, k)] * y[8 * kb + k] : 0.0;
      }
      __syncwarp();
      if (l < 8) y[8 * kb + l] = v;
    }
    __syncthreads();
    const long long tp1 = clock_after(y[8 * kb]);      // y_kb was written by warp 0 before the barrier: really after release
    if (prof && w == kChainWarp && l == 0 && TP::prof_fits(4 * kb + 3, prof_cap)) prof[4 * kb + 0] = tp1 - tp0;
    if (m == 0) break;
    // ---- trailing update C(i, j) -= X_i X_j^T, right-hand side rows, and the next diagonal tile one panel ahead
    const int ntile = m * (m + 1) / 2;
    if (w == kChainWarp) {
      double *C = TILE(kb + 1, kb + 1);
      const long long td0 = clock64();
      diag_factor(C, s_ok);
      if (prof && l == 0 && TP::prof_fits(4 * kb + 3, prof_cap)) { prof[4 * kb + 1] = gtime_ns(); prof[4 * kb + 2] = clock64() - td0; }
    } else if ((w & 3) != (kChainWarp & 3)) {
      // tile tasks p = 1 .. ntile - 1: tile (i, j) with p = i (i + 1) / 2 + j (p = 0 is the next diagonal tile: the chain warp's).
      // The warps that share the chain warp's scheduler (w % 4 == 3) take no tasks: their fp64 MMAs would queue in front of
      // every dependent fp64 operation of the chain (measured: the diagonal tile takes 4.9k cycles beside them, 2.0k alone).
      constexpr int kWorkers = kDsWarps - kDsWarps / 4;          // 12
      const int wi = w - (w >> 2);                               // dense index of this worker: 0 .. 11
      // Each worker takes a CONTIGUOUS range of the tile tasks (row-major over the lower triangle), so that the fragments of the
      // row tile X_i stay in registers while j runs along the row: the update is bound by shared-memory bandwidth (2 kB per tile:
      // two X fragments, C in and out), a cached row saves a quarter of it.
      const int ntask = ntile - 1;                               // tile tasks p = 1 .. ntile - 1
      const int per = (ntask + kWorkers - 1) / kWorkers;
      const int p0 = 1 + wi * per, p1 = min(ntile, p0 + per);
      if constexpr (!TP::kCluster) {
      if (p0 < p1) {
        int i = (int)((sqrt(8.0 * p0 + 1.0) - 1.0) * 0.5);
        while ((i + 1) * (i + 2) / 2 <= p0) ++i;
        while (i * (i + 1) / 2 > p0) --i;
        int j = p0 - i * (i + 1) / 2;
        const int o0 = swz(fr, fq), o1 = swz(fr, fq + 4), oc = swz(fr, 2 * fq);
        // The range is walked row segment by row segment with strength-reduced pointers (the generic tile_off / swizzle
        // arithmetic cost ~60 instructions per tile: with 4 warps per scheduler the update was issue bound, not MMA bound):
        // along a row the C tiles are contiguous (+64 doubles) and X_j advances by (kb + 2 + j) tiles.
        for (int p = p0; p < p1;) {
          const int jend = min(i, j + (p1 - p) - 1);
          const double *Xi = tiles + tile_off(kb + 1 + i, kb);
          const double a0 = -Xi[o0], a1 = -Xi[o1];
          double *Cp = tiles + tile_off(kb + 1 + i, kb + 1 + j) + oc;
          const double *xp = tiles + tile_off(kb + 1 + j, kb);
          int xinc = (kb + 2 + j) * 64;
          double x0 = xp[o0], x1 = xp[o1];
          double2 c = *reinterpret_cast<double2 *>(Cp);
#pragma unroll 2
          for (int jj = j; jj <= jend; ++jj) {
            const bool more = jj < jend;
            const double *xn = xp + xinc;
            double nx0 = 0.0, nx1 = 0.0;
            double2 nc = make_double2(0.0, 0.0);
            if (more) { nx0 = xn[o0]; nx1 = xn[o1]; nc = *reinterpret_cast<double2 *>(Cp + 64); }
            dmma884(c.x, c.y, a0, x0);
            dmma884(c.x, c.y, a1, x1);
            *reinterpret_cast<double2 *>(Cp) = c;
            Cp += 64; xp = xn; xinc += 64;
            x0 = nx0; x1 = nx1; c = nc;
          }
          p += jend - j + 1;
          j = 0; ++i;
        }
      }
      } else if (p0 < p1) {
        // TwoCta: the same walk, every tile address from the map (a row's tiles are spread over both CTAs)
        int i = (int)((sqrt(8.0 * p0 + 1.0) - 1.0) * 0.5);
        while ((i + 1) * (i + 2) / 2 <= p0) ++i;
        while (i * (i + 1) / 2 > p0) --i;
        int j = p0 - i * (i + 1) / 2;
        const int o0 = swz(fr, fq), o1 = swz(fr, fq + 4), oc = swz(fr, 2 * fq);
        for (int p = p0; p < p1;) {
          const int jend = min(i, j + (p1 - p) - 1);
          const double *Xi = TILE(kb + 1 + i, kb);
          const double a0 = -Xi[o0], a1 = -Xi[o1];
          double *Cp = TILE(kb + 1 + i, kb + 1 + j) + oc;
          const double *xp = TILE(kb + 1 + j, kb);
          double x0 = xp[o0], x1 = xp[o1];
          double2 c = *reinterpret_cast<double2 *>(Cp);
          for (int jj = j; jj <= jend; ++jj) {
            const bool more = jj < jend;
            double *Cn = Cp;
            double nx0 = 0.0, nx1 = 0.0;
            double2 nc = make_double2(0.0, 0.0);
            if (more) {
              const double *xn = TILE(kb + 2 + jj, kb);
              Cn = TILE(kb + 1 + i, kb + 2 + jj) + oc;
              nx0 = xn[o0]; nx1 = xn[o1]; nc = *reinterpret_cast<double2 *>(Cn);
            }
            dmma884(c.x, c.y, a0, x0);
            dmma884(c.x, c.y, a1, x1);
            *reinterpret_cast<double2 *>(Cp) = c;
            Cp = Cn; x0 = nx0; x1 = nx1; c = nc;
          }
          p += jend - j + 1;
          j = 0; ++i;
        }
      }
      // right-hand side rows of tile-row r (r = 0 .. m - 1), one per worker in turn
      if (l < 8) {
        for (int r = wi; r < m; r += kWorkers) {
          const int ib = kb + 1 + r;
          const double *X = TILE(ib, kb);
          double s = 0.0;
#pragma unroll
          for (int k = 0; k < 8; ++k) s += X[swz(l, k)] * y[8 * kb + k];
          y[8 * ib + l] -= s;
        }
      }
    }
    __syncthreads();
    if (prof && w == kChainWarp && l == 0 && TP::prof_fits(4 * kb + 3, prof_cap)) prof[4 * kb + 3] = clock_after(y[8 * (kb + 1)]) - tp1;
  }
  __syncthreads();
  const int ok = *s_ok;
  if (!ok) return 0;
  const long long tb0 = clock64();
  if (prof && w == kChainWarp && l == 0 && TP::prof_fits(4 * NB + 3, prof_cap)) prof[4 * NB + 3] = gtime_ns();
  // ---- back substitution L^T x = y over the tiles in reverse.  Only the first kBackWarps warps take part (8 NB rows): the
  // 8 threads of tile-row jb turn their finished y into x = inv(L_jj)^T y (they share a warp), one named barrier
  // publishes x, then every thread of the rows above subtracts its tile's contribution.
  if (w < TP::kBackWarps) {
    for (int jb = NB - 1; jb >= 0; --jb) {
      if ((tid >> 3) == jb) {
        const double *Li = TILE(jb, jb);
        const int c = tid & 7;
        __syncwarp(0xffu << (l & 24));
        double v0 = 0.0, v1 = 0.0;
#pragma unroll
        for (int r = 0; r < 8; r += 2) {
          v0 += (r >= c) ? Li[swz(r, c)] * y[8 * jb + r] : 0.0;
          v1 += (r + 1 >= c) ? Li[swz(r + 1, c)] * y[8 * jb + r + 1] : 0.0;
        }
        __syncwarp(0xffu << (l & 24));
        y[8 * jb + c] = v0 + v1;
      }
      double lt[8];   // this thread's column of tile (jb, ib): independent of x, fetched before the barrier
      if (tid < 8 * jb) {
        const double *Lt = TILE(jb, tid >> 3);
#pragma unroll
        for (int r = 0; r < 8; ++r) lt[r] = Lt[swz(r, tid & 7)];
      }
      asm volatile("bar.sync 1, %0;" :: "n"(32 * TP::kBackWarps) : "memory");
      if (tid < 8 * jb) {
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int r = 0; r < 8; r += 2) { s0 += lt[r] * y[8 * jb + r]; s1 += lt[r + 1] * y[8 * jb + r + 1]; }
        y[tid] -= s0 + s1;
      }
    }
  }
  __syncthreads();
  if (prof && tid == 0 && TP::prof_fits(4 * NB + 4, prof_cap)) { const long long te = clock_after(y[0]); prof[4 * NB] = te - tb0; prof[4 * NB + 4] = gtime_ns(); }
  return 1;
}

// =====================================================================================================
// element-wise gather of the normal equations
struct GatherCtx {
  int O, n, oe, np;
  bool ex_free, prior, lidar, imu, ex_prior;
  const double *Hp, *Fimu, *Fprior, *Fex, *G, *G0;
  const double *zero;     // a 0.0 in shared memory: the target of absent terms
  const int *pim_valid;   // shared-memory copy
};

__device__ __forceinline__ int prior_index(const GatherCtx &c, int a) {   // tangent -> prior canonical index, or -1
  if (a < 15 * c.O) return a;
  if (a >= c.oe) return c.ex_free ? 15 * c.O + (a - c.oe) : -1;
  return -1;
}
// lidar block id: 0 pose_0, i (1..O) pose_i, O + 1 extrinsic, -1 none; sub = index inside the 6-block
__device__ __forceinline__ int lidar_block(const GatherCtx &c, int a, int &sub) {
  if (a >= c.oe) { sub = a - c.oe; return c.ex_free ? c.O + 1 : -1; }
  const int k = a / 15, w = a - 15 * k;
  if (w >= 6) return -1;
  sub = w;
  return k;
}

// All contributions are looked up first and loaded together (one memory round trip per element instead of a chain of
// conditional loads); absent terms read a zero, so the summation order prior + lidar + imu + imu + extrinsic prior is fixed.
__device__ __forceinline__ double h_elem(const GatherCtx &c, int a, int b) {   // a >= b, both < n
  if (!c.ex_free && a >= c.oe) return (a == b) ? 1.0 : 0.0;      // frozen extrinsic: identity block, zero gradient
  const double *p0 = c.zero, *p1 = c.zero, *p2 = c.zero, *p3 = c.zero, *p4 = c.zero;
  if (c.prior) {
    const int pa = prior_index(c, a), pb = prior_index(c, b);
    if (pa >= 0 && pb >= 0) p0 = c.Hp + (size_t)pa * c.np + pb;
  }
  if (c.lidar) {
    int sa, sb;
    const int ba = lidar_block(c, a, sa), bb = lidar_block(c, b, sb);
    if (ba >= 0 && bb >= 0) {
      const bool sha = (ba == 0 || ba == c.O + 1), shb = (bb == 0 || bb == c.O + 1);
      if (sha && shb) {
        p1 = c.G0 + ((ba == 0 ? 0 : 6) + sa) * 12 + (bb == 0 ? 0 : 6) + sb;
      } else if (!sha && !shb) {
        if (ba == bb) p1 = c.G + (size_t)(ba - 1) * kFGStride + (6 + sa) * 18 + 6 + sb;
      } else {
        const int i = sha ? bb : ba;                              // the frame-specific one
        const int ra = sha ? (ba == 0 ? 0 : 12) + sa : 6 + sa, rb = shb ? (bb == 0 ? 0 : 12) + sb : 6 + sb;
        p1 = c.G + (size_t)(i - 1) * kFGStride + ra * 18 + rb;
      }
    }
  }
  if (c.imu && a < c.oe) {
    const int ka = a / 15;
    {
      const int k = ka, lb = b - 15 * k;
      if (k < c.O && c.pim_valid[k] && lb >= 0) p2 = c.Fimu + (size_t)k * kFImuStride + (a - 15 * k) * 30 + lb;
    }
    {
      const int k = ka - 1, lb = b - 15 * k;
      if (k >= 0 && k < c.O && c.pim_valid[k] && lb >= 0) p3 = c.Fimu + (size_t)k * kFImuStride + (a - 15 * k) * 30 + lb;
    }
  }
  if (c.ex_prior && b >= c.oe) p4 = c.Fex + (a - c.oe) * 6 + (b - c.oe);
  const double v0 = *p0, v1 = *p1, v2 = *p2, v3 = *p3, v4 = *p4;
  return (((v0 + v1) + v2) + v3) + v4;
}

__device__ __forceinline__ double g_elem(const GatherCtx &c, int a) {
  if (!c.ex_free && a >= c.oe) return 0.0;
  const double *p0 = c.zero, *p1 = c.zero, *p2 = c.zero, *p3 = c.zero, *p4 = c.zero;
  if (c.prior) { const int pa = prior_index(c, a); if (pa >= 0) p0 = c.Fprior + pa; }
  if (c.lidar) {
    int sa;
    const int ba = lidar_block(c, a, sa);
    if (ba == 0 || ba == c.O + 1) p1 = c.G0 + 144 + (ba == 0 ? 0 : 6) + sa;
    else if (ba > 0) p1 = c.G + (size_t)(ba - 1) * kFGStride + 324 + 6 + sa;
  }
  if (c.imu && a < c.oe) {
    const int ka = a / 15;
    if (ka < c.O && c.pim_valid[ka]) p2 = c.Fimu + (size_t)ka * kFImuStride + 900 + (a - 15 * ka);
    if (ka >= 1 && ka - 1 < c.O && c.pim_valid[ka - 1]) p3 = c.Fimu + (size_t)(ka - 1) * kFImuStride + 900 + (a - 15 * (ka - 1));
  }
  if (c.ex_prior && a >= c.oe) p4 = c.Fex + 36 + (a - c.oe);
  const double v0 = *p0, v1 = *p1, v2 = *p2, v3 = *p3, v4 = *p4;
  return (((v0 + v1) + v2) + v3) + v4;
}

// Lidar-independent share of the normal equations at the evaluated state, element-wise into Hpart (lower triangle,
// unscaled) and gpart: prior + ImuFactors + extrinsic PriorFactor.  Runs on many CTAs beside asm_ppp (second stream), so
// that the single-CTA step kernel only has to add the lidar blocks while it streams the rows into its Cholesky tiles.
// hflags records the structure (free extrinsic, prior in use) the gather assumed: the convergence gates of evaluation 0
// can still change it, in which case k_step falls back to its own full gather.
__global__ void __launch_bounds__(256)
k_hpart(DevSolveState *__restrict__ S, const double *__restrict__ Hp, FPtrs F, double *__restrict__ Hpart, double *__restrict__ HpartT, int eval_index) {
  __shared__ double s_zero;
  __shared__ int s_pimv[kMaxOpt];
  if (S->sc.done) return;
  const int O = S->sc.O, n = S->sc.n;
  if (threadIdx.x < kMaxOpt) s_pimv[threadIdx.x] = S->pim_valid[threadIdx.x];
  if (threadIdx.x == 32) s_zero = 0.0;
  __syncthreads();
  GatherCtx gc;
  gc.O = O; gc.n = n; gc.oe = 15 * (O + 1); gc.np = 15 * O + 6;
  gc.ex_free = S->sc.ex_free != 0; gc.prior = S->sc.marginalization_factor && S->sc.prior_valid; gc.lidar = false;
  gc.imu = S->sc.imu_factor != 0; gc.ex_prior = gc.ex_free && S->sc.prior_factor;
  gc.Hp = Hp; gc.Fimu = F.imu; gc.Fprior = F.prior; gc.Fex = F.ex; gc.G = nullptr; gc.G0 = nullptr; gc.pim_valid = s_pimv; gc.zero = &s_zero;
  double *gpart = Hpart + (size_t)n * n;
  if (eval_index == 0) {
    for (int a = blockIdx.x; a < n; a += gridDim.x) {
      for (int b = threadIdx.x; b <= a; b += blockDim.x) Hpart[(size_t)a * n + b] = h_elem(gc, a, b);
      if (threadIdx.x == blockDim.x - 1) gpart[a] = g_elem(gc, a);
    }
  } else {
    // the Jacobi scaling is fixed since evaluation 0: write the scaled entries straight in the step kernel's swizzled tile
    // layout (identity on the padding rows), so that k_step fetches its Cholesky tiles with one coalesced copy
    const int NP = ((n + 7) / 8) * 8;
    for (int a = blockIdx.x; a < NP; a += gridDim.x) {
      if (a < n) {
        const double sa = S->scale[a];
        for (int b = threadIdx.x; b <= a; b += blockDim.x)
          HpartT[tile_off(a >> 3, b >> 3) + swz(a & 7, b & 7)] = h_elem(gc, a, b) * sa * S->scale[b];
        if (threadIdx.x == blockDim.x - 1) gpart[a] = g_elem(gc, a);
      } else {
        for (int b = threadIdx.x; b <= a; b += blockDim.x) HpartT[tile_off(a >> 3, b >> 3) + swz(a & 7, b & 7)] = (a == b) ? 1.0 : 0.0;
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    gpart[n] = gc.ex_free ? 1.0 : 0.0;
    gpart[n + 1] = gc.prior ? 1.0 : 0.0;
    gpart[n + 2] = eval_index == 0 ? 0.0 : 1.0;   // which of Hpart / HpartT this launch wrote
    if (gc.prior) {   // cost of the marginalisation prior from the slices of k_factors, in slice order
      double tot = 0;
      for (int p = 0; p < kFPriorCtas; ++p) tot += F.prior[kDsMaxNp + 1 + p];
      F.prior[kDsMaxNp] = 0.5 * (S->c0 + tot);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp_max(S, eval_index, 14);
}

// lidar share of H(a, b), a >= b (zero when either index is not a pose / free-extrinsic entry)
__device__ __forceinline__ double lidar_h(const GatherCtx &c, int ba, int sa, int b) {
  int sb;
  const int bb = lidar_block(c, b, sb);
  if (bb < 0) return 0.0;
  const bool sha = (ba == 0 || ba == c.O + 1), shb = (bb == 0 || bb == c.O + 1);
  if (sha && shb) return c.G0[((ba == 0 ? 0 : 6) + sa) * 12 + (bb == 0 ? 0 : 6) + sb];
  if (!sha && !shb) return ba == bb ? c.G[(size_t)(ba - 1) * kFGStride + (6 + sa) * 18 + 6 + sb] : 0.0;
  const int i = sha ? bb : ba;
  const int ra = sha ? (ba == 0 ? 0 : 12) + sa : 6 + sa, rb = shb ? (bb == 0 ? 0 : 12) + sb : 6 + sb;
  return c.G[(size_t)(i - 1) * kFGStride + ra * 18 + rb];
}
__device__ __forceinline__ double lidar_g(const GatherCtx &c, int ba, int sa) {
  if (ba == 0 || ba == c.O + 1) return c.G0[144 + (ba == 0 ? 0 : 6) + sa];
  return c.G[(size_t)(ba - 1) * kFGStride + 324 + 6 + sa];
}

// G_i = M_i^T S_gg M_i (18 x 18), M_i^T S_gr (18) per frame, and the blocks shared by all frames (pose_0 / extrinsic rows
// and columns, 12 x 12 + 12) summed in frame order.  scratch: O * 108 doubles of shared memory.
// G_i = M_i^T S_i M_i (18 x 18 + 18 gradient terms per frame) and the block G0 shared by pose_0 and the extrinsic.  The inputs
// (M_i: 108 doubles, S_i: 29) are staged in shared memory first and every product runs from there: the three phases used to
// fetch their operands from global memory one dependent round trip after the other (4.8 us for 10 frames).
// scratch: >= O * (108 + 32 + 108 + 342) doubles of shared memory (the Cholesky tiles are not in use yet).
template <int kLoads>
__device__ void lidar_blocks(int O, const double *__restrict__ Sblk, const double *__restrict__ FM, double *G, double *G0, double *scratch, long long *marks = nullptr) {
  const int tid = threadIdx.x, T = blockDim.x;
  if (marks && tid == 0) marks[0] = clock64();
  double *sM = scratch, *sS = sM + O * 108, *sSM = sS + O * 32, *sG = sSM + O * 108;
  {   // all of a thread's loads are issued before the first store (O * 140 <= kLoads * 512)
    double v[kLoads];
    int dst[kLoads];
#pragma unroll
    for (int k = 0; k < kLoads; ++k) {
      const int p = tid + k * T;
      dst[k] = -1; v[k] = 0.0;
      if (p < O * 140) {
        const int i = p / 140, q = p - i * 140;
        if (q < 108) { dst[k] = i * 108 + q; v[k] = FM[(size_t)i * kFMStride + q]; }
        else if (q < 108 + 29) { dst[k] = O * 108 + i * 32 + (q - 108); v[k] = Sblk[i * kAsmStride + (q - 108)]; }
      }
    }
#pragma unroll
    for (int k = 0; k < kLoads; ++k) if (dst[k] >= 0) scratch[dst[k]] = v[k];
  }
  __syncthreads();
  if (marks && threadIdx.x == 0) marks[1] = clock_after(scratch[0]);
  for (int p = tid; p < O * 108; p += T) {     // SM_i = S_gg M_i (6 x 18)
    const int i = p / 108, q = p - i * 108, a = q / 18, c = q - a * 18;
    const double *Sb = sS + i * 32, *M = sM + i * 108;
    double s = 0;
#pragma unroll
    for (int b = 0; b < 6; ++b) s += Sb[a < b ? s_idx(a, b) : s_idx(b, a)] * M[b * 18 + c];
    sSM[p] = s;
  }
  __syncthreads();
  if (marks && threadIdx.x == 0) marks[2] = clock_after(scratch[0]);
  // G_i = M_i^T (S_gg M_i): an (18 x 6)(6 x 18) product per frame - on the fp64 tensor path (DMMA m8n8k4): 3 x 3 output tiles of
  // 8 x 8 per frame, K = 6 padded to 8 (two k-steps), one warp per tile.  (As scalar code - 6 multiply-adds per output, every
  // operand from shared memory - this phase was shared-memory-bandwidth bound: 4.0k cycles for 10 frames.)
  {
    const int w = warp_id(), l = lane_id(), fr = l >> 2, fq = l & 3;
    for (int task = w; task < O * 9; task += kDsWarps) {
      const int i = task / 9, t9 = task - i * 9, mt = t9 / 3, nt = t9 - mt * 3;
      const double *M = sM + i * 108, *SM = sSM + i * 108;
      const int m = 8 * mt + fr, nn = 8 * nt + fr;
      double d0 = 0.0, d1 = 0.0;
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const int k = 4 * kk + fq;
        const double a = (k < 6 && m < 18) ? M[k * 18 + m] : 0.0;      // A[m][k] = M^T[m][k]
        const double b = (k < 6 && nn < 18) ? SM[k * 18 + nn] : 0.0;   // B[k][n] = (S M)[k][n]
        dmma884(d0, d1, a, b);
      }
      const int n0 = 8 * nt + 2 * fq;
      if (m < 18) {
        if (n0 < 18) { sG[i * 342 + m * 18 + n0] = d0; G[(size_t)i * kFGStride + m * 18 + n0] = d0; }
        if (n0 + 1 < 18) { sG[i * 342 + m * 18 + n0 + 1] = d1; G[(size_t)i * kFGStride + m * 18 + n0 + 1] = d1; }
      }
    }
  }
  for (int p = tid; p < O * 18; p += T) {   // gradient terms M_i^T S_gr
    const int i = p / 18, a = p - i * 18;
    const double *M = sM + i * 108, *Sb = sS + i * 32;
    double v = 0;
#pragma unroll
    for (int k = 0; k < 6; ++k) v += M[k * 18 + a] * Sb[s_idx(k, 6)];
    sG[i * 342 + 324 + a] = v;
    G[(size_t)i * kFGStride + 324 + a] = v;
  }
  __syncthreads();
  if (marks && threadIdx.x == 0) marks[3] = clock_after(scratch[0]);
  for (int p = tid; p < 156; p += T) {
    double s = 0;
    if (p < 144) {
      const int ra = p / 12, rb = p - ra * 12;
      const int a = ra < 6 ? ra : ra + 6, b = rb < 6 ? rb : rb + 6;
      for (int i = 0; i < O; ++i) s += sG[i * 342 + a * 18 + b];
    } else {
      const int ra = p - 144, a = ra < 6 ? ra : ra + 6;
      for (int i = 0; i < O; ++i) s += sG[i * 342 + 324 + a];
    }
    G0[p] = s;
  }
  __syncthreads();
}

// y = H v with H the symmetric matrix whose lower triangle sits in the (unfactored) tiles; v, y in shared memory.
// Two threads per row, each over every other column; the tile address advances incrementally along the row / down the
// column.  OneCta: n <= blockDim.x / 2.  TwoCta: rows a and a + blockDim.x / 2, every tile address from the map.
template <class TP>
__device__ void symv_tiles(const double *tiles, int n, const double *v, double *y) {
  if constexpr (TP::kCluster) {
    const int q = threadIdx.x & 1;
    for (int a0 = 0; a0 < n; a0 += blockDim.x >> 1) {   // uniform trip count: the shuffle below has every lane
      const int a = a0 + (threadIdx.x >> 1);
      double s0 = 0.0, s1 = 0.0;
      if (a < n) {
        const int ta = a >> 3, ra = a & 7;
        for (int jb = 0; jb < ta; ++jb) {
          const double *row = TILE(ta, jb);
#pragma unroll
          for (int c = 0; c < 8; c += 4) {
            s0 += row[swz(ra, c + q)] * v[8 * jb + c + q];
            s1 += row[swz(ra, c + 2 + q)] * v[8 * jb + c + 2 + q];
          }
        }
        const double *row = TILE(ta, ta);
        for (int c = q; c <= ra; c += 2) s0 += row[swz(ra, c)] * v[8 * ta + c];
        for (int r = ra + 1 + q; r < 8 && 8 * ta + r < n; r += 2) s1 += row[swz(r, ra)] * v[8 * ta + r];
        const int NB = (n + 7) >> 3;
        for (int ib = ta + 1; ib < NB; ++ib) {
          const double *col = TILE(ib, ta);
#pragma unroll
          for (int r = 0; r < 8; r += 4) {
            s0 += col[swz(r + q, ra)] * v[8 * ib + r + q];
            s1 += col[swz(r + 2 + q, ra)] * v[8 * ib + r + 2 + q];
          }
        }
      }
      double s = s0 + s1;
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if (a < n && q == 0) y[a] = s;
    }
    __syncthreads();
    return;
  }
  const int a = threadIdx.x >> 1, q = threadIdx.x & 1;
  double s0 = 0.0, s1 = 0.0;
  if (a < n) {
    const int ta = a >> 3, ra = a & 7;
    const double *row = tiles + tile_off(ta, 0);            // tiles (ta, jb), jb = 0 .. ta: contiguous, 64 doubles apart
    for (int jb = 0; jb < ta; ++jb, row += 64) {
#pragma unroll
      for (int c = 0; c < 8; c += 4) {
        s0 += row[swz(ra, c + q)] * v[8 * jb + c + q];
        s1 += row[swz(ra, c + 2 + q)] * v[8 * jb + c + 2 + q];
      }
    }
    for (int c = q; c <= ra; c += 2) s0 += row[swz(ra, c)] * v[8 * ta + c];               // diagonal tile, lower part
    for (int r = ra + 1 + q; r < 8 && 8 * ta + r < n; r += 2) s1 += row[swz(r, ra)] * v[8 * ta + r];   // its mirror
    const int NB = (n + 7) >> 3;
    for (int ib = ta + 1; ib < NB; ++ib) {                                                  // column ra of the tiles below
      const double *col = tiles + tile_off(ib, ta);
#pragma unroll
      for (int r = 0; r < 8; r += 4) {
        s0 += col[swz(r + q, ra)] * v[8 * ib + r + q];
        s1 += col[swz(r + 2 + q, ra)] * v[8 * ib + r + 2 + q];
      }
    }
  }
  double s = s0 + s1;
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  if (a < n && q == 0) y[a] = s;
  __syncthreads();
}

// block-wide copy of a tile set (ndoubles = tiles x 64) between global and shared memory, 16 bytes per access, eight in flight
__device__ __forceinline__ void copy_tiles(double *__restrict__ dst, const double *__restrict__ src, int ndoubles) {
  const int n2 = ndoubles >> 1, T = blockDim.x;
  const double2 *s2 = reinterpret_cast<const double2 *>(src);
  double2 *d2 = reinterpret_cast<double2 *>(dst);
  int k = threadIdx.x;
  for (; k + 7 * T < n2; k += 8 * T) {
    double2 v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = s2[k + q * T];
#pragma unroll
    for (int q = 0; q < 8; ++q) d2[k + q * T] = v[q];
  }
  for (; k < n2; k += T) d2[k] = s2[k];
}
// Copy between a global tile set in the canonical layout (tile_off) and the tiles where TP keeps them.  OneCta: one flat
// copy.  TwoCta: the same 16-byte accesses, eight in flight, each shared-memory address from the map.
__device__ __forceinline__ int tile_row(int t) {   // ib of the canonical tile index t = ib (ib + 1) / 2 + jb
  int ib = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((ib + 1) * (ib + 2) / 2 <= t) ++ib;
  while (ib * (ib + 1) / 2 > t) --ib;
  return ib;
}
template <class TP> __device__ __forceinline__ double2 *tile_vec(double *tiles, int k) {   // 16-byte word k of the canonical set
  const int t = k >> 5, ib = tile_row(t);
  return reinterpret_cast<double2 *>(TILE(ib, t - ib * (ib + 1) / 2)) + (k & 31);
}
template <class TP, bool kLoad>
__device__ __forceinline__ void copy_tiles_map(double *tiles, double *glob, int ntd) {   // ntd = tiles x 64
  if constexpr (!TP::kCluster) {
    if (kLoad) copy_tiles(tiles, glob, ntd); else copy_tiles(glob, tiles, ntd);
  } else {
    const int n2 = ntd >> 1, T = blockDim.x;
    double2 *g2 = reinterpret_cast<double2 *>(glob);
    int k = threadIdx.x;
    for (; k + 7 * T < n2; k += 8 * T) {
      double2 v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = kLoad ? g2[k + q * T] : *tile_vec<TP>(tiles, k + q * T);
#pragma unroll
      for (int q = 0; q < 8; ++q) { if (kLoad) *tile_vec<TP>(tiles, k + q * T) = v[q]; else g2[k + q * T] = v[q]; }
    }
    for (; k < n2; k += T) { if (kLoad) *tile_vec<TP>(tiles, k) = g2[k]; else g2[k] = *tile_vec<TP>(tiles, k); }
  }
}
// (re)load the pure scaled H of the current x (tile layout, saved by the evaluation that built it)
template <class TP>
__device__ void refill_tiles(double *tiles, const double *__restrict__ HsT, int ntd) {
  copy_tiles_map<TP, true>(tiles, const_cast<double *>(HsT), ntd);
  __syncthreads();
}

__device__ __noinline__ void write_terms(int O, const double *xe, double *Rt) {
  double M[108];
  ppp_frame_terms_impl(x_pose(xe, 0), x_pose(xe, threadIdx.x + 1), xe + 16 * (O + 1), Rt + threadIdx.x * kAsmRtStride,
                       Rt + threadIdx.x * kAsmRtStride + 9, M);
}

#define DS_MARK(k) do { if (tid == 0 && eval_index < 24) S->dbg[eval_index][k] = clock64(); } while (0)

struct StepShared {
  double sred[100];
  double zero;
  DevScalars sc;
  int flag[4], ok, pim_valid[kMaxOpt];
};

template <class TP>
__device__ void step_body(DevSolveState *S, StepShared &sh, double *dsm, double *Hs, const double *__restrict__ Hp, double *H0, double *g0,
                          const double *__restrict__ Sblk, FPtrs F, const double *__restrict__ Hpart, const double *__restrict__ HpartT, double *Rt,
                          int eval_index) {
  DevScalars &sc = sh.sc;
  double *sred = sh.sred;
  int *s_flag = sh.flag;
  int &s_ok = sh.ok;
  const int tid = threadIdx.x, T = blockDim.x;
  if (tid == 0 && eval_index < 24) { for (int k = 0; k < 12; ++k) S->dbg[eval_index][k] = 0; S->dbg[eval_index][0] = gtime_ns(); }
  DS_MARK(1);
  const int O = sc.O, n = sc.n;
  const int NB = (n + 7) / 8, NP = NB * 8, ntd = (NB * (NB + 1) / 2) * 64;
  double *tiles = dsm;
  double *v_g = dsm + TP::local_doubles(NB);   // scaled gradient of the current x
  double *v_scale = v_g + NP, *v_diag = v_scale + NP, *v_grad = v_diag + NP, *v_gn = v_grad + NP, *v_step = v_gn + NP;
  double *v_tmp = v_step + NP, *v_y = v_tmp + NP, *v_hsg = v_y + NP;
  const double min_diagonal = 1e-6, max_diagonal = 1e32, min_mu = 1e-8, max_mu = 1.0, mu_factor = 10.0;
  const double initial_radius = 1e4, max_radius = 1e16, min_radius = 1e-32, min_relative_decrease = 1e-3;
  const double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
  const int xdim = 16 * (O + 1) + 7;
  const int oe = 15 * (O + 1), np = 15 * O + 6;
  double *G = F.G, *G0 = F.G + (size_t)kMaxOpt * kFGStride;

  // persistent vectors: global -> shared
  for (int i = tid; i < NP; i += T) {
    const bool in = i < n;
    v_g[i] = in ? S->g[i] : 0.0; v_scale[i] = in ? S->scale[i] : 1.0; v_diag[i] = in ? S->diagonal[i] : 1.0;
    v_grad[i] = in ? S->gradient[i] : 0.0; v_gn[i] = in ? S->gn[i] : 0.0; v_hsg[i] = in ? S->hsg[i] : 0.0;
  }
  __syncthreads();

  // ---------------- cost of the evaluated state and the verdict ----------------
  int build = 0;   // 1: (re)build H, g at the evaluated state and make it the current point
  int tiles_ready = 0;      // the gather below leaves the pure scaled H in the Cholesky tiles
  if (warp_id() == 0) {   // cost components: lane i fetches frame i's terms, summed in frame order by lane 0
    const int l = lane_id();
    double cp = (l < O && sc.point_distance_factor) ? 0.5 * Sblk[l * kAsmStride + 28] : 0.0;
    double ci = (l < O && sc.imu_factor && sh.pim_valid[l]) ? F.imu[(size_t)l * kFImuStride + 930] : 0.0;
    double c_ppp = 0, c_pim = 0;
    for (int i = 0; i < O; ++i) { c_ppp += __shfl_sync(0xffffffffu, cp, i); c_pim += __shfl_sync(0xffffffffu, ci, i); }
    if (l == 0) {
    const double c_marg = (sc.marginalization_factor && sc.prior_valid) ? F.prior[kDsMaxNp] : 0.0;
    sred[90] = c_ppp; sred[91] = c_pim; sred[92] = c_marg;
    if (eval_index == 0 && !sc.skip_gates) {
      // residuals before optimisation + gates (Estimator.cc:1924-1985)
      sc.cost_ppp = c_ppp; sc.cost_pim = c_pim; sc.cost_marg = c_marg;
      int turn_off = 1;
      if (sc.imu_factor) turn_off = c_pim > 1e3;
      sc.turn_off = turn_off;
      const double ratio = c_marg / (c_ppp + c_pim);
      if (!sc.convergence_flag && !turn_off && ratio <= 2 && ratio != 0) sc.convergence_flag = 1;
      if (!sc.convergence_flag) { sc.ex_free = 0; sc.prior_valid = 0; }
    }
    }
  }
  __syncthreads();
  const bool ex_free = sc.ex_free != 0;
  const bool use_prior = sc.marginalization_factor && sc.prior_valid;
  const bool ex_prior = ex_free && sc.prior_factor;
  const double cost_eval = sred[90] + sred[91] + (use_prior ? sred[92] : 0.0) + (ex_prior ? F.ex[42] : 0.0);
  const int xd = ex_free ? xdim : xdim - 7;
  if (eval_index == 0) {
    build = 1;
  } else {
    double sn = 0, dummy1 = 0, dummy2 = 0;
    for (int i = tid; i < xd; i += T) { const double d = S->x[i] - S->cand[i]; sn += d * d; }
    block_sum3(sn, dummy1, dummy2, sred);
    if (tid == 0) {
      double cand_cost = cost_eval;
      if (!isfinite(cand_cost)) cand_cost = 1e300;
      sc.cand_cost = cand_cost;
      sc.evaluations += 1;
      int verdict = 0;  // 0 reject, 1 accept, 2 terminate (converged)
      const double cost_change = sc.x_cost - cand_cost;
      if (sqrt(sn) <= parameter_tolerance * (sc.x_norm + parameter_tolerance)) { verdict = 2; sc.termination = 1; }
      else if (fabs(cost_change) <= function_tolerance * sc.x_cost) { verdict = 2; sc.termination = 1; }
      else {
        const double rd = cost_change / sc.model_cost_change;
        if (rd > min_relative_decrease) {
          verdict = 1;
          sc.x_cost = cand_cost;
          sc.successful += 1;
          if (rd < 0.25) sc.radius *= 0.5;
          if (rd > 0.75) sc.radius = fmin(max_radius, fmax(sc.radius, 3.0 * sc.dogleg_step_norm));
          sc.mu = fmax(min_mu, 2.0 * sc.mu / mu_factor);
          sc.reuse = 0;
        } else {
          sc.radius *= 0.5;
          sc.reuse = 1;
        }
      }
      s_flag[1] = verdict;
    }
    __syncthreads();
    const int verdict = s_flag[1];
    if (verdict == 2) { if (tid == 0) sc.done = 1; return; }
    build = verdict == 1;
    if (build) {
      for (int p = tid; p < xdim; p += T) S->x[p] = S->cand[p];
      __syncthreads();
    }
  }

  DS_MARK(2);
  GatherCtx gc;
  gc.O = O; gc.n = n; gc.oe = oe; gc.np = np;
  gc.ex_free = ex_free; gc.prior = use_prior; gc.lidar = sc.point_distance_factor != 0; gc.imu = sc.imu_factor != 0; gc.ex_prior = ex_prior;
  gc.Hp = Hp; gc.Fimu = F.imu; gc.Fprior = F.prior; gc.Fex = F.ex; gc.G = G; gc.G0 = G0; gc.pim_valid = sh.pim_valid; gc.zero = &sh.zero;

  if (build) {
    // ---------------- normal equations at the new current point ----------------
    if (gc.lidar) lidar_blocks<TP::kLidarLoads>(O, Sblk, F.M, G, G0, tiles, eval_index == 2 ? &S->dbg[16][0] : nullptr);
    DS_MARK(3);
    // unscaled diagonal, gradient; Jacobi scaling is fixed at iteration zero
    // k_hpart's gather is usable when it assumed the structure that is in force now (the gates may have changed it)
    const double *gpart = Hpart + (size_t)n * n;
    const bool fast = (gpart[n] != 0.0) == ex_free && (gpart[n + 1] != 0.0) == use_prior;
    double gm = 0, xn = 0;
    for (int a = tid; a < n; a += T) {
      int sa = 0;
      const int ba = (fast && gc.lidar) ? lidar_block(gc, a, sa) : -1;
      const double ga = fast ? gpart[a] + (ba >= 0 ? lidar_g(gc, ba, sa) : 0.0) : g_elem(gc, a);
      gm = fmax(gm, fabs(ga));
      if (eval_index == 0) {
        const double haa = fast ? Hpart[(size_t)a * n + a] + (ba >= 0 ? lidar_h(gc, ba, sa, a) : 0.0) : h_elem(gc, a, a);
        const double sc = 1.0 / (1.0 + sqrt(haa));
        v_scale[a] = sc; S->scale[a] = sc;
        g0[a] = ga;
      }
      v_g[a] = ga;   // unscaled for the moment
    }
    for (int i = tid; i < xd; i += T) xn += S->x[i] * S->x[i];
    gm = block_max(gm, sred);
    { double d1 = 0, d2 = 0; block_sum3(xn, d1, d2, sred); }
    for (int a = tid; a < n; a += T) { v_g[a] *= v_scale[a]; S->g[a] = v_g[a]; }
    if (tid == 0) {
      sc.x_norm = sqrt(xn);
      int stop = 0;
      if (eval_index == 0) {
        sc.x_cost = cost_eval; sc.initial_cost = cost_eval; sc.cost0 = cost_eval;
        sc.evaluations = 1;
        sc.radius = initial_radius; sc.mu = min_mu; sc.reuse = 0; sc.invalid = 0; sc.iteration = 0; sc.successful = 0; sc.termination = 0;
        if (!isfinite(cost_eval)) { sc.termination = 2; stop = 1; }
        else if (gm <= gradient_tolerance) { sc.termination = 1; stop = 1; }
      } else if (gm <= gradient_tolerance) { sc.termination = 1; stop = 1; }
      if (stop) sc.done = 1;
      s_flag[2] = stop;
    }
    __syncthreads();
    if (s_flag[2]) return;
    DS_MARK(4);
    // scaled H of the current point (lower triangle) -> global and straight into the Cholesky tiles.  One warp per 15 x 15 parameter block pair (K >= L; block O + 1 = extrinsic, 6 wide): inside a block
    // every contribution is a plain sub-matrix (prior rows, the 6 x 6 pose part of a lidar G, ImuFactor quadrants), so
    // the per-element work is five pointer offsets, their loads and the stores.
    if (fast && eval_index >= 1 && gpart[n + 2] != 0.0) {
      // k_hpart left the scaled lidar-independent share in tile layout: one coalesced copy, then the lidar entries (pose rows
      // and the free extrinsic only: <= 72 x 72 / 2 candidates) are added in place
      copy_tiles_map<TP, true>(tiles, const_cast<double *>(HpartT), ntd);
      __syncthreads();
      if (gc.lidar) {
        // the structurally non-zero lidar entries only: per frame the 6 pose_i rows against [pose_0 | pose_i | extrinsic]
        // (108 candidates, lower part kept), then the 12 x 12 block shared by pose_0 and the extrinsic; <= 4 per thread, all
        // their loads independent
        const int total = O * 108 + 144;
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // O <= 16: 1872 candidates <= 4 x 512
          const int e = tid + k * kDsThreads;
          if (e >= total) continue;
          int a, b;
          if (e < O * 108) {
            const int f = e / 108, q = e - f * 108, r = q / 18, c = q - r * 18;
            a = 15 * (f + 1) + r;
            if (c < 6) b = c;                                                   // pose_i x pose_0
            else if (c < 12) { if (c - 6 > r) continue; b = 15 * (f + 1) + (c - 6); }   // pose_i x pose_i, lower part
            else { if (!ex_free) continue; b = a; a = oe + (c - 12); }          // extrinsic x pose_i (the extrinsic rows are the last)
          } else {
            const int q = e - O * 108, r = q / 12, c = q - r * 12;
            a = r < 6 ? r : oe + (r - 6);
            b = c < 6 ? c : oe + (c - 6);
            if (b > a || (!ex_free && a >= oe)) continue;
          }
          int sa = 0;
          const int ba = lidar_block(gc, a, sa);
          const double lh = lidar_h(gc, ba, sa, b);
          if (lh != 0.0) TILE(a >> 3, b >> 3)[swz(a & 7, b & 7)] += lh * v_scale[a] * v_scale[b];
        }
        __syncthreads();
      }
      for (int a = tid; a < n; a += T) {
        const double d = sqrt(fmin(fmax(TILE(a >> 3, a >> 3)[swz(a & 7, a & 7)], min_diagonal), max_diagonal));
        v_diag[a] = d; S->diagonal[a] = d;
      }
    } else if (fast) {
      // one warp per row: the row of Hpart is streamed (all its 32-column slices in flight), the lidar block entry is added
      const int l = lane_id();
      for (int a = warp_id(); a < NP; a += kDsWarps) {
        if (a >= n) {   // padding rows: identity
          for (int b2 = l; b2 <= a; b2 += 32) TILE(a >> 3, b2 >> 3)[swz(a & 7, b2 & 7)] = (a == b2) ? 1.0 : 0.0;
          continue;
        }
        int sa = 0;
        const int ba = gc.lidar ? lidar_block(gc, a, sa) : -1;
        const double sca = v_scale[a];
        double hq[TP::kRowSlices];
#pragma unroll
        for (int q = 0; q < TP::kRowSlices; ++q) { const int b = l + 32 * q; hq[q] = (b <= a) ? Hpart[(size_t)a * n + b] : 0.0; }
#pragma unroll
        for (int q = 0; q < TP::kRowSlices; ++q) {
          const int b = l + 32 * q;
          if (b > a) continue;
          const double h = hq[q] + (ba >= 0 ? lidar_h(gc, ba, sa, b) : 0.0);
          if (eval_index == 0) { H0[(size_t)a * n + b] = h; H0[(size_t)b * n + a] = h; }
          const double hs = h * sca * v_scale[b];
          if (a == b) {
            const double d = sqrt(fmin(fmax(hs, min_diagonal), max_diagonal));
            v_diag[a] = d; S->diagonal[a] = d;
          }
          TILE(a >> 3, b >> 3)[swz(a & 7, b & 7)] = hs;
        }
      }
    } else {
      const int l = lane_id();
      const int nblk = O + 2, npair = nblk * (nblk + 1) / 2;
      for (int pp = warp_id(); pp < npair; pp += kDsWarps) {
        int K = 0, L = pp;
        while (L > K) { L -= K + 1; ++K; }
        const int szK = K == O + 1 ? 6 : 15, szL = L == O + 1 ? 6 : 15;
        const int baseK = K == O + 1 ? oe : 15 * K, baseL = L == O + 1 ? oe : 15 * L;
        const bool exK = K == O + 1, exL = L == O + 1;
        const bool frozen = exK && !ex_free;          // identity rows, nothing else
        // prior: rows/cols of frames < O and of a free extrinsic
        const int pK = K < O ? 15 * K : (exK && ex_free ? 15 * O : -1), pL = L < O ? 15 * L : (exL && ex_free ? 15 * O : -1);
        const double *q0 = (!frozen && use_prior && pK >= 0 && pL >= 0) ? Hp + (size_t)pK * np + pL : nullptr;
        // lidar: 6 x 6 pose sub-block (rows r < 6, cols c < 6) of G0 or of one frame's G
        const double *q1 = nullptr;
        int ld1 = 18;
        if (!frozen && gc.lidar) {
          const bool shK = K == 0 || exK, shL = L == 0 || exL;
          if (shK && shL) { q1 = G0 + (exK ? 6 : 0) * 12 + (exL ? 6 : 0); ld1 = 12; }
          else if (!shK && !shL) { if (K == L) q1 = G + (size_t)(K - 1) * kFGStride + 6 * 18 + 6; }
          else if (shK) q1 = G + (size_t)(L - 1) * kFGStride + 12 * 18 + 6;              // K = extrinsic, L = frame
          else q1 = G + (size_t)(K - 1) * kFGStride + 6 * 18 + (exL ? 12 : 0);             // K = frame, L = pose_0
        }
        // ImuFactors: factor k covers blocks k and k + 1
        const double *q2 = nullptr, *q3 = nullptr;
        if (!frozen && gc.imu && !exK) {
          if (K == L) {
            if (K < O && sh.pim_valid[K]) q2 = F.imu + (size_t)K * kFImuStride;
            if (K >= 1 && sh.pim_valid[K - 1]) q3 = F.imu + (size_t)(K - 1) * kFImuStride + 15 * 30 + 15;
          } else if (L == K - 1 && sh.pim_valid[L]) {
            q3 = F.imu + (size_t)L * kFImuStride + 15 * 30;
          }
        }
        const double *q4 = (!frozen && ex_prior && exK && exL) ? F.ex : nullptr;
        for (int e = l; e < szK * szL; e += 32) {
          const int r = e / szL, c = e - r * szL;
          if (K == L && c > r) continue;
          const int ga = baseK + r, gb = baseL + c;
          double h;
          if (frozen) h = (ga == gb) ? 1.0 : 0.0;
          else {
            const bool pose = r < 6 && c < 6;
            const double v0 = q0 ? q0[(size_t)r * np + c] : 0.0;
            const double v1 = (q1 && pose) ? q1[r * ld1 + c] : 0.0;
            const double v2 = q2 ? q2[r * 30 + c] : 0.0;
            const double v3 = q3 ? q3[r * 30 + c] : 0.0;
            const double v4 = q4 ? q4[r * 6 + c] : 0.0;
            h = (((v0 + v1) + v2) + v3) + v4;
          }
          if (eval_index == 0) { H0[(size_t)ga * n + gb] = h; H0[(size_t)gb * n + ga] = h; }
          const double hs = h * v_scale[ga] * v_scale[gb];
          if (ga == gb) {
            const double d = sqrt(fmin(fmax(hs, min_diagonal), max_diagonal));
            v_diag[ga] = d; S->diagonal[ga] = d;
          }
          TILE(ga >> 3, gb >> 3)[swz(ga & 7, gb & 7)] = hs;
        }
      }
      for (int a2 = n + warp_id(); a2 < NP; a2 += kDsWarps)   // padding rows: identity
        for (int b2 = l; b2 <= a2; b2 += 32) TILE(a2 >> 3, b2 >> 3)[swz(a2 & 7, b2 & 7)] = (a2 == b2) ? 1.0 : 0.0;
    }
    tiles_ready = 1;
    __syncthreads();
    copy_tiles_map<TP, false>(tiles, Hs, ntd);   // kept for a mu retry / an invalid step of a later evaluation (plain stores, nobody waits for them)
    for (int i = tid; i < n; i += T) { v_grad[i] = v_g[i] / v_diag[i]; S->gradient[i] = v_grad[i]; }
    __syncthreads();
    DS_MARK(5);
  }

  // ---------------- next step (loops over invalid steps without a new evaluation) ----------------
  while (true) {
    if (tid == 0) {
      int stop = 0;
      if (sc.iteration >= sc.max_it) { sc.termination = 0; stop = 1; }
      else if (sc.radius < min_radius) { sc.termination = 1; stop = 1; }
      else sc.iteration += 1;
      s_flag[1] = stop;
      s_flag[3] = sc.reuse;
    }
    __syncthreads();
    if (s_flag[1]) { if (tid == 0) sc.done = 1; return; }
    int linear_ok = 1;
    if (!s_flag[3]) {
      // Cauchy point scale: alpha = |gradient|^2 / (sg^T H sg), sg = gradient / D; H sg is kept (model cost change)
      if (!tiles_ready) refill_tiles<TP>(tiles, Hs, ntd);
      for (int i = tid; i < NP; i += T) v_tmp[i] = i < n ? v_g[i] / (v_diag[i] * v_diag[i]) : 0.0;
      __syncthreads();
      symv_tiles<TP>(tiles, n, v_tmp, v_hsg);
      double pa = 0, pb = 0, pc = 0;
      for (int i = tid; i < n; i += T) { pa += v_grad[i] * v_grad[i]; pb += v_tmp[i] * v_hsg[i]; S->hsg[i] = v_hsg[i]; }
      block_sum3(pa, pb, pc, sred);
      double mu = sc.mu;
      if (tid == 0) { sc.alpha = pa / pb; sc.reuse = 1; }
      DS_MARK(6);
      linear_ok = 0;
      bool pure = true;   // the tiles hold the pure H
      while (mu < max_mu) {
        // tiles of H + mu D^2 (lower triangle; identity on the padding), right-hand side g
        if (!pure) refill_tiles<TP>(tiles, Hs, ntd);
        for (int i = tid; i < n; i += T) TILE(i >> 3, i >> 3)[swz(i & 7, i & 7)] += mu * v_diag[i] * v_diag[i];
        pure = false;
        tiles_ready = 0;
        for (int i = tid; i < NP; i += T) v_y[i] = i < n ? v_g[i] : 0.0;
        __syncthreads();
        DS_MARK(7);
        int ok = chol_solve_tiles<TP>(tiles, NB, v_y, &s_ok, eval_index == 1 ? S->chol_prof : nullptr, 4 * 28 + 4);
        DS_MARK(8);
        if (ok) {
          double bad = 0;
          for (int i = tid; i < n; i += T) if (!isfinite(v_y[i])) bad = 1.0;
          bad = block_max(bad, sred);
          ok = bad == 0.0;
        }
        if (!ok) { mu *= mu_factor; __syncthreads(); continue; }
        for (int i = tid; i < n; i += T) { v_gn[i] = -v_diag[i] * v_y[i]; S->gn[i] = v_gn[i]; }
        linear_ok = 1;
        break;
      }
      if (tid == 0) { sc.mu = mu; sc.mu_fact = mu; }
      __syncthreads();
    }
    int step_valid = linear_ok;
    if (linear_ok) {
      double p1 = 0, p2 = 0, p3 = 0;
      for (int i = tid; i < n; i += T) { p1 += v_grad[i] * v_grad[i]; p2 += v_gn[i] * v_gn[i]; p3 += v_grad[i] * v_gn[i]; }
      block_sum3(p1, p2, p3, sred);
      const double gradient_norm = sqrt(p1), gn_norm = sqrt(p2), g_dot_gn = p3;
      const double radius = sc.radius, alpha = sc.alpha;
      double c_grad, c_gn, dsn;
      if (gn_norm <= radius) { c_grad = 0.0; c_gn = 1.0; dsn = gn_norm; }
      else if (gradient_norm * alpha >= radius) { c_grad = -(radius / gradient_norm); c_gn = 0.0; dsn = radius; }
      else {
        const double b_dot_a = -alpha * g_dot_gn;
        const double a2 = pow(alpha * gradient_norm, 2.0);
        const double bma2 = a2 - 2 * b_dot_a + pow(gn_norm, 2);
        const double c = b_dot_a - a2;
        const double d = sqrt(c * c + bma2 * (pow(radius, 2.0) - a2));
        const double beta = (c <= 0) ? (d - c) / bma2 : (radius * radius - a2) / (d + c);
        c_grad = -alpha * (1.0 - beta); c_gn = beta; dsn = -1.0;
      }
      double pn = 0, z1 = 0, z2 = 0;
      for (int i = tid; i < n; i += T) {
        const double sv = c_grad * v_grad[i] + c_gn * v_gn[i];
        pn += sv * sv;
        v_step[i] = sv / v_diag[i];
      }
      block_sum3(pn, z1, z2, sred);
      if (dsn < 0) dsn = sqrt(pn);
      // H step without a matrix pass: step = c_grad sg - c_gn y with (H + mu D^2) y = g and gn = -D y, hence
      // H step = c_grad (H sg) - c_gn (g + mu D gn)
      const double mu_f = sc.mu_fact;
      double q1 = 0, q2 = 0, q3 = 0;
      for (int i = tid; i < n; i += T) {
        const double hstep = c_grad * v_hsg[i] - c_gn * (v_g[i] + mu_f * v_diag[i] * v_gn[i]);
        q1 += v_step[i] * v_g[i]; q2 += v_step[i] * hstep;
      }
      block_sum3(q1, q2, q3, sred);
      const double mcc = -q1 - 0.5 * q2;
      step_valid = mcc > 0.0;
      if (tid == 0) { sc.model_cost_change = mcc; sc.dogleg_step_norm = dsn; }
    }
    __syncthreads();
    if (!step_valid) {
      if (tid == 0) {
        sc.invalid += 1;
        s_flag[1] = sc.invalid >= 5;
        if (s_flag[1]) { sc.termination = 2; sc.done = 1; }
        sc.mu *= mu_factor;
        sc.reuse = 0;
      }
      __syncthreads();
      if (s_flag[1]) return;
      continue;
    }
    if (tid == 0) sc.invalid = 0;
    break;
  }
  DS_MARK(9);
  // candidate = Plus(x, step .* scale); frame terms of the candidate for the next asm_ppp launch
  for (int i = tid; i < n; i += T) v_tmp[i] = v_step[i] * v_scale[i];
  __syncthreads();
  if (tid <= O) {
    const int k = tid;
    pose_plus_impl(S->x + 16 * k, v_tmp + 15 * k, S->cand + 16 * k);
    for (int a = 0; a < 9; ++a) S->cand[16 * k + 7 + a] = S->x[16 * k + 7 + a] + v_tmp[15 * k + 6 + a];
  } else if (tid == O + 1) {
    if (ex_free) pose_plus_impl(S->x + 16 * (O + 1), v_tmp + 15 * (O + 1), S->cand + 16 * (O + 1));
    else for (int a = 0; a < 7; ++a) S->cand[16 * (O + 1) + a] = S->x[16 * (O + 1) + a];
  }
  __syncthreads();
  if (tid < O) write_terms(O, S->cand, Rt);
  __syncthreads();
  DS_MARK(10);
  if (tid == 0 && eval_index < 24) S->dbg[eval_index][11] = gtime_ns();
}

__global__ void __launch_bounds__(kDsThreads, 1)
k_step(DevSolveState *S, double *Hs, const double *__restrict__ Hp, double *H0, double *g0, const double *__restrict__ Sblk,
       FPtrs F, const double *__restrict__ Hpart, const double *__restrict__ HpartT, double *Rt, int eval_index) {
  extern __shared__ __align__(16) double dsm[];
  __shared__ StepShared sh;
  static_assert(sizeof(DevScalars) % 8 == 0, "DevScalars is copied as 8-byte words");
  if (S->sc.done) return;
  const int tid = threadIdx.x;
  if (tid < (int)(sizeof(DevScalars) / 8)) reinterpret_cast<long long *>(&sh.sc)[tid] = reinterpret_cast<const long long *>(&S->sc)[tid];
  if (tid >= 64 && tid < 64 + kMaxOpt) sh.pim_valid[tid - 64] = S->pim_valid[tid - 64];
  if (tid == 128) sh.zero = 0.0;
  __syncthreads();
  step_body<OneCta>(S, sh, dsm, Hs, Hp, H0, g0, Sblk, F, Hpart, HpartT, Rt, eval_index);
  __syncthreads();
  if (tid < (int)(sizeof(DevScalars) / 8)) reinterpret_cast<long long *>(&S->sc)[tid] = reinterpret_cast<const long long *>(&sh.sc)[tid];
}

// Opt windows 14..16: the same step on a cluster of two CTAs.  Rank 0 runs k_step's body with the tiles mapped by TwoCta;
// rank 1 only lends its shared memory.  Exits are uniform over the cluster by construction: no thread returns from this
// kernel before the final cluster barrier.  Rank 1 does nothing between the two barriers; rank 0's early exits (sc.done at
// entry, the verdict / gradient / iteration stops and the failed-step limit inside step_body) all return to the code below,
// and a failed pivot only raises mu inside step_body.  The entry barrier orders rank 1's start before rank 0's first remote
// access; the exit barrier keeps rank 1's shared memory alive until rank 0's last one (its stores are complete: arrive has
// release semantics, wait acquire).
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kDsThreads, 1)
k_step_x2(DevSolveState *S, double *Hs, const double *__restrict__ Hp, double *H0, double *g0, const double *__restrict__ Sblk,
          FPtrs F, const double *__restrict__ Hpart, const double *__restrict__ HpartT, double *Rt, int eval_index) {
  extern __shared__ __align__(16) double dsm[];
  __shared__ StepShared sh;
  cg::cluster_group cluster = cg::this_cluster();
  cluster.sync();
  // uniform over rank 0: nothing writes S->sc before every thread of rank 0 has passed the barrier behind this read
  if (cluster.block_rank() == 0 && !S->sc.done) {
    const int tid = threadIdx.x;
    if (tid < (int)(sizeof(DevScalars) / 8)) reinterpret_cast<long long *>(&sh.sc)[tid] = reinterpret_cast<const long long *>(&S->sc)[tid];
    if (tid >= 64 && tid < 64 + kMaxOpt) sh.pim_valid[tid - 64] = S->pim_valid[tid - 64];
    if (tid == 128) sh.zero = 0.0;
    __syncthreads();
    step_body<TwoCta>(S, sh, dsm, Hs, Hp, H0, g0, Sblk, F, Hpart, HpartT, Rt, eval_index);
    __syncthreads();
    if (tid < (int)(sizeof(DevScalars) / 8)) reinterpret_cast<long long *>(&S->sc)[tid] = reinterpret_cast<const long long *>(&sh.sc)[tid];
  }
  cluster.sync();
}

// =====================================================================================================
static size_t step_smem_bytes(int O) {
  const int n = 15 * (O + 1) + 6, NB = (n + 7) / 8;
  return sizeof(double) * ((size_t)(NB * (NB + 1) / 2) * 64 + 9 * (size_t)NB * 8);
}

// k_step_x2: each CTA of the pair gets rank 0's share (fixed TwoCta layout: local tiles + the nine vectors at NB = 33)
static size_t step_x2_smem_bytes() {
  return sizeof(double) * ((size_t)TwoCta::kLocalTiles * 64 + 9 * (size_t)TwoCta::kMaxNB * 8);
}
static_assert(TwoCta::kPeerTiles * 64 <= TwoCta::kLocalTiles * 64 + 9 * TwoCta::kMaxNB * 8, "rank 1's tiles fit the same allocation");

// The cluster kernel's shared-memory size is set and one two-CTA cluster must be able to be resident on the current device.
static bool cluster_step_resident() {
  const size_t smem = step_x2_smem_bytes();
  if (cudaFuncSetAttribute(k_step_x2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return false; }
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(2); lc.blockDim = dim3(kDsThreads); lc.dynamicSmemBytes = smem;
  int nc = 0;
  if (cudaOccupancyMaxActiveClusters(&nc, k_step_x2, &lc) != cudaSuccess) { cudaGetLastError(); return false; }
  return nc >= 1;
}

// O <= 13: one CTA; O = 14..16: the two-CTA cluster, when the device can hold one (decided once, at estimator creation)
bool DevSolver::supports(int O_) const {
  if (O_ >= 1 && O_ <= kDsMaxOpt1) return step_smem_bytes(O_) <= 225 * 1024;
  return O_ > kDsMaxOpt1 && O_ <= kDsMaxOpt && cluster_step_resident();
}

int DevSolver::init(int O_) {
  O = O_;
  const int n = 15 * (O + 1) + 6, np = 15 * O + 6;
  smem_bytes = O <= kDsMaxOpt1 ? step_smem_bytes(O) : step_x2_smem_bytes();
  if (!alloc(st, 1) || !alloc(Hs, n * n) || !alloc(H0, n * n) || !alloc(g0, n) || !alloc(Hp, np * np) || !alloc(F, f_doubles()) ||
      !alloc(Hpart, (size_t)n * n + n + 8))
    return -1;
  if (cudaMemset(Hpart, 0, sizeof(double) * ((size_t)n * n + n + 8)) != cudaSuccess) return -1;
  {
    const size_t NBt = (n + 7) / 8, ntd = NBt * (NBt + 1) / 2 * 64;
    if (!alloc(HpartT, ntd) || cudaMemset(HpartT, 0, sizeof(double) * ntd) != cudaSuccess) return -1;
    if (cudaMemset(Hs, 0, sizeof(double) * n * n) != cudaSuccess) return -1;
  }
  if (!alloc_host(h_st, 1)) return -1;
  if (cudaMemset(st, 0, sizeof(DevSolveState)) != cudaSuccess) return -1;
  if (cudaMemset(F, 0, sizeof(double) * f_doubles()) != cudaSuccess) return -1;
  if (O <= kDsMaxOpt1) {
    if (cudaFuncSetAttribute(k_step, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes) != cudaSuccess) return -1;
  } else if (cudaFuncSetAttribute(k_step_x2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes) != cudaSuccess) {
    return -1;
  }
  return create(aux) && create(ev_fork) && create(ev_join) ? 0 : -1;
}

static FPtrs fptrs(const DevSolver &ds) {
  FPtrs f;
  f.imu = ds.F + ds.off_imu(); f.M = ds.F + ds.off_M(); f.prior = ds.F + ds.off_prior(); f.ex = ds.F + ds.off_ex(); f.G = ds.F + ds.off_G();
  return f;
}

int dev_solver_factors(DevSolver &ds, int eval_index, cudaStream_t st, int *launches) {
  cudaError_t e = cudaEventRecord(ds.ev_fork, st);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(ds.aux, ds.ev_fork, 0);
  if (e == cudaSuccess) {
    k_factors<<<ds.O + 1 + kFPriorCtas, kFThreads, 0, ds.aux>>>(ds.st, ds.Hp, fptrs(ds), eval_index);
    k_hpart<<<64, 256, 0, ds.aux>>>(ds.st, ds.Hp, fptrs(ds), ds.Hpart, ds.HpartT, eval_index);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(ds.ev_join, ds.aux);
  if (launches) *launches += 2;
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

int dev_solver_step(DevSolver &ds, const double *S_dev, double *Rt_dev, int eval_index, cudaStream_t st, int *launches) {
  cudaError_t e = cudaStreamWaitEvent(st, ds.ev_join, 0);
  if (e == cudaSuccess) {
    if (ds.O <= kDsMaxOpt1)
      k_step<<<1, kDsThreads, ds.smem_bytes, st>>>(ds.st, ds.Hs, ds.Hp, ds.H0, ds.g0, S_dev, fptrs(ds), ds.Hpart, ds.HpartT, Rt_dev, eval_index);
    else   // one cluster of two CTAs (__cluster_dims__)
      k_step_x2<<<2, kDsThreads, ds.smem_bytes, st>>>(ds.st, ds.Hs, ds.Hp, ds.H0, ds.g0, S_dev, fptrs(ds), ds.Hpart, ds.HpartT, Rt_dev, eval_index);
    e = cudaGetLastError();
  }
  if (launches) *launches += 1;
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

}  // namespace lio

// ---- test seam: the tiled shared-memory Cholesky alone, on an explicit host system ------------------------------------
namespace lio {
template <class TP>
__device__ void chol_test_body(double *dsm, int &s_ok, const double *__restrict__ A, const double *__restrict__ b, int n,
                               double *__restrict__ x, int *__restrict__ ok_out, long long *__restrict__ prof) {
  const int tid = threadIdx.x, T = blockDim.x;
  const int NB = (n + 7) / 8, NP = NB * 8;
  double *tiles = dsm, *y = dsm + TP::local_doubles(NB);
  for (int p = tid; p < (NB * (NB + 1) / 2) * 64; p += T) {
    const int t = p >> 6, e = p & 63, r = e >> 3, cs = e & 7, c = cs ^ ((r & 2) << 1);
    int ib = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
    while ((ib + 1) * (ib + 2) / 2 <= t) ++ib;
    while (ib * (ib + 1) / 2 > t) --ib;
    const int jb = t - ib * (ib + 1) / 2;
    const int a = 8 * ib + r, bb = 8 * jb + c;
    const double v = (a < n && bb < n) ? A[(size_t)a * n + bb] : (a == bb ? 1.0 : 0.0);
    if constexpr (TP::kCluster) TILE(ib, jb)[e] = v; else tiles[p] = v;
  }
  for (int i = tid; i < NP; i += T) y[i] = i < n ? b[i] : 0.0;
  __syncthreads();
  const int ok = chol_solve_tiles<TP>(tiles, NB, y, &s_ok, prof, 4 * NB + 5);
  for (int i = tid; i < n; i += T) x[i] = y[i];
  if (tid == 0) *ok_out = ok;
}

__global__ void __launch_bounds__(kDsThreads, 1)
k_chol_test(const double *__restrict__ A, const double *__restrict__ b, int n, double *__restrict__ x, int *__restrict__ ok_out,
            long long *__restrict__ prof) {
  extern __shared__ __align__(16) double dsm[];
  __shared__ int s_ok;
  chol_test_body<OneCta>(dsm, s_ok, A, b, n, x, ok_out, prof);
}

// n = 217..261 on a cluster of two CTAs, as k_step_x2: rank 1 lends its shared memory between the two cluster barriers, and
// no thread leaves before the second (a failed pivot ends chol_solve_tiles on all of rank 0 together).
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kDsThreads, 1)
k_chol_test_x2(const double *__restrict__ A, const double *__restrict__ b, int n, double *__restrict__ x, int *__restrict__ ok_out,
               long long *__restrict__ prof) {
  extern __shared__ __align__(16) double dsm[];
  __shared__ int s_ok;
  cg::cluster_group cluster = cg::this_cluster();
  cluster.sync();
  if (cluster.block_rank() == 0) chol_test_body<TwoCta>(dsm, s_ok, A, b, n, x, ok_out, prof);
  cluster.sync();
}
}  // namespace lio

// Solves A x = b (A symmetric positive definite, n x n row-major, n <= 261) with the device solver's tiled Cholesky: one CTA
// for n <= 216 (k_step's), the two-CTA cluster above (k_step_x2's).
extern "C" int lio_dev_cholesky_solve_host(const double *A, const double *b, int n, double *x, int *ok, long long *prof, int device) {
  using namespace lio;
  if (!A || !b || !x || !ok || n < 1 || n > 15 * (kDsMaxOpt + 1) + 6) return LIO_ERR_INVALID;
  LIO_TRY(select_device(device));
  const int NB = (n + 7) / 8;
  const bool one = n <= 15 * (kDsMaxOpt1 + 1) + 6;
  const size_t smem = sizeof(double) * ((one ? (size_t)(NB * (NB + 1) / 2) * 64 : (size_t)TwoCta::kLocalTiles * 64) + (size_t)NB * 8);
  DevBufs d;
  double *dA = nullptr, *db = nullptr, *dx = nullptr;
  int *dok = nullptr;
  long long *dprof = nullptr;
  const size_t nprof = 4 * (size_t)NB + 1, nprof_dev = nprof + 4;   // + 4 in-kernel phase stamps (not returned)
  if (!d.alloc(&dA, (size_t)n * n) || !d.alloc(&db, n) || !d.alloc(&dx, n) || !d.alloc(&dok, 1) || !d.alloc(&dprof, nprof_dev) ||
      !d.up(dA, A, (size_t)n * n) || !d.up(db, b, n) ||
      !d.ok(cudaFuncSetAttribute(one ? k_chol_test : k_chol_test_x2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) ||
      !d.ok(cudaMemset(dprof, 0, sizeof(long long) * nprof_dev)))
    return LIO_ERR_CUDA;
  if (one) k_chol_test<<<1, kDsThreads, smem>>>(dA, db, n, dx, dok, prof ? dprof : nullptr);
  else k_chol_test_x2<<<2, kDsThreads, smem>>>(dA, db, n, dx, dok, prof ? dprof : nullptr);
  if (!d.ok(cudaGetLastError())) return LIO_ERR_CUDA;
  if (!d.down(x, dx, n) || (prof && !d.down(prof, dprof, nprof))) return LIO_ERR_CUDA;
  if (prof) {   // the four %globaltimer stamps become durations (ns) appended behind the per-panel cycles when the caller left room
    long long st[4];
    if (!d.down(st, dprof + nprof, 4)) return LIO_ERR_CUDA;
    std::fprintf(stderr, "[k_chol_test] ns: entry->loop %lld, loop %lld, backsub %lld, total %lld\n", st[1] - st[0], st[2] - st[1], st[3] - st[2], st[3] - st[0]);
  }
  return d.down(ok, dok, 1) ? LIO_OK : LIO_ERR_CUDA;
}
