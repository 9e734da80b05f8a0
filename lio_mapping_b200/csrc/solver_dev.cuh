// Device-resident trust-region (traditional dogleg) solver — see solver_dev.cu.
#pragma once
#include "assemble.cuh"
#include "factors_impl.h"

namespace lio {

constexpr int kDsMaxN = 15 * (kMaxOpt + 1) + 6;  // 261
constexpr int kDsMaxNp = 15 * kMaxOpt + 6;       // 246
constexpr int kFPriorCtas = 13;                  // CTAs of k_factors that share the prior's matrix-vector product
constexpr int kDsXDim = 16 * (kMaxOpt + 1) + 7;
constexpr int kDsMaxOpt1 = 13;                   // largest opt window whose Cholesky tiles fit one SM's shared memory (k_step)
constexpr int kDsMaxOpt = kMaxOpt;               // larger windows (14..16) spread the tiles over a two-CTA cluster (k_step_x2)

// Scalar part of the solver state.  k_step keeps a copy in shared memory for the duration of a launch (thread 0 runs the
// trust-region bookkeeping on it without global round trips) and writes it back on exit.
struct DevScalars {
  int O, n, max_it;
  int imu_factor, point_distance_factor, prior_factor, marginalization_factor;
  int ex_free, prior_valid, convergence_flag, turn_off;
  int iteration, successful, evaluations, termination, done, reuse, invalid;
  int skip_gates, pad_;   // skip_gates: pure assembly (lio_est_assemble): the convergence gates of Estimator.cc:1924-1985 are not applied
  // trust region
  double radius, mu, alpha, x_cost, cand_cost, model_cost_change, dogleg_step_norm, x_norm;
  double initial_cost, cost_pim, cost_ppp, cost_marg;
  double ex0_pos[3], ex0_quat[4];  // PriorFactor target (transform_lb_ at problem build), quat x y z w
  double cost0;                    // first linearisation (parity / debugging)
  double mu_fact;                  // the mu the current Gauss-Newton step was factored with
};

struct DevSolveState {
  // parameters: [pose_k(7) sb_k(9)] k = 0..O, then extrinsic pose(7)
  double x[kDsXDim], cand[kDsXDim];
  DevScalars sc;
  // ---- everything above is read back after a solve (offsetof(scale) bytes) ----
  double scale[kDsMaxN], diagonal[kDsMaxN], gradient[kDsMaxN], gn[kDsMaxN], g[kDsMaxN];
  double hsg[kDsMaxN];   // H (g / D^2) of the current linearisation: Cauchy-point scale and the model cost change need it
  // marginalisation prior (canonical order [pose_0,sb_0,...,pose_{O-1},sb_{O-1},ex])
  double bp[kDsMaxNp], c0;
  double x0_pose[7 * kMaxOpt], x0_sb[9 * kMaxOpt], x0_ex[7];
  // IMU factors i -> i+1
  PimData pim[kMaxOpt];
  int pim_valid[kMaxOpt];
  // device-side timeline (layout documented at lio_est_solver_trace in lio_b200.h): rows 0..11 k_step phases + gap kernels per
  // evaluation, rows 12..14 asm_ppp stamps, row 16 lidar block expansion
  long long dbg[24][16];
  long long chol_prof[4 * 28 + 4];   // per-panel cycles of the Cholesky of evaluation 1 (see lio_dev_cholesky_solve_host); opt
                                     // windows 14..16 (29..33 tile columns) record panels 0..28 only and no tail stamps
};

// Scratch written by k_factors (state-dependent, lidar-independent terms at the state being evaluated) and read by
// k_step.  Strides in doubles.
constexpr int kFImuStride = 936;   // J^T J (30 x 30) | J^T r (30) | cost | pad
constexpr int kFMStride = 108;     // M_i (6 x 18) of the PivotPointPlane frame terms
constexpr int kFGStride = 344;     // G_i = M_i^T S_gg M_i (18 x 18) | M_i^T S_gr (18) | pad   (written by k_step itself)

struct DevSolver {
  DevMem<DevSolveState> st;       // device
  DevMem<double> Hs;               // the Jacobi-scaled normal matrix of the current x as the step kernel's swizzled lower tiles (mu-retry / invalid-step reload)
  DevMem<double> HpartT;           // evaluations >= 1: scaled lidar-independent share of H in the same tile layout (bulk-copied into shared memory)
                                   // (only re-read when a factorisation has to be repeated with a larger mu)
  DevMem<double> Hp;               // prior np x np
  DevMem<double> H0, g0;           // first linearisation, unscaled (parity getter)
  DevMem<double> F;                // factor scratch: imu | M | prior vec | ex prior | G
  DevMem<double> Hpart;            // n x n row-major, lower triangle: prior + ImuFactor + PriorFactor part of H at the state
                                   // being evaluated (unscaled), gathered by k_hpart beside asm_ppp; then n gradient entries
                                   // and 2 words recording the structure flags it was built with
  HostMem<DevSolveState> h_st;     // pinned staging copy
  size_t smem_bytes = 0;
  int O = 0;
  Stream aux;                      // k_factors runs beside asm_ppp
  Event ev_fork, ev_join;
  int init(int O);
  bool supports(int O) const;
  // scratch offsets (doubles)
  size_t off_imu() const { return 0; }
  size_t off_M() const { return (size_t)kMaxOpt * kFImuStride; }
  size_t off_prior() const { return off_M() + (size_t)kMaxOpt * kFMStride; }                    // np gradient terms | cost
  size_t off_ex() const { return off_prior() + kDsMaxNp + 8 + 16; }                                   // 36 J^T J | 6 J^T r | cost
  size_t off_G() const { return off_ex() + 48; }                                                 // O x kFGStride | 144 + 12 shared
  size_t f_doubles() const { return off_G() + (size_t)kMaxOpt * kFGStride + 160; }
};

// Enqueues the lidar-independent factor evaluation (ImuFactors, marginalisation prior, extrinsic PriorFactor, frame
// terms M_i, then the element-wise gather of their share of H and g) at the state the coming asm_ppp launch evaluates: x for eval_index 0, the candidate afterwards.
// Runs on ds.aux, ordered after everything enqueued so far on `st`; dev_solver_step joins it.
int dev_solver_factors(DevSolver &ds, int eval_index, cudaStream_t st, int *launches);
// Enqueues one evaluation step of the solver on `st` (no host synchronisation):
//   eval_index 0: build the normal equations at x from S_dev, run the convergence gates, take the first step;
//   eval_index k > 0: judge the candidate evaluated by the preceding asm_ppp launch, then take the next step.
// After each call Rt_dev holds the frame terms of the next state to evaluate.
int dev_solver_step(DevSolver &ds, const double *S_dev, double *Rt_dev, int eval_index, cudaStream_t st, int *launches);

}  // namespace lio
