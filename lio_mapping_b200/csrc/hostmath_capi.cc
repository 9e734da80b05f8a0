// lio_mapping_b200 — C-ABI seams of the host shell's dense fp64 kernels (hostmath.cc), so that the CPU test-suite can pin
// them against LAPACK without a device: the blocked Cholesky used by the dogleg step (Ceres DENSE_SCHUR equivalent,
// Estimator.cc:1909-1921) and the symmetric eigen-solver used by the marginalisation (Eigen::SelfAdjointEigenSolver call
// sites MarginalizationFactor.cc:276, :293).  Also the pre-integration handle (lio_pim_*) and the ImuFactor on it
// (factors_host.cc), which lio_est_init_frame consumes.
#include <cstring>
#include "../../include/lio_b200.h"
#include "factors_host.h"
#include "hostmath.h"
#include "imu_init.h"
#include "solver_host.h"
#include <cmath>
#include <new>

void lio_set_last_error(const char *file, int line, const char *msg);  // capi_common.cu

using namespace lio;
using namespace lio::hm;

extern "C" int lio_host_cholesky_solve(int n, const double *A, const double *b, double *L_out, double *x) {
  if (n <= 0 || !A || !b || !x) return LIO_ERR_INVALID;
  Mat M(n, n);
  std::memcpy(M.d.data(), A, sizeof(double) * n * n);
  if (!cholesky(M)) {
    lio_set_last_error(__FILE__, __LINE__, "matrix is not positive definite");
    return LIO_ERR_NUMERIC;
  }
  Vec v(b, b + n);
  cholesky_solve(M, v);
  std::memcpy(x, v.data(), sizeof(double) * n);
  if (L_out)
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) L_out[(size_t)i * n + j] = j <= i ? M(i, j) : 0.0;  // only the lower triangle is defined
  return LIO_OK;
}

extern "C" int lio_host_sym_eigen(int n, const double *A, double *evals, double *evecs, int threads) {
  if (n <= 0 || !A || !evals || !evecs) return LIO_ERR_INVALID;
  Mat M(n, n), Z;
  std::memcpy(M.d.data(), A, sizeof(double) * n * n);
  Vec d;
  sym_eigen(M, d, Z, threads < 1 ? 1 : threads);
  std::memcpy(evals, d.data(), sizeof(double) * n);
  std::memcpy(evecs, Z.d.data(), sizeof(double) * n * n);
  return LIO_OK;
}

// The dogleg controller (solver_host.cc, stand-in for ceres::Solve as configured at Estimator.cc:1909-1921) on a toy
// nonlinear least-squares problem assembled on the host:  r_k = a_k . x + amp sin(b_k . x) - y_k, optional CauchyLoss(1.0)
// with the Ceres corrector (rho'' <= 0: residual and Jacobian scaled by sqrt(rho')).  The normal equations are built
// exactly the way the window solver consumes them (H = J^T J, g = J^T r, cost = 1/2 sum rho).  summary = {iterations,
// successful steps, termination, initial cost, final cost, evaluations}.
extern "C" int lio_host_dogleg_toy(int n, int m, const double *A, const double *B, const double *y, double amp, int use_cauchy,
                                   double *x, int max_iter, double *summary) {
  if (n <= 0 || m <= 0 || !A || !B || !y || !x || !summary || max_iter < 0) return LIO_ERR_INVALID;
  using namespace lio;
  Vec state(x, x + n);
  DoglegProblem P;
  P.n = n;
  P.get_state = [&](Vec &o) { o = state; };
  P.set_state = [&](const Vec &v) { state = v; };
  P.plus = [&](const Vec &a, const Vec &d, Vec &o) { o = a; for (int i = 0; i < n; ++i) o[i] += d[i]; };
  P.linearize = [&](Mat &H, Vec &g, double &cost) {
    if (H.r != n) H = Mat(n, n); else H.zero();
    g.assign(n, 0.0);
    cost = 0.0;
    Vec J(n);
    for (int k = 0; k < m; ++k) {
      const double *a = A + (size_t)k * n, *b = B + (size_t)k * n;
      double s = 0, t = 0;
      for (int j = 0; j < n; ++j) { s += a[j] * state[j]; t += b[j] * state[j]; }
      double r = s + amp * std::sin(t) - y[k];
      const double cb = amp * std::cos(t);
      for (int j = 0; j < n; ++j) J[j] = a[j] + cb * b[j];
      if (use_cauchy) {
        const double sq = r * r, rho1 = 1.0 / (1.0 + sq);
        cost += 0.5 * std::log(1.0 + sq);
        const double w = std::sqrt(rho1);
        r *= w;
        for (int j = 0; j < n; ++j) J[j] *= w;
      } else {
        cost += 0.5 * r * r;
      }
      for (int i = 0; i < n; ++i) {
        const double ji = J[i];
        g[i] += ji * r;
        double *row = &H.d[(size_t)i * n];
        for (int j = 0; j < n; ++j) row[j] += ji * J[j];
      }
    }
    return std::isfinite(cost);
  };
  DoglegOptions opt;
  opt.max_num_iterations = max_iter;
  DoglegSummary sum;
  dogleg_solve(opt, P, &sum);
  for (int i = 0; i < n; ++i) x[i] = state[i];
  summary[0] = sum.iterations; summary[1] = sum.successful_steps; summary[2] = sum.termination;
  summary[3] = sum.initial_cost; summary[4] = sum.final_cost; summary[5] = sum.evaluations;
  return LIO_OK;
}

// ---- IntegrationBase and ImuFactor (factors_host.cc) on a pre-integration handle
extern "C" int lio_pim_create(const double a0[3], const double g0[3], const double ba[3], const double bg[3], const double n5[5], lio_pim **out) {
  if (!a0 || !g0 || !ba || !bg || !n5 || !out) return LIO_ERR_INVALID;
  ImuNoise nz;
  nz.acc_n = n5[0]; nz.gyr_n = n5[1]; nz.acc_w = n5[2]; nz.gyr_w = n5[3]; nz.g_norm = n5[4];
  lio_pim *p = new (std::nothrow) lio_pim();
  if (!p) return LIO_ERR_INVALID;
  p->p = std::make_shared<Preintegration>(V3(a0), V3(g0), V3(ba), V3(bg), nz);
  *out = p;
  return LIO_OK;
}
extern "C" int lio_pim_destroy(lio_pim *p) { delete p; return LIO_OK; }
extern "C" int lio_pim_push_back(lio_pim *p, double dt, const double a[3], const double g[3]) {
  if (!p || !a || !g) return LIO_ERR_INVALID;
  p->p->push_back(dt, V3(a), V3(g));
  return LIO_OK;
}
extern "C" int lio_pim_get(lio_pim *p, double *s, double *jac, double *cov) {
  if (!p || !s) return LIO_ERR_INVALID;
  const Preintegration &q = *p->p;
  s[0] = q.delta_p.x; s[1] = q.delta_p.y; s[2] = q.delta_p.z; s[3] = q.delta_q.x; s[4] = q.delta_q.y; s[5] = q.delta_q.z; s[6] = q.delta_q.w;
  s[7] = q.delta_v.x; s[8] = q.delta_v.y; s[9] = q.delta_v.z; s[10] = q.sum_dt;
  if (jac) std::memcpy(jac, q.jac, sizeof(q.jac));
  if (cov) std::memcpy(cov, q.cov, sizeof(q.cov));
  return LIO_OK;
}
extern "C" int lio_imu_factor_evaluate(lio_pim *p, const double pose_i[7], const double sb_i[9], const double pose_j[7],
                                       const double sb_j[9], double *res15, double *J0, double *J1, double *J2, double *J3) {
  if (!p || !pose_i || !sb_i || !pose_j || !sb_j || !res15) return LIO_ERR_INVALID;
  double Ji[15][6], Jsi[15][9], Jj[15][6], Jsj[15][9];
  const bool need = J0 || J1 || J2 || J3;
  imu_factor_evaluate(*p->p, pose_i, sb_i, pose_j, sb_j, res15, need ? Ji : nullptr, Jsi, Jj, Jsj);
  if (need) {
    for (int a = 0; a < 15; ++a) {
      for (int c = 0; c < 7; ++c) { if (J0) J0[a * 7 + c] = c < 6 ? Ji[a][c] : 0.0; if (J2) J2[a * 7 + c] = c < 6 ? Jj[a][c] : 0.0; }
      for (int c = 0; c < 9; ++c) { if (J1) J1[a * 9 + c] = Jsi[a][c]; if (J3) J3[a * 9 + c] = Jsj[a][c]; }
    }
  }
  return LIO_OK;
}

extern "C" int lio_imu_run_initialization_host(int W, const float *laser_tf7, lio_pim *const *pims, const float tlb7[7], double g_norm,
                                               const double *bas, double *bgs, double *vs, double R_WI9[9], double *ps, double *rs, double g3[3],
                                               int *outcome) {
  if (W < 5 || !laser_tf7 || !pims || !tlb7 || !bas || !bgs || !vs || !R_WI9 || !ps || !rs || !g3 || !outcome) return LIO_ERR_INVALID;
  std::vector<TwistF> tf(W + 1);
  std::vector<Preintegration *> pre(W + 1);
  std::vector<V3> Ba(W + 1), Bg(W + 1), Vs(W + 1), Ps(W + 1);
  std::vector<M3> Rs(W + 1);
  for (int i = 0; i <= W; ++i) {
    if (!pims[i]) return LIO_ERR_INVALID;
    const float *t = laser_tf7 + 7 * i;
    tf[i] = TwistF{t[0], t[1], t[2], t[3], t[4], t[5], t[6]};
    pre[i] = pims[i]->p.get();
    Ba[i] = V3(bas + 3 * i); Bg[i] = V3(bgs + 3 * i); Vs[i] = V3(vs + 3 * i);
  }
  M3 R_WI;
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) R_WI(a, b) = R_WI9[3 * a + b];
  V3 g;
  const TwistF tlb{tlb7[0], tlb7[1], tlb7[2], tlb7[3], tlb7[4], tlb7[5], tlb7[6]};
  const int rc = run_initialization(W, tf.data(), pre.data(), tlb, g_norm, Ba.data(), Bg.data(), Vs.data(), R_WI, Ps.data(), Rs.data(), g);
  if (rc == kInitNotFinite) {
    lio_set_last_error(__FILE__, __LINE__, "RunInitialization: non-finite result");
    return LIO_ERR_NUMERIC;
  }
  *outcome = rc;
  if (rc == kInitLowExcitation) return LIO_OK;
  for (int i = 0; i <= W; ++i)
    for (int k = 0; k < 3; ++k) {
      bgs[3 * i + k] = Bg[i][k]; vs[3 * i + k] = Vs[i][k]; ps[3 * i + k] = Ps[i][k];
      for (int c = 0; c < 3; ++c) rs[9 * i + 3 * k + c] = Rs[i](k, c);
    }
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) R_WI9[3 * a + b] = R_WI(a, b);
  for (int k = 0; k < 3; ++k) g3[k] = g[k];
  return LIO_OK;
}

extern "C" int lio_imu_estimate_extrinsic_rotation_host(int W, const float *laser_tf7, lio_pim *const *pims, float tlb7[7], double sv4[4], int *ok) {
  if (W < 1 || !laser_tf7 || !pims || !tlb7 || !sv4 || !ok) return LIO_ERR_INVALID;
  std::vector<TwistF> tf(W + 1);
  std::vector<Preintegration *> pre(W + 1);
  for (int i = 0; i <= W; ++i) {
    if (!pims[i]) return LIO_ERR_INVALID;
    const float *t = laser_tf7 + 7 * i;
    tf[i] = TwistF{t[0], t[1], t[2], t[3], t[4], t[5], t[6]};
    pre[i] = pims[i]->p.get();
  }
  TwistF tlb{tlb7[0], tlb7[1], tlb7[2], tlb7[3], tlb7[4], tlb7[5], tlb7[6]};
  *ok = estimate_extrinsic_rotation(W, tf.data(), pre.data(), tlb, sv4) ? 1 : 0;
  tlb7[0] = tlb.qx; tlb7[1] = tlb.qy; tlb7[2] = tlb.qz; tlb7[3] = tlb.qw;
  return LIO_OK;
}
