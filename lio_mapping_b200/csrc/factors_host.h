// lio_mapping_b200 — the window's small fp64 factors evaluated on the host (O <= 16 IMU blocks, one
// marginalisation prior, one extrinsic prior: a few kflop per iteration), and the per-frame terms
// the fused lidar kernel needs.  Reference files are cited per function in factors_host.cc.
#pragma once
#include "hostmath.h"
#include <memory>

namespace lio { struct PimData; }

namespace lio {

struct ImuNoise {  // IntegrationBaseConfig (include/imu_processor/IntegrationBase.h:64-70)
  double acc_n = 0.1, gyr_n = 0.01, acc_w = 0.0002, gyr_w = 2.0e-5, g_norm = 9.805;
};

// IntegrationBase (include/imu_processor/IntegrationBase.h:72-388), mid-point scheme
struct Preintegration {
  hm::V3 acc0, gyr0, lin_acc, lin_gyr, lin_ba, lin_bg;
  hm::V3 delta_p, delta_v;
  hm::Q delta_q;
  double sum_dt = 0;
  double jac[15][15];
  double cov[15][15];
  double noise_diag[18];
  double g_norm;
  // whitening matrix LLT(cov^-1).matrixL()^T, cached after the last push_back
  double sqrt_info[15][15];
  bool sqrt_info_valid = false;
  bool keep_samples = true;         // false: repropagate is never called (the estimator's INITED pre-integrations)
  std::vector<double> dt_buf;       // the samples pushed so far, for repropagate
  std::vector<hm::V3> acc_buf, gyr_buf;
  Preintegration(const hm::V3 &acc0, const hm::V3 &gyr0, const hm::V3 &ba, const hm::V3 &bg, const ImuNoise &n);
  void push_back(double dt, const hm::V3 &acc, const hm::V3 &gyr);
  // IntegrationBase::Repropagate (IntegrationBase.h:110-125): start over from the first sample with new linearisation biases
  void repropagate(const hm::V3 &ba, const hm::V3 &bg);
  void propagate(double dt, const hm::V3 &acc, const hm::V3 &gyr);   // one mid-point step (Propagate :278-307)
  void ensure_sqrt_info();
  void to_data(struct PimData &d);
  const struct PimData &data();  // cached plain-data view (valid until the next push_back)
  std::shared_ptr<struct PimData> cache;
};

// ImuFactor::Evaluate (include/factor/ImuFactor.h:53-167).  J blocks are 15x6 / 15x9 (tangent
// columns only; the reference's 7th pose column is identically zero), row-major; pass J = nullptr
// for residual-only evaluation.
void imu_factor_evaluate(Preintegration &pim, const double *pose_i, const double *sb_i, const double *pose_j, const double *sb_j,
                         double r[15], double (*Ji)[6], double (*Jsi)[9], double (*Jj)[6], double (*Jsj)[9]);
// Same with the combined 15 x 30 Jacobian over [pose_i | sb_i | pose_j | sb_j] (nullptr: residual only).
void imu_factor_evaluate30(Preintegration &pim, const double *pose_i, const double *sb_i, const double *pose_j, const double *sb_j,
                           double r[15], double (*J)[30]);

// PivotPointPlaneFactor::Evaluate for ONE factor on the host (src/factor/PivotPointPlaneFactor.cc:43-137);
// J blocks 1x7 row-major or nullptr.  Operator-seam entry (lio_ppp_evaluate), not used in the solve loop.
void ppp_evaluate_single(const double point[3], const double coeff[4], const double *pose_pivot, const double *pose_i,
                         const double *pose_ex, double *residual, double *J0, double *J1, double *J2);

// Per-frame terms of the fused lidar kernel: R = R_lpi (row-major), t = R_lpi^T P_lpi, and the
// 6x18 matrix M with J(1x18) = [a ; p x a]^T M over (pose_pivot, pose_i, extrinsic) tangents.
void ppp_frame_terms(const double *pose_pivot, const double *pose_i, const double *pose_ex, double R[9], double t[3], double M[6 * 18]);

// PriorFactor::Evaluate (src/factor/PriorFactor.cc:35-67) on the extrinsic; J is 6x6 (tangent).
void prior_factor_evaluate(const hm::V3 &pos0, const hm::Q &rot0, const double *pose_ex, double r[6], double (*J)[6]);

// PoseLocalParameterization::Plus (src/factor/PoseLocalParameterization.cc:35-52)
void pose_plus(const double *x, const double *delta, double *out);

// mathutils::R2ypr / ypr2R (include/utils/math_utils.h:188-232), degrees
hm::V3 R2ypr(const hm::M3 &R);
hm::M3 ypr2R(const hm::V3 &ypr);

}  // namespace lio

// The C-ABI's pre-integration handle (lio_pim_*): lio_est_init_frame takes over its pre-integration
struct lio_pim {
  std::shared_ptr<lio::Preintegration> p;
};
