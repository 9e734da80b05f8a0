// ORACLE — TEST INFRASTRUCTURE ONLY (see o_linalg.h header).
// ImuInitializer::EstimateExtrinsicRotation (src/imu_processor/ImuInitializer.cc:353-419) restated on IntegrationBase (o_factors.cc),
// with
//   LeftQuatMatrix / RightQuatMatrix   include/utils/math_utils.h:140-161 (coefficient order x y z w)
//   Eigen::JacobiSVD                   a one-sided (Hestenes) Jacobi SVD of A itself, singular values sorted descending with V's columns
// The library solves the same system through the eigen-decomposition of A^T A, so the two share no solver code.
#include "o_factors.h"
#include <algorithm>

namespace orc {

static Quat<double> ex_cast(const Quat<float> &q) { return Quat<double>((double)q.w, (double)q.x, (double)q.y, (double)q.z); }

static void LeftQuatMatrix(const Quat<double> &q, double m[4][4]) {   // math_utils.h:140-149
  const double v[3] = {q.x, q.y, q.z};
  const double sk[3][3] = {{0, -v[2], v[1]}, {v[2], 0, -v[0]}, {-v[1], v[0], 0}};
  for (int a = 0; a < 3; ++a) {
    for (int c = 0; c < 3; ++c) m[a][c] = (a == c ? q.w : 0.0) + sk[a][c];
    m[3][a] = -v[a];
    m[a][3] = v[a];
  }
  m[3][3] = q.w;
}

static void RightQuatMatrix(const Quat<double> &p, double m[4][4]) {   // math_utils.h:151-161
  const double v[3] = {p.x, p.y, p.z};
  const double sk[3][3] = {{0, -v[2], v[1]}, {v[2], 0, -v[0]}, {-v[1], v[0], 0}};
  for (int a = 0; a < 3; ++a) {
    for (int c = 0; c < 3; ++c) m[a][c] = (a == c ? p.w : 0.0) - sk[a][c];
    m[3][a] = -v[a];
    m[a][3] = v[a];
  }
  m[3][3] = p.w;
}

// One-sided Jacobi SVD of the m x 4 matrix A (row-major, overwritten by U Sigma): sweeps of plane rotations of column pairs until every
// pair is orthogonal to machine precision; sigma = the column norms, V the accumulated rotations, both sorted by descending sigma.
static void ex_jacobi_svd(int m, std::vector<double> &A, double sigma[4], double V[4][4]) {
  for (int a = 0; a < 4; ++a) for (int c = 0; c < 4; ++c) V[a][c] = a == c ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 4; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int r = 0; r < m; ++r) {
          const double ap = A[4 * r + p], aq = A[4 * r + q];
          alpha += ap * ap; beta += aq * aq; gamma += ap * aq;
        }
        if (gamma == 0.0 || std::fabs(gamma) <= 1e-15 * std::sqrt(alpha * beta)) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / std::sqrt(1.0 + t * t), s = c * t;
        for (int r = 0; r < m; ++r) {
          const double ap = A[4 * r + p], aq = A[4 * r + q];
          A[4 * r + p] = c * ap - s * aq;
          A[4 * r + q] = s * ap + c * aq;
        }
        for (int r = 0; r < 4; ++r) {
          const double vp = V[r][p], vq = V[r][q];
          V[r][p] = c * vp - s * vq;
          V[r][q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  double s[4];
  for (int c = 0; c < 4; ++c) {
    double n = 0;
    for (int r = 0; r < m; ++r) n += A[4 * r + c] * A[4 * r + c];
    s[c] = std::sqrt(n);
  }
  int order[4] = {0, 1, 2, 3};
  std::sort(order, order + 4, [&](int a, int b) { return s[a] > s[b]; });
  double Vs[4][4];
  for (int k = 0; k < 4; ++k) {
    sigma[k] = s[order[k]];
    for (int r = 0; r < 4; ++r) Vs[r][k] = V[r][order[k]];
  }
  for (int r = 0; r < 4; ++r) for (int k = 0; k < 4; ++k) V[r][k] = Vs[r][k];
}

static bool EstimateExtrinsicRotation(int W, const std::vector<Twist<float>> &tf, const std::vector<std::shared_ptr<IntegrationBase>> &pre,
                                      Twist<float> &transform_lb, double sv[4]) {
  const Twist<float> transform_bl = transform_lb.inverse();                                           // :356
  const Quat<double> rot_bl = ex_cast(transform_bl.rot);                                              // :357
  std::vector<double> A((size_t)16 * W, 0.0);                                                         // :361
  for (int i = 0; i < W; ++i) {                                                                       // :363
    const Quat<double> delta_qij_imu = pre[i + 1]->delta_q_;                                          // :367
    const Quat<double> delta_qij_laser = ex_cast(tf[i].rot.conjugate() * tf[i + 1].rot);              // :369-370
    const Quat<double> delta_qij_laser_from_imu = rot_bl.conjugate() * delta_qij_imu * rot_bl;        // :372
    const double angular_distance = 180 / M_PI * delta_qij_laser.angularDistance(delta_qij_laser_from_imu);   // :374
    const double huber = angular_distance > 5.0 ? 5.0 / angular_distance : 1.0;                       // :378
    double lq[4][4], rq[4][4];
    LeftQuatMatrix(delta_qij_laser, lq);                                                              // :380
    RightQuatMatrix(delta_qij_imu, rq);                                                               // :381
    for (int a = 0; a < 4; ++a) for (int c = 0; c < 4; ++c) A[4 * (4 * i + a) + c] = huber * (lq[a][c] - rq[a][c]);   // :383
  }
  double V[4][4];
  ex_jacobi_svd(4 * W, A, sv, V);                                                                     // :398
  const Quat<double> estimated_qlb(V[3][3], V[0][3], V[1][3], V[2][3]);                               // :399-400, x y z w
  const Quat<float> qf = estimated_qlb.cast<float>();
  transform_lb.rot = Quat<float>::fromRotationMatrix(qf.toRotationMatrix());                          // :402
  return sv[2] > 0.25;                                                                                // :404-417
}

}  // namespace orc

using namespace orc;

extern "C" {

// lio_imu_estimate_extrinsic_rotation_host on the oracle's pre-integrations (orc_pim_create handles); same layout, returns ok
int orc_imu_estimate_extrinsic_rotation(int W, const float *laser_tf7, void *const *pims, float *tlb7, double *sv4) {
  auto tf_of = [](const float *a) { return Twist<float>(Quat<float>(a[3], a[0], a[1], a[2]), Vec3<float>(a[4], a[5], a[6])); };
  std::vector<Twist<float>> tf;
  std::vector<std::shared_ptr<IntegrationBase>> pre;
  for (int i = 0; i <= W; ++i) {
    tf.push_back(tf_of(laser_tf7 + 7 * i));
    pre.push_back(*(std::shared_ptr<IntegrationBase> *)pims[i]);
  }
  Twist<float> lb = tf_of(tlb7);
  const bool ok = EstimateExtrinsicRotation(W, tf, pre, lb, sv4);
  tlb7[0] = lb.rot.x; tlb7[1] = lb.rot.y; tlb7[2] = lb.rot.z; tlb7[3] = lb.rot.w;
  return ok ? 1 : 0;
}

}  // extern "C"
