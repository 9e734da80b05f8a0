// lio_mapping_b200 — the IMU start-up of the imu_factor = 1 estimator on the host: Estimator::RunInitialization
// (src/imu_processor/Estimator.cc:858-958) with ImuInitializer::Initialization (src/imu_processor/ImuInitializer.cc:35-308,
// :421-452), and the extrinsic-rotation calibration before it, ImuInitializer::EstimateExtrinsicRotation (:353-419).  One attempt
// solves a 3 x 3 gyro-bias system, a 3 x 3 gravity system and five (3(W+1)+2)^2 refinements, one calibration a 4W x 4 least-squares
// system; every input (the mapped laser poses, the pre-integrations) is host state, so both run here and not on the device.
#include "imu_init.h"
#include <algorithm>
#include <cmath>
#include <limits>

namespace lio {
using namespace hm;

namespace {

// Eigen::LDLT<MatrixXd>::compute + solve (diagonal pivoting on the largest remaining |D|), on a dense row-major n x n matrix
void ldlt_solve(std::vector<double> A, int n, const std::vector<double> &b, std::vector<double> &x) {
  std::vector<int> perm(n);
  std::vector<double> tmp(n);
  for (int k = 0; k < n; ++k) {
    int big = k;
    for (int i = k + 1; i < n; ++i) if (std::fabs(A[i * n + i]) > std::fabs(A[big * n + big])) big = i;
    perm[k] = big;
    if (big != k) {
      for (int j = 0; j < n; ++j) std::swap(A[k * n + j], A[big * n + j]);
      for (int i = 0; i < n; ++i) std::swap(A[i * n + k], A[i * n + big]);
    }
    for (int j = 0; j < k; ++j) tmp[j] = A[j * n + j] * A[k * n + j];
    double akk = A[k * n + k];
    for (int j = 0; j < k; ++j) akk -= A[k * n + j] * tmp[j];
    A[k * n + k] = akk;
    for (int i = k + 1; i < n; ++i) {
      double s = A[i * n + k];
      for (int j = 0; j < k; ++j) s -= A[i * n + j] * tmp[j];
      A[i * n + k] = std::fabs(akk) > 0 ? s / akk : s;
    }
  }
  x = b;
  for (int k = 0; k < n; ++k) std::swap(x[k], x[perm[k]]);
  for (int i = 0; i < n; ++i) for (int j = 0; j < i; ++j) x[i] -= A[i * n + j] * x[j];
  for (int i = 0; i < n; ++i) x[i] = std::fabs(A[i * n + i]) > std::numeric_limits<double>::min() ? x[i] / A[i * n + i] : 0.0;
  for (int i = n - 1; i >= 0; --i) for (int j = i + 1; j < n; ++j) x[i] -= A[j * n + i] * x[j];
  for (int k = n - 1; k >= 0; --k) std::swap(x[k], x[perm[k]]);
}

V3 div(const V3 &v, double s) { return V3(v.x / s, v.y / s, v.z / s); }
V3 normalized3(const V3 &v) { return div(v, norm(v)); }

// rot.cast<double>().toRotationMatrix(), optionally after a float normalized()
M3 rot_of(const TwistF &t, bool normalise) {
  float qx = t.qx, qy = t.qy, qz = t.qz, qw = t.qw;
  if (normalise) {
    const float n = std::sqrt(qx * qx + qy * qy + qz * qz + qw * qw);
    qx /= n; qy /= n; qz /= n; qw /= n;
  }
  return toR(Q((double)qw, (double)qx, (double)qy, (double)qz));
}
V3 pos_of(const TwistF &t) { return V3((double)t.px, (double)t.py, (double)t.pz); }

// TangentBasis (ImuInitializer.cc:35-47): the exact comparison with (0, 0, 1) is the reference's
void tangent_basis(const V3 &g0, V3 &b, V3 &c) {
  const V3 a = normalized3(g0);
  V3 tmp(0, 0, 1);
  if (a.x == tmp.x && a.y == tmp.y && a.z == tmp.z) tmp = V3(1, 0, 0);
  b = normalized3(tmp - a * dot(a, tmp));
  c = cross(a, b);
}

// (q_i^* q_j).cast<double>() with the product in float: the laser rotation between two pushes (:58-60, :369-370)
Q laser_delta_q(const TwistF &ti, const TwistF &tj) {
  const float cx = -ti.qx, cy = -ti.qy, cz = -ti.qz, cw = ti.qw;
  const float wx = cw * tj.qx + cx * tj.qw + cy * tj.qz - cz * tj.qy;
  const float wy = cw * tj.qy + cy * tj.qw + cz * tj.qx - cx * tj.qz;
  const float wz = cw * tj.qz + cz * tj.qw + cx * tj.qy - cy * tj.qx;
  const float ww = cw * tj.qw - cx * tj.qx - cy * tj.qy - cz * tj.qz;
  return Q((double)ww, (double)wx, (double)wy, (double)wz);
}

// EstimateGyroBias (:49-90)
void estimate_gyro_bias(int W, const TwistF *tf, Preintegration *const *pre, V3 *Bgs) {
  std::vector<double> A(9, 0.0), b(3, 0.0), dbg;
  for (int i = 0; i < W; ++i) {
    const Q q_ij = laser_delta_q(tf[i], tf[i + 1]);
    const Preintegration &p = *pre[i + 1];
    const V3 tb = (conj(p.delta_q) * q_ij).vec() * 2.0;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) {
        double s = 0;
        for (int k = 0; k < 3; ++k) s += p.jac[3 + k][12 + r] * p.jac[3 + k][12 + c];
        A[3 * r + c] += s;
      }
      double s = 0;
      for (int k = 0; k < 3; ++k) s += p.jac[3 + k][12 + r] * tb[k];
      b[r] += s;
    }
  }
  ldlt_solve(A, 3, b, dbg);
  for (int i = 0; i <= W; ++i) Bgs[i] = Bgs[i] + V3(dbg[0], dbg[1], dbg[2]);
  for (int i = 0; i < W; ++i) pre[i + 1]->repropagate(V3(), Bgs[0]);
}

// ApproximateGravity (:92-172); W >= 5
bool approximate_gravity(int W, const TwistF *tf, Preintegration *const *pre, const TwistF &tlb, double g_norm, V3 &g) {
  double a = 0;
  V3 bv;
  const V3 plb = pos_of(tlb);
  const M3 rlb = rot_of(tlb, false);
  for (int i = 0; i < W - 1; ++i) {
    const Preintegration &pj = *pre[i + 1], &pk = *pre[i + 2];
    const double dt12 = pj.sum_dt, dt23 = pk.sum_dt;
    const V3 pl1 = pos_of(tf[i]), pl2 = pos_of(tf[i + 1]), pl3 = pos_of(tf[i + 2]);
    const M3 rl1 = rot_of(tf[i], false), rl2 = rot_of(tf[i + 1], false), rl3 = rot_of(tf[i + 2], false);
    const double ta = 0.5 * (dt12 * dt12 * dt23 + dt23 * dt23 * dt12);   // tmp_A = ta * I
    const V3 tb = (pl2 - pl1) * dt23 - (pl3 - pl2) * dt12 + ((rl2 - rl1) * plb) * dt23 - ((rl3 - rl2) * plb) * dt12 +
                  ((rl2 * rlb) * pk.delta_p) * dt12 + ((rl1 * rlb) * pj.delta_v) * dt12 * dt23 -
                  ((rl1 * rlb) * pj.delta_p) * dt23;
    a += ta * ta;
    bv = bv - tb * ta;
  }
  std::vector<double> A(9, 0.0), b = {bv.x * 10000.0, bv.y * 10000.0, bv.z * 10000.0}, x;
  A[0] = A[4] = A[8] = a * 10000.0;
  ldlt_solve(A, 3, b, x);
  g = V3(x[0], x[1], x[2]);
  return std::fabs(norm(g) - g_norm) <= 1.0;
}

// RefineGravityAccBias (:174-308).  A and b are not cleared between the five rounds: each round adds its terms to the
// previous round's (already scaled) system and scales the sum by 1000 again, as the reference does.
void refine_gravity(int W, const TwistF *tf, Preintegration *const *pre, const TwistF &tlb, double g_norm, V3 &g, V3 *Vs, M3 &R_WI) {
  const int n = 3 * (W + 1) + 2;
  std::vector<double> A((size_t)n * n, 0.0), b(n, 0.0), x(n, 0.0);
  const V3 plb = pos_of(tlb);
  const M3 rlb = rot_of(tlb, true);
  g = normalized3(g) * g_norm;
  for (int round = 0; round < 5; ++round) {
    V3 lx, ly;
    tangent_basis(g, lx, ly);
    for (int i = 0; i < W; ++i) {
      const Preintegration &pj = *pre[i + 1];
      const double dt = pj.sum_dt;
      const V3 pl1 = pos_of(tf[i]), pl2 = pos_of(tf[i + 1]);
      const M3 rl1 = rot_of(tf[i], true), rl2 = rot_of(tf[i + 1], true);
      double J[6][8] = {};
      double r[6];
      for (int k = 0; k < 3; ++k) {
        J[k][k] = dt;
        J[k][6] = 0.5 * lx[k] * dt * dt; J[k][7] = 0.5 * ly[k] * dt * dt;
        J[3 + k][k] = 1.0; J[3 + k][3 + k] = -1.0;
        J[3 + k][6] = lx[k] * dt; J[3 + k][7] = ly[k] * dt;
      }
      const V3 r0 = pl2 - pl1 - (rl1 * rlb) * pj.delta_p - (rl1 - rl2) * plb - g * 0.5 * dt * dt;
      const V3 r1 = -((rl1 * rlb) * pj.delta_v) - g * dt;
      for (int k = 0; k < 3; ++k) { r[k] = r0[k]; r[3 + k] = r1[k]; }
      double rA[8][8], rb[8];
      for (int p = 0; p < 8; ++p) {
        for (int q = 0; q < 8; ++q) { double s = 0; for (int k = 0; k < 6; ++k) s += J[k][p] * J[k][q]; rA[p][q] = s; }
        double s = 0;
        for (int k = 0; k < 6; ++k) s += J[k][p] * r[k];
        rb[p] = s;
      }
      const int o = 3 * i;
      for (int p = 0; p < 6; ++p) {
        for (int q = 0; q < 6; ++q) A[(size_t)(o + p) * n + o + q] += rA[p][q];
        b[o + p] += rb[p];
      }
      for (int p = 0; p < 2; ++p) {
        for (int q = 0; q < 2; ++q) A[(size_t)(n - 2 + p) * n + n - 2 + q] += rA[6 + p][6 + q];
        b[n - 2 + p] += rb[6 + p];
      }
      for (int p = 0; p < 6; ++p)
        for (int q = 0; q < 2; ++q) {
          A[(size_t)(o + p) * n + n - 2 + q] += rA[p][6 + q];
          A[(size_t)(n - 2 + q) * n + o + p] += rA[6 + q][p];
        }
    }
    for (double &v : A) v *= 1000.0;
    for (double &v : b) v *= 1000.0;
    ldlt_solve(A, n, b, x);
    g = normalized3(g + lx * x[n - 2] + ly * x[n - 1]) * g_norm;
  }
  const V3 gI(0.0, 0.0, -1.0), gW = normalized3(g), c = cross(gI, gW);
  const V3 v = div(c, norm(c));
  const double ang = std::atan2(norm(c), dot(gI, gW));
  // Sophus::SO3d::exp(ang * v).matrix()
  const V3 w = v * ang;
  const double th2 = dot(w, w), th = std::sqrt(th2);
  double imag, real;
  if (th < 1e-10) {
    imag = 0.5 - (1.0 / 48.0) * th2 + (1.0 / 3840.0) * th2 * th2;
    real = 1.0 - (1.0 / 8.0) * th2 + (1.0 / 384.0) * th2 * th2;
  } else {
    imag = std::sin(0.5 * th) / th;
    real = std::cos(0.5 * th);
  }
  R_WI = toR(Q(real, imag * w.x, imag * w.y, imag * w.z));
  for (int i = 0; i <= W; ++i) Vs[i] = V3(x[3 * i], x[3 * i + 1], x[3 * i + 2]);
}

bool finite3(const V3 &v) { return std::isfinite(v.x) && std::isfinite(v.y) && std::isfinite(v.z); }

}  // namespace

int run_initialization(int W, const TwistF *tf, Preintegration *const *pre, const TwistF &tlb, double g_norm, const V3 *Bas, V3 *Bgs,
                       V3 *Vs, M3 &R_WI, V3 *Ps, M3 *Rs, V3 &g_vec) {
  {  // the excitation check (:860-894); sum_g is read uninitialised there, taken as zero here (DESIGN.md §5)
    V3 sum_g;
    for (int i = 0; i < W; ++i) sum_g = sum_g + div(pre[i + 1]->delta_v, pre[i + 1]->sum_dt);
    const V3 aver_g = div(sum_g * 1.0, (double)W);
    double var = 0;
    for (int i = 0; i < W; ++i) {
      const V3 d = div(pre[i + 1]->delta_v, pre[i + 1]->sum_dt) - aver_g;
      var += dot(d, d);
    }
    var = std::sqrt(var / W);
    if (var < 0.25) return kInitLowExcitation;
  }
  V3 g_in_laser;
  estimate_gyro_bias(W, tf, pre, Bgs);
  bool ok = approximate_gravity(W, tf, pre, tlb, g_norm, g_in_laser);
  if (ok) refine_gravity(W, tf, pre, tlb, g_norm, g_in_laser, Vs, R_WI);
  for (int i = 0; i <= W; ++i) {   // :906-919
    const TwistF tb = twist_mul(tf[i], tlb);
    float R[9];
    quat_to_matrix_normalized(tb, R);
    Ps[i] = V3((double)tb.px, (double)tb.py, (double)tb.pz);
    for (int a = 0; a < 3; ++a) for (int c = 0; c < 3; ++c) Rs[i](a, c) = (double)R[3 * a + c];
  }
  M3 R0 = T(R_WI);   // :921-929
  const double yaw = R2ypr(R0 * Rs[0]).x;
  R0 = ypr2R(V3(-yaw, 0, 0)) * R0;
  R_WI = T(R0);
  g_vec = R0 * g_in_laser;
  for (int i = 0; i <= W; ++i) pre[i]->repropagate(Bas[i], Bgs[i]);
  for (int i = 0; i <= W; ++i) { Ps[i] = R0 * Ps[i]; Rs[i] = R0 * Rs[i]; Vs[i] = R0 * Vs[i]; }
  bool finite = finite3(g_vec);
  for (int a = 0; a < 3; ++a) finite = finite && finite3(V3(R_WI(a, 0), R_WI(a, 1), R_WI(a, 2)));
  for (int i = 0; i <= W; ++i) finite = finite && finite3(Ps[i]) && finite3(Vs[i]) && finite3(Bgs[i]);
  if (!finite) return kInitNotFinite;
  return ok ? kInitSuccess : kInitGravityFailed;
}

// EstimateExtrinsicRotation (ImuInitializer.cc:353-419).  Row block i of A is huber_i (LeftQuatMatrix(q_laser) - RightQuatMatrix(q_imu))
// (math_utils.h:140-161, coefficient order x y z w).  The reference takes Eigen::JacobiSVD of A; here the singular values and V come
// from the symmetric eigen-decomposition of the 4 x 4 A^T A (hm::sym_eigen: Householder tridiagonalisation, then implicit QL), with
// sigma_k = sqrt(lambda_k) and x the eigenvector of the smallest eigenvalue.  Every block row has norm <= 2 huber, and a success needs
// sigma_2 > 0.25, so there the gap below it bounds x's error to about 1e-13; on a failure x is what the reference would write to the
// same accuracy only when the two smallest singular values are apart.
bool estimate_extrinsic_rotation(int W, const TwistF *tf, Preintegration *const *pre, TwistF &tlb, double sv[4]) {
  const TwistF bl = twist_inverse(tlb);   // transform_lb.inverse(), rot cast to double (:356-357)
  const Q rot_bl((double)bl.qw, (double)bl.qx, (double)bl.qy, (double)bl.qz);
  Mat AtA(4, 4);
  for (int i = 0; i < W; ++i) {
    const Q q_imu = pre[i + 1]->delta_q;                 // :367
    const Q q_laser = laser_delta_q(tf[i], tf[i + 1]);   // :369-370
    const Q q_from_imu = conj(rot_bl) * q_imu * rot_bl;  // :372
    const Q d = q_laser * conj(q_from_imu);              // Eigen angularDistance, in degrees (:374)
    const double deg = 180 / M_PI * (2.0 * std::atan2(std::sqrt(d.x * d.x + d.y * d.y + d.z * d.z), std::fabs(d.w)));
    const double huber = deg > 5.0 ? 5.0 / deg : 1.0;   // :378
    const double lv[3] = {q_laser.x, q_laser.y, q_laser.z}, rv[3] = {q_imu.x, q_imu.y, q_imu.z};
    double L[4][4] = {}, R[4][4] = {}, B[4][4];
    const double ls[3][3] = {{0, -lv[2], lv[1]}, {lv[2], 0, -lv[0]}, {-lv[1], lv[0], 0}};
    const double rs[3][3] = {{0, -rv[2], rv[1]}, {rv[2], 0, -rv[0]}, {-rv[1], rv[0], 0}};
    for (int a = 0; a < 3; ++a) {
      for (int c = 0; c < 3; ++c) {
        L[a][c] = (a == c ? q_laser.w : 0.0) + ls[a][c];
        R[a][c] = (a == c ? q_imu.w : 0.0) - rs[a][c];
      }
      L[3][a] = -lv[a]; L[a][3] = lv[a];
      R[3][a] = -rv[a]; R[a][3] = rv[a];
    }
    L[3][3] = q_laser.w; R[3][3] = q_imu.w;
    for (int a = 0; a < 4; ++a) for (int c = 0; c < 4; ++c) B[a][c] = huber * (L[a][c] - R[a][c]);   // :383
    for (int a = 0; a < 4; ++a)
      for (int c = 0; c < 4; ++c) for (int k = 0; k < 4; ++k) AtA(a, c) += B[k][a] * B[k][c];
  }
  Vec lambda;
  Mat V;
  sym_eigen(AtA, lambda, V, 1);   // ascending
  for (int k = 0; k < 4; ++k) sv[k] = std::sqrt(std::max(lambda[3 - k], 0.0));
  // Quaterniond(x) with x = V.col(3) (coefficients x y z w), then transform_lb.rot = x.cast<float>().toRotationMatrix() (:399-402):
  // Eigen's quaternion-to-matrix formula without normalisation, then its matrix-to-quaternion.  The sign of x cancels.
  const float qx = (float)V(0, 0), qy = (float)V(1, 0), qz = (float)V(2, 0), qw = (float)V(3, 0);
  const float tx = 2.f * qx, ty = 2.f * qy, tz = 2.f * qz;
  const float twx = tx * qw, twy = ty * qw, twz = tz * qw, txx = tx * qx, txy = ty * qx, txz = tz * qx, tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  const float M[9] = {1.f - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.f - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1.f - (txx + tyy)};
  float q[4];
  matrix_to_quat(M, q);
  tlb.qx = q[0]; tlb.qy = q[1]; tlb.qz = q[2]; tlb.qw = q[3];
  return sv[2] > 0.25;   // singularValues().tail<3>()(1) > 0.25 (:404-413)
}

}  // namespace lio
