// ORACLE — TEST INFRASTRUCTURE ONLY (see o_linalg.h header).
// Estimator::RunInitialization (src/imu_processor/Estimator.cc:858-958) and ImuInitializer::Initialization
// (src/imu_processor/ImuInitializer.cc:35-308, :421-452) restated on IntegrationBase (o_factors.cc), with
//   Eigen::LDLT                  diagonal pivoting on the largest remaining |D|, solve with D entries below DBL_MIN taken as zero
//   Sophus::SO3d::exp            3rdparty/sophus/so3.hpp expAndTheta (no renormalisation)
//   mathutils::R2ypr / ypr2R     include/utils/math_utils.h:188-232
// sum_g of the excitation check is read uninitialised by the reference (:863); it is zero here.
#include "o_factors.h"
#include <cfloat>
#include <cstring>

namespace orc {

typedef Twist<float> TransformF;
enum { II_O_R = 3, II_O_BG = 12 };

static void ii_ldlt_solve(MatX A, const VecX &b, VecX &x) {
  const int n = A.r;
  std::vector<int> tr(n);
  VecX t(n);
  for (int k = 0; k < n; ++k) {
    int p = k;
    for (int i = k + 1; i < n; ++i) if (std::fabs(A(i, i)) > std::fabs(A(p, p))) p = i;
    tr[k] = p;
    if (p != k) {
      for (int j = 0; j < n; ++j) std::swap(A(k, j), A(p, j));
      for (int i = 0; i < n; ++i) std::swap(A(i, k), A(i, p));
    }
    for (int j = 0; j < k; ++j) t[j] = A(j, j) * A(k, j);
    double d = A(k, k);
    for (int j = 0; j < k; ++j) d -= A(k, j) * t[j];
    A(k, k) = d;
    for (int i = k + 1; i < n; ++i) {
      double s = A(i, k);
      for (int j = 0; j < k; ++j) s -= A(i, j) * t[j];
      A(i, k) = std::fabs(d) > 0 ? s / d : s;
    }
  }
  x = b;
  for (int k = 0; k < n; ++k) std::swap(x[k], x[tr[k]]);
  for (int i = 0; i < n; ++i) for (int j = 0; j < i; ++j) x[i] -= A(i, j) * x[j];
  for (int i = 0; i < n; ++i) x[i] = std::fabs(A(i, i)) > DBL_MIN ? x[i] / A(i, i) : 0.0;
  for (int i = n - 1; i >= 0; --i) for (int j = i + 1; j < n; ++j) x[i] -= A(j, i) * x[j];
  for (int k = n - 1; k >= 0; --k) std::swap(x[k], x[tr[k]]);
}

static V3 ii_normalized(const V3 &v) { return v / std::sqrt(v.dot(v)); }
static double ii_norm(const V3 &v) { return std::sqrt(v.dot(v)); }

static V3 R2ypr(const M3 &R) {
  const V3 n = R.col(0), o = R.col(1), a = R.col(2);
  const double y = std::atan2(n.y, n.x);
  const double p = std::atan2(-n.z, n.x * std::cos(y) + n.y * std::sin(y));
  const double r = std::atan2(a.x * std::sin(y) - a.y * std::cos(y), -o.x * std::sin(y) + o.y * std::cos(y));
  return V3(y, p, r) / M_PI * 180.0;
}
static M3 ypr2R(const V3 &ypr) {
  const double y = ypr.x / 180.0 * M_PI, p = ypr.y / 180.0 * M_PI, r = ypr.z / 180.0 * M_PI;
  M3 Rz, Ry, Rx;
  Rz(0, 0) = std::cos(y); Rz(0, 1) = -std::sin(y); Rz(1, 0) = std::sin(y); Rz(1, 1) = std::cos(y); Rz(2, 2) = 1;
  Ry(0, 0) = std::cos(p); Ry(0, 2) = std::sin(p); Ry(1, 1) = 1; Ry(2, 0) = -std::sin(p); Ry(2, 2) = std::cos(p);
  Rx(0, 0) = 1; Rx(1, 1) = std::cos(r); Rx(1, 2) = -std::sin(r); Rx(2, 1) = std::sin(r); Rx(2, 2) = std::cos(r);
  return Rz * Ry * Rx;
}

static M3 SO3Exp(const V3 &omega) {
  const double theta_sq = omega.dot(omega), theta = std::sqrt(theta_sq), half = 0.5 * theta;
  double imag, real;
  if (theta < 1e-10) {
    const double t4 = theta_sq * theta_sq;
    imag = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * t4;
    real = 1.0 - (1.0 / 8.0) * theta_sq + (1.0 / 384.0) * t4;
  } else {
    imag = std::sin(half) / theta;
    real = std::cos(half);
  }
  return Qd(real, imag * omega.x, imag * omega.y, imag * omega.z).toRotationMatrix();
}

struct ImuWindow {   // all_laser_transforms_ with their shared pre-integrations
  int W;
  std::vector<TransformF> tf;
  std::vector<std::shared_ptr<IntegrationBase>> pre;
};

static void EstimateGyroBias(ImuWindow &w, std::vector<V3> &Bgs) {
  MatX A(3, 3);
  VecX b(3, 0.0), dbg;
  for (int i = 0; i < w.W; ++i) {
    const Quat<float> qf = w.tf[i].rot.conjugate() * w.tf[i + 1].rot;
    const Qd q_ij((double)qf.w, (double)qf.x, (double)qf.y, (double)qf.z);
    const IntegrationBase &p = *w.pre[i + 1];
    const V3 tb = (p.delta_q_.conjugate() * q_ij).vec() * 2.0;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) {
        double s = 0;
        for (int k = 0; k < 3; ++k) s += p.jacobian_(II_O_R + k, II_O_BG + r) * p.jacobian_(II_O_R + k, II_O_BG + c);
        A(r, c) += s;
      }
      double s = 0;
      for (int k = 0; k < 3; ++k) s += p.jacobian_(II_O_R + k, II_O_BG + r) * tb[k];
      b[r] += s;
    }
  }
  ii_ldlt_solve(A, b, dbg);
  for (int i = 0; i <= w.W; ++i) Bgs[i] += V3(dbg[0], dbg[1], dbg[2]);
  for (int i = 0; i < w.W; ++i) w.pre[i + 1]->Repropagate(V3(), Bgs[0]);
}

static bool ApproximateGravity(ImuWindow &w, V3 &g, const TransformF &lb, double g_norm) {
  MatX A(3, 3);
  VecX b(3, 0.0), x;
  const V3 plb = lb.pos.cast<double>();
  const M3 rlb = lb.rot.cast<double>().toRotationMatrix();
  for (int i = 0; i < w.W - 1; ++i) {
    const IntegrationBase &pj = *w.pre[i + 1], &pk = *w.pre[i + 2];
    const double dt12 = pj.sum_dt_, dt23 = pk.sum_dt_;
    const V3 pl1 = w.tf[i].pos.cast<double>(), pl2 = w.tf[i + 1].pos.cast<double>(), pl3 = w.tf[i + 2].pos.cast<double>();
    const M3 rl1 = w.tf[i].rot.cast<double>().toRotationMatrix(), rl2 = w.tf[i + 1].rot.cast<double>().toRotationMatrix(),
             rl3 = w.tf[i + 2].rot.cast<double>().toRotationMatrix();
    const double a = 0.5 * (dt12 * dt12 * dt23 + dt23 * dt23 * dt12);
    const V3 tb = (pl2 - pl1) * dt23 - (pl3 - pl2) * dt12 + ((rl2 - rl1) * plb) * dt23 - ((rl3 - rl2) * plb) * dt12 +
                  ((rl2 * rlb) * pk.delta_p_) * dt12 + ((rl1 * rlb) * pj.delta_v_) * dt12 * dt23 - ((rl1 * rlb) * pj.delta_p_) * dt23;
    for (int k = 0; k < 3; ++k) { A(k, k) += a * a; b[k] -= a * tb[k]; }
  }
  for (double &v : A.d) v *= 10000.0;
  for (double &v : b) v *= 10000.0;
  ii_ldlt_solve(A, b, x);
  g = V3(x[0], x[1], x[2]);
  return std::fabs(ii_norm(g) - g_norm) <= 1.0;
}

static void TangentBasis(const V3 &g0, V3 &b, V3 &c) {
  const V3 a = ii_normalized(g0);
  V3 tmp(0, 0, 1);
  if (a.x == tmp.x && a.y == tmp.y && a.z == tmp.z) tmp = V3(1, 0, 0);
  b = ii_normalized(tmp - a * a.dot(tmp));
  c = a.cross(b);
}

static void RefineGravityAccBias(ImuWindow &w, std::vector<V3> &Vs, V3 &g, const TransformF &lb, double g_norm, M3 &R_WI) {
  const int n = 3 * (w.W + 1) + 2;
  MatX A(n, n);
  VecX b(n, 0.0), x(n, 0.0);
  const V3 plb = lb.pos.cast<double>();
  const M3 rlb = lb.rot.normalized().cast<double>().toRotationMatrix();
  g = ii_normalized(g) * g_norm;
  for (int k = 0; k < 5; ++k) {
    V3 lx, ly;
    TangentBasis(g, lx, ly);
    for (int i = 0; i < w.W; ++i) {
      const IntegrationBase &pj = *w.pre[i + 1];
      const double dt = pj.sum_dt_;
      const V3 pl1 = w.tf[i].pos.cast<double>(), pl2 = w.tf[i + 1].pos.cast<double>();
      const M3 rl1 = w.tf[i].rot.normalized().cast<double>().toRotationMatrix(), rl2 = w.tf[i + 1].rot.normalized().cast<double>().toRotationMatrix();
      MatX tA(6, 8);
      VecX tb(6, 0.0);
      for (int q = 0; q < 3; ++q) {
        tA(q, q) = dt;
        tA(q, 6) = 0.5 * lx[q] * dt * dt; tA(q, 7) = 0.5 * ly[q] * dt * dt;
        tA(3 + q, q) = 1.0; tA(3 + q, 3 + q) = -1.0;
        tA(3 + q, 6) = lx[q] * dt; tA(3 + q, 7) = ly[q] * dt;
      }
      const V3 r0 = pl2 - pl1 - (rl1 * rlb) * pj.delta_p_ - (rl1 - rl2) * plb - g * 0.5 * dt * dt;
      const V3 r1 = -((rl1 * rlb) * pj.delta_v_) - g * dt;
      for (int q = 0; q < 3; ++q) { tb[q] = r0[q]; tb[3 + q] = r1[q]; }
      MatX rA(8, 8);
      VecX rb(8, 0.0);
      for (int p = 0; p < 8; ++p) {
        for (int q = 0; q < 8; ++q) { double s = 0; for (int m = 0; m < 6; ++m) s += tA(m, p) * tA(m, q); rA(p, q) = s; }
        double s = 0;
        for (int m = 0; m < 6; ++m) s += tA(m, p) * tb[m];
        rb[p] = s;
      }
      const int o = 3 * i;
      for (int p = 0; p < 6; ++p) { for (int q = 0; q < 6; ++q) A(o + p, o + q) += rA(p, q); b[o + p] += rb[p]; }
      for (int p = 0; p < 2; ++p) { for (int q = 0; q < 2; ++q) A(n - 2 + p, n - 2 + q) += rA(6 + p, 6 + q); b[n - 2 + p] += rb[6 + p]; }
      for (int p = 0; p < 6; ++p)
        for (int q = 0; q < 2; ++q) { A(o + p, n - 2 + q) += rA(p, 6 + q); A(n - 2 + q, o + p) += rA(6 + q, p); }
    }
    for (double &v : A.d) v *= 1000.0;   // A and b carry over between the rounds (:193-196 are outside the loop)
    for (double &v : b) v *= 1000.0;
    ii_ldlt_solve(A, b, x);
    g = ii_normalized(g + lx * x[n - 2] + ly * x[n - 1]) * g_norm;
  }
  const V3 gI(0.0, 0.0, -1.0), gW = ii_normalized(g), c = gI.cross(gW);
  const V3 v = c / ii_norm(c);
  const double ang = std::atan2(ii_norm(c), gI.dot(gW));
  R_WI = SO3Exp(v * ang);
  for (int i = 0; i <= w.W; ++i) Vs[i] = V3(x[3 * i], x[3 * i + 1], x[3 * i + 2]);
}

// outcome: 0 excitation, 1 gravity check, 2 success
static int RunInitialization(ImuWindow &w, const TransformF &lb, double g_norm, const std::vector<V3> &Bas, std::vector<V3> &Bgs,
                             std::vector<V3> &Vs, M3 &R_WI, std::vector<V3> &Ps, std::vector<M3> &Rs, V3 &g_vec) {
  const int W = w.W;
  {
    V3 sum_g;
    for (int i = 0; i < W; ++i) sum_g += w.pre[i + 1]->delta_v_ / w.pre[i + 1]->sum_dt_;
    const V3 aver_g = sum_g * 1.0 / (double)W;
    double var = 0;
    for (int i = 0; i < W; ++i) {
      const V3 d = w.pre[i + 1]->delta_v_ / w.pre[i + 1]->sum_dt_ - aver_g;
      var += d.dot(d);
    }
    var = std::sqrt(var / W);
    if (var < 0.25) return 0;
  }
  V3 g_in_laser;
  EstimateGyroBias(w, Bgs);
  const bool ok = ApproximateGravity(w, g_in_laser, lb, g_norm);
  if (ok) RefineGravityAccBias(w, Vs, g_in_laser, lb, g_norm, R_WI);
  for (int i = 0; i <= W; ++i) {
    const TransformF tb = w.tf[i] * lb;
    Ps[i] = tb.pos.cast<double>();
    Rs[i] = tb.rot.normalized().toRotationMatrix().cast<double>();
  }
  M3 R0 = R_WI.transpose();
  const double yaw = R2ypr(R0 * Rs[0]).x;
  R0 = ypr2R(V3(-yaw, 0, 0)) * R0;
  R_WI = R0.transpose();
  g_vec = R0 * g_in_laser;
  for (int i = 0; i <= W; ++i) w.pre[i]->Repropagate(Bas[i], Bgs[i]);
  for (int i = 0; i <= W; ++i) { Ps[i] = R0 * Ps[i]; Rs[i] = R0 * Rs[i]; Vs[i] = R0 * Vs[i]; }
  return ok ? 2 : 1;
}

}  // namespace orc

using namespace orc;

extern "C" {

// lio_imu_run_initialization_host on the oracle's pre-integrations (orc_pim_create handles); same layout, returns the outcome
int orc_imu_run_initialization(int W, const float *laser_tf7, void *const *pims, const float *tlb7, double g_norm, const double *bas, double *bgs,
                               double *vs, double *R_WI9, double *ps, double *rs, double *g3) {
  ImuWindow w;
  w.W = W;
  auto tf_of = [](const float *a) { return TransformF(Quat<float>(a[3], a[0], a[1], a[2]), Vec3<float>(a[4], a[5], a[6])); };
  std::vector<V3> Ba(W + 1), Bg(W + 1), Vs(W + 1), Ps(W + 1);
  std::vector<M3> Rs(W + 1);
  for (int i = 0; i <= W; ++i) {
    w.tf.push_back(tf_of(laser_tf7 + 7 * i));
    w.pre.push_back(*(std::shared_ptr<IntegrationBase> *)pims[i]);
    Ba[i] = V3(bas[3 * i], bas[3 * i + 1], bas[3 * i + 2]);
    Bg[i] = V3(bgs[3 * i], bgs[3 * i + 1], bgs[3 * i + 2]);
    Vs[i] = V3(vs[3 * i], vs[3 * i + 1], vs[3 * i + 2]);
  }
  M3 R_WI;
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) R_WI(a, b) = R_WI9[3 * a + b];
  V3 g;
  const int out = RunInitialization(w, tf_of(tlb7), g_norm, Ba, Bg, Vs, R_WI, Ps, Rs, g);
  if (out == 0) return 0;
  for (int i = 0; i <= W; ++i)
    for (int k = 0; k < 3; ++k) {
      bgs[3 * i + k] = Bg[i][k]; vs[3 * i + k] = Vs[i][k]; ps[3 * i + k] = Ps[i][k];
      for (int c = 0; c < 3; ++c) rs[9 * i + 3 * k + c] = Rs[i](k, c);
    }
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) R_WI9[3 * a + b] = R_WI(a, b);
  for (int k = 0; k < 3; ++k) g3[k] = g[k];
  return out;
}

}  // extern "C"
