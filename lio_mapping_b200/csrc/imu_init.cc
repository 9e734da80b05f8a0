// lio_mapping_b200 — the IMU start-up of the imu_factor = 1 estimator on the host: Estimator::RunInitialization
// (src/imu_processor/Estimator.cc:858-958) with ImuInitializer::Initialization (src/imu_processor/ImuInitializer.cc:35-308,
// :421-452).  One attempt solves a 3 x 3 gyro-bias system, a 3 x 3 gravity system and five (3(W+1)+2)^2 refinements; every
// input (the mapped laser poses, the pre-integrations) is host state, so it runs here and not on the device.
#include "imu_init.h"
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

// EstimateGyroBias (:49-90)
void estimate_gyro_bias(int W, const TwistF *tf, Preintegration *const *pre, V3 *Bgs) {
  std::vector<double> A(9, 0.0), b(3, 0.0), dbg;
  for (int i = 0; i < W; ++i) {
    // Quaterniond(q_i^* q_j) with the product in float
    const TwistF &ti = tf[i], &tj = tf[i + 1];
    const float cx = -ti.qx, cy = -ti.qy, cz = -ti.qz, cw = ti.qw;
    const float wx = cw * tj.qx + cx * tj.qw + cy * tj.qz - cz * tj.qy;
    const float wy = cw * tj.qy + cy * tj.qw + cz * tj.qx - cx * tj.qz;
    const float wz = cw * tj.qz + cz * tj.qw + cx * tj.qy - cy * tj.qx;
    const float ww = cw * tj.qw - cx * tj.qx - cy * tj.qy - cz * tj.qz;
    const Q q_ij((double)ww, (double)wx, (double)wy, (double)wz);
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

}  // namespace lio
