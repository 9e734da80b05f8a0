// lio_mapping_b200 — host fp64 factors (see factors_host.h).
#include "factors_host.h"
#include "factors_impl.h"

namespace lio {
using namespace hm;

using namespace fi;

// ---- pre-integration (IntegrationBase.h:77-101 ctor, :127-208 MidPointIntegration, :278-307 Propagate)
Preintegration::Preintegration(const V3 &a0, const V3 &g0, const V3 &ba, const V3 &bg, const ImuNoise &n)
    : acc0(a0), gyr0(g0), lin_acc(a0), lin_gyr(g0), lin_ba(ba), lin_bg(bg), g_norm(n.g_norm) {
  std::memset(jac, 0, sizeof(jac));
  std::memset(cov, 0, sizeof(cov));
  for (int i = 0; i < 15; ++i) jac[i][i] = 1.0;
  for (int k = 0; k < 3; ++k) {
    noise_diag[0 + k] = n.acc_n * n.acc_n; noise_diag[3 + k] = n.gyr_n * n.gyr_n;
    noise_diag[6 + k] = n.acc_n * n.acc_n; noise_diag[9 + k] = n.gyr_n * n.gyr_n;
    noise_diag[12 + k] = n.acc_w * n.acc_w; noise_diag[15 + k] = n.gyr_w * n.gyr_w;
  }
}

void Preintegration::push_back(double dt, const V3 &acc1, const V3 &gyr1) {
  if (keep_samples) { dt_buf.push_back(dt); acc_buf.push_back(acc1); gyr_buf.push_back(gyr1); }
  propagate(dt, acc1, gyr1);
}

void Preintegration::repropagate(const V3 &ba, const V3 &bg) {
  sum_dt = 0;
  acc0 = lin_acc; gyr0 = lin_gyr;
  delta_p = V3(); delta_q = Q(); delta_v = V3();
  lin_ba = ba; lin_bg = bg;
  std::memset(jac, 0, sizeof(jac));
  std::memset(cov, 0, sizeof(cov));
  for (int i = 0; i < 15; ++i) jac[i][i] = 1.0;
  for (size_t i = 0; i < dt_buf.size(); ++i) propagate(dt_buf[i], acc_buf[i], gyr_buf[i]);
  sqrt_info_valid = false;
  cache.reset();
}

void Preintegration::propagate(double dt, const V3 &acc1, const V3 &gyr1) {
  sqrt_info_valid = false;
  cache.reset();
  const V3 un_acc_0 = rotate(delta_q, acc0 - lin_ba);
  const V3 un_gyr = 0.5 * (gyr0 + gyr1) - lin_bg;
  const Q rq = delta_q * Q(1, un_gyr.x * dt / 2, un_gyr.y * dt / 2, un_gyr.z * dt / 2);
  const V3 un_acc_1 = rotate(rq, acc1 - lin_ba);
  const V3 un_acc = 0.5 * (un_acc_0 + un_acc_1);
  const V3 rp = delta_p + delta_v * dt + 0.5 * un_acc * dt * dt;
  const V3 rv = delta_v + un_acc * dt;
  {
    const V3 w_x = un_gyr, a_0_x = acc0 - lin_ba, a_1_x = acc1 - lin_ba;
    const M3 R_w_x = skew(w_x), R_a_0_x = skew(a_0_x), R_a_1_x = skew(a_1_x);
    const M3 I3 = M3::I();
    const M3 dR = toR(delta_q), rR = toR(rq);
    double F[15][15], V[15][18];
    std::memset(F, 0, sizeof(F));
    std::memset(V, 0, sizeof(V));
    const M3 IwR = I3 - R_w_x * dt;
    put33(&F[0][0], 15, 0, 0, I3);
    put33(&F[0][0], 15, 0, 3, dR * R_a_0_x * (-0.25 * dt * dt) + rR * R_a_1_x * IwR * (-0.25 * dt * dt));
    put33(&F[0][0], 15, 0, 6, I3 * dt);
    put33(&F[0][0], 15, 0, 9, (dR + rR) * (-0.25 * dt * dt));
    put33(&F[0][0], 15, 0, 12, rR * R_a_1_x * (-0.1667 * dt * dt * -dt));
    put33(&F[0][0], 15, 3, 3, IwR);
    put33(&F[0][0], 15, 3, 12, I3 * (-1.0 * dt));
    put33(&F[0][0], 15, 6, 3, dR * R_a_0_x * (-0.5 * dt) + rR * R_a_1_x * IwR * (-0.5 * dt));
    put33(&F[0][0], 15, 6, 6, I3);
    put33(&F[0][0], 15, 6, 9, (dR + rR) * (-0.5 * dt));
    put33(&F[0][0], 15, 6, 12, rR * R_a_1_x * (-0.5 * dt * -dt));
    put33(&F[0][0], 15, 9, 9, I3);
    put33(&F[0][0], 15, 12, 12, I3);
    const M3 v03 = (-rR) * R_a_1_x * (0.25 * dt * dt * 0.5 * dt);
    const M3 v63 = (-rR) * R_a_1_x * (0.5 * dt * 0.5 * dt);
    put33(&V[0][0], 18, 0, 0, dR * (0.5 * dt * dt));
    put33(&V[0][0], 18, 0, 3, v03);
    put33(&V[0][0], 18, 0, 6, rR * (0.5 * dt * dt));
    put33(&V[0][0], 18, 0, 9, v03);
    put33(&V[0][0], 18, 3, 3, I3 * (0.5 * dt));
    put33(&V[0][0], 18, 3, 9, I3 * (0.5 * dt));
    put33(&V[0][0], 18, 6, 0, dR * (0.5 * dt));
    put33(&V[0][0], 18, 6, 3, v63);
    put33(&V[0][0], 18, 6, 6, rR * (0.5 * dt));
    put33(&V[0][0], 18, 6, 9, v63);
    put33(&V[0][0], 18, 9, 12, I3 * dt);
    put33(&V[0][0], 18, 12, 15, I3 * dt);
    double nj[15][15], fc[15][15], nc[15][15];
    for (int i = 0; i < 15; ++i)
      for (int j = 0; j < 15; ++j) {
        double s = 0, s2 = 0;
        for (int k = 0; k < 15; ++k) { s += F[i][k] * jac[k][j]; s2 += F[i][k] * cov[k][j]; }
        nj[i][j] = s; fc[i][j] = s2;
      }
    for (int i = 0; i < 15; ++i)
      for (int j = 0; j < 15; ++j) {
        double s = 0;
        for (int k = 0; k < 15; ++k) s += fc[i][k] * F[j][k];
        double s2 = 0;
        for (int k = 0; k < 18; ++k) s2 += V[i][k] * noise_diag[k] * V[j][k];
        nc[i][j] = s + s2;
      }
    std::memcpy(jac, nj, sizeof(jac));
    std::memcpy(cov, nc, sizeof(cov));
  }
  delta_p = rp; delta_v = rv;
  delta_q = normalized(rq);
  sum_dt += dt;
  acc0 = acc1; gyr0 = gyr1;
}

// ImuFactor.h:74-75: sqrt_info = LLT(covariance^-1).matrixL().transpose()
void Preintegration::ensure_sqrt_info() {
  if (sqrt_info_valid) return;
  Mat L(15, 15);
  for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) L(i, j) = cov[i][j];
  Mat inv(15, 15);
  if (cholesky(L)) {
    for (int c = 0; c < 15; ++c) {
      Vec e(15, 0.0);
      e[c] = 1.0;
      cholesky_solve(L, e);
      for (int r = 0; r < 15; ++r) inv(r, c) = e[r];
    }
    for (int i = 0; i < 15; ++i) for (int j = i + 1; j < 15; ++j) { double s = 0.5 * (inv(i, j) + inv(j, i)); inv(i, j) = inv(j, i) = s; }
  }
  Mat Li = inv;
  bool ok = cholesky(Li);
  for (int i = 0; i < 15; ++i) for (int j = 0; j < 15; ++j) sqrt_info[i][j] = (ok && j >= i) ? Li(j, i) : 0.0;
  sqrt_info_valid = true;
}

static void fill_pim(const Preintegration &p, PimData &d) {
  for (int k = 0; k < 3; ++k) { d.delta_p[k] = p.delta_p[k]; d.delta_v[k] = p.delta_v[k]; d.lin_ba[k] = p.lin_ba[k]; d.lin_bg[k] = p.lin_bg[k]; }
  d.delta_q[0] = p.delta_q.x; d.delta_q[1] = p.delta_q.y; d.delta_q[2] = p.delta_q.z; d.delta_q[3] = p.delta_q.w;
  d.sum_dt = p.sum_dt; d.g_norm = p.g_norm;
  std::memcpy(d.jac, p.jac, sizeof(d.jac));
  std::memcpy(d.sqrt_info, p.sqrt_info, sizeof(d.sqrt_info));
}

void Preintegration::to_data(PimData &d) {
  ensure_sqrt_info();
  fill_pim(*this, d);
}

const PimData &Preintegration::data() {
  if (!cache || !sqrt_info_valid) {
    if (!cache) cache = std::make_shared<PimData>();
    to_data(*cache);
  }
  return *cache;
}

#if defined(__x86_64__) && defined(__GNUC__) && !defined(__clang__)
__attribute__((target_clones("arch=x86-64-v3", "default")))
#endif
void imu_factor_evaluate30(Preintegration &pim, const double *pose_i, const double *sb_i, const double *pose_j, const double *sb_j,
                           double r[15], double (*J)[30]) {
  imu_factor_eval30(pim.data(), pose_i, sb_i, pose_j, sb_j, r, J);
}

void imu_factor_evaluate(Preintegration &pim, const double *pose_i, const double *sb_i, const double *pose_j, const double *sb_j,
                         double r[15], double (*Ji)[6], double (*Jsi)[9], double (*Jj)[6], double (*Jsj)[9]) {
  PimData d;
  pim.to_data(d);
  imu_factor_eval_impl(d, pose_i, sb_i, pose_j, sb_j, r, Ji, Jsi, Jj, Jsj);
}

// ---- lidar factor -------------------------------------------------------------------------------
static inline V3 row_times(const V3 &w, const M3 &m) {
  return V3(w.x * m(0, 0) + w.y * m(1, 0) + w.z * m(2, 0), w.x * m(0, 1) + w.y * m(1, 1) + w.z * m(2, 1),
            w.x * m(0, 2) + w.y * m(1, 2) + w.z * m(2, 2));
}

void ppp_evaluate_single(const double point[3], const double coeff[4], const double *pose_pivot, const double *pose_i,
                         const double *pose_ex, double *residual, double *J0, double *J1, double *J2) {
  const V3 P_pivot(pose_pivot), Pi(pose_i), tlb(pose_ex), p(point), w(coeff);
  const Q Q_pivot = pose_q(pose_pivot), Qi = pose_q(pose_i), qlb = pose_q(pose_ex);
  const Q Qlpivot = Q_pivot * conj(qlb);
  const V3 Plpivot = P_pivot - rotate(Qlpivot, tlb);
  const Q Qli = Qi * conj(qlb);
  const V3 Pli = Pi - rotate(Qli, tlb);
  const Q Qlpi = conj(Qlpivot) * Qli;
  const V3 Plpi = rotate(conj(Qlpivot), Pli - Plpivot);
  *residual = dot(w, rotate(Qlpi, p) + Plpi) + coeff[3];
  if (!J0 && !J1 && !J2) return;
  const M3 Ri = toR(Qi), Rp = toR(Q_pivot), rlb = toR(qlb);
  auto put = [](double *J, const V3 &a, const V3 &b) { J[0] = a.x; J[1] = a.y; J[2] = a.z; J[3] = b.x; J[4] = b.y; J[5] = b.z; J[6] = 0.0; };
  if (J0) {
    M3 S = skew(T(Rp) * (Ri * (T(rlb) * (p - tlb)))) + skew(T(Rp) * (Pi - P_pivot));
    put(J0, -row_times(w, rlb * T(Rp)), row_times(w, rlb * S));
  }
  if (J1) {
    M3 A = rlb * T(Rp);
    M3 S = skew(T(rlb) * tlb) - skew(T(rlb) * p);
    put(J1, row_times(w, A), row_times(w, A * Ri * S));
  }
  if (J2) {
    M3 S = T(Rp) * Ri * skew(T(rlb) * (p - tlb)) - skew(T(Rp) * (Ri * (T(rlb) * (p - tlb)))) - skew(T(Rp) * (Pi - P_pivot));
    put(J2, row_times(w, M3::I() - rlb * T(Rp) * Ri * T(rlb)), row_times(w, rlb * S));
  }
}

void ppp_frame_terms(const double *pose_pivot, const double *pose_i, const double *pose_ex, double Rout[9], double tout[3], double Mout[6 * 18]) {
  ppp_frame_terms_impl(pose_pivot, pose_i, pose_ex, Rout, tout, Mout);
}

void prior_factor_evaluate(const V3 &pos0, const Q &rot0, const double *pose_ex, double r[6], double (*J)[6]) {
  prior_factor_impl(pos0, rot0, pose_ex, r, J);
}

void pose_plus(const double *x, const double *delta, double *out) { pose_plus_impl(x, delta, out); }

V3 R2ypr(const M3 &R) {
  const V3 n(R(0, 0), R(1, 0), R(2, 0)), o(R(0, 1), R(1, 1), R(2, 1)), a(R(0, 2), R(1, 2), R(2, 2));
  const double y = std::atan2(n.y, n.x);
  const double p = std::atan2(-n.z, n.x * std::cos(y) + n.y * std::sin(y));
  const double r = std::atan2(a.x * std::sin(y) - a.y * std::cos(y), -o.x * std::sin(y) + o.y * std::cos(y));
  return V3(y, p, r) * (180.0 / M_PI);
}
M3 ypr2R(const V3 &ypr) {
  const double y = ypr.x / 180.0 * M_PI, p = ypr.y / 180.0 * M_PI, r = ypr.z / 180.0 * M_PI;
  M3 Rz, Ry, Rx;
  Rz(0, 0) = std::cos(y); Rz(0, 1) = -std::sin(y); Rz(1, 0) = std::sin(y); Rz(1, 1) = std::cos(y); Rz(2, 2) = 1;
  Ry(0, 0) = std::cos(p); Ry(0, 2) = std::sin(p); Ry(1, 1) = 1; Ry(2, 0) = -std::sin(p); Ry(2, 2) = std::cos(p);
  Rx(0, 0) = 1; Rx(1, 1) = std::cos(r); Rx(1, 2) = -std::sin(r); Rx(2, 1) = std::sin(r); Rx(2, 2) = std::cos(r);
  return Rz * Ry * Rx;
}

}  // namespace lio
