// lio::Twist<float> (include/utils/Twist.h:40-97) on the host, in float and in the reference's operation order: the pose
// compositions of PointMapping::Process / PointOdometry::Process that run once per sweep stay on the CPU (cubemap.cu, podom.cu).
#pragma once
#include <cmath>

namespace lio {

struct TwistF {   // lio::Twist<float> (include/utils/Twist.h:40-97): compositions go through the 3 x 3 matrix like the reference
  float qx = 0, qy = 0, qz = 0, qw = 1, px = 0, py = 0, pz = 0;
};

inline void quat_to_matrix_normalized(const TwistF &t, float R[9]) {   // rot.normalized().toRotationMatrix()
  const float n = std::sqrt(t.qx * t.qx + t.qy * t.qy + t.qz * t.qz + t.qw * t.qw);
  const float x = t.qx / n, y = t.qy / n, z = t.qz / n, w = t.qw / n;
  const float tx = 2.f * x, ty = 2.f * y, tz = 2.f * z;
  const float twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1.f - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1.f - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.f - (txx + tyy);
}

// q * v (Eigen _transformVector) in float: the host copy of the device odom_qmul_vec (odom.cuh), its steps volatile so that
// the host compiler keeps them in the device expression's order.
inline void rotate_host(const TwistF &t, float vx, float vy, float vz, float &ox, float &oy, float &oz) {
  volatile float ux = t.qy * vz - t.qz * vy, uy = t.qz * vx - t.qx * vz, uz = t.qx * vy - t.qy * vx;
  volatile float ux2 = ux + ux, uy2 = uy + uy, uz2 = uz + uz;
  volatile float cx = t.qy * uz2 - t.qz * uy2, cy = t.qz * ux2 - t.qx * uz2, cz = t.qx * uy2 - t.qy * ux2;
  volatile float ax = ux2 * t.qw, ay = uy2 * t.qw, az = uz2 * t.qw;
  volatile float rx = vx + ax, ry = vy + ay, rz = vz + az;
  ox = rx + cx; oy = ry + cy; oz = rz + cz;
}

inline void matrix_to_quat(const float m[9], float q[4]) {   // Eigen quaternionbase_assign_impl<Matrix3> (Shepperd); x y z w
  float t = m[0] + m[4] + m[8];
  if (t > 0.f) {
    t = std::sqrt(t + 1.0f);
    q[3] = 0.5f * t;
    t = 0.5f / t;
    q[0] = (m[7] - m[5]) * t; q[1] = (m[2] - m[6]) * t; q[2] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[i * 3 + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0f);
    q[i] = 0.5f * t;
    t = 0.5f / t;
    q[3] = (m[k * 3 + j] - m[j * 3 + k]) * t;
    q[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
    q[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
  }
}

inline TwistF twist_inverse(const TwistF &a) {   // Twist::inverse :67-73: R^T, -(R^T t); rot not re-normalised
  float R[9], Rt[9], q[4];
  quat_to_matrix_normalized(a, R);
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = R[j * 3 + i];
  matrix_to_quat(Rt, q);
  TwistF r;
  r.qx = q[0]; r.qy = q[1]; r.qz = q[2]; r.qw = q[3];
  r.px = -(Rt[0] * a.px + Rt[1] * a.py + Rt[2] * a.pz);
  r.py = -(Rt[3] * a.px + Rt[4] * a.py + Rt[5] * a.pz);
  r.pz = -(Rt[6] * a.px + Rt[7] * a.py + Rt[8] * a.pz);
  return r;
}

inline TwistF twist_mul(const TwistF &a, const TwistF &b) {   // Twist::operator* :75-78
  float Ra[9], Rb[9], R[9], q[4];
  quat_to_matrix_normalized(a, Ra);
  quat_to_matrix_normalized(b, Rb);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { float s = 0.f; for (int k = 0; k < 3; ++k) s += Ra[i * 3 + k] * Rb[k * 3 + j]; R[i * 3 + j] = s; }
  matrix_to_quat(R, q);
  const float n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  TwistF r;
  r.qx = q[0] / n; r.qy = q[1] / n; r.qz = q[2] / n; r.qw = q[3] / n;
  r.px = (Ra[0] * b.px + Ra[1] * b.py + Ra[2] * b.pz) + a.px;
  r.py = (Ra[3] * b.px + Ra[4] * b.py + Ra[5] * b.pz) + a.py;
  r.pz = (Ra[6] * b.px + Ra[7] * b.py + Ra[8] * b.pz) + a.pz;
  return r;
}

}  // namespace lio
