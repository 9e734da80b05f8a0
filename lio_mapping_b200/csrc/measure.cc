// MeasurementManager's pairing and ProcessEstimation's IMU loop (see measure.h), and the host seam lio_measure_replay.
#include "measure.h"
#include "../../include/lio_b200.h"

namespace lio {

bool MeasurementPairing::push_imu(const ImuMsg &m) {
  if (m.t <= imu_last_time_) {   // MeasurementManager.cc:111-114
    ++imu_dropped_;
    return false;
  }
  imu_last_time_ = m.t;
  imu_.push_back(m);
  return true;
}

MeasurementPairing::Decision MeasurementPairing::next(int *id, double *stamp, std::vector<ImuMsg> *list) {
  list->clear();
  if (imu_.empty() || msgs_.empty()) return kWait;                               // :62-64
  const double t = msgs_.front().second;
  if (imu_.back().t <= t + delay_) return kWait;                                 // :66-71
  *id = msgs_.front().first;
  *stamp = t;
  msgs_.pop_front();
  if (imu_.front().t >= t + delay_) return kDropped;                             // :73-78
  while (imu_.front().t < t + delay_) {                                          // :83-87
    list->push_back(imu_.front());
    imu_.pop_front();
  }
  list->push_back(imu_.front());                                                 // :90, the next message stays queued
  return kReleased;
}

void MeasurementPairing::integrate(double stamp, const std::vector<ImuMsg> &list, std::vector<ImuCall> *calls) {
  double ax = 0, ay = 0, az = 0, rx = 0, ry = 0, rz = 0;                          // Estimator.cc:2686
  for (const ImuMsg &m : list) {
    const double imu_time = m.t;
    const double laser_odom_time = stamp + delay_;
    ImuCall c;
    c.stamp = m.t;                                                               // imu_msg->header
    if (imu_time <= laser_odom_time) {                                           // :2692-2708
      if (curr_time_ < 0) curr_time_ = imu_time;
      const double dt = imu_time - curr_time_;
      curr_time_ = imu_time;
      ax = m.acc[0]; ay = m.acc[1]; az = m.acc[2];
      rx = m.gyr[0]; ry = m.gyr[1]; rz = m.gyr[2];
      c.dt = dt;
    } else {                                                                     // :2710-2727, interpolation at the laser time
      const double dt_1 = laser_odom_time - curr_time_;
      const double dt_2 = imu_time - laser_odom_time;
      curr_time_ = laser_odom_time;
      const double w1 = dt_2 / (dt_1 + dt_2);
      const double w2 = dt_1 / (dt_1 + dt_2);
      ax = w1 * ax + w2 * m.acc[0];
      ay = w1 * ay + w2 * m.acc[1];
      az = w1 * az + w2 * m.acc[2];
      rx = w1 * rx + w2 * m.gyr[0];
      ry = w1 * ry + w2 * m.gyr[1];
      rz = w1 * rz + w2 * m.gyr[2];
      c.dt = dt_1;
    }
    c.acc[0] = ax; c.acc[1] = ay; c.acc[2] = az;
    c.gyr[0] = rx; c.gyr[1] = ry; c.gyr[2] = rz;
    calls->push_back(c);
  }
}

}  // namespace lio

using lio::ImuCall;
using lio::ImuMsg;
using lio::MeasurementPairing;

extern "C" int lio_measure_replay(double msg_time_delay, int n, const int *kind, const double *stamp, const double *acc3, const double *gyr3,
                                  double *calls8, int cap_calls, int *n_calls, int *events3, int cap_events, int *n_events, int *imu_dropped) {
  if (n < 0 || (n > 0 && (!kind || !stamp || !acc3 || !gyr3)) || !calls8 || !n_calls || !events3 || !n_events || !imu_dropped ||
      cap_calls < 0 || cap_events < 0)
    return LIO_ERR_INVALID;
  MeasurementPairing mp(msg_time_delay);
  std::vector<ImuCall> calls;
  std::vector<ImuMsg> list;
  int ne = 0;
  for (int i = 0; i < n; ++i) {
    if (kind[i] == 0) {
      ImuMsg m{stamp[i], {acc3[3 * i], acc3[3 * i + 1], acc3[3 * i + 2]}, {gyr3[3 * i], gyr3[3 * i + 1], gyr3[3 * i + 2]}};
      mp.push_imu(m);
    } else {
      mp.push_message(i, stamp[i]);
    }
    for (;;) {
      int id = -1;
      double t = 0;
      const MeasurementPairing::Decision d = mp.next(&id, &t, &list);
      if (d == MeasurementPairing::kWait) break;
      if (ne >= cap_events) return LIO_ERR_CAPACITY;
      events3[3 * ne] = id;
      events3[3 * ne + 1] = d == MeasurementPairing::kReleased ? 1 : 0;
      events3[3 * ne + 2] = (int)calls.size();
      ++ne;
      if (d == MeasurementPairing::kReleased) mp.integrate(t, list, &calls);
    }
  }
  if ((int)calls.size() > cap_calls) return LIO_ERR_CAPACITY;
  for (size_t k = 0; k < calls.size(); ++k) {
    double *o = calls8 + 8 * k;
    o[0] = calls[k].dt;
    for (int a = 0; a < 3; ++a) { o[1 + a] = calls[k].acc[a]; o[4 + a] = calls[k].gyr[a]; }
    o[7] = calls[k].stamp;
  }
  *n_calls = (int)calls.size();
  *n_events = ne;
  *imu_dropped = (int)mp.imu_dropped();
  return LIO_OK;
}
