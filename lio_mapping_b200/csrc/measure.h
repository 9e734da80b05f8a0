// The pairing of /compact_data messages with IMU messages that the reference's estimator_node runs on its measurement thread, restated
// as host arithmetic on host data (like imu_init.cc).  Reference:
//   MeasurementManager::ImuHandler        src/imu_processor/MeasurementManager.cc:110-116   out-of-order IMU dropped
//   MeasurementManager::GetMeasurements   src/imu_processor/MeasurementManager.cc:54-108    enable_imu = true (MeasurementManager.h:79)
//   Estimator::ProcessEstimation          src/imu_processor/Estimator.cc:2682-2736          the ProcessImu calls of one message
// Compiled without FP contraction, so that the interpolation rounds as the reference writes it.
#pragma once
#include <deque>
#include <utility>
#include <vector>

namespace lio {

struct ImuMsg {
  double t;
  double acc[3], gyr[3];
};

// One Estimator::ProcessImu call: dt, the (possibly interpolated) sample and the IMU message's own header stamp.
struct ImuCall {
  double dt;
  double acc[3], gyr[3];
  double stamp;
};

class MeasurementPairing {
 public:
  enum Decision { kWait = 0, kDropped = 1, kReleased = 2 };

  explicit MeasurementPairing(double msg_time_delay) : delay_(msg_time_delay) {}
  // ImuHandler: a message not later than the last accepted one is dropped (returns false) and counted
  bool push_imu(const ImuMsg &m);
  void push_message(int id, double stamp) { msgs_.emplace_back(id, stamp); }
  // One step of GetMeasurements' loop.  kWait: nothing can be decided yet.  kDropped: the front message was dropped (*id, *stamp).
  // kReleased: the front message was popped (*id, *stamp) with its IMU list in *list: every queued message with stamp < stamp + delay
  // (popped) and then the next one, which stays queued.
  Decision next(int *id, double *stamp, std::vector<ImuMsg> *list);
  // ProcessEstimation's loop over one released message's list; appends its ProcessImu calls.  curr_time_ persists across messages.
  void integrate(double stamp, const std::vector<ImuMsg> &list, std::vector<ImuCall> *calls);
  int pending() const { return (int)msgs_.size(); }
  long long imu_dropped() const { return imu_dropped_; }

 private:
  double delay_;
  double imu_last_time_ = -1;   // MeasurementManager.h:105
  double curr_time_ = -1;       // Estimator::curr_time_
  long long imu_dropped_ = 0;
  std::deque<ImuMsg> imu_;
  std::deque<std::pair<int, double>> msgs_;
};

}  // namespace lio
