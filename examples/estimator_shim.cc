// A dependency-free mock of the reference's lio::Estimator that keeps its member names and the control flow of the INITED
// branch (src/imu_processor/Estimator.cc: ProcessImu :338-427, ProcessLaserOdom :618-774, SolveOptimization :1648-2438,
// SlideWindow :2570-2666) and forwards the heavy parts to liblio_b200.so through the C ABI - the shim a maintainer would
// write inside the real class (INTEGRATION.md section 2), compiled and run here without Eigen / PCL / Ceres / ROS.
//
//   g++ -std=c++14 -Iinclude examples/estimator_shim.cc -Llio_mapping_b200 -llio_b200 -Wl,-rpath,$PWD/lio_mapping_b200 -o estimator_shim
//   ./estimator_shim scenario.bin states_out.bin [stepwise]
//
// scenario.bin (written by tests/test_cxx_shim_gpu.py), little endian:
//   int32 W, O, n_scans ; float32 tf_lb[7] ; then W warm-start frames { float64 state16[16]; int32 n_imu; n_imu x {float64 dt, acc[3],
//   gyr[3]}; float64 acc0[3], gyr0[3]; int32 n_pts; float32 xyzi[n_pts][4] } ; float64 acc_last[3], gyr_last[3] ;
//   then n_scans x { int32 n_imu; n_imu x {float64 dt, acc[3], gyr[3], stamp}; int32 n_pts; float32 xyzi[n_pts][4] }
// states_out.bin: n_scans x (W + 1) x 16 float64 window states after every scan.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "lio_b200.h"

namespace lio {

struct EstimatorConfig {   // include/imu_processor/Estimator.h:77-108 (the fields this path reads)
  int window_size = 10, opt_window_size = 10;
  float min_match_sq_dis = 1.0f, min_plane_dis = 0.2f, surf_filter_size = 0.4f;
  bool imu_factor = true, point_distance_factor = true, prior_factor = true, marginalization_factor = true;
  int estimate_extrinsic = 1, opt_extrinsic = 1;
  int init_window_factor = 1;
};

class Estimator {
 public:
  explicit Estimator(const EstimatorConfig &config) : estimator_config_(config) {}
  ~Estimator() { if (gpu_) lio_est_destroy(gpu_); }

  // stage_flag_ becomes INITED (Estimator.cc:551-560): hand the window to the library once
  bool SetupGpu(const float tf_lb[7]) {
    lio_est_config c;
    lio_est_default_config(&c);
    c.window_size = estimator_config_.window_size; c.opt_window_size = estimator_config_.opt_window_size;
    c.min_match_sq_dis = estimator_config_.min_match_sq_dis; c.min_plane_dis = estimator_config_.min_plane_dis;
    c.surf_filter_size = estimator_config_.surf_filter_size;
    c.imu_factor = estimator_config_.imu_factor; c.point_distance_factor = estimator_config_.point_distance_factor;
    c.prior_factor = estimator_config_.prior_factor; c.marginalization_factor = estimator_config_.marginalization_factor;
    c.estimate_extrinsic = estimator_config_.estimate_extrinsic; c.opt_extrinsic = estimator_config_.opt_extrinsic;
    c.max_frame_points = 1 << 15; c.max_scan_points = 1 << 17;
    c.init_window_factor = estimator_config_.init_window_factor;
    const int rc = lio_est_create(&c, 0, nullptr, &gpu_);
    if (rc != LIO_OK) { std::fprintf(stderr, "lio_est_create: %d %s\n", rc, lio_last_error()); return false; }
    return lio_est_set_extrinsic(gpu_, tf_lb) == LIO_OK;
  }

  // void Estimator::ProcessImu(double dt, const Vector3d &linear_acceleration, const Vector3d &angular_velocity, const std_msgs::Header &header)
  void ProcessImu(double dt, const double linear_acceleration[3], const double angular_velocity[3], double stamp) {
    if (lio_est_process_imu(gpu_, dt, linear_acceleration, angular_velocity, stamp) != LIO_OK) std::fprintf(stderr, "ProcessImu: %s\n", lio_last_error());
  }

  // void Estimator::ProcessLaserOdom(const Transform &transform_in, const std_msgs::Header &header), INITED branch:
  // laser_cloud_surf_last_ comes from PointMapping::CompactDataHandler; the reference then runs SolveOptimization() and
  // SlideWindow() (Estimator.cc:700-707)
  bool ProcessLaserOdom(const std::vector<float> &laser_cloud_surf_last, bool stepwise) {
    const int n = (int)(laser_cloud_surf_last.size() / 4);
    if (!stepwise) return Check(lio_est_process_scan_host(gpu_, laser_cloud_surf_last.data(), n), "lio_est_process_scan_host");
    // the reference's own order, phase by phase
    if (!Check(lio_est_open_scan_host(gpu_, laser_cloud_surf_last.data(), n), "BuildLocalMap")) return false;   // :1361-1646
    const int O = estimator_config_.opt_window_size;
    std::vector<double> para_pose_(7 * (O + 1)), para_speed_bias_(9 * (O + 1));
    double para_ex_pose_[7];
    if (!Check(lio_est_get_parameters(gpu_, para_pose_.data(), para_speed_bias_.data(), para_ex_pose_), "VectorToDouble")) return false;
    int n_tangent = 0;
    double cost = 0;
    if (!Check(lio_est_assemble(gpu_, para_pose_.data(), para_speed_bias_.data(), para_ex_pose_, nullptr, nullptr, &cost, &n_tangent), "problem.Evaluate"))
      return false;
    double summary[8];
    if (!Check(lio_est_solve(gpu_, para_pose_.data(), para_speed_bias_.data(), para_ex_pose_, 10, summary), "ceres::Solve")) return false;   // :1989
    last_initial_cost_ = cost; last_summary_initial_cost_ = summary[3];
    return Check(lio_est_close_scan(gpu_, para_pose_.data(), para_speed_bias_.data(), para_ex_pose_), "DoubleToVector/Marginalize/SlideWindow");
  }

  lio_est *gpu() { return gpu_; }
  double last_initial_cost_ = 0, last_summary_initial_cost_ = 0;

 private:
  bool Check(int rc, const char *what) {
    if (rc == LIO_OK) return true;
    std::fprintf(stderr, "%s: status %d: %s\n", what, rc, lio_last_error());   // the reference logs through glog and carries on
    return false;
  }
  EstimatorConfig estimator_config_;
  lio_est *gpu_ = nullptr;
};

}  // namespace lio

template <typename T> static bool rd(FILE *f, T *p, size_t n = 1) { return std::fread(p, sizeof(T), n, f) == n; }

int main(int argc, char **argv) {
  std::printf("liblio_b200 version %d, %d CUDA device(s)\n", lio_version(), lio_device_count());
  if (lio_device_count() <= 0) {
    lio::EstimatorConfig cfg;
    lio::Estimator est(cfg);
    const float tf[7] = {0, 0, 0, 1, 0, 0, -0.1f};
    if (!est.SetupGpu(tf)) { std::printf("no device: the estimator cannot be created (status %d, no CPU fallback)\n", LIO_ERR_NO_DEVICE); return 0; }
    return 1;
  }
  if (argc < 3) { std::fprintf(stderr, "usage: %s scenario.bin states_out.bin [stepwise]\n", argv[0]); return 2; }
  const bool stepwise = argc > 3 && std::string(argv[3]) == "stepwise";
  FILE *f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  int32_t W = 0, O = 0, n_scans = 0;
  float tf_lb[7];
  if (!rd(f, &W) || !rd(f, &O) || !rd(f, &n_scans) || !rd(f, tf_lb, 7)) return 4;
  lio::EstimatorConfig cfg;
  cfg.window_size = W; cfg.opt_window_size = O;
  lio::Estimator est(cfg);
  if (!est.SetupGpu(tf_lb)) return 5;
  const double n5[5] = {0.2, 0.02, 2e-4, 2e-5, 9.805};
  const double zero3[3] = {0, 0, 0};
  for (int k = 0; k < W; ++k) {   // Ps_/Rs_/Vs_/Bas_/Bgs_[k], surf_stack_[k], pre_integrations_[k]
    double state16[16], acc0[3], gyr0[3];
    int32_t n_imu = 0, n_pts = 0;
    if (!rd(f, state16, 16) || !rd(f, &n_imu)) return 6;
    std::vector<double> imu(7 * (size_t)n_imu);
    if (n_imu && !rd(f, imu.data(), imu.size())) return 6;
    if (!rd(f, acc0, 3) || !rd(f, gyr0, 3) || !rd(f, &n_pts)) return 6;
    std::vector<float> pts(4 * (size_t)n_pts);
    if (n_pts && !rd(f, pts.data(), pts.size())) return 6;
    lio_pim *pim = nullptr;
    if (k > 0) {
      if (lio_pim_create(acc0, gyr0, zero3, zero3, n5, &pim) != LIO_OK) return 7;
      for (int j = 0; j < n_imu; ++j) lio_pim_push_back(pim, imu[7 * j], &imu[7 * j + 1], &imu[7 * j + 4]);
    }
    if (lio_est_init_frame(est.gpu(), k, state16, pts.data(), n_pts, pim) != LIO_OK) { std::fprintf(stderr, "%s\n", lio_last_error()); return 8; }
  }
  double acc_last[3], gyr_last[3];
  if (!rd(f, acc_last, 3) || !rd(f, gyr_last, 3)) return 9;
  if (lio_est_finish_init(est.gpu(), acc_last, gyr_last) != LIO_OK) return 10;
  FILE *out = std::fopen(argv[2], "wb");
  if (!out) return 11;
  std::vector<double> states(16 * (size_t)(W + 1));
  for (int s = 0; s < n_scans; ++s) {
    int32_t n_imu = 0, n_pts = 0;
    if (!rd(f, &n_imu)) return 12;
    std::vector<double> imu(8 * (size_t)n_imu);
    if (n_imu && !rd(f, imu.data(), imu.size())) return 12;
    for (int j = 0; j < n_imu; ++j) est.ProcessImu(imu[8 * j], &imu[8 * j + 1], &imu[8 * j + 4], imu[8 * j + 7]);
    if (!rd(f, &n_pts)) return 12;
    std::vector<float> pts(4 * (size_t)n_pts);
    if (n_pts && !rd(f, pts.data(), pts.size())) return 12;
    if (!est.ProcessLaserOdom(pts, stepwise)) return 13;
    if (lio_est_get_states(est.gpu(), states.data()) != LIO_OK) return 14;
    std::fwrite(states.data(), sizeof(double), states.size(), out);
    if (stepwise) std::printf("scan %d: cost at the initial point %.9g (assemble) %.9g (solver summary)\n", s, est.last_initial_cost_, est.last_summary_initial_cost_);
  }
  std::fclose(out);
  std::fclose(f);
  std::printf("estimator_shim OK: %d scans, %s\n", n_scans, stepwise ? "stepwise (open / assemble / solve / close)" : "lio_est_process_scan_host");
  return 0;
}
