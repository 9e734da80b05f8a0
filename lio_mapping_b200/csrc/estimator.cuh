// The device window estimator's context (lio_est) and the helpers its units share; internal to the library (the C-ABI is
// include/lio_b200.h).  The units:
//   estimator.cu   creation, IMU, the scan shell and its C-ABI entries, the stepwise API, shard set-up, getters
//   est_solve.cu   BuildLocalMap, the stage-C lidar reduction, linearisation, marginalisation, both solvers, SlideWindow
//   est_map.cu     the /local clouds, the attached cube map and the imu_factor = 0 mapping
// Every unit is compiled with -fmad=false (the host arithmetic and the kernels are bit-exact against the CPU path).
#pragma once
#include "assemble.cuh"
#include "cubemap.cuh"
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include "factors_host.h"
#include "factors_impl.h"
#include "imu_init.h"
#include "knn.cuh"
#include "odom.cuh"
#include "qr.cuh"
#include "solver_dev.cuh"
#include "solver_host.h"
#include "voxel.cuh"
#include <array>
#include <chrono>
#include <cstddef>
#include <memory>
#include <new>
#include <vector>

namespace lio {
constexpr int kMaxWindow = 32;
}  // namespace lio

using namespace lio;
using namespace lio::hm;

inline double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct ImuStampedF {
  double time;
  float q[4];  // x y z w
  float p[3];
};

struct MargPrior {
  bool valid = false;
  int n = 0;      // 15*O + 6
  Mat Hp;         // J^T J
  Vec bp;         // J^T r0
  double c0 = 0;  // r0^T r0
  std::vector<double> x0_pose, x0_sb;  // O x 7, O x 9
  double x0_ex[7];
};

// Marginalisation split in two: the linearised system (A, b) of the dropped + kept blocks is built right after the
// solve (it needs the device reduction and the converged parameters); the dense algebra (Schur complement + two
// symmetric eigen-decompositions, ~n^3) is a pure function of that snapshot and runs on a worker thread while the next
// scan's front end (deskew, voxel grid, local map, k-NN features) keeps the device busy.  The worker is started at
// the ENTRY of the next lio_est_process_scan_* call, not earlier, so none of it runs outside a caller's timed step.
struct MargJob {
  bool stashed = false, running = false;
  int O = 0;
  Mat A;
  Vec b;
  std::vector<double> x0_pose, x0_sb;
  double x0_ex[7];
  MargPrior result;
};

// One persistent helper thread per estimator context (created on first use): starting a std::thread per scan costs
// ~0.1 ms on the bench host.  Hand-off: the helper spins for spin_us after each job before it sleeps on the condition
// variable, so the jobs of one solve (one every ~150 us) never pay a futex wake-up; between scans it sleeps.
struct Worker {
  double spin_us = 400.0;   // hand-off spin window; shortened for sharded runs (one process per GPU shares the host cores)
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::function<void()> job;
  std::atomic<int> has_job{0}, busy{0}, sleeping{0};
  bool quit = false, started = false;
  static inline void relax() {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
  void submit(std::function<void()> f) {
    wait();                                // the previous job has fully retired
    if (!started) { started = true; th = std::thread([this]() { loop(); }); }
    job = std::move(f);
    busy.store(1);
    has_job.store(1);
    if (sleeping.load()) { std::lock_guard<std::mutex> lk(mu); cv.notify_all(); }
  }
  void wait() {
    const double t0 = now_s();
    while (busy.load()) {
      relax();
      if ((now_s() - t0) * 1e6 > spin_us) {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [this]() { return busy.load() == 0; });
        return;
      }
    }
  }
  void loop() {
    while (true) {
      const double t0 = now_s();
      bool got = false;
      while ((now_s() - t0) * 1e6 <= spin_us) {
        if (has_job.load()) { got = true; break; }
        relax();
      }
      if (!got) {
        std::unique_lock<std::mutex> lk(mu);
        sleeping.store(1);
        cv.wait(lk, [this]() { return has_job.load() != 0 || quit; });
        sleeping.store(0);
        if (!has_job.load()) return;  // quit
      }
      has_job.store(0);
      job();
      busy.store(0);
      { std::lock_guard<std::mutex> lk(mu); cv.notify_all(); }
    }
  }
  ~Worker() {
    if (started) {
      wait();
      { std::lock_guard<std::mutex> lk(mu); quit = true; cv.notify_all(); }
      th.join();
    }
  }
};

// ---- the optional parts of a context: each is off until its enable / attach call succeeds.  The call builds the part in a local and
// moves it in on success, so a call that fails half-way leaves the context as it was.

// /local/* publication (lio_est_enable_local_clouds): corner_stack_ / full_stack_ beside the surf slots.  The per-frame work runs on
// `stream`, forked from the scan's stream after the surf push and joined before SlideWindow.
struct LocalClouds {
  bool on = false, staged = false, pending = false;
  float corner_leaf = 0.2f;
  int cap[2] = {0, 0};             // corner, full points per slot (and per staged cloud)
  std::vector<DevMem<float4>> slot[2];   // physical slots [corner / full][slot], rotated through slot_of with the surf slots
  DevMem<int> d_slot_n;            // [0, W] corner counts per physical slot, [W + 1, 2W + 1] full counts
  DevMem<float4> d_stage[2];       // staged corner / full cloud of the next push
  DevMem<int> d_stage_n;           // [2]
  DevMem<float4> d_pub[3];         // published corner / surf / full of frame W - O (lio_mb_* argument order)
  DevMem<int> d_pub_n;             // [3]
  int pub_cap[3] = {0, 0, 0};
  VoxelGrid vg;                    // down_size_filter_corner_ (its own workspace: it runs beside the surf filter)
  Stream stream;
  Event ev_fork, ev_join;
};

// The global cube map after initialisation (lio_est_attach_map / lio_est_attach_mapping): the PointMapping the reference's Estimator
// is.  Its work runs on the map's stream, forked after the solve (ev_in) and joined at the next scan's entry and staging (ev_done).
struct AttachedMap {
  lio_pm *pm = nullptr;
  int scans = 0;                   // INITED scans since the attach: opt_point_coeff_mask_.first() is false from scan O on
  bool pending = false;
  DevMem<float4> d_keep[2];        // W == O with de-skew: the previous frame's corner / surf cloud, kept until its insert
  DevMem<int> d_keep_n;            // [2]
  Event ev_in, ev_done;
  lio::TwistF insert;              // opt_transforms_.first() of the last insert
  int info[4] = {0, 0, 0, 0};      // inserted, points inserted, surround published, last surround size
  void detach();                   // waits for the pending map work, then detaches the handle (the map is not owned)
};

// imu_factor = 0 from the odometry's clouds (lio_est_attach_mapping): the estimator's own PointMapping::Process on every message,
// the NOT_INITED window of the mapped poses and the start-up (ProcessCompactData / ProcessLaserOdom, Estimator.cc:430-856).
// imu_factor = 1 (lio_est_attach_imu_mapping): the same window, started by RunInitialization (:505-602, :858-958).
struct Mapping {
  bool on = false;
  bool inited = false;                // stage_flag_ == INITED
  bool quiet = false;                 // the start-up's solve: no estimator insert or publication on the NOT_INITED path
  int cir_count = 0, recv_count = 0;  // cir_buf_count_, laser_odom_recv_count_
  std::vector<lio::TwistF> laser_tf;  // all_laser_transforms_ (transform_aft_mapped_ of each push), logical frames
  std::vector<std::vector<size_t>> opt_valid;   // opt_valid_idx_, logical frames
  std::vector<std::array<int, 3>> opt_centre;   // opt_cube_centers_, logical frames
  int compact_info[4] = {0, 0, 0, 0}; // inited, cir_buf_count_, pushed by the last call, solved by the last call
  // imu_factor = 1
  double initial_time = -1;           // initial_time_: the stamp of the last attempt
  int attempts = 0, outcome = -1;     // RunInitialization calls, result of the last (kInit*)
  bool attempted = false;             // the last message ran an attempt
  M3 R_WI = M3::I();                  // R_WI_
  std::vector<double> attempt_states; // (W+1) x 16 (lio_est_get_states layout) as the last attempt left them, before any solve
};

// estimate_extrinsic = 2 on an IMU mapping (lio_est_enable_extrinsic_calibration): EstimateExtrinsicRotation before RunInitialization
struct ExtrinsicCalib {
  bool on = false;
  int runs = 0, result = -1;          // calls, result of the last (0 failed, 1 success)
  bool ran = false;                   // the last message ran one
  double sv[4] = {0, 0, 0, 0};        // the last call's singular values, descending
};

// Peer memory of a sharded context.  Rows exchange: one device allocation per rank, laid out as
//   [2 parities][kMaxOpt * kAsmStride doubles] | unsigned flag[kMaxPeers] | int err
// Feature exchange: all feature buffers (xyz+score, coefficients, counts) live in ONE allocation with two parities, so that a sharded
// run can exchange the features themselves once per scan (lio_est_set_feature_peers): every rank then owns all frames' features and
// the whole solve runs exactly like a single-GPU solve - no rendezvous inside the 11 evaluations.  The slab is also where a
// single-GPU context keeps its features.
constexpr size_t kXRowBytes = sizeof(double) * kMaxOpt * kAsmStride;
constexpr size_t kXFlagOff = 2 * kXRowBytes;
constexpr size_t kXErrOff = kXFlagOff + sizeof(unsigned) * kMaxPeers;
constexpr size_t kXBytes = kXErrOff + 64;

struct PeerExchange {
  DevMem<char> xbuf;
  char *peer_base[kMaxPeers] = {};
  int npeers = 0;
  unsigned xepoch = 0;
  DevMem<char> fslab;
  size_t fslab_bytes = 0, fpar_stride = 0, foff_cnt = 0, foff_flags = 0;
  std::vector<size_t> foff_pts, foff_coef;
  bool fpeers = false;
  char *fpeer_base[kMaxPeers] = {};
  unsigned fepoch = 0;
  int fparity = 0;
};

struct lio_est {
  lio_est_config cfg;
  MargJob mjob;
  Worker worker;
  PeerExchange px;
  Mat hp_exp;             // prior Hp scattered into the current tangent layout (cache of one solve)
  bool hp_exp_valid = false;
  struct ImuBlockStore { double JtJ[30 * 30], Jtr[30], cost; bool used; } imu_blocks_store[kMaxOpt];
  std::atomic<int> imu_next{0}, imu_done{0};  // shared pool of ImuFactor indices of one linearisation (caller + helper)
  double t_marg_wait = 0;
  char err[512] = "";         // text of the last failed call on THIS handle (lio_est_last_error)
  bool window_open = false;   // between lio_est_open_scan_* and lio_est_close_scan (stepwise API)
  bool poisoned = false;   // a scan failed half-way: the window bookkeeping is inconsistent, every later call fails fast
  int W = 0, O = 0, device = 0;
  cudaStream_t stream = 0;
  int sm_count = 132;
  // ---- host window state
  std::vector<V3> Ps, Vs, Bas, Bgs;
  std::vector<M3> Rs;
  std::vector<std::shared_ptr<Preintegration>> pre;
  std::shared_ptr<Preintegration> tmp_pre;
  ImuNoise noise;
  V3 acc_last, gyr_last, g_vec;
  bool first_imu = false;
  float tlb_q[4] = {0, 0, 0, 1}, tlb_p[3] = {0, 0, -0.1f};  // transform_lb_ (Twist<float>)
  std::vector<ImuStampedF> imu_stamped;
  std::vector<std::vector<double>> para_pose, para_sb;
  double para_ex[7];
  MargPrior prior;
  bool convergence_flag = false, init_local_map = false;
  int extrinsic_stage = 1;
  bool ex_constant = false;
  ExtrinsicCalib calib;
  // ---- device
  std::vector<DevMem<float4>> slot_ptr;   // physical slots
  std::vector<int> slot_of;          // logical frame -> physical slot
  DevMem<int> d_slot_n;              // counts per physical slot
  std::vector<int> size_surf_stack;  // host mirror of each frame's own size (logical)
  DevMem<int> d_own_n;               // device: own size per physical slot (for SlideWindow's skip)
  int slot_cap = 0;
  DevMem<float4> d_scan, d_local, d_map, d_tmp;
  int local_cap = 0;
  DevMem<int> d_counts;     // [0] scan n [1] local n [2] map n [3] tmp n
  VoxelGrid vg;
  CellHash hash;
  KnnWork knn;
  KnnWork knn2;                     // launch state of the LaserOdom chain, which runs beside the frame-batched k-NN launch
  Stream ostream;                   // stream of that chain
  Event ev_map, ev_odom;
  std::vector<FeatureOut> feats;  // logical frame index: pts / coef / count in the feature slab, src in feat_src
  std::vector<DevMem<int>> feat_src;
  int *d_feat_counts = nullptr;   // W+1 (inside the feature slab, current parity)
  DevMem<TransformF> d_tf;        // W+1
  HostMem<TransformF> h_tf;       // pinned
  AsmWork asmw;
  HostMem<double> h_Rt;     // pinned kMaxOpt*kAsmRtStride
  DevMem<double> d_Rt;
  HostMem<double> h_S;      // pinned kMaxOpt*kAsmStride
  HostMem<int> h_counts;    // pinned
  int *h_xerr = nullptr;    // h_counts + W + 10: the rows exchange's bounded-wait error word (the feature exchange's is W + 9)
  DevMem<OdomState> d_odom;
  DevMem<double> d_odom_partial;
  // ---- sharding
  int rank = 0, world = 1;
  lio_allreduce_fn allreduce = nullptr;
  void *allreduce_user = nullptr;
  // ---- results / stats
  std::vector<int> h_feat_n;
  int h_map_n = 0;
  std::vector<TransformF> local_tf;
  DoglegSummary summary;
  double cost_pim = 0, cost_ppp = 0, cost_marg = 0;
  bool turn_off = true;
  int odom_iters = 0;
  double t_build = 0, t_feat = 0, t_solve = 0, t_marg = 0, t_total = 0;
  bool S_pending = false;
  long long S_pending_feats = 0;
  double t_lin_wait = 0, t_lin_host = 0, t_lin_lidar = 0;  // per scan: blocked on the device / host factor work / lidar block expansion
  int launches = 0;
  Mat H0;
  Vec g0;
  double cost0 = 0;
  bool have_H0 = false;
  // device-resident solver
  DevSolver ds;
  bool use_dev_solver = false;
  // the device solver's launches of one solve, captured once and replayed (single-GPU contexts)
  Stream gstream;
  Graph sgraph;
  GraphExec sexec;                    // declared after sgraph, so destroyed before it
  std::vector<cudaGraphNode_t> asm_nodes;   // nodes of sgraph, re-parameterised on sexec every scan
  Event ev_gin, ev_gout;
  int graph_launches = 0;
  bool prior_uploaded = false;
  bool ds_prepared = false, ds_prepared_asm = false;   // solve_dev_prepare ran for the current parameters
  int ds_prepared_it = 0;
  Event evp[2 * 24];
  // cached lidar reduction for the current parameter values
  bool S_valid = false;
  // CUDA-event timing of the fused kernel (on the launching stream)
  Event ev0, ev1, evk0, evk1;
  double knn_ms_sum = 0;
  long long knn_launch_count = 0, knn_query_sum = 0;
  bool knn_timed = false;
  double asm_ms_sum = 0;
  long long asm_launch_count = 0, asm_feat_sum = 0;
  bool frames_started = false;        // an init_frame or scan has run: too late to enable local clouds
  bool scanned = false;               // a process_scan / open_scan has run: too late to attach a map
  TransformF es{0, 0, 0, 1, 0, 0, 0};   // transform_es_ (Estimator.h), kept across scans like the member
  LocalClouds lc;
  AttachedMap map;
  Mapping mapping;
  // The members go in reverse declaration order once these waits are done.  The running marginalisation job is joined first.  The
  // attached map's pending insert reads the estimator's slots and the map is not owned: it is waited for and the map detached before
  // any slot is freed.  The local clouds' stream is drained before its buffers and the slots it reads go.
  ~lio_est() {
    if (mjob.running) worker.wait();
    map.detach();
    if (lc.stream) cudaStreamSynchronize(lc.stream);
  }
};


template <typename T> void push_shift(std::vector<T> &v, T x) { v.erase(v.begin()); v.push_back(x); }

// transform_es_ is computed, and the attached map keeps or inserts the de-skewed clouds, whenever either de-skew flag is set
inline bool map_deskew(const lio_est *e) { return e->cfg.enable_deskew || e->cfg.cutoff_deskew; }

// ---- estimator.cu
Tw tlb_double(const lio_est *e);
Tw lidar_pose(const V3 &P, const M3 &R, const Tw &tlb);   // Estimator.cc:1387-1390
// k_copy_cloud: min(max(*n_src, 0), n_max) points and the count to *n_dst, on min(grid_cap, n_max / 256) blocks
void copy_cloud(const float4 *src, const int *n_src, int n_max, float4 *dst, int *n_dst, int grid_cap, cudaStream_t st);
// k_deskew: TransformToEnd of at most n_max points in place
void deskew(float4 *cloud, const int *n_dev, int n_max, TransformF es, float time_factor, bool keep_intensity, cudaStream_t st);
// A scan call that failed: its error text is kept on the handle (lio_est_last_error); with poison the window is left half-advanced,
// so every later scan call is refused.  Returns rc.
int scan_failed(lio_est *e, int rc, bool poison = true);
int refuse_poisoned(lio_est *e);   // sets the "context poisoned" error, returns LIO_ERR_INVALID
// A push of lio_est_process_compact_* (imu_factor = 0): surf_ds / surf_ds_n, when set, is PointMapping's down-sampled surf stack, copied
// into the frame slot instead of the VoxelGrid of the scan (:474-480); corner_filtered: the staged corner cloud is that stack's corner
// cloud, copied likewise; startup: the NOT_INITED push that reaches a full window (:505-517), no transform_es_.
// tmp_bg: Bgs_[W] as it was when the push made tmp_pre_integration_ (:453), before RunInitialization moved it.
struct CompactPush { const float4 *surf_ds; const int *surf_ds_n; bool corner_filtered, startup; V3 tmp_bg; };
int process_scan_body(lio_est *e, const float4 *scan_dev, const int *n_dev, int n_max, bool open_only, const CompactPush *cp = nullptr);

// ---- est_solve.cu
void set_feature_parity(lio_est *e, int par);
int build_local_map(lio_est *e, const std::function<int()> &before_sync = nullptr);
void vector_to_double(lio_est *e);
void double_to_vector(lio_est *e);
int linearize(lio_est *e, Mat &H, Vec &g, double &cost, double *c_pim, double *c_ppp, double *c_marg);
int marginalize(lio_est *e);
void marg_start(lio_est *e);
void prior_join(lio_est *e);
int solve_host(lio_est *e, int max_it);
int solve_dev_prepare(lio_est *e, int max_it, bool assemble_only);
int solve_dev(lio_est *e, int max_it, bool assemble_only);
int slide_window(lio_est *e);

// ---- est_map.cu
int lc_push(lio_est *e, bool deskew_corner, bool corner_filtered = false);
int lc_join(lio_est *e);
int map_scan_entry(lio_est *e, bool predict);
int map_step(lio_est *e);
void predict_state_w(lio_est *e);
