// lio_node: the reference's test_*.launch graph - lio_processor_node (src/processor_node.cc) and lio_estimator_node
// (src/estimator_node.cc: PointOdometry on its own thread, Estimator::ProcessEstimation on the measurement thread) - as one handle on
// one stream.  Stage A, the odometry, the estimator and its attached PointMapping are the existing handles; this unit only restates
// the glue between them: the /compact_data queue (the odometry's published clouds copied into HBM slots), MeasurementManager's
// pairing and ProcessEstimation's IMU loop (measure.cc), and the /enable_odom call.  No kernel of its own: the slot copies are the
// count-guarded copy_cloud of the estimator.  Optionally it also runs map_4D*.launch's map_builder_node on the estimator's /local/*
// clouds (lio_node_enable_map_builder) and feeds drive maps (lio_node_attach_registered_map): the map builder's kernels and
// lio_rm_insert_dev, enqueued on the same stream.  With lio_node_enable_odometry it keeps every pose the two nodes publish in host
// queues, read from host state the handles already hold.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <deque>
#include <new>
#include <vector>
#include "estimator.cuh"
#include "measure.h"
#include "regmap.cuh"

namespace {

struct Slot {                 // one published /compact_data message waiting for its IMU
  lio::DevMem<float4> cloud[3];   // /laser_cloud_corner_last, /laser_cloud_surf_last, the full cloud
  lio::DevMem<int> d_n;       // their device counts
  int n[3] = {};              // the same counts as the host knows them (the bounds handed on)
  float sum7[7] = {};         // transform_sum_
  double stamp = 0;           // header.stamp
};

struct MbRow {                // one map builder call: the set's stamp, transform_tobe_mapped_, transform_aft_mapped_, info6
  double stamp;
  float tobe7[7], aft7[7];
  int info6[6];
};

struct DriveMap {             // an attached lio_rm and the /cloud_registered it takes
  lio_rm *rm;
  int source;
};

// One odometry topic (lio_node_enable_odometry): a ring of capacity rows of 16 doubles {stamp, tf7, extras7, seq}; a push onto a full
// ring drops the oldest row, as a ROS publisher queue does
struct OdomTopic {
  std::vector<double> rows;
  int head = 0, count = 0;    // the oldest row and the number queued
  long long seq = 0;          // publications so far
  int capacity() const { return (int)rows.size() / 16; }
  void push(double stamp, const double tf7[7], const double *extra7) {
    const int cap = capacity();
    if (count == cap) { head = head + 1 == cap ? 0 : head + 1; --count; }
    const int tail = count < cap - head ? head + count : count - (cap - head);
    double *r = rows.data() + 16 * (size_t)tail;
    r[0] = stamp;
    std::memcpy(r + 1, tf7, 7 * sizeof(double));
    for (int k = 0; k < 7; ++k) r[8 + k] = extra7 ? extra7[k] : 0.0;
    r[15] = (double)++seq;
    ++count;
  }
};

static void widen7(const float *f, double *d) { for (int k = 0; k < 7; ++k) d[k] = (double)f[k]; }

// The sub-handles a node creates, destroyed through their own entries (each counts as one live resource)
template <class T, int (*Destroy)(T *)> struct DestroyHandle { void operator()(T *h) const { Destroy(h); } };
template <class T, int (*Destroy)(T *)> using SubHandle = lio::Own<T *, DestroyHandle<T, Destroy>>;

// create(&h) of one sub-handle; the node owns it from here
template <class T, class D, class F> int make(lio::Own<T *, D> &h, F create) {
  T *p = nullptr;
  const int rc = create(&p);
  if (rc == LIO_OK) h.take(cudaSuccess, p, nullptr);
  return rc;
}

}  // namespace

struct lio_node {
  lio_node_config cfg{};
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  lio::DevMem<float4> d_in;            // upload target of lio_node_push_sweep_host
  lio::DevMem<uint16_t> d_rings;
  std::vector<Slot> slots;
  // The sub-handles go before the node's own buffers, in the order mb, est, pm, po, pp (reverse declaration order): the estimator
  // detaches pm, so it goes before pm.
  SubHandle<lio_pp, lio_pp_destroy> pp;
  SubHandle<lio_po, lio_po_destroy> po;
  SubHandle<lio_pm, lio_pm_destroy> pm;
  SubHandle<lio_est, lio_est_destroy> est;
  SubHandle<lio_pm, lio_pm_destroy> mb;   // lio_node_enable_map_builder
  std::vector<int> free_slots;
  lio::MeasurementPairing pairing{0};
  std::vector<lio::ImuMsg> list;
  std::vector<lio::ImuCall> calls;
  long long po_calls = 0;              // successful odometry calls (the io_ratio gate follows from them)
  long long sweeps = 0, published = 0, processed = 0, dropped = 0;
  bool odom_on = true, inited = false, poisoned = false;
  double last_stamp = -1;
  std::deque<double> headers;          // Headers_ (Estimator.cc:441): the stamps of the last W + 1 pushed messages
  std::vector<MbRow> mb_rows;
  std::vector<DriveMap> maps;          // lio_node_attach_registered_map, in attach order
  bool odometry = false;               // lio_node_enable_odometry
  OdomTopic topics[LIO_NODE_ODOM_TOPICS];
  std::vector<double> states;          // (W + 1) x 16, lio_est_get_states for /predict_odom
};

static bool ring_sensor(const lio_node *nd) { return nd->cfg.sensor_type == 320; }

// processor_node.cc:72-73: only the 320 preset reads the ring field (an empty sweep may come without it)
static int check_rings(const lio_node *nd, bool has_rings, int n) {
  if (ring_sensor(nd) ? (has_rings || n == 0) : !has_rings) return LIO_OK;
  lio_set_last_error(__FILE__, __LINE__, "lio_node: rings are required with sensor_type 320 and refused otherwise");
  return LIO_ERR_INVALID;
}

extern "C" void lio_node_default_config(lio_node_config *c) {
  if (!c) return;
  std::memset(c, 0, sizeof(*c));
  c->sensor_type = 16;
  lio_pp_default_config(&c->pp);
  c->odom_io = 2;                       // PointOdometry(scan_period, io_ratio = 2) default
  c->msg_time_delay = 0;                // MeasurementManager.h:78
  lio_est_default_config(&c->est);
  c->tf_lb7[3] = 1.0f;
  c->corner_filter_size = 0.2f;         // PointMapping leaves (config/*.yaml)
  c->surf_filter_size = 0.4f;
  c->map_filter_size = 0.6f;
  c->max_points = 1 << 18;
  c->max_feature_points = 1 << 16;
  c->max_pending = 16;
}

extern "C" int lio_node_create(const lio_node_config *cfg, int device, void *cuda_stream, lio_node **out) {
  if (!cfg || !out) return LIO_ERR_INVALID;
  *out = nullptr;
  const int st = cfg->sensor_type;
  if ((st != 16 && st != 32 && st != 64 && st != 320) || cfg->odom_io < 1 || !(cfg->msg_time_delay >= 0) || cfg->max_points <= 0 ||
      cfg->max_feature_points <= 0 || cfg->max_pending < 1 || !(cfg->map_filter_size > 0)) {
    lio_set_last_error(__FILE__, __LINE__, "lio_node_create: sensor_type must be 16, 32, 64 or 320; odom_io, capacities and max_pending >= 1");
    return LIO_ERR_INVALID;
  }
  std::unique_ptr<lio_node> nd(new (std::nothrow) lio_node());
  if (!nd) return LIO_ERR_INVALID;
  LIO_TRY(select_device(device, &nd->sm_count));
  nd->cfg = *cfg;
  nd->device = device;
  nd->stream = (cudaStream_t)cuda_stream;
  nd->pairing = lio::MeasurementPairing(cfg->msg_time_delay);
  // processor_node.cc:64-74: the sensor presets (320 = RS-32 with the ring field)
  lio_pp_config pc = cfg->pp;
  if (st == 16) { pc.lower_bound = -15.f; pc.upper_bound = 15.f; pc.num_rings = 16; }
  else if (st == 32) { pc.lower_bound = -30.67f; pc.upper_bound = 10.67f; pc.num_rings = 32; }
  else if (st == 64) { pc.lower_bound = -24.9f; pc.upper_bound = 2.f; pc.num_rings = 64; }
  else { pc.lower_bound = -25.f; pc.upper_bound = 15.f; pc.num_rings = 32; }
  const int F = cfg->max_feature_points, N = cfg->max_points;
  const lio_est_config &ec = cfg->est;
  int rc;
  if ((rc = make(nd->pp, [&](lio_pp **h) { return lio_pp_create(&pc, N, device, cuda_stream, h); })) != LIO_OK) return rc;
  // estimator_node.cc:145-147: PointOdometry(0.1, odom_io) with its default 25 iterations
  if ((rc = make(nd->po, [&](lio_po **h) { return lio_po_create(0.1f, cfg->odom_io, 25, F, N, device, cuda_stream, h); })) != LIO_OK) return rc;
  // the Estimator is a PointMapping (num_max_iterations_ 10, PointMapping.h:171) with the YAML's leaves
  if ((rc = make(nd->pm, [&](lio_pm **h) {
         return lio_pm_create(F, cfg->corner_filter_size, cfg->surf_filter_size, ec.min_match_sq_dis, ec.min_plane_dis, 10, device, cuda_stream, h);
       })) != LIO_OK)
    return rc;
  if ((rc = lio_pm_enable_publish(nd->pm, cfg->map_filter_size, N)) != LIO_OK) return rc;
  if ((rc = make(nd->est, [&](lio_est **h) { return lio_est_create(&ec, device, cuda_stream, h); })) != LIO_OK) return rc;
  if ((rc = lio_est_set_extrinsic(nd->est, cfg->tf_lb7)) != LIO_OK) return rc;
  if ((rc = lio_est_enable_local_clouds(nd->est, cfg->corner_filter_size, F, N)) != LIO_OK) return rc;
  if (ec.imu_factor && ec.estimate_extrinsic == 2 && (rc = lio_est_enable_extrinsic_calibration(nd->est)) != LIO_OK) return rc;
  rc = ec.imu_factor ? lio_est_attach_imu_mapping(nd->est, nd->pm) : lio_est_attach_mapping(nd->est, nd->pm);
  if (rc != LIO_OK) return rc;
  nd->slots.resize(cfg->max_pending);
  for (int k = cfg->max_pending - 1; k >= 0; --k) {
    Slot &s = nd->slots[k];
    if (!lio::alloc(s.cloud[0], F) || !lio::alloc(s.cloud[1], F) || !lio::alloc(s.cloud[2], N) || !lio::alloc(s.d_n, 3)) {
      lio_set_last_error(__FILE__, __LINE__, "lio_node_create: cudaMalloc of a queue slot failed");
      return LIO_ERR_CUDA;
    }
    nd->free_slots.push_back(k);
  }
  *out = nd.release();
  return LIO_OK;
}

extern "C" int lio_node_destroy(lio_node *nd) {
  if (!nd) return LIO_OK;
  cudaSetDevice(nd->device);   // the buffers belong to the node's device, whichever is current
  delete nd;
  return LIO_OK;
}

// map_builder_node on the set the estimator has just published (INITED messages only, see lio_node_enable_map_builder): its /local/*
// clouds and /local_laser_odom as they lie in HBM, on the node's stream; then the pose row.
static int map_builder_step(lio_node *nd) {
  const float *ptr[3];
  const int *n_dev = nullptr;
  int n_host[3];
  MbRow row{};
  int rc = lio_est_local_clouds_dev(nd->est, ptr, &n_dev, n_host);
  float sum7[7];
  if (rc == LIO_OK) rc = lio_est_local_laser_odom(nd->est, sum7);
  if (rc == LIO_OK) rc = lio_mb_process_map_dev(nd->mb, ptr[0], ptr[1], ptr[2], n_dev, n_host, sum7, row.tobe7, row.aft7, row.info6);
  if (rc != LIO_OK) return rc;
  // Headers_[pivot_idx + 1] (Estimator.cc:727, :2364), the stamp of both the clouds and /local_laser_odom: Headers_ is full (W + 1)
  // once INITED, so this is the message pushed O - 1 pushes before the newest
  row.stamp = nd->headers[nd->headers.size() - nd->cfg.est.opt_window_size];
  nd->mb_rows.push_back(row);
  return LIO_OK;
}

// save_bag_to_pcd on the attached maps: the registered cloud of every publication of their source, stream-ordered, no host wait.
static int insert_registered(lio_node *nd, int source) {
  const float *p = nullptr;
  int n = 0, rc = LIO_OK;
  for (const DriveMap &d : nd->maps) {
    if (d.source != source) continue;
    if (!p && (rc = lio_mb_full_dev(source == LIO_NODE_MAP_ESTIMATOR ? nd->pm : nd->mb, &p, &n)) != LIO_OK) return rc;
    if ((rc = lio_rm_insert_dev(d.rm, p, n)) != LIO_OK) return rc;
  }
  return LIO_OK;
}

// /predict_odom after a ProcessImu call made INITED (Estimator.cc:406-425): Ps_.last(), Quaterniond(Rs_.last()), Vs_.last() and
// Bas_.last() (the reference's twist.angular) are row W of lio_est_get_states; the stamp is the IMU message's that the call carries
// (:2706, :2725).
static int record_predict_odom(lio_node *nd, double stamp) {
  LIO_TRY(lio_est_get_states(nd->est, nd->states.data()));
  const double *s = nd->states.data() + 16 * nd->cfg.est.window_size;
  const double tf7[7] = {s[3], s[4], s[5], s[6], s[0], s[1], s[2]};
  const double v_ba[7] = {s[7], s[8], s[9], s[10], s[11], s[12], 0.0};
  nd->topics[LIO_NODE_ODOM_PREDICT_ODOM].push(stamp, tf7, v_ba);
  return LIO_OK;
}

// The estimator's publications of one processed message (see lio_node_enable_odometry), once its call has returned: /aft_mapped_to_init
// always, /extrinsic_lb when the call solved, /predict_laser_odom and /local_laser_odom when the message arrived INITED.
static int record_message(lio_node *nd, const Slot &s, bool was_inited, bool solved) {
  float f7[7];
  double tf7[7];
  // PointMapping::PublishResults (PointMapping.cc:1255-1276): transform_aft_mapped_, stamped time_laser_odometry_ (:230)
  LIO_TRY(lio_est_map_poses(nd->est, nullptr, f7, nullptr, nullptr));
  widen7(f7, tf7);
  nd->topics[LIO_NODE_ODOM_AFT_MAPPED_TO_INIT].push(s.stamp, tf7, nullptr);
  if (solved) {   // SolveOptimization's update_laser_imu block (Estimator.cc:2343-2353): transform_lb_.cast<double>(), Headers_.last()
    LIO_TRY(lio_est_get_extrinsic(nd->est, f7));
    widen7(f7, tf7);
    nd->topics[LIO_NODE_ODOM_EXTRINSIC_LB].push(nd->headers.back(), tf7, nullptr);
  }
  if (was_inited) {   // ProcessLaserOdom's INITED branch after SlideWindow (:725-758), outside the opt_point_coeff_map_ check
    double local7[7];
    LIO_TRY(lio_est_laser_odom(nd->est, tf7, local7));
    nd->topics[LIO_NODE_ODOM_PREDICT_LASER_ODOM].push(s.stamp, tf7, nullptr);
    nd->topics[LIO_NODE_ODOM_LOCAL_LASER_ODOM].push(nd->headers[nd->headers.size() - nd->cfg.est.opt_window_size], local7, nullptr);
  }
  return LIO_OK;
}

// One released message: ProcessEstimation's ProcessImu calls, then ProcessCompactData on its slot (Estimator.cc:2682-2736), then the
// /enable_odom call of the RunInitialization success path (:542-560); with odometry topics, the message's rows; with a map builder, its
// call when the message arrived INITED; then the drive-map inserts.  Any failure poisons the node.
static int process_message(lio_node *nd, const Slot &s) {
  nd->calls.clear();
  nd->pairing.integrate(s.stamp, nd->list, &nd->calls);
  int rc = LIO_OK;
  const bool was_inited = nd->inited;
  for (const lio::ImuCall &c : nd->calls) {
    if ((rc = lio_est_process_imu(nd->est, c.dt, c.acc, c.gyr, c.stamp)) != LIO_OK) break;
    if (nd->odometry && was_inited && (rc = record_predict_odom(nd, c.stamp)) != LIO_OK) break;
  }
  if (rc == LIO_OK) rc = lio_est_process_compact_stamped_dev(nd->est, (const float *)s.cloud[0].get(), (const float *)s.cloud[1].get(), (const float *)s.cloud[2].get(),
                                                            s.d_n, s.n, s.sum7, s.stamp);
  int info[4] = {};
  if (rc == LIO_OK) rc = lio_est_compact_status(nd->est, info);
  if (rc != LIO_OK) { nd->poisoned = true; return rc; }
  ++nd->processed;
  nd->last_stamp = s.stamp;
  if (info[2]) {   // the message passed the init_window_factor gate (:436-439) and was pushed: Headers_.push(header) (:441)
    nd->headers.push_back(s.stamp);
    if ((int)nd->headers.size() > nd->cfg.est.window_size + 1) nd->headers.pop_front();
  }
  const bool now_inited = info[0] != 0;
  const lio_est_config &ec = nd->cfg.est;
  if (ec.imu_factor && !nd->inited && now_inited && (ec.enable_deskew || ec.cutoff_deskew)) {
    if ((rc = lio_po_set_enable_odom(nd->po, 0)) != LIO_OK) { nd->poisoned = true; return rc; }
    nd->odom_on = false;
  }
  nd->inited = now_inited;
  if (nd->odometry && (rc = record_message(nd, s, was_inited, info[3] != 0)) != LIO_OK) { nd->poisoned = true; return rc; }
  if (nd->mb && was_inited && (rc = map_builder_step(nd)) != LIO_OK) { nd->poisoned = true; return rc; }
  // the estimator's PointMapping publishes /cloud_registered once per processed message (see lio_node_attach_registered_map)
  if ((rc = insert_registered(nd, LIO_NODE_MAP_ESTIMATOR)) != LIO_OK) { nd->poisoned = true; return rc; }
  if (nd->mb && was_inited && (rc = insert_registered(nd, LIO_NODE_MAP_BUILDER)) != LIO_OK) { nd->poisoned = true; return rc; }
  return LIO_OK;
}

// GetMeasurements until it waits: every message it releases is processed, every one it drops frees its slot.
static int drain(lio_node *nd) {
  for (;;) {
    int id = -1;
    double t = 0;
    const lio::MeasurementPairing::Decision d = nd->pairing.next(&id, &t, &nd->list);
    if (d == lio::MeasurementPairing::kWait) return LIO_OK;
    nd->free_slots.push_back(id);
    if (d == lio::MeasurementPairing::kDropped) { ++nd->dropped; continue; }
    const int rc = process_message(nd, nd->slots[id]);
    if (rc != LIO_OK) return rc;
  }
}

static int refuse_poisoned(lio_node *nd) {
  if (!nd->poisoned) return LIO_OK;
  lio_set_last_error(__FILE__, __LINE__, "lio_node: an earlier estimator or map builder failure poisoned the node; destroy and re-create it");
  return LIO_ERR_INVALID;
}

extern "C" int lio_node_push_imu_batch(lio_node *nd, int n, const double *stamp, const double *acc3, const double *gyr3) {
  LIO_ENTER(nd);
  if (n < 0 || (n > 0 && (!stamp || !acc3 || !gyr3))) return LIO_ERR_INVALID;
  int rc = refuse_poisoned(nd);
  if (rc != LIO_OK) return rc;
  for (int k = 0; k < n; ++k) {
    lio::ImuMsg m{stamp[k], {acc3[3 * k], acc3[3 * k + 1], acc3[3 * k + 2]}, {gyr3[3 * k], gyr3[3 * k + 1], gyr3[3 * k + 2]}};
    if (nd->pairing.push_imu(m) && (rc = drain(nd)) != LIO_OK) return rc;
  }
  return LIO_OK;
}

extern "C" int lio_node_push_imu(lio_node *nd, double stamp, const double acc[3], const double gyr[3]) {
  LIO_ENTER(nd);
  if (!acc || !gyr) return LIO_ERR_INVALID;
  return lio_node_push_imu_batch(nd, 1, &stamp, acc, gyr);
}

extern "C" int lio_node_push_sweep_dev(lio_node *nd, const float *xyzi_dev, const uint16_t *rings_dev, int n, double stamp) {
  LIO_ENTER(nd);
  if (n < 0 || (n > 0 && !xyzi_dev) || std::isnan(stamp)) return LIO_ERR_INVALID;
  int rc = check_rings(nd, rings_dev != nullptr, n);
  if (rc != LIO_OK) return rc;
  if ((rc = refuse_poisoned(nd)) != LIO_OK) return rc;
  if (n > nd->cfg.max_points) return LIO_ERR_CAPACITY;
  // the io_ratio gate of the coming odometry call (PointOdometry.cc:302-310, :725): the first call never publishes
  const long long c = nd->po_calls;
  const bool will_publish = c >= 1 && (nd->cfg.odom_io < 2 || c % nd->cfg.odom_io == 1);
  if (will_publish && nd->free_slots.empty()) {
    lio_set_last_error(__FILE__, __LINE__, "lio_node: the /compact_data queue is full (max_pending messages wait for IMU)");
    return LIO_ERR_CAPACITY;
  }
  rc = ring_sensor(nd) ? lio_pp_process_dev_ring(nd->pp, xyzi_dev, rings_dev, n) : lio_pp_process_dev(nd->pp, xyzi_dev, n);
  if (rc != LIO_OK) return rc;
  static const int which[5] = {LIO_PP_CORNER_SHARP, LIO_PP_CORNER_LESS_SHARP, LIO_PP_SURF_FLAT, LIO_PP_SURF_LESS_FLAT, LIO_PP_CLOUD_IN_RINGS};
  const float *clouds[5];
  const int *counts[5];
  for (int k = 0; k < 5; ++k) {
    if ((rc = lio_pp_cloud_dev(nd->pp, which[k], &clouds[k])) != LIO_OK) return rc;
    if ((rc = lio_pp_cloud_count_dev(nd->pp, which[k], &counts[k])) != LIO_OK) return rc;
  }
  const int F = nd->cfg.max_feature_points;
  const int n_max[5] = {F, F, F, F, nd->cfg.max_points};
  float sum7[7], es7[7];
  int info4[4];
  if ((rc = lio_po_process_dev(nd->po, clouds, counts, n_max, sum7, es7, info4)) != LIO_OK) return rc;
  ++nd->po_calls;
  ++nd->sweeps;
  if (nd->odometry && c >= 1) {   // PublishResults (:681-721), pass-through included: transform_sum_, then transform_es_ as the extras
    double tf7[7], ex7[7];
    widen7(sum7, tf7);
    widen7(es7, ex7);
    nd->topics[LIO_NODE_ODOM_LASER_ODOM_TO_INIT].push(stamp, tf7, ex7);
  }
  if (info4[1]) {   // published (:727): copy the three clouds, transform_sum_ and the stamp into a queue slot
    const float *ptr[3];
    const int *n_dev;
    int n_host[3];
    if ((rc = lio_po_clouds_dev(nd->po, ptr, &n_dev, n_host)) != LIO_OK) return rc;
    const int id = nd->free_slots.back();
    nd->free_slots.pop_back();
    Slot &s = nd->slots[id];
    for (int w = 0; w < 3; ++w) {
      copy_cloud(reinterpret_cast<const float4 *>(ptr[w]), n_dev + w, n_host[w], s.cloud[w], s.d_n + w, 2 * nd->sm_count, nd->stream);
      s.n[w] = n_host[w];
    }
    LIO_CUDA_OK(cudaGetLastError());
    std::memcpy(s.sum7, sum7, sizeof(sum7));
    s.stamp = stamp;
    nd->pairing.push_message(id, stamp);
    ++nd->published;
  }
  return drain(nd);
}

extern "C" int lio_node_push_sweep_host(lio_node *nd, const float *xyzi, const uint16_t *rings, int n, double stamp) {
  LIO_ENTER(nd);
  if (n < 0 || (n > 0 && !xyzi) || std::isnan(stamp)) return LIO_ERR_INVALID;
  int rc = check_rings(nd, rings != nullptr, n);
  if (rc != LIO_OK) return rc;
  if ((rc = refuse_poisoned(nd)) != LIO_OK) return rc;
  if (n > nd->cfg.max_points) return LIO_ERR_CAPACITY;
  if (!nd->d_in && !lio::alloc(nd->d_in, nd->cfg.max_points)) return LIO_ERR_CUDA;
  if (rings && !nd->d_rings && !lio::alloc(nd->d_rings, nd->cfg.max_points)) return LIO_ERR_CUDA;
  if (n > 0) {
    LIO_CUDA_OK(cudaMemcpyAsync(nd->d_in, xyzi, sizeof(float4) * n, cudaMemcpyHostToDevice, nd->stream));
    if (rings) LIO_CUDA_OK(cudaMemcpyAsync(nd->d_rings, rings, sizeof(uint16_t) * n, cudaMemcpyHostToDevice, nd->stream));
  }
  rc = lio_node_push_sweep_dev(nd, (const float *)nd->d_in.get(), rings ? nd->d_rings.get() : nullptr, n, stamp);
  const cudaError_t e = cudaStreamSynchronize(nd->stream);   // the caller's buffers may be reused on return
  if (rc == LIO_OK && e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return rc;
}

extern "C" int lio_node_status(lio_node *nd, lio_node_info *s) {
  LIO_ENTER_HOST(nd);
  if (!s) return LIO_ERR_INVALID;
  s->sweeps = nd->sweeps;
  s->published = nd->published;
  s->processed = nd->processed;
  s->dropped = nd->dropped;
  s->pending = nd->pairing.pending();
  s->imu_dropped = nd->pairing.imu_dropped();
  s->odom_enabled = nd->odom_on ? 1 : 0;
  s->inited = nd->inited ? 1 : 0;
  s->poisoned = nd->poisoned ? 1 : 0;
  s->last_stamp = nd->last_stamp;
  return LIO_OK;
}

extern "C" int lio_node_handles(lio_node *nd, lio_pp **pp, lio_po **po, lio_est **est, lio_pm **pm) {
  LIO_ENTER_HOST(nd);
  if (pp) *pp = nd->pp;
  if (po) *po = nd->po;
  if (est) *est = nd->est;
  if (pm) *pm = nd->pm;
  return LIO_OK;
}

extern "C" int lio_node_enable_map_builder(lio_node *nd, const lio_mb_config *cfg) {
  LIO_ENTER(nd);
  if (!cfg) return LIO_ERR_INVALID;
  if (nd->mb || nd->sweeps > 0 || nd->poisoned) {
    lio_set_last_error(__FILE__, __LINE__, "lio_node_enable_map_builder: once, before the first sweep");
    return LIO_ERR_INVALID;
  }
  const float *ptr[3];
  const int *n_dev = nullptr;
  int n_host[3];
  LIO_TRY(lio_est_local_clouds_dev(nd->est, ptr, &n_dev, n_host));
  return make(nd->mb, [&](lio_pm **h) { return lio_mb_create(cfg, std::max(n_host[0], n_host[1]), n_host[2], nd->device, nd->stream, h); });
}

extern "C" int lio_node_map_builder(lio_node *nd, lio_pm **mb) {
  LIO_ENTER_HOST(nd);
  if (!mb) return LIO_ERR_INVALID;
  *mb = nd->mb;
  if (nd->mb) return LIO_OK;
  lio_set_last_error(__FILE__, __LINE__, "lio_node_map_builder: no map builder (lio_node_enable_map_builder)");
  return LIO_ERR_INVALID;
}

extern "C" int lio_node_map_builder_poses(lio_node *nd, double *stamp, float *tobe7, float *aft7, int *info6, int cap, int *n) {
  LIO_ENTER_HOST(nd);
  if (!n || cap < 0) return LIO_ERR_INVALID;
  if (!nd->mb) {
    lio_set_last_error(__FILE__, __LINE__, "lio_node_map_builder_poses: no map builder (lio_node_enable_map_builder)");
    return LIO_ERR_INVALID;
  }
  const int rows = (int)nd->mb_rows.size();
  *n = rows;
  if (rows > cap) return LIO_ERR_CAPACITY;
  for (int r = 0; r < rows; ++r) {
    const MbRow &row = nd->mb_rows[r];
    if (stamp) stamp[r] = row.stamp;
    if (tobe7) std::memcpy(tobe7 + 7 * r, row.tobe7, sizeof(row.tobe7));
    if (aft7) std::memcpy(aft7 + 7 * r, row.aft7, sizeof(row.aft7));
    if (info6) std::memcpy(info6 + 6 * r, row.info6, sizeof(row.info6));
  }
  return LIO_OK;
}

extern "C" int lio_node_enable_odometry(lio_node *nd, int capacity) {
  LIO_ENTER_HOST(nd);
  if (capacity < 1 || nd->odometry || nd->sweeps > 0 || nd->poisoned) {
    lio_set_last_error(__FILE__, __LINE__, "lio_node_enable_odometry: capacity >= 1, once, before the first sweep, on a node that is not poisoned");
    return LIO_ERR_INVALID;
  }
  try {
    for (OdomTopic &t : nd->topics) t.rows.assign(16 * (size_t)capacity, 0.0);
    nd->states.assign(16 * (size_t)(nd->cfg.est.window_size + 1), 0.0);
  } catch (const std::bad_alloc &) {
    for (OdomTopic &t : nd->topics) std::vector<double>().swap(t.rows);
    lio_set_last_error(__FILE__, __LINE__, "lio_node_enable_odometry: the queues do not fit in host memory");
    return LIO_ERR_CAPACITY;
  }
  nd->odometry = true;
  return LIO_OK;
}

extern "C" int lio_node_take_odometry(lio_node *nd, int topic, double *rows16, int cap, int *n, int *left) {
  LIO_ENTER_HOST(nd);
  if (!n || cap < 0 || (cap > 0 && !rows16)) return LIO_ERR_INVALID;
  *n = 0;
  const char *why = nullptr;
  if (topic < 0 || topic >= LIO_NODE_ODOM_TOPICS) why = "lio_node_take_odometry: unknown topic";
  else if (!nd->odometry) why = "lio_node_take_odometry: no odometry topics (lio_node_enable_odometry)";
  if (why) { lio_set_last_error(__FILE__, __LINE__, why); return LIO_ERR_INVALID; }
  OdomTopic &t = nd->topics[topic];
  const int k = std::min(cap, t.count), size = t.capacity();
  for (int r = 0; r < k; ++r) {
    std::memcpy(rows16 + 16 * (size_t)r, t.rows.data() + 16 * (size_t)t.head, 16 * sizeof(double));
    t.head = t.head + 1 == size ? 0 : t.head + 1;
  }
  t.count -= k;
  *n = k;
  if (left) *left = t.count;
  return LIO_OK;
}

extern "C" int lio_node_attach_registered_map(lio_node *nd, lio_rm *rm, int source) {
  LIO_ENTER_HOST(nd);
  if (!rm) return LIO_ERR_INVALID;
  const char *why = nullptr;
  if (source != LIO_NODE_MAP_ESTIMATOR && source != LIO_NODE_MAP_BUILDER) why = "lio_node_attach_registered_map: unknown source";
  else if (source == LIO_NODE_MAP_BUILDER && !nd->mb) why = "lio_node_attach_registered_map: the map builder's source needs lio_node_enable_map_builder first";
  else if (rm_device(rm) != nd->device || rm_stream(rm) != nd->stream) why = "lio_node_attach_registered_map: the map must be on the node's device and stream";
  else if (nd->poisoned) why = "lio_node_attach_registered_map: the node is poisoned";
  for (const DriveMap &d : nd->maps)
    if (!why && d.rm == rm) why = "lio_node_attach_registered_map: the map is attached already";
  if (why) { lio_set_last_error(__FILE__, __LINE__, why); return LIO_ERR_INVALID; }
  nd->maps.push_back(DriveMap{rm, source});
  return LIO_OK;
}
