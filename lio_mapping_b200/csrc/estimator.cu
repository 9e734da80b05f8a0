// lio::Estimator (steady state) on sm_90a — the host shell keeps the reference's control flow
// (window bookkeeping, gates, slide; src/imu_processor/Estimator.cc) while every per-point /
// per-feature loop runs in the CUDA kernels of this library:
//   ProcessLaserOdom INITED branch :618-774 -> process_scan   (de-skew kernel, device VoxelGrid)
//   BuildLocalMap :1361-1646                -> build_local_map (est_solve.cu: concat+transform kernel, VoxelGrid, cell hash,
//                                              voxel-hash kNN + plane fit per frame, device LaserOdom chain)
//   SolveOptimization :1648-2438            -> solve_host / solve_dev (est_solve.cu: fused residual+Jacobian+J^T J kernel per
//                                              iteration, dogleg controller, marginalisation)
//   SlideWindow :2570-2666                  -> slide_window (est_solve.cu)
// There is no CPU path for the per-point work: without a CUDA device create() fails.
#include "estimator.cuh"

namespace lio {

// TransformToEnd (Estimator.cc:62-103), in place; keep_intensity leaves the intensity as is (the full-cloud call, :2416)
__global__ void __launch_bounds__(256)
k_deskew(float4 *__restrict__ cloud, const int *__restrict__ n_dev, TransformF es, float time_factor, bool keep_intensity = false) {
  const int n = *n_dev;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = cloud[i];
  float s = time_factor * (p.w - (float)(int)p.w);
  p.x -= s * es.px; p.y -= s * es.py; p.z -= s * es.pz;
  if (!keep_intensity) p.w -= (float)(int)p.w;
  // q_s = identity.slerp(s, q_e)  (Eigen QuaternionBase::slerp)
  const float one = 1.0f - FLT_EPSILON;
  float d = es.qw;  // identity . q_e
  float absD = fabsf(d);
  float scale0, scale1;
  if (absD >= one) { scale0 = 1.0f - s; scale1 = s; }
  else {
    float theta = acosf(absD);
    float sinTheta = sinf(theta);
    scale0 = sinf((1.0f - s) * theta) / sinTheta;
    scale1 = sinf(s * theta) / sinTheta;
  }
  if (d < 0.f) scale1 = -scale1;
  float sw = scale0 + scale1 * es.qw, sx = scale1 * es.qx, sy = scale1 * es.qy, sz = scale1 * es.qz;
  // q_s.conjugate().normalized()
  float nn = sqrtf(sx * sx + sy * sy + sz * sz + sw * sw);
  float cx = -sx / nn, cy = -sy / nn, cz = -sz / nn, cw = sw / nn;
  float ax, ay, az;
  odom_qmul_vec(cx, cy, cz, cw, p.x, p.y, p.z, ax, ay, az);
  float bx, by, bz;
  odom_qmul_vec(es.qx, es.qy, es.qz, es.qw, ax, ay, az, bx, by, bz);
  cloud[i] = make_float4(bx + es.px, by + es.py, bz + es.pz, p.w);
}

// Count-guarded cloud copy: min(max(*n_src, 0), n_max) points, the count itself to *n_dst (src, dst and the counts do not alias)
__global__ void __launch_bounds__(256)
k_copy_cloud(const float4 *__restrict__ src, const int *__restrict__ n_src, int n_max, float4 *__restrict__ dst, int *__restrict__ n_dst) {
  const int n = min(max(*n_src, 0), n_max);
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_dst = n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = __ldg(src + i);
}

}  // namespace lio

void deskew(float4 *cloud, const int *n_dev, int n_max, TransformF es, float time_factor, bool keep_intensity, cudaStream_t st) {
  k_deskew<<<(n_max + 255) / 256, 256, 0, st>>>(cloud, n_dev, es, time_factor, keep_intensity);
}

void copy_cloud(const float4 *src, const int *n_src, int n_max, float4 *dst, int *n_dst, int grid_cap, cudaStream_t st) {
  k_copy_cloud<<<std::max(1, std::min(grid_cap, (n_max + 255) / 256)), 256, 0, st>>>(src, n_src, n_max, dst, n_dst);
}

Tw tlb_double(const lio_est *e) {
  return Tw(Q(e->tlb_q[3], e->tlb_q[0], e->tlb_q[1], e->tlb_q[2]), V3(e->tlb_p[0], e->tlb_p[1], e->tlb_p[2]));
}

Tw lidar_pose(const V3 &P, const M3 &R, const Tw &tlb) {
  Q rot = fromR(R * toR(inverse(tlb.rot)));
  V3 pos = P - rotate(rot, tlb.pos);
  return Tw(rot, pos);
}

// ---- creation -----------------------------------------------------------------------------------
extern "C" void lio_est_default_config(lio_est_config *c) {
  c->window_size = 10; c->opt_window_size = 10;
  c->min_match_sq_dis = 1.0f; c->min_plane_dis = 0.2f; c->surf_filter_size = 0.4f;
  c->keep_features = 0; c->estimate_extrinsic = 1; c->opt_extrinsic = 1;
  c->imu_factor = 1; c->point_distance_factor = 1; c->prior_factor = 0; c->marginalization_factor = 1;
  c->enable_deskew = 1; c->cutoff_deskew = 1;
  c->acc_n = 0.2; c->gyr_n = 0.02; c->acc_w = 2e-4; c->gyr_w = 2e-5; c->g_norm = 9.805;
  c->max_num_iterations = 10; c->odom_max_iterations = 10;
  c->max_frame_points = 1 << 16; c->max_scan_points = 1 << 18;
  c->device_solver = 1;   // GPU-resident dogleg loop (solver_dev.cu; O = 14..16 on a two-CTA cluster); 0 keeps the host controller
  c->overlap_marginalization = 1;
  c->solver_graph = 1;
  c->init_window_factor = 1;
}

extern "C" int lio_est_destroy(lio_est *e) {
  if (!e) return LIO_OK;
  cudaSetDevice(e->device);   // the resources belong to the context's device, whichever is current
  delete e;
  return LIO_OK;
}

extern "C" int lio_est_create(const lio_est_config *cfg, int device, void *cuda_stream, lio_est **out) {
  if (!cfg || !out) return LIO_ERR_INVALID;
  const int W = cfg->window_size, O = cfg->opt_window_size;
  if (W < 1 || W >= kMaxWindow || O < 1 || O > W || O > kMaxOpt || cfg->max_frame_points < 16 || cfg->max_scan_points < 16 ||
      !(cfg->surf_filter_size > 0) || !(cfg->min_match_sq_dis > 0) || cfg->odom_max_iterations < 1 || cfg->init_window_factor < 1) {
    lio_set_last_error(__FILE__, __LINE__, "lio_est_create: configuration outside supported limits");
    return LIO_ERR_INVALID;
  }
  std::unique_ptr<lio_est> e(new (std::nothrow) lio_est());
  if (!e) return LIO_ERR_INVALID;
  LIO_TRY(select_device(device, &e->sm_count));
  e->cfg = *cfg; e->W = W; e->O = O; e->device = device; e->stream = (cudaStream_t)cuda_stream;
  e->noise.acc_n = cfg->acc_n; e->noise.gyr_n = cfg->gyr_n; e->noise.acc_w = cfg->acc_w; e->noise.gyr_w = cfg->gyr_w; e->noise.g_norm = cfg->g_norm;
  e->g_vec = V3(0, 0, -cfg->g_norm);
  e->extrinsic_stage = cfg->estimate_extrinsic;
  e->Ps.assign(W + 1, V3()); e->Vs.assign(W + 1, V3()); e->Bas.assign(W + 1, V3()); e->Bgs.assign(W + 1, V3());
  e->Rs.assign(W + 1, M3::I());
  e->pre.assign(W + 1, nullptr);
  e->para_pose.assign(O + 1, std::vector<double>(7, 0.0));
  e->para_sb.assign(O + 1, std::vector<double>(9, 0.0));
  std::memset(e->para_ex, 0, sizeof(e->para_ex));
  e->size_surf_stack.assign(W + 1, 0);
  e->h_feat_n.assign(W + 1, 0);
  e->local_tf.assign(W + 1, TransformF{0, 0, 0, 1, 0, 0, 0});
  const int pivot = W - O;
  e->slot_cap = cfg->max_frame_points * (pivot + 1);
  e->slot_ptr.resize(W + 1);
  e->slot_of.resize(W + 1);
  bool ok = true;
  for (int k = 0; k <= W; ++k) {
    e->slot_of[k] = k;
    ok = ok && alloc(e->slot_ptr[k], e->slot_cap);
  }
  e->local_cap = e->slot_cap + cfg->max_frame_points * (O > 1 ? O - 1 : 1);
  ok = ok && alloc(e->d_slot_n, W + 1) && alloc(e->d_own_n, W + 1) && alloc(e->d_scan, cfg->max_scan_points) && alloc(e->d_local, e->local_cap) &&
       alloc(e->d_map, e->local_cap) && alloc(e->d_tmp, e->slot_cap) && alloc(e->d_counts, 8) && alloc(e->d_tf, W + 1) && alloc(e->d_odom, 1) &&
       alloc(e->d_odom_partial, 32 * 1024) && alloc_host(e->h_tf, W + 1) && alloc_host(e->h_S, kMaxOpt * kAsmStride) &&
       alloc_host(e->h_Rt, kMaxOpt * kAsmRtStride) && alloc(e->d_Rt, kMaxOpt * kAsmRtStride) && alloc_host(e->h_counts, W + 16);
  if (ok) { std::memset(e->h_counts, 0, sizeof(int) * (W + 16)); e->h_xerr = e->h_counts + W + 10; }
  int vg_cap = std::max(e->local_cap, cfg->max_scan_points);
  ok = ok && e->vg.init(vg_cap) == 0;
  ok = ok && e->hash.init(e->local_cap) == 0;
  ok = ok && e->knn.init(cfg->max_frame_points * (O + 1)) == 0;
  ok = ok && e->knn2.init(cfg->max_frame_points) == 0;
  ok = ok && create(e->ostream) && create(e->ev_map) && create(e->ev_odom);
  e->feats.assign(W + 1, FeatureOut());
  e->feat_src.resize(W + 1);
  long long total_feat = 0;
  {
    e->px.foff_pts.assign(W + 1, 0); e->px.foff_coef.assign(W + 1, 0);
    size_t off = 0;
    for (int k = pivot + 1; k <= W; ++k) {
      const int cap = cfg->max_frame_points * ((k == W && cfg->keep_features) ? cfg->odom_max_iterations : 1);
      e->feats[k].cap = cap;
      e->px.foff_pts[k] = off; off += sizeof(float4) * (size_t)cap;
      e->px.foff_coef[k] = off; off += sizeof(float4) * (size_t)cap;
      total_feat += cap;
    }
    e->px.foff_cnt = off; off += ((sizeof(int) * (size_t)(W + 1) + 255) / 256) * 256;
    e->px.fpar_stride = off;
    e->px.foff_flags = 2 * off;
    e->px.fslab_bytes = 2 * off + 256;   // epoch flags (one per source rank) + error word behind the two parities
    ok = ok && alloc(e->px.fslab, e->px.fslab_bytes) && cudaMemset(e->px.fslab, 0, e->px.fslab_bytes) == cudaSuccess;
    for (int k = pivot + 1; k <= W && ok; ++k) {
      ok = alloc(e->feat_src[k], e->feats[k].cap);
      e->feats[k].src = e->feat_src[k];
    }
    if (ok) set_feature_parity(e.get(), 0);
  }
  ok = ok && e->asmw.init((int)std::min<long long>(total_feat, 1ll << 30)) == 0 && cudaMemset(e->d_slot_n, 0, sizeof(int) * (W + 1)) == cudaSuccess &&
       cudaMemset(e->d_own_n, 0, sizeof(int) * (W + 1)) == cudaSuccess && cudaMemset(e->d_counts, 0, sizeof(int) * 8) == cudaSuccess;
  ok = ok && create(e->ev0, cudaEventDefault) && create(e->ev1, cudaEventDefault) && create(e->evk0, cudaEventDefault) &&
       create(e->evk1, cudaEventDefault);
  ok = ok && alloc(e->px.xbuf, kXBytes) && cudaMemset(e->px.xbuf, 0, kXBytes) == cudaSuccess;
  for (int k = 0; k < 48 && ok; ++k) ok = create(e->evp[k], cudaEventDefault);
  e->use_dev_solver = cfg->device_solver != 0 && e->ds.supports(O) && cfg->max_num_iterations <= 22;
  if (e->use_dev_solver) ok = ok && e->ds.init(O) == 0;
  if (e->use_dev_solver && cfg->solver_graph) ok = ok && create(e->gstream) && create(e->ev_gin) && create(e->ev_gout);
  if (!ok) {
    lio_set_last_error(__FILE__, __LINE__, "lio_est_create: device allocation failed");
    return LIO_ERR_CUDA;
  }
  *out = e.release();
  return LIO_OK;
}

extern "C" int lio_est_set_extrinsic(lio_est *e, const float tf7[7]) {
  LIO_ENTER_HOST(e);
  if (!tf7) return LIO_ERR_INVALID;
  for (int k = 0; k < 4; ++k) e->tlb_q[k] = tf7[k];
  for (int k = 0; k < 3; ++k) e->tlb_p[k] = tf7[4 + k];
  return LIO_OK;
}
extern "C" int lio_est_get_extrinsic(lio_est *e, float tf7[7]) {
  LIO_ENTER_HOST(e);
  if (!tf7) return LIO_ERR_INVALID;
  for (int k = 0; k < 4; ++k) tf7[k] = e->tlb_q[k];
  for (int k = 0; k < 3; ++k) tf7[4 + k] = e->tlb_p[k];
  return LIO_OK;
}

extern "C" int lio_est_init_frame(lio_est *e, int k, const double s[16], const float *surf_ds, int n, lio_pim *pim) {
  LIO_ENTER(e);
  if (!s || k < 0 || k >= e->W || n < 0 || (n > 0 && !surf_ds)) return LIO_ERR_INVALID;
  if (n > e->cfg.max_frame_points) return LIO_ERR_CAPACITY;
  if (e->lc.on && !e->lc.staged) {
    lio_set_last_error(__FILE__, __LINE__, "local clouds are on: stage the frame's corner / full cloud with lio_est_set_scan_clouds_* first");
    return LIO_ERR_INVALID;
  }
  e->frames_started = true;
  if (e->mapping.on) { lio_set_last_error(__FILE__, __LINE__, "a mapping is attached: the window starts from the mapped poses"); return LIO_ERR_INVALID; }
  if (e->lc.on) {   // the pre-initialisation corner_stack_ / full_stack_ entries (Estimator.cc:474-482), verbatim
    const int slot = e->slot_of[k + 1];
    for (int w = 0; w < 2; ++w) {
      copy_cloud(e->lc.d_stage[w], e->lc.d_stage_n + w, e->lc.cap[w], e->lc.slot[w][slot], e->lc.d_slot_n + w * (e->W + 1) + slot, e->sm_count * 2,
                 e->stream);
    }
    LIO_CUDA_OK(cudaGetLastError());
    e->lc.staged = false;
  }
  e->Ps[k] = V3(s); e->Rs[k] = toR(normalized(Q(s[6], s[3], s[4], s[5]))); e->Vs[k] = V3(s + 7); e->Bas[k] = V3(s + 10); e->Bgs[k] = V3(s + 13);
  const int slot = e->slot_of[k + 1];  // one slot to the right: the first process_scan pushes (see oracle InitFrame)
  if (n > 0) LIO_CUDA_OK(cudaMemcpyAsync(e->slot_ptr[slot], surf_ds, sizeof(float4) * n, cudaMemcpyHostToDevice, e->stream));
  LIO_CUDA_OK(cudaMemcpyAsync(e->d_slot_n + slot, &n, sizeof(int), cudaMemcpyHostToDevice, e->stream));
  LIO_CUDA_OK(cudaMemcpyAsync(e->d_own_n + slot, &n, sizeof(int), cudaMemcpyHostToDevice, e->stream));
  LIO_CUDA_OK(cudaStreamSynchronize(e->stream));
  e->size_surf_stack[k + 1] = n;
  e->pre[k + 1] = pim ? pim->p : nullptr;
  if (pim) delete pim;
  return LIO_OK;
}

extern "C" int lio_est_finish_init(lio_est *e, const double a[3], const double g[3]) {
  LIO_ENTER_HOST(e);
  if (!a || !g || e->mapping.on) return LIO_ERR_INVALID;
  const int W = e->W;
  e->Ps[W] = e->Ps[W - 1]; e->Rs[W] = e->Rs[W - 1]; e->Vs[W] = e->Vs[W - 1]; e->Bas[W] = e->Bas[W - 1]; e->Bgs[W] = e->Bgs[W - 1];
  e->acc_last = V3(a); e->gyr_last = V3(g);
  e->first_imu = true;
  e->tmp_pre = std::make_shared<Preintegration>(e->acc_last, e->gyr_last, e->Bas[W], e->Bgs[W], e->noise);
  e->imu_stamped.clear();
  return LIO_OK;
}

extern "C" int lio_est_process_imu(lio_est *e, double dt, const double a[3], const double g[3], double stamp) {
  LIO_ENTER_HOST(e);
  if (!a || !g) return LIO_ERR_INVALID;
  const V3 acc(a), gyr(g);
  if (!e->first_imu) { e->first_imu = true; e->acc_last = acc; e->gyr_last = gyr; }
  if (!e->tmp_pre) return LIO_ERR_INVALID;
  if (e->mapping.on && !e->mapping.inited && e->mapping.cir_count == 0) { e->acc_last = acc; e->gyr_last = gyr; return LIO_OK; }   // :379: no laser yet
  const int j = (e->mapping.on && !e->mapping.inited) ? e->mapping.cir_count : e->W;
  e->tmp_pre->push_back(dt, acc, gyr);
  const V3 un_acc_0 = e->Rs[j] * (e->acc_last - e->Bas[j]) + e->g_vec;
  const V3 un_gyr = 0.5 * (e->gyr_last + gyr) - e->Bgs[j];
  e->Rs[j] = e->Rs[j] * toR(deltaQ(un_gyr * dt));
  const V3 un_acc_1 = e->Rs[j] * (acc - e->Bas[j]) + e->g_vec;
  const V3 un_acc = 0.5 * (un_acc_0 + un_acc_1);
  e->Ps[j] = e->Ps[j] + dt * e->Vs[j] + 0.5 * dt * dt * un_acc;
  e->Vs[j] = e->Vs[j] + dt * un_acc;
  ImuStampedF tt;
  tt.time = stamp;
  tt.p[0] = (float)e->Ps[j].x; tt.p[1] = (float)e->Ps[j].y; tt.p[2] = (float)e->Ps[j].z;
  {  // Quaternionf(Rs.cast<float>())
    M3 Rf;
    for (int a2 = 0; a2 < 3; ++a2) for (int b = 0; b < 3; ++b) Rf(a2, b) = (double)(float)e->Rs[j](a2, b);
    Q q = fromR(Rf);
    tt.q[0] = (float)q.x; tt.q[1] = (float)q.y; tt.q[2] = (float)q.z; tt.q[3] = (float)q.w;
  }
  e->imu_stamped.push_back(tt);
  if (e->imu_stamped.size() > 100) e->imu_stamped.erase(e->imu_stamped.begin());
  e->acc_last = acc; e->gyr_last = gyr;
  return LIO_OK;
}

extern "C" int lio_est_process_imu_batch(lio_est *e, int n, const double *dt, const double *acc3, const double *gyr3, const double *stamp) {
  LIO_ENTER_HOST(e);
  if (n < 0 || (n > 0 && (!dt || !acc3 || !gyr3 || !stamp))) return LIO_ERR_INVALID;
  for (int k = 0; k < n; ++k) {
    LIO_TRY(lio_est_process_imu(e, dt[k], acc3 + 3 * k, gyr3 + 3 * k, stamp[k]));
  }
  return LIO_OK;
}

// SolveOptimization (Estimator.cc:1648-2438) in three phases, also exported one by one (lio_est_open_scan_* / lio_est_solve /
// lio_est_close_scan) for callers that keep the reference's control flow:
//   scan_open   BuildLocalMap, join the previous marginalisation, VectorToDouble                       (:1361-1646, :2440-2478)
//   scan_solve  problem build + gates + ceres::Solve from the para_* blocks                            (:1747-1990)
//   scan_close  DoubleToVector, marginalisation of the oldest frame, SlideWindow                        (:2479-2568, :2040-2275, :2570-2666)
static int scan_open_window(lio_est *e) {
  e->turn_off = true;
  e->ds_prepared = false;
  int rc = build_local_map(e, [e]() -> int {
    prior_join(e);  // the previous scan's marginalisation algebra ran beside the front end enqueued above
    e->ex_constant = (e->extrinsic_stage == 0 || e->cfg.opt_extrinsic == 0);
    vector_to_double(e);
    // the device solver's state does not depend on the features: prepare and upload it before waiting for them
    if (e->use_dev_solver) return solve_dev_prepare(e, e->cfg.max_num_iterations, false);
    return LIO_OK;
  });
  if (rc != LIO_OK) return rc;
  e->window_open = true;
  return LIO_OK;
}

static int scan_close_window(lio_est *e) {
  double_to_vector(e);
  const double t1 = now_s();
  if (e->cfg.marginalization_factor && !e->turn_off) {
    vector_to_double(e);
    const int rc = marginalize(e);
    if (rc != LIO_OK) return rc;
    e->prior_uploaded = false;
  }
  e->t_marg = now_s() - t1;
  e->window_open = false;
  int rc = lc_join(e);   // the forked /local/* work reads the surf slot that SlideWindow replaces
  if (rc != LIO_OK) return rc;
  if (e->map.pm && !e->mapping.quiet && (rc = map_step(e)) != LIO_OK) return rc;   // UpdateMapDatabase + PublishResults come before SlideWindow (:703-723)
  return slide_window(e);
}

static int scan_solve(lio_est *e, int max_it) { return e->use_dev_solver ? solve_dev(e, max_it, false) : solve_host(e, max_it); }

int scan_failed(lio_est *e, int rc, bool poison) {
  if (poison) e->poisoned = true;
  std::snprintf(e->err, sizeof(e->err), "%s", lio_last_error());
  return rc;
}

int refuse_poisoned(lio_est *e) {
  lio_set_last_error(__FILE__, __LINE__, "estimator context poisoned by an earlier failed scan: destroy and re-create it");
  return LIO_ERR_INVALID;
}

// The pre-integration buffer, the slot rotation and size_surf_stack advance before the fallible device work.  A failure
// after that point leaves the window half-slid, so the context is poisoned: later calls return LIO_ERR_INVALID instead of
// running on inconsistent state (documented in lio_b200.h).
static int process_scan_common(lio_est *e, const float4 *scan_dev, const int *n_dev, int n_max, bool open_only) {
  if (e->window_open) { lio_set_last_error(__FILE__, __LINE__, "a scan is open: finish it with lio_est_close_scan first"); return LIO_ERR_INVALID; }
  if (e->poisoned) return refuse_poisoned(e);
  if (!e->tmp_pre) { lio_set_last_error(__FILE__, __LINE__, "process_scan before finish_init"); return LIO_ERR_INVALID; }
  if (e->mapping.on) {
    lio_set_last_error(__FILE__, __LINE__, "a mapping is attached: feed the odometry's clouds with lio_est_process_compact_*");
    return LIO_ERR_INVALID;
  }
  if (e->lc.on && !e->lc.staged) {   // before the window advances: the context stays usable
    lio_set_last_error(__FILE__, __LINE__, "local clouds are on: stage the scan's corner / full cloud with lio_est_set_scan_clouds_* first");
    return scan_failed(e, LIO_ERR_INVALID, false);
  }
  e->frames_started = true;
  e->scanned = true;
  const int rc = process_scan_body(e, scan_dev, n_dev, n_max, open_only);
  return rc != LIO_OK ? scan_failed(e, rc) : rc;
}

int process_scan_body(lio_est *e, const float4 *scan_dev, const int *n_dev, int n_max, bool open_only, const CompactPush *cp) {
  const int W = e->W;
  cudaStream_t st = e->stream;
  marg_start(e);
  const double t0 = now_s();
  e->launches = 0;
  e->t_lin_wait = e->t_lin_host = e->t_lin_lidar = e->t_marg_wait = 0;
  e->have_H0 = false;
  if (!e->tmp_pre) { lio_set_last_error(__FILE__, __LINE__, "process_scan before finish_init"); return LIO_ERR_INVALID; }
  if (e->map.pm) {
    const int rc0 = map_scan_entry(e, !(cp && cp->startup));
    if (rc0 != LIO_OK) return rc0;
  }
  push_shift(e->pre, e->tmp_pre);
  e->tmp_pre = std::make_shared<Preintegration>(e->acc_last, e->gyr_last, e->Bas[W], cp ? cp->tmp_bg : e->Bgs[W], e->noise);
  e->tmp_pre->keep_samples = false;   // from here on the window is INITED: only RunInitialization repropagates
  // frame slot rotation (CircularBuffer push): the dropped logical frame 0 becomes the new frame W
  {
    const int freed = e->slot_of[0];
    e->slot_of.erase(e->slot_of.begin());
    e->slot_of.push_back(freed);
  }
  const int slot = e->slot_of[W];
  const float4 *src = scan_dev;
  // transform_es_ is computed whenever either flag is set (:628-664); the surf (and corner) clouds are de-skewed with it only
  // without cutoff_deskew (:666-673), the full cloud always (:2416, local clouds on)
  const bool es_on = map_deskew(e) && !e->imu_stamped.empty() && !(cp && cp->startup);
  const bool deskew_surf = es_on && !e->cfg.cutoff_deskew;
  if (es_on) {
    // transform_es_ from the IMU-propagated poses of the last 0.1 s (:632-664), float Twist algebra on the host
    const ImuStampedF &te = e->imu_stamped.back();
    ImuStampedF ts = te;
    for (int i = (int)e->imu_stamped.size() - 1; i >= 0; --i) {
      ts = e->imu_stamped[i];
      if (te.time - e->imu_stamped[i].time >= 0.1) break;
    }
    auto twf = [](const float *q, const float *p) { return Tw(Q(q[3], q[0], q[1], q[2]), V3(p[0], p[1], p[2])); };
    // evaluated in double and rounded: the float op order of Eigen::Transform<float> is not reproduced (tolerance-checked)
    Tw body_es = tw_mul(tw_inverse(twf(te.q, te.p)), twf(ts.q, ts.p));
    {
      const float s = (float)(0.1 / (te.time - ts.time));
      Q qe = body_es.rot;
      double d = qe.w, absD = std::fabs(d), s0, s1;
      if (absD >= 1.0 - 1.1920929e-7) { s0 = 1.0 - s; s1 = s; }
      else { double th = std::acos(absD), sn = std::sin(th); s0 = std::sin((1.0 - s) * th) / sn; s1 = std::sin(s * th) / sn; }
      if (d < 0) s1 = -s1;
      body_es.rot = Q(s0 + s1 * qe.w, s1 * qe.x, s1 * qe.y, s1 * qe.z);
      body_es.pos = body_es.pos * (double)s;
    }
    const Tw tlb = tlb_double(e);
    const Tw es = tw_mul(tw_mul(tlb, body_es), tw_inverse(tlb));
    e->es = TransformF{(float)es.rot.x, (float)es.rot.y, (float)es.rot.z, (float)es.rot.w, (float)es.pos.x, (float)es.pos.y, (float)es.pos.z};
  }
  if (deskew_surf) {
    if (scan_dev != e->d_scan) {
      LIO_CUDA_OK(cudaMemcpyAsync(e->d_scan, scan_dev, sizeof(float4) * n_max, cudaMemcpyDeviceToDevice, st));
    }
    deskew(e->d_scan, n_dev, n_max, e->es, 10.f, false, st);
    ++e->launches;
    src = e->d_scan;
  }
  int rc = LIO_OK;
  if (cp && cp->surf_ds) {
    copy_cloud(cp->surf_ds, cp->surf_ds_n, e->cfg.max_frame_points, e->slot_ptr[slot], e->d_slot_n + slot, e->sm_count * 2, st);
    ++e->launches;
    LIO_CUDA_OK(cudaGetLastError());
  } else {
    rc = e->vg.run(src, n_dev, n_max, e->cfg.surf_filter_size, e->slot_ptr[slot], e->cfg.max_frame_points, e->d_slot_n + slot, nullptr, st, &e->launches);
    if (rc != LIO_OK) return rc;
  }
  LIO_CUDA_OK(cudaMemcpyAsync(e->d_own_n + slot, e->d_slot_n + slot, sizeof(int), cudaMemcpyDeviceToDevice, st));
  if (e->lc.on && (rc = lc_push(e, deskew_surf, cp && cp->corner_filtered)) != LIO_OK) return rc;
  push_shift(e->size_surf_stack, 0);
  if (cp && !e->cfg.imu_factor) predict_state_w(e);
  rc = scan_open_window(e);
  if (rc != LIO_OK || open_only) return rc;
  rc = scan_solve(e, e->cfg.max_num_iterations);
  if (rc != LIO_OK) return rc;
  rc = scan_close_window(e);
  if (rc != LIO_OK) return rc;
  e->t_total = now_s() - t0;
  return LIO_OK;
}

extern "C" int lio_est_begin_scan(lio_est *e) {
  LIO_ENTER_HOST(e);
  if (e->cfg.overlap_marginalization) marg_start(e);
  return LIO_OK;
}

// The host entries upload surf_last into d_scan and its count into d_counts[0]; the device entries read the caller's buffers.
static int scan_host(lio_est *e, const float *surf_last, int n, bool open_only) {
  if (n < 0 || (n > 0 && !surf_last)) return LIO_ERR_INVALID;
  if (n > e->cfg.max_scan_points) return LIO_ERR_CAPACITY;
  if (n > 0) LIO_CUDA_OK(cudaMemcpyAsync(e->d_scan, surf_last, sizeof(float4) * n, cudaMemcpyHostToDevice, e->stream));
  e->h_counts[e->W + 8] = n;
  LIO_CUDA_OK(cudaMemcpyAsync(e->d_counts, e->h_counts + e->W + 8, sizeof(int), cudaMemcpyHostToDevice, e->stream));
  return process_scan_common(e, e->d_scan, e->d_counts, n > 0 ? n : 1, open_only);
}

static int scan_dev(lio_est *e, const float *surf_last_dev, const int *n_dev, int n_max, bool open_only) {
  if (!surf_last_dev || !n_dev || n_max <= 0) return LIO_ERR_INVALID;
  if (n_max > e->cfg.max_scan_points) n_max = e->cfg.max_scan_points;   // the voxel filter clamps *n_dev to n_max on the device
  return process_scan_common(e, reinterpret_cast<const float4 *>(surf_last_dev), n_dev, n_max, open_only);
}

extern "C" int lio_est_process_scan_host(lio_est *e, const float *surf_last, int n) { LIO_ENTER(e); return scan_host(e, surf_last, n, false); }

extern "C" int lio_est_process_scan_dev(lio_est *e, const float *surf_last_dev, const int *n_dev, int n_max) {
  LIO_ENTER(e);
  return scan_dev(e, surf_last_dev, n_dev, n_max, false);
}

// ---- stepwise API: the phases of ProcessLaserOdom / SolveOptimization one by one ----------------------------------------
extern "C" int lio_est_open_scan_host(lio_est *e, const float *surf_last, int n) { LIO_ENTER(e); return scan_host(e, surf_last, n, true); }

extern "C" int lio_est_open_scan_dev(lio_est *e, const float *surf_last_dev, const int *n_dev, int n_max) {
  LIO_ENTER(e);
  return scan_dev(e, surf_last_dev, n_dev, n_max, true);
}

static int need_open(lio_est *e) {
  if (e->poisoned) return scan_failed(e, refuse_poisoned(e), false);
  if (e->window_open) return LIO_OK;
  lio_set_last_error(__FILE__, __LINE__, "no open scan: call lio_est_open_scan_host / _dev first");
  return scan_failed(e, LIO_ERR_INVALID, false);
}

static void load_parameters(lio_est *e, const double *pose, const double *sb, const double *ex) {
  for (int k = 0; k <= e->O; ++k) {
    if (pose) std::memcpy(e->para_pose[k].data(), pose + 7 * k, 7 * sizeof(double));
    if (sb) std::memcpy(e->para_sb[k].data(), sb + 9 * k, 9 * sizeof(double));
  }
  if (ex) std::memcpy(e->para_ex, ex, 7 * sizeof(double));
  e->S_valid = false;
  e->ds_prepared = false;   // the uploaded solver state belongs to the previous parameter values
}
static void store_parameters(const lio_est *e, double *pose, double *sb, double *ex) {
  for (int k = 0; k <= e->O; ++k) {
    if (pose) std::memcpy(pose + 7 * k, e->para_pose[k].data(), 7 * sizeof(double));
    if (sb) std::memcpy(sb + 9 * k, e->para_sb[k].data(), 9 * sizeof(double));
  }
  if (ex) std::memcpy(ex, e->para_ex, 7 * sizeof(double));
}

extern "C" int lio_est_get_parameters(lio_est *e, double *pose, double *speed_bias, double *ex) {
  LIO_ENTER_HOST(e);
  LIO_TRY(need_open(e));
  store_parameters(e, pose, speed_bias, ex);
  return LIO_OK;
}

extern "C" int lio_est_last_normal_equations(lio_est *e, double *H, double *g, double *cost, int *n);

extern "C" int lio_est_assemble(lio_est *e, const double *pose, const double *speed_bias, const double *ex, double *H, double *g,
                                double *cost, int *n) {
  LIO_ENTER(e);
  if (!n) return LIO_ERR_INVALID;
  int rc = need_open(e);
  if (rc != LIO_OK) return rc;
  // evaluate at the caller's blocks, then put the estimator's own blocks back
  std::vector<double> kp(7 * (e->O + 1)), ks(9 * (e->O + 1));
  double kx[7];
  store_parameters(e, kp.data(), ks.data(), kx);
  load_parameters(e, pose, speed_bias, ex);
  if (e->use_dev_solver) {
    rc = solve_dev(e, 0, true);
    if (rc == LIO_OK) rc = lio_est_last_normal_equations(e, H, g, cost, n);
  } else {
    Mat Hh;
    Vec gg;
    double c = 0;
    rc = linearize(e, Hh, gg, c, nullptr, nullptr, nullptr);
    if (rc == LIO_ERR_NUMERIC) lio_set_last_error(__FILE__, __LINE__, "non-finite cost");
    if (rc == LIO_OK) {
      *n = Hh.r;
      if (H) std::memcpy(H, Hh.d.data(), sizeof(double) * Hh.r * Hh.r);
      if (g) std::memcpy(g, gg.data(), sizeof(double) * Hh.r);
      if (cost) *cost = c;
    }
  }
  load_parameters(e, kp.data(), ks.data(), kx);
  return rc;
}

extern "C" int lio_est_solve(lio_est *e, double *pose, double *speed_bias, double *ex, int max_iter, double summary[8]) {
  LIO_ENTER(e);
  if (max_iter < 0) return LIO_ERR_INVALID;
  int rc = need_open(e);
  if (rc != LIO_OK) return rc;
  if (e->use_dev_solver && max_iter > 22) return LIO_ERR_INVALID;
  load_parameters(e, pose, speed_bias, ex);
  rc = scan_solve(e, max_iter);
  if (rc != LIO_OK) return scan_failed(e, rc);
  store_parameters(e, pose, speed_bias, ex);
  if (summary) {
    summary[0] = e->summary.iterations; summary[1] = e->summary.successful_steps; summary[2] = e->summary.termination;
    summary[3] = e->summary.initial_cost; summary[4] = e->summary.final_cost; summary[5] = e->summary.evaluations;
    summary[6] = e->convergence_flag ? 1 : 0; summary[7] = e->ex_constant ? 1 : 0;
  }
  return LIO_OK;
}

extern "C" int lio_est_close_scan(lio_est *e, const double *pose, const double *speed_bias, const double *ex) {
  LIO_ENTER(e);
  int rc = need_open(e);
  if (rc != LIO_OK) return rc;
  load_parameters(e, pose, speed_bias, ex);
  rc = scan_close_window(e);
  return rc != LIO_OK ? scan_failed(e, rc) : rc;
}

extern "C" int lio_est_frame_owner(int frame_rel, int world) {  // frame_rel in 1..O (relative to the pivot)
  if (world < 1 || frame_rel < 1) return -1;
  return (frame_rel - 1) % world;
}

extern "C" int lio_est_set_shard(lio_est *e, int rank, int world, lio_allreduce_fn fn, void *user) {
  LIO_ENTER_HOST(e);
  if (world < 1 || rank < 0 || rank >= world) return LIO_ERR_INVALID;
  if (e->lc.on) { lio_set_last_error(__FILE__, __LINE__, "local clouds are not supported on a sharded context"); return LIO_ERR_INVALID; }
  e->rank = rank; e->world = world; e->allreduce = fn; e->allreduce_user = user;
  e->px.npeers = 0;
  e->px.fpeers = false;
  e->worker.spin_us = world > 1 ? std::max(25.0, 400.0 / world) : 400.0;  // N processes share the host: spin less
  return LIO_OK;
}

extern "C" int lio_est_exchange_buffer(lio_est *e, void **dev_ptr, size_t *bytes) {
  LIO_ENTER_HOST(e);
  if (!dev_ptr) return LIO_ERR_INVALID;
  *dev_ptr = e->px.xbuf;
  if (bytes) *bytes = kXBytes;
  return LIO_OK;
}

extern "C" int lio_est_set_peers(lio_est *e, int world, void *const *peer_ptrs) {
  LIO_ENTER_HOST(e);
  if (!peer_ptrs || world != e->world || world < 2 || world > kMaxPeers || e->lc.on) return LIO_ERR_INVALID;
  for (int r = 0; r < world; ++r) {
    e->px.peer_base[r] = r == e->rank ? e->px.xbuf : static_cast<char *>(peer_ptrs[r]);
    if (!e->px.peer_base[r]) return LIO_ERR_INVALID;
  }
  e->px.npeers = world;
  return LIO_OK;
}

extern "C" int lio_est_feature_slab(lio_est *e, void **dev_ptr, size_t *bytes) {
  LIO_ENTER_HOST(e);
  if (!dev_ptr) return LIO_ERR_INVALID;
  *dev_ptr = e->px.fslab;
  if (bytes) *bytes = e->px.fslab_bytes;
  return LIO_OK;
}

extern "C" int lio_est_set_feature_peers(lio_est *e, int world, void *const *peer_slabs) {
  LIO_ENTER_HOST(e);
  if (!peer_slabs || world != e->world || world < 2 || world > kMaxPeers || e->lc.on) return LIO_ERR_INVALID;
  if (e->window_open) { lio_set_last_error(__FILE__, __LINE__, "lio_est_set_feature_peers inside an open scan"); return LIO_ERR_INVALID; }
  for (int r = 0; r < world; ++r) {
    e->px.fpeer_base[r] = r == e->rank ? e->px.fslab : static_cast<char *>(peer_slabs[r]);
    if (!e->px.fpeer_base[r]) return LIO_ERR_INVALID;
  }
  e->px.fpeers = true;
  e->px.npeers = 0;
  return LIO_OK;
}

extern "C" int lio_ipc_export(const void *dev_ptr, unsigned char handle[64]) {
  if (!dev_ptr || !handle) return LIO_ERR_INVALID;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  cudaIpcMemHandle_t h;
  LIO_CUDA_OK(cudaIpcGetMemHandle(&h, const_cast<void *>(dev_ptr)));
  std::memcpy(handle, &h, 64);
  return LIO_OK;
}

extern "C" int lio_ipc_open(const unsigned char handle[64], void **dev_ptr) {
  if (!handle || !dev_ptr) return LIO_ERR_INVALID;
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle, 64);
  LIO_CUDA_OK(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return LIO_OK;
}

extern "C" int lio_ipc_close(void *dev_ptr) {
  if (!dev_ptr) return LIO_OK;
  LIO_CUDA_OK(cudaIpcCloseMemHandle(dev_ptr));
  return LIO_OK;
}

// ---- getters --------------------------------------------------------------------------------------
extern "C" int lio_est_get_states(lio_est *e, double *out) {
  LIO_ENTER_HOST(e);
  if (!out) return LIO_ERR_INVALID;
  for (int k = 0; k <= e->W; ++k) {
    double *s = out + 16 * k;
    Q q = fromR(e->Rs[k]);
    s[0] = e->Ps[k].x; s[1] = e->Ps[k].y; s[2] = e->Ps[k].z; s[3] = q.x; s[4] = q.y; s[5] = q.z; s[6] = q.w;
    for (int a = 0; a < 3; ++a) { s[7 + a] = e->Vs[k][a]; s[10 + a] = e->Bas[k][a]; s[13 + a] = e->Bgs[k][a]; }
  }
  return LIO_OK;
}

extern "C" int lio_est_summary(lio_est *e, double *o) {
  LIO_ENTER_HOST(e);
  if (!o) return LIO_ERR_INVALID;
  const bool has_prior = e->prior.valid || e->mjob.stashed || e->mjob.running;  // does not force the pending algebra
  for (int k = 0; k < 32; ++k) o[k] = 0;
  o[0] = e->summary.iterations; o[1] = e->summary.successful_steps; o[2] = e->summary.termination;
  o[3] = e->summary.initial_cost; o[4] = e->summary.final_cost; o[5] = e->cost_pim; o[6] = e->cost_ppp; o[7] = e->cost_marg;
  o[8] = e->turn_off; o[9] = e->convergence_flag; o[10] = e->h_map_n;
  long long nf = 0;
  for (int v : e->h_feat_n) nf += v;
  o[11] = (double)nf; o[12] = e->odom_iters;
  o[13] = e->t_build; o[14] = e->t_feat; o[15] = e->t_solve; o[16] = e->t_marg; o[17] = e->t_total;
  o[18] = has_prior ? 1 : 0; o[19] = e->summary.evaluations; o[20] = e->summary.evaluations; o[21] = e->launches;
  o[22] = e->t_lin_wait; o[23] = e->t_lin_host; o[24] = e->t_lin_lidar; o[25] = e->t_marg_wait;
  return LIO_OK;
}

extern "C" int lio_est_feature_count(lio_est *e, int frame, int *n) {
  LIO_ENTER_HOST(e);
  if (!n || frame < 0 || frame > e->W) return LIO_ERR_INVALID;
  *n = e->h_feat_n[frame];
  return LIO_OK;
}

extern "C" int lio_est_get_features(lio_est *e, int frame, float *pts4, float *coef4, int32_t *src, int cap) {
  LIO_ENTER(e);
  if (frame < 0 || frame > e->W) return LIO_ERR_INVALID;
  const int n = e->h_feat_n[frame];
  if (n > cap) return LIO_ERR_CAPACITY;
  if (n == 0) return LIO_OK;
  const FeatureOut &f = e->feats[frame];
  if (pts4) LIO_TRY(read_back((float4 *)pts4, f.pts, n, cap, e->stream));
  if (coef4) LIO_TRY(read_back((float4 *)coef4, f.coef, n, cap, e->stream));
  if (src) LIO_TRY(read_back((int *)src, f.src, n, cap, e->stream));
  return LIO_OK;
}

extern "C" int lio_est_map_size(lio_est *e, int *n) {
  LIO_ENTER_HOST(e);
  if (!n) return LIO_ERR_INVALID;
  *n = e->h_map_n;
  return LIO_OK;
}
extern "C" int lio_est_get_map(lio_est *e, float *out, int cap) {
  LIO_ENTER(e);
  if (!out) return LIO_ERR_INVALID;
  return read_back((float4 *)out, e->d_map, e->h_map_n, cap, e->stream);
}
extern "C" int lio_est_frame_size(lio_est *e, int frame, int *n) {
  LIO_ENTER(e);
  if (!n || frame < 0 || frame > e->W) return LIO_ERR_INVALID;
  return read_back(n, e->d_slot_n + e->slot_of[frame], 1, 1, e->stream);
}
extern "C" int lio_est_get_frame(lio_est *e, int frame, float *out, int cap) {
  LIO_ENTER(e);
  int n = 0;
  LIO_TRY(lio_est_frame_size(e, frame, &n));
  return read_back((float4 *)out, e->slot_ptr[e->slot_of[frame]], n, cap, e->stream);
}
extern "C" int lio_est_get_local_transform(lio_est *e, int frame, float tf7[7]) {
  LIO_ENTER_HOST(e);
  if (!tf7 || frame < 0 || frame > e->W) return LIO_ERR_INVALID;
  const TransformF &t = e->local_tf[frame];
  tf7[0] = t.qx; tf7[1] = t.qy; tf7[2] = t.qz; tf7[3] = t.qw; tf7[4] = t.px; tf7[5] = t.py; tf7[6] = t.pz;
  return LIO_OK;
}
// /local_laser_odom (Estimator.cc:725-742): rot = Quaterniond(Rs_[pivot] * transform_lb.rot.inverse()), pos = Ps_[pivot] - rot *
// transform_lb.pos with transform_lb = transform_lb_.cast<double>(), rounded to float like LaserOdometryHandler (PointMapping.cc:267-282)
extern "C" int lio_est_local_laser_odom(lio_est *e, float tf7[7]) {
  LIO_ENTER_HOST(e);
  if (!tf7) return LIO_ERR_INVALID;
  const int pivot = e->W - e->O;
  const Tw t = lidar_pose(e->Ps[pivot], e->Rs[pivot], tlb_double(e));
  tf7[0] = (float)t.rot.x; tf7[1] = (float)t.rot.y; tf7[2] = (float)t.rot.z; tf7[3] = (float)t.rot.w;
  tf7[4] = (float)t.pos.x; tf7[5] = (float)t.pos.y; tf7[6] = (float)t.pos.z;
  return LIO_OK;
}
// /predict_laser_odom (Estimator.cc:744-758, state W) and /local_laser_odom (:725-742, state W - O) in double, as they are published:
// the same lidar_pose as lio_est_local_laser_odom, not rounded
extern "C" int lio_est_laser_odom(lio_est *e, double predict7[7], double local7[7]) {
  LIO_ENTER_HOST(e);
  if (!predict7 && !local7) return LIO_ERR_INVALID;
  const Tw tlb = tlb_double(e);
  auto out = [](const Tw &t, double *o) {
    o[0] = t.rot.x; o[1] = t.rot.y; o[2] = t.rot.z; o[3] = t.rot.w; o[4] = t.pos.x; o[5] = t.pos.y; o[6] = t.pos.z;
  };
  if (predict7) out(lidar_pose(e->Ps[e->W], e->Rs[e->W], tlb), predict7);
  if (local7) out(lidar_pose(e->Ps[e->W - e->O], e->Rs[e->W - e->O], tlb), local7);
  return LIO_OK;
}
extern "C" int lio_est_prior_dim(lio_est *e, int *n) {
  LIO_ENTER_HOST(e);
  if (!n) return LIO_ERR_INVALID;
  prior_join(e);
  *n = e->prior.valid ? e->prior.n : 0;
  return LIO_OK;
}
extern "C" int lio_est_get_prior(lio_est *e, double *Hp, double *bp) {
  LIO_ENTER_HOST(e);
  if (!Hp || !bp) return LIO_ERR_INVALID;
  prior_join(e);
  if (!e->prior.valid) return LIO_ERR_INVALID;
  std::memcpy(Hp, e->prior.Hp.d.data(), sizeof(double) * e->prior.n * e->prior.n);
  std::memcpy(bp, e->prior.bp.data(), sizeof(double) * e->prior.n);
  return LIO_OK;
}
extern "C" int lio_est_last_normal_equations(lio_est *e, double *H, double *g, double *cost, int *n) {
  LIO_ENTER(e);
  if (!n) return LIO_ERR_INVALID;
  if (!e->have_H0) { *n = 0; return LIO_OK; }
  if (e->use_dev_solver) {
    // device layout keeps the 6 extrinsic slots; report the reduced system when the extrinsic was constant
    const int nf = 15 * (e->O + 1) + 6, nr = e->ex_constant ? nf - 6 : nf;
    *n = nr;
    std::vector<double> Hf((size_t)nf * nf), gf(nf);
    LIO_CUDA_OK(cudaMemcpy(Hf.data(), e->ds.H0, sizeof(double) * nf * nf, cudaMemcpyDeviceToHost));
    LIO_CUDA_OK(cudaMemcpy(gf.data(), e->ds.g0, sizeof(double) * nf, cudaMemcpyDeviceToHost));
    if (H) for (int r = 0; r < nr; ++r) std::memcpy(H + (size_t)r * nr, &Hf[(size_t)r * nf], sizeof(double) * nr);
    if (g) std::memcpy(g, gf.data(), sizeof(double) * nr);
    if (cost) *cost = e->cost0;
    return LIO_OK;
  }
  *n = e->H0.r;
  if (H) std::memcpy(H, e->H0.d.data(), sizeof(double) * e->H0.r * e->H0.r);
  if (g) std::memcpy(g, e->g0.data(), sizeof(double) * e->H0.r);
  if (cost) *cost = e->cost0;
  return LIO_OK;
}
extern "C" int lio_est_last_launches(lio_est *e) { return e ? e->launches : 0; }
extern "C" const char *lio_est_last_error(lio_est *e) { return e ? e->err : "null handle"; }

extern "C" int lio_est_solver_trace(lio_est *e, long long *out, int cap) {
  LIO_ENTER(e);
  if (!out || cap < 24 * 16 + 4 * 28 + 4) return LIO_ERR_INVALID;
  if (!e->use_dev_solver) { std::memset(out, 0, sizeof(long long) * (24 * 16 + 4 * 28 + 4)); return LIO_OK; }
  LIO_CUDA_OK(cudaMemcpy(out, reinterpret_cast<const char *>(e->ds.st.get()) + offsetof(DevSolveState, dbg), sizeof(long long) * (24 * 16 + 4 * 28 + 4), cudaMemcpyDeviceToHost));
  return LIO_OK;
}

extern "C" int lio_est_kernel_profile(lio_est *e, double out[8], int reset) {
  LIO_ENTER_HOST(e);
  if (!out) return LIO_ERR_INVALID;
  out[0] = e->asm_ms_sum; out[1] = (double)e->asm_launch_count; out[2] = (double)e->asm_feat_sum; out[3] = 32.0;
  out[4] = e->knn_ms_sum; out[5] = (double)e->knn_launch_count; out[6] = (double)e->knn_query_sum; out[7] = 128.0;
  if (reset) { e->asm_ms_sum = 0; e->asm_launch_count = 0; e->asm_feat_sum = 0; e->knn_ms_sum = 0; e->knn_launch_count = 0; e->knn_query_sum = 0; }
  return LIO_OK;
}

// ---- C-ABI: TransformToEnd on an explicit host array (parity entry) ----------------------------------------------
extern "C" int lio_transform_to_end_host(float *cloud, int n, const float *tf7_es, float time_factor, int device) {
  if (!cloud || !tf7_es || n < 0) return LIO_ERR_INVALID;
  LIO_TRY(select_device(device));
  if (n == 0) return LIO_OK;
  DevBufs db;
  float4 *d = nullptr;
  int *dn = nullptr;
  if (!db.alloc(&d, n) || !db.alloc(&dn, 1) || !db.up(d, (const float4 *)cloud, n) || !db.up(dn, &n, 1)) return LIO_ERR_CUDA;
  TransformF es;
  std::memcpy(&es, tf7_es, sizeof(es));
  deskew(d, dn, n, es, time_factor, false, 0);
  return db.down((float4 *)cloud, d, n) ? LIO_OK : LIO_ERR_CUDA;
}
