// The optional map-side parts of the device estimator: the /local/* clouds (lio_est_enable_local_clouds), the global cube map after
// initialisation (lio_est_attach_map) and the imu_factor = 0 mapping from the odometry's clouds (lio_est_attach_mapping).
#include "estimator.cuh"

namespace lio {

// The /local/* publication (Estimator.cc:2362-2375): corner, surf and full cloud of one frame into the publication buffers,
// one blockIdx.y per cloud, counts to n_out[0..2]
struct LocalGather {
  const float4 *src[3];
  const int *n[3];
  float4 *dst[3];
  int cap[3];
};
__global__ void __launch_bounds__(256)
k_local_gather(const LocalGather G, int *__restrict__ n_out) {
  const int w = blockIdx.y;
  const int n = min(max(*G.n[w], 0), G.cap[w]);
  if (blockIdx.x == 0 && threadIdx.x == 0) n_out[w] = n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) G.dst[w][i] = __ldg(G.src[w] + i);
}

}  // namespace lio

// ---- /local/* clouds (Estimator.cc:474-482, :628-693, :2355-2375, :2416) ------------------------------------------------
extern "C" int lio_est_enable_local_clouds(lio_est *e, float corner_filter_size, int max_corner_points, int max_full_points) {
  LIO_ENTER(e);
  if (!(corner_filter_size > 0) || max_corner_points < 1 || max_full_points < 1) return LIO_ERR_INVALID;
  if (e->lc.on || e->frames_started) {
    lio_set_last_error(__FILE__, __LINE__, "lio_est_enable_local_clouds: call it once, before the first lio_est_init_frame");
    return LIO_ERR_INVALID;
  }
  if (e->world > 1 || e->px.npeers || e->px.fpeers) {
    lio_set_last_error(__FILE__, __LINE__, "lio_est_enable_local_clouds: not supported on a sharded context");
    return LIO_ERR_INVALID;
  }
  const int W = e->W;
  LocalClouds lc;
  lc.corner_leaf = corner_filter_size;
  lc.cap[0] = max_corner_points; lc.cap[1] = max_full_points;
  lc.pub_cap[0] = max_corner_points; lc.pub_cap[1] = e->cfg.max_frame_points; lc.pub_cap[2] = max_full_points;
  bool ok = true;
  for (int w = 0; w < 2; ++w) {
    lc.slot[w].resize(W + 1);
    for (int k = 0; k <= W; ++k) ok = ok && alloc(lc.slot[w][k], lc.cap[w]);
    ok = ok && alloc(lc.d_stage[w], lc.cap[w]);
  }
  for (int w = 0; w < 3; ++w) ok = ok && alloc(lc.d_pub[w], lc.pub_cap[w]);
  ok = ok && alloc(lc.d_slot_n, 2 * (W + 1)) && alloc(lc.d_stage_n, 2) && alloc(lc.d_pub_n, 3) &&
       cudaMemset(lc.d_slot_n, 0, sizeof(int) * 2 * (W + 1)) == cudaSuccess && cudaMemset(lc.d_stage_n, 0, sizeof(int) * 2) == cudaSuccess &&
       cudaMemset(lc.d_pub_n, 0, sizeof(int) * 3) == cudaSuccess && lc.vg.init(max_corner_points) == 0 && create(lc.stream) &&
       create(lc.ev_fork) && create(lc.ev_join) &&
       cudaDeviceSynchronize() == cudaSuccess;   // the memsets above ran on the legacy stream
  if (!ok) {   // lc goes: the handle stays usable with local clouds off
    lio_set_last_error(__FILE__, __LINE__, "lio_est_enable_local_clouds: device allocation failed");
    return LIO_ERR_CUDA;
  }
  lc.on = true;
  e->lc = std::move(lc);
  return LIO_OK;
}

// The staging buffers may still be read by the previous push's forked work (stepwise API: staging inside an open scan)
static int lc_stage_wait(lio_est *e) {
  if (e->map.pm && e->window_open) {   // the open scan's /cloud_registered is registered from the staged full cloud when it closes
    lio_set_last_error(__FILE__, __LINE__, "a map is attached: stage the next scan's clouds after lio_est_close_scan");
    return LIO_ERR_INVALID;
  }
  if (e->lc.pending) LIO_CUDA_OK(cudaStreamWaitEvent(e->stream, e->lc.ev_join, 0));
  if (e->map.pending) LIO_CUDA_OK(cudaStreamWaitEvent(e->stream, e->map.ev_done, 0));   // the registration reads the staged full cloud
  return LIO_OK;
}

extern "C" int lio_est_set_scan_clouds_host(lio_est *e, const float *corner, int nc, const float *full, int nf) {
  LIO_ENTER(e);
  if (nc < 0 || nf < 0 || (nc > 0 && !corner) || (nf > 0 && !full)) return LIO_ERR_INVALID;
  if (!e->lc.on) { lio_set_last_error(__FILE__, __LINE__, "local clouds are off: call lio_est_enable_local_clouds first"); return LIO_ERR_INVALID; }
  if (nc > e->lc.cap[0] || nf > e->lc.cap[1]) { lio_set_last_error(__FILE__, __LINE__, "staged cloud exceeds the local-cloud capacity"); return LIO_ERR_CAPACITY; }
  LIO_TRY(lc_stage_wait(e));
  const int hn[2] = {nc, nf};
  if (nc > 0) LIO_CUDA_OK(cudaMemcpyAsync(e->lc.d_stage[0], corner, sizeof(float4) * nc, cudaMemcpyHostToDevice, e->stream));
  if (nf > 0) LIO_CUDA_OK(cudaMemcpyAsync(e->lc.d_stage[1], full, sizeof(float4) * nf, cudaMemcpyHostToDevice, e->stream));
  LIO_CUDA_OK(cudaMemcpyAsync(e->lc.d_stage_n, hn, sizeof(hn), cudaMemcpyHostToDevice, e->stream));
  LIO_CUDA_OK(cudaStreamSynchronize(e->stream));   // hn is a stack array; the caller's buffers are free on return
  e->lc.staged = true;
  return LIO_OK;
}

extern "C" int lio_est_set_scan_clouds_dev(lio_est *e, const float *corner_dev, const int *nc_dev, int nc_max, const float *full_dev,
                                           const int *nf_dev, int nf_max) {
  LIO_ENTER(e);
  if (!corner_dev || !nc_dev || !full_dev || !nf_dev || nc_max < 0 || nf_max < 0) return LIO_ERR_INVALID;
  if (!e->lc.on) { lio_set_last_error(__FILE__, __LINE__, "local clouds are off: call lio_est_enable_local_clouds first"); return LIO_ERR_INVALID; }
  LIO_TRY(lc_stage_wait(e));
  const float *src[2] = {corner_dev, full_dev};
  const int *n_src[2] = {nc_dev, nf_dev};
  const int n_max[2] = {std::min(nc_max, e->lc.cap[0]), std::min(nf_max, e->lc.cap[1])};   // counts are clamped on the device
  for (int w = 0; w < 2; ++w) {
    copy_cloud(reinterpret_cast<const float4 *>(src[w]), n_src[w], n_max[w], e->lc.d_stage[w], e->lc.d_stage_n + w, e->sm_count * 2, e->stream);
  }
  LIO_CUDA_OK(cudaGetLastError());
  e->lc.staged = true;
  return LIO_OK;
}

// The INITED push of the staged clouds and the publication, on lc.stream (forked after the surf push, joined before SlideWindow):
// corner TransformToEnd under the surf cloud's condition + VoxelGrid(corner_filter_size) into corner_stack_[W] (:662-693),
// full_stack_[W] = the staged full cloud (:482), the /local/* gather of frame pivot + 1 (:2362-2375), then TransformToEnd of the
// newest full cloud with keep_intensity (:2416) - after the gather, so that with O = 1 the frame is published before it, as there.
int lc_push(lio_est *e, bool deskew_corner, bool corner_filtered) {
  const int W = e->W, pivot = W - e->O, slot = e->slot_of[W], pub = e->slot_of[pivot + 1];
  cudaStream_t ls = e->lc.stream;
  const int grid_c = std::max(1, std::min(e->sm_count * 2, (e->lc.cap[0] + 255) / 256));
  const int grid_f = std::max(1, std::min(e->sm_count * 4, (e->lc.cap[1] + 255) / 256));
  LIO_CUDA_OK(cudaEventRecord(e->lc.ev_fork, e->stream));
  LIO_CUDA_OK(cudaStreamWaitEvent(ls, e->lc.ev_fork, 0));
  e->lc.pending = true;
  e->lc.staged = false;
  int *n_corner = e->lc.d_slot_n, *n_full = e->lc.d_slot_n + W + 1;
  if (deskew_corner) {
    deskew(e->lc.d_stage[0], e->lc.d_stage_n, e->lc.cap[0], e->es, 10.f, false, ls);
    ++e->launches;
  }
  if (corner_filtered) {   // PointMapping's laser_cloud_corner_stack_downsampled_ (lio_est_attach_mapping, :478)
    copy_cloud(e->lc.d_stage[0], e->lc.d_stage_n, e->lc.cap[0], e->lc.slot[0][slot], n_corner + slot, e->sm_count * 2, ls);
    ++e->launches;
  } else {
    int rc = e->lc.vg.run(e->lc.d_stage[0], e->lc.d_stage_n, e->lc.cap[0], e->lc.corner_leaf, e->lc.slot[0][slot], e->lc.cap[0], n_corner + slot,
                          nullptr, ls, &e->launches);
    if (rc != LIO_OK) return rc;
  }
  copy_cloud(e->lc.d_stage[1], e->lc.d_stage_n + 1, e->lc.cap[1], e->lc.slot[1][slot], n_full + slot, e->sm_count * 4, ls);
  LocalGather G;
  G.src[0] = e->lc.slot[0][pub]; G.n[0] = n_corner + pub;
  G.src[1] = e->slot_ptr[pub]; G.n[1] = e->d_slot_n + pub;
  G.src[2] = e->lc.slot[1][pub]; G.n[2] = n_full + pub;
  for (int w = 0; w < 3; ++w) { G.dst[w] = e->lc.d_pub[w]; G.cap[w] = e->lc.pub_cap[w]; }
  k_local_gather<<<dim3(std::max(grid_c, grid_f), 3), 256, 0, ls>>>(G, e->lc.d_pub_n);
  deskew(e->lc.slot[1][slot], n_full + slot, e->lc.cap[1], e->es, 10.f, true, ls);
  e->launches += 3;
  LIO_CUDA_OK(cudaGetLastError());
  LIO_CUDA_OK(cudaEventRecord(e->lc.ev_join, ls));
  return LIO_OK;
}

int lc_join(lio_est *e) {
  if (!e->lc.pending) return LIO_OK;
  LIO_CUDA_OK(cudaStreamWaitEvent(e->stream, e->lc.ev_join, 0));
  e->lc.pending = false;
  return LIO_OK;
}

extern "C" int lio_est_local_clouds_dev(lio_est *e, const float *ptr[3], const int **n_dev, int n_host[3]) {
  LIO_ENTER_HOST(e);
  if (!e->lc.on) { lio_set_last_error(__FILE__, __LINE__, "local clouds are off"); return LIO_ERR_INVALID; }
  for (int w = 0; w < 3; ++w) {
    if (ptr) ptr[w] = reinterpret_cast<const float *>(e->lc.d_pub[w].get());
    if (n_host) n_host[w] = e->lc.pub_cap[w];
  }
  if (n_dev) *n_dev = e->lc.d_pub_n;
  return LIO_OK;
}
extern "C" int lio_est_local_clouds_download(lio_est *e, int which, float *out, int cap, int *n) {
  LIO_ENTER(e);
  if (!n || which < 0 || which > 2 || (cap > 0 && !out)) return LIO_ERR_INVALID;
  if (!e->lc.on) { lio_set_last_error(__FILE__, __LINE__, "local clouds are off"); return LIO_ERR_INVALID; }
  if (e->lc.pending) LIO_CUDA_OK(cudaStreamSynchronize(e->lc.stream));   // inside an open scan: the forked work has not been joined yet
  int *count = e->h_counts + e->W + 12;
  LIO_TRY(read_back(count, e->lc.d_pub_n + which, 1, 1, e->stream));
  return read_back((float4 *)out, e->lc.d_pub[which], *count, cap, e->stream, n);
}

// ---- the global cube map after initialisation (lio_est_attach_map; Estimator.cc:703-723, :776-812) -------------------------
// transform_lb_ as the float Twist it is
static lio::TwistF lb_twist(const lio_est *e) {
  return lio::TwistF{e->tlb_q[0], e->tlb_q[1], e->tlb_q[2], e->tlb_q[3], e->tlb_p[0], e->tlb_p[1], e->tlb_p[2]};
}

// Scan entry: join the previous scan's map work (it reads frame slots the push below may reuse, and the staged full cloud), predict
// transform_tobe_mapped_ (ProcessCompactData :776-809, imu_factor: tobe * lb * (prev^-1 * curr) * lb^-1 in float Twist, prev / curr
// the float casts of the states W - 1 and W; only on INITED messages: predict is false for the start-up's) and, when W == O with
// de-skew, keep the clouds of the frame that leaves the window: they are the ones this scan inserts (see map_step).
int map_scan_entry(lio_est *e, bool predict) {
  const int W = e->W, O = e->O;
  cudaStream_t st = e->stream;
  if (e->map.pending) { LIO_CUDA_OK(cudaStreamWaitEvent(st, e->map.ev_done, 0)); e->map.pending = false; }
  auto twist_of = [](const M3 &R, const V3 &P) {
    const Q q = fromR(R);
    return lio::TwistF{(float)q.x, (float)q.y, (float)q.z, (float)q.w, (float)P.x, (float)P.y, (float)P.z};
  };
  if (e->cfg.imu_factor && predict) {   // imu_factor = 0: TransformAssociateToMap, run by the mapping's Process (:804)
    const lio::TwistF d = lio::twist_mul(lio::twist_inverse(twist_of(e->Rs[W - 1], e->Ps[W - 1])), twist_of(e->Rs[W], e->Ps[W]));
    const lio::TwistF lb = lb_twist(e);
    lio::TwistF *tobe = pm_tobe(e->map.pm);
    *tobe = lio::twist_mul(lio::twist_mul(lio::twist_mul(*tobe, lb), d), lio::twist_inverse(lb));
  }
  if (W == O && map_deskew(e) && e->map.scans >= O) {
    const int s0 = e->slot_of[0];
    copy_cloud(e->lc.slot[0][s0], e->lc.d_slot_n + s0, e->lc.cap[0], e->map.d_keep[0], e->map.d_keep_n, e->sm_count * 2, st);
    copy_cloud(e->slot_ptr[s0], e->d_slot_n + s0, e->slot_cap, e->map.d_keep[1], e->map.d_keep_n + 1, e->sm_count * 2, st);
    e->launches += 2;
    LIO_CUDA_OK(cudaGetLastError());
  }
  return LIO_OK;
}

// After the solve, before SlideWindow: UpdateMapDatabase of opt_*_stack_.first() (:703-708) from scan O on (the warm-start frames
// count as mapped: opt_point_coeff_mask_ is true for them, :616, and false for INITED frames, :467), then PublishResults (:721).
// The clouds those entries alias (:474-485, :689-693): with either de-skew flag the INITED push of a frame's clouds comes after its
// opt entry was recorded, so the entry is the previous frame's cloud objects - logical frame pivot - 1 now, or the copy kept at the
// scan's entry when W == O.  Without de-skew it is the frame's own objects, logical frame pivot.  The surf object is the slot as
// SlideWindow (:2615) has accumulated it in place; the corner object is never rewritten.  With W == O SlideWindow's prepend drops
// all of surf_stack_[0] (its size is size_surf_stack_[0]), so the frame's own cloud is what the reference inserts there too.
// The pose is opt_transforms_[0] as SolveOptimization overwrites it (:2279-2286).  The work runs on the map's stream.
int map_step(lio_est *e) {
  const int W = e->W, O = e->O, pivot = W - O;
  const bool insert = e->map.scans >= O;
  ++e->map.scans;
  const float4 *src[2] = {nullptr, nullptr};
  const int *n_dev[2] = {nullptr, nullptr};
  int bound[2] = {0, 0};
  if (insert) {
    if (map_deskew(e) && pivot == 0) {
      src[0] = e->map.d_keep[0]; src[1] = e->map.d_keep[1];
      n_dev[0] = e->map.d_keep_n; n_dev[1] = e->map.d_keep_n + 1;
    } else {
      const int s = e->slot_of[map_deskew(e) ? pivot - 1 : pivot];
      src[0] = e->lc.slot[0][s]; src[1] = e->slot_ptr[s];
      n_dev[0] = e->lc.d_slot_n + s; n_dev[1] = e->d_slot_n + s;
    }
    bound[0] = e->lc.cap[0]; bound[1] = e->slot_cap;
    const Tw tlb = tlb_double(e);
    const Q rot = fromR(e->Rs[pivot] * toR(normalized(conj(tlb.rot))));
    const V3 pos = e->Ps[pivot] - rotate(rot, tlb.pos);
    e->map.insert = lio::TwistF{(float)rot.x, (float)rot.y, (float)rot.z, (float)rot.w, (float)pos.x, (float)pos.y, (float)pos.z};
  }
  cudaStream_t ms = pm_stream(e->map.pm);
  LIO_CUDA_OK(cudaEventRecord(e->map.ev_in, e->stream));
  LIO_CUDA_OK(cudaStreamWaitEvent(ms, e->map.ev_in, 0));
  e->map.pending = true;
  // imu_factor = 0: the frame's own valid list and the cube centre it was computed with (opt_valid_idx_ / opt_cube_centers_.first());
  // imu_factor = 1: the lists of the last Process, frozen since
  const bool own = e->mapping.on && !e->cfg.imu_factor;
  const std::vector<size_t> *valid = own ? &e->mapping.opt_valid[pivot] : nullptr;
  const int *centre = own ? e->mapping.opt_centre[pivot].data() : nullptr;
  const int rc = pm_est_step(e->map.pm, insert, src, n_dev, bound, e->map.insert, valid, centre, e->lc.d_stage[1], e->lc.d_stage_n + 1, e->h_counts[W + 13],
                             e->map.info);
  if (rc != LIO_OK) return rc;
  LIO_CUDA_OK(cudaEventRecord(e->map.ev_done, ms));
  return LIO_OK;
}

void AttachedMap::detach() {
  if (!pm) return;
  if (pending) cudaEventSynchronize(ev_done);   // the pending insert reads the estimator's slots
  pm_detach(pm);
  pm = nullptr;
  pending = false;
}

// The estimator's side of both attaches: the map-step events, the W == O de-skew copies, and the handle's own checks (pm_attach).
static int attach_common(lio_est *e, lio_pm *pm, bool fresh) {
  const bool keep = e->W == e->O && map_deskew(e);
  AttachedMap map;
  bool ok = create(map.ev_in) && create(map.ev_done);
  if (keep) ok = ok && alloc(map.d_keep[0], e->lc.cap[0]) && alloc(map.d_keep[1], e->slot_cap) && alloc(map.d_keep_n, 2);
  int rc = ok ? LIO_OK : LIO_ERR_CUDA;
  if (!ok) lio_set_last_error(__FILE__, __LINE__, "lio_est_attach_map: device allocation failed");
  // an accumulated surf slot holds up to max_frame_points * (W - O + 1) points: the map's insert buffers grow to it
  if (ok) rc = pm_attach(pm, e->device, e->lc.corner_leaf, e->cfg.surf_filter_size, e->lc.cap[0] + e->slot_cap, e->lc.cap[1], fresh);
  if (rc != LIO_OK) return rc;   // nothing changed: map goes, the handle stays usable without a map
  map.pm = pm;
  e->map = std::move(map);
  return LIO_OK;
}

extern "C" int lio_est_attach_map(lio_est *e, lio_pm *pm) {
  LIO_ENTER(e);
  if (!pm) return LIO_ERR_INVALID;
  const char *why = nullptr;
  if (e->map.pm) why = "lio_est_attach_map: a map is attached already";
  else if (!e->tmp_pre) why = "lio_est_attach_map: call it after lio_est_finish_init";
  else if (e->scanned) why = "lio_est_attach_map: call it before the first scan";
  else if (!e->lc.on) why = "lio_est_attach_map: local clouds are off (lio_est_enable_local_clouds)";
  else if (!e->cfg.imu_factor) why = "lio_est_attach_map: needs imu_factor = 1";
  else if (e->world > 1 || e->px.npeers || e->px.fpeers) why = "lio_est_attach_map: not supported on a sharded context";
  if (why) { lio_set_last_error(__FILE__, __LINE__, why); return LIO_ERR_INVALID; }
  return attach_common(e, pm, false);
}

extern "C" int lio_est_map_poses(lio_est *e, float tobe7[7], float aft7[7], float insert7[7], int info4[4]) {
  LIO_ENTER_HOST(e);
  if (!e->map.pm) { lio_set_last_error(__FILE__, __LINE__, "no map attached (lio_est_attach_map)"); return LIO_ERR_INVALID; }
  auto out = [](const lio::TwistF &t, float *o) { if (o) { o[0] = t.qx; o[1] = t.qy; o[2] = t.qz; o[3] = t.qw; o[4] = t.px; o[5] = t.py; o[6] = t.pz; } };
  out(*pm_tobe(e->map.pm), tobe7);
  out(pm_aft(e->map.pm), aft7);
  out(e->map.insert, insert7);
  if (info4) for (int k = 0; k < 4; ++k) info4[k] = e->map.info[k];
  return LIO_OK;
}

// ---- imu_factor = 0 from the odometry's clouds (lio_est_attach_mapping; Estimator.cc:430-856) ------------------------------
// SolveOptimization :1670-1676: state W from the increment of the last two pushed laser transforms, incre = (lb^-1 * T_{W-1}^-1 * T_W
// * lb) in float Twist, cast to double; Ps_[W] = Rs_[W-1] * incre.pos + Ps_[W-1], Rs_[W] = Rs_[W-1] * incre.rot.  Every input is host
// state (the mapping's optimiser reads its pose back before the call returns), so this is host arithmetic with no device round trip.
void predict_state_w(lio_est *e) {
  const int W = e->W;
  const lio::TwistF lb = lb_twist(e);
  const lio::TwistF inc = lio::twist_mul(lio::twist_mul(lio::twist_mul(lio::twist_inverse(lb), lio::twist_inverse(e->mapping.laser_tf[W - 1])), e->mapping.laser_tf[W]), lb);
  const V3 p((double)inc.px, (double)inc.py, (double)inc.pz);
  e->Ps[W] = e->Rs[W - 1] * p + e->Ps[W - 1];
  e->Rs[W] = e->Rs[W - 1] * toR(Q((double)inc.qw, (double)inc.qx, (double)inc.qy, (double)inc.qz));
}

static int attach_mapping(lio_est *e, lio_pm *pm, bool imu) {
  if (!pm) return LIO_ERR_INVALID;
  const char *why = nullptr;
  if (e->map.pm) why = "a map is attached already";
  else if (e->frames_started || e->tmp_pre) why = "call it before lio_est_init_frame / lio_est_finish_init and the first scan";
  else if (!e->lc.on) why = "local clouds are off (lio_est_enable_local_clouds)";
  else if (!imu && e->cfg.imu_factor) why = "lio_est_attach_mapping needs imu_factor = 0 (lio_est_attach_imu_mapping takes imu_factor = 1)";
  else if (imu && !e->cfg.imu_factor) why = "lio_est_attach_imu_mapping needs imu_factor = 1";
  else if (imu && e->W < 5) why = "lio_est_attach_imu_mapping: ImuInitializer needs window_size >= 5 (ApproximateGravity)";
  else if (imu && e->extrinsic_stage == 2 && !e->calib.on)
    why = "lio_est_attach_imu_mapping: estimate_extrinsic = 2 needs lio_est_enable_extrinsic_calibration first";
  else if (e->world > 1 || e->px.npeers || e->px.fpeers) why = "not supported on a sharded context";
  if (why) { lio_set_last_error(__FILE__, __LINE__, why); return LIO_ERR_INVALID; }
  const int rc = attach_common(e, pm, true);
  if (rc != LIO_OK) return rc;
  const int W = e->W;
  e->mapping.on = true;
  e->mapping.laser_tf.assign(W + 1, lio::TwistF{});
  e->mapping.opt_valid.assign(W + 1, std::vector<size_t>());
  e->mapping.opt_centre.assign(W + 1, std::array<int, 3>{0, 0, 0});
  // ProcessImu needs a pre-integration to fill once the first laser frame is in (:379-381); ImuFactors are not part of the solve
  e->tmp_pre = std::make_shared<Preintegration>(e->acc_last, e->gyr_last, e->Bas[0], e->Bgs[0], e->noise);
  return LIO_OK;
}

extern "C" int lio_est_attach_mapping(lio_est *e, lio_pm *pm) { LIO_ENTER(e); return attach_mapping(e, pm, false); }
extern "C" int lio_est_attach_imu_mapping(lio_est *e, lio_pm *pm) { LIO_ENTER(e); return attach_mapping(e, pm, true); }

extern "C" int lio_est_enable_extrinsic_calibration(lio_est *e) {
  LIO_ENTER_HOST(e);
  const char *why = nullptr;
  if (!e->cfg.imu_factor || e->extrinsic_stage != 2) why = "lio_est_enable_extrinsic_calibration needs imu_factor = 1 and estimate_extrinsic = 2";
  else if (e->calib.on) why = "lio_est_enable_extrinsic_calibration: call it once";
  else if (e->mapping.on || e->map.pm || e->frames_started || e->tmp_pre) why = "lio_est_enable_extrinsic_calibration: call it before the attach and any frame";
  if (why) { lio_set_last_error(__FILE__, __LINE__, why); return LIO_ERR_INVALID; }
  e->calib.on = true;
  return LIO_OK;
}

// all_laser_transforms_ 0..W's pre-integrations on the window the push has just filled: pre_[1..W] and tmp_pre (the push moves them one
// place later; the objects, which an attempt repropagates, are the same)
static std::vector<Preintegration *> window_pre(lio_est *e) {
  const int W = e->W;
  std::vector<Preintegration *> pre(W + 1);
  for (int i = 0; i < W; ++i) pre[i] = e->pre[i + 1].get();
  pre[W] = e->tmp_pre.get();
  return pre;
}

// EstimateExtrinsicRotation (:520-531) on that window, with no stamp gate: transform_lb_'s rotation is overwritten whether or not it
// succeeds; a success ends extrinsic stage 2
static void calib_attempt(lio_est *e) {
  const std::vector<Preintegration *> pre = window_pre(e);
  lio::TwistF tlb = lb_twist(e);
  const bool ok = estimate_extrinsic_rotation(e->W, e->mapping.laser_tf.data(), pre.data(), tlb, e->calib.sv);
  e->tlb_q[0] = tlb.qx; e->tlb_q[1] = tlb.qy; e->tlb_q[2] = tlb.qz; e->tlb_q[3] = tlb.qw;
  ++e->calib.runs;
  e->calib.result = ok ? 1 : 0;
  e->calib.ran = true;
  if (ok) e->extrinsic_stage = 1;
}

// RunInitialization (:858-958) on the same window
static int imu_attempt(lio_est *e, double stamp) {
  const int W = e->W;
  const std::vector<Preintegration *> pre = window_pre(e);
  const int rc = run_initialization(W, e->mapping.laser_tf.data(), pre.data(), lb_twist(e), e->noise.g_norm, e->Bas.data(), e->Bgs.data(),
                                    e->Vs.data(), e->mapping.R_WI, e->Ps.data(), e->Rs.data(), e->g_vec);
  ++e->mapping.attempts;
  e->mapping.attempted = true;
  e->mapping.attempt_states.resize(16 * (W + 1));
  lio_est_get_states(e, e->mapping.attempt_states.data());
  e->mapping.initial_time = stamp;   // :536
  if (rc == kInitNotFinite) {
    lio_set_last_error(__FILE__, __LINE__, "RunInitialization: non-finite result (TangentBasis of a gravity exactly along +z)");
    return LIO_ERR_NUMERIC;
  }
  e->mapping.outcome = rc;
  return LIO_OK;
}

// ProcessCompactData (:776-856) with update_laser_imu: PointMapping::Process on the mapping's stream (not once imu_factor = 1 is
// inited, :810-812), then ProcessLaserOdom.  corner / surf / full and n3_dev are the message's clouds and counts, n_max their bounds
// (already capped by the mapping's capacities); stamp is header.stamp (imu_factor = 1 only).
static int compact_body(lio_est *e, const float4 *const src[3], const int *n3_dev, const int n_max[3], const float sum7[7], double stamp) {
  const int W = e->W;
  cudaStream_t st = e->stream, ms = pm_stream(e->map.pm);
  const bool process = !(e->mapping.inited && e->cfg.imu_factor);
  // Process overwrites the handle's stacks and full cloud, which the estimator's previous pushes read on its own stream; without it
  // the estimator's stream still waits for the host entry's upload on the mapping's stream
  LIO_CUDA_OK(cudaEventRecord(e->map.ev_in, st));
  LIO_CUDA_OK(cudaStreamWaitEvent(ms, e->map.ev_in, 0));
  int rc = process ? pm_est_process(e->map.pm, src, src[2], n3_dev, n_max, sum7) : LIO_OK;
  if (rc != LIO_OK) return rc;
  LIO_CUDA_OK(cudaEventRecord(e->map.ev_done, ms));
  LIO_CUDA_OK(cudaStreamWaitEvent(st, e->map.ev_done, 0));
  e->map.pending = false;
  ++e->mapping.recv_count;
  e->mapping.compact_info[0] = e->mapping.inited ? 1 : 0; e->mapping.compact_info[1] = e->mapping.cir_count; e->mapping.compact_info[2] = e->mapping.compact_info[3] = 0;
  e->mapping.attempted = false;
  e->calib.ran = false;
  if (!e->mapping.inited && e->mapping.recv_count % e->cfg.init_window_factor != 0) return LIO_OK;   // :436-439
  // the push (:441-487): the laser transform is transform_aft_mapped_, the stacks PointMapping's down-sampled ones unless the INITED
  // de-skew rules push their own (:474-480, :628-693)
  const bool pm_stacks = !e->mapping.inited || !map_deskew(e);
  const int nds[2] = {pm_ds_n(e->map.pm, 0), pm_ds_n(e->map.pm, 1)};
  if (pm_stacks && (nds[1] > e->cfg.max_frame_points || nds[0] > e->lc.cap[0])) {
    lio_set_last_error(__FILE__, __LINE__, "the mapping's down-sampled stacks exceed max_frame_points / the local corner capacity");
    return LIO_ERR_CAPACITY;
  }
  const int *cnt = pm_counts_dev(e->map.pm);   // {corner in, surf in, corner ds, surf ds, full}
  const int *n_in = process ? cnt : n3_dev;     // the message's counts: Process's copies, or the caller's own
  rc = lc_stage_wait(e);
  if (rc != LIO_OK) return rc;
  {
    const float4 *sc[2] = {pm_stacks ? pm_ds(e->map.pm, 0) : src[0], process ? pm_full_in(e->map.pm) : src[2]};
    const int *nc[2] = {pm_stacks ? cnt + 2 : n_in, process ? cnt + 4 : n3_dev + 2};
    const int nb[2] = {process || pm_stacks ? e->lc.cap[0] : n_max[0], n_max[2]};
    for (int w = 0; w < 2; ++w) copy_cloud(sc[w], nc[w], nb[w], e->lc.d_stage[w], e->lc.d_stage_n + w, e->sm_count * 2, st);
    LIO_CUDA_OK(cudaGetLastError());
    e->lc.staged = true;
  }
  push_shift(e->mapping.laser_tf, pm_aft(e->map.pm));
  push_shift(e->mapping.opt_valid, pm_valid(e->map.pm));
  {
    std::array<int, 3> c;
    pm_centre(e->map.pm, c.data());
    push_shift(e->mapping.opt_centre, c);
  }
  e->mapping.compact_info[2] = 1;
  const int c = e->mapping.cir_count;
  const V3 tmp_bg = e->Bgs[c];
  bool startup = !e->mapping.inited && c == W;
  if (startup && e->cfg.imu_factor) {   // :520-537
    startup = false;
    if (e->extrinsic_stage == 2) calib_attempt(e);
    if (e->extrinsic_stage != 2 && stamp - e->mapping.initial_time > 0.1) {
      if ((rc = imu_attempt(e, stamp)) != LIO_OK) return rc;
      startup = e->mapping.outcome == kInitSuccess;
    }
  }
  if (!e->mapping.inited && !startup) {   // NOT_INITED without a start-up: push, then SlideWindow's state copy (:600-614)
    push_shift(e->pre, e->tmp_pre);
    e->tmp_pre = std::make_shared<Preintegration>(e->acc_last, e->gyr_last, e->Bas[c], tmp_bg, e->noise);
    const int freed = e->slot_of[0];
    e->slot_of.erase(e->slot_of.begin());
    e->slot_of.push_back(freed);
    const int slot = e->slot_of[W];
    copy_cloud(pm_ds(e->map.pm, 1), cnt + 3, e->cfg.max_frame_points, e->slot_ptr[slot], e->d_slot_n + slot, e->sm_count * 2, st);
    for (int w = 0; w < 2; ++w)
      copy_cloud(e->lc.d_stage[w], e->lc.d_stage_n + w, e->lc.cap[w], e->lc.slot[w][slot], e->lc.d_slot_n + w * (W + 1) + slot, e->sm_count * 2, st);
    LIO_CUDA_OK(cudaGetLastError());
    LIO_CUDA_OK(cudaMemcpyAsync(e->d_own_n + slot, e->d_slot_n + slot, sizeof(int), cudaMemcpyDeviceToDevice, st));
    e->lc.staged = false;
    push_shift(e->size_surf_stack, nds[1]);
    if (c < W) {   // ++cir_buf_count_ (:613)
      e->Ps[c + 1] = e->Ps[c]; e->Vs[c + 1] = e->Vs[c]; e->Rs[c + 1] = e->Rs[c]; e->Bas[c + 1] = e->Bas[c]; e->Bgs[c + 1] = e->Bgs[c];
      e->mapping.compact_info[1] = ++e->mapping.cir_count;
    } else {       // imu_factor = 1, full window, no successful attempt (:600-602): the buffers move on, state W is kept
      push_shift(e->Ps, e->Ps[W]); push_shift(e->Vs, e->Vs[W]); push_shift(e->Rs, e->Rs[W]); push_shift(e->Bas, e->Bas[W]);
      push_shift(e->Bgs, e->Bgs[W]);
    }
    return LIO_OK;
  }
  CompactPush cp{nullptr, nullptr, pm_stacks, !e->mapping.inited, tmp_bg};
  if (pm_stacks) { cp.surf_ds = pm_ds(e->map.pm, 1); cp.surf_ds_n = cnt + 3; }
  if (!e->mapping.inited && !e->cfg.imu_factor) {   // the start-up (:505-517): states 0..W from the W + 1 pushed laser transforms
    const lio::TwistF lb = lb_twist(e);
    for (int i = 0; i <= W; ++i) {
      const lio::TwistF tb = lio::twist_mul(e->mapping.laser_tf[i], lb);
      float R[9];
      lio::quat_to_matrix_normalized(tb, R);
      e->Ps[i] = V3((double)tb.px, (double)tb.py, (double)tb.pz);
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) e->Rs[i](a, b) = (double)R[3 * a + b];
    }
  }
  if (!e->mapping.inited) {   // then (either mode) the first solve and SlideWindow
    e->mapping.inited = true;
    pm_set_imu_inited(e->map.pm);   // SetInitFlag(true) (:544)
    e->mapping.quiet = true;
  }
  rc = process_scan_body(e, src[1], n_in + 1, std::max(1, std::min(n_max[1], e->cfg.max_scan_points)), false, &cp);
  e->mapping.quiet = false;
  if (rc != LIO_OK) return rc;
  e->mapping.compact_info[0] = 1; e->mapping.compact_info[3] = 1;
  return LIO_OK;
}

static int compact_common(lio_est *e, const float4 *const src[3], const int *n3_dev, const int n_max[3], const float sum7[7], double stamp) {
  if (e->poisoned) return refuse_poisoned(e);
  // the full cloud is pushed into a local full slot, and with a de-skew flag the raw corner cloud is staged after initialisation:
  // bounds above those capacities are refused before anything changes, as lio_est_set_scan_clouds_* refuses them
  if (n_max[2] > e->lc.cap[1] || (map_deskew(e) && n_max[0] > e->lc.cap[0])) {
    lio_set_last_error(__FILE__, __LINE__, "a cloud bound exceeds the local-cloud capacity (lio_est_enable_local_clouds)");
    return LIO_ERR_CAPACITY;
  }
  e->frames_started = true;
  e->scanned = true;
  const int rc = compact_body(e, src, n3_dev, n_max, sum7, stamp);
  return rc != LIO_OK ? scan_failed(e, rc) : rc;
}

static int compact_check(lio_est *e) {
  if (!e->mapping.on) { lio_set_last_error(__FILE__, __LINE__, "no mapping attached (lio_est_attach_mapping)"); return LIO_ERR_INVALID; }
  return LIO_OK;
}

// The unstamped entries pass a NaN stamp, which an IMU mapping refuses: its attempts are gated on the stamps
static int compact_check(lio_est *e, double stamp) {
  const int rc = compact_check(e);
  if (rc != LIO_OK) return rc;
  if (e->cfg.imu_factor && std::isnan(stamp)) {
    lio_set_last_error(__FILE__, __LINE__, "an IMU mapping takes the message stamps: lio_est_process_compact_stamped_*");
    return LIO_ERR_INVALID;
  }
  return LIO_OK;
}

static int compact_dev(lio_est *e, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev, const int n3_max[3],
                       const float transform_sum7[7], double stamp) {
  if (!n3_dev || !n3_max || !transform_sum7 || n3_max[0] < 0 || n3_max[1] < 0 || n3_max[2] < 0 || (n3_max[0] > 0 && !corner_dev) ||
      (n3_max[1] > 0 && !surf_dev) || (n3_max[2] > 0 && !full_dev))
    return LIO_ERR_INVALID;
  LIO_TRY(compact_check(e, stamp));
  int n_max[3];
  pm_est_caps(e->map.pm, n3_max, n_max);
  const float4 *src[3] = {reinterpret_cast<const float4 *>(corner_dev), reinterpret_cast<const float4 *>(surf_dev), reinterpret_cast<const float4 *>(full_dev)};
  return compact_common(e, src, n3_dev, n_max, transform_sum7, stamp);
}

static int compact_host(lio_est *e, const float *corner, int nc, const float *surf, int ns, const float *full, int nf, const float transform_sum7[7],
                        double stamp) {
  if (!transform_sum7 || nc < 0 || ns < 0 || nf < 0 || (nc > 0 && !corner) || (ns > 0 && !surf) || (nf > 0 && !full)) return LIO_ERR_INVALID;
  int rc = compact_check(e, stamp);
  if (rc != LIO_OK) return rc;
  if (e->poisoned || nf > e->lc.cap[1] || (map_deskew(e) && nc > e->lc.cap[0])) {
    const int n_max[3] = {nc, ns, nf};
    return compact_common(e, nullptr, nullptr, n_max, transform_sum7, stamp);
  }
  // the handle's input buffers are rewritten: the previous message's pushes (on the estimator's stream) read them
  LIO_CUDA_OK(cudaStreamSynchronize(e->stream));
  const float4 *src[3];
  const int *n3_dev = nullptr;
  if ((rc = pm_est_upload(e->map.pm, corner, nc, surf, ns, full, nf, src, &n3_dev)) != LIO_OK) return rc;
  const int n_max[3] = {nc, ns, nf};
  return compact_common(e, src, n3_dev, n_max, transform_sum7, stamp);
}

extern "C" int lio_est_process_compact_dev(lio_est *e, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev,
                                           const int n3_max[3], const float transform_sum7[7]) {
  LIO_ENTER(e);
  return compact_dev(e, corner_dev, surf_dev, full_dev, n3_dev, n3_max, transform_sum7, std::nan(""));
}
extern "C" int lio_est_process_compact_host(lio_est *e, const float *corner, int nc, const float *surf, int ns, const float *full, int nf,
                                            const float transform_sum7[7]) {
  LIO_ENTER(e);
  return compact_host(e, corner, nc, surf, ns, full, nf, transform_sum7, std::nan(""));
}
extern "C" int lio_est_process_compact_stamped_dev(lio_est *e, const float *corner_dev, const float *surf_dev, const float *full_dev,
                                                   const int *n3_dev, const int n3_max[3], const float transform_sum7[7], double stamp) {
  LIO_ENTER(e);
  if (std::isnan(stamp)) return LIO_ERR_INVALID;
  return compact_dev(e, corner_dev, surf_dev, full_dev, n3_dev, n3_max, transform_sum7, stamp);
}
extern "C" int lio_est_process_compact_stamped_host(lio_est *e, const float *corner, int nc, const float *surf, int ns, const float *full, int nf,
                                                    const float transform_sum7[7], double stamp) {
  LIO_ENTER(e);
  if (std::isnan(stamp)) return LIO_ERR_INVALID;
  return compact_host(e, corner, nc, surf, ns, full, nf, transform_sum7, stamp);
}

extern "C" int lio_est_compact_status(lio_est *e, int info4[4]) {
  LIO_ENTER_HOST(e);
  if (!info4) return LIO_ERR_INVALID;
  LIO_TRY(compact_check(e));
  for (int k = 0; k < 4; ++k) info4[k] = e->mapping.compact_info[k];
  return LIO_OK;
}

extern "C" int lio_est_imu_init_status(lio_est *e, int info4[4], double g3[3], double R_WI9[9], double *states16) {
  LIO_ENTER_HOST(e);
  if (!info4) return LIO_ERR_INVALID;
  LIO_TRY(compact_check(e));
  info4[0] = e->mapping.attempts; info4[1] = e->mapping.outcome; info4[2] = e->mapping.attempted ? 1 : 0; info4[3] = e->mapping.inited ? 1 : 0;
  if (g3) for (int k = 0; k < 3; ++k) g3[k] = e->g_vec[k];
  if (R_WI9) for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) R_WI9[3 * a + b] = e->mapping.R_WI(a, b);
  if (states16 && !e->mapping.attempt_states.empty())
    std::memcpy(states16, e->mapping.attempt_states.data(), sizeof(double) * e->mapping.attempt_states.size());
  return LIO_OK;
}

extern "C" int lio_est_extrinsic_calib_status(lio_est *e, int info4[4], double sv4[4]) {
  LIO_ENTER_HOST(e);
  if (!info4) return LIO_ERR_INVALID;
  info4[0] = e->calib.runs; info4[1] = e->calib.result; info4[2] = e->calib.ran ? 1 : 0; info4[3] = e->extrinsic_stage;
  if (sv4) for (int k = 0; k < 4; ++k) sv4[k] = e->calib.sv[k];
  return LIO_OK;
}
