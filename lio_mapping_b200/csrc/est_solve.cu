// The window solve of the device estimator: BuildLocalMap (Estimator.cc:1361-1646) with the per-scan feature exchange of a sharded
// context, the stage-C lidar reduction and its rows exchange, the host linearisation, the marginalisation (MarginalizationFactor.cc),
// the host and the device-resident dogleg solvers (SolveOptimization :1648-2438) and SlideWindow (:2570-2666).
#include "estimator.cuh"

namespace lio {

// ------------------------------------------------------------------------------------------------
// kernels
struct ConcatParams {
  const float4 *src[kMaxWindow];
  const int *n[kMaxWindow];
  float R[kMaxWindow][9];
  float t[kMaxWindow][3];
  float tag[kMaxWindow];
  int identity[kMaxWindow];  // copy as is (pivot frame keeps its intensity)
  int skip_first[kMaxWindow];  // drop the first k points (SlideWindow ExtractIndices), value read from *skip_n
  const int *skip_n[kMaxWindow];
  int nsrc;
};

// pcl::transformPointCloud (x' = m00 x + m01 y + m02 z + m03, left to right) + intensity tag + concat
// (Estimator.cc:1498-1507, :2600-2611).  Exact float order: compiled with -fmad=false.
__global__ void __launch_bounds__(256)
k_concat(const ConcatParams P, float4 *__restrict__ dst, int *__restrict__ n_out, int cap) {
  __shared__ int off[kMaxWindow + 1];
  __shared__ int skip[kMaxWindow];
  if (threadIdx.x == 0) {
    int run = 0;
    for (int k = 0; k < P.nsrc; ++k) {
      int sk = P.skip_first[k] ? *P.skip_n[k] : 0;
      int nk = *P.n[k] - sk;
      if (nk < 0) nk = 0;
      skip[k] = sk;
      off[k] = run;
      run += nk;
    }
    off[P.nsrc] = run;
    if (blockIdx.x == 0) *n_out = run < cap ? run : cap;
  }
  __syncthreads();
  const int total = min(off[P.nsrc], cap);
  for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < total; g += gridDim.x * blockDim.x) {
    int k = 0;
    while (k + 1 < P.nsrc && g >= off[k + 1]) ++k;
    float4 p = __ldg(P.src[k] + (g - off[k]) + skip[k]);
    if (!P.identity[k]) {
      const float *R = P.R[k];
      const float *t = P.t[k];
      float x = R[0] * p.x + R[1] * p.y + R[2] * p.z + t[0];
      float y = R[3] * p.x + R[4] * p.y + R[5] * p.z + t[1];
      float z = R[6] * p.x + R[7] * p.y + R[8] * p.z + t[2];
      p = make_float4(x, y, z, P.tag[k] >= 0.f ? P.tag[k] : p.w);
    }
    dst[g] = p;
  }
}

}  // namespace lio

// Twist<double> -> cast<float>() -> transform(): float quaternion normalised in float, float matrix
struct AffineF { float R[9]; float t[3]; TransformF tf; };
static AffineF to_affine_f(const Tw &t) {
  AffineF a;
  lio::TwistF tw;
  tw.qx = (float)t.rot.x; tw.qy = (float)t.rot.y; tw.qz = (float)t.rot.z; tw.qw = (float)t.rot.w;
  quat_to_matrix_normalized(tw, a.R);
  a.t[0] = (float)t.pos.x; a.t[1] = (float)t.pos.y; a.t[2] = (float)t.pos.z;
  // Twist<float>(Affine3f): Quaternionf(linear).normalized()
  float q[4];
  matrix_to_quat(a.R, q);
  float qn = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  a.tf.qx = q[0] / qn; a.tf.qy = q[1] / qn; a.tf.qz = q[2] / qn; a.tf.qw = q[3] / qn;
  a.tf.px = a.t[0]; a.tf.py = a.t[1]; a.tf.pz = a.t[2];
  return a;
}

// point the per-frame feature descriptors at one parity of the slab
void set_feature_parity(lio_est *e, int par) {
  char *base = e->px.fslab + (size_t)par * e->px.fpar_stride;
  e->d_feat_counts = reinterpret_cast<int *>(base + e->px.foff_cnt);
  const int pivot = e->W - e->O;
  for (int k = pivot + 1; k <= e->W; ++k) {
    FeatureOut &f = e->feats[k];
    f.pts = reinterpret_cast<float4 *>(base + e->px.foff_pts[k]);
    f.coef = reinterpret_cast<float4 *>(base + e->px.foff_coef[k]);
    f.count = e->d_feat_counts + k;
  }
  e->px.fparity = par;
}

// ---- per-scan feature exchange over peer memory (sharded runs) ----------------------------------------------------------
struct FeaturePeers {
  float4 *pts[kMaxPeers], *coef[kMaxPeers];
  int *count[kMaxPeers];
  int npeers, self;
};
// An owned frame's features go to the same place in every peer's slab (plain P2P stores over NVLink / NVSwitch).
__global__ void __launch_bounds__(256)
k_publish_features(const float4 *__restrict__ pts, const float4 *__restrict__ coef, const int *__restrict__ count, int cap, FeaturePeers P) {
  const int n = min(*count, cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 v = pts[i], w = coef[i];
    for (int r = 0; r < P.npeers; ++r) if (r != P.self) { P.pts[r][i] = v; P.coef[r][i] = w; }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) for (int r = 0; r < P.npeers; ++r) if (r != P.self) *P.count[r] = *count;
}
struct FlagPeers { unsigned *flag[kMaxPeers]; int npeers, self; };
// after the publishing kernels of this rank have completed (stream order): the scan's epoch into every rank's flag slot
__global__ void k_publish_flag(FlagPeers P, unsigned epoch) {
  __threadfence_system();
  if ((int)threadIdx.x < P.npeers) {
    unsigned *fl = P.flag[threadIdx.x] + P.self;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(fl), "r"(epoch) : "memory");
  }
}

// ---- parameter <-> state ---------------------------------------------------------------------------
void vector_to_double(lio_est *e) {  // Estimator.cc:2440-2478
  const int pivot = e->W - e->O;
  for (int i = 0, oi = pivot; i <= e->O; ++i, ++oi) {
    double *pp = e->para_pose[i].data(), *sb = e->para_sb[i].data();
    pp[0] = e->Ps[oi].x; pp[1] = e->Ps[oi].y; pp[2] = e->Ps[oi].z;
    Q q = fromR(e->Rs[oi]);
    pp[3] = q.x; pp[4] = q.y; pp[5] = q.z; pp[6] = q.w;
    for (int k = 0; k < 3; ++k) { sb[k] = e->Vs[oi][k]; sb[3 + k] = e->Bas[oi][k]; sb[6 + k] = e->Bgs[oi][k]; }
  }
  e->para_ex[0] = e->tlb_p[0]; e->para_ex[1] = e->tlb_p[1]; e->para_ex[2] = e->tlb_p[2];
  e->para_ex[3] = e->tlb_q[0]; e->para_ex[4] = e->tlb_q[1]; e->para_ex[5] = e->tlb_q[2]; e->para_ex[6] = e->tlb_q[3];
  e->S_valid = false;
}

void double_to_vector(lio_est *e) {  // Estimator.cc:2479-2568
  const int pivot = e->W - e->O, O = e->O;
  const V3 origin_P0 = e->Ps[pivot];
  const V3 origin_R0 = R2ypr(e->Rs[pivot]);
  auto qpose = [&](int i) { const double *p = e->para_pose[i].data(); return toR(normalized(Q(p[6], p[3], p[4], p[5]))); };
  const V3 origin_R00 = R2ypr(qpose(0));
  const double y_diff = origin_R0.x - origin_R00.x;
  M3 rot_diff = ypr2R(V3(y_diff, 0, 0));
  if (std::fabs(std::fabs(origin_R0.y) - 90) < 1.0 || std::fabs(std::fabs(origin_R00.y) - 90) < 1.0) rot_diff = e->Rs[pivot] * T(qpose(0));
  {
    Tw trans_pivot(fromR(e->Rs[pivot]), e->Ps[pivot]);
    Tw trans_opt_pivot(fromR(rot_diff * qpose(0)), origin_P0);
    for (int idx = 0; idx < pivot; ++idx) {
      Tw trans_idx(fromR(e->Rs[idx]), e->Ps[idx]);
      Tw o = tw_mul(tw_mul(trans_opt_pivot, tw_inverse(trans_pivot)), trans_idx);
      e->Ps[idx] = o.pos;
      e->Rs[idx] = toR(normalized(o.rot));
    }
  }
  for (int i = 0, oi = pivot; i <= O; ++i, ++oi) {
    const double *pp = e->para_pose[i].data(), *p0 = e->para_pose[0].data(), *sb = e->para_sb[i].data();
    e->Rs[oi] = rot_diff * qpose(i);
    e->Ps[oi] = rot_diff * V3(pp[0] - p0[0], pp[1] - p0[1], pp[2] - p0[2]) + origin_P0;
    e->Vs[oi] = rot_diff * V3(sb[0], sb[1], sb[2]);
    e->Bas[oi] = V3(sb[3], sb[4], sb[5]);
    e->Bgs[oi] = V3(sb[6], sb[7], sb[8]);
  }
  e->tlb_p[0] = (float)e->para_ex[0]; e->tlb_p[1] = (float)e->para_ex[1]; e->tlb_p[2] = (float)e->para_ex[2];
  e->tlb_q[0] = (float)e->para_ex[3]; e->tlb_q[1] = (float)e->para_ex[4]; e->tlb_q[2] = (float)e->para_ex[5]; e->tlb_q[3] = (float)e->para_ex[6];
}

// ---- stage B orchestration -----------------------------------------------------------------------
// How a sharded context completes the lidar reduction of a solve.  features: the features themselves were exchanged, so every rank
// holds all of them and solves like a single GPU (this wins even when the rows exchange was also set up); rows: the peer-memory
// exchange of the S rows (lio_est_set_peers), which wins over the allreduce callback; missing: a sharded context with neither.
enum class Exchange { none, features, rows, callback, missing };
static Exchange exchange_of(const lio_est *e) {
  if (e->world == 1) return Exchange::none;
  if (e->px.fpeers) return Exchange::features;
  if (e->px.npeers == e->world) return Exchange::rows;
  return e->allreduce ? Exchange::callback : Exchange::missing;
}
static bool owns_frame(const lio_est *e, int idx) {  // idx: logical frame > pivot
  const int pivot = e->W - e->O;
  return lio_est_frame_owner(idx - pivot, e->world) == e->rank;
}

__global__ void k_xwait(const unsigned *__restrict__ flags, int npeers, unsigned epoch, int *__restrict__ err, const int *__restrict__ skip);

// Reports a bounded peer wait (k_xwait) of the feature or rows exchange that gave up, after its error word was read back.  The word
// is one-shot: its device and host copies are cleared with the report.
static int xwait_report(lio_est *e, Exchange x, cudaStream_t st) {
  const bool features = x == Exchange::features;
  int *h = features ? e->h_counts + e->W + 9 : e->h_xerr;
  if (!*h) return LIO_OK;
  cudaMemsetAsync(features ? e->px.fslab + e->px.foff_flags + 128 : e->px.xbuf + kXErrOff, 0, sizeof(int), st);
  *h = 0;
  lio_set_last_error(__FILE__, __LINE__, features ? "feature exchange timed out (a rank did not publish its frames)"
                                                  : "peer exchange timed out (a rank did not publish its rows)");
  return LIO_ERR_CUDA;
}

int build_local_map(lio_est *e, const std::function<int()> &before_sync) {
  const int W = e->W, O = e->O, pivot = W - O;
  cudaStream_t st = e->stream;
  const double t0 = now_s();
  const Tw tlb = tlb_double(e);
  const Tw transform_pivot = lidar_pose(e->Ps[pivot], e->Rs[pivot], tlb);
  const Tw pivot_inv = tw_inverse(transform_pivot);
  if (!e->init_local_map) {  // :1409-1441 merge frames 0..pivot into the pivot cloud
    if (pivot > 0) {
      ConcatParams cp;
      std::memset(&cp, 0, sizeof(cp));
      cp.nsrc = pivot + 1;
      for (int i = 0; i <= pivot; ++i) {
        AffineF a = to_affine_f(tw_mul(pivot_inv, lidar_pose(e->Ps[i], e->Rs[i], tlb)));
        cp.src[i] = e->slot_ptr[e->slot_of[i]];
        cp.n[i] = e->d_slot_n + e->slot_of[i];
        std::memcpy(cp.R[i], a.R, sizeof(a.R)); std::memcpy(cp.t[i], a.t, sizeof(a.t));
        cp.tag[i] = -1.f;  // keep intensity
      }
      k_concat<<<std::max(1, std::min(e->sm_count * 2, (e->slot_cap + 255) / 256)), 256, 0, st>>>(cp, e->d_tmp, e->d_counts + 3, e->slot_cap);
      ++e->launches;
      const int ps = e->slot_of[pivot];
      LIO_CUDA_OK(cudaMemcpyAsync(e->slot_ptr[ps], e->d_tmp, sizeof(float4) * e->slot_cap, cudaMemcpyDeviceToDevice, st));
      LIO_CUDA_OK(cudaMemcpyAsync(e->d_slot_n + ps, e->d_counts + 3, sizeof(int), cudaMemcpyDeviceToDevice, st));
    }
    e->init_local_map = true;
  }
  ConcatParams cp;
  std::memset(&cp, 0, sizeof(cp));
  int ns = 0;
  for (int i = 0; i <= W; ++i) {
    AffineF a = to_affine_f(tw_mul(pivot_inv, lidar_pose(e->Ps[i], e->Rs[i], tlb)));
    e->local_tf[i] = a.tf;
    e->h_tf[i] = a.tf;
    if (i < pivot || i == W) continue;
    cp.src[ns] = e->slot_ptr[e->slot_of[i]];
    cp.n[ns] = e->d_slot_n + e->slot_of[i];
    if (i == pivot) cp.identity[ns] = 1;
    else { std::memcpy(cp.R[ns], a.R, sizeof(a.R)); std::memcpy(cp.t[ns], a.t, sizeof(a.t)); cp.tag[ns] = (float)i; }
    ++ns;
  }
  cp.nsrc = ns;
  LIO_CUDA_OK(cudaMemcpyAsync(e->d_tf, e->h_tf, sizeof(TransformF) * (W + 1), cudaMemcpyHostToDevice, st));
  k_concat<<<std::max(1, std::min(e->sm_count * 4, (e->local_cap + 255) / 256)), 256, 0, st>>>(cp, e->d_local, e->d_counts + 1, e->local_cap);
  ++e->launches;
  // Host-side bound of the concatenated cloud: the frames' own sizes are mirrored on the host (the merged pivot cloud is
  // at most the sum of the frames merged into it), so the voxel grid, its sort and the hash build are sized for the data,
  // not for the worst-case capacity.
  long long bound = 64;
  for (int i = 0; i < W; ++i) bound += e->size_surf_stack[i] > 0 ? e->size_surf_stack[i] : e->cfg.max_frame_points;
  const int n_bound = (int)std::min<long long>(e->local_cap, bound);
  int rc = e->vg.run(e->d_local, e->d_counts + 1, n_bound, e->cfg.surf_filter_size, e->d_map, e->local_cap, e->d_counts + 2, nullptr, st, &e->launches);
  if (rc != LIO_OK) return rc;
  const float cell = std::sqrt(e->cfg.min_match_sq_dis) * (1.0f + 1.0f / 1024.0f);
  rc = e->hash.build(e->d_map, e->d_counts + 2, n_bound, cell, st, &e->launches);
  if (rc != LIO_OK) return rc;
  e->t_build = now_s() - t0;
  const double t1 = now_s();
  if (e->px.fpeers) {
    // feature exchange: this scan's features go to the other parity (a rank that is one scan ahead writes into the parity nobody
    // reads any more); only the counts of the frames this rank matches are reset - the others arrive from their owners
    set_feature_parity(e, e->px.fparity ^ 1);
    ++e->px.fepoch;
    for (int idx = pivot + 1; idx <= W; ++idx)
      if (owns_frame(e, idx)) LIO_CUDA_OK(cudaMemsetAsync(e->d_feat_counts + idx, 0, sizeof(int), st));
  } else {
    LIO_CUDA_OK(cudaMemsetAsync(e->d_feat_counts, 0, sizeof(int) * (W + 1), st));
  }
  // CalculateLaserOdom on the newest frame: rounds after convergence are no-ops on the device (done flag), but each still costs two
  // launches.  The chain is therefore enqueued in two batches: the first kOdomFirstBatch rounds ride with the scan's one
  // synchronisation (it converges in 2-3 rounds); only if the flag is still clear are the remaining rounds enqueued.
  constexpr int kOdomFirstBatch = 3;
  const bool odom = e->cfg.imu_factor && owns_frame(e, W);
  auto rounds = [&](int from, int to, cudaStream_t q) {
    const int slot = e->slot_of[W];
    return odom_rounds(e->hash, e->slot_ptr[slot], e->d_slot_n + slot, e->cfg.max_frame_points, e->d_tf + W, e->feats[W], e->cfg.keep_features,
                       e->d_odom, e->d_odom_partial, e->knn2, e->cfg.min_match_sq_dis, e->cfg.min_plane_dis, from, to, e->sm_count, q, &e->launches);
  };
  const int odom_total = odom ? e->cfg.odom_max_iterations : 0;
  const int odom_first = e->px.fpeers ? odom_total : std::min(odom_total, kOdomFirstBatch);   // exchanged features must be final
  if (odom) {
    // the chain is a string of small latency-bound launches: it runs on its own stream beside the frame-batched launch below
    // (both only read the map and its hash; the feature buffers are per frame) and joins before the read-back
    LIO_CUDA_OK(cudaEventRecord(e->ev_map, st));
    LIO_CUDA_OK(cudaStreamWaitEvent(e->ostream, e->ev_map, 0));
    LIO_CUDA_OK(cudaMemsetAsync(e->d_odom, 0, sizeof(OdomState), e->ostream));
    rc = rounds(0, odom_first, e->ostream);
    if (rc != LIO_OK) return rc;
    LIO_CUDA_OK(cudaEventRecord(e->ev_odom, e->ostream));
  }
  {
    // every owned frame except a LaserOdom-driven newest frame: ONE batched kNN + plane-fit launch
    KnnBatch b;
    b.nframes = 0;
    for (int idx = pivot + 1; idx <= W; ++idx) {
      if (!owns_frame(e, idx)) continue;
      if (idx == W && e->cfg.imu_factor) continue;
      const int slot = e->slot_of[idx];
      KnnFrame &f = b.f[b.nframes++];
      f.surf = e->slot_ptr[slot]; f.n_dev = e->d_slot_n + slot; f.tf = e->d_tf + idx;
      const int known = e->size_surf_stack[idx];
      f.n_bound = (known > 0 && idx < W) ? known : e->cfg.max_frame_points;
      f.out_p = e->feats[idx].pts; f.out_c = e->feats[idx].coef; f.out_src = e->feats[idx].src; f.out_count = e->feats[idx].count;
      f.append = 0; f.tile0 = 0;
    }
    e->knn_timed = b.nframes > 0 && e->evk0 && e->evk1;
    if (e->knn_timed) cudaEventRecord(e->evk0, st);
    rc = calculate_features_batch(e->hash, b, e->cfg.min_match_sq_dis, e->cfg.min_plane_dis, nullptr, e->knn, st, &e->launches);
    if (rc != LIO_OK) return rc;
    if (e->knn_timed) cudaEventRecord(e->evk1, st);
  }
  // one synchronisation: feature counts, map size, odom iterations
  auto readback = [&]() -> int {
    LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts, e->d_feat_counts, sizeof(int) * (W + 1), cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts + W + 1, e->d_counts, sizeof(int) * 4, cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts + W + 5, &e->d_odom->iter, sizeof(int), cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaMemcpyAsync(e->h_tf + W, e->d_tf + W, sizeof(TransformF), cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts + W + 6, e->d_slot_n + e->slot_of[W], sizeof(int), cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts + W + 7, e->vg.overflow_flag(), sizeof(int), cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts + W + 8, &e->d_odom->done, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (e->px.fpeers) LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts + W + 9, e->px.fslab + e->px.foff_flags + 128, sizeof(int), cudaMemcpyDeviceToHost, st));
    if (e->map.pm) LIO_CUDA_OK(cudaMemcpyAsync(e->h_counts + W + 13, e->lc.d_stage_n + 1, sizeof(int), cudaMemcpyDeviceToHost, st));   // /cloud_registered size
    LIO_CUDA_OK(cudaStreamSynchronize(st));
    return LIO_OK;
  };
  if (odom) LIO_CUDA_OK(cudaStreamWaitEvent(st, e->ev_odom, 0));
  if (e->px.fpeers) {
    // all-gather of the features: every owned frame is copied into the same place of every peer's slab, then the scan's epoch is
    // published in every rank's flag slot and this rank waits for the epochs of all ranks (bounded, like the S-row exchange)
    const size_t pbase = (size_t)e->px.fparity * e->px.fpar_stride;
    FeaturePeers fp;
    std::memset(&fp, 0, sizeof(fp));
    fp.npeers = e->world; fp.self = e->rank;
    FlagPeers fl;
    std::memset(&fl, 0, sizeof(fl));
    fl.npeers = e->world; fl.self = e->rank;
    for (int r = 0; r < e->world; ++r) fl.flag[r] = reinterpret_cast<unsigned *>(e->px.fpeer_base[r] + e->px.foff_flags);
    for (int idx = pivot + 1; idx <= W; ++idx) {
      if (!owns_frame(e, idx)) continue;
      for (int r = 0; r < e->world; ++r) {
        fp.pts[r] = reinterpret_cast<float4 *>(e->px.fpeer_base[r] + pbase + e->px.foff_pts[idx]);
        fp.coef[r] = reinterpret_cast<float4 *>(e->px.fpeer_base[r] + pbase + e->px.foff_coef[idx]);
        fp.count[r] = reinterpret_cast<int *>(e->px.fpeer_base[r] + pbase + e->px.foff_cnt) + idx;
      }
      const int known = e->size_surf_stack[idx];
      const int bound = (known > 0 && idx < W) ? known : e->feats[idx].cap;
      k_publish_features<<<std::max(1, std::min(e->sm_count * 2, (bound + 255) / 256)), 256, 0, st>>>(e->feats[idx].pts, e->feats[idx].coef, e->feats[idx].count,
                                                                                                   e->feats[idx].cap, fp);
      ++e->launches;
    }
    k_publish_flag<<<1, 32, 0, st>>>(fl, e->px.fepoch);
    k_xwait<<<1, 32, 0, st>>>(reinterpret_cast<const unsigned *>(e->px.fslab + e->px.foff_flags), e->world, e->px.fepoch,
                              reinterpret_cast<int *>(e->px.fslab + e->px.foff_flags + 128), nullptr);
    e->launches += 2;
  }
  if (before_sync) {   // host work that only needs the window state runs here, while the GPU is busy with the launches above
    rc = before_sync();
    if (rc != LIO_OK) return rc;
  }
  rc = readback();
  if (rc != LIO_OK) return rc;
  if (odom && odom_first < odom_total && !e->h_counts[W + 8]) {   // not converged yet (rare): the rest of the chain, one more synchronisation
    rc = rounds(odom_first, odom_total, st);
    if (rc != LIO_OK) return rc;
    rc = readback();
    if (rc != LIO_OK) return rc;
  }
  if (e->px.fpeers && (rc = xwait_report(e, Exchange::features, st)) != LIO_OK) return rc;
  if (e->h_counts[W + 6] > e->cfg.max_frame_points) {   // vg_emit stopped storing at the capacity but kept counting
    lio_set_last_error(__FILE__, __LINE__, "down-sampled scan exceeds max_frame_points");
    return LIO_ERR_CAPACITY;
  }
  if (e->h_counts[W + 7]) {   // PCL: "Leaf size is too small for the input dataset. Integer indices would overflow."
    cudaMemsetAsync(e->vg.overflow_flag(), 0, sizeof(int), st);
    lio_set_last_error(__FILE__, __LINE__, "voxel grid index overflow (leaf size too small for the cloud extent)");
    return LIO_ERR_CAPACITY;
  }
  e->size_surf_stack[W] = e->h_counts[W + 6];
  if (e->knn_timed) {  // live duration of the frame-batched k-NN + plane-fit launch (its memsets included, ~2 us)
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e->evk0, e->evk1) == cudaSuccess) {
      long long nq = 0;
      for (int idx = pivot + 1; idx <= W; ++idx)
        if (owns_frame(e, idx) && !(idx == W && e->cfg.imu_factor)) nq += e->size_surf_stack[idx];
      e->knn_ms_sum += ms; e->knn_launch_count += 1; e->knn_query_sum += nq;
    }
  }
  for (int k = 0; k <= W; ++k) e->h_feat_n[k] = e->h_counts[k];
  e->h_map_n = e->h_counts[W + 1 + 2];
  e->odom_iters = e->h_counts[W + 5];
  e->local_tf[W] = e->h_tf[W];
  for (int k = pivot + 1; k <= W; ++k)
    if (e->h_feat_n[k] > e->feats[k].cap) { lio_set_last_error(__FILE__, __LINE__, "feature buffer overflow"); return LIO_ERR_CAPACITY; }
  if (e->h_counts[W + 1 + 1] >= e->local_cap) { lio_set_last_error(__FILE__, __LINE__, "local map capacity exceeded"); return LIO_ERR_CAPACITY; }
  if (e->h_counts[W + 1 + 1] > n_bound) { lio_set_last_error(__FILE__, __LINE__, "internal: host bound of the local cloud below its device count"); return LIO_ERR_CAPACITY; }
  e->t_feat = now_s() - t1;
  return LIO_OK;
}

// ---- fused exchange over peer memory -----------------------------------------------------------------
// Waits until every rank has published `epoch` in this rank's flag array (the rows travel with the asm_ppp tails of the
// peers as P2P stores; system-scope release / acquire).  Bounded: a peer that never arrives sets *err instead of hanging.
__global__ void k_xwait(const unsigned *__restrict__ flags, int npeers, unsigned epoch, int *__restrict__ err,
                        const int *__restrict__ skip) {
  const int p = threadIdx.x;
  if (p >= npeers) return;
  if (skip && *skip) return;   // the device solver has terminated: its asm_ppp launches publish nothing any more
  const long long t0 = clock64();
  while (true) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + p) : "memory");
    if ((int)(v - epoch) >= 0) break;
    if (clock64() - t0 > 20000000000LL) { *err = 1; break; }   // ~10 s at 1.97 GHz
    __nanosleep(64);
  }
}

// ---- stage C: lidar reduction at the current parameter values ------------------------------------
struct FrameTerms { double M[6 * 18]; };

// Frame terms at the current parameters: R, t of every window frame into h_Rt (the input of asm_ppp) and, when ft is given, the
// M blocks that expand the frame's reduced rows into the normal equations.
static void write_frame_terms(lio_est *e, std::vector<FrameTerms> *ft) {
  if (ft) ft->resize(e->O + 1);
  for (int i = 1; i <= e->O; ++i) {
    double *Rt = e->h_Rt + (i - 1) * kAsmRtStride, M[6 * 18];
    ppp_frame_terms(e->para_pose[0].data(), e->para_pose[i].data(), e->para_ex, Rt, Rt + 9, ft ? (*ft)[i].M : M);
  }
}

// The frames and tile plan of the fused lidar reduction.  A frame counts when this rank holds its features: every frame after a
// feature exchange, its own frames otherwise.  Fails before anything is enqueued when a sharded context has no exchange.
static int lidar_setup(const lio_est *e, Exchange x, AsmParams &ap, long long &nfeat) {
  if (x == Exchange::missing) {
    lio_set_last_error(__FILE__, __LINE__, "sharded context without an exchange: call lio_est_set_peers or pass an allreduce callback");
    return LIO_ERR_INVALID;
  }
  const int O = e->O, pivot = e->W - O;
  std::memset(&ap, 0, sizeof(ap));
  ap.nframes = O;
  nfeat = 0;
  for (int i = 1; i <= O; ++i) {
    AsmFrame &f = ap.f[i - 1];
    const FeatureOut &fo = e->feats[pivot + i];
    f.pts = fo.pts; f.coef = fo.coef;
    f.n = (e->cfg.point_distance_factor && (x == Exchange::features || owns_frame(e, pivot + i))) ? e->h_feat_n[pivot + i] : 0;
    nfeat += f.n;
  }
  asm_plan(ap, e->sm_count);
  return LIO_OK;
}

// Rows exchange, before each asm_ppp launch: a new epoch, and the kernel's tail scatters the owned rows into the epoch's parity of
// every rank's buffer and publishes the epoch.  Returns where all rows of the evaluation land on this rank.
static const double *exchange_targets(lio_est *e, Exchange x, AsmParams &ap) {
  if (x != Exchange::rows) return e->asmw.out;
  const int pivot = e->W - e->O;
  ap.npeers = e->px.npeers; ap.self = e->rank; ap.epoch = ++e->px.xepoch;
  ap.owned_mask = 0;
  for (int i = 1; i <= e->O; ++i) if (owns_frame(e, pivot + i)) ap.owned_mask |= 1u << (i - 1);
  const size_t par = (size_t)(ap.epoch & 1u) * kXRowBytes;
  for (int r = 0; r < e->px.npeers; ++r) {
    ap.peer_out[r] = reinterpret_cast<double *>(e->px.peer_base[r] + par);
    ap.peer_flag[r] = reinterpret_cast<unsigned *>(e->px.peer_base[r] + kXFlagOff);
  }
  return reinterpret_cast<const double *>(e->px.xbuf + par);
}

// After each asm_ppp launch: the rows exchange waits on q for every rank's epoch (skipped on the device once `*skip` is set), the
// callback exchange sums the partial rows of all ranks.
static int exchange_rows(lio_est *e, Exchange x, const AsmParams &ap, cudaStream_t q, const int *skip) {
  if (x == Exchange::rows) {
    k_xwait<<<1, 32, 0, q>>>(reinterpret_cast<const unsigned *>(e->px.xbuf + kXFlagOff), e->px.npeers, ap.epoch,
                             reinterpret_cast<int *>(e->px.xbuf + kXErrOff), skip);
    ++e->launches;
  } else if (x == Exchange::callback && e->allreduce(e->allreduce_user, e->asmw.out, e->O * kAsmStride) != 0) {
    lio_set_last_error(__FILE__, __LINE__, "allreduce callback failed");
    return LIO_ERR_CUDA;
  }
  return LIO_OK;
}

// One completed asm_ppp launch into lio_est_kernel_profile's totals.  A failed timing query is dropped and cleared, so that it does
// not surface as the next launch's error.
static void asm_time_add(lio_est *e, cudaEvent_t a, cudaEvent_t b, long long nfeat) {
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, a, b) == cudaSuccess) { e->asm_ms_sum += ms; e->asm_launch_count += 1; e->asm_feat_sum += nfeat; }
  else (void)cudaGetLastError();
}

// Enqueues the fused lidar reduction at the current parameters (no host synchronisation); eval_lidar_wait() completes it.
static int eval_lidar_launch(lio_est *e, std::vector<FrameTerms> &ft) {
  write_frame_terms(e, &ft);
  if (e->S_valid) return LIO_OK;
  const Exchange x = exchange_of(e);
  AsmParams ap;
  long long nfeat;
  int rc = lidar_setup(e, x, ap, nfeat);
  if (rc != LIO_OK) return rc;
  LIO_CUDA_OK(cudaMemcpyAsync(e->d_Rt, e->h_Rt, sizeof(double) * e->O * kAsmRtStride, cudaMemcpyHostToDevice, e->stream));
  const double *result = exchange_targets(e, x, ap);
  if (e->ev0) cudaEventRecord(e->ev0, e->stream);
  rc = asm_launch(ap, e->d_Rt, e->asmw, e->stream, &e->launches);
  if (rc != LIO_OK) return rc;
  if (e->ev1) cudaEventRecord(e->ev1, e->stream);
  rc = exchange_rows(e, x, ap, e->stream, nullptr);
  if (rc != LIO_OK) return rc;
  if (x == Exchange::rows) LIO_CUDA_OK(cudaMemcpyAsync(e->h_xerr, e->px.xbuf + kXErrOff, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  LIO_CUDA_OK(cudaMemcpyAsync(e->h_S, result, sizeof(double) * e->O * kAsmStride, cudaMemcpyDeviceToHost, e->stream));
  e->S_pending = true;
  e->S_pending_feats = nfeat;
  return LIO_OK;
}

static int eval_lidar_wait(lio_est *e) {
  if (!e->S_pending) return LIO_OK;
  const double t0 = now_s();
  LIO_CUDA_OK(cudaStreamSynchronize(e->stream));
  e->t_lin_wait += now_s() - t0;
  e->S_pending = false;
  const int rc = xwait_report(e, Exchange::rows, e->stream);
  if (rc != LIO_OK) return rc;
  asm_time_add(e, e->ev0, e->ev1, e->S_pending_feats);
  e->S_valid = true;
  return LIO_OK;
}

static int eval_lidar(lio_est *e, std::vector<FrameTerms> &ft) {
  int rc = eval_lidar_launch(e, ft);
  return rc != LIO_OK ? rc : eval_lidar_wait(e);
}

// tangent layout: [pose_k(6) sb_k(9)] k=0..O, then ex(6)
static inline int off_pose(int k) { return 15 * k; }

// adds M^T S M into H/g over (pose_0, pose_i, ex) column offsets o0, oi, oe (oe < 0: extrinsic not a variable)
static void add_lidar_block(const double *S /*kAsmStride*/, const double *M /*6x18*/, Mat *H, Vec *g, int o0, int oi, int oe) {
  double Sg[6][6], Sr[6];
  {
    int k = 0;
    for (int a = 0; a < 7; ++a) for (int b = a; b < 7; ++b) { double v = S[k++]; if (b < 6) { Sg[a][b] = v; Sg[b][a] = v; } else if (a < 6) Sr[a] = v; }
  }
  double SM[6][18];
  for (int a = 0; a < 6; ++a) for (int c = 0; c < 18; ++c) { double s = 0; for (int b = 0; b < 6; ++b) s += Sg[a][b] * M[b * 18 + c]; SM[a][c] = s; }
  const int offs[3] = {o0, oi, oe};
  for (int bi = 0; bi < 3; ++bi) {
    if (offs[bi] < 0) continue;
    for (int a = 0; a < 6; ++a) {
      const int ca = bi * 6 + a;
      double gs = 0;
      for (int k = 0; k < 6; ++k) gs += M[k * 18 + ca] * Sr[k];
      (*g)[offs[bi] + a] += gs;
      if (!H) continue;
      for (int bj = 0; bj < 3; ++bj) {
        if (offs[bj] < 0) continue;
        for (int b = 0; b < 6; ++b) {
          const int cb = bj * 6 + b;
          double s = 0;
          for (int k = 0; k < 6; ++k) s += M[k * 18 + ca] * SM[k][cb];
          (*H)(offs[bi] + a, offs[bj] + b) += s;
        }
      }
    }
  }
}

static void prior_dx(const lio_est *e, const MargPrior &pr, Vec &dx) {  // MarginalizationFactor::Evaluate :347-372
  const int O = e->O;
  dx.assign(pr.n, 0.0);
  auto pose_dx = [&](const double *x, const double *x0, double *out) {
    for (int k = 0; k < 3; ++k) out[k] = x[k] - x0[k];
    Q q0(x0[6], x0[3], x0[4], x0[5]), q(x[6], x[3], x[4], x[5]);
    Q dq = inverse(q0) * q;
    Q dn = normalized(dq);
    double s = dq.w < 0 ? -2.0 : 2.0;
    out[3] = s * dn.x; out[4] = s * dn.y; out[5] = s * dn.z;
  };
  for (int k = 0; k < O; ++k) {
    pose_dx(e->para_pose[k].data(), &pr.x0_pose[7 * k], &dx[15 * k]);
    for (int a = 0; a < 9; ++a) dx[15 * k + 6 + a] = e->para_sb[k][a] - pr.x0_sb[9 * k + a];
  }
  pose_dx(e->para_ex, pr.x0_ex, &dx[15 * O]);
}

// Drains the ImuFactor pool of the current linearisation (called concurrently by the caller thread and the helper).
static void imu_pool_run(lio_est *e, int O, int pivot) {
  int i;
  while ((i = e->imu_next.fetch_add(1)) < O) {
    lio_est::ImuBlockStore &b = e->imu_blocks_store[i];
    Preintegration &pim = *e->pre[pivot + i + 1];
    b.used = !(pim.sum_dt > 10.0);
    if (b.used) {
      double r[15], J[15][30];
      imu_factor_evaluate30(pim, e->para_pose[i].data(), e->para_sb[i].data(), e->para_pose[i + 1].data(), e->para_sb[i + 1].data(), r, J);
      JtJ_dense(&J[0][0], r, 15, 30, b.JtJ, b.Jtr);
      double sq = 0;
      for (int k = 0; k < 15; ++k) sq += r[k] * r[k];
      b.cost = 0.5 * sq;
    }
    e->imu_done.fetch_add(1);
  }
}

// Full linearisation at the current parameter values.  n_t = tangent dim (ex block present iff !ex_constant).  Returns the lidar
// evaluation's error, or LIO_ERR_NUMERIC for a non-finite cost.
int linearize(lio_est *e, Mat &H, Vec &g, double &cost, double *c_pim, double *c_ppp, double *c_marg) {
  const int O = e->O, pivot = e->W - O;
  const bool ex_free = !e->ex_constant;
  const int n = 15 * (O + 1) + (ex_free ? 6 : 0);
  const int oe = ex_free ? 15 * (O + 1) : -1;
  std::vector<FrameTerms> ft;
  int rc = eval_lidar_launch(e, ft);  // the device reduces the lidar factors while the host does the rest
  if (rc != LIO_OK) return rc;
  // H starts as the prior's information matrix scattered into the tangent layout (constant over a solve: cached), or zero
  const bool use_prior = e->cfg.marginalization_factor && e->prior.valid;
  if (use_prior) {
    if (!e->hp_exp_valid || e->hp_exp.r != n) {
      const MargPrior &pr = e->prior;
      e->hp_exp = Mat(n, n);
      const int nw = 15 * O;  // window part maps one to one, the extrinsic block moves behind pose_O / sb_O
      for (int a = 0; a < pr.n; ++a) {
        const int ta = a < nw ? a : (ex_free ? 15 * (O + 1) + (a - nw) : -1);
        if (ta < 0) continue;
        const double *row = &pr.Hp.d[(size_t)a * pr.n];
        double *hrow = &e->hp_exp.d[(size_t)ta * n];
        for (int b = 0; b < nw; ++b) hrow[b] = row[b];
        if (ex_free) for (int b = nw; b < pr.n; ++b) hrow[15 * (O + 1) + (b - nw)] = row[b];
      }
      e->hp_exp_valid = true;
    }
    if (H.r != n) H = Mat(n, n);
    std::memcpy(H.d.data(), e->hp_exp.d.data(), sizeof(double) * (size_t)n * n);
  } else {
    if (H.r != n) H = Mat(n, n); else H.zero();
  }
  g.assign(n, 0.0);
  const double th0 = now_s();
  double cp = 0, ci = 0, cm = 0;
  // ImuFactors: factors [0, i_split) go directly into H on this thread; factors [i_split, O) form a pool that the context's
  // helper thread and (after its own share and the prior) this thread drain together into private 30x30 blocks, which
  // are added in index order afterwards - the result does not depend on who evaluated which block, and a helper that
  // is late or descheduled costs nothing but its share.
  const int i_split = (e->cfg.imu_factor && O >= 4) ? O / 2 : O;
  auto imu_eval = [&](int i, double *r, double (*J)[30]) {
    Preintegration &pim = *e->pre[pivot + i + 1];
    if (pim.sum_dt > 10.0) return false;
    imu_factor_evaluate30(pim, e->para_pose[i].data(), e->para_sb[i].data(), e->para_pose[i + 1].data(), e->para_sb[i + 1].data(), r, J);
    return true;
  };
  if (e->cfg.imu_factor && i_split < O) {
    e->worker.wait();  // the previous pool job has retired before the counters are reset
    e->imu_next.store(i_split);
    e->imu_done.store(0);
    e->worker.submit([e, O, pivot]() { imu_pool_run(e, O, pivot); });
  }
  if (e->cfg.imu_factor) {
    for (int i = 0; i < i_split; ++i) {
      double r[15], J[15][30];
      if (!imu_eval(i, r, J)) continue;
      int cmap[30];
      for (int a = 0; a < 30; ++a) cmap[a] = 15 * i + a;  // pose_i, sb_i, pose_j, sb_j are contiguous in the tangent layout
      add_JtJ_mapped(&J[0][0], r, 15, 30, cmap, H, g);
      double sq = 0;
      for (int k = 0; k < 15; ++k) sq += r[k] * r[k];
      ci += 0.5 * sq;
    }
  }
  if (e->cfg.marginalization_factor && e->prior.valid) {
    const MargPrior &pr = e->prior;
    Vec dx;
    prior_dx(e, pr, dx);
    Vec Hdx;
    matvec(pr.Hp, dx, Hdx);
    cm = 0.5 * (pr.c0 + 2.0 * vdot(pr.bp, dx) + vdot(dx, Hdx));
    auto tmap = [&](int pi) { return pi < 15 * O ? pi : (ex_free ? 15 * (O + 1) + (pi - 15 * O) : -1); };
    for (int a = 0; a < pr.n; ++a) {
      const int ta = tmap(a);
      if (ta >= 0) g[ta] += Hdx[a] + pr.bp[a];
    }
  }
  if (e->cfg.imu_factor && i_split < O) {
    imu_pool_run(e, O, pivot);
    while (e->imu_done.load() < O - i_split) Worker::relax();  // at most one block still in flight on the helper
    const lio_est::ImuBlockStore *blk = e->imu_blocks_store;
    for (int i = i_split; i < O; ++i) {
      const lio_est::ImuBlockStore &b = blk[i];
      if (!b.used) continue;
      for (int a = 0; a < 30; ++a) {
        double *hrow = &H.d[(size_t)(15 * i + a) * n + 15 * i];
        const double *src = b.JtJ + 30 * a;
        for (int c = 0; c < 30; ++c) hrow[c] += src[c];
        g[15 * i + a] += b.Jtr[a];
      }
      ci += b.cost;
    }
  }
  double cprior = 0;
  if (e->cfg.prior_factor && ex_free) {  // constant extrinsic: the block is dropped from the reduced program
    const Tw tt = tlb_double(e);
    double r[6], J[6][6];
    prior_factor_evaluate(tt.pos, tt.rot, e->para_ex, r, J);
    for (int a = 0; a < 6; ++a) {
      double gs = 0;
      for (int k = 0; k < 6; ++k) gs += J[k][a] * r[k];
      g[oe + a] += gs;
      for (int b = 0; b < 6; ++b) { double s = 0; for (int k = 0; k < 6; ++k) s += J[k][a] * J[k][b]; H(oe + a, oe + b) += s; }
    }
    for (int k = 0; k < 6; ++k) cprior += 0.5 * r[k] * r[k];
  }
  e->t_lin_host += now_s() - th0;
  rc = eval_lidar_wait(e);
  if (rc != LIO_OK) return rc;
  if (e->cfg.point_distance_factor) {
    const double tl0 = now_s();
    for (int i = 1; i <= O; ++i) {
      const double *S = e->h_S + (i - 1) * kAsmStride;
      cp += 0.5 * S[28];
      add_lidar_block(S, ft[i].M, &H, &g, off_pose(0), off_pose(i), oe);
    }
    e->t_lin_lidar += now_s() - tl0;
  }
  cost = cp + ci + cm + cprior;
  if (c_pim) *c_pim = ci;
  if (c_ppp) *c_ppp = cp;
  if (c_marg) *c_marg = cm;
  return std::isfinite(cost) ? LIO_OK : LIO_ERR_NUMERIC;
}

static MargPrior marg_algebra(Mat A, Vec b, int O, std::vector<double> x0_pose, std::vector<double> x0_sb, const double *x0_ex);
// ---- marginalisation (MarginalizationInfo::PreMarginalize / Marginalize, MarginalizationFactor.cc:132-311)
int marginalize(lio_est *e) {
  const int O = e->O, pivot = e->W - O;
  const int m = 15, nr = 15 * O + 6, pos = m + nr;
  // layout: [pose_0 (6), sb_0 (9) | pose_1, sb_1, ..., pose_O, sb_O, ex]
  Mat A(pos, pos);
  Vec b(pos, 0.0);
  auto idx_pose = [&](int k) { return k == 0 ? 0 : m + 15 * (k - 1); };
  auto idx_sb = [&](int k) { return k == 0 ? 6 : m + 15 * (k - 1) + 6; };
  const int idx_ex = m + 15 * O;
  if (e->prior.valid) {  // previous prior re-wrapped with drop_set {pose_0, sb_0}
    const MargPrior &pr = e->prior;
    Vec dx;
    prior_dx(e, pr, dx);
    Vec Hdx;
    matvec(pr.Hp, dx, Hdx);
    auto map = [&](int pi) {  // prior canonical index -> A index
      if (pi >= 15 * O) return idx_ex + (pi - 15 * O);
      int k = pi / 15, a = pi % 15;
      return (a < 6 ? idx_pose(k) + a : idx_sb(k) + (a - 6));
    };
    for (int a = 0; a < pr.n; ++a) {
      const int ia = map(a);
      b[ia] += Hdx[a] + pr.bp[a];
      for (int c = 0; c < pr.n; ++c) A(ia, map(c)) += pr.Hp(a, c);
    }
  }
  if (e->cfg.imu_factor && e->pre[pivot + 1]->sum_dt < 10.0) {
    double r[15], J[15][30];
    imu_factor_evaluate30(*e->pre[pivot + 1], e->para_pose[0].data(), e->para_sb[0].data(), e->para_pose[1].data(), e->para_sb[1].data(), r, J);
    int col[30];
    for (int c = 0; c < 6; ++c) { col[c] = idx_pose(0) + c; col[15 + c] = idx_pose(1) + c; }
    for (int c = 0; c < 9; ++c) { col[6 + c] = idx_sb(0) + c; col[21 + c] = idx_sb(1) + c; }
    add_JtJ_mapped(&J[0][0], r, 15, 30, col, A, b);
  }
  if (e->cfg.point_distance_factor) {
    std::vector<FrameTerms> ft;
    int rc = eval_lidar(e, ft);
    if (rc != LIO_OK) return rc;
    for (int i = 1; i <= O; ++i) add_lidar_block(e->h_S + (i - 1) * kAsmStride, ft[i].M, &A, &b, idx_pose(0), idx_pose(i), idx_ex);
  }
  MargJob &job = e->mjob;
  job.O = O;
  job.A.r = A.r; job.A.c = A.c; job.A.d.swap(A.d);
  job.b.swap(b);
  job.x0_pose.resize(7 * O); job.x0_sb.resize(9 * O);
  for (int k = 1; k <= O; ++k) {  // addr_shift: block i -> i-1 in the next window
    std::memcpy(&job.x0_pose[7 * (k - 1)], e->para_pose[k].data(), 7 * sizeof(double));
    std::memcpy(&job.x0_sb[9 * (k - 1)], e->para_sb[k].data(), 9 * sizeof(double));
  }
  std::memcpy(job.x0_ex, e->para_ex, sizeof(job.x0_ex));
  job.stashed = true;
  if (!e->cfg.overlap_marginalization) {  // the reference's order: finish the algebra before returning from this scan
    job.stashed = false;
    e->prior = marg_algebra(std::move(job.A), std::move(job.b), job.O, std::move(job.x0_pose), std::move(job.x0_sb), job.x0_ex);
    e->hp_exp_valid = false;
  }
  return LIO_OK;
}

// Schur complement + eigen square-root form (MarginalizationInfo::Marginalize, MarginalizationFactor.cc:206-311) of a
// stashed system; layout [pose_0 (6), sb_0 (9) | pose_1, sb_1, ..., pose_O, sb_O, ex].  Pure function: worker-thread safe.
static MargPrior marg_algebra(Mat A, Vec b, int O, std::vector<double> x0_pose, std::vector<double> x0_sb, const double *x0_ex) {
  const int m = 15, nr = 15 * O + 6;
  // Schur complement with the eigen pseudo-inverse (eps = 1e-8)
  const double eps = 1e-8;
  Mat Amm(m, m);
  for (int r = 0; r < m; ++r) for (int c = 0; c < m; ++c) Amm(r, c) = 0.5 * (A(r, c) + A(c, r));
  Vec ev;
  Mat evec;
  sym_eigen(Amm, ev, evec);
  Mat Amm_inv(m, m);
  for (int r = 0; r < m; ++r)
    for (int c = 0; c < m; ++c) { double s = 0; for (int k = 0; k < m; ++k) s += evec(r, k) * (ev[k] > eps ? 1.0 / ev[k] : 0.0) * evec(c, k); Amm_inv(r, c) = s; }
  Mat Tm(nr, m);  // Arm * Amm_inv
  for (int r = 0; r < nr; ++r) for (int c = 0; c < m; ++c) { double s = 0; for (int k = 0; k < m; ++k) s += A(m + r, k) * Amm_inv(k, c); Tm(r, c) = s; }
  Mat A2(nr, nr);
  Vec b2(nr);
  for (int r = 0; r < nr; ++r) {
    for (int c = 0; c < nr; ++c) { double s = 0; for (int k = 0; k < m; ++k) s += Tm(r, k) * A(k, m + c); A2(r, c) = A(m + r, m + c) - s; }
    double s = 0;
    for (int k = 0; k < m; ++k) s += Tm(r, k) * b[k];
    b2[r] = b[m + r] - s;
  }
  // Eigen square root of the Schur complement (MarginalizationFactor.cc:276-311).  Only the factors that touch the dropped
  // blocks enter A, so the speed-bias blocks sb_2 .. sb_O (and pose_O's sb) have exactly-zero rows and columns in A2: its
  // spectrum is that of the non-zero principal sub-matrix plus zeros, which the eps test drops.  The decomposition is
  // therefore taken on the compressed matrix (75 of 156 rows for O = 10: ~9x fewer flops) and scattered back; the
  // reference decomposes the padded matrix and arrives at the same kept eigenpairs.
  std::vector<int> nz;
  for (int r = 0; r < nr; ++r) {
    bool any = b2[r] != 0.0;
    const double *row = &A2.d[(size_t)r * nr];
    for (int c = 0; c < nr && !any; ++c) any = row[c] != 0.0 || A2.d[(size_t)c * nr + r] != 0.0;
    if (any) nz.push_back(r);
  }
  const int nc = (int)nz.size();
  Mat Ac(nc, nc);
  Vec bc(nc);
  for (int r = 0; r < nc; ++r) {
    bc[r] = b2[nz[r]];
    for (int c = 0; c < nc; ++c) Ac(r, c) = A2(nz[r], nz[c]);
  }
  Vec ev2;
  Mat V2;
  if (nc > 0) sym_eigen(Ac, ev2, V2, 1);
  MargPrior np;
  np.valid = true;
  np.n = nr;
  np.Hp = Mat(nr, nr);
  np.bp.assign(nr, 0.0);
  np.c0 = 0;
  // Hp = V S V^T, bp = V_kept V_kept^T b, c0 = sum (v^T b)^2 / lambda over kept eigenpairs
  std::vector<int> kept;
  for (int k = 0; k < nc; ++k) if (ev2[k] > eps) kept.push_back(k);
  Vec vb(nc, 0.0);
  for (int k : kept) { double s = 0; for (int r = 0; r < nc; ++r) s += V2(r, k) * bc[r]; vb[k] = s; np.c0 += s * s / ev2[k]; }
  Mat Hc(nc, nc);
  if (nc > 0) weighted_gram(V2, ev2, kept, Hc);
  for (int r = 0; r < nc; ++r) {
    double sb = 0;
    for (int k : kept) sb += V2(r, k) * vb[k];
    np.bp[nz[r]] = sb;
    for (int c = 0; c < nc; ++c) np.Hp(nz[r], nz[c]) = Hc(r, c);
  }
  np.x0_pose = std::move(x0_pose);
  np.x0_sb = std::move(x0_sb);
  std::memcpy(np.x0_ex, x0_ex, sizeof(np.x0_ex));
  return np;
}

void marg_start(lio_est *e) {
  MargJob &job = e->mjob;
  if (!job.stashed || job.running) return;
  job.stashed = false;
  job.running = true;
  e->worker.submit([&job]() {
    job.result = marg_algebra(std::move(job.A), std::move(job.b), job.O, std::move(job.x0_pose), std::move(job.x0_sb), job.x0_ex);
  });
}

// Makes e->prior current: runs a stashed job (inline start) and waits for a running one.
void prior_join(lio_est *e) {
  MargJob &job = e->mjob;
  if (job.stashed) marg_start(e);
  if (!job.running) return;
  const double t0 = now_s();
  e->worker.wait();
  e->prior = std::move(job.result);
  e->hp_exp_valid = false;
  job.running = false;
  e->t_marg_wait += now_s() - t0;
}

int solve_host(lio_est *e, int max_it) {
  const int O = e->O;
  const double t0 = now_s();
  // residuals before optimisation + gates (:1924-1985)
  Mat H;
  Vec g;
  double cost;
  int rc = linearize(e, H, g, cost, &e->cost_pim, &e->cost_ppp, &e->cost_marg);
  if (rc == LIO_ERR_NUMERIC) lio_set_last_error(__FILE__, __LINE__, "non-finite cost at the initial point");
  if (rc != LIO_OK) return rc;
  if (e->cfg.imu_factor) e->turn_off = e->cost_pim > 1e3;
  const bool ex_constant_before = e->ex_constant, prior_before = e->prior.valid;
  {
    const double ratio = e->cost_marg / (e->cost_ppp + e->cost_pim);
    if (!e->convergence_flag && !e->turn_off && ratio <= 2 && ratio != 0) e->convergence_flag = true;
    if (!e->convergence_flag) {
      e->ex_constant = true;
      e->prior.valid = false;
    }
  }
  DoglegProblem P;
  const bool ex_free = !e->ex_constant;
  P.n = 15 * (O + 1) + (ex_free ? 6 : 0);
  bool first = true;
  // the gate evaluation above is the solver's first linearisation when the gates left the problem structure unchanged
  bool reuse_gate = (ex_constant_before == e->ex_constant && prior_before == e->prior.valid);
  // A non-finite cost is a rejected step.  Any other failed evaluation ends the solve with its error: the remaining iterations of
  // dogleg_solve evaluate nothing.
  int eval_rc = LIO_OK;
  P.linearize = [&](Mat &Hh, Vec &gg, double &c) {
    if (eval_rc != LIO_OK) return false;
    int r2 = LIO_OK;
    if (reuse_gate && first) { Hh.d.swap(H.d); Hh.r = H.r; Hh.c = H.c; gg.swap(g); c = cost; }
    else r2 = linearize(e, Hh, gg, c, nullptr, nullptr, nullptr);
    if (r2 != LIO_OK && r2 != LIO_ERR_NUMERIC) eval_rc = r2;
    if (r2 == LIO_OK && first) { e->H0 = Hh; e->g0 = gg; e->cost0 = c; e->have_H0 = true; first = false; }
    return r2 == LIO_OK;
  };
  P.get_state = [&](Vec &x) {
    x.clear();
    for (int k = 0; k <= O; ++k) { x.insert(x.end(), e->para_pose[k].begin(), e->para_pose[k].end()); x.insert(x.end(), e->para_sb[k].begin(), e->para_sb[k].end()); }
    if (ex_free) x.insert(x.end(), e->para_ex, e->para_ex + 7);
  };
  P.set_state = [&](const Vec &x) {
    for (int k = 0; k <= O; ++k) { std::memcpy(e->para_pose[k].data(), &x[16 * k], 7 * sizeof(double)); std::memcpy(e->para_sb[k].data(), &x[16 * k + 7], 9 * sizeof(double)); }
    if (ex_free) std::memcpy(e->para_ex, &x[16 * (O + 1)], 7 * sizeof(double));
    e->S_valid = false;
  };
  P.plus = [&](const Vec &x, const Vec &d, Vec &out) {
    out = x;
    for (int k = 0; k <= O; ++k) {
      pose_plus(&x[16 * k], &d[15 * k], &out[16 * k]);
      for (int a = 0; a < 9; ++a) out[16 * k + 7 + a] = x[16 * k + 7 + a] + d[15 * k + 6 + a];
    }
    if (ex_free) pose_plus(&x[16 * (O + 1)], &d[15 * (O + 1)], &out[16 * (O + 1)]);
  };
  DoglegOptions opt;
  opt.max_num_iterations = max_it;
  dogleg_solve(opt, P, &e->summary);
  if (eval_rc != LIO_OK) return eval_rc;
  if (e->summary.termination == 2 && !std::isfinite(e->summary.final_cost)) { lio_set_last_error(__FILE__, __LINE__, "solver breakdown"); return LIO_ERR_NUMERIC; }
  e->t_solve = now_s() - t0;
  return LIO_OK;
}

// ---- SolveOptimization with the device-resident dogleg loop --------------------------------------
// The solve from the current para_* blocks on the device.  assemble_only: one evaluation without gates or steps, nothing of
// the estimator's own state is touched (lio_est_assemble); the first linearisation stays readable in ds.H0 / ds.g0.
// Everything of a device solve that does not depend on this scan's features: the solver state (parameters, prior, pre-integrations)
// and the frame terms of the initial point, uploaded asynchronously.  process_scan calls it while the GPU is still busy with the front
// end (before the scan's one synchronisation); solve_dev repeats it only when the parameters were replaced since.
int solve_dev_prepare(lio_est *e, int max_it, bool assemble_only) {
  const int O = e->O, pivot = e->W - O;
  cudaStream_t st = e->stream;
  DevSolveState &S = *e->ds.h_st;
  S.sc.O = O; S.sc.n = 15 * (O + 1) + 6; S.sc.max_it = assemble_only ? 0 : max_it;
  S.sc.skip_gates = assemble_only ? 1 : 0; S.sc.pad_ = 0;
  S.sc.imu_factor = e->cfg.imu_factor; S.sc.point_distance_factor = e->cfg.point_distance_factor;
  S.sc.prior_factor = e->cfg.prior_factor; S.sc.marginalization_factor = e->cfg.marginalization_factor;
  S.sc.ex_free = e->ex_constant ? 0 : 1;
  S.sc.prior_valid = (e->cfg.marginalization_factor && e->prior.valid) ? 1 : 0;
  S.sc.convergence_flag = e->convergence_flag ? 1 : 0;
  S.sc.turn_off = 1; S.sc.done = 0; S.sc.iteration = 0; S.sc.successful = 0; S.sc.evaluations = 0; S.sc.termination = 0; S.sc.reuse = 0; S.sc.invalid = 0;
  for (int k = 0; k <= O; ++k) { std::memcpy(S.x + 16 * k, e->para_pose[k].data(), 7 * sizeof(double)); std::memcpy(S.x + 16 * k + 7, e->para_sb[k].data(), 9 * sizeof(double)); }
  std::memcpy(S.x + 16 * (O + 1), e->para_ex, 7 * sizeof(double));
  {
    const Tw tt = tlb_double(e);
    S.sc.ex0_pos[0] = tt.pos.x; S.sc.ex0_pos[1] = tt.pos.y; S.sc.ex0_pos[2] = tt.pos.z;
    S.sc.ex0_quat[0] = tt.rot.x; S.sc.ex0_quat[1] = tt.rot.y; S.sc.ex0_quat[2] = tt.rot.z; S.sc.ex0_quat[3] = tt.rot.w;
  }
  for (int i = 0; i < O; ++i) {
    Preintegration &pim = *e->pre[pivot + i + 1];
    S.pim_valid[i] = pim.sum_dt > 10.0 ? 0 : 1;
    S.pim[i] = pim.data();
  }
  if (S.sc.prior_valid) {
    const MargPrior &pr = e->prior;
    std::memcpy(S.bp, pr.bp.data(), sizeof(double) * pr.n);
    S.c0 = pr.c0;
    std::memcpy(S.x0_pose, pr.x0_pose.data(), sizeof(double) * 7 * O);
    std::memcpy(S.x0_sb, pr.x0_sb.data(), sizeof(double) * 9 * O);
    std::memcpy(S.x0_ex, pr.x0_ex, sizeof(double) * 7);
    if (!e->prior_uploaded) {
      LIO_CUDA_OK(cudaMemcpyAsync(e->ds.Hp, pr.Hp.d.data(), sizeof(double) * pr.n * pr.n, cudaMemcpyHostToDevice, st));
      e->prior_uploaded = true;
    }
  }
  LIO_CUDA_OK(cudaMemcpyAsync(e->ds.st, &S, sizeof(DevSolveState), cudaMemcpyHostToDevice, st));
  write_frame_terms(e, nullptr);   // frame terms of the initial point; the solver writes the candidates' terms itself
  LIO_CUDA_OK(cudaMemcpyAsync(e->d_Rt, e->h_Rt, sizeof(double) * O * kAsmRtStride, cudaMemcpyHostToDevice, st));
  e->ds_prepared = true; e->ds_prepared_it = max_it; e->ds_prepared_asm = assemble_only;
  return LIO_OK;
}

int solve_dev(lio_est *e, int max_it, bool assemble_only) {
  const int O = e->O;
  cudaStream_t st = e->stream;
  int rc = LIO_OK;
  const double t0 = now_s();
  if (!(e->ds_prepared && e->ds_prepared_it == max_it && e->ds_prepared_asm == assemble_only)) {
    rc = solve_dev_prepare(e, max_it, assemble_only);
    if (rc != LIO_OK) return rc;
  }
  e->ds_prepared = false;
  DevSolveState &S = *e->ds.h_st;
  const Exchange x = exchange_of(e);
  AsmParams ap;
  long long nfeat;
  rc = lidar_setup(e, x, ap, nfeat);
  if (rc != LIO_OK) return rc;
  ap.skip_flag = &e->ds.st->sc.done;
  ap.stamps = &e->ds.st->dbg[12][0];   // rows 12..14 of the trace: asm_ppp entry / exit stamps per evaluation
  const bool sharded = x == Exchange::rows || x == Exchange::callback;
  const bool use_graph = e->gstream && !sharded && !assemble_only && max_it == e->cfg.max_num_iterations;
  const int nevals = (assemble_only ? 0 : max_it) + 1;
  auto enqueue = [&](cudaStream_t q, bool capturing) -> int {
    // timing events inside a capture must be EXTERNAL event nodes to stay usable with cudaEventElapsedTime
    const unsigned evflag = capturing ? cudaEventRecordExternal : cudaEventRecordDefault;
    for (int ev = 0; ev < nevals; ++ev) {
      int r2 = dev_solver_factors(e->ds, ev, q, &e->launches);   // ImuFactors / prior / M_i on the second stream, beside asm_ppp
      if (r2 != LIO_OK) return r2;
      const double *result = exchange_targets(e, x, ap);
      // asm_ppp is timed on the first evaluation only: inside the captured graph every event record is a node on the critical path
      // between two k_step launches (measured: the launch behind it starts ~4 us later)
      const bool timed = ev == 0 || (!capturing && !sharded);   // sharded runs: first evaluation only, like the graph
      if (timed) cudaEventRecordWithFlags(e->evp[2 * ev], q, evflag);
      r2 = asm_launch(ap, e->d_Rt, e->asmw, q, &e->launches);
      if (r2 != LIO_OK) return r2;
      if (timed) cudaEventRecordWithFlags(e->evp[2 * ev + 1], q, evflag);
      r2 = exchange_rows(e, x, ap, q, &e->ds.st->sc.done);
      if (r2 != LIO_OK) return r2;
      r2 = dev_solver_step(e->ds, result, e->d_Rt, ev, q, &e->launches);
      if (r2 != LIO_OK) return r2;
    }
    return LIO_OK;
  };
  if (use_graph) {
    // One graph per solve: the launch sequence (and the fork / join with the factor stream) is captured the first time and
    // replayed afterwards; only the asm_ppp nodes are re-parameterised with this scan's feature counts and tile plan.
    cudaStream_t gs = e->gstream;
    LIO_CUDA_OK(cudaEventRecord(e->ev_gin, st));
    LIO_CUDA_OK(cudaStreamWaitEvent(gs, e->ev_gin, 0));
    if (!e->sexec) {
      asm_prepare();
      const int l0 = e->launches;
      LIO_CUDA_OK(cudaStreamBeginCapture(gs, cudaStreamCaptureModeThreadLocal));
      rc = enqueue(gs, true);
      Graph g;
      const cudaError_t ce = end_capture(gs, g);
      if (rc != LIO_OK) return rc;
      if (ce != cudaSuccess || !g) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(ce)); return LIO_ERR_CUDA; }
      e->sgraph = std::move(g);
      e->graph_launches = e->launches - l0;
      e->launches = l0;
      if (!instantiate(e->sexec, e->sgraph)) return LIO_ERR_CUDA;
      size_t nn = 0;
      LIO_CUDA_OK(cudaGraphGetNodes(e->sgraph, nullptr, &nn));
      std::vector<cudaGraphNode_t> nodes(nn);
      LIO_CUDA_OK(cudaGraphGetNodes(e->sgraph, nodes.data(), &nn));
      e->asm_nodes.clear();
      for (cudaGraphNode_t nd : nodes) if (asm_is_graph_node(nd)) e->asm_nodes.push_back(nd);
      if ((int)e->asm_nodes.size() != nevals) { lio_set_last_error(__FILE__, __LINE__, "solver graph: unexpected node count"); return LIO_ERR_CUDA; }
    }
    const double tu0 = now_s();
    for (cudaGraphNode_t nd : e->asm_nodes) {
      rc = asm_graph_update(e->sexec, nd, ap, e->d_Rt, e->asmw);
      if (rc != LIO_OK) return rc;
    }
    e->t_lin_lidar = now_s() - tu0;   // device-solver mode: host time of re-parameterising the asm_ppp nodes
    LIO_CUDA_OK(cudaGraphLaunch(e->sexec, gs));
    e->t_lin_host = now_s() - t0;     // device-solver mode: host time from the start of the solve to the end of the graph launch call
    e->launches += e->graph_launches;
    LIO_CUDA_OK(cudaEventRecord(e->ev_gout, gs));
    LIO_CUDA_OK(cudaStreamWaitEvent(st, e->ev_gout, 0));
  } else {
    rc = enqueue(st, false);
    if (rc != LIO_OK) return rc;
  }
  if (x == Exchange::rows) LIO_CUDA_OK(cudaMemcpyAsync(e->h_xerr, e->px.xbuf + kXErrOff, sizeof(int), cudaMemcpyDeviceToHost, st));
  LIO_CUDA_OK(cudaMemcpyAsync(&S, e->ds.st, offsetof(DevSolveState, scale), cudaMemcpyDeviceToHost, st));
  LIO_CUDA_OK(cudaStreamSynchronize(st));
  rc = xwait_report(e, Exchange::rows, st);
  if (rc != LIO_OK) return rc;
  for (int ev = 0; ev < std::min((use_graph || sharded) ? 1 : nevals, S.sc.evaluations); ++ev)
    asm_time_add(e, e->evp[2 * ev], e->evp[2 * ev + 1], nfeat);
  e->have_H0 = true; e->H0 = Mat(); e->cost0 = S.sc.initial_cost;
  if (assemble_only) return LIO_OK;
  for (int k = 0; k <= O; ++k) { std::memcpy(e->para_pose[k].data(), S.x + 16 * k, 7 * sizeof(double)); std::memcpy(e->para_sb[k].data(), S.x + 16 * k + 7, 9 * sizeof(double)); }
  std::memcpy(e->para_ex, S.x + 16 * (O + 1), 7 * sizeof(double));
  e->S_valid = false;
  e->summary = DoglegSummary();
  e->summary.iterations = S.sc.iteration; e->summary.successful_steps = S.sc.successful; e->summary.evaluations = S.sc.evaluations;
  e->summary.termination = S.sc.termination; e->summary.initial_cost = S.sc.initial_cost; e->summary.final_cost = S.sc.x_cost;
  e->cost_pim = S.sc.cost_pim; e->cost_ppp = S.sc.cost_ppp; e->cost_marg = S.sc.cost_marg;
  e->turn_off = S.sc.turn_off != 0;
  e->convergence_flag = S.sc.convergence_flag != 0;
  e->ex_constant = S.sc.ex_free == 0;
  if (!S.sc.prior_valid) e->prior.valid = false;
  if (S.sc.termination == 2 && !std::isfinite(S.sc.x_cost)) { lio_set_last_error(__FILE__, __LINE__, "solver breakdown"); return LIO_ERR_NUMERIC; }
  e->t_solve = now_s() - t0;
  return LIO_OK;
}

int slide_window(lio_est *e) {  // Estimator.cc:2570-2666
  const int W = e->W, O = e->O, pivot = W - O;
  if (e->init_local_map && pivot > 0) {
    const Tw tlb = tlb_double(e);
    const Tw transform_pivot = lidar_pose(e->Ps[pivot], e->Rs[pivot], tlb);
    const int i = pivot + 1;
    const Tw transform_li = lidar_pose(e->Ps[i], e->Rs[i], tlb);
    AffineF a = to_affine_f(tw_mul(tw_inverse(transform_li), transform_pivot));
    ConcatParams cp;
    std::memset(&cp, 0, sizeof(cp));
    cp.nsrc = 2;
    cp.src[0] = e->slot_ptr[e->slot_of[pivot]]; cp.n[0] = e->d_slot_n + e->slot_of[pivot];
    std::memcpy(cp.R[0], a.R, sizeof(a.R)); std::memcpy(cp.t[0], a.t, sizeof(a.t));
    cp.tag[0] = -1.f;
    cp.skip_first[0] = 1; cp.skip_n[0] = e->d_own_n + e->slot_of[0];  // size_surf_stack_[0]
    cp.src[1] = e->slot_ptr[e->slot_of[i]]; cp.n[1] = e->d_slot_n + e->slot_of[i];
    cp.identity[1] = 1;
    k_concat<<<std::max(1, std::min(e->sm_count * 2, (e->slot_cap + 255) / 256)), 256, 0, e->stream>>>(cp, e->d_tmp, e->d_counts + 3, e->slot_cap);
    ++e->launches;
    std::swap(e->slot_ptr[e->slot_of[i]], e->d_tmp);
    LIO_CUDA_OK(cudaMemcpyAsync(e->d_slot_n + e->slot_of[i], e->d_counts + 3, sizeof(int), cudaMemcpyDeviceToDevice, e->stream));
  }
  push_shift(e->Ps, e->Ps[W]); push_shift(e->Vs, e->Vs[W]); push_shift(e->Rs, e->Rs[W]); push_shift(e->Bas, e->Bas[W]); push_shift(e->Bgs, e->Bgs[W]);
  return LIO_OK;
}
