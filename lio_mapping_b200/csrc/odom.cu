// Estimator::CalculateLaserOdom (Estimator.cc:1242-1359) and PointMapping::OptimizeTransformTobeMapped (PointMapping.cc:325-753) on
// device-resident clouds: the reduce / solve kernels, the estimator's round driver, the scan-to-map loop and their host-array parity
// entries.  Compiled with -fmad=false, like the k-NN kernels whose features they reduce.
#include <algorithm>
#include "odom.cuh"
#include "twistf.h"

namespace lio {

constexpr int kOdomThreads = 256;

__global__ void __launch_bounds__(kOdomThreads)
k_odom_reduce(const float4 *__restrict__ pts, const float4 *__restrict__ coef, const int *__restrict__ n_dev,
              const TransformF *__restrict__ tf_dev, OdomState *__restrict__ st, double *__restrict__ partial, int mode = 0) {
  __shared__ double sred[kOdomThreads / 32][27];
  __shared__ bool is_last;
  if (st->done) return;
  const int n = *n_dev;
  const TransformF tf = *tf_dev;
  float R[9], Ri[9];
  odom_rotation(tf, R);
  // mode 2 (MapBuilder::OptimizeMap, MapBuilder.cc:905-911): J_r is post-multiplied by rot.inverse().toRotationMatrix()
  // (inverse = conjugate / squaredNorm) and the rotation information matrix diag(5e-3, 5e-3, 1)
  {
    const float n2 = tf.qx * tf.qx + tf.qy * tf.qy + tf.qz * tf.qz + tf.qw * tf.qw;
    TransformF inv = tf;
    inv.qx = -tf.qx / n2; inv.qy = -tf.qy / n2; inv.qz = -tf.qz / n2; inv.qw = tf.qw / n2;
    odom_rotation(inv, Ri);
  }
  double acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = __ldg(pts + i), c = __ldg(coef + i);
    // CalculateLaserOdom: d2 = w . (R p + t) + b (Estimator.cc:1282-1284); scan-to-map: d2 = coeff.intensity (PointMapping.cc:634)
    float row[6], d2;
    odom_row(tf, R, p, c, row, d2);
    if (mode != 0) d2 = c.w;
    if (mode == 2) {
      const float t0 = row[0] * Ri[0] + row[1] * Ri[3] + row[2] * Ri[6];
      const float t1 = row[0] * Ri[1] + row[1] * Ri[4] + row[2] * Ri[7];
      const float t2 = row[0] * Ri[2] + row[1] * Ri[5] + row[2] * Ri[8];
      row[0] = t0 * 5e-3f; row[1] = t1 * 5e-3f; row[2] = t2 * 1.0f;
    }
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
#pragma unroll
      for (int b = a; b < 6; ++b) acc[k++] += (double)(row[a] * row[b]);
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] += (double)(row[a] * (-d2));
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) {
    double v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane_id() == 0) sred[warp_id()][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 27) {
    double v = 0;
#pragma unroll
    for (int w = 0; w < kOdomThreads / 32; ++w) v += sred[w][threadIdx.x];
    partial[blockIdx.x * 32 + threadIdx.x] = v;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(&st->counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x < 27) {
    double v = 0;
    for (unsigned b = 0; b < gridDim.x; ++b) v += __ldcg(partial + b * 32 + threadIdx.x);
    if (threadIdx.x < 21) {
      int k = threadIdx.x, a = 0;
      while (k >= 6 - a) { k -= 6 - a; ++a; }
      int b = a + k;
      st->AtA[a * 6 + b] = v; st->AtA[b * 6 + a] = v;
    } else {
      st->AtB[threadIdx.x - 21] = v;
    }
  }
  if (threadIdx.x == 0) st->counter = 0u;
}

__global__ void k_odom_solve(OdomState *__restrict__ st, TransformF *__restrict__ tf_dev, double delta_r_abort, double delta_t_abort,
                             int round = -1, const int *__restrict__ n_dev = nullptr, int min_features = 0, int left_update = 0) {
  if (threadIdx.x != 0 || st->done) return;
  odom_solve_step(st, tf_dev, delta_r_abort, delta_t_abort, round, n_dev, min_features, left_update);
}

// One CalculateLaserOdom round after the k-NN launch, as a single CTA: reduce the round's features (float products
// accumulated in double, fixed thread -> feature mapping and a fixed reduction tree: deterministic), solve, and zero the
// k-NN launch state (tile status words, ticket) so that the next round's k-NN launch needs no memset.
constexpr int kOdomRoundThreads = 512;
__global__ void __launch_bounds__(kOdomRoundThreads)
k_odom_round(const float4 *__restrict__ pts, const float4 *__restrict__ coef, const int *__restrict__ n_dev, TransformF *__restrict__ tf_dev,
             OdomState *__restrict__ st, double delta_r_abort, double delta_t_abort, unsigned long long *__restrict__ knn_status, int knn_ntiles,
             int *__restrict__ knn_ticket) {
  __shared__ double sred[kOdomRoundThreads / 32][27];
  if (st->done) return;   // the k-NN launch of a finished chain was a no-op: nothing to clean
  const int n = *n_dev;
  const TransformF tf = *tf_dev;
  float R[9];
  odom_rotation(tf, R);
  double acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.0;
  // four features per trip: their eight loads are issued together (the loop is latency bound: ~25 features per thread)
#pragma unroll 1
  for (int i0 = threadIdx.x; i0 < n; i0 += 4 * kOdomRoundThreads) {
    float4 pq[4], cq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + u * kOdomRoundThreads;
      if (i < n) { pq[u] = __ldg(pts + i); cq[u] = __ldg(coef + i); }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
    if (i0 + u * kOdomRoundThreads >= n) break;
    float row[6], d2;
    odom_row(tf, R, pq[u], cq[u], row, d2);
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
#pragma unroll
      for (int b = a; b < 6; ++b) acc[k++] += (double)(row[a] * row[b]);
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] += (double)(row[a] * (-d2));
    }
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) {
    double v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane_id() == 0) sred[warp_id()][k] = v;
  }
  for (int t = threadIdx.x; t < knn_ntiles; t += kOdomRoundThreads) knn_status[t] = 0ull;
  if (threadIdx.x == 0) *knn_ticket = 0;
  __syncthreads();
  if (threadIdx.x < 27) {
    double v = 0;
#pragma unroll
    for (int w = 0; w < kOdomRoundThreads / 32; ++w) v += sred[w][threadIdx.x];
    if (threadIdx.x < 21) {
      int k = threadIdx.x, a = 0;
      while (k >= 6 - a) { k -= 6 - a; ++a; }
      const int b = a + k;
      st->AtA[a * 6 + b] = v; st->AtA[b * 6 + a] = v;
    } else {
      st->AtB[threadIdx.x - 21] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) odom_solve_step(st, tf_dev, delta_r_abort, delta_t_abort);
}

int odom_rounds(const CellHash &h, const float4 *surf, const int *n_dev, int n_bound, TransformF *tf_dev, const FeatureOut &fo,
                bool keep_features, OdomState *odom, double *partial, KnnWork &work, float min_match_sq_dis, float min_plane_dis,
                int from, int to, int sm, cudaStream_t q, int *launches) {
  if (!keep_features) {
    // two launches per round and no memset: the k-NN + plane fit of the frame, then ONE CTA that reduces the round's features
    // to A^T A / A^T b, takes the 6 x 6 Gauss-Newton step and re-arms the k-NN launch state
    KnnBatch ob;
    ob.nframes = 1;
    KnnFrame &f = ob.f[0];
    f.surf = surf; f.n_dev = n_dev; f.n_bound = n_bound; f.tf = tf_dev;
    f.out_p = fo.pts; f.out_c = fo.coef; f.out_src = fo.src; f.out_count = fo.count;
    f.append = 0; f.tile0 = 0;
    for (int it = from; it < to; ++it) {
      int rc = calculate_features_batch(h, ob, min_match_sq_dis, min_plane_dis, &odom->done, work, q, launches, 0, it > 0);
      if (rc != LIO_OK) return rc;
      k_odom_round<<<1, kOdomRoundThreads, 0, q>>>(fo.pts, fo.coef, fo.count, tf_dev, odom, 0.05, 0.05, work.status, ob.ntiles, work.ticket);
      if (launches) ++*launches;
    }
  } else {
    // keep_features: every round re-evaluates ALL kept features at the current transform (Estimator.cc:978-980), so the
    // reduction is a pass of its own
    const int nb = std::max(1, std::min(sm, (fo.cap + kOdomThreads - 1) / kOdomThreads));
    for (int it = from; it < to; ++it) {
      int rc = calculate_features_dev(h, nullptr, surf, n_dev, n_bound, tf_dev, min_match_sq_dis, min_plane_dis, fo, 1, &odom->done, work, q,
                                      launches);
      if (rc != LIO_OK) return rc;
      k_odom_reduce<<<nb, kOdomThreads, 0, q>>>(fo.pts, fo.coef, fo.count, tf_dev, odom, partial);
      k_odom_solve<<<1, 32, 0, q>>>(odom, tf_dev, 0.05, 0.05);
      if (launches) *launches += 2;
    }
  }
  return LIO_OK;
}

// ---- PointMapping::OptimizeTransformTobeMapped (PointMapping.cc:325-753) on device-resident clouds -----------------------
int ScanToMapWork::init(int cap_corner_map, int cap_surf_map, int cap_queries) {
  cap_feat = cap_queries > 0 ? cap_queries : 1;
  if (hc.init(cap_corner_map > 0 ? cap_corner_map : 1) != 0 || hs.init(cap_surf_map > 0 ? cap_surf_map : 1) != 0 || w.init(cap_feat + 1) != 0) return -1;
  if (!(alloc(d_fpts, cap_feat) && alloc(d_fcoef, cap_feat) && alloc(d_fsrc, cap_feat) && alloc(d_n, 8) && alloc(d_tf, 1) && alloc(d_odom, 1) &&
        alloc(d_partial, 32 * 1024) && alloc(d_z, 4)))
    return -1;
  fo.pts = d_fpts; fo.coef = d_fcoef; fo.src = d_fsrc;
  fo.cap = cap_feat;
  fo.count = d_n + 4;
  return 0;
}

// Maps and stacks are device arrays; Kc / Ks are known on the host (the caller assembled the maps), the stack sizes are
// device counts bounded by Mc_max / Ms_max.  tf7 (host, in/out).  No synchronisation before the final read-back.
int scan_to_map_run(ScanToMapWork &W, const float4 *d_cmap, int Kc, const float4 *d_smap, int Ks, const float4 *d_corner, const int *d_nc,
                    int Mc_max, const float4 *d_surf, const int *d_ns, int Ms_max, float *tf7, float min_match_sq_dis, float min_plane_dis,
                    int max_iter, double delta_r_abort, double delta_t_abort, int variant, int *n_out, int *iters, int sm, cudaStream_t st) {
  if (n_out) *n_out = 0;
  if (iters) *iters = 0;
  if (Kc <= 10 || Ks <= 100 || max_iter == 0) return LIO_OK;  // PointMapping.cc:327-329: nothing to optimise against
  if (Mc_max + Ms_max > W.cap_feat) { lio_set_last_error(__FILE__, __LINE__, "scan-to-map: stacks exceed the feature capacity"); return LIO_ERR_CAPACITY; }
  const int hn[2] = {Kc, Ks};
  LIO_CUDA_OK(cudaMemcpyAsync(W.d_n, hn, sizeof(hn), cudaMemcpyHostToDevice, st));
  LIO_CUDA_OK(cudaMemsetAsync(W.d_n + 4, 0, sizeof(int), st));
  LIO_CUDA_OK(cudaMemcpyAsync(W.d_tf, tf7, sizeof(TransformF), cudaMemcpyHostToDevice, st));
  LIO_CUDA_OK(cudaMemsetAsync(W.d_odom, 0, sizeof(OdomState), st));
  {  // point_on_z_axis_ = T0 * (0, 0, 10), fixed for the whole optimisation (PointMapping.cc:803-806); float, no FMA
    TwistF t0;
    t0.qx = tf7[0]; t0.qy = tf7[1]; t0.qz = tf7[2]; t0.qw = tf7[3];
    float sx, sy, sz;
    rotate_host(t0, 0.0f, 0.0f, 10.0f, sx, sy, sz);
    const float hz[4] = {sx + tf7[4], sy + tf7[5], sz + tf7[6], 0.f};
    LIO_CUDA_OK(cudaMemcpyAsync(W.d_z, hz, sizeof(hz), cudaMemcpyHostToDevice, st));
    LIO_CUDA_OK(cudaStreamSynchronize(st));   // hn / hz are stack variables
  }
  const float cell = sqrtf(min_match_sq_dis) * (1.0f + 1.0f / 1024.0f);
  int rc = W.hc.build(d_cmap, W.d_n, Kc, cell, st, nullptr);
  if (rc == LIO_OK) rc = W.hs.build(d_smap, W.d_n + 1, Ks, cell, st, nullptr);
  const int cap = std::max(1, Mc_max + Ms_max);
  const int nb = std::max(1, std::min(sm, (cap + kOdomThreads - 1) / kOdomThreads));
  for (int it = 0; it < max_iter && rc == LIO_OK; ++it) {
    rc = calculate_features_dev(W.hc, d_cmap, d_corner, d_nc, std::max(Mc_max, 1), W.d_tf, min_match_sq_dis, min_plane_dis, W.fo, 0,
                                &W.d_odom->done, W.w, st, nullptr, 3, W.d_z);
    if (rc == LIO_OK)
      rc = calculate_features_dev(W.hs, d_smap, d_surf, d_ns, std::max(Ms_max, 1), W.d_tf, min_match_sq_dis, min_plane_dis, W.fo, 1,
                                  &W.d_odom->done, W.w, st, nullptr, 2, W.d_z);
    if (rc != LIO_OK) break;
    k_odom_reduce<<<nb, kOdomThreads, 0, st>>>(W.fo.pts, W.fo.coef, W.fo.count, W.d_tf, W.d_odom, W.d_partial, variant == 1 ? 2 : 1);
    k_odom_solve<<<1, 32, 0, st>>>(W.d_odom, W.d_tf, delta_r_abort, delta_t_abort, it, W.fo.count, kScanToMapMinFeatures, variant == 1 ? 1 : 0);
  }
  if (rc != LIO_OK) return rc;
  int m = 0;
  OdomState hs2;
  cudaError_t ce = cudaMemcpyAsync(&m, W.d_n + 4, sizeof(int), cudaMemcpyDeviceToHost, st);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(&hs2, W.d_odom, sizeof(OdomState), cudaMemcpyDeviceToHost, st);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(tf7, W.d_tf, sizeof(TransformF), cudaMemcpyDeviceToHost, st);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
  if (ce != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(ce)); return LIO_ERR_CUDA; }
  if (m > cap) { lio_set_last_error(__FILE__, __LINE__, "feature buffer overflow"); return LIO_ERR_CAPACITY; }
  if (n_out) *n_out = m;
  if (iters) *iters = hs2.iter;
  return LIO_OK;
}

}  // namespace lio

using namespace lio;

// ---- C-ABI: PointMapping::OptimizeTransformTobeMapped on explicit host arrays (parity entry) ------------------------
extern "C" int lio_scan_to_map_host(const float *corner_map, int Kc, const float *surf_map, int Ks, const float *corner, int Mc,
                                    const float *surf, int Ms, float *tf7, float min_match_sq_dis, float min_plane_dis, int max_iter,
                                    double delta_r_abort, double delta_t_abort, int variant, float *pts4, float *coef4, int32_t *src,
                                    int *n_out, int *iters, int device) {
  if (!corner_map || !surf_map || !corner || !surf || !tf7 || Kc < 0 || Ks < 0 || Mc < 0 || Ms < 0 || max_iter < 0 || variant < 0 || variant > 1)
    return LIO_ERR_INVALID;
  int sm = 132;
  LIO_TRY(select_device(device, &sm));
  if (n_out) *n_out = 0;
  if (iters) *iters = 0;
  if (Kc <= 10 || Ks <= 100 || max_iter == 0) return LIO_OK;  // PointMapping.cc:327-329: nothing to optimise against
  DevBufs d;
  ScanToMapWork W;
  float4 *d_cmap = nullptr, *d_smap = nullptr, *d_corner = nullptr, *d_surf = nullptr;
  int *d_cnt = nullptr;
  int rc = LIO_OK;
  const int hn[2] = {Mc, Ms};
  if (W.init(Kc, Ks, Mc + Ms) != 0) { lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed"); rc = LIO_ERR_CUDA; }
  else if (!d.alloc(&d_cmap, Kc) || !d.alloc(&d_smap, Ks) || !d.alloc(&d_corner, Mc) || !d.alloc(&d_surf, Ms) || !d.alloc(&d_cnt, 2) ||
           !d.up(d_cmap, (const float4 *)corner_map, Kc) || !d.up(d_smap, (const float4 *)surf_map, Ks) ||
           !d.up(d_corner, (const float4 *)corner, Mc) || !d.up(d_surf, (const float4 *)surf, Ms) || !d.up(d_cnt, hn, 2))
    rc = LIO_ERR_CUDA;
  int m = 0;
  if (rc == LIO_OK)
    rc = scan_to_map_run(W, d_cmap, Kc, d_smap, Ks, d_corner, d_cnt, Mc, d_surf, d_cnt + 1, Ms, tf7, min_match_sq_dis, min_plane_dis, max_iter,
                         delta_r_abort, delta_t_abort, variant, &m, iters, sm, 0);
  if (rc == LIO_OK) {
    if (n_out) *n_out = m;
    if ((pts4 && !d.down((float4 *)pts4, W.fo.pts, m)) || (coef4 && !d.down((float4 *)coef4, W.fo.coef, m)) || (src && !d.down(src, W.fo.src, m)))
      rc = LIO_ERR_CUDA;
  }
  return rc;
}

// ---- C-ABI: Estimator::CalculateLaserOdom on explicit host arrays (parity entry) ---------------------------------
// Runs the estimator's own round driver (odom_rounds): without keep_features the batched k-NN launch and the fused k_odom_round.
extern "C" int lio_laser_odom_host(const float *map, int K, const float *surf, int M, float *tf7, float min_match_sq_dis,
                                   float min_plane_dis, int keep_features, int max_iter, float *pts4, float *coef4, int32_t *src,
                                   int *n_out, int *iters, int device) {
  if (!map || !surf || !tf7 || !n_out || K < 0 || M < 0 || max_iter < 0) return LIO_ERR_INVALID;
  int sm = 132;
  LIO_TRY(select_device(device, &sm));
  *n_out = 0;
  if (iters) *iters = 0;
  if (M == 0 || max_iter == 0) return LIO_OK;
  const int cap = M * (keep_features ? max_iter : 1);
  DevBufs d;
  CellHash h;
  KnnWork w;
  float4 *d_map = nullptr, *d_surf = nullptr;
  FeatureOut fo;
  int *d_n = nullptr;
  TransformF *d_tf = nullptr;
  OdomState *d_odom = nullptr;
  double *d_partial = nullptr;
  int rc = LIO_OK;
  const int Kc = K > 0 ? K : 1;
  const int hn[3] = {K, M, 0};
  if (h.init(Kc) != 0 || w.init(M) != 0) { lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed"); rc = LIO_ERR_CUDA; }
  else if (!d.alloc(&d_map, Kc) || !d.alloc(&d_surf, M) || !d.alloc(&fo.pts, cap) || !d.alloc(&fo.coef, cap) || !d.alloc(&fo.src, cap) ||
           !d.alloc(&d_n, 4) || !d.alloc(&d_tf, 1) || !d.alloc(&d_odom, 1) || !d.alloc(&d_partial, 32 * 1024) ||
           !d.up(d_map, (const float4 *)map, K) || !d.up(d_surf, (const float4 *)surf, M) || !d.up(d_n, hn, 3) ||
           !d.up(d_tf, (const TransformF *)tf7, 1) || !d.ok(cudaMemset(d_odom, 0, sizeof(OdomState))))
    rc = LIO_ERR_CUDA;
  if (rc == LIO_OK) {
    fo.count = d_n + 2; fo.cap = cap;
    const float cell = sqrtf(min_match_sq_dis) * (1.0f + 1.0f / 1024.0f);
    rc = h.build(d_map, d_n, Kc, cell, 0, nullptr);
    if (rc == LIO_OK)
      rc = odom_rounds(h, d_surf, d_n + 1, M, d_tf, fo, keep_features != 0, d_odom, d_partial, w, min_match_sq_dis, min_plane_dis, 0, max_iter,
                       sm, 0, nullptr);
  }
  int m = 0;
  OdomState hs;
  if (rc == LIO_OK && (!d.down(&m, d_n + 2, 1) || !d.down(&hs, d_odom, 1) || !d.down((TransformF *)tf7, d_tf, 1))) rc = LIO_ERR_CUDA;
  if (rc == LIO_OK && m > cap) { lio_set_last_error(__FILE__, __LINE__, "feature buffer overflow"); rc = LIO_ERR_CAPACITY; }
  if (rc == LIO_OK) {
    *n_out = m;
    if (iters) *iters = hs.iter;
    if ((pts4 && !d.down((float4 *)pts4, fo.pts, m)) || (coef4 && !d.down((float4 *)coef4, fo.coef, m)) || (src && !d.down(src, fo.src, m)))
      rc = LIO_ERR_CUDA;
  }
  return rc;
}

// ---- C-ABI: test seams of the 6-DoF Gauss-Newton step --------------------------------------------------------------
// The normal equations of n explicit features as one of the production reductions leaves them in OdomState.
extern "C" int lio_odom_normal_equations_host(const float *pts4, const float *coef4, int n, const float *tf7, int kernel, int blocks,
                                              double *AtA, double *AtB, int device) {
  constexpr int kMaxBlocks = 1024;
  if ((n > 0 && (!pts4 || !coef4)) || !tf7 || !AtA || !AtB || n < 0 || kernel < 0 || kernel > 3 || blocks < 0 || blocks > kMaxBlocks ||
      (kernel == 3 && blocks > 1))
    return LIO_ERR_INVALID;
  int sm = 132;
  LIO_TRY(select_device(device, &sm));
  DevBufs d;
  float4 *d_pts = nullptr, *d_coef = nullptr;
  int *d_n = nullptr;
  TransformF *d_tf = nullptr;
  OdomState *d_odom = nullptr;
  double *d_partial = nullptr;
  unsigned long long *d_status = nullptr;
  if (!d.alloc(&d_pts, n) || !d.alloc(&d_coef, n) || !d.alloc(&d_n, 2) || !d.alloc(&d_tf, 1) || !d.alloc(&d_odom, 1) ||
      !d.alloc(&d_partial, 32 * kMaxBlocks) || !d.alloc(&d_status, 1) || !d.up(d_pts, (const float4 *)pts4, n) ||
      !d.up(d_coef, (const float4 *)coef4, n) || !d.up(d_n, &n, 1) || !d.up(d_tf, (const TransformF *)tf7, 1) ||
      !d.ok(cudaMemset(d_odom, 0, sizeof(OdomState))))
    return LIO_ERR_CUDA;
  if (kernel < 3) {
    const int nb = blocks ? blocks : std::max(1, std::min(sm, (n + kOdomThreads - 1) / kOdomThreads));
    k_odom_reduce<<<nb, kOdomThreads>>>(d_pts, d_coef, d_n, d_tf, d_odom, d_partial, kernel);
  } else {
    k_odom_round<<<1, kOdomRoundThreads>>>(d_pts, d_coef, d_n, d_tf, d_odom, 0.05, 0.05, d_status, 0, d_n + 1);
  }
  OdomState hs;
  if (!d.ok(cudaGetLastError()) || !d.down(&hs, d_odom, 1)) return LIO_ERR_CUDA;
  for (int k = 0; k < 36; ++k) AtA[k] = hs.AtA[k];
  for (int k = 0; k < 6; ++k) AtB[k] = hs.AtB[k];
  return LIO_OK;
}

// variant 0 CalculateLaserOdom, 1 PointMapping, 2 MapBuilder (left update), 3 PointOdometry, with the parameters of their loops
__global__ void k_odom_step_variant(OdomState *__restrict__ st, TransformF *__restrict__ tf_dev, double delta_r_abort, double delta_t_abort,
                                    int variant, int round, const int *__restrict__ n_dev) {
  if (threadIdx.x != 0 || st->done) return;
  if (variant == 0) odom_solve_step(st, tf_dev, delta_r_abort, delta_t_abort);
  else if (variant == 1) odom_solve_step(st, tf_dev, delta_r_abort, delta_t_abort, round, n_dev, kScanToMapMinFeatures, 0);
  else if (variant == 2) odom_solve_step(st, tf_dev, delta_r_abort, delta_t_abort, round, n_dev, kScanToMapMinFeatures, 1);
  else odom_solve_step(st, tf_dev, delta_r_abort, delta_t_abort, round, n_dev, kPoMinFeatures, 0, kPoEigThre);
}

// `rounds` steps of one chain from a cleared OdomState: round r stores AtA[36 r..], AtB[6 r..] and n_feat[r] and takes the step.
extern "C" int lio_odom_step_host(int rounds, const double *AtA, const double *AtB, const int *n_feat, int variant, double delta_r_abort,
                                  double delta_t_abort, float *tf7, float *tf_per_round, int *state_out, float *matP, int device) {
  if (rounds < 0 || (rounds > 0 && (!AtA || !AtB || !n_feat)) || !tf7 || variant < 0 || variant > 3) return LIO_ERR_INVALID;
  LIO_TRY(select_device(device));
  DevBufs d;
  TransformF *d_tf = nullptr;
  OdomState *d_odom = nullptr;
  int *d_n = nullptr;
  if (!d.alloc(&d_tf, 1) || !d.alloc(&d_odom, 1) || !d.alloc(&d_n, 1) || !d.up(d_tf, (const TransformF *)tf7, 1) ||
      !d.ok(cudaMemset(d_odom, 0, sizeof(OdomState))))
    return LIO_ERR_CUDA;
  for (int r = 0; r < rounds; ++r) {
    if (!d.up(d_odom->AtA, AtA + 36 * r, 36) || !d.up(d_odom->AtB, AtB + 6 * r, 6) || !d.up(d_n, n_feat + r, 1)) return LIO_ERR_CUDA;
    k_odom_step_variant<<<1, 1>>>(d_odom, d_tf, delta_r_abort, delta_t_abort, variant, r, d_n);
    if (!d.ok(cudaGetLastError())) return LIO_ERR_CUDA;
    if (tf_per_round && !d.down((TransformF *)(tf_per_round + 7 * r), d_tf, 1)) return LIO_ERR_CUDA;
  }
  OdomState hs;
  if (!d.down(&hs, d_odom, 1) || !d.down((TransformF *)tf7, d_tf, 1)) return LIO_ERR_CUDA;
  if (state_out) { state_out[0] = hs.degenerate; state_out[1] = hs.done; state_out[2] = hs.iter; }
  if (matP) for (int k = 0; k < 36; ++k) matP[k] = hs.matP[k];
  return LIO_OK;
}
