// HBM-resident voxel-hash k-NN + plane fit (stage B), see knn.cu.
#pragma once
#include "primitives.cuh"

namespace lio {

struct TransformF {  // Twist<float>: rot (x,y,z,w) + pos
  float qx, qy, qz, qw, px, py, pz;
};

struct CellHash {
  int table_size = 0;  // allocated slots, power of two
  int eff_size = 0;    // slots in use by the current build: the power of two >= 2 x its point bound (<= table_size)
  int cap_points = 0;
  float cell = 1.0f, inv_cell = 1.0f;
  DevMem<unsigned long long> keys;     // [table_size], ~0 = empty
  DevMem<int> count;                   // [table_size]
  DevMem<int> start;                   // [table_size]
  DevMem<int> slot_of, rank_of;        // [cap_points]
  DevMem<float4> cellpts;              // [cap_points] xyz + bitcast(map index)
  DevMem<unsigned long long> status;
  DevMem<int> ticket;
  int init(int cap_points);
  // Builds the hash over map[0..*n_dev): cells of edge `cell` (>= search radius).  n_max bounds *n_dev; the table, its
  // memsets and the scan are sized from n_max, so a tight bound (the caller usually knows one) keeps the build cheap.
  int build(const float4 *map, const int *n_dev, int n_max, float cell_size, cudaStream_t st, int *launches);
};

struct FeatureOut {
  float4 *pts = nullptr;   // xyz = point_ori, w = score s
  float4 *coef = nullptr;  // s*(pa,pb,pc,pd)
  int *src = nullptr;      // index of the originating surf point
  int *count = nullptr;    // device counter (appended to when keep_features)
  int cap = 0;
};

constexpr int kMaxKnnFrames = 16;

struct KnnFrame {
  const float4 *surf;
  const int *n_dev;        // device count of surf points
  int n_bound;             // host-side upper bound of *n_dev (grid sizing).  Contract: *n_dev <= n_bound.  With more points than
                           // the bound the frame's last tile is never dealt, so *out_count is never written.
  const TransformF *tf;    // device transform (frame -> pivot frame)
  float4 *out_p, *out_c;
  int *out_src, *out_count;
  int append;
  int tile0;
  const float *zaxis = nullptr;  // optional device float[3]: a fixed point_on_z_axis_ for the FOV test (PointMapping.cc:803-806)
};

struct KnnBatch {
  KnnFrame f[kMaxKnnFrames];
  int nframes = 0;
  int ntiles = 0;
};

struct KnnWork {
  DevMem<unsigned long long> status;
  DevMem<int> ticket;
  int ntiles_max = 0;
  int init(int max_queries_total);
};

// CalculateFeatures for several frames against the same map in ONE launch (tiles are dealt frame-major so each
// frame's accepted features are compacted in query order).
// state_clean: work.status[0 .. ntiles) and work.ticket are already zero (a previous k_odom_round re-armed them): no memsets.
int calculate_features_batch(const CellHash &h, KnnBatch &b, float min_match_sq_dis, float min_plane_dis, const int *done_flag,
                             KnnWork &work, cudaStream_t st, int *launches, int fit = 0, bool state_clean = false);

// fit = 2 / 3: the scan-to-map flavours of PointMapping::OptimizeTransformTobeMapped (PointMapping.cc:514-606 surf with the
// sign-normalised coefficient and intensity = s |pd2|; :381-512 corner with ONE feature per line, intensity = s ld2).
// fit = 0: point-to-plane (surf branch); fit = 1: point-to-line (USE_CORNER branch, Estimator.cc:1101-1227), which
// emits two consecutive half-weight features per accepted query (out buffers sized 2 x queries).
// Estimator::CalculateFeatures (Estimator.cc:970-1097) for one frame.  Appends to `out` starting at
// *out.count when `append` is non-zero, else overwrites from 0.  `done_flag` (optional device int):
// when non-null and *done_flag != 0 the launch is a no-op (used by the LaserOdom iteration chain).
int calculate_features_dev(const CellHash &h, const float4 *map, const float4 *surf, const int *nsurf_dev, int nsurf_max,
                           const TransformF *tf_dev, float min_match_sq_dis, float min_plane_dis, FeatureOut out, int append,
                           const int *done_flag, KnnWork &work, cudaStream_t st, int *launches, int fit = 0, const float *zaxis_dev = nullptr);

}  // namespace lio
