/* lio_b200.h — C-ABI of liblio_b200.so: the H100-native (sm_90a) replacement of the compute hot
 * path of hyye/lio-mapping.  Plain pointers and sizes only; no C++/torch types.
 *
 * Each entry point names the reference interface (file:line under the reference tree) it stands
 * in for.  The reference has no FFI layer of its own: the seams are its C++ member functions and
 * the ceres::CostFunction contract (SURVEY.md §8b); INTEGRATION.md shows the shim a maintainer
 * adds at each seam.
 *
 * Conventions
 *   - point clouds are arrays of float4 {x, y, z, intensity}  (pcl::PointXYZI payload);
 *   - poses are double[7] {px,py,pz,qx,qy,qz,qw} (para_pose_ layout, Estimator.cc:2445-2452),
 *     float transforms are float[7] {qx,qy,qz,qw,px,py,pz} (Twist<float>);
 *   - every function returns LIO_OK (0) or a negative lio_status; lio_last_error() gives text;
 *   - an entry that enqueues work on, copies from or waits for a handle's device makes that device current and leaves it
 *     current, whatever device was current before; an entry that only reads or writes host state leaves it alone;
 *   - "_host" variants take host buffers and copy in/out on the context's stream (synchronous
 *     on return); "_dev" variants take device pointers and are stream-ordered (asynchronous);
 *   - one thread drives a given handle at a time (same rule as the reference objects).
 */
#ifndef LIO_B200_H_
#define LIO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum lio_status {
  LIO_OK = 0,
  LIO_ERR_CUDA = -1,        /* a CUDA runtime call failed (text in lio_last_error) */
  LIO_ERR_INVALID = -2,     /* bad argument */
  LIO_ERR_CAPACITY = -3,    /* input exceeds the capacity given at create time */
  LIO_ERR_NO_DEVICE = -4,   /* no CUDA device: there is NO CPU fallback in this library */
  LIO_ERR_NUMERIC = -5      /* solver breakdown (non-finite / not positive definite) */
} lio_status;

const char *lio_last_error(void);
int lio_version(void);
/* Number of usable CUDA devices (0 => every compute entry point returns LIO_ERR_NO_DEVICE). */
int lio_device_count(void);

/* ------------------------------------------------------------------------------------------
 * Stage A — lio::PointProcessor  (include/point_processor/PointProcessor.h:122-229,
 *           src/point_processor/PointProcessor.cc:185-783)
 * ---------------------------------------------------------------------------------------- */
typedef struct lio_pp_config {      /* PointProcessorConfig, PointProcessor.h:104-120 + ctor :76-80 */
  float lower_bound;                /* deg */
  float upper_bound;                /* deg */
  int num_rings;
  double scan_period;
  int num_scan_subregions;
  int num_curvature_regions;
  float surf_curv_th;
  int max_corner_sharp;
  int max_corner_less_sharp;
  int max_surf_flat;
  float less_flat_filter_size;
} lio_pp_config;

typedef struct lio_pp lio_pp;

/* Which output of the processor (names follow the reference members, PointProcessor.h:170-194). */
typedef enum lio_pp_cloud {
  LIO_PP_LASER_SCANS = 0,           /* laser_scans concatenated: intensity = ring + rel_time      */
  LIO_PP_CLOUD_IN_RINGS = 1,        /* cloud_in_rings_: intensity = int(I) + rel_time             */
  LIO_PP_CORNER_SHARP = 2,          /* corner_points_sharp_                                       */
  LIO_PP_CORNER_LESS_SHARP = 3,     /* corner_points_less_sharp_                                  */
  LIO_PP_SURF_FLAT = 4,             /* surface_points_flat_                                       */
  LIO_PP_SURF_LESS_FLAT = 5,        /* surface_points_less_flat_ (per-ring VoxelGrid(0.2) output) */
  LIO_PP_NUM_CLOUDS = 6
} lio_pp_cloud;

typedef enum lio_pp_index {         /* index sets into the ring-ordered cloud (parity / debug)   */
  LIO_PP_IDX_SHARP = 0,
  LIO_PP_IDX_LESS_SHARP = 1,
  LIO_PP_IDX_FLAT = 2,
  LIO_PP_IDX_ORIG = 3               /* input index of every ring-ordered point                   */
} lio_pp_index;

void lio_pp_default_config(lio_pp_config *cfg);                 /* PointProcessor.h:104-120 defaults */
/* PointProcessor::PointProcessor(lower, upper, rings) + SetupConfig  (PointProcessor.cc:74-95) */
int lio_pp_create(const lio_pp_config *cfg, int max_points, int device, void *cuda_stream, lio_pp **out);
int lio_pp_destroy(lio_pp *pp);
/* SetInputCloud + PointToRing + ExtractFeaturePoints (PointProcessor.cc:96-100,140-172,185-783);
 * xyzi: n x float4 on the HOST (pinned or pageable).  Synchronous. */
int lio_pp_process_host(lio_pp *pp, const float *xyzi, int n);
/* Same, input already on the device; asynchronous on the stream. */
int lio_pp_process_dev(lio_pp *pp, const float *xyzi_dev, int n);
/* The overload for sensors that deliver the ring index (lio::PointXYZIR, include/point_processor/point_types.h:37-52):
 * PointToRing(PointCloud<PointIR>) PointProcessor.cc:428-536 — ring id from `rings` (n x uint16), rel_time scaled by the
 * observed azimuth range end_ori_ - start_ori_ — followed by the shared ExtractFeaturePoints.  Synchronous.
 * Checked against the oracle (tests/test_zz_ring_field_gpu.py) and against a plain numpy statement of PointProcessor at
 * its edges (tests/test_stage_a_edges_gpu.py) on the device. */
int lio_pp_process_host_ring(lio_pp *pp, const float *xyzi, const uint16_t *rings, int n);
/* The same with xyzi (n x float4) and rings (n x uint16) already on the device, e.g. a sensor driver's DMA target: the kernels of
 * lio_pp_process_host_ring without its uploads (which is "upload, then this entry").  Stream rule and count accessors as for
 * lio_pp_process_dev: asynchronous on the stream, the inputs are read by work enqueued there; lio_pp_cloud_sizes waits. */
int lio_pp_process_dev_ring(lio_pp *pp, const float *xyzi_dev, const uint16_t *rings_dev, int n);
/* Sizes of the six output clouds (synchronises the stream). */
int lio_pp_cloud_sizes(lio_pp *pp, int sizes[LIO_PP_NUM_CLOUDS]);
/* Copy one output cloud to the host (cap in points).  Returns the point count via *n. */
int lio_pp_download_cloud(lio_pp *pp, int which, float *out, int cap, int *n);
/* Device pointer of one output cloud (float4 array, valid until the next process call). */
int lio_pp_cloud_dev(lio_pp *pp, int which, const float **ptr);
int lio_pp_download_index(lio_pp *pp, int which, int32_t *out, int cap, int *n);
/* scan_ranges (PointProcessor.h:172): R pairs (start,end) exactly as the reference stores them. */
int lio_pp_download_scan_ranges(lio_pp *pp, int32_t *out_2R);
/* scan_ring_mask_ after the last subregion and PointLabel of every ring-ordered point. */
int lio_pp_download_mask_labels(lio_pp *pp, uint8_t *mask, int8_t *labels, int cap);
int lio_pp_start_ori(lio_pp *pp, float *start_ori);
/* Number of kernels launched by the last process call (bench bookkeeping). */
int lio_pp_last_launches(lio_pp *pp);

/* ------------------------------------------------------------------------------------------
 * Stage B primitives on explicit host arrays (parity entries; the estimator context below keeps
 * the same kernels device-resident).
 * ---------------------------------------------------------------------------------------- */
/* pcl::VoxelGrid<PointXYZI>::filter with setLeafSize(leaf,leaf,leaf)
 * (call sites Estimator.cc:679-687, :1518-1519; PointProcessor.cc:737-751).  out sized cap points. */
int lio_voxel_grid_host(const float *cloud, int n, float leaf, float *out, int cap, int *n_out, int device);
/* Estimator::CalculateFeatures (Estimator.cc:970-1097) with the kd-tree replaced by the voxel-hash
 * k-NN: map (K x float4) = local_surf_points_filtered_ptr_, surf (M x float4) = surf_stack_[idx],
 * tf7 = local_transform {qx,qy,qz,qw,px,py,pz}.  Outputs (sized M): pts4 = {point.xyz, score},
 * coef4 = coeffs, src = index of the originating surf point. */
int lio_calculate_features_host(const float *map, int K, const float *surf, int M, const float *tf7,
                                float min_match_sq_dis, float min_plane_dis, float *pts4, float *coef4, int32_t *src,
                                int *n_out, int device);
/* Point-to-line branch of Estimator::CalculateFeatures (Estimator.cc:1101-1227, compiled out in the reference build:
 * USE_CORNER is undefined, Estimator.h:55-56) == the live corner matching of PointMapping::OptimizeTransformTobeMapped
 * (PointMapping.cc:381-512): 5-NN in the corner map, centroid + 3x3 covariance eigen-decomposition, line accepted iff
 * lambda_3 > 3 lambda_2; a line is emitted as TWO consecutive half-weight plane-like features (normal_to_point and
 * normal_cross_point), which go through the same PivotPointPlaneFactor / fused stage-C kernel.
 * corner_map (K x float4) = local corner map, corner (M x float4) = corner stack of the frame; outputs sized 2*M. */
int lio_calculate_line_features_host(const float *corner_map, int K, const float *corner, int M, const float *tf7,
                                     float min_match_sq_dis, float *pts4, float *coef4, int32_t *src, int *n_out, int device);
/* TransformToEnd (Estimator.cc:62-103): in-place motion compensation of a sweep whose intensity carries
 * ring + relative time; tf7_es = transform_es {qx,qy,qz,qw,px,py,pz}; time_factor = 10 at the call site
 * (Estimator.cc:560).  float32, device sinf/acosf: parity tolerance 2e-6 relative to the range. */
int lio_transform_to_end_host(float *cloud, int n, const float *tf7_es, float time_factor, int device);
/* Estimator::CalculateLaserOdom (Estimator.cc:1099-1360): up to max_iter rounds of CalculateFeatures +
 * 6-DoF point-to-plane Gauss-Newton (float features, double normal equations, degeneracy projection at
 * the first round) refining tf7 in place.  Outputs are sized M * (keep_features ? max_iter : 1); *iters =
 * rounds executed before the delta_r / delta_t < 0.05 exit.  Runs the estimator's own chain: without
 * keep_features each round is the batched k-NN launch plus the fused single-CTA k_odom_round, with it the
 * k-NN launch plus k_odom_reduce / k_odom_solve over all kept features. */
int lio_laser_odom_host(const float *map, int K, const float *surf, int M, float *tf7, float min_match_sq_dis,
                        float min_plane_dis, int keep_features, int max_iter, float *pts4, float *coef4, int32_t *src,
                        int *n_out, int *iters, int device);
/* Test seam of the reductions under the 6-DoF Gauss-Newton step: the A^T A (36, row-major) / A^T b (6) that one production
 * kernel stores for n features (pts4, coef4: n float4) at the transform tf7.  kernel 0..2 = k_odom_reduce in mode 0
 * (CalculateLaserOdom), 1 (scan-to-map) or 2 (MapBuilder's rotation information matrix) on `blocks` CTAs (1..1024; 0 = the
 * callers' grid max(1, min(SMs, ceil(n / 256)))); kernel 3 = the fused single-CTA k_odom_round (blocks 0 or 1) with no k-NN
 * tiles to clear.  Synchronous. */
int lio_odom_normal_equations_host(const float *pts4, const float *coef4, int n, const float *tf7, int kernel, int blocks,
                                   double *AtA, double *AtB, int device);
/* Test seam of the step itself (odom_solve_step): `rounds` steps of one chain from a cleared OdomState and the pose tf7
 * (in/out).  Round r stores AtA[36 r..] / AtB[6 r..] and the match count n_feat[r], then one thread takes the step of
 * variant 0 CalculateLaserOdom (first executed round analyses degeneracy, threshold 100, no match minimum), 1 PointMapping
 * (loop index r, rounds under 50 matches skipped, threshold 100), 2 MapBuilder (as 1, left update) or 3 PointOdometry (loop
 * index r, minimum 10, threshold 10); a finished chain (done) skips its rounds, as the callers' kernels do.  Optional outputs:
 * tf_per_round (7 per round), state_out {degenerate, done, iter}, matP (36, row-major).  Synchronous. */
int lio_odom_step_host(int rounds, const double *AtA, const double *AtB, const int *n_feat, int variant, double delta_r_abort,
                       double delta_t_abort, float *tf7, float *tf_per_round, int *state_out, float *matP, int device);

/* ---- lio::PointMapping with its rolling cube map resident in HBM (src/point_processor/PointMapping.cc) -------------------
 * The 21 x 21 x 11 cubes of 50 m (:77-82, :121-122) hold their corner / surf clouds as HBM segments; the cube directory
 * (pointer, count, capacity) is host state.  lio_pm_process_host is PointMapping::Process (:765-1052, imu_inited_ == false,
 * num_stack_frames_ == 1): associate the odometry increment (:753-756), bring the last features to the map frame and back
 * (:782-800, :1013-1016), re-centre the cube array (:809-931), select the cubes in the field of view (:944-1003), pull
 * laser_cloud_{corner,surf}_from_map_ (:1005-1011), VoxelGrid the stacks (:1016-1022), OptimizeTransformTobeMapped
 * (:325-753) and UpdateMapDatabase (:1112-1208: order-preserving insert + VoxelGrid of every valid cube).
 * transform_sum7 = transform_sum_ from the odometry (qx qy qz qw px py pz); out: transform_tobe_mapped_ and
 * info3 = {iterations, corner_from_map size, surf_from_map size}.  Cube index = i + 21 j + 441 k (PointMapping.h:150-153). */
typedef struct lio_pm lio_pm;
int lio_pm_create(int max_points, float corner_filter_size, float surf_filter_size, float min_match_sq_dis, float min_plane_dis,
                  int max_iterations, int device, void *cuda_stream, lio_pm **out);
int lio_pm_destroy(lio_pm *pm);
int lio_pm_process_host(lio_pm *pm, const float *corner_last, int nc, const float *surf_last, int ns, const float transform_sum7[7],
                        float transform_tobe_mapped7[7], int info3[3]);
int lio_pm_map_centre(lio_pm *pm, int centre3[3]);                 /* laser_cloud_cen_length_ / width_ / height_ */
/* laser_cloud_valid_idx_ and laser_cloud_surround_idx_ (the latter on publishing and map-builder handles) of the last process call,
 * n2 = their counts (<= 125 each); valid / surround may be NULL.  An attached map keeps them frozen (lio_est_attach_map). */
int lio_pm_cube_lists(lio_pm *pm, long long valid[125], long long surround[125], int n2[2]);
int lio_pm_cube_size(lio_pm *pm, int cube_index, int which, int *n);  /* which: 0 corner, 1 surf */
int lio_pm_cube_download(lio_pm *pm, int cube_index, int which, float *out_xyzi, int cap);
/* lio_pm_process_host with the clouds already in HBM, e.g. the odometry's published clouds (lio_po_clouds_dev): corner_dev / surf_dev
 * / full_dev are float4 arrays (/laser_cloud_corner_last, /laser_cloud_surf_last, /full_odom_cloud), n3_dev points to their device
 * counts int[3] {corner, surf, full}.  The counts are read and clamped on the device to n3_max, which is itself capped by max_points /
 * max_full_points; n3_max also sizes the launches, so pass tight bounds.  Same steps, outputs and host synchronisations as the host
 * entry (which is "upload, then these steps"), bit for bit.  A count above its bound returns LIO_ERR_CAPACITY once the down-sampling
 * read-back sees it; by then this call's pose association and map re-centring have already been applied, so treat the handle's pose
 * as advanced by the dropped frame.  On a handle that does not publish the full cloud is not read and its count has no bound:
 * full_dev may be NULL.  Outputs (any may be NULL): transform_tobe_mapped_, transform_aft_mapped_ (/aft_mapped_to_init; it takes
 * tobe on calls that optimised, TransformUpdate :716, and is held otherwise) and info5 = {iterations, corner_from_map size,
 * surf_from_map size, surround map published by this call, size of the last published surround map} (the last two 0 without
 * publishing).  An lio_mb handle returns LIO_ERR_INVALID.
 * Stream rule: the inputs are read by work enqueued on the mapping stream.  When the producer (e.g. lio_po_process_dev) runs on the
 * same stream nothing else is needed; otherwise the caller records an event on the producer's stream, makes the mapping stream wait
 * for it and keeps the inputs unchanged until this call returns. */
int lio_pm_process_dev(lio_pm *pm, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev,
                       const int n3_max[3], const float transform_sum7[7], float transform_tobe_mapped7[7], float transform_aft_mapped7[7],
                       int info5[5]);
/* PointMapping::PublishResults (:1210-1270) on a plain PointMapping handle: after this, every lio_pm_process_dev also publishes
 *   /laser_cloud_surround   on the first call and every num_map_frames_ (5)-th call after it (calls 1, 6, 11, ...; map_frame_count_
 *                           starts at num_map_frames_ - 1, :104): every surround cube's corner then surf cloud through
 *                           VoxelGrid(map_filter_size) (0.6, :123) - lio_mb_surround_download / lio_mb_surround_dev;
 *   /cloud_registered       the call's full cloud through PointAssociateToMap with the final transform_tobe_mapped_ (:1245-1251) -
 *                           lio_mb_full_download / lio_mb_full_dev;
 *   /aft_mapped_to_init     transform_aft_mapped_ (:1254-1262), the aft output of lio_pm_process_dev.
 * It allocates the full cloud in / registered (max_full_points float4 each) and the surround buffers of the map-builder mode, and
 * adds one synchronisation on calls that publish the surround map (its size).  Call it once, before the first process call; a later
 * call, a second call or an lio_mb handle returns LIO_ERR_INVALID.  A publishing handle rejects lio_pm_process_host (it has no full
 * cloud) with LIO_ERR_INVALID.  Without it the handle behaves as before and the lio_mb_* accessors return LIO_ERR_INVALID. */
int lio_pm_enable_publish(lio_pm *pm, float map_filter_size, int max_full_points);
/* PointMapping::UpdateMapDatabase (:1112-1208) on its own, for a caller that keeps the estimator's loop and calls it where the
 * reference's Estimator does (Estimator.cc:703-708): corner_ds / surf_ds (host, nc / ns float4 points <= max_points) are the
 * down-sampled clouds in the sensor frame, tf7 the insert pose, valid (nv <= 125 distinct cube indices) the valid list as computed
 * with the cube-array centre margin_centre3 (which may differ from the current one, lio_pm_map_centre).  Inserts every point into
 * its cube in order, then VoxelGrids every valid cube that still lies in the array, corner cubes with corner_filter_size and surf
 * cubes with surf_filter_size.  lio_pm_process_* and lio_mb_process_map_* run the same code.
 * The insert waits for the device once, plus once for every cube segment it moves to a larger one; the re-filter is one segmented
 * VoxelGrid with a launch count independent of the number of cubes, and its new cube sizes are read back without a wait in this
 * call: the next call on the handle or lio_pm_cube_size / lio_pm_cube_download wait for them (one host wait, after the call).
 * When a cube's voxel grid exceeded 2^24 voxels (a leaf below ~0.2 m for a full 50 m cube) that reader returns LIO_ERR_CAPACITY,
 * and so does every later call that reads or updates the cubes: the map is invalid and the handle must be re-created.
 * Bad arguments, an index outside [0, 4851) or a repeated index return LIO_ERR_INVALID, too many points or valid cubes
 * LIO_ERR_CAPACITY, before anything changes.  The clouds are copied before the call returns. */
int lio_pm_update_map_database_host(lio_pm *pm, const float *corner_ds, int nc, const float *surf_ds, int ns, const long long *valid, int nv,
                                    const float tf7[7], const int margin_centre3[3]);
/* The last UpdateMapDatabase on the handle (any entry): info4 = {cube jobs re-filtered, kernel launches, host waits, points inserted}.
 * The waits include the one for the re-filtered sizes that the next reader of the cubes makes. */
int lio_pm_update_stats(lio_pm *pm, int info4[4]);

/* ---- lio::MapBuilder, the global 4-D mapper (src/map_builder/MapBuilder.cc, src/map_builder_node.cc) ---------------------
 * MapBuilder derives from PointMapping; here a map-builder context is an lio_pm handle created by lio_mb_create, so
 * lio_pm_map_centre / lio_pm_cube_size / lio_pm_cube_download / lio_pm_destroy apply to it unchanged.  lio_pm_process_host on a
 * map-builder handle, and lio_mb_* on a plain lio_pm handle, return LIO_ERR_INVALID. */
typedef struct lio_mb_config {    /* MapBuilderConfig (include/map_builder/MapBuilder.h:41-48) + node parameters */
  float corner_filter_size;       /* 0.2 */
  float surf_filter_size;         /* 0.4 */
  float map_filter_size;          /* 0.2: map_builder_node.cc overrides the struct's 0.6 (down_size_filter_map_, :96) */
  float min_match_sq_dis;         /* 1.0 */
  float min_plane_dis;            /* 0.2 */
  int enable_4d;                  /* 1: Transform4DAssociateToMap + OptimizeMap; 0: the PointMapping steps (:246-251, :529-543) */
  int skip_count;                 /* 2: optimise on every skip_count-th frame (MapBuilder.cc:109-110, :529) */
  int max_iterations;             /* 10: num_max_iterations_ (PointMapping.cc:67-104) */
} lio_mb_config;
void lio_mb_default_config(lio_mb_config *cfg);   /* the node's values above */
/* MapBuilder::MapBuilder(config) + SetupRos parameters (:92-110).  max_points bounds the corner / surf clouds of one call,
 * max_full_points the full-resolution cloud.  The surround-map buffers grow on demand. */
int lio_mb_create(const lio_mb_config *cfg, int max_points, int max_full_points, int device, void *cuda_stream, lio_pm **out);
/* MapBuilder::ProcessMap (:220-622) for one matched set of the clouds and the odometry that HasNewData()
 * (PointMapping.cc:291-297) gates: corner_last / surf_last / full_cloud are /laser_cloud_corner_last, /laser_cloud_surf_last and
 * /full_odom_cloud, transform_sum7 the /laser_odom_to_init pose rounded to float as LaserOdometryHandler (PointMapping.cc:267-282)
 * does.  The first call sets bef = tobe = aft = sum (:227-232).  Then Transform4DAssociateToMap (:55-75), the PointMapping stacks,
 * re-centring, cube selection, map extraction and VoxelGrid (:286-526), the gate (:529-544: OptimizeMap on every skip_count-th
 * call, Transform4DUpdate otherwise), UpdateMapDatabase (:553-557) and PublishMapBuilderResults (:144-218).
 * Outputs (any may be NULL): transform_tobe_mapped_, transform_aft_mapped_ (/aft_4d_mapped) and
 * info6 = {iterations, gate chose optimisation, corner_from_map size, surf_from_map size, surround map published by this call,
 * size of the last published surround map}.  Synchronises the stream except for the registered full cloud's kernel. */
int lio_mb_process_map_host(lio_pm *pm, const float *corner_last, int nc, const float *surf_last, int ns, const float *full_cloud, int nf,
                            const float transform_sum7[7], float transform_tobe_mapped7[7], float transform_aft_mapped7[7], int info6[6]);
/* laser_cloud_surround_downsampled_ (:156-168, published on calls 1, 6, 11, ...): the corner then surf cloud of every cube of the
 * 5 x 5 x 5 block around the sensor (no FOV test) through VoxelGrid(map_filter_size) with one bounding box; equal to its input
 * when PCL's voxel-index overflow check fires.  The last published map stays until the next publishing call. */
int lio_mb_surround_download(lio_pm *pm, float *out_xyzi, int cap, int *n);
/* full_cloud_ after PointAssociateToMap with the final transform_tobe_mapped_ (/cloud_registered, :178-185), last call. */
int lio_mb_full_download(lio_pm *pm, float *out_xyzi, int cap, int *n);
/* Device pointers (float4) and counts of the same clouds, valid until the next lio_mb_process_map_*; stream-ordered.  The four
 * accessors also serve a publishing PointMapping handle (lio_pm_enable_publish), valid until its next lio_pm_process_dev. */
int lio_mb_surround_dev(lio_pm *pm, const float **ptr, int *n);
int lio_mb_full_dev(lio_pm *pm, const float **ptr, int *n);
/* lio_mb_process_map_host with the three clouds already in HBM, e.g. the estimator's /local/{corner,surf,full}_points publication
 * (lio_est_local_clouds_dev): corner_dev / surf_dev / full_dev are float4 arrays, n3_dev points to their counts {corner, surf, full}
 * on the device.  The counts are read and clamped on the device to n3_max, which is itself capped by max_points / max_full_points;
 * n3_max also sizes the launches, so pass tight bounds.  Same semantics, outputs and host synchronisations as the host entry (which
 * is "upload, then these steps"); the full cloud is copied with a count-guarded kernel.  A count above its bound returns
 * LIO_ERR_CAPACITY once the down-sampling read-back sees it; by then this call's pose association and map re-centring have
 * already been applied, so treat the handle's pose as advanced by the dropped frame.
 * Stream rule: the inputs are read by work enqueued on the map builder's stream.  When the producer (e.g. the estimator) runs on
 * the same stream nothing else is needed; otherwise the caller orders the two streams (an event recorded on the producer's
 * stream and waited on by the map builder's) and keeps the inputs unchanged until this call returns. */
int lio_mb_process_map_dev(lio_pm *pm, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev,
                           const int n3_max[3], const float transform_sum7[7], float transform_tobe_mapped7[7],
                           float transform_aft_mapped7[7], int info6[6]);

/* ---- lio::PointOdometry: scan-to-scan odometry of the pre-initialisation phase + the /compact_data pass-through ---------
 * (src/point_processor/PointOdometry.cc; include/point_processor/PointOdometry.h).  lio_po_create mirrors the constructor
 * PointOdometry(scan_period, io_ratio, num_max_iterations) (:66-86; defaults 0.1, 2, 25); the capacities bound the four feature
 * clouds and the full-resolution cloud of one sweep.  lio_po_process_host is Process() + PublishResults() (:294-766) for one
 * synchronised set of the five /laser_cloud_* topics (what HasNewData() :227-235 gates): the first sweep only becomes the
 * "last" clouds (:302-310); afterwards, while odometry is enabled, up to num_max_iterations rounds of corner (:338-441) and
 * surf (:443-549) matching against the last sweep + the damped 6 x 6 float Gauss-Newton (:551-664) refine transform_es_
 * (sweep end -> start), transform_sum_ accumulates its inverse (:667-669) and the less-sharp / less-flat clouds are de-skewed
 * to the sweep end (:673-674) before they replace the last clouds.  After lio_po_set_enable_odom(po, 0) - the /enable_odom
 * service the estimator calls once the IMU is initialised (:126-131) - the call is the pure pass-through: clouds swapped in,
 * transform_sum_ untouched.  Outputs (any may be NULL): transform_sum_ and transform_es_ as (qx qy qz qw px py pz),
 * info4 = {iterations executed, published (io_ratio gate :726), frame_count_, matches of the last round}.
 * lio_po_compact_data writes the /compact_data payload of the sweep just processed (:732-762, 3 + corner + surf + full points of
 * 4 floats; LIO_ERR_INVALID when the io_ratio gate did not publish it) - feed it to lio_xyzi_to_pcl32 for the PointCloud2 bytes or
 * to lio_compact_decode / lio_pm_process_host on the receiving side.  which: 0 last_corner_cloud_, 1 last_surf_cloud_,
 * 2 full_cloud_ (de-skewed when published while odometry is enabled, :728-730). */
typedef struct lio_po lio_po;
int lio_po_create(float scan_period, int io_ratio, int num_max_iterations, int max_feature_points, int max_full_points, int device,
                  void *cuda_stream, lio_po **out);
int lio_po_destroy(lio_po *po);
int lio_po_set_enable_odom(lio_po *po, int enable);
int lio_po_process_host(lio_po *po, const float *corner_points_sharp, int n_sharp, const float *corner_points_less_sharp, int n_less_sharp,
                        const float *surf_points_flat, int n_flat, const float *surf_points_less_flat, int n_less_flat,
                        const float *full_cloud, int n_full, float transform_sum7[7], float transform_es7[7], int info4[4]);
int lio_po_cloud_size(lio_po *po, int which, int *n);
int lio_po_cloud_download(lio_po *po, int which, float *out_xyzi, int cap);
int lio_po_compact_data(lio_po *po, float *out_xyzi, int cap_points, int *n_points);
int lio_po_last_launches(lio_po *po);
int lio_po_matches(lio_po *po, int kind, int32_t *out, int cap_queries);   /* test aid: indices of the last search, 2 (corner) / 3 (surf) per query */
/* lio_po_process_host with the five clouds already in HBM, e.g. stage A's outputs (lio_pp_cloud_dev / lio_pp_cloud_count_dev):
 * clouds_dev = float4 arrays {sharp, less_sharp, flat, less_flat, full} (LIO_PP_CORNER_SHARP, LIO_PP_CORNER_LESS_SHARP,
 * LIO_PP_SURF_FLAT, LIO_PP_SURF_LESS_FLAT, LIO_PP_CLOUD_IN_RINGS), n_dev = one device int per cloud with its count, n_max = host
 * bounds of the counts.  A bound above the capacities given to lio_po_create returns LIO_ERR_CAPACITY; so does a device count above
 * its bound, before anything of the handle changes (no swap, no frame_count_ increment: the call can be repeated with a correct
 * bound).  less_sharp, less_flat and full are copied into the handle by a count-guarded kernel (they are de-skewed in place and kept
 * as the last clouds), sharp and flat are read where they are during the call.  Then one read-back of the clamped counts and the
 * overflow flag, and the host entry's steps; the outputs are bit-identical to lio_po_process_host on the same clouds.  The call
 * synchronises the stream at most twice (the count read-back; the pose after the iterations when odometry runs) and not at its
 * end: what it enqueues last (the de-skew kernels) is ordered before later work on the same stream.
 * Stream rule: the inputs are read by work enqueued on the odometry's stream; share the producer's stream, or record an event on
 * the producer's stream and make the odometry's stream wait for it, and keep sharp / flat unchanged until that stream has passed
 * this call's work. */
int lio_po_process_dev(lio_po *po, const float *const clouds_dev[5], const int *const n_dev[5], const int n_max[5], float transform_sum7[7],
                       float transform_es7[7], int info4[4]);
/* The published clouds in HBM: ptr = {last_corner_cloud_, last_surf_cloud_, full_cloud_} (/laser_cloud_corner_last,
 * /laser_cloud_surf_last and the full cloud of /compact_data, the argument order of lio_pm_process_dev), *n_dev = a device int[3]
 * with their counts (stable for the life of the handle, written stream-ordered by every process call), n_host = the same counts as
 * the host knows them after the last call (exact, so tight bounds for n3_max).  The two last clouds swap buffers with the incoming
 * less_sharp / less_flat clouds, so the pointers are valid until the next process call only: fetch them after every call. */
int lio_po_clouds_dev(lio_po *po, const float *ptr[3], const int **n_dev, int n_host[3]);

/* PointMapping::OptimizeTransformTobeMapped (PointMapping.cc:325-753): scan-to-map 6-DoF float Gauss-Newton of
 * transform_tobe_mapped_ (tf7, in/out) against explicit corner / surf maps (laser_cloud_corner_from_map_ /
 * laser_cloud_surf_from_map_; the cube-map store that selects them is outside this operator).  Per round: corner matching
 * (:381-512, one feature per line), surf matching (:514-606, sign-normalised plane), skip when fewer than 50 matches
 * (:609-611), 6x6 normal equations + colPivHouseholderQr + first-round degeneracy projection + quaternion update (:613-715),
 * exit when delta_r < delta_r_abort (deg) and delta_t < delta_t_abort (cm).  Returns immediately (tf7 untouched) when
 * Kc <= 10 or Ks <= 100 (:327-329).  Optional outputs (sized Mc + Ms): the matches of the last executed round, corner
 * then surf; *iters = rounds executed.
 * variant 1 = MapBuilder::OptimizeMap (MapBuilder.cc:624-1014): the same loop with the rotation information matrix
 * J_r <- J_r R^-1 diag(5e-3, 5e-3, 1) (:905-911) and the left-multiplicative update rot = DeltaQ(x) * rot (:984-985). */
int lio_scan_to_map_host(const float *corner_map, int Kc, const float *surf_map, int Ks, const float *corner, int Mc,
                         const float *surf, int Ms, float *tf7, float min_match_sq_dis, float min_plane_dis, int max_iter,
                         double delta_r_abort, double delta_t_abort, int variant, float *pts4, float *coef4, int32_t *src,
                         int *n_out, int *iters, int device);

/* ------------------------------------------------------------------------------------------
 * fp64 factor operators — the ceres::CostFunction::Evaluate seam (SURVEY.md §8b).
 * Same contract as the reference: residuals always written, each jacobian pointer may be NULL,
 * blocks are row-major num_residuals x global_size (pose = 7 with a zero last column).
 * ---------------------------------------------------------------------------------------- */
/* PivotPointPlaneFactor::Evaluate (src/factor/PivotPointPlaneFactor.cc:43-137), one factor, host math. */
int lio_ppp_evaluate(const double point[3], const double coeff[4], const double pose_pivot[7], const double pose_i[7],
                     const double pose_ex[7], double *residual, double *J_pivot_1x7, double *J_i_1x7, double *J_ex_1x7);
/* The same operator for N factors sharing (pose_pivot, pose_i, pose_ex), evaluated on the GPU through
 * the rank-6 form used by the fused kernel: r_out[N], J_out[N][18] = [pivot(6) | i(6) | ex(6)] tangent columns. */
int lio_ppp_evaluate_batch_host(const float *pts4, const float *coef4, int n, const double pose_pivot[7],
                                const double pose_i[7], const double pose_ex[7], double *r_out, double *J_out, int device);

/* The fused stage-C reduction for ONE frame on explicit host arrays: with R9 = R_lpi (row-major), t3 = R_lpi^T P_lpi,
 * out32[0..27] = upper triangle (row-major) of S = sum_k rho'(r_k^2) [g_k;r_k][g_k;r_k]^T, out32[28] = sum_k rho(r_k^2)
 * (CauchyLoss(1.0), Estimator.cc:1664).  J^T J / J^T r of the frame's PivotPointPlaneFactors = M^T S M. */
int lio_asm_ppp_host(const float *pts4, const float *coef4, int n, const double R9[9], const double t3[3],
                     double out32[32], int device);

/* Streaming-rate measurement of the fused stage-C kernel on n synthetic features (32 B each) split over 8 frames;
 * CUDA events around each launch.  out = {avg ms / launch, min ms, algorithmic bytes / launch, launches}. */
int lio_asm_stream_bench(long long n_features, int iters, int device, double out[4]);
/* Test seam: number of TMA stages between folds of the per-thread product of (1 + r^2) into the cost accumulator of the
 * fused kernel (default 1024, i.e. one log per 2048 features and thread). */
int lio_asm_set_fold_chunks(int chunks);

/* Test seam of the device-resident solver: solves A x = b (A symmetric positive definite, n x n row-major, n <= 261) with
 * the tiled shared-memory Cholesky (n <= 216: one CTA, as k_step; 217..261: a cluster of two CTAs whose shared memory holds
 * the tiles together, as k_step_x2) (fp64 tensor-core MMA trailing update) that the dogleg step of the device solver uses
 * in place of Ceres' dense factorisation (Estimator.cc:1911 DENSE_SCHUR).  *ok = 0 when a pivot is not positive.
 * prof (optional, 4 * ceil(n / 8) + 1 entries): SM cycles per 8-column panel {panel solve, own tile update, diagonal-tile
 * factorisation, trailing update incl. barrier} as seen by the warp that runs the serial chain, then the back substitution. */
int lio_dev_cholesky_solve_host(const double *A, const double *b, int n, double *x, int *ok, long long *prof, int device);

/* Test seam of the library's resource ownership: the device and pinned host allocations, streams, events, graphs, graph execs
 * and node sub-handles currently held by every handle of the process.  Creation, enable / attach calls, a first solve's graph capture and
 * map regrowth move it; destroying a handle returns it to where it was before the handle's creation. */
long long lio_live_resources(void);
/* Test seam of the sort under every device VoxelGrid and the cube-map insert: the stable LSD radix sort of (key, value) pairs
 * by the low key_bits (1..32) bits, rounded up to whole 8-bit passes, on n host pairs; the result is read from whichever
 * buffer pair the last pass wrote.  Synchronous. */
int lio_radix_sort_pairs_host(const uint32_t *keys, const uint32_t *vals, int n, int key_bits, uint32_t *keys_out,
                              uint32_t *vals_out, int device);
/* Test seam of the segmented VoxelGrid of UpdateMapDatabase's re-filter: njobs (1..256) clouds of n_per_job[j] >= 1 points,
 * concatenated in xyzi (float4), each filtered as its own pcl::VoxelGrid with leaf_per_job[j].  out (sum of n_per_job float4)
 * receives job j's centroids at the job's own input offset, n_out_per_job[j] their count; what follows them in the job's
 * span is unspecified.  A job whose floor-space grid exceeds 2^24 voxels sets *index_bound_error and returns LIO_ERR_CAPACITY
 * without writing out.  Synchronous. */
int lio_seg_voxel_grid_host(const float *xyzi, const int *n_per_job, const float *leaf_per_job, int njobs, float *out,
                            int *n_out_per_job, int *index_bound_error, int device);
/* Test seam of the cell hash under the voxel-hash k-NN: a hash of capacity cap_points is built over map (n x float4, device count
 * n, host bound n_max >= n) with cells of edge cell_size, after an optional earlier build over prev_map (prev_n points, bound
 * prev_n) that leaves its state behind.  *eff_size = slots in use (a power of two); keys / count / start receive that many
 * entries (size them for the power of two >= max(1024, 2 * cap_points)), cellpts n float4 {x, y, z, bit-cast map index}: slot s
 * with keys[s] != ~0 holds the packed cell of the points cellpts[start[s] .. start[s] + count[s]).  Synchronous. */
int lio_cell_hash_build_host(const float *map, int n, int n_max, int cap_points, float cell_size, const float *prev_map,
                             int prev_n, int *eff_size, unsigned long long *keys, int *count, int *start, float *cellpts,
                             int device);
/* Test seam of the batched feature launch: one cell hash over map (K x float4, cells of edge cell_size), one work area sized
 * for work_queries queries, ONE launch matching nframes (1..16) frames.  Frame k: n_per_frame[k] points (consecutive in
 * surf_cat) under the grid bound n_bound_per_frame[k] >= n, transform tf7_per_frame[7k..], append_per_frame[k]; zaxis3
 * (optional, shared) replaces every frame's transformed (0, 0, 10) in the field-of-view test.  fit: 0 plane, 1 line (two
 * features per query), 2 / 3 the scan-to-map flavours.  done_flag_value: < 0 launches without a flag, else the flag's value.
 * Frame k owns out_cap_per_frame[k] consecutive entries of pts4_cat / coef4_cat / src_cat (in its frame order) and
 * count_per_frame[k]; all four are uploaded as given, so the caller sees what was and was not written.  out_cap must hold
 * the frame's initial count (when appending) plus one entry (fit 1: two) per query.  A launch plan larger than the work area
 * returns LIO_ERR_CAPACITY before anything runs.  Synchronous. */
int lio_calculate_features_batch_host(const float *map, int K, float cell_size, float min_match_sq_dis, float min_plane_dis,
                                      int nframes, const float *surf_cat, const int *n_per_frame, const int *n_bound_per_frame,
                                      const float *tf7_per_frame, const int *append_per_frame, const float *zaxis3, int fit,
                                      int done_flag_value, int work_queries, const int *out_cap_per_frame, float *pts4_cat,
                                      float *coef4_cat, int32_t *src_cat, int *count_per_frame, int device);

/* IntegrationBase (include/imu_processor/IntegrationBase.h:72-388) */
typedef struct lio_pim lio_pim;
int lio_pim_create(const double acc0[3], const double gyr0[3], const double ba[3], const double bg[3],
                   const double noise5[5] /* acc_n gyr_n acc_w gyr_w g_norm */, lio_pim **out);
int lio_pim_destroy(lio_pim *p);
int lio_pim_push_back(lio_pim *p, double dt, const double acc[3], const double gyr[3]);
/* state11 = delta_p(3) delta_q(xyzw) delta_v(3) sum_dt; jac225 / cov225 row-major 15x15 (may be NULL) */
int lio_pim_get(lio_pim *p, double *state11, double *jac225, double *cov225);
/* ImuFactor::Evaluate (include/factor/ImuFactor.h:53-167): J blocks 15x7, 15x9, 15x7, 15x9 row-major or NULL */
int lio_imu_factor_evaluate(lio_pim *p, const double pose_i[7], const double sb_i[9], const double pose_j[7],
                            const double sb_j[9], double *res15, double *J0, double *J1, double *J2, double *J3);
/* Estimator::RunInitialization (src/imu_processor/Estimator.cc:858-958) with ImuInitializer::Initialization (ImuInitializer.cc:35-308,
 * :421-452) on host arrays: the arithmetic the imu_factor = 1 estimator runs on its full window (lio_est_attach_imu_mapping).
 * W >= 5 (ApproximateGravity needs it; LIO_ERR_INVALID otherwise); laser_tf7 (W+1) x 7 float transforms (x y z w, px py pz), pims W + 1
 * handles (frame i's pre-integration ends at frame i; the excitation check reads 1..W), tlb7 transform_lb_; bas / bgs / vs (W+1) x 3,
 * R_WI9 row-major.  outcome: 0 excitation below 0.25 (nothing changes), 1 gravity norm check failed, 2 success.  With 1 and 2 the
 * reference's side effects all happen: bgs += delta_bg, pims 1..W repropagated with (0, bgs[0]) and then pims 0..W with (bas[i], bgs[i]),
 * ps / rs (row-major 3x3 each) from the laser transforms, R0 = ypr2R(-yaw, 0, 0) R_WI^T applied to ps, rs, vs, R_WI9 = R0^T and
 * g3 = R0 g_in_laser; vs is the refined velocities only on success.  A non-finite result returns LIO_ERR_NUMERIC. */
int lio_imu_run_initialization_host(int W, const float *laser_tf7, lio_pim *const *pims, const float tlb7[7], double g_norm, const double *bas,
                                    double *bgs, double *vs, double R_WI9[9], double *ps, double *rs, double g3[3], int *outcome);
/* ImuInitializer::EstimateExtrinsicRotation (src/imu_processor/ImuInitializer.cc:353-419) on host arrays: the calibration the imu_factor = 1
 * estimator runs before RunInitialization with estimate_extrinsic = 2 (lio_est_enable_extrinsic_calibration).  W >= 1; laser_tf7 and pims as
 * for lio_imu_run_initialization_host (pims 1..W are read, none is changed); tlb7 transform_lb_ in / out.  The rotation of tlb7 is overwritten
 * whether or not the call succeeds, its position never.  sv4 = the singular values of the 4W x 4 system, descending; ok = 1 iff sv4[2] > 0.25.
 * Needs no device. */
int lio_imu_estimate_extrinsic_rotation_host(int W, const float *laser_tf7, lio_pim *const *pims, float tlb7[7], double sv4[4], int *ok);

/* ------------------------------------------------------------------------------------------
 * Stages B+C+D — lio::Estimator in steady state (stage_flag_ == INITED)
 * (include/imu_processor/Estimator.h:110-170, src/imu_processor/Estimator.cc:338-427, 430-774,
 *  970-1646, 1648-2438, 2440-2666).
 * ---------------------------------------------------------------------------------------- */
typedef struct lio_est_config {   /* EstimatorConfig (Estimator.h:77-108), lidar/solver subset */
  int window_size;
  int opt_window_size;
  float min_match_sq_dis;
  float min_plane_dis;
  float surf_filter_size;
  int keep_features;
  int estimate_extrinsic;
  int opt_extrinsic;
  int imu_factor;
  int point_distance_factor;
  int prior_factor;
  int marginalization_factor;
  int enable_deskew;
  int cutoff_deskew;
  double acc_n, gyr_n, acc_w, gyr_w, g_norm;   /* IntegrationBaseConfig */
  int max_num_iterations;        /* ceres options.max_num_iterations, Estimator.cc:1916 */
  int odom_max_iterations;       /* PointMapping num_max_iterations_, PointMapping.h:171 */
  int max_frame_points;          /* capacity of one down-sampled frame cloud (surf_stack_ entry) */
  int max_scan_points;           /* capacity of the incoming laser_cloud_surf_last_ */
  int device_solver;             /* 1 (default): ImuFactor / marginalisation prior / PriorFactor evaluation, the dense normal
                                    equations, the tiled Cholesky and the dogleg controller all resident on the GPU (no host
                                    sync inside a solve; opt windows up to 16: 14..16 on a two-CTA cluster, where the device
                                    can hold one; otherwise, or with max_num_iterations > 22, the host controller);
                                    0: host controller around the fused kernel */
  int overlap_marginalization;   /* 1 (default): the Schur-complement / eigen algebra of scan k's marginalisation runs on a
                                    worker thread beside scan k+1's device front end (started at that call's entry, joined
                                    before its solve); 0: inline at the end of scan k, the reference's order.  Same result. */
  int solver_graph;              /* 1 (default): the device solver's launches of one solve are captured once as a CUDA graph
                                    and replayed per scan (single-GPU contexts); 0: plain stream launches.  Same result. */
  int init_window_factor;        /* 1 (default): with a mapping attached (imu_factor = 0), only every init_window_factor-th message
                                    is pushed before initialisation (Estimator.cc:436-439); values < 1 are refused */
} lio_est_config;

typedef struct lio_est lio_est;

void lio_est_default_config(lio_est_config *cfg);
int lio_est_create(const lio_est_config *cfg, int device, void *cuda_stream, lio_est **out);
int lio_est_destroy(lio_est *est);
/* transform_lb_ (Estimator.h:89): float {qx,qy,qz,qw,px,py,pz} */
int lio_est_set_extrinsic(lio_est *est, const float tf7[7]);
int lio_est_get_extrinsic(lio_est *est, float tf7[7]);
/* Warm start of window frame k in [0, W): state16 = P(3) Q(xyzw) V(3) Ba(3) Bg(3), the frame's own
 * down-sampled surf cloud (host), and the pre-integration ending at the frame (NULL for k = 0;
 * ownership of pim passes to the estimator). */
int lio_est_init_frame(lio_est *est, int k, const double state16[16], const float *surf_ds, int n, lio_pim *pim);
int lio_est_finish_init(lio_est *est, const double acc_last[3], const double gyr_last[3]);
/* Estimator::ProcessImu (Estimator.cc:338-427) */
int lio_est_process_imu(lio_est *est, double dt, const double acc[3], const double gyr[3], double stamp);
/* The same for n consecutive messages (dt[n], acc3[n][3], gyr3[n][3], stamp[n]) in one call: bag playback / batched drivers. */
int lio_est_process_imu_batch(lio_est *est, int n, const double *dt, const double *acc3, const double *gyr3, const double *stamp);
/* Estimator::ProcessLaserOdom, INITED branch (Estimator.cc:618-774): de-skew + VoxelGrid + SolveOptimization +
 * SlideWindow.  surf_last = laser_cloud_surf_last_ (surface_points_less_flat of the new sweep), HOST buffer.
 * Error behaviour: the window bookkeeping (pre-integration buffer, frame slots) advances before the device work, as in
 * the reference.  If a scan fails after that point (LIO_ERR_CAPACITY: down-sampled scan > max_frame_points, local map or
 * feature buffers full, voxel index overflow; LIO_ERR_NUMERIC; LIO_ERR_CUDA) the context is POISONED: every later
 * lio_est_process_scan_* call returns LIO_ERR_INVALID until the context is destroyed and re-created. */
int lio_est_process_scan_host(lio_est *est, const float *surf_last, int n);
/* ---- The same scan, phase by phase - for callers that keep the reference's control flow (Estimator::ProcessLaserOdom ->
 * SolveOptimization, Estimator.cc:618-774, 1648-2438) and only swap the heavy parts:
 *
 *   lio_est_open_scan_host / _dev   push the sweep (TransformToEnd :62-103, VoxelGrid :678-693), BuildLocalMap (:1361-1646:
 *                                   local map, k-NN + plane fit of every window frame, CalculateLaserOdom), VectorToDouble
 *                                   (:2440-2478).  The window stays "open" until lio_est_close_scan.
 *   lio_est_get_parameters          the ceres parameter blocks para_pose_ (O + 1 x 7: px py pz qx qy qz qw), para_speed_bias_
 *                                   (O + 1 x 9: v ba bg), para_ex_pose_ (7) of the open window (Estimator.h:282-284)
 *   lio_est_assemble                what ceres::Problem would evaluate at the given blocks (NULL = the estimator's own): the
 *                                   normal equations H = J^T J (n x n row-major), g = J^T r and the cost 1/2 sum rho, over
 *                                   every residual block added at :1747-1904 (ImuFactors, PivotPointPlaneFactors with
 *                                   CauchyLoss, MarginalizationFactor, PriorFactor).  n = 15 (O + 1) + 6, or 6 less while the
 *                                   extrinsic block is constant.  No gates, no step; nothing of the estimator changes.
 *   lio_est_solve                   ceres::Solve (:1989-1990) from the given blocks (in/out; NULL = the estimator's own) with
 *                                   at most max_iter iterations (<= 22 with the device solver); gates :1924-1985 included.
 *                                   summary[8] = iterations, successful steps, termination (0 no convergence / 1 convergence /
 *                                   2 failure), initial cost, final cost, evaluations, convergence_flag, extrinsic held constant.
 *   lio_est_close_scan              DoubleToVector (:2479-2568) from the given blocks (NULL = the estimator's own),
 *                                   marginalisation of the oldest frame (:2040-2275), SlideWindow (:2570-2666).
 *
 * lio_est_process_scan_* == open + solve(max_num_iterations) + close.  Errors poison the context as described above;
 * LIO_ERR_INVALID when the calls come out of order. */
int lio_est_open_scan_host(lio_est *est, const float *surf_last, int n);
int lio_est_open_scan_dev(lio_est *est, const float *surf_last_dev, const int *n_dev, int n_max);
int lio_est_get_parameters(lio_est *est, double *pose, double *speed_bias, double *ex);
int lio_est_assemble(lio_est *est, const double *pose, const double *speed_bias, const double *ex, double *H, double *g,
                     double *cost, int *n);
int lio_est_solve(lio_est *est, double *pose, double *speed_bias, double *ex, int max_iter, double summary[8]);
int lio_est_close_scan(lio_est *est, const double *pose, const double *speed_bias, const double *ex);
/* Optional: announce that the next sweep has arrived (call before stage A / lio_pp_process_*).  Starts the background
 * marginalisation algebra of the previous scan now instead of at the lio_est_process_scan_* entry, so it also overlaps
 * the feature extraction of the new sweep.  No effect with overlap_marginalization = 0. */
int lio_est_begin_scan(lio_est *est);
/* Same with the cloud already on the device (e.g. lio_pp_cloud_dev(LIO_PP_SURF_LESS_FLAT)); n is read
 * from *n_dev on the device and clamped there to n_max (n_max itself is clamped to max_scan_points). */
int lio_est_process_scan_dev(lio_est *est, const float *surf_last_dev, const int *n_dev, int n_max);
/* Device pointer to the point count of one stage-A output cloud, to chain stage A into the estimator. */
int lio_pp_cloud_count_dev(lio_pp *pp, int which, const int **n_dev);
/* ---- The estimator's /local/{corner,surf,full}_points publication, the input of lio::MapBuilder (launch/map_4D.launch remaps the map builder's
 * /laser_cloud_corner_last, /laser_cloud_surf_last, /full_odom_cloud and /laser_odom_to_init to /local/corner_points,
 * /local/surf_points, /local/full_points and /local_laser_odom).  Opt-in; while it is off nothing of the estimator changes.
 *
 *   lio_est_enable_local_clouds     allocates W + 1 corner and W + 1 full slots (corner_stack_ / full_stack_, rotated with the
 *                                   surf slots), the staging buffers and the publication buffers.  Call it once, before the
 *                                   first lio_est_init_frame; later calls return LIO_ERR_INVALID.  Not available on a sharded
 *                                   context: it returns LIO_ERR_INVALID after lio_est_set_shard / _set_peers / _set_feature_peers,
 *                                   and those return LIO_ERR_INVALID once local clouds are on.
 *   lio_est_set_scan_clouds_*       stages /laser_cloud_corner_last (stage A's LIO_PP_CORNER_LESS_SHARP) and the full cloud
 *                                   (LIO_PP_CLOUD_IN_RINGS, what the odometry pass-through carries) for the next frame push.  Each
 *                                   staged pair is consumed by exactly one push; staging again before the push replaces it.
 *                                   _host: counts above max_corner_points / max_full_points return LIO_ERR_CAPACITY and change
 *                                   nothing; the clouds are copied before the call returns (it synchronises the stream), so the
 *                                   caller's buffers may be reused at once.
 *                                   _dev: counts are read on the device and clamped there to nc_max / nf_max (themselves capped by
 *                                   the capacities); a count-guarded kernel copies the clouds into the estimator's staging buffers,
 *                                   stream-ordered on the estimator's stream: the caller's buffers may be overwritten by any work
 *                                   enqueued on that stream after this call (or after the caller has waited for it).
 *   pushes                          lio_est_init_frame(k) stores the staged clouds verbatim as frame k's pre-initialisation stack
 *                                   entries (the corner cloud is expected down-sampled, like surf_ds).  lio_est_process_scan_* /
 *                                   lio_est_open_scan_* apply the INITED rules (Estimator.cc:628-693): transform_es_ is computed
 *                                   whenever enable_deskew || cutoff_deskew; without cutoff_deskew the corner cloud goes through
 *                                   TransformToEnd(.., 10) like the surf cloud; then VoxelGrid(corner_filter_size).  The full cloud
 *                                   is pushed raw (:482) and de-skewed after the publication with TransformToEnd(.., 10,
 *                                   keep_intensity) and the scan's transform_es_ (:2416, also under cutoff_deskew).  With local
 *                                   clouds on, a push with nothing staged returns LIO_ERR_INVALID before anything advances (the
 *                                   context is NOT poisoned).  This work does not feed the solve: it runs on a stream forked after
 *                                   the surf push and joined back into the estimator's stream before SlideWindow.
 *   lio_est_local_clouds_dev        after lio_est_process_scan_* / lio_est_close_scan: the clouds SolveOptimization publishes
 *                                   (:2362-2375) - corner_stack_, surf_stack_ and full_stack_ of frame W - O + 1 before the slide,
 *                                   i.e. of the scan received O - 1 scans before the newest.  The surf cloud is that frame's OWN
 *                                   down-sampled cloud (not the accumulated slot lio_est_get_frame returns).  ptr[3] = device float4
 *                                   arrays {corner, surf, full} (the argument order of lio_mb_process_map_*), *n_dev = their device
 *                                   counts int[3], n_host[3] = their capacities (bounds to pass on as n3_max).  Pointers are stable
 *                                   for the life of the handle; the contents are valid until the next scan entry and are written by
 *                                   stream-ordered work on the estimator's stream (hand them to a map builder on the same stream,
 *                                   or order the streams).
 *   lio_est_local_clouds_download   which: 0 corner, 1 surf, 2 full; copies one of them to the host (synchronous; *n = count,
 *                                   LIO_ERR_CAPACITY when it exceeds cap).
 * Without lio_est_enable_local_clouds the accessors and lio_est_set_scan_clouds_* return LIO_ERR_INVALID. */
int lio_est_enable_local_clouds(lio_est *est, float corner_filter_size, int max_corner_points, int max_full_points);
int lio_est_set_scan_clouds_host(lio_est *est, const float *corner, int nc, const float *full, int nf);
int lio_est_set_scan_clouds_dev(lio_est *est, const float *corner_dev, const int *nc_dev, int nc_max, const float *full_dev,
                                const int *nf_dev, int nf_max);
int lio_est_local_clouds_dev(lio_est *est, const float *ptr[3], const int **n_dev, int n_host[3]);
int lio_est_local_clouds_download(lio_est *est, int which, float *out, int cap, int *n);
/* /local_laser_odom (Estimator.cc:725-742), after lio_est_process_scan_* / lio_est_close_scan: the lidar pose of window slot W - O,
 * rot = Quaterniond(Rs_[W-O] * transform_lb.rot.inverse()), pos = Ps_[W-O] - rot * transform_lb.pos in double with
 * transform_lb = transform_lb_.cast<double>(), rounded to float as the map builder's LaserOdometryHandler keeps it
 * (PointMapping.cc:267-282): tf7 = {qx,qy,qz,qw,px,py,pz}.  Works with or without local clouds. */
int lio_est_local_laser_odom(lio_est *est, float tf7[7]);
/* The two poses ProcessLaserOdom's INITED branch publishes after SlideWindow, in double as nav_msgs/Odometry carries them:
 * predict7 = /predict_laser_odom (Estimator.cc:744-758), the lidar pose of window slot W (rot = Quaterniond(Rs_.last() *
 * transform_lb.rot.inverse()), pos = Ps_.last() - rot * transform_lb.pos); local7 = /local_laser_odom (:725-742), the same at slot
 * W - O, i.e. lio_est_local_laser_odom before its rounding to float.  {qx,qy,qz,qw,px,py,pz}; either pointer may be NULL, not both. */
int lio_est_laser_odom(lio_est *est, double predict7[7], double local7[7]);
/* The global cube map after initialisation.  The reference's Estimator is a PointMapping: on every INITED scan it predicts
 * transform_tobe_mapped_ (ProcessCompactData, Estimator.cc:776-809), inserts the oldest optimised frame into the cube map
 * (UpdateMapDatabase, :703-708) and publishes (PublishResults, :721; PointMapping.cc:1210-1270).  PointMapping::Process is not run
 * (:810-812), so the cube centre, the valid and surround cube lists and transform_aft_mapped_ stay at their pre-initialisation values.
 *   lio_est_attach_map   hands the pre-initialisation map to the estimator: pm is a publishing PointMapping (lio_pm_enable_publish,
 *                        not lio_mb_create) on the estimator's device that has run at least one process call.  Call it after
 *                        lio_est_finish_init and before the first scan.  The estimator needs local clouds (the corner and full
 *                        clouds come from there), imu_factor = 1 and no sharding; the map's corner / surf leaf sizes must equal
 *                        corner_filter_size / surf_filter_size (the same members in the reference).  Any violation, a second attach
 *                        or an attach after the first scan returns LIO_ERR_INVALID before anything changes; a map whose
 *                        max_full_points is below the estimator's max_full_points returns LIO_ERR_CAPACITY.  An accumulated surf slot
 *                        holds up to max_frame_points * (W - O + 1) points: the map's insert buffers grow to that at attach.
 *                        While attached, lio_pm_process_*, lio_pm_update_map_database_host and lio_pm_destroy on pm return
 *                        LIO_ERR_INVALID; the cube accessors, lio_pm_map_centre, lio_pm_update_stats and lio_mb_surround_* /
 *                        lio_mb_full_* keep working and show the estimator's map.  lio_est_destroy releases the attachment.
 *   per scan             at the scan entry tobe = tobe * lb * (prev^-1 * curr) * lb^-1 in float Twist, prev / curr the float casts
 *                        of the states W - 1 and W (lb = transform_lb_).  After the solve, from the (O+1)-th scan on (the warm-start
 *                        frames count as mapped), UpdateMapDatabase of the clouds opt_corner_stack_ / opt_surf_stack_.first() alias:
 *                        with enable_deskew or cutoff_deskew the previous frame's (window frame W - O - 1, or the frame that has just
 *                        left the window when W == O), otherwise frame W - O's; the surf cloud as SlideWindow has accumulated it, the
 *                        corner cloud as pushed.  Pose: opt_transforms_[0] (:2279-2286), Quaterniond(Rs_[W-O] *
 *                        transform_lb.rot.conjugate().normalized()), Ps_[W-O] - rot * transform_lb.pos, cast to float.  Then the
 *                        surround map (every 5th call, counting on from the pre-initialisation calls) and /cloud_registered (the
 *                        scan's raw staged full cloud through PointAssociateToMap with the predicted tobe).  The work runs on pm's
 *                        stream, after the solve, ordered by events; the next scan entry and the next lio_est_set_scan_clouds_* wait
 *                        for it.  /cloud_registered reads the staged full cloud when the scan closes, so with a map attached
 *                        lio_est_set_scan_clouds_* inside an open scan (stepwise API) returns LIO_ERR_INVALID (not poisoning).  A failed map step poisons the estimator like any failed scan.
 *   lio_est_map_poses    after lio_est_process_scan_* / lio_est_close_scan: tobe7 = transform_tobe_mapped_, aft7 = the frozen
 *                        transform_aft_mapped_ (/aft_mapped_to_init), insert7 = the pose of the last insert, info4 = {inserted this
 *                        scan, points inserted, surround published this scan, size of the last surround map}; any pointer may be NULL.
 *                        LIO_ERR_INVALID without an attached map. */
int lio_est_attach_map(lio_est *est, lio_pm *pm);
int lio_est_map_poses(lio_est *est, float tobe7[7], float aft7[7], float insert7[7], int info4[4]);
/* ---- imu_factor = 0 from the odometry's clouds: the estimator starts itself from the mapped lidar poses, without ImuInitializer
 * (Estimator::ProcessCompactData :776-856, ProcessLaserOdom :430-774 with update_laser_imu).
 *   lio_est_attach_mapping       hands a FRESH publishing PointMapping (lio_pm_enable_publish done, no process call yet) on the estimator's
 *                                device to an imu_factor = 0 estimator with local clouds on, no sharding, leaf sizes equal to the map's,
 *                                before any lio_est_init_frame / lio_est_finish_init / scan.  Any violation returns LIO_ERR_INVALID and
 *                                changes nothing; a map whose max_full_points is below the local full capacity LIO_ERR_CAPACITY.  While
 *                                attached pm refuses the same calls as under lio_est_attach_map, and so do lio_est_process_scan_* /
 *                                open_scan_* / init_frame / finish_init on the estimator; lio_est_destroy releases pm.
 *   lio_est_process_compact_dev  one /compact_data message: corner_dev / surf_dev / full_dev / n3_dev / n3_max as lio_pm_process_dev takes
 *                                them (lio_po_clouds_dev gives them), transform_sum7 the odometry's transform_sum_.
 *                                NOT_INITED: PointMapping::Process in full (association, optimisation, UpdateMapDatabase, PublishResults);
 *                                every init_window_factor-th message then pushes the frame: transform_aft_mapped_, PointMapping's
 *                                down-sampled corner / surf stacks, the raw full cloud, the valid cube list and the cube centre.  The push
 *                                that fills the window (the (W+1)-th) sets states 0..W to trans_li * transform_lb_ (float Twist, cast to
 *                                double), switches pm to its IMU-inited mode, runs the first solve (no estimator insert or publication) and
 *                                SlideWindow.
 *                                INITED: Process without insert and publication (PointMapping.cc:784, :1033), then the INITED push rules
 *                                of lio_est_process_scan_* (with either de-skew flag the scan's own VoxelGrid of surf_last and the staged
 *                                corner, otherwise PointMapping's stacks), state W from the pushed transforms (:1670-1676), the solve with
 *                                lidar, marginalisation and prior factors, from the (O+1)-th INITED message on UpdateMapDatabase of the
 *                                oldest optimised frame with ITS saved valid list and cube centre (:703-708), PublishResults and
 *                                SlideWindow.  The IMU (lio_est_process_imu) is optional: before initialisation it propagates state
 *                                cir_buf_count_ (:379-401), afterwards state W as usual, and feeds transform_es_.
 *                                Stream rule: the inputs are read on pm's stream (Process) and on the estimator's stream, which waits for
 *                                Process.  A bound n3_max[2] above the local max_full_points, or with a de-skew flag n3_max[0] above
 *                                max_corner_points, returns LIO_ERR_CAPACITY before anything changes.  Other errors poison the
 *                                context as scans do.
 *   lio_est_process_compact_host the same from host clouds: upload into pm's input buffers, then the same steps, bit for bit.
 *   lio_est_compact_status       info4 = {inited, cir_buf_count_, frame pushed by the last call, window solved by the last call}.
 * lio_est_map_poses works in this mode; its aft7 is the live transform_aft_mapped_. */
int lio_est_attach_mapping(lio_est *est, lio_pm *pm);
int lio_est_process_compact_dev(lio_est *est, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev,
                                const int n3_max[3], const float transform_sum7[7]);
int lio_est_process_compact_host(lio_est *est, const float *corner, int nc, const float *surf, int ns, const float *full, int nf,
                                 const float transform_sum7[7]);
int lio_est_compact_status(lio_est *est, int info4[4]);
/* ---- imu_factor = 1 from the odometry's clouds and the IMU: the estimator starts itself with ImuInitializer (ProcessLaserOdom NOT_INITED
 * :505-602, RunInitialization :858-958) and then runs the lio_est_attach_map path.
 *   lio_est_attach_imu_mapping   as lio_est_attach_mapping, with imu_factor = 1 and W >= 5; estimate_extrinsic = 2 is refused unless
 *                                lio_est_enable_extrinsic_calibration was called.  Refusals return LIO_ERR_INVALID and change nothing.
 *   lio_est_process_compact_stamped_dev / _host
 *                                the compact entries with the message's header.stamp, which the 0.1 s gate between attempts (:533-536)
 *                                compares; feed the IMU samples up to that stamp before the call.  On an imu_factor = 0 mapping they
 *                                equal the unstamped entries; on an IMU mapping the unstamped entries return LIO_ERR_INVALID.
 *                                NOT_INITED: as under lio_est_attach_mapping.  The push that fills the window, and every later push
 *                                until one succeeds, runs RunInitialization when stamp - (stamp of the last attempt) > 0.1 (the first
 *                                always).  Success: the rotated states, Vs, Bgs and g_vec_ are taken, pm switches to its IMU-inited mode,
 *                                the first solve runs (no insert or publication), then SlideWindow.  Otherwise SlideWindow's state copy and
 *                                the attempt's side effects stay (see lio_imu_run_initialization_host); a non-finite result returns
 *                                LIO_ERR_NUMERIC and poisons the context.
 *                                INITED: no Process; tobe is predicted as lio_est_attach_map predicts it, the INITED push rules take the
 *                                message's clouds (without a de-skew flag PointMapping's last stacks, which no longer change), from the
 *                                (O+1)-th INITED message on the oldest optimised frame is inserted with the frozen valid list, then
 *                                PublishResults.  With a de-skew flag the caller turns its odometry into a pass-through once
 *                                lio_est_imu_init_status reports inited (lio_po_set_enable_odom(po, 0); the reference's /enable_odom).
 *   lio_est_imu_init_status      info4 = {attempts, outcome of the last (-1 none, 0 excitation, 1 gravity check, 2 success), whether the
 *                                last message ran an attempt, inited}; g3 = g_vec_, R_WI9 = R_WI_ row-major; states16 (W+1) x 16 in the
 *                                lio_est_get_states layout as the last attempt left them (on success: before the first solve; untouched
 *                                before the first attempt).  g3, R_WI9 and states16 may be NULL.
 *   lio_est_enable_extrinsic_calibration
 *                                opt-in for estimate_extrinsic = 2 (the reference's extrinsic stage 2, Estimator.cc:520-531): accepted only
 *                                on an imu_factor = 1, estimate_extrinsic = 2 context, once, before lio_est_attach_imu_mapping and before
 *                                any frame; anything else returns LIO_ERR_INVALID and changes nothing.  With it, every full-window
 *                                NOT_INITED push runs EstimateExtrinsicRotation (lio_imu_estimate_extrinsic_rotation_host) on the window,
 *                                with no stamp gate, before the gated RunInitialization, until one succeeds.  Each call overwrites the
 *                                rotation of transform_lb_ (lio_est_get_extrinsic; the position never changes), which the attempt, the
 *                                start-up states, the prediction, de-skew and the solve then use.  While no call has succeeded no
 *                                RunInitialization runs and the push ends in SlideWindow's state copy; after a success the extrinsic
 *                                stage is 1 and the same message goes on to the gate.
 *   lio_est_extrinsic_calib_status
 *                                info4 = {calibrations run, result of the last (-1 none, 0 failed, 1 success), whether the last message
 *                                ran one, current extrinsic stage}; sv4 = the last call's singular values, descending (may be NULL).
 *                                lio_est_imu_init_status's attempts count RunInitialization calls only. */
int lio_est_attach_imu_mapping(lio_est *est, lio_pm *pm);
int lio_est_enable_extrinsic_calibration(lio_est *est);
int lio_est_extrinsic_calib_status(lio_est *est, int info4[4], double sv4[4]);
int lio_est_process_compact_stamped_dev(lio_est *est, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev,
                                        const int n3_max[3], const float transform_sum7[7], double stamp);
int lio_est_process_compact_stamped_host(lio_est *est, const float *corner, int nc, const float *surf, int ns, const float *full, int nf,
                                         const float transform_sum7[7], double stamp);
int lio_est_imu_init_status(lio_est *est, int info4[4], double g3[3], double R_WI9[9], double *states16);
/* window states: (W+1) x 16 doubles (layout of state16) */
int lio_est_get_states(lio_est *est, double *out);
/* summary[32]: see lio_mapping_b200/estimator.py SUMMARY_KEYS */
int lio_est_summary(lio_est *est, double *out32);
int lio_est_feature_count(lio_est *est, int frame, int *n);
int lio_est_get_features(lio_est *est, int frame, float *pts4, float *coef4, int32_t *src, int cap);
int lio_est_map_size(lio_est *est, int *n);
int lio_est_get_map(lio_est *est, float *out, int cap);
int lio_est_frame_size(lio_est *est, int frame, int *n);
int lio_est_get_frame(lio_est *est, int frame, float *out, int cap);
int lio_est_get_local_transform(lio_est *est, int frame, float tf7[7]);
/* Marginalisation prior kept for the next solve, as normal-equation terms over the kept blocks in
 * canonical order [pose_0,sb_0,...,pose_{O-1},sb_{O-1},ex] (tangent, 15*O+6): Hp = J^T J, bp = J^T r0. */
int lio_est_prior_dim(lio_est *est, int *n);
int lio_est_get_prior(lio_est *est, double *Hp, double *bp);
/* Normal equations at the INITIAL point of the last solve (after the convergence gates; tangent order
 * [pose_0,sb_0,...,pose_O,sb_O,ex], n = 15*(O+1)+6): H n x n row-major, g n, cost. */
int lio_est_last_normal_equations(lio_est *est, double *H, double *g, double *cost, int *n);
/* Kernels launched by the last process_scan call. */
int lio_est_last_launches(lio_est *est);
/* Text of the last failed scan-level call on THIS context (lio_last_error() is per calling thread; a process that drives
 * several estimators from one thread reads the per-handle copy). */
const char *lio_est_last_error(lio_est *est);
/* Diagnostic: the device-side timeline of the last solve, stamped by the kernels themselves.  out[24][16]:
 * rows 0..11 = evaluations: [0] / [11] %globaltimer (ns) at k_step entry / exit, [1..10] SM clock at its phase boundaries (entry,
 * verdict, lidar blocks, gradient, H tiles, Cauchy scale, tiles ready, Cholesky + solve, dogleg, exit), [12] / [13] %globaltimer when
 * the first k_factors CTA starts / the last one ends, [14] when the last k_hpart CTA ends;
 * row 12 = launch counters of asm_ppp, row 13 / 14 = %globaltimer when its first CTA starts / its tail ends, one column per
 * evaluation; row 16 = SM clock inside the lidar block expansion of evaluation 2 (entry, operands staged, S M, M^T (S M)).
 * Followed by 4 * 28 + 4 entries: the per-panel profile of evaluation 1's Cholesky in the layout of
 * lio_dev_cholesky_solve_host's prof (column 1 = %globaltimer at the start of the panel's diagonal tile), and after the back
 * substitution cycles four %globaltimer stamps (entry, loop start, loop end, exit).  Opt windows 14..16 (29..33 panels) fill
 * the 116 entries with panels 0..28 and leave out the back substitution and the four stamps.  cap >= 24 * 16 + 116.  Zeros
 * when the host controller is in use.  `LIO_BENCH_TRACE=1 python bench.py` prints it. */
int lio_est_solver_trace(lio_est *est, long long *out, int cap);
/* CUDA-event timing of the fused residual+Jacobian kernel accumulated since the last reset (events recorded
 * on the estimator's stream around every launch): out[0..3] = {sum ms, launches, features processed, bytes/feature};
 * out[4..7] = the same for the frame-batched k-NN + plane-fit launch of BuildLocalMap {sum ms, launches, queries,
 * algorithmic bytes/query = 128}. */
int lio_est_kernel_profile(lio_est *est, double out[8], int reset);
/* Multi-GPU (SURVEY.md §8e): frames i with (i-1) % world == rank are matched/assembled locally; the
 * callback must sum-allreduce `count` doubles in place on the DEVICE buffer `buf` across ranks
 * (e.g. ncclAllReduce / torch.distributed.all_reduce on the estimator's stream). */
typedef int (*lio_allreduce_fn)(void *user, double *buf_dev, int count);
int lio_est_set_shard(lio_est *est, int rank, int world, lio_allreduce_fn fn, void *user);
/* Fused exchange over peer memory (preferred on one NVLink / NVSwitch node; `fn` may then be NULL in set_shard).  Every
 * rank owns one small device exchange buffer; once each rank knows the device pointers of all of them (its own, and the
 * peers' opened through CUDA IPC with lio_ipc_export / lio_ipc_open, or raw pointers when the contexts share a process),
 * the last CTA of the fused stage-C kernel stores the S blocks of the frames it owns straight into EVERY rank's buffer
 * (P2P stores) and publishes an epoch with system-scope release; a one-warp kernel on each rank acquires the epochs of
 * all ranks before the 2.5 kB result goes to the host.  No collective call, no extra pass over the data. */
int lio_est_exchange_buffer(lio_est *est, void **dev_ptr, size_t *bytes);
int lio_est_set_peers(lio_est *est, int world, void *const *peer_ptrs /* [world], entry [rank] ignored */);
/* Per-scan feature exchange (preferred on one NVLink / NVSwitch node).  After lio_est_set_shard(rank, world, NULL, NULL) each rank
 * still matches only the frames it owns, but copies their features (xyz + score, coefficients, count) into the same place of every
 * peer's feature slab with P2P stores and publishes the scan's epoch; once all epochs have arrived every rank holds ALL frames'
 * features and runs the complete solve exactly like a single-GPU context (one rendezvous per scan instead of one per evaluation, the
 * solve graph stays in use).  lio_est_feature_slab returns this context's slab (all feature buffers of both scan parities, the
 * counts and the epoch flags are ONE allocation: export it with lio_ipc_export); lio_est_set_feature_peers takes every rank's slab
 * as mapped in this process (entry [rank] ignored).  Replaces a previous lio_est_set_peers; LIO_ERR_INVALID inside an open scan. */
int lio_est_feature_slab(lio_est *est, void **dev_ptr, size_t *bytes);
int lio_est_set_feature_peers(lio_est *est, int world, void *const *peer_slabs /* [world], entry [rank] ignored */);
int lio_ipc_export(const void *dev_ptr, unsigned char handle[64]);      /* cudaIpcGetMemHandle */
int lio_ipc_open(const unsigned char handle[64], void **dev_ptr);       /* cudaIpcOpenMemHandle, lazy peer access */
int lio_ipc_close(void *dev_ptr);
/* Owner rank of window frame pivot+frame_rel (frame_rel = 1..O) under `world` ranks: (frame_rel-1) % world. */
int lio_est_frame_owner(int frame_rel, int world);

/* ------------------------------------------------------------------------------------------
 * /compact_data wire format (host only; no device needed).  Encoder PointOdometry.cc:732-762, decoder
 * PointMapping::CompactDataHandler PointMapping.cc:171-238: point 0 = transform_sum_.pos, point 1 = quaternion
 * (x, y, z | intensity = w), point 2 = (corner_size, surf_size, full_size) as floats, then corner || surf || full.
 * Clouds are packed (x, y, z, intensity) float4; tf7 = {qx,qy,qz,qw,px,py,pz}.
 * ---------------------------------------------------------------------------------------- */
/* out_xyzi sized cap_points float4; *n_points = 3 + nc + ns + nf.  LIO_ERR_CAPACITY when a size is >= 2^24 (not exact as
 * a float) or the output is too small. */
int lio_compact_encode(const float tf7[7], const float *corner, int nc, const float *surf, int ns, const float *full, int nf,
                       float *out_xyzi, int cap_points, int *n_points);
/* Header check of the decoder (:180-195): LIO_ERR_INVALID when n_points < 4 or 3 + sizes != n_points. */
int lio_compact_sizes(const float *xyzi, int n_points, int sizes[3]);
/* corner / surf / full sized by lio_compact_sizes. */
int lio_compact_decode(const float *xyzi, int n_points, float tf7[7], float *corner, float *surf, float *full);
/* packed float4 <-> the 32-byte pcl::PointXYZI records a sensor_msgs/PointCloud2 of this type carries
 * (x, y, z at 0/4/8, data[3] = 1.0f, intensity at 16). */
int lio_xyzi_to_pcl32(const float *xyzi, int n, uint8_t *out32);
int lio_pcl32_to_xyzi(const uint8_t *in32, int n, float *xyzi);

/* ------------------------------------------------------------------------------------------
 * The map of a whole drive (src/save_bag_to_pcd.cc): the registered clouds accumulated in HBM, written as one PCD.
 * ---------------------------------------------------------------------------------------- */
/* save_bag_to_pcd.cc appends every /cloud_registered message to one cloud (`map_points += transformed_cloud`, :111-115; its
 * transform is the identity, :95-109) and writes it with pcl::PCDWriter::writeBinary (:156-160).  An lio_rm handle does the same
 * in HBM, one insert per publishing step:
 *   leaf == 0   raw mode, the tool's behaviour: the concatenation of every inserted point in insert order, non-finite points kept;
 *               capacity counts points.
 *   leaf > 0    voxel mode; capacity counts voxels.  A point's voxel is (int64) floorf(c * (1.0f / leaf)) per axis in float32
 *               (PCL's VoxelGrid arithmetic without its 32-bit voxel index).  Points with a non-finite x, y or z, or a voxel
 *               coordinate outside [-2^20, 2^20), are dropped.  Each voxel keeps fp64 sums of x, y, z, intensity and a count, and
 *               every point is added to them one at a time in arrival order (insert order, then index in the cloud): the sums
 *               equal np.add.at on float64 arrays.  A voxel's id is given when its first point arrives.
 * The handle owns HBM for the map (raw: 16 B per point; voxel: about 80 B per voxel) and grows its per-insert scratch with
 * stream-ordered allocations.  All work runs on cuda_stream (0 = the legacy default stream).
 * Bad arguments return LIO_ERR_INVALID (voxel mode takes capacity <= 2^30), no device LIO_ERR_NO_DEVICE. */
typedef struct lio_rm lio_rm;
int lio_rm_create(float leaf, long long capacity, int device, void *cuda_stream, lio_rm **out);
int lio_rm_destroy(lio_rm *rm);
/* Insert one cloud of n float4 {x, y, z, intensity} (save_bag_to_pcd.cc:111-115).  _dev takes a device array and the host count,
 * e.g. what lio_mb_full_dev returns on a publishing lio_pm, a map-builder handle or the map attached to an estimator.  It is
 * stream-ordered on the handle's stream and never waits on the host: the cloud is written by stream-ordered work on the mapping's
 * stream, so create the handle on that stream or order the two streams with an event.  Work enqueued on the handle's stream after
 * the call may reuse the caller's buffer.  _host copies a host array before it returns.
 * An insert that would exceed the capacity changes nothing and sets a sticky overflow flag; every later insert is then a no-op
 * until lio_rm_reset.  A voxel-mode insert is 17 stream operations whatever n is (one more for the upload of _host), a raw-mode
 * insert one copy. */
int lio_rm_insert_dev(lio_rm *rm, const float *xyzi_dev, int n);
int lio_rm_insert_host(lio_rm *rm, const float *xyzi, int n);
/* out8 = {insert calls, points offered by them, map size (points or voxels), overflow flag, points accepted, points dropped (voxel
 * mode: non-finite or out of range), host waits of the handle so far (this call's included), stream operations of the last insert}.
 * Synchronises the handle's stream. */
int lio_rm_stats(lio_rm *rm, long long out8[8]);
/* The map as float4, raw points in insert order or voxels in id order as float(sum / count) per channel.  _dev synchronises for
 * the size, then gathers into a stable export buffer on the stream; the pointer is valid until the next insert or reset.
 * _download copies it to out (cap float4 records; LIO_ERR_CAPACITY with *n set when the map is larger). */
int lio_rm_export_dev(lio_rm *rm, const float **ptr, long long *n);
int lio_rm_download(lio_rm *rm, float *out_xyzi, long long cap, long long *n);
/* Empties the map and clears the overflow flag (stream-ordered); the counters of lio_rm_stats keep counting. */
int lio_rm_reset(lio_rm *rm);
/* A binary PCD v0.7 file in the layout pcl::PCDWriter::writeBinary gives pcl::PointXYZI (save_bag_to_pcd.cc:156-160), restated
 * from PCL's published format: the header lines "# .PCD v0.7 - Point Cloud Data file format", "VERSION 0.7",
 * "FIELDS x y z intensity", "SIZE 4 4 4 4", "TYPE F F F F", "COUNT 1 1 1 1", "WIDTH n", "HEIGHT 1", "VIEWPOINT 0 0 0 1 0 0 0",
 * "POINTS n", "DATA binary", each ended by '\n', then n records of 16 bytes (x, y, z, intensity; no padding fields).
 * lio_pcd_write_xyzi is host only and needs no device; a path that cannot be written returns LIO_ERR_INVALID. */
int lio_pcd_write_xyzi(const char *path, const float *xyzi_host, long long n);
int lio_rm_write_pcd(lio_rm *rm, const char *path);

/* ------------------------------------------------------------------------------------------
 * lio_node — lio_processor_node + lio_estimator_node (src/processor_node.cc, src/estimator_node.cc; the graph of the
 * launch/test_*.launch files) as one device-resident handle: raw sweeps and IMU messages in, everything else inside.
 * ---------------------------------------------------------------------------------------- */
/* The pairing the reference's measurement thread runs, as a host seam that needs no device.  Arrivals i = 0..n-1 in order: kind[i] 0 an
 * IMU message (stamp[i], acc3 / gyr3 row i), 1 a /compact_data message (stamp[i]; its acc / gyr rows are ignored).  After every arrival
 * MeasurementManager::GetMeasurements (MeasurementManager.cc:54-108, enable_imu = true as MeasurementManager.h:79 leaves it) runs until it
 * waits:
 *   - an IMU message not later than the last accepted one is dropped and counted (ImuHandler :110-116);
 *   - it waits while the newest IMU stamp <= front stamp + msg_time_delay, drops the front message while the oldest IMU stamp >= its stamp
 *     + delay, and otherwise pops it with every IMU message stamped < stamp + delay, then appends the next IMU message WITHOUT popping it;
 *   - each released message runs Estimator::ProcessEstimation's loop (Estimator.cc:2682-2736) with curr_time_ kept across messages from -1:
 *     a sample at or before stamp + delay is integrated with dt = t - curr_time_; the one after it is replaced by w1 * previous + w2 * sample
 *     (dt_1 = laser - curr, w1 = dt_2 / (dt_1 + dt_2), w2 = dt_1 / (dt_1 + dt_2), no FP contraction) with dt = dt_1.  Every call carries the
 *     IMU message's own stamp.  A sample stamped exactly at stamp + delay is integrated, stays queued and is integrated again with dt = 0
 *     at the start of the next message.
 * Outputs: calls8 = the ProcessImu calls {dt, acc xyz, gyr xyz, stamp} (cap_calls rows); events3 = one row per decided message in decision
 * order {arrival index, 1 processed / 0 dropped, index of its first call}; imu_dropped = out-of-order IMU messages.  Messages still waiting at
 * the end have no row.  LIO_ERR_CAPACITY when a capacity is too small. */
int lio_measure_replay(double msg_time_delay, int n, const int *kind, const double *stamp, const double *acc3, const double *gyr3,
                       double *calls8, int cap_calls, int *n_calls, int *events3, int cap_events, int *n_events, int *imu_dropped);

typedef struct lio_node_config {
  int sensor_type;                /* 16, 32, 64 or 320: the presets of processor_node.cc:66-74 (VLP-16 -15..15 deg, HDL-32 -30.67..10.67,
                                     HDL-64 -24.9..2, 320 = RS-32 -25..15 with the ring field of every point) */
  lio_pp_config pp;               /* PointProcessorConfig; lower_bound / upper_bound / num_rings come from sensor_type */
  int odom_io;                    /* odom_io (estimator_node.cc:145-147): PointOdometry(0.1, odom_io)'s io_ratio */
  double msg_time_delay;          /* msg_time_delay (estimator_node.cc:138-139) */
  lio_est_config est;             /* the EstimatorConfig subset; imu_factor picks the start-up, estimate_extrinsic = 2 calibrates */
  float tf_lb7[7];                /* transform_lb_ {qx,qy,qz,qw,px,py,pz} (extrinsic_rotation / extrinsic_translation) */
  float corner_filter_size;       /* PointMapping leaves (corner_filter_size / surf_filter_size: surf must equal est.surf_filter_size) */
  float surf_filter_size;
  float map_filter_size;          /* the surround map's leaf */
  int max_points;                 /* capacity of one raw sweep (and of the full cloud) */
  int max_feature_points;         /* capacity of one feature cloud of a sweep (odometry, mapping, the local corner cloud) */
  int max_pending;                /* depth of the /compact_data queue: published messages waiting for their IMU */
} lio_node_config;
typedef struct lio_node lio_node;
typedef struct lio_node_status {
  long long sweeps;               /* sweeps run through stage A and the odometry */
  long long published;            /* /compact_data messages the io_ratio gate published (PointOdometry.cc:725) */
  long long processed;            /* messages paired and processed by the estimator */
  long long dropped;              /* messages the pairing dropped (no IMU before stamp + delay, MeasurementManager.cc:73-78) */
  long long imu_dropped;          /* IMU messages dropped as out of order (MeasurementManager.cc:111-114) */
  int pending;                    /* messages waiting for IMU */
  int odom_enabled;               /* 0 once the /enable_odom call has switched the odometry to its pass-through */
  int inited;                     /* the estimator's stage is INITED */
  int poisoned;                   /* an estimator failure poisoned the node */
  double last_stamp;              /* header.stamp of the last processed message (-1 before the first) */
} lio_node_info;
void lio_node_default_config(lio_node_config *cfg);
/* Creates lio_pp (sensor preset), lio_po (scan period 0.1, odom_io, 25 iterations), a publishing lio_pm (the YAML's leaves, 10 iterations,
 * min_match_sq_dis / min_plane_dis of est) and an estimator with local clouds on, all on cuda_stream; sets tf_lb7, calls
 * lio_est_enable_extrinsic_calibration when imu_factor = 1 and estimate_extrinsic = 2 (Estimator.cc:520-531), then attaches the mapping
 * with lio_est_attach_imu_mapping (imu_factor = 1) or lio_est_attach_mapping (imu_factor = 0), and allocates max_pending queue slots in
 * HBM.  A refusal of any inner create / attach is returned as its status, and nothing stays allocated. */
int lio_node_create(const lio_node_config *cfg, int device, void *cuda_stream, lio_node **out);
int lio_node_destroy(lio_node *node);
/* One IMU message (ImuHandler): dropped and counted when not later than the last accepted one; then every message that GetMeasurements now
 * releases is processed, in order (see lio_node_push_sweep_dev).  _batch: n messages, stamp[n], acc3 / gyr3 n x 3. */
int lio_node_push_imu(lio_node *node, double stamp, const double acc[3], const double gyr[3]);
int lio_node_push_imu_batch(lio_node *node, int n, const double *stamp, const double *acc3, const double *gyr3);
/* One raw sweep (xyzi n x float4, rings n x uint16 - required with sensor_type 320, refused otherwise - and its stamp): stage A
 * (lio_pp_process_dev / lio_pp_process_dev_ring), then lio_po_process_dev.  When the io_ratio gate publishes (PointOdometry.cc:725-727) the
 * three clouds are copied, count-guarded, into a queue slot in HBM with transform_sum_, their host counts and the stamp; then the pairing
 * runs as after an IMU push.  Processing one message: its ProcessImu calls (lio_est_process_imu), then lio_est_process_compact_stamped_dev
 * on the slot.  When that message initialised an imu_factor = 1 estimator and enable_deskew or cutoff_deskew is set, the node turns the
 * odometry into its pass-through (lio_po_set_enable_odom(po, 0), the /enable_odom call of Estimator.cc:542-560, made only on the
 * RunInitialization success path: the imu_factor = 0 start-up, :505-517, leaves the odometry on).  It takes effect from the next sweep,
 * exactly once; the reference's service call is asynchronous, so there the switch lands at a sweep that depends on thread timing.
 * Refusals, before anything changes: a sweep the gate would publish while max_pending messages wait returns LIO_ERR_CAPACITY, n above
 * max_points LIO_ERR_CAPACITY, rings on the wrong sensor type LIO_ERR_INVALID.  Inner failures return their status; an estimator failure
 * poisons the node as it poisons the estimator: every later push returns LIO_ERR_INVALID.
 * Waits: the odometry's one or two (lio_po_process_dev) and the estimator's per processed message; the node adds none to the device
 * entry.  _dev is stream-ordered (the caller's buffers are read by work on the stream); _host uploads, runs the same and synchronises once. */
int lio_node_push_sweep_dev(lio_node *node, const float *xyzi_dev, const uint16_t *rings_dev, int n, double stamp);
int lio_node_push_sweep_host(lio_node *node, const float *xyzi, const uint16_t *rings, int n, double stamp);
int lio_node_status(lio_node *node, lio_node_info *status);
/* The inner handles, for the existing getters and _dev accessors (lio_est_get_states, lio_est_map_poses, lio_est_imu_init_status,
 * lio_est_extrinsic_calib_status, lio_est_local_clouds_dev, lio_mb_surround_dev / lio_mb_full_dev for lio_rm_insert_dev, lio_pp_cloud_dev,
 * ...).  Their process, set-up, attach and destroy entries must not be called: the node owns them.  Any pointer may be NULL. */
int lio_node_handles(lio_node *node, lio_pp **pp, lio_po **po, lio_est **est, lio_pm **pm);

/* ---- map_4D.launch / map_4D_indoor.launch beside the node: map_builder_node (src/map_builder_node.cc) on the estimator's /local
 * clouds, and save_bag_to_pcd (src/save_bag_to_pcd.cc) on a /cloud_registered topic.
 *   lio_node_enable_map_builder     creates an lio_mb handle (lio_mb_create with cfg; lio_mb_default_config holds the values of both
 *                                   launch files: compact_data false, enable_4d true, map_filter_size 0.2 from map_builder_node.cc) on the
 *                                   node's device and stream, sized from lio_est_local_clouds_dev's capacities: max_points = max(corner,
 *                                   surf), max_full_points = full.  Only once and only before the first sweep; otherwise LIO_ERR_INVALID
 *                                   and nothing changes.  A refusal of lio_mb_create is returned as its status.
 *   which messages                  map_builder_node runs ProcessMap when HasNewData() (PointMapping.cc:291-297) sees its four topics new
 *                                   with stamps within 5 ms.  The three clouds are published by SolveOptimization (Estimator.cc:2355-2375,
 *                                   stamp Headers_[pivot+1]); /local_laser_odom only in the INITED branch of ProcessLaserOdom (:725-742,
 *                                   the same stamp: SlideWindow does not move Headers_, :441 / :2650).  The start-up solve (:575 with
 *                                   imu_factor = 1, :505-517 with imu_factor = 0) publishes clouds without /local_laser_odom, and the next
 *                                   message's clouds replace them.  So the map builder runs once for every message that reaches the
 *                                   estimator already INITED: after that message's successful estimator call, lio_est_local_clouds_dev and
 *                                   lio_est_local_laser_odom go to lio_mb_process_map_dev on the node's stream; then its pose row is kept.
 *                                   The reference's map builder is a separate process whose subscriber queues hold 2 messages, so under
 *                                   load it can skip sets, depending on thread timing; the node processes every set, in order, on its
 *                                   one stream.  The call adds the map builder's own host waits (lio_mb_process_map_dev) to the message.
 *                                   A map builder failure poisons the node as an estimator failure does; note that lio_mb_process_map_dev
 *                                   can return LIO_ERR_CAPACITY after it has advanced the handle's pose.
 *   lio_node_map_builder            the lio_mb handle, for lio_pm_map_centre, the cube accessors, lio_mb_surround_* and lio_mb_full_*.
 *                                   Its process and destroy entries must not be called (as for lio_node_handles).  LIO_ERR_INVALID
 *                                   without a map builder.
 *   lio_node_map_builder_poses      the drive's 4-D trajectory, one row per map builder call in call order: stamp = the set's header stamp
 *                                   (Headers_[pivot+1]: the message pushed O - 1 pushes before the newest), tobe7 = transform_tobe_mapped_,
 *                                   aft7 = transform_aft_mapped_ (/aft_mapped_to_init of PublishMapBuilderResults, MapBuilder.cc:186-200),
 *                                   info6 as lio_mb_process_map_*.  Kept on the host.  *n = the number of rows; LIO_ERR_CAPACITY and
 *                                   nothing copied when it exceeds cap.  Any array may be NULL.  LIO_ERR_INVALID without a map builder.
 *   lio_node_attach_registered_map  every cloud that source publishes is inserted into rm with lio_rm_insert_dev, stream-ordered (no host
 *                                   wait), in publication order.  LIO_NODE_MAP_ESTIMATOR: the estimator's PointMapping /cloud_registered,
 *                                   save_bag_to_pcd's default topic (:66).  It publishes once per processed message: PointMapping::Process
 *                                   publishes on the messages that arrive NOT INITED (the start-up message included: Process runs before
 *                                   SetInitFlag, :544, and the start-up solve runs no PublishResults), PublishResults (:721) on the messages
 *                                   that arrive INITED (Process skips it there, PointMapping.cc:1033, or is not run, :810-812).
 *                                   LIO_NODE_MAP_BUILDER: the map builder's cloud_registered (MapBuilder.cc:113, :178-185), once per map
 *                                   builder call; it needs lio_node_enable_map_builder first.  rm must be on the node's device and stream,
 *                                   attached once, and must outlive the node (there is no detach).  A full map sets rm's sticky overflow
 *                                   flag and does not fail the node.  Refusals (an unknown source, the map builder's source without a map
 *                                   builder, another device or stream, an rm attached already, a poisoned node) return LIO_ERR_INVALID and
 *                                   change nothing. */
enum { LIO_NODE_MAP_ESTIMATOR = 0, LIO_NODE_MAP_BUILDER = 1 };
int lio_node_enable_map_builder(lio_node *node, const lio_mb_config *cfg);
int lio_node_map_builder(lio_node *node, lio_pm **mb);
int lio_node_map_builder_poses(lio_node *node, double *stamp, float *tobe7, float *aft7, int *info6, int cap, int *n);
int lio_node_attach_registered_map(lio_node *node, lio_rm *rm, int source);

/* ---- The node's odometry topics: every pose the processor and estimator nodes publish, one row per publication, kept in host queues
 * that the caller drains.  One push can release several messages and each message makes many ProcessImu calls, so the getters above
 * (lio_est_get_states, lio_est_map_poses) only show the last of them; these queues keep every one.
 *   lio_node_enable_odometry  opt-in: one queue per topic, each of capacity rows; a push onto a full queue drops its oldest row (a ROS
 *                             publisher queue's behaviour, which bounds memory for a caller that never drains).  Only once, only before
 *                             the first sweep, capacity >= 1 and not on a poisoned node; otherwise LIO_ERR_INVALID and nothing changes.
 *                             Without it the node records nothing.  Recording reads host state only: no launch, no copy, no host wait.
 *   row layout                16 doubles for every topic: [0] stamp, [1..7] tf7 {qx,qy,qz,qw,px,py,pz}, [8..14] the topic's extras
 *                             (zero where it has none), [15] seq, the topic's publication count from 1 (a dropped row leaves a gap).
 *                             Float sources are widened exactly, as nav_msgs/Odometry carries double.
 *   topic                     publisher (reference), when, pose, extras, stamp:
 *   LASER_ODOM_TO_INIT        PointOdometry::PublishResults (PointOdometry.cc:685-704): every odometry call but the first sweep's, which
 *                             returns at :302-310; the pass-through after /enable_odom false still reaches :681.  transform_sum_;
 *                             extras = transform_es_ (tf7, /laser_odom_to_last, :712-721); the sweep's stamp.
 *   AFT_MAPPED_TO_INIT        PointMapping::PublishResults (PointMapping.cc:1255-1276): once per processed message (Process before
 *                             INITED, decimated messages included; Estimator.cc:721 after; the rule of LIO_NODE_MAP_ESTIMATOR above).
 *                             transform_aft_mapped_ (lio_est_map_poses aft7); the message's stamp (time_laser_odometry_, :230).
 *   PREDICT_ODOM              Estimator::ProcessImu (Estimator.cc:406-425): after every ProcessImu call of a message that arrived INITED
 *                             (not the start-up message's calls).  Ps_.last(), Quaterniond(Rs_.last()) (row W of lio_est_get_states);
 *                             extras = Vs_.last() then Bas_.last() (the reference's twist.angular); the IMU message's stamp the call
 *                             carries (:2706, :2725).
 *   PREDICT_LASER_ODOM        ProcessLaserOdom, INITED branch after SlideWindow (:744-758), outside the opt_point_coeff_map_ size check:
 *                             every message that arrives INITED.  lio_est_laser_odom predict7; the message's stamp.
 *   LOCAL_LASER_ODOM          the same block (:725-742), the same messages.  lio_est_laser_odom local7; Headers_[pivot + 1] (the stamp of
 *                             lio_node_map_builder_poses).
 *   EXTRINSIC_LB              SolveOptimization's update_laser_imu block (:2279-2433, publish :2343-2353; every shipped YAML sets
 *                             update_laser_imu): after every solve the estimator records (lio_est_compact_status info4[3]): the start-up
 *                             solve (:505-517 with imu_factor = 0, :575 with imu_factor = 1) and every INITED solve.
 *                             transform_lb_.cast<double>() after DoubleToVector (lio_est_get_extrinsic); Headers_.last().
 *   lio_node_take_odometry    copies the min(cap, queued) oldest rows of topic into rows16 (16 doubles each), removes them, *n = the
 *                             rows copied, *left (may be NULL) = the rows still queued.  Unknown topic, cap < 0 or no
 *                             lio_node_enable_odometry: LIO_ERR_INVALID and nothing removed.  Works on a poisoned node. */
enum {
  LIO_NODE_ODOM_LASER_ODOM_TO_INIT = 0,   /* /laser_odom_to_init */
  LIO_NODE_ODOM_AFT_MAPPED_TO_INIT = 1,   /* /aft_mapped_to_init */
  LIO_NODE_ODOM_PREDICT_ODOM = 2,         /* /predict_odom */
  LIO_NODE_ODOM_PREDICT_LASER_ODOM = 3,   /* /predict_laser_odom */
  LIO_NODE_ODOM_LOCAL_LASER_ODOM = 4,     /* /local_laser_odom */
  LIO_NODE_ODOM_EXTRINSIC_LB = 5,         /* /extrinsic_lb */
  LIO_NODE_ODOM_TOPICS = 6
};
int lio_node_enable_odometry(lio_node *node, int capacity);
int lio_node_take_odometry(lio_node *node, int topic, double *rows16, int cap, int *n, int *left);

/* ------------------------------------------------------------------------------------------
 * Dense fp64 kernels of the host shell (host only; test seams).
 * ---------------------------------------------------------------------------------------- */
/* Lower Cholesky A = L L^T (blocked, the factorisation behind every dogleg step: Ceres DENSE_SCHUR at n <= 261,
 * Estimator.cc:1909-1921) and the solve A x = b.  A n x n row-major symmetric (lower triangle read); L_out optional
 * (n x n, upper triangle zeroed).  LIO_ERR_NUMERIC when A is not positive definite. */
int lio_host_cholesky_solve(int n, const double *A, const double *b, double *L_out, double *x);
/* Symmetric eigen-decomposition (Eigen::SelfAdjointEigenSolver call sites MarginalizationFactor.cc:276, :293):
 * ascending eigenvalues, eigenvectors in the COLUMNS of evecs (n x n row-major).  threads > 1 applies the QL rotations
 * on disjoint row ranges in parallel (bit-identical result). */
int lio_host_sym_eigen(int n, const double *A, double *evals, double *evecs, int threads);
/* The trust-region / traditional-dogleg controller that stands in for ceres::Solve (options of Estimator.cc:1909-1921,
 * Ceres 1.14 defaults otherwise) on a toy nonlinear least-squares problem assembled on the host:
 * r_k = a_k . x + amp sin(b_k . x) - y_k  (A, B: m x n row-major), optional CauchyLoss(1.0) with the Ceres corrector.
 * x in/out; summary[8] = {iterations, successful steps, termination (0 no convergence, 1 convergence, 2 failure),
 * initial cost, final cost, evaluations}. */
int lio_host_dogleg_toy(int n, int m, const double *A, const double *B, const double *y, double amp, int use_cauchy, double *x,
                        int max_iter, double *summary);

#ifdef __cplusplus
}
#endif
#endif /* LIO_B200_H_ */
