// lio::PointMapping's rolling cube map and its Process() step (pre-initialisation scan-to-map path) with the map resident in
// HBM - SURVEY section 8 row f2.  Reference: src/point_processor/PointMapping.cc
//   constants / ToIndex        :77-82, :121-122, include/point_processor/PointMapping.h:150-159   (21 x 21 x 11 cubes of 50 m)
//   re-centring                :809-931      cube descriptors are shifted on the host: no point moves in HBM
//   cube selection             :944-1003     5 x 5 x 5 neighbourhood, FOV test on the eight cube corners (host, <= 125 cubes)
//   map extraction             :1005-1011    one gather kernel over the valid cubes' HBM segments
//   Process                    :765-1052     PointAssociateToMap / TobeMapped kernels, VoxelGrid of the stacks,
//                                            OptimizeTransformTobeMapped (scan_to_map_run: voxel-hash k-NN + 6 x 6 float GN)
//   UpdateMapDatabase          :1112-1208    order-preserving insert (cube keys, stable sort and append positions on the device,
//                                            one wait for the touched cubes) + one segmented VoxelGrid of every valid cube
//                                            (voxel.cu SegVoxelGrid); also an entry of its own, lio_pm_update_map_database_host
//   PublishResults             :1210-1270    after lio_pm_enable_publish: the map-builder mode's surround map (every 5th call) and
//                                            registered full cloud, shared with PublishMapBuilderResults (pm_publish)
// Host entries upload into the context's own buffers and run the same steps as the device entries (lio_pm_process_dev,
// lio_mb_process_map_dev), whose clouds and counts stay in HBM.
// lio::MapBuilder::ProcessMap (src/map_builder/MapBuilder.cc:220-622) is the same context in map-builder mode (lio_mb_*):
//   Transform4DAssociateToMap  :55-75       yaw-only correction of the odometry rotation (host, once per frame)
//   optimisation gate          :529-544     OptimizeMap = scan_to_map_run variant 1 on every skip_count-th frame
//   PublishMapBuilderResults   :144-218     surround map (k_gather_segments over <= 250 cube segments + VoxelGrid) every 5th
//                                            frame, registered full cloud (k_associate mode 0) every frame
// Per-point work runs in kernels; the 4851-entry cube directory (pointer, count, capacity per cube) lives on the host and is
// the only thing the control logic touches.  Compiled with -fmad=false: the float expressions follow the reference's order,
// clouds, cube contents and the mapped pose are compared with the oracle (oracle/o_cubemap.cc; the map-builder mode with oracle/o_mapbuilder.cc).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <new>
#include <vector>
#include "odom.cuh"
#include "voxel.cuh"
#include "cubemap.cuh"

namespace lio {

constexpr int kCubeL = 21, kCubeW = 21, kCubeH = 11, kCubes = kCubeL * kCubeW * kCubeH;

// q * v (Eigen _transformVector) in float, host copy of the device expression
static void rotate_host(const TwistF &t, float vx, float vy, float vz, float &ox, float &oy, float &oz) {
  volatile float ux = t.qy * vz - t.qz * vy, uy = t.qz * vx - t.qx * vz, uz = t.qx * vy - t.qy * vx;
  volatile float ux2 = ux + ux, uy2 = uy + uy, uz2 = uz + uz;
  volatile float cx = t.qy * uz2 - t.qz * uy2, cy = t.qz * ux2 - t.qx * uz2, cz = t.qx * uy2 - t.qy * ux2;
  volatile float ax = ux2 * t.qw, ay = uy2 * t.qw, az = uz2 * t.qw;
  volatile float rx = vx + ax, ry = vy + ay, rz = vz + az;
  ox = rx + cx; oy = ry + cy; oz = rz + cz;
}

// ---- kernels ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void rotate_dev(float qx, float qy, float qz, float qw, float vx, float vy, float vz, float &ox, float &oy, float &oz) {
  float ux = qy * vz - qz * vy, uy = qz * vx - qx * vz, uz = qx * vy - qy * vx;
  ux += ux; uy += uy; uz += uz;
  const float cx = qy * uz - qz * uy, cy = qz * ux - qx * uz, cz = qx * uy - qy * ux;
  ox = vx + ux * qw + cx; oy = vy + uy * qw + cy; oz = vz + uz * qw + cz;
}

// mode 0: PointAssociateToMap (po = q * pi + t, :303-314); mode 1: PointAssociateTobeMapped (po = q^* * (pi - t), :316-323)
__global__ void __launch_bounds__(256)
k_associate(const float4 *__restrict__ in, float4 *__restrict__ out, const int *__restrict__ n_dev, TwistF t, int mode) {
  const int n = *n_dev;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = __ldg(in + i);
  float x, y, z;
  if (mode == 0) {
    rotate_dev(t.qx, t.qy, t.qz, t.qw, p.x, p.y, p.z, x, y, z);
    x += t.px; y += t.py; z += t.pz;
  } else {
    rotate_dev(-t.qx, -t.qy, -t.qz, t.qw, p.x - t.px, p.y - t.py, p.z - t.pz, x, y, z);
  }
  out[i] = make_float4(x, y, z, p.w);
}

// int((v + 25.0) / 50.0) + cen, minus one for negatives (:812-819) - double arithmetic like the reference
__device__ __forceinline__ int cube_of(float v, int cen) {
  int c = int(((double)v + 25.0) / 50.0) + cen;
  if ((double)v + 25.0 < 0) --c;
  return c;
}

// UpdateMapDatabase insert (:1123-1168).  The corner (n0 points) then surf cloud are one sequence; a point's key is its cloud's
// cube array entry w * kCubes + cube, kInsOutside when it falls outside the array.  A stable sort by key then puts every cube's new
// points together in push_back order.
constexpr int kInsOutside = 2 * kCubes, kInsKeyBits = 14;   // 2 * 4851 < 2^14
static_assert(kInsOutside < (1 << kInsKeyBits), "insert key bits");

// phase 1: map-frame point and key of every point; the counts *nc_dev / *ns_dev are clamped to [0, bc] / [0, bs] here;
// n_ins[0] = n (the sort's count), n_ins[1] = 0 (phase 2's run counter)
__global__ void __launch_bounds__(256)
k_ins_keys(const float4 *__restrict__ corner, const float4 *__restrict__ surf, const int *__restrict__ nc_dev, const int *__restrict__ ns_dev,
           int bc, int bs, TwistF t, int cen_l, int cen_w, int cen_h, float4 *__restrict__ mapped, unsigned *__restrict__ keys,
           unsigned *__restrict__ vals, int *__restrict__ n_ins) {
  const int n0 = min(max(*nc_dev, 0), bc), n = n0 + min(max(*ns_dev, 0), bs);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) { n_ins[0] = n; n_ins[1] = 0; }
  if (i >= n) return;
  const int w = i < n0 ? 0 : 1;
  const float4 p = w == 0 ? __ldg(corner + i) : __ldg(surf + (i - n0));
  float x, y, z;
  rotate_dev(t.qx, t.qy, t.qz, t.qw, p.x, p.y, p.z, x, y, z);
  x += t.px; y += t.py; z += t.pz;
  mapped[i] = make_float4(x, y, z, p.w);
  const int ci = cube_of(x, cen_l), cj = cube_of(y, cen_w), ck = cube_of(z, cen_h);
  const bool in = ci >= 0 && ci < kCubeL && cj >= 0 && cj < kCubeW && ck >= 0 && ck < kCubeH;
  keys[i] = in ? (unsigned)(w * kCubes + ci + kCubeL * cj + kCubeL * kCubeW * ck) : (unsigned)kInsOutside;
  vals[i] = (unsigned)i;
}

struct InsRun { int key, n; };
// phase 2: one run per touched cube, found at its last sorted point: the run goes to the host's pinned list (runs, mapped into
// the device's address space) in slot order, its slot and first sorted position to slot_of / start_of
__global__ void __launch_bounds__(256)
k_ins_runs(const unsigned *__restrict__ keys, const int *__restrict__ n_ins, int *__restrict__ nruns, InsRun *__restrict__ runs,
           int *__restrict__ slot_of, int *__restrict__ start_of) {
  const int n = n_ins[0];
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const unsigned k = keys[p];
  if (k >= (unsigned)kInsOutside || (p + 1 < n && keys[p + 1] == k)) return;
  int lo = 0, hi = p;   // first position of key k
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (keys[mid] < k) lo = mid + 1; else hi = mid; }
  const int slot = atomicAdd(nruns, 1);
  runs[slot] = InsRun{(int)k, p + 1 - lo};
  slot_of[k] = slot;
  start_of[k] = lo;
}

struct CubeEnd { float4 *p; int n; };   // a touched cube's segment and its count before the insert
// phase 3: every point to its append position, its rank inside the run
__global__ void __launch_bounds__(256)
k_ins_scatter(const unsigned *__restrict__ keys, const unsigned *__restrict__ vals, const float4 *__restrict__ mapped, const int *__restrict__ n_ins,
              const int *__restrict__ slot_of, const int *__restrict__ start_of, const CubeEnd *__restrict__ tab) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_ins[0]) return;
  const unsigned k = keys[p];
  if (k >= (unsigned)kInsOutside) return;
  const CubeEnd c = tab[slot_of[k]];
  c.p[c.n + p - start_of[k]] = __ldg(mapped + vals[p]);
}

// Input counts of one call {corner, surf, full}, read on the device and clamped to n_max: cnt[0], cnt[1], cnt[4]; cnt[7] = 1 when
// a count exceeded its bound (reported as LIO_ERR_CAPACITY at the down-sampling read-back)
__global__ void k_clamp_counts(const int *__restrict__ in, int3 n_max, int *__restrict__ cnt) {
  if (threadIdx.x != 0) return;
  const int mx[3] = {n_max.x, n_max.y, n_max.z};
  int v[3], over = 0;
  for (int w = 0; w < 3; ++w) {
    v[w] = in[w];
    if (v[w] > mx[w]) { over = 1; v[w] = mx[w]; }
    if (v[w] < 0) v[w] = 0;
  }
  cnt[0] = v[0]; cnt[1] = v[1]; cnt[4] = v[2]; cnt[7] = over;
}

// count-guarded copy of the full cloud (its count in *n_dev)
__global__ void __launch_bounds__(256)
k_copy_counted(const float4 *__restrict__ in, float4 *__restrict__ out, const int *__restrict__ n_dev) {
  const int n = *n_dev;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = __ldg(in + i);
}

struct Segment { const float4 *src; int n; int off; };
// concatenation of cube segments (laser_cloud_*_from_map_, :1005-1011); one block range per segment
__global__ void __launch_bounds__(256)
k_gather_segments(const Segment *__restrict__ seg, int nseg, float4 *__restrict__ out) {
  for (int s = blockIdx.y; s < nseg; s += gridDim.y) {
    const Segment sg = seg[s];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < sg.n; i += gridDim.x * blockDim.x) out[sg.off + i] = __ldg(sg.src + i);
  }
}

}  // namespace lio

using namespace lio;

struct lio_pm {
  struct Cube { float4 *p = nullptr; int n = 0, cap = 0; };
  int device = 0;
  cudaStream_t stream = nullptr;
  int sm = 132;
  int max_points = 0;
  std::vector<Cube> cube[2];           // [0] corner, [1] surf: kCubes descriptors each
  int cen_l = 10, cen_w = 10, cen_h = 5;
  float leaf[2] = {0.2f, 0.4f};
  float min_match_sq_dis = 1.0f, min_plane_dis = 0.2f;
  int max_iter = 10;
  double delta_r_abort = 0.05, delta_t_abort = 0.05;
  TwistF sum, bef, aft, tobe;          // transform_sum_, transform_bef_mapped_, transform_aft_mapped_, transform_tobe_mapped_
  // device scratch
  float4 *d_in[2] = {nullptr, nullptr}, *d_stack[2] = {nullptr, nullptr}, *d_ds[2] = {nullptr, nullptr}, *d_mapped = nullptr;
  float4 *d_map[2] = {nullptr, nullptr};
  int map_cap[2] = {0, 0};
  int *d_cnt = nullptr;                // [0,1] input sizes, [2,3] down-sampled sizes, [4] full cloud, [5,6] surround map in / out,
                                       // [7] input count over its bound, [8..10] counts uploaded by the host entries
  int h_cnt[8] = {};                   // read-back of d_cnt[0..7] after the down-sampling
  Segment *d_seg = nullptr;
  VoxelGrid vg;
  ScanToMapWork stm;
  int stm_cap[3] = {0, 0, 0};
  int last_iters = 0, last_from_map[2] = {0, 0};
  std::vector<size_t> last_valid, last_surround;   // laser_cloud_valid_idx_ / laser_cloud_surround_idx_ of the last process call
  // UpdateMapDatabase (pm_update).  Insert: sort buffers for ins_cap (initially 2 * max_points) keys, per-key slot / first position, the run list
  // (pinned, written by the device), the touched cubes' table (pinned and its device copy).
  unsigned *d_ins_k[2] = {nullptr, nullptr}, *d_ins_v[2] = {nullptr, nullptr};
  RadixSortTemp ins_rs;
  int ins_cap = 0;
  int *d_ins_n = nullptr;              // [0] points, [1] runs
  int *d_slot_of = nullptr, *d_start_of = nullptr;
  InsRun *h_runs = nullptr, *h_runs_dev = nullptr;
  int *h_nruns = nullptr;              // read-back of d_ins_n: [0] points inserted, [1] runs
  CubeEnd *h_tab = nullptr, *d_tab = nullptr;
  cudaEvent_t ev_ins = nullptr;
  // Re-filter: one segmented VoxelGrid over the jobs; their output counts arrive in h_jn (pinned) behind ev_counts and are applied
  // to the directory by pm_counts before anything reads it.
  SegVoxelGrid svg;
  VgJob *h_jobs = nullptr;
  int *h_jn = nullptr;
  std::vector<std::pair<int, size_t>> pend_jobs;   // (cloud, cube) of every job whose count is in flight
  bool counts_pending = false;
  bool counts_broken = false;          // a job exceeded the 2^24-voxel bound: its cubes are wrong, every later reader fails
  cudaEvent_t ev_counts = nullptr;
  int upd_stats[4] = {0, 0, 0, 0};     // last UpdateMapDatabase: cube jobs, kernel launches, host waits (the later wait for the
                                       // re-filtered counts included), points inserted
  bool started = false;               // a process call has run (lio_pm_enable_publish must come before it)
  bool publish = false;                // lio_pm_enable_publish: PointMapping::PublishResults on every lio_pm_process_dev
  bool attached = false;               // lio_est_attach_map: the estimator owns the map (its process / update / destroy entries refuse)
  // map-builder mode (lio_mb_*: MapBuilder : PointMapping, src/map_builder/MapBuilder.cc)
  bool mb = false, enable_4d = true, system_init = false;
  int skip_count = 2, odom_count = 0;
  int map_frame_count = 4;             // num_map_frames_ - 1 (PointMapping.cc:104): the first frame publishes
  float map_leaf = 0.2f;               // down_size_filter_map_ (PointMapping.cc:123 0.6, map_builder_node 0.2)
  int max_full = 0, n_full = 0, n_surround = 0, sur_cap = 0;
  float4 *d_full_in = nullptr, *d_full_out = nullptr, *d_sur = nullptr, *d_sur_ds = nullptr;
  Segment *d_sur_seg = nullptr, *h_sur_seg = nullptr;   // h_sur_seg / h_sur_n: pinned, so their uploads need no sync
  int *h_sur_n = nullptr;
  VoxelGrid vg_sur;                    // down_size_filter_map_, sized for the surround map
};

static size_t to_index(int i, int j, int k) { return (size_t)i + (size_t)kCubeL * j + (size_t)kCubeL * kCubeW * k; }
static int cube_of_host(float v, int cen) {
  int c = int(((double)v + 25.0) / 50.0) + cen;
  if ((double)v + 25.0 < 0) --c;
  return c;
}

extern "C" int lio_pm_destroy(lio_pm *m) {
  if (!m) return LIO_OK;
  if (m->attached) { lio_set_last_error(__FILE__, __LINE__, "lio_pm_destroy: the map is attached to an estimator (lio_est_destroy releases it)"); return LIO_ERR_INVALID; }
  cudaSetDevice(m->device);
  for (int w = 0; w < 2; ++w) {
    for (lio_pm::Cube &c : m->cube[w]) if (c.p) cudaFree(c.p);
    void *fr[] = {m->d_in[w], m->d_stack[w], m->d_ds[w], m->d_map[w]};
    for (void *q : fr) if (q) cudaFree(q);
  }
  void *fr[] = {m->d_mapped, m->d_cnt, m->d_seg, m->d_full_in, m->d_full_out, m->d_sur, m->d_sur_ds, m->d_sur_seg, m->d_ins_k[0],
                m->d_ins_k[1], m->d_ins_v[0], m->d_ins_v[1], m->d_ins_n, m->d_slot_of, m->d_start_of, m->d_tab};
  for (void *q : fr) if (q) cudaFree(q);
  void *frh[] = {m->h_sur_seg, m->h_sur_n, m->h_runs, m->h_nruns, m->h_tab, m->h_jobs, m->h_jn};
  for (void *q : frh) if (q) cudaFreeHost(q);
  if (m->ev_ins) cudaEventDestroy(m->ev_ins);
  if (m->ev_counts) cudaEventDestroy(m->ev_counts);
  m->vg.destroy();
  m->vg_sur.destroy();
  m->svg.destroy();
  m->ins_rs.destroy();
  m->stm.destroy();
  delete m;
  return LIO_OK;
}

extern "C" int lio_pm_create(int max_points, float corner_filter_size, float surf_filter_size, float min_match_sq_dis, float min_plane_dis,
                             int max_iterations, int device, void *cuda_stream, lio_pm **out) {
  if (!out || max_points < 16 || !(corner_filter_size > 0) || !(surf_filter_size > 0) || max_iterations < 0) return LIO_ERR_INVALID;
  if (lio_device_count() <= 0) return LIO_ERR_NO_DEVICE;
  LIO_CUDA_OK(cudaSetDevice(device));
  lio_pm *m = new (std::nothrow) lio_pm();
  if (!m) return LIO_ERR_INVALID;
  m->device = device; m->stream = (cudaStream_t)cuda_stream; m->max_points = max_points;
  m->leaf[0] = corner_filter_size; m->leaf[1] = surf_filter_size;
  m->min_match_sq_dis = min_match_sq_dis; m->min_plane_dis = min_plane_dis; m->max_iter = max_iterations;
  cudaDeviceGetAttribute(&m->sm, cudaDevAttrMultiProcessorCount, device);
  m->cube[0].assign(kCubes, lio_pm::Cube());
  m->cube[1].assign(kCubes, lio_pm::Cube());
  bool ok = true;
  for (int w = 0; w < 2 && ok; ++w) {
    ok = ok && cudaMalloc(&m->d_in[w], sizeof(float4) * max_points) == cudaSuccess;
    ok = ok && cudaMalloc(&m->d_stack[w], sizeof(float4) * max_points) == cudaSuccess;
    ok = ok && cudaMalloc(&m->d_ds[w], sizeof(float4) * max_points) == cudaSuccess;
  }
  m->ins_cap = 2 * max_points;
  ok = ok && cudaMalloc(&m->d_mapped, sizeof(float4) * 2 * max_points) == cudaSuccess;
  ok = ok && cudaMalloc(&m->d_cnt, sizeof(int) * 12) == cudaSuccess;
  ok = ok && cudaMalloc(&m->d_seg, sizeof(Segment) * 256) == cudaSuccess;
  ok = ok && m->vg.init(max_points) == 0;
  for (int b = 0; b < 2 && ok; ++b) {
    ok = ok && cudaMalloc(&m->d_ins_k[b], sizeof(unsigned) * 2 * max_points) == cudaSuccess;
    ok = ok && cudaMalloc(&m->d_ins_v[b], sizeof(unsigned) * 2 * max_points) == cudaSuccess;
  }
  ok = ok && m->ins_rs.init(2 * max_points) == 0;
  ok = ok && cudaMalloc(&m->d_ins_n, sizeof(int) * 2) == cudaSuccess;
  ok = ok && cudaMalloc(&m->d_slot_of, sizeof(int) * kInsOutside) == cudaSuccess;
  ok = ok && cudaMalloc(&m->d_start_of, sizeof(int) * kInsOutside) == cudaSuccess;
  ok = ok && cudaMalloc(&m->d_tab, sizeof(CubeEnd) * kInsOutside) == cudaSuccess;
  ok = ok && cudaHostAlloc(&m->h_runs, sizeof(InsRun) * kInsOutside, cudaHostAllocMapped) == cudaSuccess;
  ok = ok && cudaHostGetDevicePointer(&m->h_runs_dev, m->h_runs, 0) == cudaSuccess;
  ok = ok && cudaMallocHost(&m->h_nruns, sizeof(int) * 2) == cudaSuccess;
  ok = ok && cudaMallocHost(&m->h_tab, sizeof(CubeEnd) * kInsOutside) == cudaSuccess;
  ok = ok && m->svg.init() == 0;
  ok = ok && cudaMallocHost(&m->h_jobs, sizeof(VgJob) * kVgMaxJobs) == cudaSuccess;
  ok = ok && cudaMallocHost(&m->h_jn, sizeof(int) * (kVgMaxJobs + 1)) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&m->ev_ins, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&m->ev_counts, cudaEventDisableTiming) == cudaSuccess;
  if (!ok) { lio_set_last_error(__FILE__, __LINE__, "lio_pm_create: device allocation failed"); lio_pm_destroy(m); return LIO_ERR_CUDA; }
  *out = m;
  return LIO_OK;
}

// ---- host-side directory logic (the reference's own index arithmetic) ---------------------------------------------------
static void pm_recentre(lio_pm *m, float px, float py, float pz, int &ci, int &cj, int &ck) {   // :812-931
  ci = cube_of_host(px, m->cen_l); cj = cube_of_host(py, m->cen_w); ck = cube_of_host(pz, m->cen_h);
  auto shift = [&](int axis, int dir) {  // dir +1: contents move towards higher indices, the low face is cleared
    const int n[3] = {kCubeL, kCubeW, kCubeH};
    int idx[3];
    for (idx[(axis + 1) % 3] = 0; idx[(axis + 1) % 3] < n[(axis + 1) % 3]; ++idx[(axis + 1) % 3])
      for (idx[(axis + 2) % 3] = 0; idx[(axis + 2) % 3] < n[(axis + 2) % 3]; ++idx[(axis + 2) % 3]) {
        if (dir > 0) {
          for (int a = n[axis] - 1; a >= 1; --a) {
            idx[axis] = a; const size_t ia = to_index(idx[0], idx[1], idx[2]);
            idx[axis] = a - 1; const size_t ib = to_index(idx[0], idx[1], idx[2]);
            std::swap(m->cube[0][ia], m->cube[0][ib]); std::swap(m->cube[1][ia], m->cube[1][ib]);
          }
          idx[axis] = 0;
        } else {
          for (int a = 0; a < n[axis] - 1; ++a) {
            idx[axis] = a; const size_t ia = to_index(idx[0], idx[1], idx[2]);
            idx[axis] = a + 1; const size_t ib = to_index(idx[0], idx[1], idx[2]);
            std::swap(m->cube[0][ia], m->cube[0][ib]); std::swap(m->cube[1][ia], m->cube[1][ib]);
          }
          idx[axis] = n[axis] - 1;
        }
        const size_t ic = to_index(idx[0], idx[1], idx[2]);
        m->cube[0][ic].n = 0; m->cube[1][ic].n = 0;   // clear(): the HBM segment is kept for re-use
      }
  };
  while (ci < 3) { shift(0, +1); ++ci; ++m->cen_l; }
  while (ci >= kCubeL - 3) { shift(0, -1); --ci; --m->cen_l; }
  while (cj < 3) { shift(1, +1); ++cj; ++m->cen_w; }
  while (cj >= kCubeW - 3) { shift(1, -1); --cj; --m->cen_w; }
  while (ck < 3) { shift(2, +1); ++ck; ++m->cen_h; }
  while (ck >= kCubeH - 3) { shift(2, -1); --ck; --m->cen_h; }
}

// valid: laser_cloud_valid_idx_; surround (optional): laser_cloud_surround_idx_, every in-range cube without the FOV test
static void pm_select(const lio_pm *m, float px, float py, float pz, const float z[3], int ci, int cj, int ck, std::vector<size_t> &valid,
                      std::vector<size_t> *surround) {   // :944-1003
  valid.clear();
  if (surround) surround->clear();
  for (int i = ci - 2; i <= ci + 2; ++i)
    for (int j = cj - 2; j <= cj + 2; ++j)
      for (int k = ck - 2; k <= ck + 2; ++k) {
        if (!(i >= 0 && i < kCubeL && j >= 0 && j < kCubeW && k >= 0 && k < kCubeH)) continue;
        const float center_x = 50.0f * (i - m->cen_l), center_y = 50.0f * (j - m->cen_w), center_z = 50.0f * (k - m->cen_h);
        bool is_in_laser_fov = false;
        for (int ii = -1; ii <= 1; ii += 2)
          for (int jj = -1; jj <= 1; jj += 2)
            for (int kk = -1; kk <= 1; kk += 2) {
              const float cx = center_x + 25.0f * ii, cy = center_y + 25.0f * jj, cz = center_z + 25.0f * kk;
              const float d0 = px - cx, d1 = py - cy, d2 = pz - cz;
              volatile float s1 = d0 * d0; s1 = s1 + d1 * d1; s1 = s1 + d2 * d2;
              const float e0 = z[0] - cx, e1 = z[1] - cy, e2 = z[2] - cz;
              volatile float s2 = e0 * e0; s2 = s2 + e1 * e1; s2 = s2 + e2 * e2;
              const float squared_side1 = s1, squared_side2 = s2;
              const float check1 = 100.0f + squared_side1 - squared_side2 - 10.0f * std::sqrt(3.0f) * std::sqrt(squared_side1);
              const float check2 = 100.0f + squared_side1 - squared_side2 + 10.0f * std::sqrt(3.0f) * std::sqrt(squared_side1);
              if (check1 < 0 && check2 > 0) is_in_laser_fov = true;
            }
        if (is_in_laser_fov) valid.push_back(to_index(i, j, k));
        if (surround) surround->push_back(to_index(i, j, k));
      }
}

static int pm_grow(lio_pm *m, lio_pm::Cube &c, int need) {
  if (need <= c.cap) return LIO_OK;
  int cap = std::max(1024, c.cap);
  while (cap < need) cap *= 2;
  float4 *p = nullptr;
  LIO_CUDA_OK(cudaMalloc(&p, sizeof(float4) * cap));
  if (c.p && c.n > 0) LIO_CUDA_OK(cudaMemcpyAsync(p, c.p, sizeof(float4) * c.n, cudaMemcpyDeviceToDevice, m->stream));
  if (c.p) { LIO_CUDA_OK(cudaStreamSynchronize(m->stream)); cudaFree(c.p); }
  c.p = p; c.cap = cap;
  return LIO_OK;
}

// laser_cloud_*_from_map_: concatenate the valid cubes (in `valid` order) into d_map[w]
static int pm_from_map(lio_pm *m, const std::vector<size_t> &valid, int w, int &total) {
  std::vector<Segment> seg;
  total = 0;
  for (size_t v : valid) {
    const lio_pm::Cube &c = m->cube[w][v];
    if (c.n > 0) { seg.push_back(Segment{c.p, c.n, total}); total += c.n; }
  }
  if (total > m->map_cap[w]) {
    if (m->d_map[w]) cudaFree(m->d_map[w]);
    m->map_cap[w] = std::max(2 * total, 1 << 16);
    LIO_CUDA_OK(cudaMalloc(&m->d_map[w], sizeof(float4) * m->map_cap[w]));
  }
  if (seg.empty()) return LIO_OK;
  if (seg.size() > 256) return LIO_ERR_CAPACITY;
  LIO_CUDA_OK(cudaMemcpyAsync(m->d_seg, seg.data(), sizeof(Segment) * seg.size(), cudaMemcpyHostToDevice, m->stream));
  LIO_CUDA_OK(cudaStreamSynchronize(m->stream));   // seg is a stack vector
  k_gather_segments<<<dim3(16, (unsigned)seg.size()), 256, 0, m->stream>>>(m->d_seg, (int)seg.size(), m->d_map[w]);
  return LIO_OK;
}

// The re-filter's output counts of the last UpdateMapDatabase into the directory; every reader of the cube counts calls this first.
// This is the update's one host wait after it returned (counted in its upd_stats).  Once a job has exceeded the 2^24-voxel bound
// its cubes hold wrong centroids: the error is sticky, this and every later call return LIO_ERR_CAPACITY.
static int pm_counts(lio_pm *m) {
  if (m->counts_broken) {
    lio_set_last_error(__FILE__, __LINE__, "UpdateMapDatabase: an earlier re-filter exceeded the 2^24-voxel bound; the cube map is invalid");
    return LIO_ERR_CAPACITY;
  }
  if (!m->counts_pending) return LIO_OK;
  m->counts_pending = false;
  LIO_CUDA_OK(cudaEventSynchronize(m->ev_counts));
  const int nj = (int)m->pend_jobs.size();
  if (m->h_jn[nj]) {
    m->counts_broken = true;
    lio_set_last_error(__FILE__, __LINE__, "UpdateMapDatabase: a cube's voxel index range exceeds 2^24 (leaf too small for a 50 m cube)");
    return LIO_ERR_CAPACITY;
  }
  for (int j = 0; j < nj; ++j) m->cube[m->pend_jobs[j].first][m->pend_jobs[j].second].n = m->h_jn[j];
  return LIO_OK;
}

// UpdateMapDatabase (:1112-1208) of the corner src[0] and surf src[1] clouds in HBM with the pose t.  Their counts are read on the
// device (*n_dev[w], clamped to [0, bound[w]]); bound[0] + bound[1] <= ins_cap.  valid holds cube indices
// of the margin centre mc (:1173-1183 move them to the current centre).  Insert: the keys, a stable sort by key and the run list
// on the device; the host waits once for the runs to size the touched segments (and once per segment it moves to a larger one),
// then uploads their {segment, count} table.  Re-filter: one segmented VoxelGrid over every non-empty valid cube, corner and surf,
// whose output counts reach the directory through pm_counts without a wait here (the next reader waits; upd_stats counts that wait).
static int pm_update(lio_pm *m, const std::vector<size_t> &valid, const float4 *const src[2], const int *const n_dev[2], const int bound[2],
                     const TwistF &t, const int mc[3]) {
  cudaStream_t st = m->stream;
  int rc = pm_counts(m);
  if (rc != LIO_OK) return rc;
  if (bound[0] + bound[1] > m->ins_cap) { lio_set_last_error(__FILE__, __LINE__, "UpdateMapDatabase: clouds exceed the insert buffers"); return LIO_ERR_CAPACITY; }
  int launches = 0, waits = 0, n = 0;
  const int nb = bound[0] + bound[1];
  if (nb > 0) {
    const int blocks = (nb + 255) / 256;
    k_ins_keys<<<blocks, 256, 0, st>>>(src[0], src[1], n_dev[0], n_dev[1], bound[0], bound[1], t, m->cen_l, m->cen_w, m->cen_h, m->d_mapped,
                                       m->d_ins_k[0], m->d_ins_v[0], m->d_ins_n);
    ++launches;
    const int b = radix_sort_pairs(m->d_ins_k[0], m->d_ins_v[0], m->d_ins_k[1], m->d_ins_v[1], m->d_ins_n, nb, kInsKeyBits, m->ins_rs, st, &launches);
    if (b < 0) return LIO_ERR_CAPACITY;
    k_ins_runs<<<blocks, 256, 0, st>>>(m->d_ins_k[b], m->d_ins_n, m->d_ins_n + 1, m->h_runs_dev, m->d_slot_of, m->d_start_of);
    ++launches;
    LIO_CUDA_OK(cudaMemcpyAsync(m->h_nruns, m->d_ins_n, sizeof(int) * 2, cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaEventRecord(m->ev_ins, st));
    LIO_CUDA_OK(cudaEventSynchronize(m->ev_ins));
    ++waits;
    n = m->h_nruns[0];
    const int nr = m->h_nruns[1];
    for (int r = 0; r < nr; ++r) {
      const InsRun run = m->h_runs[r];
      lio_pm::Cube &c = m->cube[run.key / kCubes][run.key % kCubes];
      if (c.n + run.n > c.cap && c.p) ++waits;
      if ((rc = pm_grow(m, c, c.n + run.n)) != LIO_OK) return rc;
      m->h_tab[r] = CubeEnd{c.p, c.n};
      c.n += run.n;
    }
    if (nr > 0) {
      LIO_CUDA_OK(cudaMemcpyAsync(m->d_tab, m->h_tab, sizeof(CubeEnd) * nr, cudaMemcpyHostToDevice, st));
      k_ins_scatter<<<blocks, 256, 0, st>>>(m->d_ins_k[b], m->d_ins_v[b], m->d_mapped, m->d_ins_n, m->d_slot_of, m->d_start_of, m->d_tab);
      ++launches;
    }
  }
  // re-filter every valid cube (corner then surf), each with its own bounding box like pcl::VoxelGrid on that cube's cloud
  m->pend_jobs.clear();
  int total = 0;
  for (size_t index : valid) {
    int li, lj, lk;
    { int residual = (int)(index % (kCubeL * kCubeW)); lk = (int)(index / (kCubeL * kCubeW)); lj = residual / kCubeL; li = residual % kCubeL; }
    const float center_x = 50.0f * (li - mc[0]), center_y = 50.0f * (lj - mc[1]), center_z = 50.0f * (lk - mc[2]);
    const int ci = cube_of_host(center_x, m->cen_l), cj = cube_of_host(center_y, m->cen_w), ck = cube_of_host(center_z, m->cen_h);
    if (!(ci >= 0 && ci < kCubeL && cj >= 0 && cj < kCubeW && ck >= 0 && ck < kCubeH)) continue;
    const size_t idx = to_index(ci, cj, ck);
    for (int w = 0; w < 2; ++w) {
      const lio_pm::Cube &c = m->cube[w][idx];
      if (c.n == 0) continue;
      if ((int)m->pend_jobs.size() == kVgMaxJobs || c.n > INT_MAX / 2 - total) {
        m->pend_jobs.clear();
        lio_set_last_error(__FILE__, __LINE__, "UpdateMapDatabase: more than 256 cube jobs");
        return LIO_ERR_CAPACITY;
      }
      m->h_jobs[m->pend_jobs.size()] = VgJob{c.p, c.n, total, m->leaf[w]};
      m->pend_jobs.emplace_back(w, idx);
      total += c.n;
    }
  }
  const int nj = (int)m->pend_jobs.size();
  if (nj > 0) {
    if (m->svg.reserve(total) != 0) { m->pend_jobs.clear(); lio_set_last_error(__FILE__, __LINE__, "UpdateMapDatabase: workspace allocation failed"); return LIO_ERR_CUDA; }
    if ((rc = m->svg.run(m->h_jobs, nj, total, m->h_jn, st, &launches)) != LIO_OK) { m->pend_jobs.clear(); return rc; }
    LIO_CUDA_OK(cudaEventRecord(m->ev_counts, st));
    m->counts_pending = true;
    ++waits;   // pm_counts, at the next call or cube accessor (or in this call's surround publication)
  }
  m->upd_stats[0] = nj; m->upd_stats[1] = launches; m->upd_stats[2] = waits; m->upd_stats[3] = n;
  return LIO_OK;
}

// ---- the steps of PointMapping::Process that MapBuilder::ProcessMap shares ------------------------------------------------
// Host entries: the clouds and their counts go to the context's own input buffers (d_in, d_full_in, d_cnt[8..10]); the steps
// below then run exactly as for device inputs.
static int pm_upload(lio_pm *m, const float *const src[2], const int nin[2], const float *full, int nf) {
  cudaStream_t st = m->stream;
  const int hcnt[3] = {nin[0], nin[1], nf};
  LIO_CUDA_OK(cudaMemcpyAsync(m->d_cnt + 8, hcnt, sizeof(hcnt), cudaMemcpyHostToDevice, st));
  for (int w = 0; w < 2; ++w)
    if (nin[w] > 0) LIO_CUDA_OK(cudaMemcpyAsync(m->d_in[w], src[w], sizeof(float4) * nin[w], cudaMemcpyHostToDevice, st));
  if (m->mb && nf > 0) LIO_CUDA_OK(cudaMemcpyAsync(m->d_full_in, full, sizeof(float4) * nf, cudaMemcpyHostToDevice, st));
  LIO_CUDA_OK(cudaStreamSynchronize(st));   // hcnt is a stack array
  return LIO_OK;
}

// Stacks (:782-800, :1013-1016): the last features to the map frame with the predicted pose, and back.  Sources and counts
// {corner, surf, full} are on the device; n_max bounds them (the counts are clamped on the device).  In map-builder mode and on a
// publishing PointMapping the full-resolution cloud is copied into d_full_in in the same pass.
static int pm_stack(lio_pm *m, const float4 *const src[2], const float4 *full, const int *n3_dev, const int n_max[3]) {
  cudaStream_t st = m->stream;
  k_clamp_counts<<<1, 32, 0, st>>>(n3_dev, make_int3(n_max[0], n_max[1], n_max[2]), m->d_cnt);
  for (int w = 0; w < 2; ++w) {
    if (n_max[w] == 0) continue;
    k_associate<<<(n_max[w] + 255) / 256, 256, 0, st>>>(src[w], m->d_stack[w], m->d_cnt + w, m->tobe, 0);
    k_associate<<<(n_max[w] + 255) / 256, 256, 0, st>>>(m->d_stack[w], m->d_stack[w], m->d_cnt + w, m->tobe, 1);
  }
  if ((m->mb || m->publish) && n_max[2] > 0 && full != m->d_full_in)
    k_copy_counted<<<std::max(1, std::min(4 * m->sm, (n_max[2] + 255) / 256)), 256, 0, st>>>(full, m->d_full_in, m->d_cnt + 4);
  LIO_CUDA_OK(cudaGetLastError());
  return LIO_OK;
}

// point_on_z_axis_ (:801-806), re-centring (:809-931), cube selection (:944-1003) and laser_cloud_*_from_map_ (:1005-1011)
static int pm_locate(lio_pm *m, std::vector<size_t> &valid, std::vector<size_t> *surround, int K[2]) {
  float z[3];
  rotate_host(m->tobe, 0.0f, 0.0f, 10.0f, z[0], z[1], z[2]);
  z[0] += m->tobe.px; z[1] += m->tobe.py; z[2] += m->tobe.pz;
  int ci, cj, ck;
  pm_recentre(m, m->tobe.px, m->tobe.py, m->tobe.pz, ci, cj, ck);
  pm_select(m, m->tobe.px, m->tobe.py, m->tobe.pz, z, ci, cj, ck, valid, surround);
  for (int w = 0; w < 2; ++w) { int rc = pm_from_map(m, valid, w, K[w]); if (rc != LIO_OK) return rc; }
  m->last_from_map[0] = K[0]; m->last_from_map[1] = K[1];
  return LIO_OK;
}

// VoxelGrid of the stacks (:1016-1022)
static int pm_downsample(lio_pm *m, const int nin[2], int n_ds[2]) {
  cudaStream_t st = m->stream;
  for (int w = 0; w < 2; ++w) {
    if (nin[w] == 0) { LIO_CUDA_OK(cudaMemsetAsync(m->d_cnt + 2 + w, 0, sizeof(int), st)); continue; }
    int rc = m->vg.run(m->d_stack[w], m->d_cnt + w, nin[w], m->leaf[w], m->d_ds[w], m->max_points, m->d_cnt + 2 + w, nullptr, st, nullptr);
    if (rc != LIO_OK) return rc;
  }
  // one read-back for the down-sampled sizes, the clamped input counts and their overflow flag
  LIO_CUDA_OK(cudaMemcpyAsync(m->h_cnt, m->d_cnt, sizeof(m->h_cnt), cudaMemcpyDeviceToHost, st));
  LIO_CUDA_OK(cudaStreamSynchronize(st));
  n_ds[0] = m->h_cnt[2]; n_ds[1] = m->h_cnt[3];
  if (m->h_cnt[7]) { lio_set_last_error(__FILE__, __LINE__, "input cloud count exceeds its bound n3_max"); return LIO_ERR_CAPACITY; }
  return LIO_OK;
}

// OptimizeTransformTobeMapped (variant 0, :325-753) / MapBuilder::OptimizeMap (variant 1, MapBuilder.cc:624-1014) of tobe against
// the pulled map; the caller has checked the early return (Kc <= 10 or Ks <= 100)
static int pm_optimise(lio_pm *m, const int K[2], const int n_ds[2], int variant) {
  m->last_iters = 0;
  if (m->max_iter <= 0) return LIO_OK;
  if (K[0] > m->stm_cap[0] || K[1] > m->stm_cap[1] || n_ds[0] + n_ds[1] > m->stm_cap[2]) {
    m->stm.destroy();
    m->stm_cap[0] = std::max(2 * K[0], 1 << 15); m->stm_cap[1] = std::max(2 * K[1], 1 << 16); m->stm_cap[2] = std::max(2 * (n_ds[0] + n_ds[1]), 1 << 15);
    if (m->stm.init(m->stm_cap[0], m->stm_cap[1], m->stm_cap[2]) != 0) { lio_set_last_error(__FILE__, __LINE__, "scan-to-map workspace allocation failed"); return LIO_ERR_CUDA; }
  }
  float tf7[7] = {m->tobe.qx, m->tobe.qy, m->tobe.qz, m->tobe.qw, m->tobe.px, m->tobe.py, m->tobe.pz};
  int rc = scan_to_map_run(m->stm, m->d_map[0], K[0], m->d_map[1], K[1], m->d_ds[0], m->d_cnt + 2, std::max(n_ds[0], 1), m->d_ds[1], m->d_cnt + 3,
                           std::max(n_ds[1], 1), tf7, m->min_match_sq_dis, m->min_plane_dis, m->max_iter, m->delta_r_abort, m->delta_t_abort, variant,
                           nullptr, &m->last_iters, m->sm, m->stream);
  if (rc != LIO_OK) return rc;
  m->tobe = TwistF{tf7[0], tf7[1], tf7[2], tf7[3], tf7[4], tf7[5], tf7[6]};
  return LIO_OK;
}

static TwistF tf7_to_twist(const float t[7]) { return TwistF{t[0], t[1], t[2], t[3], t[4], t[5], t[6]}; }
static void twist_to_tf7(const TwistF &t, float o[7]) { o[0] = t.qx; o[1] = t.qy; o[2] = t.qz; o[3] = t.qw; o[4] = t.px; o[5] = t.py; o[6] = t.pz; }

static int mb_surround(lio_pm *m, const std::vector<size_t> &surround);

// PublishResults (PointMapping.cc:1210-1270) / PublishMapBuilderResults (MapBuilder.cc:144-218): the surround map every
// num_map_frames_ (5) calls, the first call included, and the full cloud `full` (count *nf_dev, host value nf <= max_full) to the
// map frame with the final tobe every call.  The only synchronisation is the read of the surround size on calls that publish it.
static int pm_publish(lio_pm *m, const std::vector<size_t> &surround, const float4 *full, const int *nf_dev, int nf, bool &published) {
  cudaStream_t st = m->stream;
  published = ++m->map_frame_count >= 5;
  if (published) {
    m->map_frame_count = 0;
    int rc = mb_surround(m, surround);
    if (rc != LIO_OK) return rc;
  }
  if (nf > 0) k_associate<<<(nf + 255) / 256, 256, 0, st>>>(full, m->d_full_out, nf_dev, m->tobe, 0);
  m->n_full = nf;
  if (published) {
    LIO_CUDA_OK(cudaMemcpyAsync(m->h_sur_n, m->d_cnt + 6, sizeof(int), cudaMemcpyDeviceToHost, st));
    LIO_CUDA_OK(cudaStreamSynchronize(st));
    m->n_surround = *m->h_sur_n;
  }
  LIO_CUDA_OK(cudaGetLastError());
  return LIO_OK;
}

// PointMapping::Process (:765-1052), imu_inited_ == false, num_stack_frames_ == 1, followed on a publishing handle by
// PublishResults (:1210-1270).  Device sources, device counts {corner, surf, full}, host bounds n_max (already capped).
static int pm_process(lio_pm *m, const float4 *const src[2], const float4 *full, const int *n3_dev, const int n_max[3], const float transform_sum7[7],
                      float transform_tobe_mapped7[7], float transform_aft_mapped7[7], int *info, int n_info) {
  const int nin[2] = {n_max[0], n_max[1]};
  m->started = true;
  int rc = pm_counts(m);
  if (rc != LIO_OK) return rc;
  m->sum = tf7_to_twist(transform_sum7);
  m->tobe = twist_mul(m->tobe, twist_mul(twist_inverse(m->bef), m->sum));   // TransformAssociateToMap :753-756
  if ((rc = pm_stack(m, src, full, n3_dev, n_max)) != LIO_OK) return rc;
  int K[2] = {0, 0}, n_ds[2] = {0, 0};
  if ((rc = pm_locate(m, m->last_valid, m->publish ? &m->last_surround : nullptr, K)) != LIO_OK) return rc;
  if ((rc = pm_downsample(m, nin, n_ds)) != LIO_OK) return rc;
  const bool optimised = !(K[0] <= 10 || K[1] <= 100);
  m->last_iters = 0;
  if (optimised && (rc = pm_optimise(m, K, n_ds, 0)) != LIO_OK) return rc;
  if (optimised) { m->bef = m->sum; m->aft = m->tobe; }   // TransformUpdate sits behind the optimiser's early return (:327-329, :716)
  const int cen[3] = {m->cen_l, m->cen_w, m->cen_h};   // margin centre == current centre: the valid list is this call's
  const float4 *ds[2] = {m->d_ds[0], m->d_ds[1]};
  const int *n_ds_dev[2] = {m->d_cnt + 2, m->d_cnt + 3};
  if ((rc = pm_update(m, m->last_valid, ds, n_ds_dev, n_ds, m->tobe, cen)) != LIO_OK) return rc;
  bool published = false;
  if (m->publish && (rc = pm_publish(m, m->last_surround, m->d_full_in, m->d_cnt + 4, n_max[2] > 0 ? m->h_cnt[4] : 0, published)) != LIO_OK) return rc;
  if (transform_tobe_mapped7) twist_to_tf7(m->tobe, transform_tobe_mapped7);
  if (transform_aft_mapped7) twist_to_tf7(m->aft, transform_aft_mapped7);
  const int out[5] = {m->last_iters, K[0], K[1], published ? 1 : 0, m->publish ? m->n_surround : 0};
  if (info) for (int k = 0; k < n_info; ++k) info[k] = out[k];
  return LIO_OK;
}

// Clouds: HOST arrays of n x 4 floats.
extern "C" int lio_pm_process_host(lio_pm *m, const float *corner_last, int nc, const float *surf_last, int ns, const float transform_sum7[7],
                                   float transform_tobe_mapped7[7], int info3[3]) {
  if (!m || m->mb || m->publish || m->attached || !transform_sum7 || nc < 0 || ns < 0 || (nc > 0 && !corner_last) || (ns > 0 && !surf_last))
    return LIO_ERR_INVALID;
  if (nc > m->max_points || ns > m->max_points) return LIO_ERR_CAPACITY;
  LIO_CUDA_OK(cudaSetDevice(m->device));
  const float *src[2] = {corner_last, surf_last};
  const int nin[2] = {nc, ns};
  int rc = pm_upload(m, src, nin, nullptr, 0);
  if (rc != LIO_OK) return rc;
  const float4 *dsrc[2] = {m->d_in[0], m->d_in[1]};
  const int n_max[3] = {nc, ns, 0};
  return pm_process(m, dsrc, nullptr, m->d_cnt + 8, n_max, transform_sum7, transform_tobe_mapped7, nullptr, info3, 3);
}

extern "C" int lio_pm_process_dev(lio_pm *m, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev,
                                  const int n3_max[3], const float transform_sum7[7], float transform_tobe_mapped7[7], float transform_aft_mapped7[7],
                                  int info5[5]) {
  if (!m || m->mb || m->attached || !transform_sum7 || !n3_dev || !n3_max || n3_max[0] < 0 || n3_max[1] < 0 || n3_max[2] < 0 || (n3_max[0] > 0 && !corner_dev) ||
      (n3_max[1] > 0 && !surf_dev) || (m->publish && n3_max[2] > 0 && !full_dev))
    return LIO_ERR_INVALID;
  LIO_CUDA_OK(cudaSetDevice(m->device));
  const float4 *dsrc[2] = {reinterpret_cast<const float4 *>(corner_dev), reinterpret_cast<const float4 *>(surf_dev)};
  // without publishing the full cloud is not read: its count gets no bound, so it never reports an overflow
  const int n_max[3] = {std::min(n3_max[0], m->max_points), std::min(n3_max[1], m->max_points), m->publish ? std::min(n3_max[2], m->max_full) : INT_MAX};
  return pm_process(m, dsrc, m->publish ? reinterpret_cast<const float4 *>(full_dev) : nullptr, n3_dev, n_max, transform_sum7, transform_tobe_mapped7,
                    transform_aft_mapped7, info5, 5);
}

extern "C" int lio_pm_update_map_database_host(lio_pm *m, const float *corner_ds, int nc, const float *surf_ds, int ns, const long long *valid,
                                               int nv, const float tf7[7], const int margin_centre3[3]) {
  if (!m || m->attached || !tf7 || !margin_centre3 || nc < 0 || ns < 0 || nv < 0 || (nc > 0 && !corner_ds) || (ns > 0 && !surf_ds) || (nv > 0 && !valid))
    return LIO_ERR_INVALID;
  if (nc > m->max_points || ns > m->max_points || nv > 125) return LIO_ERR_CAPACITY;
  std::vector<size_t> v(valid, valid + nv);
  for (int i = 0; i < nv; ++i) {
    if (valid[i] < 0 || valid[i] >= kCubes) return LIO_ERR_INVALID;
    for (int k = 0; k < i; ++k) if (valid[k] == valid[i]) return LIO_ERR_INVALID;
  }
  LIO_CUDA_OK(cudaSetDevice(m->device));
  cudaStream_t st = m->stream;
  const int n_ds[2] = {nc, ns};
  if (nc > 0) LIO_CUDA_OK(cudaMemcpyAsync(m->d_ds[0], corner_ds, sizeof(float4) * nc, cudaMemcpyHostToDevice, st));
  if (ns > 0) LIO_CUDA_OK(cudaMemcpyAsync(m->d_ds[1], surf_ds, sizeof(float4) * ns, cudaMemcpyHostToDevice, st));
  LIO_CUDA_OK(cudaMemcpyAsync(m->d_cnt + 8, n_ds, sizeof(n_ds), cudaMemcpyHostToDevice, st));   // pageable: staged before the call returns
  const float4 *ds[2] = {m->d_ds[0], m->d_ds[1]};
  const int *n_ds_dev[2] = {m->d_cnt + 8, m->d_cnt + 9};
  return pm_update(m, v, ds, n_ds_dev, n_ds, tf7_to_twist(tf7), margin_centre3);
}

extern "C" int lio_pm_update_stats(lio_pm *m, int info4[4]) {
  if (!m || !info4) return LIO_ERR_INVALID;
  for (int k = 0; k < 4; ++k) info4[k] = m->upd_stats[k];
  return LIO_OK;
}

// ---- lio::MapBuilder (src/map_builder/MapBuilder.cc) -----------------------------------------------------------------------
static void mat3_mul(const float A[9], const float B[9], float C[9]) {   // Eigen's 3 x 3 float product, sum in k order
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { float s = 0.f; for (int k = 0; k < 3; ++k) s += A[i * 3 + k] * B[k * 3 + j]; C[i * 3 + j] = s; }
}

// Transform4DAssociateToMap (:55-75, DEBUG undefined): the odometry increment as in TransformAssociateToMap gives full_transform;
// tobe keeps its position and takes sum's rotation turned about z by the yaw difference yaw(full) - yaw(sum).
// R2ypr(R.cast<double>()).x() = atan2(R(1,0), R(0,0)) / M_PI * 180.0 (math_utils.h:188-203); ypr2R in float (:205-230) takes
// (float)y_diff / 180.0 * M_PI in double, rounds it to float and evaluates cos / sin in double.  The product rot_diff * sum.rot
// is a Matrix3f assigned to the quaternion by Eigen's matrix-to-quaternion conversion, without normalisation.
static TwistF transform_4d_associate(const TwistF &tobe, const TwistF &bef, const TwistF &sum) {
  const TwistF full = twist_mul(tobe, twist_mul(twist_inverse(bef), sum));
  float Rf[9], Rs[9];
  quat_to_matrix_normalized(full, Rf);
  quat_to_matrix_normalized(sum, Rs);
  const double yaw_full = std::atan2((double)Rf[3], (double)Rf[0]) / M_PI * 180.0;
  const double yaw_sum = std::atan2((double)Rs[3], (double)Rs[0]) / M_PI * 180.0;
  const float ypr[3] = {(float)(yaw_full - yaw_sum), 0.f, 0.f};
  float a[3], c[3], s[3];
  for (int i = 0; i < 3; ++i) { a[i] = (float)(ypr[i] / 180.0 * M_PI); c[i] = (float)std::cos((double)a[i]); s[i] = (float)std::sin((double)a[i]); }
  const float Rz[9] = {c[0], -s[0], 0.f, s[0], c[0], 0.f, 0.f, 0.f, 1.f};
  const float Ry[9] = {c[1], 0.f, s[1], 0.f, 1.f, 0.f, -s[1], 0.f, c[1]};
  const float Rx[9] = {1.f, 0.f, 0.f, 0.f, c[2], -s[2], 0.f, s[2], c[2]};
  float Rzy[9], rot_diff[9], R[9], q[4];
  mat3_mul(Rz, Ry, Rzy);
  mat3_mul(Rzy, Rx, rot_diff);
  mat3_mul(rot_diff, Rs, R);
  matrix_to_quat(R, q);
  return TwistF{q[0], q[1], q[2], q[3], full.px, full.py, full.pz};
}

// laser_cloud_surround_ (:156-163): each surround cube's corner cloud then its surf cloud, gathered into d_sur, followed by
// down_size_filter_map_ over the whole cloud (:166-168).  Buffers grow on demand; the count stays on the device in d_cnt[6].
static int mb_surround(lio_pm *m, const std::vector<size_t> &surround) {
  cudaStream_t st = m->stream;
  int rc = pm_counts(m);
  if (rc != LIO_OK) return rc;
  int nseg = 0, total = 0;
  for (size_t v : surround)
    for (int w = 0; w < 2; ++w) {
      const lio_pm::Cube &c = m->cube[w][v];
      if (c.n > 0) { m->h_sur_seg[nseg++] = Segment{c.p, c.n, total}; total += c.n; }
    }
  if (total == 0) { LIO_CUDA_OK(cudaMemsetAsync(m->d_cnt + 6, 0, sizeof(int), st)); return LIO_OK; }
  if (total > m->sur_cap) {
    if (m->d_sur) cudaFree(m->d_sur);
    if (m->d_sur_ds) cudaFree(m->d_sur_ds);
    m->d_sur = m->d_sur_ds = nullptr;
    m->vg_sur.destroy();
    m->sur_cap = 0;
    const int cap = std::max(2 * total, 1 << 16);
    LIO_CUDA_OK(cudaMalloc(&m->d_sur, sizeof(float4) * cap));
    LIO_CUDA_OK(cudaMalloc(&m->d_sur_ds, sizeof(float4) * cap));
    if (m->vg_sur.init(cap) != 0) { lio_set_last_error(__FILE__, __LINE__, "surround VoxelGrid allocation failed"); return LIO_ERR_CUDA; }
    m->sur_cap = cap;
  }
  *m->h_sur_n = total;
  LIO_CUDA_OK(cudaMemcpyAsync(m->d_sur_seg, m->h_sur_seg, sizeof(Segment) * nseg, cudaMemcpyHostToDevice, st));
  LIO_CUDA_OK(cudaMemcpyAsync(m->d_cnt + 5, m->h_sur_n, sizeof(int), cudaMemcpyHostToDevice, st));
  k_gather_segments<<<dim3(16, (unsigned)nseg), 256, 0, st>>>(m->d_sur_seg, nseg, m->d_sur);
  return m->vg_sur.run(m->d_sur, m->d_cnt + 5, total, m->map_leaf, m->d_sur_ds, m->sur_cap, m->d_cnt + 6, nullptr, st, nullptr);
}

// Buffers of the published clouds (full cloud in / registered, surround segments); the surround map itself grows on demand.
// On failure nothing stays allocated and the handle does not publish.
static bool pm_alloc_publish(lio_pm *m, int max_full_points) {
  m->max_full = max_full_points;
  bool ok = cudaMalloc(&m->d_full_in, sizeof(float4) * max_full_points) == cudaSuccess;
  ok = ok && cudaMalloc(&m->d_full_out, sizeof(float4) * max_full_points) == cudaSuccess;
  ok = ok && cudaMalloc(&m->d_sur_seg, sizeof(Segment) * 2 * 125) == cudaSuccess;
  ok = ok && cudaMallocHost(&m->h_sur_seg, sizeof(Segment) * 2 * 125) == cudaSuccess;
  ok = ok && cudaMallocHost(&m->h_sur_n, sizeof(int)) == cudaSuccess;
  if (!ok) {
    void *fr[] = {m->d_full_in, m->d_full_out, m->d_sur_seg};
    for (void *q : fr) if (q) cudaFree(q);
    if (m->h_sur_seg) cudaFreeHost(m->h_sur_seg);
    if (m->h_sur_n) cudaFreeHost(m->h_sur_n);
    m->d_full_in = m->d_full_out = nullptr; m->d_sur_seg = m->h_sur_seg = nullptr; m->h_sur_n = nullptr;
    m->max_full = 0;
  }
  return ok;
}

extern "C" void lio_mb_default_config(lio_mb_config *cfg) {
  if (!cfg) return;
  cfg->corner_filter_size = 0.2f; cfg->surf_filter_size = 0.4f; cfg->map_filter_size = 0.2f;
  cfg->min_match_sq_dis = 1.0f; cfg->min_plane_dis = 0.2f;
  cfg->enable_4d = 1; cfg->skip_count = 2; cfg->max_iterations = 10;
}

extern "C" int lio_mb_create(const lio_mb_config *cfg, int max_points, int max_full_points, int device, void *cuda_stream, lio_pm **out) {
  if (!cfg || !out || max_full_points < 1 || !(cfg->map_filter_size > 0) || cfg->skip_count < 1) return LIO_ERR_INVALID;
  lio_pm *m = nullptr;
  int rc = lio_pm_create(max_points, cfg->corner_filter_size, cfg->surf_filter_size, cfg->min_match_sq_dis, cfg->min_plane_dis,
                         cfg->max_iterations, device, cuda_stream, &m);
  if (rc != LIO_OK) return rc;
  m->mb = true; m->enable_4d = cfg->enable_4d != 0; m->skip_count = cfg->skip_count; m->map_leaf = cfg->map_filter_size;
  if (!pm_alloc_publish(m, max_full_points)) { lio_set_last_error(__FILE__, __LINE__, "lio_mb_create: allocation failed"); lio_pm_destroy(m); return LIO_ERR_CUDA; }
  *out = m;
  return LIO_OK;
}

extern "C" int lio_pm_enable_publish(lio_pm *m, float map_filter_size, int max_full_points) {
  if (!m || m->mb || m->publish || m->started || !(map_filter_size > 0) || max_full_points < 1) {
    if (m && (m->mb || m->publish || m->started))
      lio_set_last_error(__FILE__, __LINE__, "lio_pm_enable_publish: only once, on a plain PointMapping handle, before its first process call");
    return LIO_ERR_INVALID;
  }
  LIO_CUDA_OK(cudaSetDevice(m->device));
  if (!pm_alloc_publish(m, max_full_points)) { lio_set_last_error(__FILE__, __LINE__, "lio_pm_enable_publish: allocation failed"); return LIO_ERR_CUDA; }
  m->map_leaf = map_filter_size;
  m->publish = true;
  return LIO_OK;
}

// MapBuilder::ProcessMap (:220-622) for one synchronised (corner, surf, full, odometry) set + PublishMapBuilderResults (:144-218).
// Device sources, device counts {corner, surf, full}, host bounds n_max (already capped by the capacities).
static int mb_process_map(lio_pm *m, const float4 *const src[2], const float4 *full, const int *n3_dev, const int n_max[3],
                          const float transform_sum7[7], float transform_tobe_mapped7[7], float transform_aft_mapped7[7], int info6[6]) {
  const int nin[2] = {n_max[0], n_max[1]};
  int rc = pm_counts(m);
  if (rc != LIO_OK) return rc;
  m->sum = tf7_to_twist(transform_sum7);
  if (!m->system_init) { m->system_init = true; m->bef = m->sum; m->tobe = m->sum; m->aft = m->tobe; }   // :227-232
  if (m->enable_4d) m->tobe = transform_4d_associate(m->tobe, m->bef, m->sum);
  else m->tobe = twist_mul(m->tobe, twist_mul(twist_inverse(m->bef), m->sum));   // TransformAssociateToMap (PointMapping.cc:755-758)
  if ((rc = pm_stack(m, src, full, n3_dev, n_max)) != LIO_OK) return rc;
  int K[2] = {0, 0}, n_ds[2] = {0, 0};
  if ((rc = pm_locate(m, m->last_valid, &m->last_surround, K)) != LIO_OK) return rc;
  if ((rc = pm_downsample(m, nin, n_ds)) != LIO_OK) return rc;
  const int nf = n_max[2] > 0 ? m->h_cnt[4] : 0;
  // optimisation gate (:529-544): OptimizeMap / OptimizeTransformTobeMapped end with the update behind their early return
  // (:625-628, :1013); the skipped frames take Transform4DUpdate / TransformUpdate (:77-90)
  const bool gate = m->odom_count % m->skip_count == 0;
  m->last_iters = 0;
  if (gate) {
    const bool optimised = !(K[0] <= 10 || K[1] <= 100);
    if (optimised && (rc = pm_optimise(m, K, n_ds, m->enable_4d ? 1 : 0)) != LIO_OK) return rc;
    if (optimised) { m->bef = m->sum; m->aft = m->tobe; }
  } else {
    m->bef = m->sum; m->aft = m->tobe;
  }
  ++m->odom_count;
  const int cen[3] = {m->cen_l, m->cen_w, m->cen_h};   // margin centre == current centre: the valid list is this call's
  const float4 *ds[2] = {m->d_ds[0], m->d_ds[1]};
  const int *n_ds_dev[2] = {m->d_cnt + 2, m->d_cnt + 3};
  if ((rc = pm_update(m, m->last_valid, ds, n_ds_dev, n_ds, m->tobe, cen)) != LIO_OK) return rc;
  // PublishMapBuilderResults: surround map every num_map_frames_ (5) frames, registered full cloud every frame
  bool publish = false;
  if ((rc = pm_publish(m, m->last_surround, m->d_full_in, m->d_cnt + 4, nf, publish)) != LIO_OK) return rc;
  if (transform_tobe_mapped7) twist_to_tf7(m->tobe, transform_tobe_mapped7);
  if (transform_aft_mapped7) twist_to_tf7(m->aft, transform_aft_mapped7);
  if (info6) { info6[0] = m->last_iters; info6[1] = gate; info6[2] = K[0]; info6[3] = K[1]; info6[4] = publish; info6[5] = m->n_surround; }
  return LIO_OK;
}

extern "C" int lio_mb_process_map_host(lio_pm *m, const float *corner_last, int nc, const float *surf_last, int ns, const float *full_cloud, int nf,
                                       const float transform_sum7[7], float transform_tobe_mapped7[7], float transform_aft_mapped7[7], int info6[6]) {
  if (!m || !m->mb || !transform_sum7 || nc < 0 || ns < 0 || nf < 0 || (nc > 0 && !corner_last) || (ns > 0 && !surf_last) ||
      (nf > 0 && !full_cloud))
    return LIO_ERR_INVALID;
  if (nc > m->max_points || ns > m->max_points || nf > m->max_full) return LIO_ERR_CAPACITY;
  LIO_CUDA_OK(cudaSetDevice(m->device));
  const float *src[2] = {corner_last, surf_last};
  const int nin[2] = {nc, ns};
  int rc = pm_upload(m, src, nin, full_cloud, nf);
  if (rc != LIO_OK) return rc;
  const float4 *dsrc[2] = {m->d_in[0], m->d_in[1]};
  const int n_max[3] = {nc, ns, nf};
  return mb_process_map(m, dsrc, m->d_full_in, m->d_cnt + 8, n_max, transform_sum7, transform_tobe_mapped7, transform_aft_mapped7, info6);
}

extern "C" int lio_mb_process_map_dev(lio_pm *m, const float *corner_dev, const float *surf_dev, const float *full_dev, const int *n3_dev,
                                      const int n3_max[3], const float transform_sum7[7], float transform_tobe_mapped7[7],
                                      float transform_aft_mapped7[7], int info6[6]) {
  if (!m || !m->mb || !transform_sum7 || !n3_dev || !n3_max || n3_max[0] < 0 || n3_max[1] < 0 || n3_max[2] < 0 ||
      (n3_max[0] > 0 && !corner_dev) || (n3_max[1] > 0 && !surf_dev) || (n3_max[2] > 0 && !full_dev))
    return LIO_ERR_INVALID;
  LIO_CUDA_OK(cudaSetDevice(m->device));
  const float4 *dsrc[2] = {reinterpret_cast<const float4 *>(corner_dev), reinterpret_cast<const float4 *>(surf_dev)};
  const int n_max[3] = {std::min(n3_max[0], m->max_points), std::min(n3_max[1], m->max_points), std::min(n3_max[2], m->max_full)};
  return mb_process_map(m, dsrc, reinterpret_cast<const float4 *>(full_dev), n3_dev, n_max, transform_sum7, transform_tobe_mapped7,
                        transform_aft_mapped7, info6);
}

extern "C" int lio_mb_surround_dev(lio_pm *m, const float **ptr, int *n) {
  if (!m || !(m->mb || m->publish) || !ptr || !n) return LIO_ERR_INVALID;
  *ptr = (const float *)m->d_sur_ds; *n = m->n_surround;
  return LIO_OK;
}

extern "C" int lio_mb_full_dev(lio_pm *m, const float **ptr, int *n) {
  if (!m || !(m->mb || m->publish) || !ptr || !n) return LIO_ERR_INVALID;
  *ptr = (const float *)m->d_full_out; *n = m->n_full;
  return LIO_OK;
}

static int mb_download(lio_pm *m, const float4 *src, int count, float *out, int cap, int *n) {
  *n = count;
  if (count > cap) return LIO_ERR_CAPACITY;
  LIO_CUDA_OK(cudaSetDevice(m->device));
  if (count > 0) LIO_CUDA_OK(cudaMemcpyAsync(out, src, sizeof(float4) * count, cudaMemcpyDeviceToHost, m->stream));
  LIO_CUDA_OK(cudaStreamSynchronize(m->stream));
  return LIO_OK;
}

extern "C" int lio_mb_surround_download(lio_pm *m, float *out_xyzi, int cap, int *n) {
  if (!m || !(m->mb || m->publish) || !n || (!out_xyzi && cap > 0)) return LIO_ERR_INVALID;
  return mb_download(m, m->d_sur_ds, m->n_surround, out_xyzi, cap, n);
}

extern "C" int lio_mb_full_download(lio_pm *m, float *out_xyzi, int cap, int *n) {
  if (!m || !(m->mb || m->publish) || !n || (!out_xyzi && cap > 0)) return LIO_ERR_INVALID;
  return mb_download(m, m->d_full_out, m->n_full, out_xyzi, cap, n);
}

extern "C" int lio_pm_map_centre(lio_pm *m, int centre3[3]) {
  if (!m || !centre3) return LIO_ERR_INVALID;
  centre3[0] = m->cen_l; centre3[1] = m->cen_w; centre3[2] = m->cen_h;
  return LIO_OK;
}

extern "C" int lio_pm_cube_lists(lio_pm *m, long long valid[125], long long surround[125], int n2[2]) {
  if (!m || !n2) return LIO_ERR_INVALID;
  n2[0] = (int)m->last_valid.size(); n2[1] = (int)m->last_surround.size();
  if (valid) for (int i = 0; i < n2[0]; ++i) valid[i] = (long long)m->last_valid[i];
  if (surround) for (int i = 0; i < n2[1]; ++i) surround[i] = (long long)m->last_surround[i];
  return LIO_OK;
}

extern "C" int lio_pm_cube_size(lio_pm *m, int cube_index, int which, int *n) {
  if (!m || !n || cube_index < 0 || cube_index >= kCubes || which < 0 || which > 1) return LIO_ERR_INVALID;
  LIO_CUDA_OK(cudaSetDevice(m->device));
  int rc = pm_counts(m);
  if (rc != LIO_OK) return rc;
  *n = m->cube[which][cube_index].n;
  return LIO_OK;
}

extern "C" int lio_pm_cube_download(lio_pm *m, int cube_index, int which, float *out_xyzi, int cap) {
  if (!m || !out_xyzi || cube_index < 0 || cube_index >= kCubes || which < 0 || which > 1) return LIO_ERR_INVALID;
  LIO_CUDA_OK(cudaSetDevice(m->device));
  int rc = pm_counts(m);
  if (rc != LIO_OK) return rc;
  const lio_pm::Cube &c = m->cube[which][cube_index];
  if (c.n > cap) return LIO_ERR_CAPACITY;
  if (c.n > 0) LIO_CUDA_OK(cudaMemcpyAsync(out_xyzi, c.p, sizeof(float4) * c.n, cudaMemcpyDeviceToHost, m->stream));
  LIO_CUDA_OK(cudaStreamSynchronize(m->stream));
  return LIO_OK;
}

// ---- the device estimator's map after initialisation (cubemap.cuh, lio_est_attach_map) ------------------------------------
int pm_attach(lio_pm *m, int device, float corner_leaf, float surf_leaf, int ins_bound, int full_bound) {
  if (!m || m->mb || !m->publish || !m->started || m->attached || m->device != device) {
    lio_set_last_error(__FILE__, __LINE__, "lio_est_attach_map: needs a publishing PointMapping (lio_pm_enable_publish) on the estimator's device "
                                           "that has run a process call and is not attached");
    return LIO_ERR_INVALID;
  }
  if (m->leaf[0] != corner_leaf || m->leaf[1] != surf_leaf) {
    lio_set_last_error(__FILE__, __LINE__, "lio_est_attach_map: the map's corner / surf leaf sizes differ from the estimator's");
    return LIO_ERR_INVALID;
  }
  if (m->max_full < full_bound) {
    lio_set_last_error(__FILE__, __LINE__, "lio_est_attach_map: the map's max_full_points is below the estimator's full-cloud capacity");
    return LIO_ERR_CAPACITY;
  }
  LIO_CUDA_OK(cudaSetDevice(m->device));
  int rc = pm_counts(m);
  if (rc != LIO_OK) return rc;
  if (ins_bound > m->ins_cap) {   // an accumulated surf slot exceeds 2 * max_points: new insert buffers, swapped in on success
    LIO_CUDA_OK(cudaStreamSynchronize(m->stream));
    float4 *mapped = nullptr;
    unsigned *k[2] = {nullptr, nullptr}, *v[2] = {nullptr, nullptr};
    RadixSortTemp rs;
    bool ok = cudaMalloc(&mapped, sizeof(float4) * ins_bound) == cudaSuccess;
    for (int b = 0; b < 2 && ok; ++b) {
      ok = ok && cudaMalloc(&k[b], sizeof(unsigned) * ins_bound) == cudaSuccess;
      ok = ok && cudaMalloc(&v[b], sizeof(unsigned) * ins_bound) == cudaSuccess;
    }
    ok = ok && rs.init(ins_bound) == 0;
    if (!ok) {
      void *fr[] = {mapped, k[0], k[1], v[0], v[1]};
      for (void *q : fr) if (q) cudaFree(q);
      rs.destroy();
      lio_set_last_error(__FILE__, __LINE__, "lio_est_attach_map: insert buffer allocation failed");
      return LIO_ERR_CUDA;
    }
    void *fr[] = {m->d_mapped, m->d_ins_k[0], m->d_ins_k[1], m->d_ins_v[0], m->d_ins_v[1]};
    for (void *q : fr) cudaFree(q);
    m->ins_rs.destroy();
    m->d_mapped = mapped;
    for (int b = 0; b < 2; ++b) { m->d_ins_k[b] = k[b]; m->d_ins_v[b] = v[b]; }
    m->ins_rs = rs;
    m->ins_cap = ins_bound;
  }
  m->attached = true;
  return LIO_OK;
}

void pm_detach(lio_pm *m) { if (m) m->attached = false; }
cudaStream_t pm_stream(const lio_pm *m) { return m->stream; }
TwistF *pm_tobe(lio_pm *m) { return &m->tobe; }
TwistF pm_aft(const lio_pm *m) { return m->aft; }

int pm_est_step(lio_pm *m, bool insert, const float4 *const src[2], const int *const n_dev[2], const int bound[2], const TwistF &pose,
                const float4 *full, const int *nf_dev, int nf, int info4[4]) {
  int rc = LIO_OK;
  if (insert) {
    const int cen[3] = {m->cen_l, m->cen_w, m->cen_h};   // opt_cube_centers_: the centre is frozen with the valid list
    if ((rc = pm_update(m, m->last_valid, src, n_dev, bound, pose, cen)) != LIO_OK) return rc;
  }
  bool published = false;
  if ((rc = pm_publish(m, m->last_surround, full, nf_dev, nf, published)) != LIO_OK) return rc;
  info4[0] = insert ? 1 : 0; info4[1] = insert ? m->upd_stats[3] : 0; info4[2] = published ? 1 : 0; info4[3] = m->n_surround;
  return LIO_OK;
}
