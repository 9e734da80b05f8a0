// Device pcl::VoxelGrid<PointXYZI> (PCL 1.8 semantics, SURVEY.md App. A.2) for the estimator's
// call sites (reference: src/imu_processor/Estimator.cc:679-687, :1518-1519).  Compiled with
// -fmad=false: voxel indices, output order (ascending voxel index) and centroids (float sums in
// input order inside a voxel, divided by the float count) are bit-identical to the CPU path.
//
//   vg_bbox   : min/max of the cloud (order-preserving uint encoding + atomics)
//   vg_keys   : ijk = floor(p*inv_leaf) - min_b, key = i + j*dx + k*dx*dy, value = input index
//   radix sort: stable, 4 x 8-bit passes (sort.cu)
//   vg_emit   : heads of equal-key runs -> ordered compaction by decoupled look-back, one centroid
//               per occupied voxel
//
// SegVoxelGrid runs the same steps over many clouds at once (UpdateMapDatabase's re-filter of the valid cubes).
#include <algorithm>
#include <vector>
#include "voxel.cuh"

namespace lio {

__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// Also publishes n_eff = min(*n_dev, n_max): every later kernel of the filter (and the radix sort) reads the clamped
// count, so a caller-side count above the grid / scratch bound cannot run past the buffers.
__global__ void vg_reset(unsigned *bbox, int *ticket, const int *__restrict__ n_dev, int n_max, int *__restrict__ n_eff) {
  if (threadIdx.x < 3) bbox[threadIdx.x] = 0xffffffffu;
  else if (threadIdx.x < 6) bbox[threadIdx.x] = 0u;
  if (threadIdx.x == 6) *ticket = 0;
  if (threadIdx.x == 7) { int n = *n_dev; *n_eff = n < 0 ? 0 : (n > n_max ? n_max : n); }
}

__global__ void __launch_bounds__(256)
vg_bbox(const float4 *__restrict__ in, const int *__restrict__ n_dev, unsigned *__restrict__ bbox) {
  const int n = *n_dev;
  float mn0 = INFINITY, mn1 = INFINITY, mn2 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY, mx2 = -INFINITY;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float4 p = __ldg(in + i);
    mn0 = fminf(mn0, p.x); mn1 = fminf(mn1, p.y); mn2 = fminf(mn2, p.z);
    mx0 = fmaxf(mx0, p.x); mx1 = fmaxf(mx1, p.y); mx2 = fmaxf(mx2, p.z);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn0 = fminf(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mn1 = fminf(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
    mn2 = fminf(mn2, __shfl_xor_sync(0xffffffffu, mn2, o)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o)); mx2 = fmaxf(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
  }
  // one set of atomics per CTA, not per warp: with hundreds of CTAs the six addresses serialise (17 us measured)
  __shared__ float sm[256 / 32][6];
  if (lane_id() == 0) { float *r = sm[warp_id()]; r[0] = mn0; r[1] = mn1; r[2] = mn2; r[3] = mx0; r[4] = mx1; r[5] = mx2; }
  __syncthreads();
  if (threadIdx.x < 6) {
    const bool is_min = threadIdx.x < 3;
    float v = sm[0][threadIdx.x];
#pragma unroll
    for (int w = 1; w < 256 / 32; ++w) v = is_min ? fminf(v, sm[w][threadIdx.x]) : fmaxf(v, sm[w][threadIdx.x]);
    if (is_min) { if (v != INFINITY) atomicMin(bbox + threadIdx.x, f2ord(v)); }
    else { if (v != -INFINITY) atomicMax(bbox + threadIdx.x, f2ord(v)); }
  }
}

__global__ void __launch_bounds__(256)
vg_keys(const float4 *__restrict__ in, const int *__restrict__ n_dev, const unsigned *__restrict__ bbox, float leaf,
        unsigned *__restrict__ keys, unsigned *__restrict__ vals, int *__restrict__ overflow) {
  __shared__ int sp[6];
  const int n = *n_dev;
  if (blockIdx.x * blockDim.x >= n) return;
  const float inv = 1.0f / leaf;
  if (threadIdx.x == 0) {
    float a[6];
    for (int q = 0; q < 6; ++q) a[q] = ord2f(bbox[q]);
    long long ddx = (long long)((a[3] - a[0]) * inv) + 1, ddy = (long long)((a[4] - a[1]) * inv) + 1,
              ddz = (long long)((a[5] - a[2]) * inv) + 1;
    int ovf = (ddx * ddy * ddz > 2147483647LL) ? 1 : 0;
    int mb0 = (int)floorf(a[0] * inv), mb1 = (int)floorf(a[1] * inv), mb2 = (int)floorf(a[2] * inv);
    int xb0 = (int)floorf(a[3] * inv), xb1 = (int)floorf(a[4] * inv);
    sp[0] = mb0; sp[1] = mb1; sp[2] = mb2;
    sp[3] = xb0 - mb0 + 1;
    sp[4] = (xb0 - mb0 + 1) * (xb1 - mb1 + 1);
    sp[5] = ovf;
    if (blockIdx.x == 0 && ovf) *overflow = 1;   // sticky until the host reads and clears it
  }
  __syncthreads();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    float4 p = __ldg(in + i);
    int ijk0 = (int)(floorf(p.x * inv) - (float)sp[0]);
    int ijk1 = (int)(floorf(p.y * inv) - (float)sp[1]);
    int ijk2 = (int)(floorf(p.z * inv) - (float)sp[2]);
    keys[i] = sp[5] ? (unsigned)i : (unsigned)(ijk0 + ijk1 * sp[3] + ijk2 * sp[4]);
    vals[i] = (unsigned)i;
  }
}

constexpr int kEmitThreads = 256;

__global__ void __launch_bounds__(kEmitThreads)
vg_emit(const float4 *__restrict__ in, const int *__restrict__ n_dev, const unsigned *__restrict__ keys,
        const unsigned *__restrict__ vals, float4 *__restrict__ out, int out_cap, int *__restrict__ nout_dev,
        unsigned *__restrict__ vox_key_out, unsigned long long *__restrict__ status, int *__restrict__ ticket) {
  __shared__ int sscan[40];
  __shared__ int stile, sbc;
  const int n = *n_dev;
  const int ntiles = (n + kEmitThreads - 1) / kEmitThreads;
  if (threadIdx.x == 0) stile = atomicAdd(ticket, 1);
  __syncthreads();
  const int tile = stile;
  if (tile >= ntiles) {
    if (n == 0 && tile == 0 && threadIdx.x == 0) *nout_dev = 0;
    return;
  }
  const int c = tile * kEmitThreads + threadIdx.x;
  int head = 0;
  unsigned v = 0;
  if (c < n) {
    v = keys[c];
    head = (c == 0) || (v != keys[c - 1]);
  }
  int tot;
  int lpos = block_scan_excl(head, sscan, &tot);
  int excl = lookback_exclusive(status, tile, tot, &sbc);
  if (head) {
    float ax = 0.f, ay = 0.f, az = 0.f, ai = 0.f;
    int cnt = 0;
    for (int c2 = c; c2 < n && keys[c2] == v; ++c2) {
      float4 p = __ldg(in + vals[c2]);
      ax += p.x; ay += p.y; az += p.z; ai += p.w;
      ++cnt;
    }
    float fn = (float)cnt;
    if (excl + lpos < out_cap) {   // the count below keeps growing: the host compares it with the capacity
      out[excl + lpos] = make_float4(ax / fn, ay / fn, az / fn, ai / fn);
      if (vox_key_out) vox_key_out[excl + lpos] = v;
    }
  }
  if (tile == ntiles - 1 && threadIdx.x == 0) *nout_dev = excl + tot;
}

int VoxelGrid::init(int cap_) {
  cap = cap_;
  nstatus = (cap + kEmitThreads - 1) / kEmitThreads + 1;
  if (!alloc(keys_a, cap) || !alloc(vals_a, cap) || !alloc(keys_b, cap) || !alloc(vals_b, cap) || rs.init(cap) != 0 ||
      !alloc(status, nstatus) || !alloc(bbox, 8) || !alloc(ticket, 4) || cudaMemset(ticket, 0, sizeof(int) * 4) != cudaSuccess)
    return -1;
  return 0;
}

int VoxelGrid::run(const float4 *in, const int *n_dev_in, int n_max, float leaf, float4 *out, int out_cap, int *nout_dev,
                   unsigned *vox_key_out, cudaStream_t st, int *launches) {
  if (n_max > cap) return LIO_ERR_CAPACITY;
  if (n_max <= 0) n_max = 1;
  int *overflow = ticket + 1;
  int *n_dev = ticket + 2;   // clamped copy of the caller's count
  vg_reset<<<1, 32, 0, st>>>(bbox, ticket, n_dev_in, n_max, n_dev);
  int nblk = (n_max + 255) / 256;
  int bb_blocks = nblk < 592 ? nblk : 592;
  vg_bbox<<<bb_blocks, 256, 0, st>>>(in, n_dev, bbox);
  vg_keys<<<nblk, 256, 0, st>>>(in, n_dev, bbox, leaf, keys_a, vals_a, overflow);
  if (launches) *launches += 3;
  int which = radix_sort_pairs(keys_a, vals_a, keys_b, vals_b, n_dev, n_max, 32, rs, st, launches);
  if (which < 0) return LIO_ERR_CAPACITY;
  const unsigned *k = which ? keys_b : keys_a, *v = which ? vals_b : vals_a;
  int etiles = (n_max + kEmitThreads - 1) / kEmitThreads;
  cudaMemsetAsync(status, 0, sizeof(unsigned long long) * (size_t)(etiles + 1), st);
  vg_emit<<<etiles, kEmitThreads, 0, st>>>(in, n_dev, k, v, out, out_cap, nout_dev, vox_key_out, status, ticket);
  if (launches) *launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

// ---- segmented VoxelGrid ------------------------------------------------------------------------------------------------
// The kernels repeat vg_bbox / vg_keys / vg_emit per job, in the same float expressions.
__global__ void vg_seg_reset(unsigned *__restrict__ jbbox, int njobs, int total, int *__restrict__ ticket) {
  for (int t = threadIdx.x; t < 6 * njobs; t += blockDim.x) jbbox[t] = (t % 6 < 3) ? 0xffffffffu : 0u;
  if (threadIdx.x == 0) { ticket[0] = 0; ticket[1] = 0; ticket[2] = total; }
}

// concatenation of the jobs (blockIdx.y = job), the job id of every point (into the key buffer) and every job's bounding box
__global__ void __launch_bounds__(256)
vg_seg_gather(const VgJob *__restrict__ jobs, float4 *__restrict__ cat, unsigned *__restrict__ job_of, unsigned *__restrict__ jbbox) {
  const int j = blockIdx.y;
  const VgJob jb = jobs[j];
  float mn0 = INFINITY, mn1 = INFINITY, mn2 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY, mx2 = -INFINITY;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < jb.n; i += gridDim.x * blockDim.x) {
    const float4 p = jb.p[i];
    cat[jb.off + i] = p;
    job_of[jb.off + i] = (unsigned)j;
    mn0 = fminf(mn0, p.x); mn1 = fminf(mn1, p.y); mn2 = fminf(mn2, p.z);
    mx0 = fmaxf(mx0, p.x); mx1 = fmaxf(mx1, p.y); mx2 = fmaxf(mx2, p.z);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn0 = fminf(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mn1 = fminf(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
    mn2 = fminf(mn2, __shfl_xor_sync(0xffffffffu, mn2, o)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o)); mx2 = fmaxf(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
  }
  __shared__ float sm[256 / 32][6];
  if (lane_id() == 0) { float *r = sm[warp_id()]; r[0] = mn0; r[1] = mn1; r[2] = mn2; r[3] = mx0; r[4] = mx1; r[5] = mx2; }
  __syncthreads();
  if (threadIdx.x < 6) {
    const bool is_min = threadIdx.x < 3;
    float v = sm[0][threadIdx.x];
#pragma unroll
    for (int w = 1; w < 256 / 32; ++w) v = is_min ? fminf(v, sm[w][threadIdx.x]) : fmaxf(v, sm[w][threadIdx.x]);
    if (is_min) { if (v != INFINITY) atomicMin(jbbox + 6 * j + threadIdx.x, f2ord(v)); }
    else { if (v != -INFINITY) atomicMax(jbbox + 6 * j + threadIdx.x, f2ord(v)); }
  }
}

// key = (job << 24) | PCL voxel index inside the job's own grid, value = position in the concatenation.  keys holds the job ids on
// entry.  A job whose grid has more than 2^24 voxels raises the error flag (below that bound PCL's INT_MAX check cannot fire).
__global__ void __launch_bounds__(256)
vg_seg_keys(const float4 *__restrict__ cat, const int *__restrict__ n_dev, const VgJob *__restrict__ jobs, const unsigned *__restrict__ jbbox,
            unsigned *__restrict__ keys, unsigned *__restrict__ vals, int *__restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *n_dev) return;
  const unsigned j = keys[i];
  const float inv = 1.0f / jobs[j].leaf;
  float a[6];
  for (int q = 0; q < 6; ++q) a[q] = ord2f(jbbox[6 * j + q]);
  const int mb0 = (int)floorf(a[0] * inv), mb1 = (int)floorf(a[1] * inv), mb2 = (int)floorf(a[2] * inv);
  const int xb0 = (int)floorf(a[3] * inv), xb1 = (int)floorf(a[4] * inv), xb2 = (int)floorf(a[5] * inv);
  const long long d0 = (long long)xb0 - mb0 + 1, d1 = (long long)xb1 - mb1 + 1, d2 = (long long)xb2 - mb2 + 1;
  if (d0 * d1 * d2 > (1LL << kVgJobBits)) *err = 1;
  const int s3 = (int)d0, s4 = (int)(d0 * d1);
  const float4 p = __ldg(cat + i);
  const int ijk0 = (int)(floorf(p.x * inv) - (float)mb0);
  const int ijk1 = (int)(floorf(p.y * inv) - (float)mb1);
  const int ijk2 = (int)(floorf(p.z * inv) - (float)mb2);
  keys[i] = (j << kVgJobBits) | ((unsigned)(ijk0 + ijk1 * s3 + ijk2 * s4) & ((1u << kVgJobBits) - 1u));
  vals[i] = (unsigned)i;
}

// vg_emit over the sorted concatenation; the first centroid of every job records where the job's output starts
__global__ void __launch_bounds__(kEmitThreads)
vg_seg_emit(const float4 *__restrict__ in, const int *__restrict__ n_dev, const unsigned *__restrict__ keys, const unsigned *__restrict__ vals,
            float4 *__restrict__ out, int njobs, int *__restrict__ jstart, unsigned long long *__restrict__ status, int *__restrict__ ticket) {
  __shared__ int sscan[40];
  __shared__ int stile, sbc;
  const int n = *n_dev;
  const int ntiles = (n + kEmitThreads - 1) / kEmitThreads;
  if (threadIdx.x == 0) stile = atomicAdd(ticket, 1);
  __syncthreads();
  const int tile = stile;
  if (tile >= ntiles) return;
  const int c = tile * kEmitThreads + threadIdx.x;
  int head = 0;
  unsigned v = 0;
  if (c < n) {
    v = keys[c];
    head = (c == 0) || (v != keys[c - 1]);
  }
  int tot;
  const int lpos = block_scan_excl(head, sscan, &tot);
  const int excl = lookback_exclusive(status, tile, tot, &sbc);
  if (head) {
    float ax = 0.f, ay = 0.f, az = 0.f, ai = 0.f;
    int cnt = 0;
    for (int c2 = c; c2 < n && keys[c2] == v; ++c2) {
      float4 p = __ldg(in + vals[c2]);
      ax += p.x; ay += p.y; az += p.z; ai += p.w;
      ++cnt;
    }
    float fn = (float)cnt;
    out[excl + lpos] = make_float4(ax / fn, ay / fn, az / fn, ai / fn);
    if (c == 0 || (keys[c - 1] >> kVgJobBits) != (v >> kVgJobBits)) jstart[v >> kVgJobBits] = excl + lpos;
  }
  if (tile == ntiles - 1 && threadIdx.x == 0) jstart[njobs] = excl + tot;
}

// every job's centroids back over its own input (blockIdx.y = job), its output count, and the error flag after the last job
__global__ void __launch_bounds__(256)
vg_seg_scatter(const VgJob *__restrict__ jobs, int njobs, const float4 *__restrict__ out, const int *__restrict__ jstart,
               const int *__restrict__ ticket, int *__restrict__ jn) {
  const int j = blockIdx.y;
  const int s = jstart[j], e = jstart[j + 1];
  float4 *dst = jobs[j].p;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < e - s; i += gridDim.x * blockDim.x) dst[i] = out[s + i];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    jn[j] = e - s;
    if (j == 0) jn[njobs] = ticket[1];
  }
}

int SegVoxelGrid::init() {
  return alloc(d_jobs, kVgMaxJobs) && alloc(jbbox, 6 * kVgMaxJobs) && alloc(jstart, kVgMaxJobs + 1) && alloc(jn, kVgMaxJobs + 1) ? 0 : -1;
}

int SegVoxelGrid::reserve(int total) {
  if (total <= cap) return 0;
  // the old workspace goes before the new one is allocated: nothing in it outlives a run
  ws = VoxelGrid{};
  cat = {};
  out = {};
  cap = 0;
  const int c = std::max(2 * total, 1 << 16);
  if (ws.init(c) != 0 || !alloc(cat, c) || !alloc(out, c)) return -1;
  cap = c;
  return 0;
}

int SegVoxelGrid::run(const VgJob *h_jobs, int njobs, int total, int *h_jn, cudaStream_t st, int *launches) {
  if (njobs < 1 || njobs > kVgMaxJobs || total < 1 || total > cap) return LIO_ERR_CAPACITY;
  LIO_CUDA_OK(cudaMemcpyAsync(d_jobs, h_jobs, sizeof(VgJob) * njobs, cudaMemcpyHostToDevice, st));
  int *n_dev = ws.ticket + 2;
  vg_seg_reset<<<1, 256, 0, st>>>(jbbox, njobs, total, ws.ticket);
  vg_seg_gather<<<dim3(16, (unsigned)njobs), 256, 0, st>>>(d_jobs, cat, ws.keys_a, jbbox);
  vg_seg_keys<<<(total + 255) / 256, 256, 0, st>>>(cat, n_dev, d_jobs, jbbox, ws.keys_a, ws.vals_a, ws.ticket + 1);
  if (launches) *launches += 3;
  const int which = radix_sort_pairs(ws.keys_a, ws.vals_a, ws.keys_b, ws.vals_b, n_dev, total, 32, ws.rs, st, launches);
  if (which < 0) return LIO_ERR_CAPACITY;
  const unsigned *k = which ? ws.keys_b : ws.keys_a, *v = which ? ws.vals_b : ws.vals_a;
  const int etiles = (total + kEmitThreads - 1) / kEmitThreads;
  LIO_CUDA_OK(cudaMemsetAsync(ws.status, 0, sizeof(unsigned long long) * (size_t)(etiles + 1), st));
  vg_seg_emit<<<etiles, kEmitThreads, 0, st>>>(cat, n_dev, k, v, out, njobs, jstart, ws.status, ws.ticket);
  vg_seg_scatter<<<dim3(16, (unsigned)njobs), 256, 0, st>>>(d_jobs, njobs, out, jstart, ws.ticket, jn);
  if (launches) *launches += 2;
  LIO_CUDA_OK(cudaMemcpyAsync(h_jn, jn, sizeof(int) * (njobs + 1), cudaMemcpyDeviceToHost, st));
  LIO_CUDA_OK(cudaGetLastError());
  return LIO_OK;
}

}  // namespace lio

// ---- C-ABI: standalone voxel filter on host buffers (parity entry for the PCL call sites) -------
using namespace lio;

extern "C" int lio_voxel_grid_host(const float *cloud, int n, float leaf, float *out, int cap, int *n_out, int device) {
  if ((!cloud && n > 0) || n < 0 || !n_out || !(leaf > 0)) return LIO_ERR_INVALID;
  LIO_TRY(select_device(device));
  *n_out = 0;
  if (n == 0) return LIO_OK;
  DevBufs d;
  VoxelGrid vg;
  float4 *d_in = nullptr, *d_out = nullptr;
  int *d_n = nullptr;
  int rc = LIO_OK;
  if (vg.init(n) != 0) { lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed"); rc = LIO_ERR_CUDA; }
  else if (!d.alloc(&d_in, n) || !d.alloc(&d_out, n) || !d.alloc(&d_n, 2) || !d.up(d_in, (const float4 *)cloud, n) || !d.up(d_n, &n, 1))
    rc = LIO_ERR_CUDA;
  if (rc == LIO_OK) rc = vg.run(d_in, d_n, n, leaf, d_out, n, d_n + 1, nullptr, 0, nullptr);
  int m = 0;
  if (rc == LIO_OK && !d.down(&m, d_n + 1, 1)) rc = LIO_ERR_CUDA;
  if (rc == LIO_OK) {
    *n_out = m;
    if (m > cap) rc = LIO_ERR_CAPACITY;
    else if (!d.down((float4 *)out, d_out, m)) rc = LIO_ERR_CUDA;
  }
  return rc;
}

// ---- C-ABI test aid: SegVoxelGrid::run on concatenated host clouds ------------------------------------------------------
extern "C" int lio_seg_voxel_grid_host(const float *xyzi, const int *n_per_job, const float *leaf_per_job, int njobs, float *out,
                                       int *n_out_per_job, int *index_bound_error, int device) {
  if (!xyzi || !n_per_job || !leaf_per_job || !out || !n_out_per_job || !index_bound_error || njobs < 1) return LIO_ERR_INVALID;
  long long total = 0;
  for (int j = 0; j < njobs; ++j) {
    if (n_per_job[j] < 1 || !(leaf_per_job[j] > 0)) return LIO_ERR_INVALID;
    total += n_per_job[j];
  }
  if (njobs > kVgMaxJobs || total >= (1LL << 30)) return LIO_ERR_CAPACITY;
  LIO_TRY(select_device(device));
  *index_bound_error = 0;
  DevBufs db;
  SegVoxelGrid sg;
  float4 *d = nullptr;
  std::vector<VgJob> jobs(njobs);
  std::vector<int> jn(njobs + 1, 0);
  int rc = LIO_OK;
  if (sg.init() != 0 || sg.reserve((int)total) != 0) { lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed"); rc = LIO_ERR_CUDA; }
  else if (!db.alloc(&d, total) || !db.up(d, (const float4 *)xyzi, total)) rc = LIO_ERR_CUDA;
  if (rc == LIO_OK) {
    for (int j = 0, off = 0; j < njobs; off += n_per_job[j], ++j) jobs[j] = VgJob{d + off, n_per_job[j], off, leaf_per_job[j]};
    rc = sg.run(jobs.data(), njobs, (int)total, jn.data(), 0, nullptr);
    if (rc == LIO_OK && !db.ok(cudaDeviceSynchronize())) rc = LIO_ERR_CUDA;
  }
  if (rc == LIO_OK) {
    for (int j = 0; j < njobs; ++j) n_out_per_job[j] = jn[j];
    *index_bound_error = jn[njobs] != 0;
    if (*index_bound_error) {
      lio_set_last_error(__FILE__, __LINE__, "a job's voxel grid exceeds 2^24 voxels");
      rc = LIO_ERR_CAPACITY;
    } else if (!db.down((float4 *)out, d, total)) {
      rc = LIO_ERR_CUDA;
    }
  }
  return rc;
}
