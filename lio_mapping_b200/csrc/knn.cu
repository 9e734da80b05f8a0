// Stage B on sm_90a — HBM-resident voxel-hash fixed-radius k-NN + plane fit, replacing
// pcl::KdTreeFLANN::nearestKSearch + the per-point body of Estimator::CalculateFeatures
// (reference: src/imu_processor/Estimator.cc:970-1097; PointAssociateToMap PointMapping.cc:303-314).
//
// Exactness argument (SURVEY.md §7.1-4): the reference rejects a match whose 5th neighbour has
// d^2 >= min_match_sq_dis, so an exact top-5 among all map points within sqrt(min_match_sq_dis)
// equals the unbounded kd-tree answer for every accepted feature.  With cells of edge >= that
// radius (+2^-10 margin) all such points lie in the 3x3x3 cell block around the query.  Ties are
// broken by (d^2, map index), the oracle's documented order.  Compiled with -fmad=false; float
// expressions follow the reference's source order, so accepted feature sets and coefficients are
// bit-identical to the CPU path.
//
//   ch_insert / ch_scan / ch_scatter : open-addressing hash of occupied cells -> contiguous
//                                      per-cell point ranges (counting sort by hash slot)
//   knn_plane : one thread per surf point: transform, scan 27 cells keeping the top-5 in
//               registers, 5x3 column-pivoted Householder QR plane fit, validity / score / FOV
//               tests, ordered compaction of accepted features by decoupled look-back
#include "knn.cuh"
#include "qr.cuh"

namespace lio {

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int kHashThreads = 256;
constexpr int kKnnThreads = 256;

__device__ __forceinline__ unsigned long long pack_cell(int cx, int cy, int cz) {
  const int off = 1 << 20;
  unsigned long long a = (unsigned)(min(max(cx + off, 0), (1 << 21) - 1));
  unsigned long long b = (unsigned)(min(max(cy + off, 0), (1 << 21) - 1));
  unsigned long long c = (unsigned)(min(max(cz + off, 0), (1 << 21) - 1));
  return a | (b << 21) | (c << 42);
}
__device__ __forceinline__ unsigned hash_cell(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (unsigned)k;
}

__global__ void __launch_bounds__(kHashThreads)
ch_insert(const float4 *__restrict__ map, const int *__restrict__ n_dev, float inv_cell, unsigned long long *__restrict__ keys,
          int *__restrict__ count, int mask, int *__restrict__ slot_of, int *__restrict__ rank_of) {
  const int n = *n_dev;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = __ldg(map + i);
  unsigned long long key = pack_cell((int)floorf(p.x * inv_cell), (int)floorf(p.y * inv_cell), (int)floorf(p.z * inv_cell));
  unsigned s = hash_cell(key) & mask;
  while (true) {
    unsigned long long prev = atomicCAS(keys + s, kEmptyKey, key);
    if (prev == kEmptyKey || prev == key) break;
    s = (s + 1) & mask;
  }
  slot_of[i] = (int)s;
  rank_of[i] = atomicAdd(count + s, 1);
}

// exclusive scan of count[0..table_size) -> start[], single pass with decoupled look-back
constexpr int kScanPer = 4;
__global__ void __launch_bounds__(kHashThreads)
ch_scan(const int *__restrict__ count, int *__restrict__ start, int table_size, unsigned long long *__restrict__ status,
        int *__restrict__ ticket) {
  __shared__ int sscan[40];
  __shared__ int stile, sbc;
  if (threadIdx.x == 0) stile = atomicAdd(ticket, 1);
  __syncthreads();
  const int tile = stile;
  const int base = tile * kHashThreads * kScanPer + threadIdx.x * kScanPer;
  int v[kScanPer], s = 0;
#pragma unroll
  for (int k = 0; k < kScanPer; ++k) { v[k] = (base + k < table_size) ? count[base + k] : 0; s += v[k]; }
  int tot;
  int lex = block_scan_excl(s, sscan, &tot);
  int excl = lookback_exclusive(status, tile, tot, &sbc);
  int run = excl + lex;
#pragma unroll
  for (int k = 0; k < kScanPer; ++k) { if (base + k < table_size) start[base + k] = run; run += v[k]; }
}

__global__ void __launch_bounds__(kHashThreads)
ch_scatter(const float4 *__restrict__ map, const int *__restrict__ n_dev, const int *__restrict__ start,
           const int *__restrict__ slot_of, const int *__restrict__ rank_of, float4 *__restrict__ cellpts) {
  const int n = *n_dev;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = __ldg(map + i);
  cellpts[start[slot_of[i]] + rank_of[i]] = make_float4(p.x, p.y, p.z, __int_as_float(i));
}

int CellHash::init(int cap) {
  cap_points = cap;
  table_size = 1024;
  while (table_size < 2 * cap) table_size <<= 1;
  eff_size = table_size;
  int ntiles = table_size / (kHashThreads * kScanPer) + 1;
  if (cudaMalloc(&keys, sizeof(unsigned long long) * table_size) != cudaSuccess) return -1;
  if (cudaMalloc(&count, sizeof(int) * table_size) != cudaSuccess) return -1;
  if (cudaMalloc(&start, sizeof(int) * table_size) != cudaSuccess) return -1;
  if (cudaMalloc(&slot_of, sizeof(int) * cap) != cudaSuccess) return -1;
  if (cudaMalloc(&rank_of, sizeof(int) * cap) != cudaSuccess) return -1;
  if (cudaMalloc(&cellpts, sizeof(float4) * cap) != cudaSuccess) return -1;
  if (cudaMalloc(&status, sizeof(unsigned long long) * ntiles) != cudaSuccess) return -1;
  if (cudaMalloc(&ticket, sizeof(int)) != cudaSuccess) return -1;
  return 0;
}
void CellHash::destroy() {
  void *p[] = {keys, count, start, slot_of, rank_of, cellpts, status, ticket};
  for (void *q : p) if (q) cudaFree(q);
  keys = nullptr; count = start = slot_of = rank_of = ticket = nullptr; cellpts = nullptr; status = nullptr;
}

int CellHash::build(const float4 *map, const int *n_dev, int n_max, float cell_size, cudaStream_t st, int *launches) {
  if (n_max > cap_points) return LIO_ERR_CAPACITY;
  cell = cell_size;
  inv_cell = 1.0f / cell_size;
  eff_size = 1024;
  while (eff_size < 2 * n_max) eff_size <<= 1;
  if (eff_size > table_size) eff_size = table_size;
  const int table_size = eff_size;   // everything below works on the slots in use
  int ntiles = (table_size + kHashThreads * kScanPer - 1) / (kHashThreads * kScanPer);
  cudaMemsetAsync(keys, 0xff, sizeof(unsigned long long) * table_size, st);
  cudaMemsetAsync(count, 0, sizeof(int) * table_size, st);
  cudaMemsetAsync(status, 0, sizeof(unsigned long long) * ntiles, st);
  cudaMemsetAsync(ticket, 0, sizeof(int), st);
  int nb = (n_max + kHashThreads - 1) / kHashThreads;
  if (nb < 1) nb = 1;
  ch_insert<<<nb, kHashThreads, 0, st>>>(map, n_dev, inv_cell, keys, count, table_size - 1, slot_of, rank_of);
  ch_scan<<<ntiles, kHashThreads, 0, st>>>(count, start, table_size, status, ticket);
  ch_scatter<<<nb, kHashThreads, 0, st>>>(map, n_dev, start, slot_of, rank_of, cellpts);
  if (launches) *launches += 3;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

// Eigen quaternion * vector, then + pos (PointAssociateToMap)
__device__ __forceinline__ void assoc_to_map(const TransformF &t, float vx, float vy, float vz, float &ox, float &oy, float &oz) {
  float ux = t.qy * vz - t.qz * vy, uy = t.qz * vx - t.qx * vz, uz = t.qx * vy - t.qy * vx;
  ux += ux; uy += uy; uz += uz;
  float cx = t.qy * uz - t.qz * uy, cy = t.qz * ux - t.qx * uz, cz = t.qx * uy - t.qy * ux;
  float rx = vx + ux * t.qw + cx, ry = vy + uy * t.qw + cy, rz = vz + uz * t.qw + cz;
  ox = rx + t.px; oy = ry + t.py; oz = rz + t.pz;
}

// (d^2, map index) packed so that unsigned order == the oracle's total order (d^2 >= 0)
__device__ __forceinline__ unsigned long long pack_key(float d, int mi) {
  return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)mi;
}
constexpr unsigned long long kInfKey = 0x7f8000007fffffffull;  // (+inf, INT_MAX)

constexpr int kGroup = 8;                               // lanes cooperating on one query
constexpr int kQueriesPerBlock = kKnnThreads / kGroup;  // 32: the fits of a block fill exactly one warp

// cyclic Jacobi eigen-decomposition of a symmetric 3x3 (float), ascending eigenvalues, vectors in columns — the same
// operation order as the oracle's sym_eigen_jacobi<float>(3, ...) (stand-in for SelfAdjointEigenSolver<Matrix3f>)
__device__ __forceinline__ void sym_eigen3(const float *Ain, float *evals, float *V) {
  float A[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) { A[i] = Ain[i]; V[i] = (i % 4 == 0) ? 1.f : 0.f; }
  for (int sweep = 0; sweep < 100; ++sweep) {
    float off = 0.f, diag = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      diag += A[i * 3 + i] * A[i * 3 + i];
#pragma unroll
      for (int j = i + 1; j < 3; ++j) off += A[i * 3 + j] * A[i * 3 + j];
    }
    if (off <= FLT_EPSILON * FLT_EPSILON * diag || off == 0.f) break;
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int q = p + 1; q < 3; ++q) {
        const float apq = A[p * 3 + q];
        if (apq == 0.f) continue;
        const float theta = (A[q * 3 + q] - A[p * 3 + p]) / (2.f * apq);
        const float t = (theta >= 0.f ? 1.f : -1.f) / (fabsf(theta) + sqrtf(theta * theta + 1.f));
        const float c = 1.f / sqrtf(t * t + 1.f), sn = t * c;
#pragma unroll
        for (int k = 0; k < 3; ++k) { float a = A[k * 3 + p], b = A[k * 3 + q]; A[k * 3 + p] = c * a - sn * b; A[k * 3 + q] = sn * a + c * b; }
#pragma unroll
        for (int k = 0; k < 3; ++k) { float a = A[p * 3 + k], b = A[q * 3 + k]; A[p * 3 + k] = c * a - sn * b; A[q * 3 + k] = sn * a + c * b; }
#pragma unroll
        for (int k = 0; k < 3; ++k) { float a = V[k * 3 + p], b = V[k * 3 + q]; V[k * 3 + p] = c * a - sn * b; V[k * 3 + q] = sn * a + c * b; }
      }
  }
  // ascending order of the diagonal (3-element sort, first index wins ties like the oracle's comparator sort)
  int i0 = 0, i1 = 1, i2 = 2;
  if (A[i1 * 3 + i1] < A[i0 * 3 + i0]) { int t = i0; i0 = i1; i1 = t; }
  if (A[i2 * 3 + i2] < A[i1 * 3 + i1]) { int t = i1; i1 = i2; i2 = t; }
  if (A[i1 * 3 + i1] < A[i0 * 3 + i0]) { int t = i0; i0 = i1; i1 = t; }
  float Vc[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) Vc[i] = V[i];
  const int idx[3] = {i0, i1, i2};
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    evals[j] = A[idx[j] * 3 + idx[j]];
#pragma unroll
    for (int k = 0; k < 3; ++k) V[k * 3 + j] = Vc[k * 3 + idx[j]];
  }
}

// kFit = 0: point-to-plane (Estimator::CalculateFeatures surf branch), one feature per accepted query;
// kFit = 1: point-to-line (USE_CORNER branch :1101-1227 / PointMapping.cc:381-512), two half-weight features.
// One 8-lane group per query: lane g scans cells g, g+8, g+16, g+24 of the 3x3x3 block keeping a local
// sorted top-5; the groups' lists are merged by five rounds of a (d^2, idx) min-reduction (shuffles), which
// yields exactly the sequence a single sorted scan would.  The 32 merged neighbour lists of the block are handed to
// warp 0 through shared memory, one query per LANE, so the long fit (QR / eigen, tests) issues once per block at full
// lane occupancy instead of on one lane in eight of every warp.
template <int kFit>
__global__ void __launch_bounds__(kKnnThreads)
knn_plane(const KnnBatch B, const unsigned long long *__restrict__ hkeys, const int *__restrict__ hcount,
          const int *__restrict__ hstart, int hmask, float inv_cell, const float4 *__restrict__ cellpts, float min_match_sq_dis,
          float min_plane_dis, const int *__restrict__ done_flag, unsigned long long *__restrict__ status, int *__restrict__ ticket) {
  __shared__ int sscan[40];
  __shared__ int stile, sbc;
  if (done_flag && *done_flag) return;
  if (threadIdx.x == 0) stile = atomicAdd(ticket, 1);
  __syncthreads();
  const int tile = stile;
  if (tile >= B.ntiles) return;
  int fi = 0;
#pragma unroll 1
  for (int k = 1; k < B.nframes; ++k) if (tile >= B.f[k].tile0) fi = k;
  const KnnFrame &F = B.f[fi];
  const int ltile = tile - F.tile0;
  const int n = *F.n_dev;
  const int ntiles = (n + kQueriesPerBlock - 1) / kQueriesPerBlock;
  const int base_count = F.append ? *F.out_count : 0;  // read before the frame's last tile rewrites it
  if (ltile >= ntiles) {
    if (n == 0 && ltile == 0 && threadIdx.x == 0 && !F.append) *F.out_count = 0;
    return;
  }
  const TransformF tf = *F.tf;
  const int g = threadIdx.x & (kGroup - 1);
  const int q = ltile * kQueriesPerBlock + (threadIdx.x / kGroup);
  const unsigned gmask = 0xffu << ((lane_id() / kGroup) * kGroup);
  bool valid = false;
  float4 po = make_float4(0, 0, 0, 0), co = make_float4(0, 0, 0, 0), co2 = make_float4(0, 0, 0, 0);
  const bool active = q < n;
  float sx = 0.f, sy = 0.f, sz = 0.f;
  float4 p = make_float4(0, 0, 0, 0);
  unsigned long long bk[5];
  int bp[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) { bk[k] = kInfKey; bp[k] = -1; }
  // Balanced scan.  The 27 cells of a query hold very different numbers of points, so a lane that owns whole cells idles
  // while its neighbours work (14.9 of 32 lanes active in round 1).  Instead: each lane looks up its <= 4 cells (the four
  // first probes in flight together), the group lays the cell ranges end to end (lane-major order; an exclusive scan of the
  // lane totals by shuffles), and lane g takes candidates g, g + 8, ... of that list, four loads in flight at a time.
  // The top-5 by (d^2, map index) does not depend on the order candidates are seen in.
  __shared__ int s_cst[kQueriesPerBlock][32];    // first cellpts index of every range
  __shared__ int s_cpre[kQueriesPerBlock][33];   // exclusive prefix of the range sizes, [32] = total
  const int ql = threadIdx.x / kGroup;
  if (active) {
    p = __ldg(F.surf + q);
    assoc_to_map(tf, p.x, p.y, p.z, sx, sy, sz);
    const int cx = (int)floorf(sx * inv_cell), cy = (int)floorf(sy * inv_cell), cz = (int)floorf(sz * inv_cell);
    unsigned long long key4[4], got4[4];
    unsigned s4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = g + kGroup * k;
      const int dz = c / 9 - 1, dy = (c / 3) % 3 - 1, dx = c % 3 - 1;
      key4[k] = pack_cell(cx + dx, cy + dy, cz + dz);
      s4[k] = hash_cell(key4[k]) & hmask;
      got4[k] = (c < 27) ? hkeys[s4[k]] : kEmptyKey;
    }
    int st4[4], cn4[4], tot = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      while (got4[k] != key4[k] && got4[k] != kEmptyKey) { s4[k] = (s4[k] + 1) & hmask; got4[k] = hkeys[s4[k]]; }
      const bool found = got4[k] == key4[k];
      st4[k] = found ? hstart[s4[k]] : 0;
      cn4[k] = found ? hcount[s4[k]] : 0;
      tot += cn4[k];
    }
    int incl = tot;
#pragma unroll
    for (int o = 1; o < kGroup; o <<= 1) {
      const int t = __shfl_up_sync(gmask, incl, o, kGroup);
      if (g >= o) incl += t;
    }
    const int T = __shfl_sync(gmask, incl, kGroup - 1, kGroup);
    int run = incl - tot;
#pragma unroll
    for (int k = 0; k < 4; ++k) { s_cst[ql][4 * g + k] = st4[k]; s_cpre[ql][4 * g + k] = run; run += cn4[k]; }
    if (g == kGroup - 1) s_cpre[ql][32] = run;
    __syncwarp(gmask);
    int r = 0;
    for (int f0 = g; f0 < T; f0 += kGroup * 4) {
      int addr[4];
      float4 m4[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int f = f0 + kGroup * u;
        addr[u] = -1;
        if (f < T) {
          while (f >= s_cpre[ql][r + 1]) ++r;
          addr[u] = s_cst[ql][r] + (f - s_cpre[ql][r]);
          m4[u] = __ldg(cellpts + addr[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (addr[u] < 0) continue;
        const float4 m = m4[u];
        // flann::L2_Simple<float>: sequential diff*diff accumulation over x, y, z
        const float d0 = sx - m.x, d1 = sy - m.y, d2 = sz - m.z;
        float d = 0.f;
        d += d0 * d0; d += d1 * d1; d += d2 * d2;
        const unsigned long long kk = pack_key(d, __float_as_int(m.w));
        if (kk < bk[4]) {
          bk[4] = kk; bp[4] = addr[u];
#pragma unroll
          for (int t = 4; t > 0; --t) {
            if (bk[t] < bk[t - 1]) {
              unsigned long long tk = bk[t]; bk[t] = bk[t - 1]; bk[t - 1] = tk;
              int ti = bp[t]; bp[t] = bp[t - 1]; bp[t - 1] = ti;
            }
          }
        }
      }
    }
  }
  // merge the 8 sorted lists: five pops of the group-wide minimum head
  unsigned long long top_k[5];
  int top_p[5];
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    unsigned long long m = bk[0];
#pragma unroll
    for (int o = kGroup / 2; o > 0; o >>= 1) {
      unsigned long long other = __shfl_xor_sync(gmask, m, o);
      m = other < m ? other : m;
    }
    const bool mine = (bk[0] == m) && (m != kInfKey);
    const unsigned wb = __ballot_sync(gmask, mine) & gmask;   // keys are unique per map point: at most one lane
    const int wl = wb ? (__ffs(wb) - 1) : (int)(lane_id() & ~(kGroup - 1));
    top_k[r] = m;
    top_p[r] = __shfl_sync(gmask, bp[0], wl);
    if (mine) {
#pragma unroll
      for (int t = 0; t < 4; ++t) { bk[t] = bk[t + 1]; bp[t] = bp[t + 1]; }
      bk[4] = kInfKey; bp[4] = -1;
    }
  }
  __shared__ int s_tp[kQueriesPerBlock][5];
  __shared__ float s_d5[kQueriesPerBlock];
  __shared__ float4 s_sel[kQueriesPerBlock], s_ori[kQueriesPerBlock];
  if (g == 0) {
    const int ql = threadIdx.x / kGroup;
#pragma unroll
    for (int j = 0; j < 5; ++j) s_tp[ql][j] = top_p[j];
    // d5 < 0 marks "no fit": inactive query or fewer than five neighbours in the 27 cells
    s_d5[ql] = (active && top_k[4] != kInfKey) ? __uint_as_float((unsigned)(top_k[4] >> 32)) : -1.f;
    s_sel[ql] = make_float4(sx, sy, sz, 0.f);
    s_ori[ql] = p;
  }
  __syncthreads();
  const int qf = ltile * kQueriesPerBlock + threadIdx.x;   // the query this thread fits (warp 0 only)
  if (threadIdx.x < kQueriesPerBlock && s_d5[threadIdx.x] >= 0.f) {
    const float d5 = s_d5[threadIdx.x];
    int top_p[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) top_p[j] = s_tp[threadIdx.x][j];
    const float4 sel = s_sel[threadIdx.x];
    const float sx = sel.x, sy = sel.y, sz = sel.z;
    const float4 p = s_ori[threadIdx.x];
    if ((kFit == 0 || kFit == 2) && d5 < min_match_sq_dis) {
      float A[5][3], Bv[5], X[3];
      float nx[5], ny[5], nz[5];
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const float4 m = __ldg(cellpts + top_p[j]);
        nx[j] = m.x; ny[j] = m.y; nz[j] = m.z;
        A[j][0] = m.x; A[j][1] = m.y; A[j][2] = m.z;
        Bv[j] = -1.f;
      }
      colpiv_qr_solve<5, 3>(A, Bv, X);
      float pa = X[0], pb = X[1], pc = X[2], pd = 1.f;
      const float ps = sqrtf(pa * pa + pb * pb + pc * pc);
      pa /= ps; pb /= ps; pc /= ps; pd /= ps;
      bool planeValid = true;
#pragma unroll
      for (int j = 0; j < 5; ++j)
        if (fabsf(pa * nx[j] + pb * ny[j] + pc * nz[j] + pd) > min_plane_dis) planeValid = false;
      if (planeValid) {
        const float pd2 = pa * sx + pb * sy + pc * sz + pd;
        const float dist = sqrtf(sx * sx + sy * sy + sz * sz);
        const float s = 1.f - 0.9f * fabsf(pd2) / sqrtf(dist);
        float zx, zy, zz;
        if (F.zaxis) { zx = F.zaxis[0]; zy = F.zaxis[1]; zz = F.zaxis[2]; }
        else assoc_to_map(tf, 0.0f, 0.0f, 10.0f, zx, zy, zz);
        const float e0 = tf.px - sx, e1 = tf.py - sy, e2 = tf.pz - sz;
        const float squared_side1 = e0 * e0 + e1 * e1 + e2 * e2;
        const float f0 = zx - sx, f1 = zy - sy, f2 = zz - sz;
        const float squared_side2 = f0 * f0 + f1 * f1 + f2 * f2;
        const float check1 = 100.0f + squared_side1 - squared_side2 - 10.0f * sqrtf(3.0f) * sqrtf(squared_side1);
        const float check2 = 100.0f + squared_side1 - squared_side2 + 10.0f * sqrtf(3.0f) * sqrtf(squared_side1);
        const bool in_fov = (check1 < 0.f && check2 > 0.f);
        if ((double)s > 0.1 && in_fov) {
          valid = true;
          po = make_float4(p.x, p.y, p.z, s);
          if (kFit == 2) co = pd2 > 0.f ? make_float4(s * pa, s * pb, s * pc, s * pd2) : make_float4(-s * pa, -s * pb, -s * pc, -s * pd2);
          else co = make_float4(s * pa, s * pb, s * pc, s * pd);
        }
      }
    }
    if ((kFit == 1 || kFit == 3) && d5 < min_match_sq_dis) {
      float nx[5], ny[5], nz[5];
      float vcx = 0.f, vcy = 0.f, vcz = 0.f;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const float4 m = __ldg(cellpts + top_p[j]);
        nx[j] = m.x; ny[j] = m.y; nz[j] = m.z;
        vcx += m.x; vcy += m.y; vcz += m.z;
      }
      vcx /= 5.0f; vcy /= 5.0f; vcz /= 5.0f;
      float a00 = 0.f, a10 = 0.f, a20 = 0.f, a11 = 0.f, a21 = 0.f, a22 = 0.f;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const float ax = nx[j] - vcx, ay = ny[j] - vcy, az = nz[j] - vcz;
        a00 += ax * ax; a10 += ax * ay; a20 += ax * az; a11 += ay * ay; a21 += ay * az; a22 += az * az;
      }
      float A1[9], D1[3], V1[9];
      A1[0] = a00 / 5.0f; A1[4] = a11 / 5.0f; A1[8] = a22 / 5.0f;
      A1[3] = A1[1] = a10 / 5.0f; A1[6] = A1[2] = a20 / 5.0f; A1[7] = A1[5] = a21 / 5.0f;
      sym_eigen3(A1, D1, V1);
      if (D1[2] > 3 * D1[1]) {
        // `vc + 0.1 * V(k,2)`: double arithmetic, rounded to float on assignment
        const float x1 = (float)((double)vcx + 0.1 * (double)V1[2]), y1 = (float)((double)vcy + 0.1 * (double)V1[5]),
                    z1 = (float)((double)vcz + 0.1 * (double)V1[8]);
        const float x2 = (float)((double)vcx - 0.1 * (double)V1[2]), y2 = (float)((double)vcy - 0.1 * (double)V1[5]),
                    z2 = (float)((double)vcz - 0.1 * (double)V1[8]);
        const float u0 = sx - x1, u1 = sy - y1, u2 = sz - z1;   // X0 - X1
        const float v0 = sx - x2, v1 = sy - y2, v2 = sz - z2;   // X0 - X2
        const float ax = u1 * v2 - u2 * v1, ay = u2 * v0 - u0 * v2, az = u0 * v1 - u1 * v0;   // a012_vec
        const float lx = x1 - x2, ly = y1 - y2, lz = z1 - z2;   // X1 - X2
        float tx = ly * az - lz * ay, ty = lz * ax - lx * az, tz = lx * ay - ly * ax;         // (X1-X2) x a012_vec
        {
          const float zz = tx * tx + ty * ty + tz * tz;
          if (zz > 0.f) { const float nn = sqrtf(zz); tx = tx / nn; ty = ty / nn; tz = tz / nn; }
        }
        const float cx2 = ly * tz - lz * ty, cy2 = lz * tx - lx * tz, cz2 = lx * ty - ly * tx;  // normal_cross_point
        const float a012 = sqrtf(ax * ax + ay * ay + az * az);
        const float l12 = sqrtf(lx * lx + ly * ly + lz * lz);
        const float ld2 = a012 / l12;
        const float qx = sx - tx * ld2, qy = sy - ty * ld2, qz = sz - tz * ld2;   // point_proj
        const float ld_p1 = -(tx * qx + ty * qy + tz * qz);
        const float ld_p2 = -(cx2 * qx + cy2 * qy + cz2 * qz);
        const float s = 1.f - 0.9f * fabsf(ld2);
        float zx, zy, zz;
        if (F.zaxis) { zx = F.zaxis[0]; zy = F.zaxis[1]; zz = F.zaxis[2]; }
        else assoc_to_map(tf, 0.0f, 0.0f, 10.0f, zx, zy, zz);
        const float e0 = tf.px - sx, e1 = tf.py - sy, e2 = tf.pz - sz;
        const float squared_side1 = e0 * e0 + e1 * e1 + e2 * e2;
        const float f0 = zx - sx, f1 = zy - sy, f2 = zz - sz;
        const float squared_side2 = f0 * f0 + f1 * f1 + f2 * f2;
        const float check1 = 100.0f + squared_side1 - squared_side2 - 10.0f * sqrtf(3.0f) * sqrtf(squared_side1);
        const float check2 = 100.0f + squared_side1 - squared_side2 + 10.0f * sqrtf(3.0f) * sqrtf(squared_side1);
        const bool in_fov = (check1 < 0.f && check2 > 0.f);
        if ((double)s > 0.1 && in_fov) {
          valid = true;
          if (kFit == 3) {
            po = make_float4(p.x, p.y, p.z, s);
            co = make_float4(s * tx, s * ty, s * tz, s * ld2);
          } else {
            po = make_float4(p.x, p.y, p.z, s * 0.5f);   // halving is exact
            co = make_float4((s * tx) * 0.5f, (s * ty) * 0.5f, (s * tz) * 0.5f, (s * ld_p1) * 0.5f);
            co2 = make_float4((s * cx2) * 0.5f, (s * cy2) * 0.5f, (s * cz2) * 0.5f, (s * ld_p2) * 0.5f);
          }
        }
      }
    }
  }
  int tot;
  constexpr int kPer = kFit == 1 ? 2 : 1;
  const int lpos = block_scan_excl(valid ? kPer : 0, sscan, &tot);   // thread order == query order
  const int excl = lookback_exclusive(status + F.tile0, ltile, tot, &sbc);
  if (valid) {
    const int o = base_count + excl + lpos;
    F.out_p[o] = po; F.out_c[o] = co; F.out_src[o] = qf;
    if (kFit == 1) { F.out_p[o + 1] = po; F.out_c[o + 1] = co2; F.out_src[o + 1] = qf; }
  }
  if (ltile == ntiles - 1 && threadIdx.x == 0) *F.out_count = base_count + excl + tot;
}

int KnnWork::init(int max_queries_total) {
  ntiles_max = (max_queries_total + kQueriesPerBlock - 1) / kQueriesPerBlock + kMaxKnnFrames + 1;
  if (cudaMalloc(&status, sizeof(unsigned long long) * ntiles_max) != cudaSuccess) return -1;
  if (cudaMalloc(&ticket, sizeof(int)) != cudaSuccess) return -1;
  return 0;
}
void KnnWork::destroy() {
  if (status) cudaFree(status);
  if (ticket) cudaFree(ticket);
  status = nullptr; ticket = nullptr;
}

void knn_plan(KnnBatch &b) {
  int t = 0;
  for (int k = 0; k < b.nframes; ++k) {
    b.f[k].tile0 = t;
    int nt = (b.f[k].n_bound + kQueriesPerBlock - 1) / kQueriesPerBlock;
    if (nt < 1) nt = 1;
    t += nt;
  }
  b.ntiles = t;
}

int calculate_features_batch(const CellHash &h, KnnBatch &b, float min_match_sq_dis, float min_plane_dis, const int *done_flag,
                             KnnWork &work, cudaStream_t st, int *launches, int fit, bool state_clean) {
  if (b.nframes <= 0) return LIO_OK;
  knn_plan(b);
  if (b.ntiles > work.ntiles_max) return LIO_ERR_CAPACITY;
  if (!state_clean) {
    cudaMemsetAsync(work.status, 0, sizeof(unsigned long long) * b.ntiles, st);
    cudaMemsetAsync(work.ticket, 0, sizeof(int), st);
  }
  if (fit == 2)
    knn_plane<2><<<b.ntiles, kKnnThreads, 0, st>>>(b, h.keys, h.count, h.start, h.eff_size - 1, h.inv_cell, h.cellpts, min_match_sq_dis,
                                                   min_plane_dis, done_flag, work.status, work.ticket);
  else if (fit == 3)
    knn_plane<3><<<b.ntiles, kKnnThreads, 0, st>>>(b, h.keys, h.count, h.start, h.eff_size - 1, h.inv_cell, h.cellpts, min_match_sq_dis,
                                                   min_plane_dis, done_flag, work.status, work.ticket);
  else if (fit == 1)
    knn_plane<1><<<b.ntiles, kKnnThreads, 0, st>>>(b, h.keys, h.count, h.start, h.eff_size - 1, h.inv_cell, h.cellpts, min_match_sq_dis,
                                                   min_plane_dis, done_flag, work.status, work.ticket);
  else
    knn_plane<0><<<b.ntiles, kKnnThreads, 0, st>>>(b, h.keys, h.count, h.start, h.eff_size - 1, h.inv_cell, h.cellpts, min_match_sq_dis,
                                                   min_plane_dis, done_flag, work.status, work.ticket);
  if (launches) *launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

int calculate_features_dev(const CellHash &h, const float4 *map, const float4 *surf, const int *nsurf_dev, int nsurf_max,
                           const TransformF *tf_dev, float min_match_sq_dis, float min_plane_dis, FeatureOut out, int append,
                           const int *done_flag, KnnWork &work, cudaStream_t st, int *launches, int fit, const float *zaxis_dev) {
  (void)map;
  KnnBatch b;
  b.nframes = 1;
  KnnFrame &f = b.f[0];
  f.surf = surf; f.n_dev = nsurf_dev; f.n_bound = nsurf_max; f.tf = tf_dev;
  f.out_p = out.pts; f.out_c = out.coef; f.out_src = out.src; f.out_count = out.count; f.append = append; f.tile0 = 0; f.zaxis = zaxis_dev;
  return calculate_features_batch(h, b, min_match_sq_dis, min_plane_dis, done_flag, work, st, launches, fit);
}

}  // namespace lio

// ---- C-ABI: Estimator::CalculateFeatures on explicit host arrays (parity entry) -----------------
using namespace lio;

static int calculate_features_host_impl(const float *map, int K, const float *surf, int M, const float *tf7,
                                        float min_match_sq_dis, float min_plane_dis, float *pts4, float *coef4, int32_t *src,
                                        int *n_out, int device, int fit);

extern "C" int lio_calculate_features_host(const float *map, int K, const float *surf, int M, const float *tf7,
                                           float min_match_sq_dis, float min_plane_dis, float *pts4, float *coef4, int32_t *src,
                                           int *n_out, int device) {
  return calculate_features_host_impl(map, K, surf, M, tf7, min_match_sq_dis, min_plane_dis, pts4, coef4, src, n_out, device, 0);
}

extern "C" int lio_calculate_line_features_host(const float *corner_map, int K, const float *corner, int M, const float *tf7,
                                                float min_match_sq_dis, float *pts4, float *coef4, int32_t *src, int *n_out,
                                                int device) {
  return calculate_features_host_impl(corner_map, K, corner, M, tf7, min_match_sq_dis, 0.f, pts4, coef4, src, n_out, device, 1);
}

static int calculate_features_host_impl(const float *map, int K, const float *surf, int M, const float *tf7,
                                        float min_match_sq_dis, float min_plane_dis, float *pts4, float *coef4, int32_t *src,
                                        int *n_out, int device, int fit) {
  const int per = fit == 1 ? 2 : 1;
  if (!map || !surf || !tf7 || !n_out || K < 0 || M < 0) return LIO_ERR_INVALID;
  if (lio_device_count() <= 0) return LIO_ERR_NO_DEVICE;
  LIO_CUDA_OK(cudaSetDevice(device));
  *n_out = 0;
  if (M == 0) return LIO_OK;
  CellHash h;
  KnnWork w;
  float4 *d_map = nullptr, *d_surf = nullptr;
  FeatureOut fo;
  int *d_n = nullptr;
  TransformF *d_tf = nullptr;
  int rc = LIO_OK;
  int Kc = K > 0 ? K : 1;
  if (h.init(Kc) != 0 || w.init(M) != 0) rc = LIO_ERR_CUDA;
  if (rc == LIO_OK && (cudaMalloc(&d_map, sizeof(float4) * Kc) != cudaSuccess || cudaMalloc(&d_surf, sizeof(float4) * M) != cudaSuccess ||
                       cudaMalloc(&fo.pts, sizeof(float4) * M * per) != cudaSuccess || cudaMalloc(&fo.coef, sizeof(float4) * M * per) != cudaSuccess ||
                       cudaMalloc(&fo.src, sizeof(int) * M * per) != cudaSuccess || cudaMalloc(&d_n, sizeof(int) * 4) != cudaSuccess ||
                       cudaMalloc(&d_tf, sizeof(TransformF)) != cudaSuccess))
    rc = LIO_ERR_CUDA;
  if (rc == LIO_OK) {
    int hn[3] = {K, M, 0};
    cudaMemcpy(d_map, map, sizeof(float4) * K, cudaMemcpyHostToDevice);
    cudaMemcpy(d_surf, surf, sizeof(float4) * M, cudaMemcpyHostToDevice);
    cudaMemcpy(d_n, hn, sizeof(hn), cudaMemcpyHostToDevice);
    cudaMemcpy(d_tf, tf7, sizeof(TransformF), cudaMemcpyHostToDevice);
    fo.count = d_n + 2; fo.cap = M * per;
    // cell edge >= search radius (with margin, see header)
    float cell = sqrtf(min_match_sq_dis) * (1.0f + 1.0f / 1024.0f);
    rc = h.build(d_map, d_n, Kc, cell, 0, nullptr);
    if (rc == LIO_OK) rc = calculate_features_dev(h, d_map, d_surf, d_n + 1, M, d_tf, min_match_sq_dis, min_plane_dis, fo, 0, nullptr, w, 0, nullptr, fit);
    if (rc == LIO_OK) {
      int m = 0;
      cudaError_t e = cudaMemcpy(&m, d_n + 2, sizeof(int), cudaMemcpyDeviceToHost);
      if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); rc = LIO_ERR_CUDA; }
      else {
        *n_out = m;
        if (m > 0) {
          cudaMemcpy(pts4, fo.pts, sizeof(float4) * m, cudaMemcpyDeviceToHost);
          cudaMemcpy(coef4, fo.coef, sizeof(float4) * m, cudaMemcpyDeviceToHost);
          if (src) cudaMemcpy(src, fo.src, sizeof(int) * m, cudaMemcpyDeviceToHost);
        }
      }
    }
  } else {
    lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed");
  }
  void *fr[] = {d_map, d_surf, fo.pts, fo.coef, fo.src, d_n, d_tf};
  for (void *q : fr) if (q) cudaFree(q);
  h.destroy();
  w.destroy();
  return rc;
}
