// lio_rm: the map of a whole drive, accumulated in HBM from the registered clouds (/cloud_registered) of every publishing step,
// and its binary PCD writer.  The reference builds the same map offline with src/save_bag_to_pcd.cc: every /cloud_registered
// message is appended (`map_points += transformed_cloud`, :111-115; the transform is the identity, :95-109) and the result is
// written by pcl::PCDWriter::writeBinary (:156-160).
//
// leaf == 0 (raw mode) is that tool: a concatenation in insert order.  leaf > 0 (voxel mode) keeps one running fp64 sum per voxel
// of PCL's float32 voxel key, so the map stays bounded over a drive.  Each voxel-mode insert is a fixed sequence of launches:
//   k_rm_key       voxel key of every point (3 x 21 bits, non-finite or out-of-range points get the sentinel that sorts last)
//   2 radix sorts  the existing stable 32-bit sort, low word then high word: stable LSD order on (key, index)
//   k_rm_hi        the high words in the order of the first sort
//   k_rm_lookup    segment heads look their key up in the hash (read only) and flag their first point when it misses
//   k_rm_scan      exclusive scan of the flags in point order: new voxels are numbered by their first point, and the batch is
//                  refused (sticky overflow) when size + misses > capacity, before anything changes
//   k_rm_commit    misses take their id and their slot (atomicCAS; the slot may depend on races, the id does not), then each
//                  segment adds its points to the voxel's sums one at a time in point order, from the stored sums: the sums are
//                  exactly np.add.at in arrival order.  No atomics touch the sums.
// That is 17 stream operations for any cloud size (k_rm_key, 2 x (memset + 5 sort kernels), k_rm_hi, lookup, scan, commit), plus
// the upload of a host cloud; a raw-mode insert is one copy.  No insert waits for the device.
#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>
#include "primitives.cuh"
#include "regmap.cuh"

namespace lio {

constexpr unsigned long long kRmEmpty = ~0ull;       // empty hash slot, and the key of a dropped point
constexpr int kRmRange = 1 << 20;                    // voxel coordinates in [-2^20, 2^20) per axis
constexpr int kRmThreads = 256;
constexpr int kRmScanItems = 8;
constexpr int kRmScanTile = kRmThreads * kRmScanItems;

// device state of the map: {size, overflow, accepted points, dropped points}
struct RmState { long long size, overflow, accepted, dropped; };
// one insert's batch values
struct RmBatch { int n, nvalid, ticket, ok; long long misses, size0; };

__device__ __forceinline__ unsigned long long rm_hash(unsigned long long k) {   // splitmix64 finaliser
  k ^= k >> 30; k *= 0xbf58476d1ce4e5b9ull;
  k ^= k >> 27; k *= 0x94d049bb133111ebull;
  return k ^ (k >> 31);
}

__device__ __forceinline__ long long rm_find(const unsigned long long *slot_key, const int *slot_id, long long nslots,
                                             unsigned long long key) {
  for (long long s = (long long)(rm_hash(key) % (unsigned long long)nslots);; s = (s + 1 == nslots) ? 0 : s + 1) {
    const unsigned long long k = slot_key[s];
    if (k == key) return slot_id[s];
    if (k == kRmEmpty) return -1;
  }
}

__global__ void __launch_bounds__(kRmThreads)
k_rm_key(const float4 *__restrict__ pts, int n, float inv_leaf, unsigned long long *__restrict__ key64, unsigned *__restrict__ lo,
         unsigned *__restrict__ idx, int *__restrict__ flag, unsigned long long *__restrict__ scan_status, int scan_tiles,
         RmBatch *__restrict__ b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) { b->n = n; b->nvalid = 0; b->ticket = 0; b->ok = 0; b->misses = 0; }
  if (i < scan_tiles) scan_status[i] = 0ull;
  if (i >= n) return;
  const float4 p = pts[i];
  // PCL's arithmetic in float32: floor(c * (1 / leaf)); the comparisons also drop NaN and inf
  const float vx = floorf(p.x * inv_leaf), vy = floorf(p.y * inv_leaf), vz = floorf(p.z * inv_leaf);
  const float lo_b = -(float)kRmRange, hi_b = (float)kRmRange;
  unsigned long long k = kRmEmpty;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && vx >= lo_b && vx < hi_b && vy >= lo_b && vy < hi_b && vz >= lo_b && vz < hi_b) {
    const unsigned long long ux = (unsigned long long)((long long)vx + kRmRange), uy = (unsigned long long)((long long)vy + kRmRange),
                             uz = (unsigned long long)((long long)vz + kRmRange);
    k = (ux << 42) | (uy << 21) | uz;
  }
  key64[i] = k;
  lo[i] = (unsigned)k;
  idx[i] = (unsigned)i;
  flag[i] = 0;
}

__global__ void __launch_bounds__(kRmThreads)
k_rm_hi(const unsigned long long *__restrict__ key64, const unsigned *__restrict__ idx, unsigned *__restrict__ hi, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) hi[j] = (unsigned)(key64[idx[j]] >> 32);
}

// sorted position j: the segment head looks its key up; a miss flags the segment's first point (its smallest index, by stability)
__global__ void __launch_bounds__(kRmThreads)
k_rm_lookup(const unsigned long long *__restrict__ key64, const unsigned *__restrict__ idx, int n,
            const unsigned long long *__restrict__ slot_key, const int *__restrict__ slot_id, long long nslots,
            const RmState *__restrict__ st, long long *__restrict__ seg_id, int *__restrict__ flag, RmBatch *__restrict__ b) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || st->overflow) return;
  const unsigned long long k = key64[idx[j]];
  const unsigned long long kp = j > 0 ? key64[idx[j - 1]] : kRmEmpty - 1;
  if (k == kRmEmpty) {                       // dropped points sort last: the first of them ends the valid range
    if (j == 0 || kp != kRmEmpty) b->nvalid = j;
    return;
  }
  if (j == n - 1) b->nvalid = n;
  if (j > 0 && kp == k) return;
  const long long id = rm_find(slot_key, slot_id, nslots, k);
  seg_id[j] = id;
  if (id < 0) flag[idx[j]] = 1;
}

// exclusive scan of flag[0, n) in point order (single pass, decoupled look-back), then the capacity test of the whole batch
__global__ void __launch_bounds__(kRmThreads)
k_rm_scan(const int *__restrict__ flag, int *__restrict__ rank, int n, unsigned long long *__restrict__ status,
          const RmState *__restrict__ st, long long capacity, RmBatch *__restrict__ b) {
  __shared__ int sscan[33];
  __shared__ int stile, sb;
  if (threadIdx.x == 0) stile = atomicAdd(&b->ticket, 1);
  __syncthreads();
  const int tile = stile;
  const int base = tile * kRmScanTile + threadIdx.x * kRmScanItems;
  int v[kRmScanItems], s = 0;
#pragma unroll
  for (int k = 0; k < kRmScanItems; ++k) { v[k] = base + k < n ? flag[base + k] : 0; s += v[k]; }
  int total;
  int excl = block_scan_excl(s, sscan, &total);
  excl += lookback_exclusive(status, tile, total, &sb);
#pragma unroll
  for (int k = 0; k < kRmScanItems; ++k) {
    if (base + k < n) rank[base + k] = excl;
    excl += v[k];
  }
  if (threadIdx.x == blockDim.x - 1 && (tile + 1) * kRmScanTile >= n) {
    const long long misses = excl;   // the last tile's last thread, past its items: the batch total
    b->misses = misses;
    b->size0 = st->size;
    b->ok = !st->overflow && st->size + misses <= capacity;
  }
}

__global__ void __launch_bounds__(kRmThreads)
k_rm_commit(const float4 *__restrict__ pts, const unsigned long long *__restrict__ key64, const unsigned *__restrict__ idx, int n,
            const int *__restrict__ rank, const long long *__restrict__ seg_id, unsigned long long *__restrict__ slot_key,
            int *__restrict__ slot_id, long long nslots, double4 *__restrict__ sum, long long *__restrict__ cnt,
            RmState *__restrict__ st, const RmBatch *__restrict__ b) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const RmBatch bb = *b;
  if (j == 0 && !st->overflow) {   // nothing else in this kernel reads the state
    if (bb.ok) { st->size = bb.size0 + bb.misses; st->accepted += bb.nvalid; st->dropped += bb.n - bb.nvalid; }
    else st->overflow = 1;
  }
  if (!bb.ok || j >= bb.nvalid) return;
  const unsigned long long k = key64[idx[j]];
  if (j > 0 && key64[idx[j - 1]] == k) return;
  long long id = seg_id[j];
  if (id < 0) {
    id = bb.size0 + rank[idx[j]];
    for (long long s = (long long)(rm_hash(k) % (unsigned long long)nslots);; s = (s + 1 == nslots) ? 0 : s + 1) {
      if (atomicCAS(slot_key + s, kRmEmpty, k) == kRmEmpty) { slot_id[s] = (int)id; break; }
    }
  }
  double4 a = sum[id];
  long long c = cnt[id];
  for (int q = j; q < bb.nvalid; ++q) {
    const unsigned i = idx[q];
    if (key64[i] != k) break;
    const float4 p = pts[i];
    a.x += (double)p.x; a.y += (double)p.y; a.z += (double)p.z; a.w += (double)p.w;
    ++c;
  }
  sum[id] = a;
  cnt[id] = c;
}

__global__ void __launch_bounds__(kRmThreads)
k_rm_export(const double4 *__restrict__ sum, const long long *__restrict__ cnt, long long size, float4 *__restrict__ out) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= size) return;
  const double4 a = sum[v];
  const double c = (double)cnt[v];
  out[v] = make_float4((float)(a.x / c), (float)(a.y / c), (float)(a.z / c), (float)(a.w / c));
}

}  // namespace lio

using namespace lio;

struct lio_rm {
  int device = 0;
  cudaStream_t stream = nullptr;
  float leaf = 0.f, inv_leaf = 0.f;
  long long capacity = 0;
  // raw mode: the concatenation, its size and the overflow flag are host state
  DevMem<float4> d_pts;
  long long n_raw = 0, raw_overflow = 0;
  // voxel mode
  DevMem<unsigned long long> d_slot_key;
  DevMem<int> d_slot_id;
  long long nslots = 0;
  DevMem<double4> d_sum;
  DevMem<long long> d_cnt;
  DevMem<float4> d_export;
  DevMem<RmState> d_state;
  HostMem<RmState> h_state;     // pinned
  // per-insert scratch, grown stream-ordered (cudaMallocAsync) for a larger cloud: the views below point into it
  int batch_cap = 0;
  void *d_batch_mem = nullptr;
  float4 *d_in = nullptr;
  unsigned long long *d_key64 = nullptr, *d_scan_status = nullptr;
  unsigned *d_ka = nullptr, *d_va = nullptr, *d_kb = nullptr, *d_vb = nullptr;
  int *d_flag = nullptr, *d_rank = nullptr;
  long long *d_seg_id = nullptr;
  RmBatch *d_b = nullptr;
  RadixSortTemp sort_tmp;
  // host counters: insert calls, points offered, host waits of every entry, stream operations of the last insert
  long long inserts = 0, offered = 0, waits = 0, last_launches = 0;
  // The scratch goes behind the stream's last use of it, and the stream drains before the buffers above are freed.
  ~lio_rm() {
    if (d_batch_mem) cudaFreeAsync(d_batch_mem, stream);
    cudaStreamSynchronize(stream);
  }
};

static long long rm_blocks(long long n) { return std::max(1LL, (n + kRmThreads - 1) / kRmThreads); }

// Scratch for clouds of up to n points: one stream-ordered allocation, the old one freed behind the work that used it.
static int rm_reserve(lio_rm *m, int n) {
  if (n <= m->batch_cap && m->d_batch_mem) return LIO_OK;
  const int cap = std::max(n, std::max(1 << 16, 2 * m->batch_cap));
  const int sort_tiles = (cap + kRsTile - 1) / kRsTile + 1;
  const int scan_tiles = (cap + kRmScanTile - 1) / kRmScanTile + 1;
  const size_t words = (size_t)4 * kRsBins + 8 + (size_t)4 * sort_tiles * kRsBins;
  size_t off[11], total = 0;
  const size_t bytes[11] = {sizeof(float4) * cap, sizeof(unsigned long long) * cap, sizeof(unsigned long long) * scan_tiles,
                            sizeof(unsigned) * cap, sizeof(unsigned) * cap, sizeof(unsigned) * cap, sizeof(unsigned) * cap,
                            sizeof(int) * cap, sizeof(int) * cap, sizeof(long long) * cap, sizeof(unsigned) * words};
  for (int k = 0; k < 11; ++k) { off[k] = total; total += (bytes[k] + 255) & ~(size_t)255; }
  const size_t b_off = total;
  total += sizeof(RmBatch);
  char *p = nullptr;
  LIO_CUDA_OK(cudaMallocAsync(&p, total, m->stream));
  if (m->d_batch_mem) LIO_CUDA_OK(cudaFreeAsync(m->d_batch_mem, m->stream));
  m->d_batch_mem = p;
  m->d_in = (float4 *)(p + off[0]);
  m->d_key64 = (unsigned long long *)(p + off[1]);
  m->d_scan_status = (unsigned long long *)(p + off[2]);
  m->d_ka = (unsigned *)(p + off[3]); m->d_va = (unsigned *)(p + off[4]);
  m->d_kb = (unsigned *)(p + off[5]); m->d_vb = (unsigned *)(p + off[6]);
  m->d_flag = (int *)(p + off[7]); m->d_rank = (int *)(p + off[8]);
  m->d_seg_id = (long long *)(p + off[9]);
  m->sort_tmp.buf = (unsigned *)(p + off[10]);
  m->sort_tmp.words = words;
  m->sort_tmp.ntiles_max = sort_tiles;
  m->d_b = (RmBatch *)(p + b_off);
  m->batch_cap = cap;
  return LIO_OK;
}

static int rm_clear(lio_rm *m) {
  m->n_raw = 0; m->raw_overflow = 0;
  if (m->leaf > 0.f) {
    LIO_CUDA_OK(cudaMemsetAsync(m->d_slot_key, 0xff, sizeof(unsigned long long) * m->nslots, m->stream));
    LIO_CUDA_OK(cudaMemsetAsync(m->d_sum, 0, sizeof(double4) * m->capacity, m->stream));
    LIO_CUDA_OK(cudaMemsetAsync(m->d_cnt, 0, sizeof(long long) * m->capacity, m->stream));
    LIO_CUDA_OK(cudaMemsetAsync(m->d_state, 0, sizeof(RmState), m->stream));
  }
  return LIO_OK;
}

extern "C" int lio_rm_create(float leaf, long long capacity, int device, void *cuda_stream, lio_rm **out) {
  if (!out || !(leaf >= 0.f) || !std::isfinite(leaf) || capacity < 1 || (leaf > 0.f && capacity > (1LL << 30)) ||
      (leaf > 0.f && !std::isfinite(1.0f / leaf)))
    return LIO_ERR_INVALID;
  *out = nullptr;
  if (lio_device_count() <= device || device < 0) return LIO_ERR_NO_DEVICE;
  LIO_CUDA_OK(cudaSetDevice(device));
  std::unique_ptr<lio_rm> m(new lio_rm);
  m->device = device; m->stream = (cudaStream_t)cuda_stream;
  m->leaf = leaf; m->inv_leaf = leaf > 0.f ? 1.0f / leaf : 0.f;
  m->capacity = capacity;
  bool ok = true;
  if (leaf == 0.f) {
    ok = alloc(m->d_pts, capacity);
  } else {
    m->nslots = 2 * capacity;
    ok = alloc(m->d_slot_key, m->nslots) && alloc(m->d_slot_id, m->nslots) && alloc(m->d_sum, capacity) && alloc(m->d_cnt, capacity) &&
         alloc(m->d_export, capacity) && alloc(m->d_state, 1) && alloc_host(m->h_state, 1);
  }
  if (!ok || rm_clear(m.get()) != LIO_OK || cudaStreamSynchronize(m->stream) != cudaSuccess) {
    lio_set_last_error(__FILE__, __LINE__, "lio_rm_create: allocation failed");
    cudaGetLastError();
    return LIO_ERR_CUDA;
  }
  *out = m.release();
  return LIO_OK;
}

extern "C" int lio_rm_destroy(lio_rm *m) {
  if (!m) return LIO_ERR_INVALID;
  cudaSetDevice(m->device);   // the buffers belong to the handle's device, whichever is current
  delete m;
  return LIO_OK;
}

// One cloud already in HBM, after an optional upload of a host cloud into the scratch (host_src != nullptr).
static int rm_insert(lio_rm *m, const float4 *src, const float *host_src, int n) {
  cudaStream_t st = m->stream;
  m->inserts += 1; m->offered += n;
  int launches = 0;
  if (m->leaf == 0.f) {
    if (m->raw_overflow || m->n_raw + n > m->capacity) { m->raw_overflow = 1; m->last_launches = 0; return LIO_OK; }   // host state
    LIO_CUDA_OK(cudaMemcpyAsync(m->d_pts + m->n_raw, host_src ? (const void *)host_src : (const void *)src, sizeof(float4) * n,
                                host_src ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st));
    m->n_raw += n;
    m->last_launches = 1;
    return LIO_OK;
  }
  int rc = rm_reserve(m, n);
  if (rc != LIO_OK) return rc;
  if (host_src) {
    if (n > 0) LIO_CUDA_OK(cudaMemcpyAsync(m->d_in, host_src, sizeof(float4) * n, cudaMemcpyHostToDevice, st));   // staged on return
    src = m->d_in;
    launches += n > 0;
  }
  const int g = (int)rm_blocks(n);
  const int scan_tiles = std::max(1, (n + kRmScanTile - 1) / kRmScanTile);
  RmBatch *b = m->d_b;
  k_rm_key<<<std::max(g, (scan_tiles + kRmThreads - 1) / kRmThreads), kRmThreads, 0, st>>>(
      src, n, m->inv_leaf, m->d_key64, m->d_ka, m->d_va, m->d_flag, m->d_scan_status, scan_tiles, b);
  launches += 1;
  // stable LSD on the 64-bit key: low word, then high word (each sort is a memset and five kernels, even passes end in a)
  if (radix_sort_pairs(m->d_ka, m->d_va, m->d_kb, m->d_vb, &b->n, n, 32, m->sort_tmp, st, &launches) != 0) return LIO_ERR_CAPACITY;
  k_rm_hi<<<g, kRmThreads, 0, st>>>(m->d_key64, m->d_va, m->d_ka, n);
  if (radix_sort_pairs(m->d_ka, m->d_va, m->d_kb, m->d_vb, &b->n, n, 32, m->sort_tmp, st, &launches) != 0) return LIO_ERR_CAPACITY;
  k_rm_lookup<<<g, kRmThreads, 0, st>>>(m->d_key64, m->d_va, n, m->d_slot_key, m->d_slot_id, m->nslots, m->d_state, m->d_seg_id,
                                        m->d_flag, b);
  k_rm_scan<<<scan_tiles, kRmThreads, 0, st>>>(m->d_flag, m->d_rank, n, m->d_scan_status, m->d_state, m->capacity, b);
  k_rm_commit<<<g, kRmThreads, 0, st>>>(src, m->d_key64, m->d_va, n, m->d_rank, m->d_seg_id, m->d_slot_key, m->d_slot_id, m->nslots,
                                        m->d_sum, m->d_cnt, m->d_state, b);
  launches += 2 /* memsets */ + 4;
  LIO_CUDA_OK(cudaGetLastError());
  m->last_launches = launches;
  return LIO_OK;
}

int rm_device(const lio_rm *m) { return m->device; }
cudaStream_t rm_stream(const lio_rm *m) { return m->stream; }

extern "C" int lio_rm_insert_dev(lio_rm *m, const float *xyzi_dev, int n) {
  LIO_ENTER(m);
  if (n < 0 || (n > 0 && !xyzi_dev)) return LIO_ERR_INVALID;
  return rm_insert(m, reinterpret_cast<const float4 *>(xyzi_dev), nullptr, n);
}

extern "C" int lio_rm_insert_host(lio_rm *m, const float *xyzi, int n) {
  LIO_ENTER(m);
  if (n < 0 || (n > 0 && !xyzi)) return LIO_ERR_INVALID;
  static const float kNone[4] = {0.f, 0.f, 0.f, 0.f};
  return rm_insert(m, nullptr, n > 0 ? xyzi : kNone, n);
}

// Reads the state after the work enqueued so far (one wait; raw mode keeps it on the host and only waits).  Every host wait of the
// handle is counted in waits, so that lio_rm_stats can show that inserts make none.
static int rm_read_state(lio_rm *m, RmState *s) {
  m->waits += 1;
  LIO_TRY(read_back(m->h_state.get(), m->d_state, m->leaf > 0.f ? 1 : 0, 1, m->stream));
  *s = m->leaf > 0.f ? *m->h_state : RmState{m->n_raw, m->raw_overflow, m->n_raw, 0};
  return LIO_OK;
}

extern "C" int lio_rm_stats(lio_rm *m, long long out[8]) {
  LIO_ENTER(m);
  if (!out) return LIO_ERR_INVALID;
  RmState s;
  LIO_TRY(rm_read_state(m, &s));
  const long long v[8] = {m->inserts, m->offered, s.size, s.overflow, s.accepted, s.dropped, m->waits, m->last_launches};
  std::memcpy(out, v, sizeof(v));
  return LIO_OK;
}

extern "C" int lio_rm_export_dev(lio_rm *m, const float **ptr, long long *n) {
  LIO_ENTER(m);
  if (!ptr || !n) return LIO_ERR_INVALID;
  RmState s;
  LIO_TRY(rm_read_state(m, &s));
  if (m->leaf == 0.f) { *ptr = (const float *)m->d_pts.get(); *n = m->n_raw; return LIO_OK; }
  if (s.size > 0) k_rm_export<<<(unsigned)rm_blocks(s.size), kRmThreads, 0, m->stream>>>(m->d_sum, m->d_cnt, s.size, m->d_export);
  LIO_CUDA_OK(cudaGetLastError());
  *ptr = (const float *)m->d_export.get(); *n = s.size;
  return LIO_OK;
}

extern "C" int lio_rm_download(lio_rm *m, float *out, long long cap, long long *n) {
  LIO_ENTER(m);
  if (!n || cap < 0 || (cap > 0 && !out)) return LIO_ERR_INVALID;
  const float *p = nullptr;
  LIO_TRY(lio_rm_export_dev(m, &p, n));
  if (*n > cap) return LIO_ERR_CAPACITY;
  m->waits += 1;   // lio_rm_stats counts the read-back's wait
  return read_back((float4 *)out, (const float4 *)p, *n, cap, m->stream);
}

extern "C" int lio_rm_reset(lio_rm *m) {
  LIO_ENTER(m);
  return rm_clear(m);
}

// The header pcl::PCDWriter::writeBinary writes for pcl::PointXYZI with its padding dropped, then n packed 16-byte records.
extern "C" int lio_pcd_write_xyzi(const char *path, const float *xyzi, long long n) {
  if (!path || n < 0 || (n > 0 && !xyzi)) return LIO_ERR_INVALID;
  FILE *f = fopen(path, "wb");
  if (!f) { lio_set_last_error(__FILE__, __LINE__, strerror(errno)); return LIO_ERR_INVALID; }
  const int ok_h = fprintf(f,
                           "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\n"
                           "TYPE F F F F\nCOUNT 1 1 1 1\nWIDTH %lld\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %lld\nDATA binary\n",
                           n, n) > 0;
  const bool ok_d = n == 0 || fwrite(xyzi, sizeof(float) * 4, (size_t)n, f) == (size_t)n;
  const bool ok_c = fclose(f) == 0;
  if (!ok_h || !ok_d || !ok_c) { lio_set_last_error(__FILE__, __LINE__, "lio_pcd_write_xyzi: write failed"); return LIO_ERR_INVALID; }
  return LIO_OK;
}

extern "C" int lio_rm_write_pcd(lio_rm *m, const char *path) {
  LIO_ENTER(m);
  if (!path) return LIO_ERR_INVALID;
  const float *p = nullptr;
  long long n = 0;
  LIO_TRY(lio_rm_export_dev(m, &p, &n));
  std::vector<float4> h((size_t)n);
  m->waits += 1;   // lio_rm_stats counts the read-back's wait
  LIO_TRY(read_back(h.data(), (const float4 *)p, n, n, m->stream));
  return lio_pcd_write_xyzi(path, (const float *)h.data(), n);
}
