// Stage A on sm_90a — replaces lio::PointProcessor::PointToRing / ExtractFeaturePoints
// (reference: src/point_processor/PointProcessor.cc:185-783, include/point_processor/
// PointProcessor.h:104-156, include/utils/math_utils.h:38-110; per-ring pcl::VoxelGrid(0.2)).
//
// Bit-exactness contract (SURVEY.md App. C): this translation unit is compiled with -fmad=false,
// IEEE sqrt/div, and every float expression is written in the reference's source order, so the
// ring-ordered cloud, the occlusion mask, the curvature sort and the sharp / less-sharp / flat /
// less-flat index sets are identical to the CPU path.
//
// Angle contract: the elevation and the azimuth are float(atan2 in double), i.e. atan2f correctly
// rounded up to the device's double atan2 error.  The reference calls atan2f, which glibc does not
// promise to round correctly, so a point can differ from the reference only where that rounding
// matters: its double angle lies within a few double ulps of a float rounding midpoint, or its
// ring id changes when the elevation moves one float ulp (a point on a bucket edge).  Such a point
// may land in the neighbouring ring, and its ring + rel_time / int(I) + rel_time may differ by one
// float ulp of the azimuth; every other point's ring, order, xyz and intensities are bit-exact
// (tests/pp_ref.py states the contract and its `ambiguous` points).
//
// Pipeline (one stream, 5 launches):
//   a_classify : per point ring id + azimuth, per-block ring histogram, first accepted point
//   a_scan     : ring_start[] and per-(block,ring) stable scatter offsets
//   a_scatter  : order-preserving scatter into ring order, rel_time, both intensity encodings
//   a_ring     : one CTA per ring, ring resident in shared memory: PrepareRing mask, curvature,
//                per-subregion bitonic sort of (curv,idx) keys (one warp per subregion), warp-
//                cooperative pick loops with exact MaskPickedInRing semantics, then the ring's
//                less-flat VoxelGrid (block bitonic sort by voxel index, ordered centroid emit)
//   a_compact  : concatenates per-ring results in the reference's output order
#include "common.cuh"
#include <cmath>
#include <memory>
#include <new>

namespace lio {

constexpr int kMaxRings = 128;
constexpr int kClsThreads = 256;
constexpr int kClsPerBlock = 1024;
constexpr int kRingThreads = 256;
constexpr int kMaxRingPoints = 8192;
constexpr int kMaxLessSharp = 64;
constexpr int kMaxFlat = 16;
constexpr int kMaxSub = 32;

struct PPParams {
  float lower_bound, factor;
  int num_rings;
  double scan_period;
  int S, d;
  float surf_curv_th;
  int max_sharp, max_less_sharp, max_flat;
  float leaf;
};

__device__ __forceinline__ float atan2_rn(float y, float x) { return (float)atan2((double)y, (double)x); }

// PointProcessor.cc:246-254 azimuth with the double comparison against 2*pi
__device__ __forceinline__ float azimuth_of(float x, float y) {
  float azi = (float)(2.0 * M_PI - (double)atan2_rn(y, x));
  if ((double)azi >= 2.0 * M_PI) azi = (float)((double)azi - 2.0 * M_PI);
  return azi;
}

__device__ __forceinline__ float rel_time_of(float azi, float start_ori, double scan_period) {
  float rel = azi - start_ori;  // :399
  if (rel < 0) rel = (float)((double)rel + 2.0 * M_PI);
  return (float)(scan_period * (double)rel / (2.0 * M_PI));
}

__global__ void __launch_bounds__(kClsThreads)
a_classify(const float4 *__restrict__ in, int n, PPParams P, int16_t *__restrict__ ring_id, float *__restrict__ azi_out,
           int *__restrict__ first_valid, int *__restrict__ hist) {
  __shared__ int sh[kMaxRings];
  for (int r = threadIdx.x; r < P.num_rings; r += blockDim.x) sh[r] = 0;
  __syncthreads();
  const int base = blockIdx.x * kClsPerBlock;
  int my_first = 0x7fffffff;
#pragma unroll
  for (int k = 0; k < kClsPerBlock / kClsThreads; ++k) {
    int i = base + k * kClsThreads + threadIdx.x;
    if (i < n) {
      float4 p = __ldg(in + i);
      int ring = -1;
      float azi = 0.f;
      if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        float dis = sqrtf(p.x * p.x + p.y * p.y);
        float ele = atan2_rn(p.z, dis);
        azi = azimuth_of(p.x, p.y);
        // ElevationToRing (PointProcessor.h:153-156): RadToDeg<float> in double, float subtract and
        // multiply, + 0.5 in double, truncation toward zero.
        float deg = (float)((double)ele * 180.0 / M_PI);
        double v = (double)((deg - P.lower_bound) * P.factor) + 0.5;
        int sid = (int)v;
        if (sid < P.num_rings && sid >= 0) ring = sid;
      }
      ring_id[i] = (int16_t)ring;
      azi_out[i] = azi;
      if (ring >= 0) {
        atomicAdd(&sh[ring], 1);
        my_first = min(my_first, i);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) my_first = min(my_first, __shfl_xor_sync(0xffffffffu, my_first, o));
  if (lane_id() == 0 && my_first != 0x7fffffff) atomicMin(first_valid, my_first);
  __syncthreads();
  for (int r = threadIdx.x; r < P.num_rings; r += blockDim.x) hist[blockIdx.x * P.num_rings + r] = sh[r];
}

__global__ void a_scan(const int *__restrict__ hist, int nb, int R, int *__restrict__ offsets, int *__restrict__ ring_start) {
  __shared__ int tot[kMaxRings + 1];
  int r = threadIdx.x;
  if (r < R) {
    int run = 0;
    for (int b = 0; b < nb; ++b) {
      int h = hist[b * R + r];
      offsets[b * R + r] = run;
      run += h;
    }
    tot[r] = run;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int k = 0; k < R; ++k) { int t = tot[k]; tot[k] = run; ring_start[k] = run; run += t; }
    ring_start[R] = run;
    tot[R] = run;
  }
  __syncthreads();
  if (r < R) {
    int s = tot[r];
    for (int b = 0; b < nb; ++b) offsets[b * R + r] += s;
  }
}

__global__ void __launch_bounds__(kClsThreads)
a_scatter(const float4 *__restrict__ in, int n, PPParams P, const int16_t *__restrict__ ring_id, const float *__restrict__ azi,
          const int *__restrict__ first_valid, const int *__restrict__ offsets, float4 *__restrict__ laser,
          float4 *__restrict__ full, int *__restrict__ orig, float *__restrict__ start_ori_out) {
  __shared__ int running[kMaxRings];
  __shared__ int warpcnt[kClsThreads / 32][kMaxRings];
  const int R = P.num_rings;
  for (int r = threadIdx.x; r < R; r += blockDim.x) running[r] = offsets[blockIdx.x * R + r];
  for (int k = threadIdx.x; k < (kClsThreads / 32) * kMaxRings; k += blockDim.x) (&warpcnt[0][0])[k] = 0;
  const int fv = *first_valid;
  const float start_ori = (fv >= 0 && fv < n) ? azi[fv] : 0.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) *start_ori_out = start_ori;
  __syncthreads();
  const int base = blockIdx.x * kClsPerBlock;
  const int w = warp_id();
  for (int k = 0; k < kClsPerBlock / kClsThreads; ++k) {
    int i = base + k * kClsThreads + threadIdx.x;
    int ring = (i < n) ? (int)ring_id[i] : -1;
    unsigned peers = __match_any_sync(0xffffffffu, ring);
    int lrank = __popc(peers & ((1u << lane_id()) - 1u));
    if (ring >= 0 && lrank == 0) warpcnt[w][ring] = __popc(peers);
    __syncthreads();
    if (ring >= 0) {
      int pos = running[ring] + lrank;
      for (int ww = 0; ww < w; ++ww) pos += warpcnt[ww][ring];
      float4 p = __ldg(in + i);
      float rel_time = rel_time_of(azi[i], start_ori, P.scan_period);
      laser[pos] = make_float4(p.x, p.y, p.z, (float)ring + rel_time);          // :409
      full[pos] = make_float4(p.x, p.y, p.z, (float)(int)p.w + rel_time);       // :410
      orig[pos] = i;
    }
    __syncthreads();
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
      int s = 0;
#pragma unroll
      for (int ww = 0; ww < kClsThreads / 32; ++ww) { s += warpcnt[ww][r]; warpcnt[ww][r] = 0; }
      running[r] += s;
    }
    __syncthreads();
  }
}

// ---- ring-field variant (PointToRing for lio::PointXYZIR input, PointProcessor.cc:428-536) ------------------------
// Separate kernels so that the elevation variant above stays byte-for-byte what the parity tests pinned.  The ring id
// comes from the driver's field; an azimuth before start_ori_ gets + 2 pi (the reference's half_passed branch is
// unreachable: `i > 3 * cloud_size / 2` never holds); end_ori_ is the maximum adjusted azimuth (from 0) and
// rel_time = scan_period * (azi - start_ori_) / (end_ori_ - start_ori_).
__global__ void __launch_bounds__(kClsThreads)
a_classify_ring(const float4 *__restrict__ in, const unsigned short *__restrict__ rings_in, int n, PPParams P,
                int16_t *__restrict__ ring_id, float *__restrict__ azi_out, int *__restrict__ first_valid, int *__restrict__ hist) {
  __shared__ int sh[kMaxRings];
  for (int r = threadIdx.x; r < P.num_rings; r += blockDim.x) sh[r] = 0;
  __syncthreads();
  const int base = blockIdx.x * kClsPerBlock;
  int my_first = 0x7fffffff;
#pragma unroll
  for (int k = 0; k < kClsPerBlock / kClsThreads; ++k) {
    int i = base + k * kClsThreads + threadIdx.x;
    if (i < n) {
      float4 p = __ldg(in + i);
      int ring = -1;
      float azi = 0.f;
      if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {   // :456-460
        azi = azimuth_of(p.x, p.y);
        const int sid = (int)rings_in[i];                      // :468
        if (sid < P.num_rings && sid >= 0) ring = sid;
      }
      ring_id[i] = (int16_t)ring;
      azi_out[i] = azi;
      if (ring >= 0) {
        atomicAdd(&sh[ring], 1);
        my_first = min(my_first, i);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) my_first = min(my_first, __shfl_xor_sync(0xffffffffu, my_first, o));
  if (lane_id() == 0 && my_first != 0x7fffffff) atomicMin(first_valid, my_first);
  __syncthreads();
  for (int r = threadIdx.x; r < P.num_rings; r += blockDim.x) hist[blockIdx.x * P.num_rings + r] = sh[r];
}

__device__ __forceinline__ float adjusted_azimuth(float azi, float start_ori) {
  const float rel = azi - start_ori;                                   // :482
  return rel < 0 ? (float)((double)azi + 2.0 * M_PI) : azi;           // :486-488
}

// end_ori_ = max over accepted points of the adjusted azimuth (non-negative floats order like their bit patterns)
__global__ void __launch_bounds__(256)
a_endori(const float *__restrict__ azi, const int16_t *__restrict__ ring_id, int n, const int *__restrict__ first_valid,
         int *__restrict__ end_bits) {
  const int fv = *first_valid;
  const float start_ori = (fv >= 0 && fv < n) ? azi[fv] : 0.f;
  float m = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (ring_id[i] >= 0) m = fmaxf(m, adjusted_azimuth(azi[i], start_ori));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane_id() == 0) atomicMax(end_bits, __float_as_int(m));
}

__global__ void __launch_bounds__(kClsThreads)
a_scatter_ring(const float4 *__restrict__ in, int n, PPParams P, const int16_t *__restrict__ ring_id, const float *__restrict__ azi,
               const int *__restrict__ first_valid, const int *__restrict__ end_bits, const int *__restrict__ offsets,
               float4 *__restrict__ laser, float4 *__restrict__ full, int *__restrict__ orig, float *__restrict__ start_ori_out) {
  __shared__ int running[kMaxRings];
  __shared__ int warpcnt[kClsThreads / 32][kMaxRings];
  const int R = P.num_rings;
  for (int r = threadIdx.x; r < R; r += blockDim.x) running[r] = offsets[blockIdx.x * R + r];
  for (int k = threadIdx.x; k < (kClsThreads / 32) * kMaxRings; k += blockDim.x) (&warpcnt[0][0])[k] = 0;
  const int fv = *first_valid;
  const float start_ori = (fv >= 0 && fv < n) ? azi[fv] : 0.f;
  const float range_ori = __int_as_float(*end_bits) - start_ori;       // :513
  if (blockIdx.x == 0 && threadIdx.x == 0) *start_ori_out = start_ori;
  __syncthreads();
  const int base = blockIdx.x * kClsPerBlock;
  const int w = warp_id();
  for (int k = 0; k < kClsPerBlock / kClsThreads; ++k) {
    int i = base + k * kClsThreads + threadIdx.x;
    int ring = (i < n) ? (int)ring_id[i] : -1;
    unsigned peers = __match_any_sync(0xffffffffu, ring);
    int lrank = __popc(peers & ((1u << lane_id()) - 1u));
    if (ring >= 0 && lrank == 0) warpcnt[w][ring] = __popc(peers);
    __syncthreads();
    if (ring >= 0) {
      int pos = running[ring] + lrank;
      for (int ww = 0; ww < w; ++ww) pos += warpcnt[ww][ring];
      float4 p = __ldg(in + i);
      const float azi_rel = adjusted_azimuth(azi[i], start_ori) - start_ori;                       // :526
      const float rel_time = (float)(P.scan_period * (double)azi_rel / (double)range_ori);         // :528
      laser[pos] = make_float4(p.x, p.y, p.z, (float)ring + rel_time);          // :531
      full[pos] = make_float4(p.x, p.y, p.z, (float)(int)p.w + rel_time);       // :532
      orig[pos] = i;
    }
    __syncthreads();
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
      int s2 = 0;
#pragma unroll
      for (int ww = 0; ww < kClsThreads / 32; ++ww) { s2 += warpcnt[ww][r]; warpcnt[ww][r] = 0; }
      running[r] += s2;
    }
    __syncthreads();
  }
}

// ---- helpers for the ring kernel -------------------------------------------------------------
__device__ __forceinline__ float sqdiff(const float *sx, const float *sy, const float *sz, int a, int b) {
  float dx = sx[a] - sx[b], dy = sy[a] - sy[b], dz = sz[a] - sz[b];
  return dx * dx + dy * dy + dz * dz;
}
__device__ __forceinline__ float sqdiff_w(const float *sx, const float *sy, const float *sz, int a, int b, float wb) {
  float dx = sx[a] - sx[b] * wb, dy = sy[a] - sy[b] * wb, dz = sz[a] - sz[b] * wb;
  return dx * dx + dy * dy + dz * dz;
}
__device__ __forceinline__ void cswap(unsigned long long *k, int i, int p) {
  unsigned long long a = k[i], b = k[p];
  if (a > b) { k[i] = b; k[p] = a; }
}

// Normalised bitonic network (all comparators ascending) over keys[0..m): positions >= m act as
// +inf, so comparators touching them are skipped.  `nthr` cooperating threads, `sync()` between steps.
template <typename SyncF>
__device__ __forceinline__ void bitonic_sort(unsigned long long *keys, int m, int tid, int nthr, SyncF sync) {
  int P = 1;
  while (P < m) P <<= 1;
  for (int k = 2; k <= P; k <<= 1) {
    int hk = k >> 1;
    for (int t = tid; t < (P >> 1); t += nthr) {
      int blk = t / hk, off = t - blk * hk;
      int i = blk * k + off, p = blk * k + k - 1 - off;
      if (p < m) cswap(keys, i, p);
    }
    sync();
    for (int j = k >> 2; j > 0; j >>= 1) {
      for (int t = tid; t < (P >> 1); t += nthr) {
        int i = 2 * j * (t / j) + (t % j), p = i + j;
        if (p < m) cswap(keys, i, p);
      }
      sync();
    }
  }
}

// MaskPickedInRing (PointProcessor.cc:624-645), executed by a full warp.
__device__ __forceinline__ void mask_picked(const float *sx, const float *sy, const float *sz, unsigned char *smask, int idx, int d) {
  int l = lane_id();
  bool fwd_break = false, bwd_break = false;
  if (l >= 1 && l <= d) fwd_break = (double)sqdiff(sx, sy, sz, idx + l, idx + l - 1) > 0.05;
  if (l >= 1 && l <= d) bwd_break = (double)sqdiff(sx, sy, sz, idx - l, idx - l + 1) > 0.05;
  unsigned fb = __ballot_sync(0xffffffffu, fwd_break);
  unsigned bb = __ballot_sync(0xffffffffu, bwd_break);
  int ff = fb ? (__ffs(fb) - 1) : (d + 1);  // first breaking step (1-based lane)
  int bf = bb ? (__ffs(bb) - 1) : (d + 1);
  if (l == 0) smask[idx] = 1;
  if (l >= 1 && l <= d) {
    if (l < ff) smask[idx + l] = 1;
    if (l < bf) smask[idx - l] = 1;
  }
  __syncwarp();
}

__global__ void __launch_bounds__(kRingThreads, 1)
a_ring(const float4 *__restrict__ laser, const int *__restrict__ ring_start, PPParams P, const float *__restrict__ start_ori_p,
       unsigned char *__restrict__ mask_out, signed char *__restrict__ label_out, int *__restrict__ pick_less,
       int *__restrict__ n_less, int *__restrict__ pick_flat, int *__restrict__ n_flat, float4 *__restrict__ lf_ring,
       int *__restrict__ lf_count, int *__restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int sscan[40];
  __shared__ float sred[6][kRingThreads / 32];
  __shared__ int sbox[8];
  const int ring = blockIdx.x;
  const int s0 = ring_start[ring];
  const int n = ring_start[ring + 1] - s0;
  const int d = P.d, S = P.S;
  const int tid = threadIdx.x, T = blockDim.x;
  for (int j = tid; j < S; j += T) { n_less[ring * S + j] = 0; n_flat[ring * S + j] = 0; }
  if (tid == 0) lf_count[ring] = 0;
  if (n <= 2 * d + 1 || n > kMaxRingPoints) {  // :660 (end_idx <= start_idx + 2d): ring skipped
    for (int i = tid; i < n; i += T) { mask_out[s0 + i] = 0; label_out[s0 + i] = 0; }
    if (n > kMaxRingPoints && tid == 0) atomicExch(err_flag, 1);
    return;
  }

  unsigned long long *keys = reinterpret_cast<unsigned long long *>(smem_raw);
  float *sx = reinterpret_cast<float *>(keys + n);
  float *sy = sx + n;
  float *sz = sy + n;
  float *sw = sz + n;
  unsigned char *smask = reinterpret_cast<unsigned char *>(sw + n);
  signed char *slab = reinterpret_cast<signed char *>(smask + n + 8);

  for (int i = tid; i < n; i += T) {
    float4 p = __ldg(laser + s0 + i);
    sx[i] = p.x; sy[i] = p.y; sz[i] = p.z; sw[i] = p.w;
    smask[i] = 0;
    slab[i] = 3;  // not (yet) inside a processed subregion
  }
  if (tid < 8) smask[n + tid] = 0;
  __syncthreads();

  // ---- PrepareRing (:542-585): every i only ORs ones into the mask -> order independent.
  for (int i = d + tid; i < n - d; i += T) {
    float diff_next2 = sqdiff(sx, sy, sz, i, i + 1);
    bool done = false;
    if ((double)diff_next2 > 0.1) {
      float depth = sqrtf(sx[i] * sx[i] + sy[i] * sy[i] + sz[i] * sz[i]);
      float depth_next = sqrtf(sx[i + 1] * sx[i + 1] + sy[i + 1] * sy[i + 1] + sz[i + 1] * sz[i + 1]);
      if (depth > depth_next) {
        float wd = sqrtf(sqdiff_w(sx, sy, sz, i + 1, i, depth_next / depth)) / depth_next;
        if ((double)wd < 0.1) {
          for (int k = 0; k <= d; ++k) smask[i - d + k] = 1;
          done = true;
        }
      } else {
        float wd = sqrtf(sqdiff_w(sx, sy, sz, i, i + 1, depth / depth_next)) / depth;
        if ((double)wd < 0.1) {
          for (int k = 0; k <= d; ++k) smask[i + 1 + k] = 1;  // may touch smask[n] like the reference
          done = true;
        }
      }
    }
    if (!done) {
      float diff_prev2 = sqdiff(sx, sy, sz, i, i - 1);
      float dis2 = sx[i] * sx[i] + sy[i] * sy[i] + sz[i] * sz[i];
      if ((double)diff_next2 > 0.0002 * (double)dis2 && (double)diff_prev2 > 0.0002 * (double)dis2) smask[i] = 1;
    }
  }
  // ---- curvature keys (:598-612)
  const float negk = (float)(-2 * d);
  for (int i = d + tid; i < n - d; i += T) {
    float dx = negk * sx[i], dy = negk * sy[i], dz = negk * sz[i];
    for (int j = 1; j <= d; ++j) {
      dx += sx[i + j] + sx[i - j];
      dy += sy[i + j] + sy[i - j];
      dz += sz[i + j] + sz[i - j];
    }
    float curv = dx * dx + dy * dy + dz * dz;
    keys[i] = ((unsigned long long)__float_as_uint(curv) << 32) | (unsigned)i;
  }
  __syncthreads();

  // ---- per-subregion sort: one warp per subregion (:672-675, :616)
  {
    const int w = warp_id(), nw = T >> 5;
    for (int j = w; j < S; j += nw) {
      long long sp = ((long long)d * (S - j) + (long long)(n - d) * j) / S;
      long long ep = ((long long)d * (S - 1 - j) + (long long)(n - d) * (j + 1)) / S - 1;
      if (ep <= sp) continue;
      bitonic_sort(keys + sp, (int)(ep - sp + 1), (int)lane_id(), 32, [] { __syncwarp(); });
    }
  }
  __syncthreads();

  // ---- pick loops (:686-732), warp 0, subregions in order (the mask carries across them)
  if (warp_id() == 0) {
    const int l = lane_id();
    for (int j = 0; j < S; ++j) {
      long long sp = ((long long)d * (S - j) + (long long)(n - d) * j) / S;
      long long ep = ((long long)d * (S - 1 - j) + (long long)(n - d) * (j + 1)) / S - 1;
      if (ep <= sp) continue;
      const int m = (int)(ep - sp + 1);
      const unsigned long long *kk = keys + sp;
      for (int i = (int)sp + l; i <= (int)ep; i += 32) slab[i] = 0;
      __syncwarp();
      // corners: walk from the largest curvature down
      int picked = 0, k = m;
      int *pl = pick_less + (size_t)(ring * S + j) * kMaxLessSharp;
      while (k > 0 && picked < P.max_less_sharp) {
        int c = k - 1 - l;
        bool ok = false, stop = false;
        int idx = 0;
        if (c >= 0) {
          unsigned long long key = kk[c];
          float curv = __uint_as_float((unsigned)(key >> 32));
          idx = (int)(unsigned)key;
          bool big = curv > P.surf_curv_th;
          ok = big && smask[idx] == 0;
          stop = !big;
        }
        unsigned okb = __ballot_sync(0xffffffffu, ok), stb = __ballot_sync(0xffffffffu, stop);
        int f = okb ? __ffs(okb) - 1 : 32, s = stb ? __ffs(stb) - 1 : 32;
        if (s < f) break;             // sorted: nothing below can pass the curvature test
        if (f == 32) { k -= 32; continue; }
        int pidx = __shfl_sync(0xffffffffu, idx, f);
        ++picked;
        if (l == 0) {
          slab[pidx] = (picked <= P.max_sharp) ? 2 : 1;
          pl[picked - 1] = s0 + pidx;
        }
        mask_picked(sx, sy, sz, smask, pidx, d);
        k -= f + 1;
      }
      if (l == 0) n_less[ring * S + j] = picked;
      // flats: walk from the smallest curvature up
      int fpicked = 0;
      k = 0;
      int *pf = pick_flat + (size_t)(ring * S + j) * kMaxFlat;
      while (k < m && fpicked < P.max_flat) {
        int c = k + l;
        bool ok = false, stop = false;
        int idx = 0;
        if (c < m) {
          unsigned long long key = kk[c];
          float curv = __uint_as_float((unsigned)(key >> 32));
          idx = (int)(unsigned)key;
          bool small = curv < P.surf_curv_th;
          ok = small && smask[idx] == 0;
          stop = !small;
        }
        unsigned okb = __ballot_sync(0xffffffffu, ok), stb = __ballot_sync(0xffffffffu, stop);
        int f = okb ? __ffs(okb) - 1 : 32, s = stb ? __ffs(stb) - 1 : 32;
        if (s < f) break;
        if (f == 32) { k += 32; continue; }
        int pidx = __shfl_sync(0xffffffffu, idx, f);
        ++fpicked;
        if (l == 0) {
          slab[pidx] = -1;
          pf[fpicked - 1] = s0 + pidx;
        }
        mask_picked(sx, sy, sz, smask, pidx, d);
        k += f + 1;
      }
      if (l == 0) n_flat[ring * S + j] = fpicked;
      __syncwarp();
    }
  }
  __syncthreads();

  for (int i = tid; i < n; i += T) {
    mask_out[s0 + i] = smask[i];
    signed char lb = slab[i];
    label_out[s0 + i] = (lb == 3) ? 0 : lb;
  }

  // ---- less-flat cloud of this ring (:728-751): members = label <= 0 inside processed subregions
  // ordered compaction of member indices into keys[] (low 32 bits), bbox reduction
  float mn0 = INFINITY, mn1 = INFINITY, mn2 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY, mx2 = -INFINITY;
  int L = 0;
  for (int base = 0; base < n; base += T) {
    int i = base + tid;
    int flag = (i < n && slab[i] <= 0) ? 1 : 0;
    int tot;
    int pos = block_scan_excl(flag, sscan, &tot);
    if (flag) {
      keys[L + pos] = (unsigned)i;
      mn0 = fminf(mn0, sx[i]); mn1 = fminf(mn1, sy[i]); mn2 = fminf(mn2, sz[i]);
      mx0 = fmaxf(mx0, sx[i]); mx1 = fmaxf(mx1, sy[i]); mx2 = fmaxf(mx2, sz[i]);
    }
    L += tot;
  }
  if (L == 0) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn0 = fminf(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mn1 = fminf(mn1, __shfl_xor_sync(0xffffffffu, mn1, o));
    mn2 = fminf(mn2, __shfl_xor_sync(0xffffffffu, mn2, o)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o)); mx2 = fmaxf(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
  }
  if (lane_id() == 0) {
    int w = warp_id();
    sred[0][w] = mn0; sred[1][w] = mn1; sred[2][w] = mn2; sred[3][w] = mx0; sred[4][w] = mx1; sred[5][w] = mx2;
  }
  __syncthreads();
  if (tid == 0) {
    float a[6];
    for (int q = 0; q < 6; ++q) {
      float v = sred[q][0];
      for (int w = 1; w < T / 32; ++w) v = (q < 3) ? fminf(v, sred[q][w]) : fmaxf(v, sred[q][w]);
      a[q] = v;
    }
    const float inv = 1.0f / P.leaf;
    long long ddx = (long long)((a[3] - a[0]) * inv) + 1, ddy = (long long)((a[4] - a[1]) * inv) + 1,
              ddz = (long long)((a[5] - a[2]) * inv) + 1;
    int overflow = (ddx * ddy * ddz > 2147483647LL) ? 1 : 0;
    int mb0 = (int)floorf(a[0] * inv), mb1 = (int)floorf(a[1] * inv), mb2 = (int)floorf(a[2] * inv);
    int xb0 = (int)floorf(a[3] * inv), xb1 = (int)floorf(a[4] * inv);
    sbox[0] = mb0; sbox[1] = mb1; sbox[2] = mb2;
    sbox[3] = xb0 - mb0 + 1;                       // div_b[0]
    sbox[4] = (xb0 - mb0 + 1) * (xb1 - mb1 + 1);   // div_b[0]*div_b[1]
    sbox[5] = overflow;
  }
  __syncthreads();
  const float start_ori = *start_ori_p;
  if (sbox[5]) {  // PCL: leaf too small -> output = input
    for (int c = tid; c < L; c += T) {
      int i = (int)(unsigned)keys[c];
      float azi = azimuth_of(sx[i], sy[i]);
      float rt = rel_time_of(azi, start_ori, P.scan_period);
      lf_ring[s0 + c] = make_float4(sx[i], sy[i], sz[i], (float)(int)sw[i] + rt);
    }
    if (tid == 0) lf_count[ring] = L;
    return;
  }
  {
    const float inv = 1.0f / P.leaf;
    const int mb0 = sbox[0], mb1 = sbox[1], mb2 = sbox[2], mul1 = sbox[3], mul2 = sbox[4];
    for (int c = tid; c < L; c += T) {
      int i = (int)(unsigned)keys[c];
      int ijk0 = (int)(floorf(sx[i] * inv) - (float)mb0);
      int ijk1 = (int)(floorf(sy[i] * inv) - (float)mb1);
      int ijk2 = (int)(floorf(sz[i] * inv) - (float)mb2);
      unsigned vidx = (unsigned)(ijk0 + ijk1 * mul1 + ijk2 * mul2);
      keys[c] = ((unsigned long long)vidx << 32) | (unsigned)i;
    }
  }
  __syncthreads();
  bitonic_sort(keys, L, tid, T, [] { __syncthreads(); });
  // ordered emit of one centroid per voxel (ascending voxel index; in-voxel sum in index order)
  int emitted = 0;
  for (int base = 0; base < L; base += T) {
    int c = base + tid;
    int head = 0;
    if (c < L) {
      unsigned v = (unsigned)(keys[c] >> 32);
      head = (c == 0) || (v != (unsigned)(keys[c - 1] >> 32));
    }
    int tot;
    int pos = block_scan_excl(head, sscan, &tot);
    if (head) {
      unsigned v = (unsigned)(keys[c] >> 32);
      float ax = 0.f, ay = 0.f, az = 0.f, ai = 0.f;
      int cnt = 0;
      for (int c2 = c; c2 < L && (unsigned)(keys[c2] >> 32) == v; ++c2) {
        int i = (int)(unsigned)keys[c2];
        ax += sx[i]; ay += sy[i]; az += sz[i]; ai += sw[i];
        ++cnt;
      }
      float fn = (float)cnt;
      float cx = ax / fn, cy = ay / fn, cz = az / fn, ci = ai / fn;
      float azi = azimuth_of(cx, cy);                              // :758-776
      float rt = rel_time_of(azi, start_ori, P.scan_period);
      lf_ring[s0 + emitted + pos] = make_float4(cx, cy, cz, (float)(int)ci + rt);
    }
    emitted += tot;
  }
  if (tid == 0) lf_count[ring] = emitted;
}

__global__ void __launch_bounds__(256)
a_compact(const float4 *__restrict__ laser, const int *__restrict__ ring_start, PPParams P, const int *__restrict__ pick_less,
          const int *__restrict__ n_less, const int *__restrict__ pick_flat, const int *__restrict__ n_flat,
          const float4 *__restrict__ lf_ring, const int *__restrict__ lf_count, float4 *__restrict__ out_sharp,
          float4 *__restrict__ out_less, float4 *__restrict__ out_flat, float4 *__restrict__ out_lf, int *__restrict__ idx_sharp,
          int *__restrict__ idx_less, int *__restrict__ idx_flat, int *__restrict__ counts) {
  __shared__ int sscan[40];
  __shared__ int soff[4];
  const int ring = blockIdx.x, R = P.num_rings, S = P.S, tid = threadIdx.x;
  // offsets of this ring = sums over all earlier rings (tiny arrays: R*S <= 4096 entries)
  int a_sh = 0, a_ls = 0, a_fl = 0, a_lf = 0;
  for (int e = tid; e < ring * S; e += blockDim.x) {
    int nl = n_less[e];
    a_ls += nl; a_sh += min(nl, P.max_sharp); a_fl += n_flat[e];
  }
  for (int r = tid; r < ring; r += blockDim.x) a_lf += lf_count[r];
  int t;
  block_scan_excl(a_sh, sscan, &t); if (tid == 0) soff[0] = t;
  block_scan_excl(a_ls, sscan, &t); if (tid == 0) soff[1] = t;
  block_scan_excl(a_fl, sscan, &t); if (tid == 0) soff[2] = t;
  block_scan_excl(a_lf, sscan, &t); if (tid == 0) soff[3] = t;
  __syncthreads();
  const int o_lf = soff[3];
  __shared__ int sub_sh[kMaxSub + 1], sub_ls[kMaxSub + 1], sub_fl[kMaxSub + 1];
  if (tid == 0) {
    int a = soff[0], b = soff[1], c = soff[2];
    for (int j = 0; j < S; ++j) {
      int nl = n_less[ring * S + j];
      sub_sh[j] = a; sub_ls[j] = b; sub_fl[j] = c;
      a += min(nl, P.max_sharp); b += nl; c += n_flat[ring * S + j];
    }
    sub_sh[S] = a; sub_ls[S] = b; sub_fl[S] = c;
    if (ring == R - 1) { counts[0] = a; counts[1] = b; counts[2] = c; counts[3] = o_lf + lf_count[ring]; counts[4] = ring_start[R]; }
  }
  __syncthreads();
  for (int q = tid; q < S * kMaxLessSharp; q += blockDim.x) {
    int j = q / kMaxLessSharp, k = q - j * kMaxLessSharp;
    int e = ring * S + j;
    if (k < n_less[e]) {
      int gi = pick_less[(size_t)e * kMaxLessSharp + k];
      float4 p = laser[gi];
      if (k < P.max_sharp) { out_sharp[sub_sh[j] + k] = p; idx_sharp[sub_sh[j] + k] = gi; }
      out_less[sub_ls[j] + k] = p; idx_less[sub_ls[j] + k] = gi;
    }
  }
  for (int q = tid; q < S * kMaxFlat; q += blockDim.x) {
    int j = q / kMaxFlat, k = q - j * kMaxFlat;
    int e = ring * S + j;
    if (k < n_flat[e]) {
      int gi = pick_flat[(size_t)e * kMaxFlat + k];
      out_flat[sub_fl[j] + k] = laser[gi]; idx_flat[sub_fl[j] + k] = gi;
    }
  }
  const int nlf = lf_count[ring], s0 = ring_start[ring];
  for (int i = tid; i < nlf; i += blockDim.x) out_lf[o_lf + i] = lf_ring[s0 + i];
}

}  // namespace lio

// ------------------------------------------------------------------------------------------------
// host side of the C-ABI
using namespace lio;

struct lio_pp {
  lio_pp_config cfg;
  PPParams P;
  int device;
  cudaStream_t stream;
  int max_points, nb_max;
  size_t ring_smem;
  // device buffers
  DevMem<float4> d_in, d_laser, d_full, d_lf_ring;
  DevMem<float4> d_out_sharp, d_out_less, d_out_flat, d_out_lf;
  DevMem<int16_t> d_ring_id;
  DevMem<float> d_azi, d_start_ori;
  DevMem<int> d_first_valid, d_hist, d_offsets, d_ring_start, d_orig;
  DevMem<unsigned char> d_mask;
  DevMem<signed char> d_label;
  DevMem<int> d_pick_less, d_n_less, d_pick_flat, d_n_flat, d_lf_count;
  DevMem<int> d_idx_sharp, d_idx_less, d_idx_flat, d_counts, d_err;
  DevMem<unsigned short> d_rings_in;  // ring-field variant only (allocated on first use)
  DevMem<int> d_end_bits;
  HostMem<int> h_counts;   // pinned: counts[0..4], err
  int launches = 0;
  int last_n = 0;
  bool counts_valid = false;
};

extern "C" void lio_pp_default_config(lio_pp_config *c) {
  c->lower_bound = -15.f; c->upper_bound = 15.f; c->num_rings = 16; c->scan_period = 0.1;
  c->num_scan_subregions = 8; c->num_curvature_regions = 5; c->surf_curv_th = 0.1f;
  c->max_corner_sharp = 2; c->max_corner_less_sharp = 20; c->max_surf_flat = 4; c->less_flat_filter_size = 0.2f;
}

extern "C" int lio_pp_create(const lio_pp_config *cfg, int max_points, int device, void *cuda_stream, lio_pp **out) {
  if (!cfg || !out || max_points <= 0) return LIO_ERR_INVALID;
  // a negative pick budget would make a_compact's min(n_less, max_sharp) offsets, and so the sharp count, negative
  if (cfg->num_rings < 1 || cfg->num_rings > kMaxRings || cfg->num_scan_subregions < 1 || cfg->num_scan_subregions > kMaxSub ||
      cfg->num_curvature_regions < 1 || cfg->num_curvature_regions > 16 || cfg->max_corner_less_sharp > kMaxLessSharp ||
      cfg->max_surf_flat > kMaxFlat || cfg->max_corner_sharp > cfg->max_corner_less_sharp || cfg->max_corner_sharp < 0 ||
      cfg->max_corner_less_sharp < 0 || cfg->max_surf_flat < 0 || !(cfg->less_flat_filter_size > 0) ||
      !(cfg->upper_bound > cfg->lower_bound)) {
    lio_set_last_error(__FILE__, __LINE__, "lio_pp_create: configuration outside supported limits");
    return LIO_ERR_INVALID;
  }
  LIO_TRY(select_device(device));
  std::unique_ptr<lio_pp> pp(new (std::nothrow) lio_pp());
  if (!pp) return LIO_ERR_INVALID;
  pp->cfg = *cfg;
  pp->device = device;
  pp->stream = (cudaStream_t)cuda_stream;
  pp->max_points = max_points;
  PPParams &P = pp->P;
  P.lower_bound = cfg->lower_bound;
  P.factor = (cfg->num_rings - 1) / (cfg->upper_bound - cfg->lower_bound);  // PointProcessor.cc:80 (int / float)
  P.num_rings = cfg->num_rings; P.scan_period = cfg->scan_period; P.S = cfg->num_scan_subregions; P.d = cfg->num_curvature_regions;
  P.surf_curv_th = cfg->surf_curv_th; P.max_sharp = cfg->max_corner_sharp; P.max_less_sharp = cfg->max_corner_less_sharp;
  P.max_flat = cfg->max_surf_flat; P.leaf = cfg->less_flat_filter_size;
  const int R = P.num_rings, S = P.S;
  pp->nb_max = (max_points + kClsPerBlock - 1) / kClsPerBlock;
  const size_t N = (size_t)max_points;
  const size_t RS = (size_t)R * S;
  if (!alloc(pp->d_in, N) || !alloc(pp->d_laser, N) || !alloc(pp->d_full, N) || !alloc(pp->d_lf_ring, N) || !alloc(pp->d_out_lf, N) ||
      !alloc(pp->d_out_sharp, RS * kMaxLessSharp) || !alloc(pp->d_out_less, RS * kMaxLessSharp) || !alloc(pp->d_out_flat, RS * kMaxFlat) ||
      !alloc(pp->d_ring_id, N) || !alloc(pp->d_azi, N) || !alloc(pp->d_start_ori, 1) || !alloc(pp->d_first_valid, 1) ||
      !alloc(pp->d_hist, (size_t)pp->nb_max * R) || !alloc(pp->d_offsets, (size_t)pp->nb_max * R) || !alloc(pp->d_ring_start, R + 1) ||
      !alloc(pp->d_orig, N) || !alloc(pp->d_mask, N) || !alloc(pp->d_label, N) || !alloc(pp->d_pick_less, RS * kMaxLessSharp) ||
      !alloc(pp->d_n_less, RS) || !alloc(pp->d_pick_flat, RS * kMaxFlat) || !alloc(pp->d_n_flat, RS) || !alloc(pp->d_lf_count, R) ||
      !alloc(pp->d_idx_sharp, RS * kMaxLessSharp) || !alloc(pp->d_idx_less, RS * kMaxLessSharp) || !alloc(pp->d_idx_flat, RS * kMaxFlat) ||
      !alloc(pp->d_counts, 8) || !alloc(pp->d_err, 1) || !alloc_host(pp->h_counts, 16))
    return LIO_ERR_CUDA;
  LIO_CUDA_OK(cudaMemset(pp->d_err, 0, sizeof(int)));
  // shared memory of the ring kernel: sized for the largest ring we may see
  int maxn = max_points < kMaxRingPoints ? max_points : kMaxRingPoints;
  pp->ring_smem = (size_t)maxn * (8 + 16 + 2) + 64;
  LIO_CUDA_OK(cudaFuncSetAttribute(a_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pp->ring_smem));
  *out = pp.release();
  return LIO_OK;
}

extern "C" int lio_pp_destroy(lio_pp *pp) {
  if (!pp) return LIO_OK;
  cudaSetDevice(pp->device);   // the buffers belong to the handle's device, whichever is current
  delete pp;
  return LIO_OK;
}

extern "C" int lio_pp_process_dev(lio_pp *pp, const float *xyzi_dev, int n) {
  LIO_ENTER(pp);
  if ((!xyzi_dev && n > 0) || n < 0) return LIO_ERR_INVALID;
  if (n > pp->max_points) return LIO_ERR_CAPACITY;
  cudaStream_t st = pp->stream;
  const PPParams &P = pp->P;
  const int R = P.num_rings;
  const float4 *in = reinterpret_cast<const float4 *>(xyzi_dev);
  pp->launches = 0;
  pp->last_n = n;
  pp->counts_valid = false;
  int nb = (n + kClsPerBlock - 1) / kClsPerBlock;
  if (nb < 1) nb = 1;
  LIO_CUDA_OK(cudaMemsetAsync(pp->d_first_valid, 0x7f, sizeof(int), st));
  a_classify<<<nb, kClsThreads, 0, st>>>(in, n, P, pp->d_ring_id, pp->d_azi, pp->d_first_valid, pp->d_hist);
  a_scan<<<1, kMaxRings, 0, st>>>(pp->d_hist, nb, R, pp->d_offsets, pp->d_ring_start);
  a_scatter<<<nb, kClsThreads, 0, st>>>(in, n, P, pp->d_ring_id, pp->d_azi, pp->d_first_valid, pp->d_offsets, pp->d_laser,
                                        pp->d_full, pp->d_orig, pp->d_start_ori);
  a_ring<<<R, kRingThreads, pp->ring_smem, st>>>(pp->d_laser, pp->d_ring_start, P, pp->d_start_ori, pp->d_mask, pp->d_label,
                                                 pp->d_pick_less, pp->d_n_less, pp->d_pick_flat, pp->d_n_flat, pp->d_lf_ring,
                                                 pp->d_lf_count, pp->d_err);
  a_compact<<<R, 256, 0, st>>>(pp->d_laser, pp->d_ring_start, P, pp->d_pick_less, pp->d_n_less, pp->d_pick_flat, pp->d_n_flat,
                               pp->d_lf_ring, pp->d_lf_count, pp->d_out_sharp, pp->d_out_less, pp->d_out_flat, pp->d_out_lf,
                               pp->d_idx_sharp, pp->d_idx_less, pp->d_idx_flat, pp->d_counts);
  pp->launches = 5;
  LIO_CUDA_OK(cudaGetLastError());
  LIO_CUDA_OK(cudaMemcpyAsync(pp->h_counts, pp->d_counts, 5 * sizeof(int), cudaMemcpyDeviceToHost, st));
  LIO_CUDA_OK(cudaMemcpyAsync(pp->h_counts + 8, pp->d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  return LIO_OK;
}

static int pp_sync_counts(lio_pp *pp) {
  if (pp->counts_valid) return LIO_OK;
  LIO_CUDA_OK(cudaStreamSynchronize(pp->stream));
  if (pp->h_counts[8] != 0) {
    lio_set_last_error(__FILE__, __LINE__, "stage A: a ring holds more points than the shared-memory ring kernel supports (8192)");
    cudaMemsetAsync(pp->d_err, 0, sizeof(int), pp->stream);
    return LIO_ERR_CAPACITY;
  }
  pp->counts_valid = true;
  return LIO_OK;
}

extern "C" int lio_pp_process_host(lio_pp *pp, const float *xyzi, int n) {
  LIO_ENTER(pp);
  if ((!xyzi && n > 0) || n < 0) return LIO_ERR_INVALID;
  if (n > pp->max_points) return LIO_ERR_CAPACITY;
  if (n > 0) LIO_CUDA_OK(cudaMemcpyAsync(pp->d_in, xyzi, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, pp->stream));
  LIO_TRY(lio_pp_process_dev(pp, reinterpret_cast<const float *>(pp->d_in.get()), n));
  return pp_sync_counts(pp);
}

// PointToRing (ring-field variant, PointProcessor.cc:428-536) + ExtractFeaturePoints on device buffers; stream-ordered, no wait.
extern "C" int lio_pp_process_dev_ring(lio_pp *pp, const float *xyzi_dev, const uint16_t *rings_dev, int n) {
  LIO_ENTER(pp);
  if (((!xyzi_dev || !rings_dev) && n > 0) || n < 0) return LIO_ERR_INVALID;
  if (n > pp->max_points) return LIO_ERR_CAPACITY;
  if (!pp->d_end_bits && !alloc(pp->d_end_bits, 1)) return LIO_ERR_CUDA;
  cudaStream_t st = pp->stream;
  const PPParams &P = pp->P;
  const int R = P.num_rings;
  const float4 *in = reinterpret_cast<const float4 *>(xyzi_dev);
  const unsigned short *rings = reinterpret_cast<const unsigned short *>(rings_dev);
  pp->launches = 0;
  pp->last_n = n;
  pp->counts_valid = false;
  int nb = (n + kClsPerBlock - 1) / kClsPerBlock;
  if (nb < 1) nb = 1;
  LIO_CUDA_OK(cudaMemsetAsync(pp->d_first_valid, 0x7f, sizeof(int), st));
  LIO_CUDA_OK(cudaMemsetAsync(pp->d_end_bits, 0, sizeof(int), st));   // end_ori_ = 0
  a_classify_ring<<<nb, kClsThreads, 0, st>>>(in, rings, n, P, pp->d_ring_id, pp->d_azi, pp->d_first_valid, pp->d_hist);
  a_scan<<<1, kMaxRings, 0, st>>>(pp->d_hist, nb, R, pp->d_offsets, pp->d_ring_start);
  a_endori<<<std::min(nb, 132), 256, 0, st>>>(pp->d_azi, pp->d_ring_id, n, pp->d_first_valid, pp->d_end_bits);
  a_scatter_ring<<<nb, kClsThreads, 0, st>>>(in, n, P, pp->d_ring_id, pp->d_azi, pp->d_first_valid, pp->d_end_bits, pp->d_offsets,
                                             pp->d_laser, pp->d_full, pp->d_orig, pp->d_start_ori);
  a_ring<<<R, kRingThreads, pp->ring_smem, st>>>(pp->d_laser, pp->d_ring_start, P, pp->d_start_ori, pp->d_mask, pp->d_label,
                                                 pp->d_pick_less, pp->d_n_less, pp->d_pick_flat, pp->d_n_flat, pp->d_lf_ring,
                                                 pp->d_lf_count, pp->d_err);
  a_compact<<<R, 256, 0, st>>>(pp->d_laser, pp->d_ring_start, P, pp->d_pick_less, pp->d_n_less, pp->d_pick_flat, pp->d_n_flat,
                               pp->d_lf_ring, pp->d_lf_count, pp->d_out_sharp, pp->d_out_less, pp->d_out_flat, pp->d_out_lf,
                               pp->d_idx_sharp, pp->d_idx_less, pp->d_idx_flat, pp->d_counts);
  pp->launches = 6;
  LIO_CUDA_OK(cudaGetLastError());
  LIO_CUDA_OK(cudaMemcpyAsync(pp->h_counts, pp->d_counts, 5 * sizeof(int), cudaMemcpyDeviceToHost, st));
  LIO_CUDA_OK(cudaMemcpyAsync(pp->h_counts + 8, pp->d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  return LIO_OK;
}

// SetInputCloud(PointIR) + the device entry above; host buffers, synchronous.
extern "C" int lio_pp_process_host_ring(lio_pp *pp, const float *xyzi, const uint16_t *rings, int n) {
  LIO_ENTER(pp);
  if (((!xyzi || !rings) && n > 0) || n < 0) return LIO_ERR_INVALID;
  if (n > pp->max_points) return LIO_ERR_CAPACITY;
  if (!pp->d_rings_in && !alloc(pp->d_rings_in, (size_t)pp->max_points)) return LIO_ERR_CUDA;
  if (n > 0) {
    LIO_CUDA_OK(cudaMemcpyAsync(pp->d_in, xyzi, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, pp->stream));
    LIO_CUDA_OK(cudaMemcpyAsync(pp->d_rings_in, rings, (size_t)n * sizeof(uint16_t), cudaMemcpyHostToDevice, pp->stream));
  }
  LIO_TRY(lio_pp_process_dev_ring(pp, reinterpret_cast<const float *>(pp->d_in.get()), pp->d_rings_in, n));
  return pp_sync_counts(pp);
}

extern "C" int lio_pp_cloud_sizes(lio_pp *pp, int sizes[LIO_PP_NUM_CLOUDS]) {
  LIO_ENTER(pp);
  if (!sizes) return LIO_ERR_INVALID;
  LIO_TRY(pp_sync_counts(pp));
  sizes[0] = pp->h_counts[4]; sizes[1] = pp->h_counts[4]; sizes[2] = pp->h_counts[0]; sizes[3] = pp->h_counts[1];
  sizes[4] = pp->h_counts[2]; sizes[5] = pp->h_counts[3];
  return LIO_OK;
}

static const float4 *pp_cloud_ptr(lio_pp *pp, int which) {
  switch (which) {
    case LIO_PP_LASER_SCANS: return pp->d_laser;
    case LIO_PP_CLOUD_IN_RINGS: return pp->d_full;
    case LIO_PP_CORNER_SHARP: return pp->d_out_sharp;
    case LIO_PP_CORNER_LESS_SHARP: return pp->d_out_less;
    case LIO_PP_SURF_FLAT: return pp->d_out_flat;
    case LIO_PP_SURF_LESS_FLAT: return pp->d_out_lf;
  }
  return nullptr;
}

extern "C" int lio_pp_cloud_dev(lio_pp *pp, int which, const float **ptr) {
  LIO_ENTER_HOST(pp);
  if (!ptr) return LIO_ERR_INVALID;
  const float4 *p = pp_cloud_ptr(pp, which);
  if (!p) return LIO_ERR_INVALID;
  *ptr = reinterpret_cast<const float *>(p);
  return LIO_OK;
}

extern "C" int lio_pp_download_cloud(lio_pp *pp, int which, float *out, int cap, int *n) {
  LIO_ENTER(pp);
  if (!n) return LIO_ERR_INVALID;
  int sizes[LIO_PP_NUM_CLOUDS];
  LIO_TRY(lio_pp_cloud_sizes(pp, sizes));
  if (which < 0 || which >= LIO_PP_NUM_CLOUDS) return LIO_ERR_INVALID;
  return read_back((float4 *)out, pp_cloud_ptr(pp, which), sizes[which], cap, pp->stream, n);
}

extern "C" int lio_pp_download_index(lio_pp *pp, int which, int32_t *out, int cap, int *n) {
  LIO_ENTER(pp);
  if (!n) return LIO_ERR_INVALID;
  LIO_TRY(pp_sync_counts(pp));
  const int *src = nullptr;
  int cnt = 0;
  switch (which) {
    case LIO_PP_IDX_SHARP: src = pp->d_idx_sharp; cnt = pp->h_counts[0]; break;
    case LIO_PP_IDX_LESS_SHARP: src = pp->d_idx_less; cnt = pp->h_counts[1]; break;
    case LIO_PP_IDX_FLAT: src = pp->d_idx_flat; cnt = pp->h_counts[2]; break;
    case LIO_PP_IDX_ORIG: src = pp->d_orig; cnt = pp->h_counts[4]; break;
    default: return LIO_ERR_INVALID;
  }
  return read_back((int *)out, src, cnt, cap, pp->stream, n);
}

extern "C" int lio_pp_download_scan_ranges(lio_pp *pp, int32_t *out_2R) {
  LIO_ENTER(pp);
  if (!out_2R) return LIO_ERR_INVALID;
  LIO_TRY(pp_sync_counts(pp));
  const int R = pp->P.num_rings;
  int rs[kMaxRings + 1];
  LIO_TRY(read_back(rs, pp->d_ring_start, R + 1, kMaxRings + 1, pp->stream));
  for (int r = 0; r < R; ++r) {  // PointProcessor.cc:196-200
    out_2R[2 * r] = rs[r];
    out_2R[2 * r + 1] = rs[r + 1] > 0 ? rs[r + 1] - 1 : 0;
  }
  return LIO_OK;
}

extern "C" int lio_pp_download_mask_labels(lio_pp *pp, uint8_t *mask, int8_t *labels, int cap) {
  LIO_ENTER(pp);
  LIO_TRY(pp_sync_counts(pp));
  int n = pp->h_counts[4];
  if (n > cap) return LIO_ERR_CAPACITY;
  // rings too short to be processed (PointProcessor.cc:660) leave their slots untouched: zero-fill
  if (mask) LIO_TRY(read_back(mask, pp->d_mask, n, cap, pp->stream));
  if (labels) LIO_TRY(read_back((signed char *)labels, pp->d_label, n, cap, pp->stream));
  return LIO_OK;
}

extern "C" int lio_pp_start_ori(lio_pp *pp, float *start_ori) {
  LIO_ENTER(pp);
  if (!start_ori) return LIO_ERR_INVALID;
  LIO_TRY(pp_sync_counts(pp));
  return read_back(start_ori, pp->d_start_ori, 1, 1, pp->stream);
}

extern "C" int lio_pp_last_launches(lio_pp *pp) { return pp ? pp->launches : 0; }

extern "C" int lio_pp_cloud_count_dev(lio_pp *pp, int which, const int **n_dev) {
  LIO_ENTER_HOST(pp);
  if (!n_dev) return LIO_ERR_INVALID;
  switch (which) {
    case LIO_PP_LASER_SCANS: case LIO_PP_CLOUD_IN_RINGS: *n_dev = pp->d_counts + 4; break;
    case LIO_PP_CORNER_SHARP: *n_dev = pp->d_counts + 0; break;
    case LIO_PP_CORNER_LESS_SHARP: *n_dev = pp->d_counts + 1; break;
    case LIO_PP_SURF_FLAT: *n_dev = pp->d_counts + 2; break;
    case LIO_PP_SURF_LESS_FLAT: *n_dev = pp->d_counts + 3; break;
    default: return LIO_ERR_INVALID;
  }
  return LIO_OK;
}
