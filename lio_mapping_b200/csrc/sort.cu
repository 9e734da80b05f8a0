// Stable LSD radix sort of (u32 key, u32 value) pairs, 8 bits per pass, hand-written for sm_90a.
// Used by the device VoxelGrid (key = PCL voxel index, value = input index: stability makes the
// in-voxel order the input order, which fixes the fp32 centroid summation order).
//
// One-sweep organisation: ONE histogram kernel counts all four digits of every key, then each pass is ONE kernel: a tile
// (2048 keys) counts its digit, publishes the per-bin aggregate, finds the keys of all earlier tiles per bin by decoupled
// look-back (256 independent look-backs, one per bin and thread), and scatters with stable in-tile ranks.  5 launches
// per sort instead of 12 (histogram / single-CTA scan / scatter per pass).
#include "primitives.cuh"

namespace lio {

constexpr unsigned kRsFlagAgg = 1u << 30, kRsFlagPfx = 2u << 30, kRsValMask = (1u << 30) - 1u;

__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned *p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u32(unsigned *p, unsigned v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ghist[p][b] = number of keys whose digit p equals b
__global__ void __launch_bounds__(kRsThreads)
rs_hist_all(const unsigned *__restrict__ keys, const int *__restrict__ n_dev, int passes, unsigned *__restrict__ ghist) {
  __shared__ unsigned sh[4][kRsBins];
  const int n = *n_dev;
  const int base = blockIdx.x * kRsTile;
  if (base >= n) return;
#pragma unroll
  for (int p = 0; p < 4; ++p) sh[p][threadIdx.x] = 0u;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kRsTile / kRsThreads; ++k) {
    const int i = base + k * kRsThreads + threadIdx.x;
    if (i < n) {
      const unsigned key = keys[i];
#pragma unroll
      for (int p = 0; p < 4; ++p) if (p < passes) atomicAdd(&sh[p][(key >> (8 * p)) & (kRsBins - 1)], 1u);
    }
  }
  __syncthreads();
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const unsigned c = sh[p][threadIdx.x];
    if (p < passes && c) atomicAdd(ghist + p * kRsBins + threadIdx.x, c);
  }
}

__global__ void __launch_bounds__(kRsThreads)
rs_pass(const unsigned *__restrict__ keys, const unsigned *__restrict__ vals, unsigned *__restrict__ keys_out,
        unsigned *__restrict__ vals_out, const int *__restrict__ n_dev, int shift, const unsigned *__restrict__ ghist,
        unsigned *__restrict__ status, int *__restrict__ ticket) {
  __shared__ int sscan[40];
  __shared__ int running[kRsBins];
  __shared__ int warpcnt[kRsThreads / 32][kRsBins];
  __shared__ unsigned tcount[kRsBins];
  __shared__ int stile;
  const int n = *n_dev;
  if (threadIdx.x == 0) stile = atomicAdd(ticket, 1);   // tiles in ticket order: every earlier tile is resident or done
  tcount[threadIdx.x] = 0u;
  __syncthreads();
  const int tile = stile;
  const int base = tile * kRsTile;
  if (base >= n) return;
  // global start of every bin
  int tot;
  const int gbase = block_scan_excl((int)ghist[threadIdx.x], sscan, &tot);
  // this tile's digit counts
  unsigned key[kRsTile / kRsThreads], val[kRsTile / kRsThreads];
#pragma unroll
  for (int k = 0; k < kRsTile / kRsThreads; ++k) {
    const int i = base + k * kRsThreads + threadIdx.x;
    key[k] = 0u; val[k] = 0u;
    if (i < n) { key[k] = keys[i]; val[k] = vals[i]; atomicAdd(&tcount[(key[k] >> shift) & (kRsBins - 1)], 1u); }
  }
  __syncthreads();
  {  // publish the aggregate, look back over the earlier tiles (bin = thread), publish the inclusive prefix
    const unsigned mine = tcount[threadIdx.x];
    unsigned *row = status + (size_t)tile * kRsBins + threadIdx.x;
    unsigned excl = 0u;
    if (tile > 0) {
      st_relaxed_u32(row, kRsFlagAgg | mine);
      for (int t = tile - 1; t >= 0; --t) {
        const unsigned *pr = status + (size_t)t * kRsBins + threadIdx.x;
        unsigned s;
        do { s = ld_relaxed_u32(pr); } while ((s >> 30) == 0u);
        excl += s & kRsValMask;
        if ((s >> 30) == 2u) break;
      }
    }
    st_relaxed_u32(row, kRsFlagPfx | (excl + mine));
    running[threadIdx.x] = gbase + (int)excl;
#pragma unroll
    for (int w = 0; w < kRsThreads / 32; ++w) warpcnt[w][threadIdx.x] = 0;
  }
  __syncthreads();
  // stable scatter: sub-rounds of 256 keys in input order, rank inside a warp by match, across warps by counts
  const int w = warp_id();
#pragma unroll
  for (int k = 0; k < kRsTile / kRsThreads; ++k) {
    const int i = base + k * kRsThreads + threadIdx.x;
    const int bin = (i < n) ? (int)((key[k] >> shift) & (kRsBins - 1)) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    const int lrank = __popc(peers & ((1u << lane_id()) - 1u));
    if (bin >= 0 && lrank == 0) warpcnt[w][bin] = __popc(peers);
    __syncthreads();
    if (bin >= 0) {
      int pos = running[bin] + lrank;
      for (int ww = 0; ww < w; ++ww) pos += warpcnt[ww][bin];
      keys_out[pos] = key[k];
      vals_out[pos] = val[k];
    }
    __syncthreads();
    {
      int s = 0;
#pragma unroll
      for (int ww = 0; ww < kRsThreads / 32; ++ww) { s += warpcnt[ww][threadIdx.x]; warpcnt[ww][threadIdx.x] = 0; }
      running[threadIdx.x] += s;
    }
    __syncthreads();
  }
}

int RadixSortTemp::init(int max_keys) {
  ntiles_max = (max_keys + kRsTile - 1) / kRsTile + 1;
  words = (size_t)4 * kRsBins + 8 + (size_t)4 * ntiles_max * kRsBins;   // digit histograms | tickets | per-pass tile status
  return cudaMalloc(&buf, sizeof(unsigned) * words) == cudaSuccess ? 0 : -1;
}
void RadixSortTemp::destroy() {
  if (buf) cudaFree(buf);
  buf = nullptr;
}

int radix_sort_pairs(unsigned *keys_a, unsigned *vals_a, unsigned *keys_b, unsigned *vals_b, const int *n_dev, int n_max,
                     int key_bits, RadixSortTemp &tmp, cudaStream_t st, int *launches) {
  int ntiles = (n_max + kRsTile - 1) / kRsTile;
  if (ntiles < 1) ntiles = 1;
  if (ntiles > tmp.ntiles_max) return -1;
  const int passes = (key_bits + kRsBits - 1) / kRsBits;
  unsigned *ghist = tmp.buf;
  int *tickets = reinterpret_cast<int *>(tmp.buf + 4 * kRsBins);
  unsigned *status = tmp.buf + 4 * kRsBins + 8;
  cudaMemsetAsync(tmp.buf, 0, sizeof(unsigned) * ((size_t)4 * kRsBins + 8 + (size_t)passes * ntiles * kRsBins), st);
  rs_hist_all<<<ntiles, kRsThreads, 0, st>>>(keys_a, n_dev, passes, ghist);
  unsigned *ki = keys_a, *vi = vals_a, *ko = keys_b, *vo = vals_b;
  for (int p = 0; p < passes; ++p) {
    rs_pass<<<ntiles, kRsThreads, 0, st>>>(ki, vi, ko, vo, n_dev, p * kRsBits, ghist + p * kRsBins, status + (size_t)p * ntiles * kRsBins,
                                           tickets + p);
    unsigned *t = ki; ki = ko; ko = t;
    t = vi; vi = vo; vo = t;
  }
  if (launches) *launches += 1 + passes;
  return passes & 1;
}

}  // namespace lio

// ---- C-ABI test aid: radix_sort_pairs on host buffers ------------------------------------------------------------------
using namespace lio;

extern "C" int lio_radix_sort_pairs_host(const uint32_t *keys, const uint32_t *vals, int n, int key_bits, uint32_t *keys_out,
                                         uint32_t *vals_out, int device) {
  if (n < 0 || key_bits < 1 || key_bits > 32 || (n > 0 && (!keys || !vals || !keys_out || !vals_out))) return LIO_ERR_INVALID;
  if (lio_device_count() <= 0) return LIO_ERR_NO_DEVICE;
  LIO_CUDA_OK(cudaSetDevice(device));
  if (n == 0) return LIO_OK;
  RadixSortTemp tmp;
  unsigned *ka = nullptr, *va = nullptr, *kb = nullptr, *vb = nullptr;
  int *d_n = nullptr;
  int rc = LIO_OK;
  const size_t bytes = sizeof(unsigned) * (size_t)n;
  if (tmp.init(n) != 0 || cudaMalloc(&ka, bytes) != cudaSuccess || cudaMalloc(&va, bytes) != cudaSuccess ||
      cudaMalloc(&kb, bytes) != cudaSuccess || cudaMalloc(&vb, bytes) != cudaSuccess || cudaMalloc(&d_n, sizeof(int)) != cudaSuccess) {
    lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed");
    rc = LIO_ERR_CUDA;
  }
  if (rc == LIO_OK && (cudaMemcpy(ka, keys, bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
                       cudaMemcpy(va, vals, bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
                       cudaMemcpy(d_n, &n, sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess)) {
    lio_set_last_error(__FILE__, __LINE__, "upload failed");
    rc = LIO_ERR_CUDA;
  }
  if (rc == LIO_OK) {
    const int which = radix_sort_pairs(ka, va, kb, vb, d_n, n, key_bits, tmp, 0, nullptr);
    cudaError_t e = which < 0 ? cudaSuccess : cudaDeviceSynchronize();
    if (which < 0) rc = LIO_ERR_CAPACITY;
    else if (e == cudaSuccess) e = cudaMemcpy(keys_out, which ? kb : ka, bytes, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && rc == LIO_OK) e = cudaMemcpy(vals_out, which ? vb : va, bytes, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); rc = LIO_ERR_CUDA; }
  }
  void *p[] = {ka, va, kb, vb, d_n};
  for (void *q : p) if (q) cudaFree(q);
  tmp.destroy();
  return rc;
}
