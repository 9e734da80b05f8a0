// Device-wide primitives shared by the stage-B kernels: single-pass ordered compaction support
// (decoupled look-back exclusive prefix of one int per tile) and a stable LSD radix sort of
// (u32 key, u32 value) pairs.  Hand-written; no CUB/Thrust.
#pragma once
#include "common.cuh"

namespace lio {

// ---- decoupled look-back ----------------------------------------------------------------------
// status[t] = (flag << 32) | value, flag: 0 = not ready, 1 = tile aggregate, 2 = inclusive prefix.
// The caller zeroes status[0..ntiles) (and the ticket counter) before the launch, and obtains its
// tile id from an atomic ticket so that every earlier tile is already resident (forward progress).
constexpr unsigned long long kLbAgg = 1ull << 32, kLbPfx = 2ull << 32;

__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// All threads of the block call with the same (tile, aggregate).  Returns the exclusive prefix
// (sum of the aggregates of tiles 0..tile-1).  `sbcast` is one shared int.
__device__ __forceinline__ int lookback_exclusive(unsigned long long *status, int tile, int aggregate, int *sbcast) {
  if (warp_id() == 0) {
    const int lane = lane_id();
    if (tile == 0) {
      if (lane == 0) { st_relaxed_u64(status, kLbPfx | (unsigned)aggregate); *sbcast = 0; }
    } else {
      if (lane == 0) st_relaxed_u64(status + tile, kLbAgg | (unsigned)aggregate);
      int excl = 0;
      int t = tile - 1;
      while (true) {
        int idx = t - lane;
        unsigned long long s;
        do {
          s = (idx >= 0) ? ld_relaxed_u64(status + idx) : kLbPfx;
        } while (__any_sync(0xffffffffu, (s >> 32) == 0));
        unsigned pm = __ballot_sync(0xffffffffu, (s >> 32) == 2);
        int first = pm ? (__ffs(pm) - 1) : 31;
        int v = (lane <= first) ? (int)(unsigned)s : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        excl += v;
        if (pm) break;
        t -= 32;
      }
      if (lane == 0) { st_relaxed_u64(status + tile, kLbPfx | (unsigned)(excl + aggregate)); *sbcast = excl; }
    }
  }
  __syncthreads();
  int r = *sbcast;
  __syncthreads();
  return r;
}

// ---- stable LSD radix sort ---------------------------------------------------------------------
constexpr int kRsThreads = 256;
constexpr int kRsTile = 2048;  // keys per CTA
constexpr int kRsBits = 8;
constexpr int kRsBins = 1 << kRsBits;

struct RadixSortTemp {
  DevMem<unsigned> mem;      // init's allocation; empty when buf points into a caller's own scratch
  unsigned *buf = nullptr;   // digit histograms [4][256] | tickets [8] | look-back status [4][ntiles_max][256]
  size_t words = 0;
  int ntiles_max = 0;
  int init(int max_keys);
};

// Sorts n pairs by the low `key_bits` bits (rounded up to a multiple of 8).  n is read from the
// device (n_dev) so that data-dependent sizes need no host round trip; n_max bounds the grid.
// Result ends in (keys_a, vals_a) if the number of passes is even, else in (keys_b, vals_b):
// the function returns which (0 = a, 1 = b), or -1 when n_max exceeds the workspace.
int radix_sort_pairs(unsigned *keys_a, unsigned *vals_a, unsigned *keys_b, unsigned *vals_b, const int *n_dev, int n_max,
                     int key_bits, RadixSortTemp &tmp, cudaStream_t st, int *launches);

}  // namespace lio
