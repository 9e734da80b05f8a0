// lio_mapping_b200 — shared device/host helpers for the sm_90a kernels behind the C-ABI.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <type_traits>
#include <vector>
#include "../../include/lio_b200.h"
#include "own.cuh"

#define LIO_CUDA_OK(expr)                                                                   \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(_e));                       \
      return LIO_ERR_CUDA;                                                                  \
    }                                                                                       \
  } while (0)

void lio_set_last_error(const char *file, int line, const char *msg);

// Returns the status of expr when it is not LIO_OK.
#define LIO_TRY(expr)                                                                       \
  do {                                                                                      \
    const int _rc = (expr);                                                                 \
    if (_rc != LIO_OK) return _rc;                                                          \
  } while (0)

// The first statement of every handle entry.  LIO_ENTER serves the entries that enqueue work on, copy from or wait for the
// handle's device: it makes that device current and leaves it so.  LIO_ENTER_HOST serves the entries that only touch host
// state, which leave the current device alone.  Both refuse a null handle with LIO_ERR_INVALID and text naming the entry.
#define LIO_ENTER(h) LIO_TRY(lio::enter(h, __func__, true))
#define LIO_ENTER_HOST(h) LIO_TRY(lio::enter(h, __func__, false))

namespace lio {

int refuse_null_handle(const char *entry);

template <class H> int enter(const H *h, const char *entry, bool on_device) {
  if (!h) return refuse_null_handle(entry);
  if (on_device) LIO_CUDA_OK(cudaSetDevice(h->device));
  return LIO_OK;
}

// The prologue of the create entries and the stateless host-array entries: LIO_ERR_NO_DEVICE without a device, else `device`
// made current and its SM count in *sms (when given).
int select_device(int device, int *sms = nullptr);

// Reads the n elements at src back to dst on stream s and waits for the stream.  *count (when given) receives n first; then
// n > cap returns LIO_ERR_CAPACITY and a null dst with n > 0 LIO_ERR_INVALID, both before anything is copied.
template <class T>
int read_back(T *dst, const typename std::common_type<T>::type *src, long long n, long long cap, cudaStream_t s, int *count = nullptr) {
  if (count) *count = (int)n;
  if (n > cap) return LIO_ERR_CAPACITY;
  if (n > 0) {
    if (!dst) return LIO_ERR_INVALID;
    LIO_CUDA_OK(cudaMemcpyAsync(dst, src, sizeof(T) * n, cudaMemcpyDeviceToHost, s));
  }
  LIO_CUDA_OK(cudaStreamSynchronize(s));
  return LIO_OK;
}

// Device buffers of a host-array entry, freed when the entry returns.  alloc / up / down / ok set lio_last_error and return
// false on failure, so an entry stops at the first failed allocation, copy or CUDA call.
struct DevBufs {
  std::vector<DevMem<void>> p;
  template <class T> bool alloc(T **out, size_t n) {
    DevMem<T> q;
    if (!lio::alloc(q, n)) return false;
    *out = q;
    p.push_back(std::move(q));
    return true;
  }
  // n elements of T; n == 0 copies nothing and leaves the pointers untouched.  T comes from the host side, so the device side
  // may be an owner.
  template <class T> struct Dev { using type = T; };
  template <class T> static bool up(typename Dev<T>::type *dst, const T *src, size_t n) {
    if (n == 0 || cudaMemcpy(dst, src, sizeof(T) * n, cudaMemcpyHostToDevice) == cudaSuccess) return true;
    lio_set_last_error(__FILE__, __LINE__, "upload failed");
    return false;
  }
  template <class T> static bool down(T *dst, const typename Dev<T>::type *src, size_t n) {
    return n == 0 || ok(cudaMemcpy(dst, src, sizeof(T) * n, cudaMemcpyDeviceToHost));
  }
  static bool ok(cudaError_t e) {
    if (e != cudaSuccess) lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
    return e == cudaSuccess;
  }
};

constexpr int kWarp = 32;

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ unsigned warp_id() { return threadIdx.x >> 5; }

// Inclusive warp scan (int).
__device__ __forceinline__ int warp_scan_incl(int v) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if ((int)lane_id() >= o) v += t;
  }
  return v;
}

// Block-wide exclusive scan for blockDim.x <= 1024; `smem` needs 33 ints.  Returns the exclusive
// prefix of v; *total receives the block sum.  All threads must call.
__device__ __forceinline__ int block_scan_excl(int v, int *smem, int *total) {
  int incl = warp_scan_incl(v);
  if (lane_id() == 31) smem[warp_id()] = incl;
  __syncthreads();
  if (warp_id() == 0) {
    int nw = (blockDim.x + 31) >> 5;
    int w = (int)lane_id() < nw ? smem[lane_id()] : 0;
    int wi = warp_scan_incl(w);
    smem[lane_id()] = wi - w;
    if ((int)lane_id() == nw - 1) smem[32] = wi;
  }
  __syncthreads();
  int r = smem[warp_id()] + incl - v;
  *total = smem[32];
  __syncthreads();
  return r;
}

__device__ __forceinline__ float4 ld_f4(const float4 *p) { return __ldg(p); }

}  // namespace lio
