// Micro-benchmark: fp64 FMA rate (DFMA) vs fp64 tensor rate (DMMA m8n8k4) per SM on sm_90a (H100).
// Decides whether the 7x7 weighted rank-1 update of stage C / the Cholesky trailing update should use mma.sync f64.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o dmma_rate dmma_rate.cu && ./dmma_rate
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_dfma(double *out, int iters) {
  double a[8], b = 1.0000001, c = 1e-9;
#pragma unroll
  for (int k = 0; k < 8; ++k) a[k] = threadIdx.x * 1e-3 + k;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = fma(a[k], b, c);
  }
  double s = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) s += a[k];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

template <int NACC>
__global__ void k_dmma(double *out, int iters) {
  double d0[NACC], d1[NACC];
#pragma unroll
  for (int k = 0; k < NACC; ++k) { d0[k] = 0; d1[k] = 0; }
  double a = 1e-3 * threadIdx.x, b = 1.0 + 1e-6 * threadIdx.x;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < NACC; ++k) dmma(d0[k], d1[k], a, b);
  }
  double s = 0;
#pragma unroll
  for (int k = 0; k < NACC; ++k) s += d0[k] + d1[k];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <typename F> static float time_ms(F f) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  f();  // warm-up
  cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
  return ms;
}

int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  double *out; cudaMalloc(&out, sizeof(double) * sms * 8 * 1024);
  const int iters = 20000;
  for (int warps : {4, 8, 16, 32}) {
    const int threads = warps * 32, blocks = sms * 2;
    float ms = time_ms([&] { k_dfma<<<blocks, threads>>>(out, iters); });
    double fma_per_s = (double)blocks * threads * iters * 8 / (ms * 1e-3);
    printf("DFMA  warps/CTA %2d x2 CTA/SM: %.3f ms  %.2f TFMA/s  (%.1f FMA/clk/SM @1.98GHz)\n", warps, ms, fma_per_s / 1e12, fma_per_s / sms / 1.98e9);
    float ms1 = time_ms([&] { k_dmma<1><<<blocks, threads>>>(out, iters); });
    float ms4 = time_ms([&] { k_dmma<4><<<blocks, threads>>>(out, iters); });
    float ms8 = time_ms([&] { k_dmma<8><<<blocks, threads>>>(out, iters); });
    auto rate = [&](float m, int nacc) { return (double)blocks * warps * iters * nacc * 256.0 / (m * 1e-3); };
    printf("DMMA  warps/CTA %2d x2 CTA/SM: chain1 %.3f ms %.2f TFMA/s | 4 acc %.3f ms %.2f TFMA/s | 8 acc %.3f ms %.2f TFMA/s (%.1f FMA/clk/SM)\n", warps,
           ms1, rate(ms1, 1) / 1e12, ms4, rate(ms4, 4) / 1e12, ms8, rate(ms8, 8) / 1e12, rate(ms8, 8) / sms / 1.98e9);
  }
  // single-warp latency of a dependent DMMA / DFMA chain
  float l1 = time_ms([&] { k_dmma<1><<<1, 32>>>(out, iters); });
  float l2 = time_ms([&] { k_dfma<<<1, 32>>>(out, iters); });
  printf("latency: dependent DMMA %.1f ns/op, 8-way DFMA group %.1f ns (%.1f ns per FMA issue)\n", l1 * 1e6 / iters, l2 * 1e6 / iters, l2 * 1e6 / iters / 8);
  cudaFree(out);
  return 0;
}
