// Micro-benchmark: latency of the serial pieces of the tiled Cholesky's critical path on sm_90a (H100) (one warp, one SM):
// dependent DFMA / DMUL / SHFL / rsqrt / rcp / LDS chains and the 8x8 diagonal-tile factorisation variants.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o diag_tile diag_tile.cu && ./diag_tile
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ int swz(int r, int c) { return r * 8 + (c ^ ((r & 2) << 1)); }

__global__ void k_lat(double *out, long long *cyc, int iters) {
  __shared__ double sm[64];
  const int l = threadIdx.x;
  if (l < 64) sm[l] = 1.0 + 1e-3 * l;
  __syncthreads();
  double x = 1.0 + 1e-9 * l, b = 1.0000001, c = 1e-12;
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) x = fma(x, b, c);
  long long t1 = clock64();
  if (l == 0) cyc[0] = t1 - t0;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) x = x * b;
  t1 = clock64();
  if (l == 0) cyc[1] = t1 - t0;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) x = __shfl_sync(0xffffffffu, x, (l + 1) & 31);
  t1 = clock64();
  if (l == 0) cyc[2] = t1 - t0;
  x = fabs(x) + 1.0;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) x = rsqrt(x) + 1.0;
  t1 = clock64();
  if (l == 0) cyc[3] = t1 - t0;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) x = 1.0 / x + 1.0;
  t1 = clock64();
  if (l == 0) cyc[4] = t1 - t0;
  int idx = l & 63;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) { double v = sm[idx]; idx = ((int)v + idx + 1) & 63; }
  t1 = clock64();
  if (l == 0) cyc[5] = t1 - t0;
  t0 = clock64();
  for (int i = 0; i < iters; ++i) x = sqrt(x) + 1.0;
  t1 = clock64();
  if (l == 0) cyc[6] = t1 - t0;
  out[l] = x + idx;
}

// V0: the production variant (row per lane, shuffles), incl. the inverse
__device__ void diag_v0(double *T) {
  const int l = threadIdx.x & 31;
  double a[8], dinv[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) a[c] = (l < 8 && c <= l) ? T[swz(l & 7, c)] : 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double dk = __shfl_sync(0xffffffffu, a[k], k);
    const double inv = rsqrt(dk);
    dinv[k] = inv;
    const double lk = a[k] * inv;
    a[k] = lk;
#pragma unroll
    for (int j = k + 1; j < 8; ++j) a[j] -= lk * __shfl_sync(0xffffffffu, lk, j);
  }
  if (l < 8) {
#pragma unroll
    for (int c = 0; c < 8; ++c) if (c <= l) T[swz(l, c)] = a[c];
  }
  __syncwarp();
  double x[8], sacc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sacc[i] = (i == l) ? 1.0 : 0.0; x[i] = 0.0; }
  if (l < 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      x[k] = sacc[k] * dinv[k];
#pragma unroll
      for (int i = k + 1; i < 8; ++i) sacc[i] -= T[swz(i, k)] * x[k];
    }
  }
  __syncwarp();
  if (l < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) T[swz(i, l)] = x[i];
  }
  __syncwarp();
}

// V1: factor only (no inverse), to split the cost
__device__ void diag_v1(double *T) {
  const int l = threadIdx.x & 31;
  double a[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) a[c] = (l < 8 && c <= l) ? T[swz(l & 7, c)] : 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double dk = __shfl_sync(0xffffffffu, a[k], k);
    const double lk = a[k] * rsqrt(dk);
    a[k] = lk;
#pragma unroll
    for (int j = k + 1; j < 8; ++j) a[j] -= lk * __shfl_sync(0xffffffffu, lk, j);
  }
  if (l < 8) {
#pragma unroll
    for (int c = 0; c < 8; ++c) if (c <= l) T[swz(l, c)] = a[c];
  }
  __syncwarp();
}

// V2: single lane, everything in registers (factor + inverse), no shuffles
__device__ void diag_v2(double *T) {
  const int l = threadIdx.x & 31;
  if (l == 0) {
    double a[8][8], dinv[8];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c <= r; ++c) a[r][c] = T[swz(r, c)];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const double inv = rsqrt(a[k][k]);
      dinv[k] = inv;
      a[k][k] *= inv;
#pragma unroll
      for (int i = k + 1; i < 8; ++i) a[i][k] *= inv;
#pragma unroll
      for (int i = k + 1; i < 8; ++i)
#pragma unroll
        for (int j = k + 1; j <= i; ++j) a[i][j] -= a[i][k] * a[j][k];
    }
    // inverse, column by column, right looking
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      double s[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] = (i == c) ? 1.0 : 0.0;
#pragma unroll
      for (int k = c; k < 8; ++k) {
        const double xk = s[k] * dinv[k];
        T[swz(k, c)] = xk;
#pragma unroll
        for (int i = k + 1; i < 8; ++i) s[i] -= a[i][k] * xk;
      }
#pragma unroll
      for (int k = 0; k < c; ++k) T[swz(k, c)] = 0.0;
    }
  }
  __syncwarp();
}

// V3: LDL^T style with reciprocal pivots on the chain, square roots at the end (all in parallel), row per lane
__device__ void diag_v3(double *T) {
  const int l = threadIdx.x & 31;
  double a[8], rinv[8], piv[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) a[c] = (l < 8 && c <= l) ? T[swz(l & 7, c)] : 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double dk = __shfl_sync(0xffffffffu, a[k], k);
    piv[k] = dk;
    const double r = 1.0 / dk;
    rinv[k] = r;
    const double lk = a[k] * r;       // unit-lower entry l_ik (lane i > k)
#pragma unroll
    for (int j = k + 1; j < 8; ++j) a[j] -= lk * __shfl_sync(0xffffffffu, a[k], j);   // a_ij -= l_ik a_jk
    a[k] = lk;
  }
  // L = L_unit sqrt(D): column scaling with independent square roots
#pragma unroll
  for (int k = 0; k < 8; ++k) { const double sq = piv[k] * rsqrt(piv[k]); a[k] = (l == k) ? sq : a[k] * sq; }
  if (l < 8) {
#pragma unroll
    for (int c = 0; c < 8; ++c) if (c <= l) T[swz(l, c)] = a[c];
  }
  __syncwarp();
}

template <int V>
__global__ void k_diag(double *out, long long *cyc, int reps) {
  __shared__ double T[64], T0[64];
  const int l = threadIdx.x;
  for (int e = l; e < 64; e += 32) { const int r = e >> 3, c = e & 7; T0[swz(r, c)] = (r == c ? 9.0 : 0.0) + 0.3 / (1 + r + c); }
  __syncwarp();
  long long tot = 0;
  for (int it = 0; it < reps; ++it) {
    for (int e = l; e < 64; e += 32) T[e] = T0[e];
    __syncwarp();
    const long long t0 = clock64();
    if (V == 0) diag_v0(T);
    if (V == 1) diag_v1(T);
    if (V == 2) diag_v2(T);
    if (V == 3) diag_v3(T);
    tot += clock64() - t0;
  }
  if (l == 0) cyc[0] = tot / reps;
  for (int e = l; e < 64; e += 32) out[e] = T[e];
}

int main() {
  double *out; long long *cyc;
  cudaMalloc(&out, 1024 * 8); cudaMalloc(&cyc, 64 * 8);
  long long h[16];
  const int iters = 2000;
  k_lat<<<1, 32>>>(out, cyc, iters); k_lat<<<1, 32>>>(out, cyc, iters);
  cudaMemcpy(h, cyc, sizeof(long long) * 8, cudaMemcpyDeviceToHost);
  const char *nm[] = {"DFMA", "DMUL", "SHFL.f64", "rsqrt(+DADD)", "1/x(+DADD)", "LDS.64 dependent", "sqrt(+DADD)"};
  for (int k = 0; k < 7; ++k) printf("dependent %-18s %.1f cycles/op\n", nm[k], (double)h[k] / iters);
  const char *vn[] = {"V0 production: row/lane shuffles, factor + inverse", "V1 row/lane shuffles, factor only", "V2 single lane registers, factor + inverse",
                      "V3 LDL^T reciprocal chain, sqrt at the end, factor only"};
  double hv[4][64];
  for (int v = 0; v < 4; ++v) {
    if (v == 0) { k_diag<0><<<1, 32>>>(out, cyc, 50); k_diag<0><<<1, 32>>>(out, cyc, 50); }
    if (v == 1) { k_diag<1><<<1, 32>>>(out, cyc, 50); k_diag<1><<<1, 32>>>(out, cyc, 50); }
    if (v == 2) { k_diag<2><<<1, 32>>>(out, cyc, 50); k_diag<2><<<1, 32>>>(out, cyc, 50); }
    if (v == 3) { k_diag<3><<<1, 32>>>(out, cyc, 50); k_diag<3><<<1, 32>>>(out, cyc, 50); }
    cudaMemcpy(h, cyc, sizeof(long long), cudaMemcpyDeviceToHost);
    cudaMemcpy(hv[v], out, sizeof(double) * 64, cudaMemcpyDeviceToHost);
    printf("%-60s %lld cycles per 8x8 tile\n", vn[v], h[0]);
  }
  double d02 = 0, d13 = 0;
  for (int e = 0; e < 64; ++e) { d02 = fmax(d02, fabs(hv[0][e] - hv[2][e])); d13 = fmax(d13, fabs(hv[1][e] - hv[3][e])); }
  printf("max |V0 - V2| = %.3e   max |V1 - V3| (lower part incl. garbage above) = %.3e\n", d02, d13);
  cudaError_t e = cudaDeviceSynchronize();
  printf("%s\n", cudaGetErrorString(e));
  return 0;
}
