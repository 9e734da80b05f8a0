// C-ABI seams of the window solve's lidar factor on explicit host arrays: the point-to-plane factor (one point, and a batch on the
// device), one frame of the fused stage-C reduction, its fold setting and its streaming-rate benchmark.
#include <algorithm>
#include <cmath>
#include <cstring>
#include "assemble.cuh"
#include "factors_host.h"

using namespace lio;

// ---- factor-operator seam ---------------------------------------------------------------------------
extern "C" int lio_ppp_evaluate(const double point[3], const double coeff[4], const double pose_pivot[7], const double pose_i[7],
                                const double pose_ex[7], double *residual, double *J0, double *J1, double *J2) {
  if (!point || !coeff || !pose_pivot || !pose_i || !pose_ex || !residual) return LIO_ERR_INVALID;
  ppp_evaluate_single(point, coeff, pose_pivot, pose_i, pose_ex, residual, J0, J1, J2);
  return LIO_OK;
}

namespace lio {
int ppp_rows_launch(const float4 *pts, const float4 *coef, int n, const double *Rt12_dev, const double *M_dev, double *r_out,
                    double *J_out, cudaStream_t st);
}

extern "C" int lio_ppp_evaluate_batch_host(const float *pts4, const float *coef4, int n, const double pose_pivot[7],
                                           const double pose_i[7], const double pose_ex[7], double *r_out, double *J_out, int device) {
  if (!pts4 || !coef4 || n < 0 || !pose_pivot || !pose_i || !pose_ex || !r_out || !J_out) return LIO_ERR_INVALID;
  LIO_TRY(select_device(device));
  if (n == 0) return LIO_OK;
  double Rt[12], M[108];
  ppp_frame_terms(pose_pivot, pose_i, pose_ex, Rt, Rt + 9, M);
  DevBufs d;
  float4 *dp = nullptr, *dc = nullptr;
  double *dRt = nullptr, *dM = nullptr, *dr = nullptr, *dJ = nullptr;
  if (!d.alloc(&dp, n) || !d.alloc(&dc, n) || !d.alloc(&dRt, 12) || !d.alloc(&dM, 108) || !d.alloc(&dr, n) || !d.alloc(&dJ, 18 * (size_t)n) ||
      !d.up(dp, (const float4 *)pts4, n) || !d.up(dc, (const float4 *)coef4, n) || !d.up(dRt, Rt, 12) || !d.up(dM, M, 108))
    return LIO_ERR_CUDA;
  const int rc = ppp_rows_launch(dp, dc, n, dRt, dM, dr, dJ, 0);
  if (rc != LIO_OK) return rc;
  return d.down(r_out, dr, n) && d.down(J_out, dJ, 18 * (size_t)n) ? LIO_OK : LIO_ERR_CUDA;
}

// Stage C reduction of ONE frame on explicit host arrays (parity entry for the fused kernel):
// out32[0..27] = upper triangle of S = sum rho'(r^2) [g;r][g;r]^T, out32[28] = sum log(1+r^2).
extern "C" int lio_asm_ppp_host(const float *pts4, const float *coef4, int n, const double R9[9], const double t3[3],
                                double out32[32], int device) {
  if (!pts4 || !coef4 || n < 0 || !R9 || !t3 || !out32) return LIO_ERR_INVALID;
  int sms = 132;
  LIO_TRY(select_device(device, &sms));
  DevBufs d;
  AsmWork w;
  float4 *dp = nullptr, *dc = nullptr;
  double *dRt = nullptr;
  double Rt[kAsmRtStride] = {};
  std::memcpy(Rt, R9, sizeof(double) * 9); std::memcpy(Rt + 9, t3, sizeof(double) * 3);
  int rc = LIO_OK;
  const int nn = n > 0 ? n : 1;
  if (w.init(nn) != 0) { lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed"); rc = LIO_ERR_CUDA; }
  else if (!d.alloc(&dp, nn) || !d.alloc(&dc, nn) || !d.alloc(&dRt, kAsmRtStride) || !d.up(dp, (const float4 *)pts4, n) ||
           !d.up(dc, (const float4 *)coef4, n) || !d.up(dRt, Rt, kAsmRtStride))
    rc = LIO_ERR_CUDA;
  if (rc == LIO_OK) {
    AsmParams ap;
    std::memset(&ap, 0, sizeof(ap));
    ap.nframes = 1;
    ap.f[0].pts = dp; ap.f[0].coef = dc; ap.f[0].n = n;
    asm_plan(ap, sms);
    rc = asm_launch(ap, dRt, w, 0, nullptr);
    if (rc == LIO_OK && (!d.ok(cudaDeviceSynchronize()) || !d.down(out32, w.out, kAsmStride))) rc = LIO_ERR_CUDA;
  }
  return rc;
}

// Synthetic feature stream shaped like a converged window: points within +-20 m, unit normals scaled by a score of 0.8,
// and plane offsets chosen so that the residual under the frame's (R, t) of the benchmark is a few centimetres
// (|r| <= 0.04 m), i.e. the regime the solver runs in (rho = log(1 + r^2) with r^2 << 1).
__global__ void k_fill_features(float4 *pts, float4 *coef, long long n, long long per_frame) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned h = (unsigned)(i * 2654435761u);
  float a = (float)(h & 1023) * (1.0f / 1024.0f), b = (float)((h >> 10) & 1023) * (1.0f / 1024.0f), c = (float)((h >> 20) & 1023) * (1.0f / 1024.0f);
  const float px = 40.f * (a - 0.5f), py = 40.f * (b - 0.5f), pz = 4.f * c;
  pts[i] = make_float4(px, py, pz, 0.9f);
  float nx = a - 0.5f, ny = b - 0.5f, nz = c + 0.1f, nn = rsqrtf(nx * nx + ny * ny + nz * nz);
  const float wx = 0.8f * nx * nn, wy = 0.8f * ny * nn, wz = 0.8f * nz * nn;
  // same (R, t) as lio_asm_stream_bench builds for frame k: R = Rz(0.01 k) stored row-major, t = (0.1 k, 0.02 k, 0)
  const int k = (int)(i / per_frame);
  const double cs = cos(0.01 * k), sn = sin(0.01 * k);
  const double ax = cs * wx + sn * wy, ay = -sn * wx + cs * wy, az = wz;   // a = R^T w
  const double r0 = ax * (px + 0.1 * k) + ay * (py + 0.02 * k) + az * pz;
  coef[i] = make_float4(wx, wy, wz, (float)(-r0) + 0.08f * (a - 0.5f));
}

extern "C" int lio_asm_set_fold_chunks(int chunks) {
  asm_set_fold_chunks(chunks);
  return LIO_OK;
}

// Streaming-rate measurement of the fused stage-C kernel on a synthetic feature stream of n features
// (choose n*32 B larger than L2 to measure the HBM-resident rate).  CUDA events around each launch on the
// launching stream.  out = {avg ms per launch, min ms, bytes per launch, launches}.
extern "C" int lio_asm_stream_bench(long long n_features, int iters, int device, double out[4]) {
  if (n_features <= 0 || iters <= 0 || !out) return LIO_ERR_INVALID;
  int sms = 132;
  LIO_TRY(select_device(device, &sms));
  const int O = 8;  // spread over 8 equal frames like a window
  const long long per = n_features / O;
  if (per <= 0 || per > 0x7fffffffLL) return LIO_ERR_INVALID;
  DevBufs d;
  float4 *dp = nullptr, *dc = nullptr;
  double *dRt = nullptr;
  AsmWork w;
  Event e0, e1;
  AsmParams ap;
  std::memset(&ap, 0, sizeof(ap));
  ap.nframes = O;
  double hRt[8 * kAsmRtStride];
  int rc = LIO_OK;
  if (!d.alloc(&dp, per * O) || !d.alloc(&dc, per * O)) rc = LIO_ERR_CUDA;
  else if (w.init((int)std::min<long long>(per * O, 1ll << 30)) != 0) { lio_set_last_error(__FILE__, __LINE__, "cudaMalloc failed"); rc = LIO_ERR_CUDA; }
  if (rc == LIO_OK) {
    k_fill_features<<<(unsigned)((per * O + 255) / 256), 256>>>(dp, dc, per * O, per);
    for (int k = 0; k < O; ++k) {
      ap.f[k].pts = dp + per * k; ap.f[k].coef = dc + per * k; ap.f[k].n = (int)per;
      const double c = std::cos(0.01 * k), s = std::sin(0.01 * k);
      const double Rt[kAsmRtStride] = {c, -s, 0, s, c, 0, 0, 0, 1, 0.1 * k, 0.02 * k, 0.0};
      std::memcpy(hRt + k * kAsmRtStride, Rt, sizeof(Rt));
    }
    if (!create(e0, cudaEventDefault) || !create(e1, cudaEventDefault) || !d.alloc(&dRt, 8 * kAsmRtStride) || !d.up(dRt, hRt, 8 * kAsmRtStride))
      rc = LIO_ERR_CUDA;
  }
  if (rc == LIO_OK) {
    asm_plan(ap, sms);
    double sum = 0, mn = 1e30;
    for (int it = 0; it < iters + 3 && rc == LIO_OK; ++it) {
      cudaEventRecord(e0, 0);
      rc = asm_launch(ap, dRt, w, 0, nullptr);
      cudaEventRecord(e1, 0);
      if (cudaEventSynchronize(e1) != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, "kernel failed"); rc = LIO_ERR_CUDA; break; }
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      if (it >= 3) { sum += ms; mn = std::min(mn, (double)ms); }
    }
    out[0] = sum / iters; out[1] = mn; out[2] = 32.0 * (double)(per * O); out[3] = iters;
  }
  return rc;
}
