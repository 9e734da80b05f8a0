// Column-pivoted Householder QR least squares for small fixed sizes, register resident.
// Restates Eigen 3.3 ColPivHouseholderQR::compute + solve (reference call sites
// src/imu_processor/Estimator.cc:1027 (5x3 plane fit) and :1306 (6x6 Gauss-Newton step)) in the same
// operation order as the CPU path; compile the including unit with -fmad=false.
#pragma once
#include <cfloat>
#include <cuda_runtime.h>

namespace lio {

template <int R, int C>
__device__ __forceinline__ void colpiv_qr_solve(float (&a)[R][C], float (&b)[R], float (&x)[C]) {
  constexpr int size = (R < C) ? R : C;
  float hCoeffs[size];
  int transp[size];
  float normsUpdated[C], normsDirect[C];
#pragma unroll
  for (int k = 0; k < C; ++k) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < R; ++i) s += a[i][k] * a[i][k];
    normsDirect[k] = sqrtf(s);
    normsUpdated[k] = normsDirect[k];
  }
  float maxn = normsUpdated[0];
#pragma unroll
  for (int k = 1; k < C; ++k) if (normsUpdated[k] > maxn) maxn = normsUpdated[k];
  const float eps = FLT_EPSILON;
  float th = maxn * eps;
  const float threshold_helper = (th * th) / (float)R;
  const float norm_downdate_threshold = sqrtf(eps);
  int nonzero_pivots = size;
#pragma unroll
  for (int k = 0; k < size; ++k) {
    int biggest = k;
    float bn = normsUpdated[k];
#pragma unroll
    for (int j = k + 1; j < C; ++j) if (normsUpdated[j] > bn) { bn = normsUpdated[j]; biggest = j; }
    float biggest_sq = bn * bn;
    if (nonzero_pivots == size && biggest_sq < threshold_helper * (float)(R - k)) nonzero_pivots = k;
    transp[k] = biggest;
#pragma unroll
    for (int j = k + 1; j < C; ++j) {
      if (j == biggest) {
#pragma unroll
        for (int i = 0; i < R; ++i) { float t = a[i][k]; a[i][k] = a[i][j]; a[i][j] = t; }
        float t = normsUpdated[k]; normsUpdated[k] = normsUpdated[j]; normsUpdated[j] = t;
        t = normsDirect[k]; normsDirect[k] = normsDirect[j]; normsDirect[j] = t;
      }
    }
    float tailSqNorm = 0.f;
#pragma unroll
    for (int i = k + 1; i < R; ++i) tailSqNorm += a[i][k] * a[i][k];
    float c0 = a[k][k];
    float tau, beta;
    if (R - k == 1 || tailSqNorm <= FLT_MIN) {
      tau = 0.f; beta = c0;
#pragma unroll
      for (int i = k + 1; i < R; ++i) a[i][k] = 0.f;
    } else {
      beta = sqrtf(c0 * c0 + tailSqNorm);
      if (c0 >= 0.f) beta = -beta;
      float den = c0 - beta;
#pragma unroll
      for (int i = k + 1; i < R; ++i) a[i][k] = a[i][k] / den;
      tau = (beta - c0) / beta;
    }
    hCoeffs[k] = tau;
    a[k][k] = beta;
    if (R - k == 1) {
#pragma unroll
      for (int j = k + 1; j < C; ++j) a[k][j] *= (1.f - tau);
    } else if (tau != 0.f) {
#pragma unroll
      for (int j = k + 1; j < C; ++j) {
        float tmp = 0.f;
#pragma unroll
        for (int i = k + 1; i < R; ++i) tmp += a[i][k] * a[i][j];
        tmp += a[k][j];
        a[k][j] -= tau * tmp;
#pragma unroll
        for (int i = k + 1; i < R; ++i) a[i][j] -= tau * a[i][k] * tmp;
      }
    }
#pragma unroll
    for (int j = k + 1; j < C; ++j) {
      if (normsUpdated[j] != 0.f) {
        float temp = fabsf(a[k][j]) / normsUpdated[j];
        temp = (1.f + temp) * (1.f - temp);
        temp = temp < 0.f ? 0.f : temp;
        float ratio = normsUpdated[j] / normsDirect[j];
        float temp2 = temp * (ratio * ratio);
        if (temp2 <= norm_downdate_threshold) {
          float s = 0.f;
#pragma unroll
          for (int i = k + 1; i < R; ++i) s += a[i][j] * a[i][j];
          normsDirect[j] = sqrtf(s);
          normsUpdated[j] = normsDirect[j];
        } else {
          normsUpdated[j] *= sqrtf(temp);
        }
      }
    }
  }
  int perm[C];
#pragma unroll
  for (int k = 0; k < C; ++k) perm[k] = k;
#pragma unroll
  for (int k = 0; k < size; ++k) {
#pragma unroll
    for (int j = k + 1; j < C; ++j) if (j == transp[k]) { int t = perm[k]; perm[k] = perm[j]; perm[j] = t; }
  }
#pragma unroll
  for (int k = 0; k < size; ++k) {
    if (k < nonzero_pivots) {
      float tau = hCoeffs[k];
      if (R - k == 1) { b[k] *= (1.f - tau); }
      else if (tau != 0.f) {
        float tmp = 0.f;
#pragma unroll
        for (int i = k + 1; i < R; ++i) tmp += a[i][k] * b[i];
        tmp += b[k];
        b[k] -= tau * tmp;
#pragma unroll
        for (int i = k + 1; i < R; ++i) b[i] -= tau * a[i][k] * tmp;
      }
    }
  }
#pragma unroll
  for (int i = size - 1; i >= 0; --i) {
    if (i < nonzero_pivots) {
      float s = b[i];
#pragma unroll
      for (int j = i + 1; j < size; ++j) if (j < nonzero_pivots) s -= a[i][j] * b[j];
      // Eigen's triangular solve divides only a nonzero right-hand side: a zero pivot under a zero rhs leaves 0, not 0 / 0
      b[i] = (s != 0.f) ? s / a[i][i] : s;
    }
  }
#pragma unroll
  for (int k = 0; k < C; ++k) x[k] = 0.f;
#pragma unroll
  for (int i = 0; i < size; ++i) {
    if (i < nonzero_pivots) {
#pragma unroll
      for (int j = 0; j < C; ++j) if (perm[i] == j) x[j] = b[i];
    }
  }
}


}  // namespace lio
