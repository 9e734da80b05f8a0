// Stage C on sm_90a — one fused kernel per Gauss-Newton iteration evaluates every
// PivotPointPlaneFactor (reference: src/factor/PivotPointPlaneFactor.cc:43-137, residual blocks
// added at src/imu_processor/Estimator.cc:1831-1889 with CauchyLoss(1.0), :1664) and reduces their
// contribution to the normal equations.
//
// Algebra (DESIGN.md §stage C): with T_lpi = (R, P) the lidar pose of frame i in the pivot lidar
// frame, a = R^T w, g = [a ; p x a], r = a.(p + R^T P) + b, the factor's 1x18 Jacobian row over
// (pose_pivot, pose_i, extrinsic) is g^T M_i with a 6x18 matrix M_i that depends on the state only.
// Ceres' Cauchy corrector (rho'' < 0 => alpha = 0) scales residual and Jacobian by sqrt(rho'),
// rho' = 1/(1+r^2).  Hence per frame the lidar part of J^T J, J^T r is M_i^T S_i M_i with
//     S_i = sum_k rho'(r_k^2) [g_k; r_k][g_k; r_k]^T      (7x7 symmetric, 28 numbers)
// and the cost is 1/2 sum_k log(1 + r_k^2).  The kernel streams 32 B per feature (float4 point +
// float4 plane), does the arithmetic in fp64 (inputs are exact fp32 values), and reduces with warp
// shuffles -> shared memory -> per-tile partials; the last CTA to finish sums the partials of each
// frame in tile order, so the result is deterministic and needs no second launch.
#include "assemble.cuh"
#include <cstring>

namespace lio {

constexpr int kAsmThreads = 256;

__device__ __forceinline__ float4 ld_stream(const float4 *p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

// One feature: u = [a; p x a; r] with a = R^T w, r = a.(p + t) + b, and s = 1 + r^2.  Branch-free, so that the
// kAsmPerThread features a thread handles per stage interleave (the chain a -> r -> s -> 1/s is latency bound otherwise).
__device__ __forceinline__ void feature_terms(const double (&R)[9], const double (&t)[3], float4 pf, float4 cf, double (&u)[7], double &s) {
  const double px = pf.x, py = pf.y, pz = pf.z;
  const double wx = cf.x, wy = cf.y, wz = cf.z, b = cf.w;
  // a = R^T w
  u[0] = R[0] * wx + R[3] * wy + R[6] * wz;
  u[1] = R[1] * wx + R[4] * wy + R[7] * wz;
  u[2] = R[2] * wx + R[5] * wy + R[8] * wz;
  // p x a
  u[3] = py * u[2] - pz * u[1];
  u[4] = pz * u[0] - px * u[2];
  u[5] = px * u[1] - py * u[0];
  // r = a.(p + t) + b
  u[6] = u[0] * (px + t[0]) + u[1] * (py + t[1]) + u[2] * (pz + t[2]) + b;
  s = 1.0 + u[6] * u[6];
}

// acc[0..27] += rho' [g;r][g;r]^T (upper triangle, row-major), rho' = 1/s
__device__ __forceinline__ void accumulate_outer(double (&acc)[29], const double (&u)[7], double s) {
  const double c = 1.0 / s;
  int k = 0;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const double cu = c * u[i];
#pragma unroll
    for (int j = i; j < 7; ++j) acc[k++] += cu * u[j];
  }
}

// rho = log(1 + x) = log(s).  Residuals are centimetres, so x is almost always tiny: instead of one log per feature the
// thread keeps the running PRODUCT of s (one DMUL, no dependency chain) and takes a single log when it folds (sum of
// logs == log of the product; relative error <= n ulp on the product, i.e. <= n 2^-53 absolute on rho).  Large
// residuals go through log directly so the product stays far from overflow (< 1.0625^kAsmFold).
__device__ __forceinline__ void accumulate_rho(double (&acc)[29], double &prod, double s) {
  const bool big = s >= 1.0625;
  prod *= big ? 1.0 : s;
  if (big) acc[28] += log(s);
}

// ---- TMA (bulk async copy) staging ---------------------------------------------------------------
// The feature stream is staged through shared memory by the TMA unit: one elected thread arms an mbarrier
// with the byte count and issues two cp.async.bulk (point tile + plane tile, 16 B aligned, contiguous 1-D:
// no tensor map needed); all threads wait on the barrier phase, consume their float4s from shared memory and
// hand the stage back with a CTA barrier.  kAsmStages tiles are in flight per CTA.
constexpr int kAsmPerThread = 2;                       // independent features a thread consumes per stage (ILP)
constexpr int kAsmChunk = kAsmThreads * kAsmPerThread;  // features per stage
constexpr int kAsmFold = 2048;                          // features per thread between folds of the (1 + x) product
constexpr int kAsmStages = 4;

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
  unsigned done = 0;
  while (!done) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  }
}

__global__ void __launch_bounds__(kAsmThreads, 2)
asm_ppp(const AsmParams P, const double *__restrict__ Rt, double *__restrict__ partial, double *__restrict__ out,
        unsigned *__restrict__ counter) {
  extern __shared__ __align__(128) unsigned char asm_smem[];  // kAsmStages x (point tile | plane tile)
  float4 (*s_pts)[kAsmChunk] = reinterpret_cast<float4 (*)[kAsmChunk]>(asm_smem);
  float4 (*s_coef)[kAsmChunk] = reinterpret_cast<float4 (*)[kAsmChunk]>(asm_smem + sizeof(float4) * kAsmStages * kAsmChunk);
  __shared__ __align__(8) unsigned long long full_bar[kAsmStages];
  __shared__ double sred[kAsmThreads / 32][29];
  __shared__ bool is_last;
  if (P.skip_flag && *P.skip_flag) return;
  if (P.stamps && blockIdx.x == 0 && threadIdx.x == 0) {
    const long long i = P.stamps[1]++;
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (i < 16) P.stamps[16 + i] = t;
  }
  const int tile = blockIdx.x;
  int fi = 0;
#pragma unroll 1
  for (int k = 1; k < P.nframes; ++k) if (tile >= P.f[k].tile0) fi = k;
  const AsmFrame &F = P.f[fi];
  double R[9], t[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = __ldg(Rt + fi * kAsmRtStride + k);
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = __ldg(Rt + fi * kAsmRtStride + 9 + k);
  double acc[29];
#pragma unroll
  for (int k = 0; k < 29; ++k) acc[k] = 0.0;
  double prod = 1.0;
  const int begin = (tile - F.tile0) * P.tile_feats;
  const int end = min(begin + P.tile_feats, F.n);
  const int nchunks = (end > begin) ? (end - begin + kAsmChunk - 1) / kAsmChunk : 0;
  if (nchunks == 1) {
    // A tile of one chunk (every tile of a window solve: 512 features) gains nothing from the TMA ring - arming a barrier,
    // the bulk copy and the phase wait only add latency - so each thread fetches its two features directly (16 B streaming
    // loads, all four in flight) and computes from registers.
    double u[kAsmPerThread][7], sv[kAsmPerThread];
    float4 pf[kAsmPerThread], cf[kAsmPerThread];
#pragma unroll
    for (int j = 0; j < kAsmPerThread; ++j) {
      const int idx = begin + j * kAsmThreads + threadIdx.x;
      const bool ok = idx < end;
      pf[j] = ok ? ld_stream(F.pts + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
      cf[j] = ok ? ld_stream(F.coef + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int j = 0; j < kAsmPerThread; ++j) feature_terms(R, t, pf[j], cf[j], u[j], sv[j]);
#pragma unroll
    for (int j = 0; j < kAsmPerThread; ++j) accumulate_outer(acc, u[j], sv[j]);
#pragma unroll
    for (int j = 0; j < kAsmPerThread; ++j) accumulate_rho(acc, prod, sv[j]);
  } else {
    if (threadIdx.x == 0) {
  #pragma unroll
      for (int s = 0; s < kAsmStages; ++s) mbar_init(&full_bar[s], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](int k) {  // elected thread: arm the barrier, start both bulk copies of chunk k
      const int s = k % kAsmStages;
      const int c0 = begin + k * kAsmChunk;
      const unsigned bytes = (unsigned)(min(kAsmChunk, end - c0) * (int)sizeof(float4));
      mbar_expect_tx(&full_bar[s], 2u * bytes);
      tma_load_1d(&s_pts[s][0], F.pts + c0, bytes, &full_bar[s]);
      tma_load_1d(&s_coef[s][0], F.coef + c0, bytes, &full_bar[s]);
    };
    if (threadIdx.x == 0) for (int k = 0; k < min(kAsmStages, nchunks); ++k) issue(k);
    for (int k = 0; k < nchunks; ++k) {
      const int s = k % kAsmStages;
      mbar_wait(&full_bar[s], (unsigned)((k / kAsmStages) & 1));
      {
        double u[kAsmPerThread][7], sv[kAsmPerThread];
  #pragma unroll
        for (int j = 0; j < kAsmPerThread; ++j) {
          const int li = j * kAsmThreads + threadIdx.x;
          const bool ok = begin + k * kAsmChunk + li < end;   // past the end: all-zero feature (u = 0, s = 1) contributes nothing
          float4 pf = s_pts[s][li], cf = s_coef[s][li];
          if (!ok) { pf = make_float4(0.f, 0.f, 0.f, 0.f); cf = pf; }
          feature_terms(R, t, pf, cf, u[j], sv[j]);
        }
  #pragma unroll
        for (int j = 0; j < kAsmPerThread; ++j) accumulate_outer(acc, u[j], sv[j]);
  #pragma unroll
        for (int j = 0; j < kAsmPerThread; ++j) accumulate_rho(acc, prod, sv[j]);
      }
      if ((k + 1) % P.fold_chunks == 0) { acc[28] += log(prod); prod = 1.0; }
      __syncthreads();  // stage s fully consumed
      if (threadIdx.x == 0 && k + kAsmStages < nchunks) issue(k + kAsmStages);
    }
  }
  acc[28] += log(prod);
  // warp reduce-scatter: each level halves the values a lane owns (30 shuffles instead of 29 x 5)
  {
    const unsigned lane = lane_id();
    int c = 29;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int h = (c + 1) >> 1;
      const bool up = (lane & o) != 0;
#pragma unroll
      for (int i = 0; i < 15; ++i) {
        if (i < h) {
          const double a = acc[i];
          const double b = (i + h < c) ? acc[i + h] : 0.0;
          const double send = up ? a : b;
          const double keep = up ? b : a;
          acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
      }
      c = h;
    }
    // lane L now owns component idx = 15*b16 + 8*b8 + 4*b4 + 2*b2 + b1 (when it is a real component)
    const int idx = 15 * ((lane >> 4) & 1) + 8 * ((lane >> 3) & 1) + 4 * ((lane >> 2) & 1) + 2 * ((lane >> 1) & 1) + (lane & 1);
    const bool real = ((lane >> 4) & 1) ? ((lane & 15) < 14) : ((lane & 15) < 15);
    if (real) sred[warp_id()][idx] = acc[0];
  }
  __syncthreads();
  if (threadIdx.x < 29) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kAsmThreads / 32; ++w) v += sred[w][threadIdx.x];
    partial[(size_t)tile * kAsmStride + threadIdx.x] = v;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned prev = atomicAdd(counter, 1u);
    is_last = (prev == (unsigned)(P.ntiles - 1));
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // last CTA: one warp per frame, one lane per component, sums that frame's per-tile partials in tile order (four
  // interleaved accumulators, loads issued sixteen at a time so the L2 round trips overlap); deterministic, no second launch.
  for (int f = warp_id(); f < P.nframes; f += kAsmThreads / 32) {
    const int k = lane_id();
    if (k >= 29) continue;
    if (P.npeers > 0 && !((P.owned_mask >> f) & 1u)) continue;   // a peer reduces this frame and writes the row here
    const int t0 = P.f[f].tile0;
    const int t1 = (f + 1 < P.nframes) ? P.f[f + 1].tile0 : P.ntiles;
    double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0;
    int tt = t0;
#pragma unroll 4
    for (; tt + 3 < t1; tt += 4) {
      v0 += __ldcg(partial + (size_t)tt * kAsmStride + k);
      v1 += __ldcg(partial + (size_t)(tt + 1) * kAsmStride + k);
      v2 += __ldcg(partial + (size_t)(tt + 2) * kAsmStride + k);
      v3 += __ldcg(partial + (size_t)(tt + 3) * kAsmStride + k);
    }
    for (; tt < t1; ++tt) v0 += __ldcg(partial + (size_t)tt * kAsmStride + k);
    const double v = (v0 + v1) + (v2 + v3);
    if (P.npeers > 0) {
#pragma unroll 1
      for (int pr = 0; pr < P.npeers; ++pr) P.peer_out[pr][f * kAsmStride + k] = v;   // own buffer included
    } else {
      out[f * kAsmStride + k] = v;
    }
  }
  if (P.npeers > 0) {
    __threadfence_system();   // rows visible system-wide before the flags
    __syncthreads();
    if (threadIdx.x < (unsigned)P.npeers) {
      unsigned *fl = P.peer_flag[threadIdx.x] + P.self;
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(fl), "r"(P.epoch) : "memory");
    }
  }
  if (threadIdx.x == 0) {
    *counter = 0u;
    if (P.stamps) {
      const long long i = P.stamps[0]++;
      long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (i < 16) P.stamps[32 + i] = t;
    }
  }
}

int AsmWork::init(int max_features_total) {
  ntiles_max = max_features_total / kAsmThreads + 2 * kMaxOpt + 16;
  if (cudaMalloc(&partial, sizeof(double) * (size_t)ntiles_max * kAsmStride) != cudaSuccess) return -1;
  if (cudaMalloc(&out, sizeof(double) * kMaxOpt * kAsmStride) != cudaSuccess) return -1;
  if (cudaMalloc(&counter, sizeof(unsigned)) != cudaSuccess) return -1;
  cudaMemset(counter, 0, sizeof(unsigned));
  return 0;
}
void AsmWork::destroy() {
  if (partial) cudaFree(partial);
  if (out) cudaFree(out);
  if (counter) cudaFree(counter);
  partial = out = nullptr; counter = nullptr;
}

static int g_fold_chunks = kAsmFold / kAsmPerThread;
void asm_set_fold_chunks(int chunks) { g_fold_chunks = chunks < 1 ? 1 : chunks; }

void asm_plan(AsmParams &p, int sm_count) {
  p.fold_chunks = g_fold_chunks;   // (the exchange fields are set by the caller; zero-initialised params mean single GPU)
  long long total = 0;
  for (int k = 0; k < p.nframes; ++k) total += p.f[k].n;
  // aim at ~4 tiles per SM, at least 2 loads per thread, tile a multiple of the block size
  long long per = (total + (long long)sm_count * 4 - 1) / ((long long)sm_count * 4);
  int tf = (int)((per + kAsmThreads - 1) / kAsmThreads) * kAsmThreads;
  if (tf < 2 * kAsmThreads) tf = 2 * kAsmThreads;
  p.tile_feats = tf;
  int t = 0;
  for (int k = 0; k < p.nframes; ++k) {
    p.f[k].tile0 = t;
    int nt = (p.f[k].n + tf - 1) / tf;
    if (nt < 1) nt = 1;  // every frame owns at least one (possibly empty) tile
    t += nt;
  }
  p.ntiles = t;
}

constexpr size_t kAsmSmem = 2 * sizeof(float4) * kAsmStages * kAsmChunk;

void asm_prepare() {
  static bool attr_set[64] = {};  // per device: the opt-in above 48 KB is a per-context function attribute
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63]) {
    cudaFuncSetAttribute(asm_ppp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAsmSmem);
    attr_set[dev & 63] = true;
  }
}

bool asm_is_graph_node(cudaGraphNode_t node) {
  cudaGraphNodeType ty;
  if (cudaGraphNodeGetType(node, &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel) return false;
  cudaKernelNodeParams kp;
  if (cudaGraphKernelNodeGetParams(node, &kp) != cudaSuccess) return false;
  return kp.func == reinterpret_cast<void *>(asm_ppp);
}

int asm_graph_update(cudaGraphExec_t exec, cudaGraphNode_t node, const AsmParams &p, const double *Rt_dev, AsmWork &work) {
  if (p.ntiles > work.ntiles_max) return LIO_ERR_CAPACITY;
  AsmParams pc = p;
  const double *rt = Rt_dev;
  double *partial = work.partial, *out = work.out;
  unsigned *counter = work.counter;
  void *args[] = {&pc, &rt, &partial, &out, &counter};
  cudaKernelNodeParams kp;
  std::memset(&kp, 0, sizeof(kp));
  kp.func = reinterpret_cast<void *>(asm_ppp);
  kp.gridDim = dim3((unsigned)(p.ntiles > 0 ? p.ntiles : 1));
  kp.blockDim = dim3(kAsmThreads);
  kp.sharedMemBytes = (unsigned)kAsmSmem;
  kp.kernelParams = args;
  kp.extra = nullptr;
  cudaError_t e = cudaGraphExecKernelNodeSetParams(exec, node, &kp);
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

int asm_launch(const AsmParams &p, const double *Rt_dev, AsmWork &work, cudaStream_t st, int *launches) {
  if (p.ntiles > work.ntiles_max) return LIO_ERR_CAPACITY;
  if (p.nframes <= 0) return LIO_OK;
  constexpr size_t kSmem = kAsmSmem;
  asm_prepare();
  asm_ppp<<<p.ntiles, kAsmThreads, kSmem, st>>>(p, Rt_dev, work.partial, work.out, work.counter);
  if (launches) *launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

// ---- per-factor evaluation on the device (parity entry for the ceres::CostFunction seam) -------
__global__ void ppp_rows(const float4 *__restrict__ pts, const float4 *__restrict__ coef, int n, const double *__restrict__ Rt12,
                         const double *__restrict__ M /*6x18*/, double *__restrict__ r_out, double *__restrict__ J_out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 pf = pts[i], cf = coef[i];
  const double px = pf.x, py = pf.y, pz = pf.z, wx = cf.x, wy = cf.y, wz = cf.z;
  double g[6];
  g[0] = Rt12[0] * wx + Rt12[3] * wy + Rt12[6] * wz;
  g[1] = Rt12[1] * wx + Rt12[4] * wy + Rt12[7] * wz;
  g[2] = Rt12[2] * wx + Rt12[5] * wy + Rt12[8] * wz;
  g[3] = py * g[2] - pz * g[1];
  g[4] = pz * g[0] - px * g[2];
  g[5] = px * g[1] - py * g[0];
  r_out[i] = g[0] * (px + Rt12[9]) + g[1] * (py + Rt12[10]) + g[2] * (pz + Rt12[11]) + (double)cf.w;
  for (int c = 0; c < 18; ++c) {
    double s = 0;
    for (int k = 0; k < 6; ++k) s += g[k] * M[k * 18 + c];
    J_out[(size_t)i * 18 + c] = s;
  }
}

int ppp_rows_launch(const float4 *pts, const float4 *coef, int n, const double *Rt12_dev, const double *M_dev, double *r_out,
                    double *J_out, cudaStream_t st) {
  if (n <= 0) return LIO_OK;
  ppp_rows<<<(n + 127) / 128, 128, 0, st>>>(pts, coef, n, Rt12_dev, M_dev, r_out, J_out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return LIO_ERR_CUDA; }
  return LIO_OK;
}

}  // namespace lio
