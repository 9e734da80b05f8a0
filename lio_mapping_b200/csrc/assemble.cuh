// Stage C — fused PivotPointPlane residual + Jacobian + J^T J / J^T r reduction (see assemble.cu).
#pragma once
#include "common.cuh"

namespace lio {

constexpr int kMaxOpt = 16;        // max frames carrying lidar factors (opt_window_size)
constexpr int kAsmStride = 32;     // doubles per frame in the output: 28 sym(7x7) + cost_sum + pad

struct AsmFrame {
  const float4 *pts;   // xyz = feature point (lidar frame i), w = score (unused)
  const float4 *coef;  // (w, b) of the plane in the pivot lidar frame
  int n;               // features of this frame
  int tile0;           // first tile index of this frame
};

constexpr int kMaxPeers = 8;
constexpr int kAsmRtStride = 12;  // per frame: R_lpi (9, row-major) then R_lpi^T P_lpi (3), in a DEVICE buffer

struct AsmParams {
  AsmFrame f[kMaxOpt];
  int nframes;
  int tile_feats;  // features per tile (multiple of the block size)
  int ntiles;
  int fold_chunks; // stages between folds of the per-thread (1 + r^2) product into the cost (set by asm_plan)
  const int *skip_flag;  // optional device flag: non-zero -> the launch returns at once (device solver already terminated)
  long long *stamps;     // optional trace area (3 x 16 words: counters, %globaltimer at the first CTA's entry, at the tail's exit)
  // Fused exchange over peer memory (multi-GPU, frames sharded by rank): the last CTA writes the S blocks of the frames
  // this rank owns into its own AND every peer's result buffer (P2P stores over NVLink), then publishes `epoch` in each
  // peer's flag slot with system-scope release.  npeers == 0: single-GPU behaviour (all rows written locally).
  unsigned owned_mask;              // bit f set: frame f is reduced by this rank
  int npeers, self;                 // ranks in the exchange (including this one), this rank's index
  unsigned epoch;                   // evaluation counter, identical on all ranks
  double *peer_out[kMaxPeers];      // result buffers (this rank's own at [self]), already offset to the epoch's parity
  unsigned *peer_flag[kMaxPeers];   // flag arrays (one slot per source rank)
};

struct AsmWork {
  DevMem<double> partial;     // [ntiles_max][kAsmStride]
  DevMem<double> out;         // [kMaxOpt][kAsmStride] device
  DevMem<unsigned> counter;
  int ntiles_max = 0;
  int init(int max_features_total);
};

// Test seam: stages between folds of the running (1 + r^2) product (default 1024 = 2048 features per thread).
void asm_set_fold_chunks(int chunks);
// Fills tile0 / ntiles / tile_feats of `p` from the per-frame counts (host side).
void asm_plan(AsmParams &p, int sm_count);
// Launches the fused kernel; results land in work.out (device), kAsmStride doubles per frame:
//   [0..27] upper triangle (row-major) of S = sum rho'(r^2) [g;r][g;r]^T,  [28] sum rho(r^2).
// Rt_dev: device buffer of nframes x kAsmRtStride doubles (written by the host shell or by the device solver).
int asm_launch(const AsmParams &p, const double *Rt_dev, AsmWork &work, cudaStream_t st, int *launches);
// CUDA-graph support (the device solver replays one captured graph per solve): is `node` a launch of the fused kernel, and
// re-parameterise such a node of an instantiated graph for this solve's feature counts / tile plan.
bool asm_is_graph_node(cudaGraphNode_t node);
int asm_graph_update(cudaGraphExec_t exec, cudaGraphNode_t node, const AsmParams &p, const double *Rt_dev, AsmWork &work);
// One-time per-device set-up (the dynamic shared memory opt-in); asm_launch does it lazily, graph capture wants it done before.
void asm_prepare();

}  // namespace lio
