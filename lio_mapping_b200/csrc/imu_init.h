// lio_mapping_b200 — Estimator::RunInitialization with ImuInitializer::Initialization, and ImuInitializer::EstimateExtrinsicRotation,
// on the host (imu_init.cc)
#pragma once
#include "factors_host.h"
#include "twistf.h"

namespace lio {

enum { kInitLowExcitation = 0, kInitGravityFailed = 1, kInitSuccess = 2, kInitNotFinite = -1 };

// One attempt on a full window of W + 1 frames (W >= 5): laser transforms tf[0..W] (transform_aft_mapped_ of each push), their
// pre-integrations pre[0..W] (repropagated in place), transform_lb_.  Bgs, Vs and R_WI are read and written, Ps / Rs / g_vec written.
// Returns kInitLowExcitation with nothing changed, else kInitGravityFailed / kInitSuccess with the side effects the reference has
// either way, or kInitNotFinite when a result is not finite.
int run_initialization(int W, const TwistF *tf, Preintegration *const *pre, const TwistF &tlb, double g_norm, const hm::V3 *Bas,
                       hm::V3 *Bgs, hm::V3 *Vs, hm::M3 &R_WI, hm::V3 *Ps, hm::M3 *Rs, hm::V3 &g_vec);

// EstimateExtrinsicRotation on the same window (W >= 1): laser transforms tf[0..W], pre-integrations pre[1..W] (read only), transform_lb_.
// tlb's rotation is overwritten whether or not the call succeeds, its position never.  sv = the singular values of the 4W x 4 system,
// descending.  Returns true iff sv[2] > 0.25.
bool estimate_extrinsic_rotation(int W, const TwistF *tf, Preintegration *const *pre, TwistF &tlb, double sv[4]);

}  // namespace lio
