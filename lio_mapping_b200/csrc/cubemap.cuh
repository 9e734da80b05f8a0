// The device estimator's use of a publishing PointMapping's cube map after initialisation (lio_est_attach_map, estimator.cu):
// Estimator.cc:703-721 run UpdateMapDatabase and PublishResults of the PointMapping the estimator is.  The lio_pm handle stays
// opaque to estimator.cu; these are the only entries it uses (cubemap.cu).
#pragma once
#include <cuda_runtime.h>
#include "twistf.h"
#include "../../include/lio_b200.h"

// Checks the handle (a publishing PointMapping that has run a process call on `device`, not attached, leaves equal to the
// estimator's corner / surf filter sizes, max_full >= full_bound), grows its insert buffers to ins_bound points and marks it attached.
// LIO_ERR_INVALID / LIO_ERR_CAPACITY before anything changes.
int pm_attach(lio_pm *m, int device, float corner_leaf, float surf_leaf, int ins_bound, int full_bound);
void pm_detach(lio_pm *m);
cudaStream_t pm_stream(const lio_pm *m);
lio::TwistF *pm_tobe(lio_pm *m);       // transform_tobe_mapped_ (the estimator predicts it, Estimator.cc:776-809)
lio::TwistF pm_aft(const lio_pm *m);   // transform_aft_mapped_ (frozen after initialisation)
// One INITED scan's map work on the handle's stream, which the caller has ordered after the clouds' producers: when `insert`,
// UpdateMapDatabase of src (counts *n_dev clamped to bound) with `pose`, the frozen valid list and centre (:703-708); then
// PublishResults (:721) with the frozen surround list and the full cloud `full` (count *nf_dev, host value nf).
// info4 = {inserted, points inserted, surround published, size of the last surround map}.
int pm_est_step(lio_pm *m, bool insert, const float4 *const src[2], const int *const n_dev[2], const int bound[2], const lio::TwistF &pose,
                const float4 *full, const int *nf_dev, int nf, int info4[4]);
