// The device estimator's use of a publishing PointMapping's cube map after initialisation (lio_est_attach_map, est_map.cu):
// Estimator.cc:703-721 run UpdateMapDatabase and PublishResults of the PointMapping the estimator is.  The lio_pm handle stays
// opaque to the estimator; these are the only entries it uses (cubemap.cu).
#pragma once
#include <cuda_runtime.h>
#include <vector>
#include "twistf.h"
#include "../../include/lio_b200.h"

// Checks the handle (a publishing PointMapping on `device`, not attached, leaves equal to the estimator's corner / surf filter sizes,
// max_full >= full_bound; fresh == true: no process call yet (lio_est_attach_mapping), false: at least one (lio_est_attach_map)),
// grows its insert buffers to ins_bound points and marks it attached.  LIO_ERR_INVALID / LIO_ERR_CAPACITY before anything changes.
int pm_attach(lio_pm *m, int device, float corner_leaf, float surf_leaf, int ins_bound, int full_bound, bool fresh);
void pm_detach(lio_pm *m);
cudaStream_t pm_stream(const lio_pm *m);
lio::TwistF *pm_tobe(lio_pm *m);       // transform_tobe_mapped_ (the estimator predicts it, Estimator.cc:776-809)
lio::TwistF pm_aft(const lio_pm *m);   // transform_aft_mapped_ (frozen after initialisation with imu_factor = 1)
// One INITED scan's map work on the handle's stream, which the caller has ordered after the clouds' producers: when `insert`,
// UpdateMapDatabase of src (counts *n_dev clamped to bound) with `pose`, the valid list and its margin centre (:703-708; NULL: the
// handle's last list and current centre, frozen with imu_factor = 1); then PublishResults (:721) with the last surround list and
// the full cloud `full` (count *nf_dev, host value nf).  info4 = {inserted, points inserted, surround published, last surround size}.
int pm_est_step(lio_pm *m, bool insert, const float4 *const src[2], const int *const n_dev[2], const int bound[2], const lio::TwistF &pose,
                const std::vector<size_t> *valid, const int *margin_centre, const float4 *full, const int *nf_dev, int nf, int info4[4]);

// ---- imu_factor = 0 (lio_est_attach_mapping): the estimator runs PointMapping::Process itself on every message (Estimator.cc:810-812)
// The host entry's upload into the handle's own input buffers (corner, surf, full; counts at *n3_dev), capacities checked first.
int pm_est_upload(lio_pm *m, const float *corner, int nc, const float *surf, int ns, const float *full, int nf, const float4 *src[3],
                  const int **n3_dev);
// lio_pm_process_dev on an attached handle: n3_max already capped by the caller (pm_est_caps).  While imu-inited (SetInitFlag,
// Estimator.cc:544) Process skips UpdateMapDatabase and PublishResults (PointMapping.cc:1033); the association of the odometry
// increment is the same TransformAssociateToMap that ProcessCompactData runs instead (:804).
int pm_est_process(lio_pm *m, const float4 *const src[2], const float4 *full, const int *n3_dev, const int n_max[3], const float sum7[7]);
void pm_est_caps(const lio_pm *m, const int n3_max[3], int out[3]);
void pm_set_imu_inited(lio_pm *m);
// laser_cloud_{corner,surf}_stack_downsampled_ of the last process call (device arrays, host counts), the call's full cloud as
// copied into the handle, and the device counts {corner in, surf in, corner ds, surf ds, full} (clamped to the call's bounds)
const float4 *pm_ds(const lio_pm *m, int which);
int pm_ds_n(const lio_pm *m, int which);
const float4 *pm_full_in(const lio_pm *m);
const int *pm_counts_dev(const lio_pm *m);
const std::vector<size_t> &pm_valid(const lio_pm *m);
void pm_centre(const lio_pm *m, int c[3]);
