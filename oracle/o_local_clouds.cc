// ORACLE — TEST INFRASTRUCTURE ONLY (see o_linalg.h header).
// The estimator's /local/* publication, the map builder's input (launch/map_4D.launch), restated around orc::Estimator without
// touching it (o_estimator.cc stays the restatement of the solve):
//   corner_stack_ / full_stack_ pushes      Estimator.cc:474-482 (pre-initialisation), :628-693 (INITED: TransformToEnd of the
//                                           corner cloud under the surf cloud's condition, VoxelGrid(corner_filter_size))
//   TransformToEnd(.., keep_intensity)      Estimator.cc:62-103
//   /local/{corner,surf,full}_points        Estimator.cc:2355-2375, published before SlideWindow (:2591-2615) prepends the
//                                           transformed pivot cloud to surf_stack_[pivot + 1]
//   full-cloud de-skew of the newest frame  Estimator.cc:2416 (after the publication, also under cutoff_deskew)
//   /local_laser_odom                       Estimator.cc:725-742
#include "o_estimator.h"
#include <cstring>

namespace orc {

// Estimator.cc:62-103 with the keep_intensity argument (the full-cloud call site :2416 passes true)
size_t TransformToEnd(Cloud &cloud, const Transform &transform_es, float time_factor, bool keep_intensity) {
  size_t cloud_size = cloud.size();
  for (size_t i = 0; i < cloud_size; i++) {
    PointXYZI &point = cloud[i];
    float s = time_factor * (point.intensity - int(point.intensity));
    point.x -= s * transform_es.pos.x;
    point.y -= s * transform_es.pos.y;
    point.z -= s * transform_es.pos.z;
    if (!keep_intensity) point.intensity -= int(point.intensity);
    Quat<float> q_id, q_e = transform_es.rot;
    Quat<float> q_s = q_id.slerp(s, q_e);
    Vec3<float> v(point.x, point.y, point.z);
    v = q_s.conjugate().normalized() * v;
    v = q_e * v;
    point.x = v.x + transform_es.pos.x;
    point.y = v.y + transform_es.pos.y;
    point.z = v.z + transform_es.pos.z;
  }
  return cloud_size;
}

// /local_laser_odom (:725-742): Quaterniond(Rs_[pivot] * transform_lb.rot.inverse()), Ps_[pivot] - rot * transform_lb.pos
static Twist<double> LocalLaserOdom(const V3 &P, const M3 &R, const Transform &transform_lb_f) {
  Twist<double> transform_lb = transform_lb_f.cast<double>();
  Qd rot = Qd::fromRotationMatrix(R * transform_lb.rot.inverse().toRotationMatrix());
  V3 pos = P - rot * transform_lb.pos;
  return Twist<double>(rot, pos);
}

struct LocalClouds {
  Estimator *e;
  float corner_filter_size = 0.2f;
  std::vector<Cloud> corner_stack, full_stack;
  Cloud staged_corner, staged_full;
  Cloud pub[3];   // corner, surf, full of the last scan
  Transform transform_es;   // the value used for the last scan's pushes

  LocalClouds(Estimator *est, float leaf) : e(est), corner_filter_size(leaf) {
    corner_stack.assign(e->W + 1, Cloud());
    full_stack.assign(e->W + 1, Cloud());
  }
  void InitFrame(int k) {   // frames 0..W-1 land one slot to the right, like surf_stack (o_estimator.cc InitFrame)
    corner_stack[k + 1] = staged_corner;
    full_stack[k + 1] = staged_full;
  }
  void ProcessScan(const Cloud &surf_last) {
    const int W = e->W, pivot = W - e->O;
    const bool deskew = (e->cfg.enable_deskew || e->cfg.cutoff_deskew) && !e->imu_stampedtransforms.empty() && !e->cfg.cutoff_deskew;
    e->ProcessScan(surf_last);   // computes e->transform_es (:628-664) before the solve; corner / full do not feed the solve
    transform_es = e->transform_es;
    Cloud corner = staged_corner;
    if (deskew) TransformToEnd(corner, transform_es, 10);   // :666-673
    Cloud ds;
    VoxelGridFilter(corner, corner_filter_size, ds);         // :686-689
    corner_stack.erase(corner_stack.begin()); corner_stack.push_back(ds);
    full_stack.erase(full_stack.begin()); full_stack.push_back(staged_full);   // :482
    // publication (:2362-2375) of frame pivot + 1 before SlideWindow; the oracle's SlideWindow has since prepended the transformed
    // pivot cloud to surf_stack[pivot + 1], so the published surf cloud is that slot's tail of size_surf_stack[pivot + 1] points
    pub[0] = corner_stack[pivot + 1];
    const Cloud &s = e->surf_stack[pivot + 1];
    const size_t own = (size_t)e->size_surf_stack[pivot + 1];
    pub[1].assign(s.end() - (std::ptrdiff_t)std::min(own, s.size()), s.end());
    pub[2] = full_stack[pivot + 1];
    TransformToEnd(full_stack[W], transform_es, 10, true);   // :2416, after the publication
  }
};

}  // namespace orc

using namespace orc;

extern "C" {

void *orc_lc_create(void *est, float corner_filter_size) { return new LocalClouds((Estimator *)est, corner_filter_size); }
void orc_lc_destroy(void *h) { delete (LocalClouds *)h; }
void orc_lc_set_scan_clouds(void *h, const float *corner, int nc, const float *full, int nf) {
  LocalClouds *l = (LocalClouds *)h;
  l->staged_corner.assign((const PointXYZI *)corner, (const PointXYZI *)corner + nc);
  l->staged_full.assign((const PointXYZI *)full, (const PointXYZI *)full + nf);
}
void orc_lc_init_frame(void *h, int k) { ((LocalClouds *)h)->InitFrame(k); }
void orc_lc_process_scan(void *h, const float *surf_last, int n) {
  Cloud c((const PointXYZI *)surf_last, (const PointXYZI *)surf_last + n);
  ((LocalClouds *)h)->ProcessScan(c);
}
// which: 0 corner, 1 surf, 2 full
int orc_lc_cloud_size(void *h, int which) { return (int)((LocalClouds *)h)->pub[which].size(); }
void orc_lc_cloud_copy(void *h, int which, float *out) {
  const Cloud &c = ((LocalClouds *)h)->pub[which];
  if (!c.empty()) std::memcpy(out, c.data(), sizeof(PointXYZI) * c.size());
}
void orc_lc_transform_es(void *h, float *tf7) {
  const Transform &t = ((LocalClouds *)h)->transform_es;
  tf7[0] = t.rot.x; tf7[1] = t.rot.y; tf7[2] = t.rot.z; tf7[3] = t.rot.w; tf7[4] = t.pos.x; tf7[5] = t.pos.y; tf7[6] = t.pos.z;
}
// /local_laser_odom of the estimator's current window, rounded to float (tf7)
void orc_lc_local_laser_odom(void *h, float *tf7) {
  Estimator *e = ((LocalClouds *)h)->e;
  const int pivot = e->W - e->O;
  Twist<double> t = LocalLaserOdom(e->Ps[pivot], e->Rs[pivot], e->transform_lb);
  tf7[0] = (float)t.rot.x; tf7[1] = (float)t.rot.y; tf7[2] = (float)t.rot.z; tf7[3] = (float)t.rot.w;
  tf7[4] = (float)t.pos.x; tf7[5] = (float)t.pos.y; tf7[6] = (float)t.pos.z;
}
// The same formula for an explicit state16 (P, Q xyzw, ...) and a float extrinsic tf7: Rs = Q.normalized().toRotationMatrix()
void orc_local_laser_odom_of(const double *s, const float *tlb7, float *tf7) {
  Transform tlb(Quat<float>(tlb7[3], tlb7[0], tlb7[1], tlb7[2]), Vec3<float>(tlb7[4], tlb7[5], tlb7[6]));
  M3 R = Qd(s[6], s[3], s[4], s[5]).normalized().toRotationMatrix();
  Twist<double> t = LocalLaserOdom(V3(s[0], s[1], s[2]), R, tlb);
  tf7[0] = (float)t.rot.x; tf7[1] = (float)t.rot.y; tf7[2] = (float)t.rot.z; tf7[3] = (float)t.rot.w;
  tf7[4] = (float)t.pos.x; tf7[5] = (float)t.pos.y; tf7[6] = (float)t.pos.z;
}
void orc_transform_to_end_keep(float *cloud, int n, const float *tf7, float time_factor, int keep_intensity) {
  Cloud c((const PointXYZI *)cloud, (const PointXYZI *)cloud + n);
  Transform t(Quat<float>(tf7[3], tf7[0], tf7[1], tf7[2]), Vec3<float>(tf7[4], tf7[5], tf7[6]));
  TransformToEnd(c, t, time_factor, keep_intensity != 0);
  if (n > 0) std::memcpy(cloud, c.data(), sizeof(PointXYZI) * n);
}

}  // extern "C"
