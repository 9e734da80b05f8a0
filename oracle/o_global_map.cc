// ORACLE — TEST INFRASTRUCTURE ONLY (see o_linalg.h header).
// The estimator's global cube map after initialisation, restated around orc::Estimator and the PointMappingPublishOracle of
// o_pm_publish.cc without touching either (the reference's lio::Estimator is a PointMapping, imu_factor = 1, update_laser_imu = 1):
//   pre-initialisation      PointMapping::Process + PublishResults through orc_pmp_process; laser_cloud_valid_idx_ of the last call
//                           is recomputed here from its predicted pose (the oracle keeps it local), after which it stays frozen
//   prediction              ProcessCompactData (Estimator.cc:776-809): tobe = tobe * lb * (prev^-1 * curr) * lb^-1, float Twist;
//                           PointMapping::Process is not run (:810-812)
//   opt_* buffers           :467-485 record the frame's entry (mask false for INITED frames, :467) aliasing surf_stack_.last() /
//                           corner_stack_.last(); with enable_deskew || cutoff_deskew the INITED push of the frame's clouds comes
//                           later (:689-693), so the entry is the previous frame's object.  Objects are shared_ptrs here, their
//                           contents follow the estimator's stacks in place (the init merge :1409-1441 and SlideWindow :2615 rewrite
//                           surf_stack_ entries in place); an object that left the window lives on while an entry holds it
//   UpdateMapDatabase       :703-708 after SolveOptimization, before PublishResults and SlideWindow, when the first entry is INITED;
//                           pose opt_transforms_[0] as :2279-2286 overwrites it; valid list and centre the frozen ones
//   PublishResults          :721 (PointMapping.cc:1210-1270): map_frame_count_ continues; surround map from the frozen surround list;
//                           /cloud_registered = the scan's raw full cloud through PointAssociateToMap with the predicted tobe
// The estimator's ProcessScan (o_estimator.cc) is restated step by step so that the insert sits between its SolveOptimization and
// SlideWindow; the corner push is LocalClouds' (o_local_clouds.cc).
#include "o_estimator.h"
#include <cstring>
#include <deque>
#include <memory>

extern "C" {   // o_cubemap.cc, o_pm_publish.cc
void orc_cm_recentre(void *h, const float *pos3, int *out6);
void orc_cm_select(void *h, const float *pos3, const float *zaxis3, const int *centre3, long long *valid, long long *surround, int *n2);
int orc_cm_cube_size(void *h, long long index, int which);
void orc_cm_cube_copy(void *h, long long index, int which, float *out);
void orc_cm_update(void *h, const float *corner, int nc, const float *surf, int ns, const long long *valid, int nv, const float *tf7,
                   const int *margin_centre3);
void orc_pmp_process(void *h, const float *corner, int nc, const float *surf, int ns, const float *full, int nf, const float *sum7, float *tobe7,
                     float *aft7, int *info5);
int orc_pmp_surround_idx(void *h, long long *out);
void orc_pmp_centre(void *h, int *out3);
}

namespace orc {

static Transform gm_tf_of(const float *a) { return Transform(Quat<float>(a[3], a[0], a[1], a[2]), Vec3<float>(a[4], a[5], a[6])); }
static void gm_tf_out(const Transform &t, float *o) {
  o[0] = t.rot.x; o[1] = t.rot.y; o[2] = t.rot.z; o[3] = t.rot.w; o[4] = t.pos.x; o[5] = t.pos.y; o[6] = t.pos.z;
}
typedef std::shared_ptr<Cloud> CloudPtr;

struct GlobalMap {
  Estimator *e;
  void *pmp;                         // PointMappingPublishOracle (o_pm_publish.cc)
  void *map;                         // its CubeMap: the struct's first member
  float corner_filter_size, map_filter_size;
  // PointMapping state the estimator carries on
  Transform tobe, aft, bef;
  bool have_bef = false;
  int map_frame_count = 4;           // num_map_frames_ - 1 (PointMapping.cc:104)
  std::vector<long long> valid, surround;
  int centre[3] = {10, 10, 5};
  // stacks as objects
  std::vector<CloudPtr> surf_obj, corner_obj;
  std::deque<CloudPtr> opt_surf, opt_corner;
  std::deque<bool> opt_mask;
  Cloud staged_corner, staged_full;
  // results of the last scan
  bool inserted = false, published = false;
  Transform insert_pose;
  Cloud ins_corner, ins_surf, surround_map, registered;

  GlobalMap(Estimator *est, void *pm, float corner_leaf, float map_leaf)
      : e(est), pmp(pm), map(*static_cast<void **>(pm)), corner_filter_size(corner_leaf), map_filter_size(map_leaf) {
    for (int k = 0; k <= e->W; ++k) { surf_obj.push_back(std::make_shared<Cloud>()); corner_obj.push_back(std::make_shared<Cloud>()); }
    for (int k = 0; k <= e->O; ++k) { opt_surf.push_back(nullptr); opt_corner.push_back(nullptr); opt_mask.push_back(true); }
  }

  // one pre-initialisation PointMapping::Process + PublishResults (the oracle's), and the valid list of that call
  void PreInitProcess(const Cloud &corner, const Cloud &surf, const Cloud &full, const float *sum7, int *info5) {
    const Transform sum = gm_tf_of(sum7);
    const Transform pred = tobe * (bef.inverse() * sum);   // TransformAssociateToMap :753-756, as the oracle evaluates it
    float tobe7[7], aft7[7];
    orc_pmp_process(pmp, (const float *)corner.data(), (int)corner.size(), (const float *)surf.data(), (int)surf.size(), (const float *)full.data(),
                    (int)full.size(), sum7, tobe7, aft7, info5);
    PointXYZI z, zo;
    z.x = 0.f; z.y = 0.f; z.z = 10.f; z.intensity = 0.f;
    PointAssociateToMap(z, zo, pred);
    const float pos3[3] = {pred.pos.x, pred.pos.y, pred.pos.z}, z3[3] = {zo.x, zo.y, zo.z};
    int out6[6];
    orc_cm_recentre(map, pos3, out6);   // the call has re-centred for this position already: no shift here
    long long v[125], s[125];
    int n2[2];
    orc_cm_select(map, pos3, z3, out6, v, s, n2);
    valid.assign(v, v + n2[0]);
    surround.assign(s, s + n2[1]);
    orc_pmp_centre(pmp, centre);
    tobe = gm_tf_of(tobe7);
    aft = gm_tf_of(aft7);
    if (info5[1] > 10 && info5[2] > 100) bef = sum;   // TransformUpdate behind the optimiser's early return
    if (++map_frame_count >= 5) map_frame_count = 0;
  }

  void InitFrame(int k, const Cloud &surf_ds) {   // warm-start frames land one slot to the right (o_estimator.cc InitFrame)
    *surf_obj[k + 1] = surf_ds;
    *corner_obj[k + 1] = staged_corner;
  }

  void SyncStacks() { for (int k = 0; k <= e->W; ++k) *surf_obj[k] = e->surf_stack[k]; }

  void ProcessScan(const Cloud &surf_last_in) {
    const int W = e->W, O = e->O, pivot = W - O;
    const bool deskew_flags = e->cfg.enable_deskew || e->cfg.cutoff_deskew;
    {  // prediction (:776-809)
      const Transform prev(Qd::fromRotationMatrix(e->Rs[W - 1]).cast<float>(), e->Ps[W - 1].cast<float>());
      const Transform curr(Qd::fromRotationMatrix(e->Rs[W]).cast<float>(), e->Ps[W].cast<float>());
      const Transform d_trans = prev.inverse() * curr;
      tobe = tobe * e->transform_lb * d_trans * e->transform_lb.inverse();
    }
    // o_estimator.cc ProcessScan up to the solve
    e->pre_integrations.erase(e->pre_integrations.begin());
    e->pre_integrations.push_back(e->tmp_pre_integration);
    e->tmp_pre_integration = std::make_shared<IntegrationBase>(e->acc_last, e->gyr_last, e->Bas[W], e->Bgs[W], e->cfg.pim);
    Cloud surf_last = surf_last_in, corner = staged_corner;
    if (deskew_flags && !e->imu_stampedtransforms.empty()) {
      double time_e = e->imu_stampedtransforms.back().time;
      Transform transform_e = e->imu_stampedtransforms.back().transform;
      double time_s = time_e;
      Transform transform_s = transform_e;
      for (int i = int(e->imu_stampedtransforms.size()) - 1; i >= 0; --i) {
        time_s = e->imu_stampedtransforms[i].time;
        transform_s = e->imu_stampedtransforms[i].transform;
        if (time_e - e->imu_stampedtransforms[i].time >= 0.1) break;
      }
      Transform transform_body_es = transform_e.inverse() * transform_s;
      {
        float s = 0.1 / (time_e - time_s);
        Quat<float> q_id, q_e = transform_body_es.rot;
        transform_body_es.rot = q_id.slerp(s, q_e);
        transform_body_es.pos = s * transform_body_es.pos;
      }
      e->transform_es = e->transform_lb * transform_body_es * e->transform_lb.inverse();
      if (!e->cfg.cutoff_deskew) { TransformToEnd(surf_last, e->transform_es, 10); TransformToEnd(corner, e->transform_es, 10); }
    }
    Cloud ds, corner_ds;
    VoxelGridFilter(surf_last, e->cfg.b.surf_filter_size, ds);
    VoxelGridFilter(corner, corner_filter_size, corner_ds);
    // :467-485 the opt entry, :474 / :689 the pushes
    CloudPtr new_surf = std::make_shared<Cloud>(ds), new_corner = std::make_shared<Cloud>(corner_ds);
    auto push_objects = [&]() {
      surf_obj.erase(surf_obj.begin()); surf_obj.push_back(new_surf);
      corner_obj.erase(corner_obj.begin()); corner_obj.push_back(new_corner);
    };
    if (!deskew_flags) push_objects();
    opt_surf.push_back(surf_obj.back()); opt_corner.push_back(corner_obj.back()); opt_mask.push_back(false);
    opt_surf.pop_front(); opt_corner.pop_front(); opt_mask.pop_front();
    if (deskew_flags) push_objects();
    e->surf_stack.erase(e->surf_stack.begin()); e->surf_stack.push_back(ds);
    e->size_surf_stack.erase(e->size_surf_stack.begin()); e->size_surf_stack.push_back((int)ds.size());
    e->SolveOptimization();   // the init merge rewrites surf_stack_[pivot] in place
    SyncStacks();
    // UpdateMapDatabase (:703-708)
    inserted = !opt_mask.front();
    if (inserted) {
      Twist<double> transform_lb = e->transform_lb.cast<double>();
      Qd rot_l0 = Qd::fromRotationMatrix(e->Rs[pivot] * transform_lb.rot.conjugate().normalized().toRotationMatrix());
      V3 pos_l0 = e->Ps[pivot] - rot_l0 * transform_lb.pos;
      insert_pose = Twist<double>(rot_l0, pos_l0).cast<float>();
      ins_corner = *opt_corner.front();
      ins_surf = *opt_surf.front();
      float tf7[7];
      gm_tf_out(insert_pose, tf7);
      orc_cm_update(map, (const float *)ins_corner.data(), (int)ins_corner.size(), (const float *)ins_surf.data(), (int)ins_surf.size(),
                    valid.data(), (int)valid.size(), tf7, centre);
    }
    // PublishResults (:721)
    published = false;
    if (++map_frame_count >= 5) {
      map_frame_count = 0;
      published = true;
      Cloud acc;
      for (long long index : surround)
        for (int w = 0; w < 2; ++w) {
          Cloud c((size_t)orc_cm_cube_size(map, index, w));
          if (!c.empty()) orc_cm_cube_copy(map, index, w, (float *)c.data());
          acc.insert(acc.end(), c.begin(), c.end());
        }
      VoxelGridFilter(acc, map_filter_size, surround_map);
    }
    registered.resize(staged_full.size());
    for (size_t i = 0; i < staged_full.size(); ++i) PointAssociateToMap(staged_full[i], registered[i], tobe);
    e->SlideWindow();          // rewrites surf_stack_[pivot + 1] in place
    SyncStacks();
  }
};

}  // namespace orc

using namespace orc;

extern "C" {

void *orc_gm_create(void *est, void *pmp, float corner_filter_size, float map_filter_size) {
  return new GlobalMap((Estimator *)est, pmp, corner_filter_size, map_filter_size);
}
void orc_gm_destroy(void *h) { delete (GlobalMap *)h; }
void orc_gm_set_scan_clouds(void *h, const float *corner, int nc, const float *full, int nf) {
  GlobalMap *g = (GlobalMap *)h;
  g->staged_corner.assign((const PointXYZI *)corner, (const PointXYZI *)corner + nc);
  g->staged_full.assign((const PointXYZI *)full, (const PointXYZI *)full + nf);
}
void orc_gm_pre_init_process(void *h, const float *corner, int nc, const float *surf, int ns, const float *full, int nf, const float *sum7,
                             int *info5) {
  Cloud c((const PointXYZI *)corner, (const PointXYZI *)corner + nc), s((const PointXYZI *)surf, (const PointXYZI *)surf + ns),
      f((const PointXYZI *)full, (const PointXYZI *)full + nf);
  ((GlobalMap *)h)->PreInitProcess(c, s, f, sum7, info5);
}
void orc_gm_init_frame(void *h, int k, const float *surf_ds, int n) {
  ((GlobalMap *)h)->InitFrame(k, Cloud((const PointXYZI *)surf_ds, (const PointXYZI *)surf_ds + n));
}
void orc_gm_process_scan(void *h, const float *surf_last, int n) {
  ((GlobalMap *)h)->ProcessScan(Cloud((const PointXYZI *)surf_last, (const PointXYZI *)surf_last + n));
}
// tobe7, aft7, insert7; info4 = {inserted, points inserted, surround published, size of the last surround map}
void orc_gm_poses(void *h, float *tobe7, float *aft7, float *insert7, int *info4) {
  GlobalMap *g = (GlobalMap *)h;
  gm_tf_out(g->tobe, tobe7); gm_tf_out(g->aft, aft7); gm_tf_out(g->insert_pose, insert7);
  info4[0] = g->inserted; info4[1] = g->inserted ? (int)(g->ins_corner.size() + g->ins_surf.size()) : 0;
  info4[2] = g->published; info4[3] = (int)g->surround_map.size();
}
// which: 0 inserted corner, 1 inserted surf, 2 surround map, 3 registered cloud
static const Cloud &gm_cloud(GlobalMap *g, int which) {
  return which == 0 ? g->ins_corner : which == 1 ? g->ins_surf : which == 2 ? g->surround_map : g->registered;
}
int orc_gm_cloud_size(void *h, int which) { return (int)gm_cloud((GlobalMap *)h, which).size(); }
void orc_gm_cloud_copy(void *h, int which, float *out) {
  const Cloud &c = gm_cloud((GlobalMap *)h, which);
  if (!c.empty()) std::memcpy(out, c.data(), sizeof(PointXYZI) * c.size());
}
int orc_gm_valid(void *h, long long *out) {
  GlobalMap *g = (GlobalMap *)h;
  std::memcpy(out, g->valid.data(), sizeof(long long) * g->valid.size());
  return (int)g->valid.size();
}
// ProcessCompactData's prediction on explicit states (state16: P, Q xyzw, ...) as the reference evaluates it
void orc_gm_predict(const float *tobe7, const double *s_prev, const double *s_curr, const float *tlb7, float *out7) {
  const Transform lb = gm_tf_of(tlb7);
  auto tw = [](const double *s) {
    return Transform(Qd(s[6], s[3], s[4], s[5]).cast<float>(), Vec3<float>((float)s[0], (float)s[1], (float)s[2]));
  };
  gm_tf_out(gm_tf_of(tobe7) * lb * (tw(s_prev).inverse() * tw(s_curr)) * lb.inverse(), out7);
}

}  // extern "C"
