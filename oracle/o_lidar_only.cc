// ORACLE — TEST INFRASTRUCTURE ONLY (see o_linalg.h header).
// The estimator with imu_factor = 0 fed the odometry's /compact_data messages (update_laser_imu = 1), restated around the unchanged
// orc::Estimator (ProcessCompactData Estimator.cc:776-856, ProcessLaserOdom :430-774):
//   PointMapping::Process   :765-1052 as o_pm_publish.cc states it, on a CubeMap of o_cubemap.cc driven through orc_cm_*; with
//                           imu_inited_ (after SetInitFlag, :544) no UpdateMapDatabase and no PublishResults (PointMapping.cc:1033);
//                           the association is the same TransformAssociateToMap that ProcessCompactData runs instead (:804)
//   decimation              :436-439: before initialisation only every init_window_factor-th message reaches the push
//   push                    :441-487: all_laser_transforms_ (transform_aft_mapped_), opt_point_coeff_mask_ (false, set true at the
//                           end of the NOT_INITED case :616), opt_cube_centers_, opt_valid_idx_, and the stacks: PointMapping's
//                           down-sampled ones before initialisation or without de-skew flags (:474-480), else the INITED de-skew
//                           push after the opt entry (:628-693), so that entry aliases the previous frame's objects (o_global_map.cc)
//   NOT_INITED              cir_buf_count_ < W: SlideWindow's state copy into index cir_buf_count_ + 1, ++cir_buf_count_ (:603-614);
//                           == W: Ps_ / Rs_[0..W] = trans_li * transform_lb_ (float Twist, normalised rotation, cast to double,
//                           :511-517), SolveOptimization, SlideWindow, no estimator insert or publication
//   INITED                  SolveOptimization, whose first step with !imu_factor overwrites state W (:1670-1676, restated here in
//                           front of orc::Estimator::SolveOptimization, which has no such step), UpdateMapDatabase of the first opt
//                           entry when its mask is false with its own valid list and centre (:703-708, pose :2279-2286),
//                           PublishResults (:721), SlideWindow
// Without IMU input (transform_es_ stays the identity), which is how the tests drive it.
#include "o_estimator.h"
#include <cstring>
#include <array>
#include <deque>
#include <memory>

extern "C" {   // o_cubemap.cc
void *orc_cm_create();
void orc_cm_destroy(void *h);
void orc_cm_recentre(void *h, const float *pos3, int *out6);
void orc_cm_select(void *h, const float *pos3, const float *zaxis3, const int *centre3, long long *valid, long long *surround, int *n2);
int orc_cm_cube_size(void *h, long long index, int which);
void orc_cm_cube_copy(void *h, long long index, int which, float *out);
void orc_cm_update(void *h, const float *corner, int nc, const float *surf, int ns, const long long *valid, int nv, const float *tf7,
                   const int *margin_centre3);
}

namespace orc {

static Transform lo_tf_of(const float *a) { return Transform(Quat<float>(a[3], a[0], a[1], a[2]), Vec3<float>(a[4], a[5], a[6])); }
static void lo_tf_out(const Transform &t, float *o) {
  o[0] = t.rot.x; o[1] = t.rot.y; o[2] = t.rot.z; o[3] = t.rot.w; o[4] = t.pos.x; o[5] = t.pos.y; o[6] = t.pos.z;
}
typedef std::shared_ptr<Cloud> CloudPtr;

struct LidarOnly {
  Estimator *e;
  void *map;
  StageBConfig pm_cfg;
  float corner_leaf = 0.2f, surf_leaf = 0.4f, map_filter_size = 0.6f;
  int init_window_factor = 1;
  double start_shift = 0.0;          // added to Ps_[i].x at the start-up: the divergence probe of the GPU tests
  // PointMapping
  Transform sum, bef, aft, tobe;
  int centre[3] = {10, 10, 5};
  int map_frame_count = 4;           // num_map_frames_ - 1 (PointMapping.cc:104)
  std::vector<long long> valid, surround;
  Cloud corner_ds, surf_ds;
  bool imu_inited = false;
  // Estimator
  bool inited = false;
  int cir_buf_count = 0, recv_count = 0;
  std::vector<Transform> laser_tf;   // all_laser_transforms_
  std::vector<CloudPtr> surf_obj, corner_obj;
  std::deque<CloudPtr> opt_surf, opt_corner;
  std::deque<bool> opt_mask;
  std::deque<std::vector<long long>> opt_valid;
  std::deque<std::array<int, 3>> opt_centre;
  // results of the last message
  int info[4] = {0, 0, 0, 0};        // inited, cir_buf_count, pushed, solved
  bool inserted = false, published = false, process_published = false;
  Transform insert_pose;
  Cloud ins_corner, ins_surf, surround_map, registered;
  std::vector<double> startup_states;   // (W + 1) x 16 written by the start-up, before its solve
  double pred[32] = {};                 // last overwrite: P_{W-1}(3) R_{W-1}(9) incre tf7 as float (7) P_W(3) R_W(9)

  LidarOnly(Estimator *est, int f, double shift) : e(est), map(orc_cm_create()), init_window_factor(f), start_shift(shift) {
    const int W = e->W, O = e->O;
    laser_tf.assign(W + 1, Transform());
    for (int k = 0; k <= W; ++k) { surf_obj.push_back(std::make_shared<Cloud>()); corner_obj.push_back(std::make_shared<Cloud>()); }
    for (int k = 0; k <= O; ++k) {
      opt_surf.push_back(nullptr); opt_corner.push_back(nullptr); opt_mask.push_back(true);
      opt_valid.push_back({}); opt_centre.push_back({0, 0, 0});
    }
    e->tmp_pre_integration = std::make_shared<IntegrationBase>(e->acc_last, e->gyr_last, e->Bas[0], e->Bgs[0], e->cfg.pim);
  }
  ~LidarOnly() { orc_cm_destroy(map); }

  Cloud Cube(long long index, int which) const {
    Cloud c((size_t)orc_cm_cube_size(map, index, which));
    if (!c.empty()) orc_cm_cube_copy(map, index, which, (float *)c.data());
    return c;
  }

  void Publish(const Cloud &full) {   // PointMapping::PublishResults :1210-1270
    published = false;
    if (++map_frame_count >= 5) {
      map_frame_count = 0;
      published = true;
      Cloud acc;
      for (long long index : surround)
        for (int w = 0; w < 2; ++w) { Cloud c = Cube(index, w); acc.insert(acc.end(), c.begin(), c.end()); }
      VoxelGridFilter(acc, map_filter_size, surround_map);
    }
    registered.resize(full.size());
    for (size_t i = 0; i < full.size(); ++i) PointAssociateToMap(full[i], registered[i], tobe);
  }

  void Process(const Cloud &corner_last, const Cloud &surf_last, const Cloud &full, const Transform &transform_sum) {
    sum = transform_sum;
    tobe = tobe * (bef.inverse() * sum);   // TransformAssociateToMap :753-756 (:804 once imu_inited_)
    Cloud corner_stack, surf_stack;
    PointXYZI point_sel;
    for (const PointXYZI &p : corner_last) { PointAssociateToMap(p, point_sel, tobe); corner_stack.push_back(point_sel); }
    for (const PointXYZI &p : surf_last) { PointAssociateToMap(p, point_sel, tobe); surf_stack.push_back(point_sel); }
    PointXYZI z;
    z.x = 0.0f; z.y = 0.0f; z.z = 10.0f; z.intensity = 0.f;
    PointAssociateToMap(z, z, tobe);
    const float pos3[3] = {tobe.pos.x, tobe.pos.y, tobe.pos.z}, z3[3] = {z.x, z.y, z.z};
    int out6[6];
    orc_cm_recentre(map, pos3, out6);
    centre[0] = out6[3]; centre[1] = out6[4]; centre[2] = out6[5];
    long long v[125], s[125];
    int n2[2];
    orc_cm_select(map, pos3, z3, out6, v, s, n2);
    valid.assign(v, v + n2[0]);
    surround.assign(s, s + n2[1]);
    Cloud corner_from_map, surf_from_map;
    for (long long index : valid) {
      Cloud c = Cube(index, 0), f = Cube(index, 1);
      corner_from_map.insert(corner_from_map.end(), c.begin(), c.end());
      surf_from_map.insert(surf_from_map.end(), f.begin(), f.end());
    }
    auto tobe_mapped = [&](PointXYZI &p) {   // PointAssociateTobeMapped :316-323
      Vec3<float> o = tobe.rot.conjugate() * Vec3<float>(p.x - tobe.pos.x, p.y - tobe.pos.y, p.z - tobe.pos.z);
      p.x = o.x; p.y = o.y; p.z = o.z;
    };
    for (PointXYZI &p : corner_stack) tobe_mapped(p);
    for (PointXYZI &p : surf_stack) tobe_mapped(p);
    VoxelGridFilter(corner_stack, corner_leaf, corner_ds);
    VoxelGridFilter(surf_stack, surf_leaf, surf_ds);
    const bool optimised = !(corner_from_map.size() <= 10 || surf_from_map.size() <= 100);
    int iters = 0;
    OptimizeTransformTobeMapped(corner_from_map, surf_from_map, corner_ds, surf_ds, tobe, pm_cfg, &iters, nullptr, 0);
    if (optimised) { bef = sum; aft = tobe; }
    process_published = false;
    if (!imu_inited) {
      float tf7[7];
      lo_tf_out(tobe, tf7);
      orc_cm_update(map, (const float *)corner_ds.data(), (int)corner_ds.size(), (const float *)surf_ds.data(), (int)surf_ds.size(),
                    valid.data(), (int)valid.size(), tf7, centre);
      Publish(full);
      process_published = published;
    }
  }

  void SyncStacks() { for (int k = 0; k <= e->W; ++k) *surf_obj[k] = e->surf_stack[k]; }

  void Message(const Cloud &corner_last, const Cloud &surf_last, const Cloud &full, const float *sum7) {
    const int W = e->W, O = e->O, pivot = W - O;
    Process(corner_last, surf_last, full, lo_tf_of(sum7));
    inserted = published = false;
    ++recv_count;
    info[0] = inited; info[1] = cir_buf_count; info[2] = info[3] = 0;
    if (!inited && recv_count % init_window_factor != 0) return;
    info[2] = 1;
    const bool deskew_flags = e->cfg.enable_deskew || e->cfg.cutoff_deskew;
    const bool pm_stacks = !inited || !deskew_flags;
    laser_tf.erase(laser_tf.begin()); laser_tf.push_back(aft);
    const int c = cir_buf_count;
    e->pre_integrations.erase(e->pre_integrations.begin());
    e->pre_integrations.push_back(e->tmp_pre_integration);
    e->tmp_pre_integration = std::make_shared<IntegrationBase>(e->acc_last, e->gyr_last, e->Bas[c], e->Bgs[c], e->cfg.pim);
    Cloud ds = surf_ds, cds = corner_ds;
    if (!pm_stacks) {   // INITED de-skew push (:628-693); without IMU input transform_es_ is never computed
      VoxelGridFilter(surf_last, e->cfg.b.surf_filter_size, ds);
      VoxelGridFilter(corner_last, corner_leaf, cds);
    }
    CloudPtr new_surf = std::make_shared<Cloud>(ds), new_corner = std::make_shared<Cloud>(cds);
    auto push_objects = [&]() {
      surf_obj.erase(surf_obj.begin()); surf_obj.push_back(new_surf);
      corner_obj.erase(corner_obj.begin()); corner_obj.push_back(new_corner);
    };
    if (pm_stacks) push_objects();
    opt_surf.push_back(surf_obj.back()); opt_corner.push_back(corner_obj.back()); opt_mask.push_back(false);
    opt_valid.push_back(valid); opt_centre.push_back({centre[0], centre[1], centre[2]});
    opt_surf.pop_front(); opt_corner.pop_front(); opt_mask.pop_front(); opt_valid.pop_front(); opt_centre.pop_front();
    if (!pm_stacks) push_objects();
    e->surf_stack.erase(e->surf_stack.begin()); e->surf_stack.push_back(ds);
    e->size_surf_stack.erase(e->size_surf_stack.begin()); e->size_surf_stack.push_back((int)ds.size());
    if (!inited) {
      opt_mask.back() = true;   // :616
      if (c < W) {
        e->Ps[c + 1] = e->Ps[c]; e->Vs[c + 1] = e->Vs[c]; e->Rs[c + 1] = e->Rs[c]; e->Bas[c + 1] = e->Bas[c]; e->Bgs[c + 1] = e->Bgs[c];
        info[1] = ++cir_buf_count;
        return;
      }
      startup_states.assign((W + 1) * 16, 0.0);
      for (int i = 0; i <= W; ++i) {   // :511-517
        const Transform trans_bi = laser_tf[i] * e->transform_lb;
        e->Ps[i] = trans_bi.pos.cast<double>();
        e->Ps[i].x += start_shift;
        e->Rs[i] = trans_bi.rot.normalized().toRotationMatrix().cast<double>();
        const Qd q = Qd::fromRotationMatrix(e->Rs[i]);
        double *st = &startup_states[16 * i];
        st[0] = e->Ps[i].x; st[1] = e->Ps[i].y; st[2] = e->Ps[i].z; st[3] = q.x; st[4] = q.y; st[5] = q.z; st[6] = q.w;
      }
      inited = true;
      imu_inited = true;   // SetInitFlag(true)
    }
    {  // SolveOptimization :1670-1676
      const Twist<double> incre = (e->transform_lb.inverse() * laser_tf[W - 1].inverse() * laser_tf[W] * e->transform_lb).cast<double>();
      const Transform incre_f = e->transform_lb.inverse() * laser_tf[W - 1].inverse() * laser_tf[W] * e->transform_lb;
      double *p = pred;
      p[0] = e->Ps[W - 1].x; p[1] = e->Ps[W - 1].y; p[2] = e->Ps[W - 1].z;
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) p[3 + 3 * a + b] = e->Rs[W - 1].m[a][b];
      float t7[7];
      lo_tf_out(incre_f, t7);
      for (int k = 0; k < 7; ++k) p[12 + k] = t7[k];
      e->Ps[W] = e->Rs[W - 1] * incre.pos + e->Ps[W - 1];
      e->Rs[W] = e->Rs[W - 1] * incre.rot.toRotationMatrix();
      p[19] = e->Ps[W].x; p[20] = e->Ps[W].y; p[21] = e->Ps[W].z;
      for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) p[22 + 3 * a + b] = e->Rs[W].m[a][b];
    }
    const bool startup = info[0] == 0;
    e->SolveOptimization();
    SyncStacks();
    if (!startup) {
      inserted = !opt_mask.front();
      if (inserted) {   // :703-708
        Twist<double> transform_lb = e->transform_lb.cast<double>();
        Qd rot_l0 = Qd::fromRotationMatrix(e->Rs[pivot] * transform_lb.rot.conjugate().normalized().toRotationMatrix());
        V3 pos_l0 = e->Ps[pivot] - rot_l0 * transform_lb.pos;
        insert_pose = Twist<double>(rot_l0, pos_l0).cast<float>();
        ins_corner = *opt_corner.front();
        ins_surf = *opt_surf.front();
        float tf7[7];
        lo_tf_out(insert_pose, tf7);
        orc_cm_update(map, (const float *)ins_corner.data(), (int)ins_corner.size(), (const float *)ins_surf.data(), (int)ins_surf.size(),
                      opt_valid.front().data(), (int)opt_valid.front().size(), tf7, opt_centre.front().data());
      }
      Publish(full);   // :721
    }
    e->SlideWindow();
    SyncStacks();
    info[0] = 1; info[1] = cir_buf_count; info[3] = 1;
  }
};

}  // namespace orc

using namespace orc;

extern "C" {

void *orc_lo_create(void *est, int init_window_factor, double start_shift) {
  return new LidarOnly((Estimator *)est, init_window_factor, start_shift);
}
void orc_lo_destroy(void *h) { delete (LidarOnly *)h; }
// one /compact_data message; info4 = {inited, cir_buf_count, pushed, solved}
void orc_lo_process_compact(void *h, const float *corner, int nc, const float *surf, int ns, const float *full, int nf, const float *sum7, int *info4) {
  LidarOnly *g = (LidarOnly *)h;
  g->Message(Cloud((const PointXYZI *)corner, (const PointXYZI *)corner + nc), Cloud((const PointXYZI *)surf, (const PointXYZI *)surf + ns),
             Cloud((const PointXYZI *)full, (const PointXYZI *)full + nf), sum7);
  std::memcpy(info4, g->info, sizeof(g->info));
}
// tobe7, aft7, insert7; info5 = {inserted, points inserted, surround published by the estimator, by Process, size of the surround map}
void orc_lo_poses(void *h, float *tobe7, float *aft7, float *insert7, int *info5) {
  LidarOnly *g = (LidarOnly *)h;
  lo_tf_out(g->tobe, tobe7); lo_tf_out(g->aft, aft7); lo_tf_out(g->insert_pose, insert7);
  info5[0] = g->inserted; info5[1] = g->inserted ? (int)(g->ins_corner.size() + g->ins_surf.size()) : 0;
  info5[2] = g->published; info5[3] = g->process_published; info5[4] = (int)g->surround_map.size();
}
int orc_lo_startup_states(void *h, double *out) {
  LidarOnly *g = (LidarOnly *)h;
  if (!g->startup_states.empty()) std::memcpy(out, g->startup_states.data(), sizeof(double) * g->startup_states.size());
  return (int)g->startup_states.size();
}
void orc_lo_prediction(void *h, double *out31) { std::memcpy(out31, ((LidarOnly *)h)->pred, sizeof(double) * 31); }
void orc_lo_centre(void *h, int *out3) { std::memcpy(out3, ((LidarOnly *)h)->centre, sizeof(int) * 3); }
int orc_lo_cube_size(void *h, long long index, int which) { return orc_cm_cube_size(((LidarOnly *)h)->map, index, which); }
void orc_lo_cube_copy(void *h, long long index, int which, float *out) { orc_cm_cube_copy(((LidarOnly *)h)->map, index, which, out); }
// :1670-1676 on explicit inputs: laser transforms T_{W-1}, T_W, transform_lb_ (float tf7), state W-1 (P(3), R(9) row-major);
// out = P_W(3), R_W(9)
void orc_lo_predict(const float *t_prev7, const float *t_curr7, const float *tlb7, const double *p_prev3, const double *r_prev9, double *out12) {
  const Transform lb = lo_tf_of(tlb7);
  const Twist<double> incre = (lb.inverse() * lo_tf_of(t_prev7).inverse() * lo_tf_of(t_curr7) * lb).cast<double>();
  M3 R;
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) R.m[a][b] = r_prev9[3 * a + b];
  const V3 P = R * incre.pos + V3(p_prev3[0], p_prev3[1], p_prev3[2]);
  const M3 Rw = R * incre.rot.toRotationMatrix();
  out12[0] = P.x; out12[1] = P.y; out12[2] = P.z;
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) out12[3 + 3 * a + b] = Rw.m[a][b];
}

}  // extern "C"
