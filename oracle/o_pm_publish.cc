// ORACLE — TEST INFRASTRUCTURE ONLY (see o_linalg.h header).
//
// CPU restatement of lio::PointMapping::Process followed by PointMapping::PublishResults (src/point_processor/PointMapping.cc),
// what the mapping node does with every synchronised set of /laser_cloud_corner_last, /laser_cloud_surf_last, /full_odom_cloud and
// /laser_odom_to_init:
//   Process                     :765-1052   the PointMappingOracle steps of o_cubemap.cc (imu_inited_ == false, num_stack_frames_ 1)
//   PublishResults              :1210-1270  map_frame_count_ starts at num_map_frames_ - 1 (:104): the surround map (every surround
//                                           cube's corner then surf cloud, VoxelGrid(0.6), :123) on calls 1, 6, 11, ...; the full
//                                           cloud through PointAssociateToMap with the final transform_tobe_mapped_; and
//                                           transform_aft_mapped_ (/aft_mapped_to_init)
// The cube map is the one of o_cubemap.cc, driven through its C API (orc_cm_*), as o_mapbuilder.cc does; the cube leaves are
// CubeMap's 0.2 / 0.4.  Device counterpart: lio_pm_enable_publish + lio_pm_process_dev in lio_mapping_b200/csrc/cubemap.cu,
// compared in tests/test_lidar_chain_gpu.py.
#include "o_api.h"
#include <cstring>

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

static Transform pmp_tf_of(const float *a) { return Transform(Quat<float>(a[3], a[0], a[1], a[2]), Vec3<float>(a[4], a[5], a[6])); }
static void pmp_tf_out(const Transform &t, float *o) {
  o[0] = t.rot.x; o[1] = t.rot.y; o[2] = t.rot.z; o[3] = t.rot.w; o[4] = t.pos.x; o[5] = t.pos.y; o[6] = t.pos.z;
}

struct PointMappingPublishOracle {
  void *map = nullptr;                   // o_cubemap.cc CubeMap
  int centre[3] = {10, 10, 5};
  Transform sum, bef, aft, tobe;         // transform_sum_, transform_bef_mapped_, transform_aft_mapped_, transform_tobe_mapped_
  StageBConfig cfg;
  float corner_leaf = 0.2f, surf_leaf = 0.4f, map_filter_size = 0.6f;
  static constexpr int num_map_frames = 5;
  int map_frame_count = num_map_frames - 1;
  int last_iters = 0, last_published = 0;
  size_t last_corner_from_map = 0, last_surf_from_map = 0;
  std::vector<long long> surround_idx;   // laser_cloud_surround_idx_ of the last call
  Cloud surround, full_registered;

  PointMappingPublishOracle() : map(orc_cm_create()) {}
  ~PointMappingPublishOracle() { orc_cm_destroy(map); }

  Cloud Cube(long long index, int which) const {
    Cloud c((size_t)orc_cm_cube_size(map, index, which));
    if (!c.empty()) orc_cm_cube_copy(map, index, which, (float *)c.data());
    return c;
  }

  static void PointAssociateTobeMapped(const PointXYZI &pi, PointXYZI &po, const Transform &t) {   // :316-323
    Vec3<float> v(pi.x - t.pos.x, pi.y - t.pos.y, pi.z - t.pos.z);
    Vec3<float> o = t.rot.conjugate() * v;
    po.x = o.x; po.y = o.y; po.z = o.z; po.intensity = pi.intensity;
  }

  void Process(const Cloud &corner_last, const Cloud &surf_last, const Cloud &full_cloud, const Transform &transform_sum) {
    sum = transform_sum;
    {  // TransformAssociateToMap :753-756
      Transform incre = bef.inverse() * sum;
      tobe = tobe * incre;
    }
    Cloud corner_stack, surf_stack;
    PointXYZI point_sel;
    for (const PointXYZI &p : corner_last) { PointAssociateToMap(p, point_sel, tobe); corner_stack.push_back(point_sel); }
    for (const PointXYZI &p : surf_last) { PointAssociateToMap(p, point_sel, tobe); surf_stack.push_back(point_sel); }
    PointXYZI point_on_z_axis;
    point_on_z_axis.x = 0.0f; point_on_z_axis.y = 0.0f; point_on_z_axis.z = 10.0f; point_on_z_axis.intensity = 0.f;
    PointAssociateToMap(point_on_z_axis, point_on_z_axis, tobe);
    // re-centring (:809-931), cube selection (:944-1003)
    const float pos3[3] = {tobe.pos.x, tobe.pos.y, tobe.pos.z}, z3[3] = {point_on_z_axis.x, point_on_z_axis.y, point_on_z_axis.z};
    int out6[6];
    orc_cm_recentre(map, pos3, out6);
    centre[0] = out6[3]; centre[1] = out6[4]; centre[2] = out6[5];
    long long valid[125], sur[125];
    int n2[2];
    orc_cm_select(map, pos3, z3, out6, valid, sur, n2);
    surround_idx.assign(sur, sur + n2[1]);
    // laser_cloud_*_from_map_ (:1005-1011)
    Cloud corner_from_map, surf_from_map;
    for (int i = 0; i < n2[0]; ++i) {
      Cloud c = Cube(valid[i], 0), s = Cube(valid[i], 1);
      corner_from_map.insert(corner_from_map.end(), c.begin(), c.end());
      surf_from_map.insert(surf_from_map.end(), s.begin(), s.end());
    }
    last_corner_from_map = corner_from_map.size(); last_surf_from_map = surf_from_map.size();
    for (PointXYZI &p : corner_stack) PointAssociateTobeMapped(p, p, tobe);
    for (PointXYZI &p : surf_stack) PointAssociateTobeMapped(p, p, tobe);
    Cloud corner_ds, surf_ds;
    VoxelGridFilter(corner_stack, corner_leaf, corner_ds);
    VoxelGridFilter(surf_stack, surf_leaf, surf_ds);
    const bool optimised = !(corner_from_map.size() <= 10 || surf_from_map.size() <= 100);
    last_iters = 0;
    OptimizeTransformTobeMapped(corner_from_map, surf_from_map, corner_ds, surf_ds, tobe, cfg, &last_iters, nullptr, 0);
    if (optimised) { bef = sum; aft = tobe; }   // TransformUpdate() sits behind the early return of the optimiser (:327-329, :716)
    float tf7[7];
    pmp_tf_out(tobe, tf7);
    orc_cm_update(map, (const float *)corner_ds.data(), (int)corner_ds.size(), (const float *)surf_ds.data(), (int)surf_ds.size(), valid, n2[0],
                  tf7, centre);
    PublishResults(full_cloud);
  }

  void PublishResults(const Cloud &full_cloud) {   // :1210-1270
    last_published = 0;
    if (++map_frame_count >= num_map_frames) {
      map_frame_count = 0;
      last_published = 1;
      Cloud acc;
      for (long long index : surround_idx) {
        Cloud c = Cube(index, 0), s = Cube(index, 1);
        acc.insert(acc.end(), c.begin(), c.end());
        acc.insert(acc.end(), s.begin(), s.end());
      }
      VoxelGridFilter(acc, map_filter_size, surround);
    }
    full_registered.resize(full_cloud.size());
    for (size_t i = 0; i < full_cloud.size(); ++i) PointAssociateToMap(full_cloud[i], full_registered[i], tobe);
  }
};

}  // namespace orc

using namespace orc;
extern "C" {
// cfg: {map_filter_size, min_match_sq_dis, min_plane_dis, max_iterations}
void *orc_pmp_create(const float *cfg4) {
  PointMappingPublishOracle *m = new PointMappingPublishOracle();
  m->map_filter_size = cfg4[0]; m->cfg.min_match_sq_dis = cfg4[1]; m->cfg.min_plane_dis = cfg4[2]; m->cfg.num_max_iterations = (int)cfg4[3];
  return m;
}
void orc_pmp_destroy(void *h) { delete (PointMappingPublishOracle *)h; }
// out: tobe tf7, aft tf7, info5 = {iterations, corner_from_map, surf_from_map, surround published, size of the last surround map}
void orc_pmp_process(void *h, const float *corner, int nc, const float *surf, int ns, const float *full, int nf, const float *sum7, float *tobe7,
                     float *aft7, int *info5) {
  PointMappingPublishOracle *m = (PointMappingPublishOracle *)h;
  Cloud c((const PointXYZI *)corner, (const PointXYZI *)corner + nc), s((const PointXYZI *)surf, (const PointXYZI *)surf + ns),
      f((const PointXYZI *)full, (const PointXYZI *)full + nf);
  m->Process(c, s, f, pmp_tf_of(sum7));
  pmp_tf_out(m->tobe, tobe7);
  pmp_tf_out(m->aft, aft7);
  info5[0] = m->last_iters; info5[1] = (int)m->last_corner_from_map; info5[2] = (int)m->last_surf_from_map; info5[3] = m->last_published;
  info5[4] = (int)m->surround.size();
}
// which: 0 surround map (last published), 1 registered full cloud (last call)
int orc_pmp_cloud_size(void *h, int which) {
  PointMappingPublishOracle *m = (PointMappingPublishOracle *)h;
  return (int)(which == 0 ? m->surround : m->full_registered).size();
}
void orc_pmp_cloud_copy(void *h, int which, float *out) {
  PointMappingPublishOracle *m = (PointMappingPublishOracle *)h;
  const Cloud &c = which == 0 ? m->surround : m->full_registered;
  std::memcpy(out, c.data(), sizeof(PointXYZI) * c.size());
}
// laser_cloud_surround_idx_ of the last call (<= 125 cube indices, the order PublishResults concatenates them in); returns the count
int orc_pmp_surround_idx(void *h, long long *out) {
  PointMappingPublishOracle *m = (PointMappingPublishOracle *)h;
  std::memcpy(out, m->surround_idx.data(), sizeof(long long) * m->surround_idx.size());
  return (int)m->surround_idx.size();
}
int orc_pmp_cube_size(void *h, long long index, int which) { return orc_cm_cube_size(((PointMappingPublishOracle *)h)->map, index, which); }
void orc_pmp_cube_copy(void *h, long long index, int which, float *out) { orc_cm_cube_copy(((PointMappingPublishOracle *)h)->map, index, which, out); }
void orc_pmp_centre(void *h, int *out3) { std::memcpy(out3, ((PointMappingPublishOracle *)h)->centre, sizeof(int) * 3); }
// PointAssociateToMap (:303-314) of a whole cloud with one tf7
void orc_associate_to_map(const float *in, int n, const float *tf7, float *out) {
  const Transform t = pmp_tf_of(tf7);
  const PointXYZI *pi = (const PointXYZI *)in;
  PointXYZI *po = (PointXYZI *)out;
  for (int i = 0; i < n; ++i) PointAssociateToMap(pi[i], po[i], t);
}
}
