// ORACLE — TEST INFRASTRUCTURE ONLY (see o_linalg.h header).
//
// CPU restatement of lio::MapBuilder::ProcessMap (src/map_builder/MapBuilder.cc:144-622) with the node's configuration
// (src/map_builder_node.cc: map_filter_size 0.2; enable_4d / skip_count :109-110) and DEBUG undefined (:36):
//   Transform4DAssociateToMap   :55-75    yaw-only correction of the odometry rotation
//   ProcessMap                  :220-622  PointMapping::Process with the 4-D association and the skip_count optimisation gate
//   PublishMapBuilderResults    :144-218  surround map every num_map_frames_ frames, registered full cloud
// The cube map is the one of o_cubemap.cc, driven through its C API (orc_cm_*); the cube leaves are CubeMap's 0.2 / 0.4, the
// node's values.  Device counterpart: lio_mapping_b200/csrc/cubemap.cu (lio_mb_*), compared in tests/test_map_builder_gpu.py.
#include "o_api.h"
#include <cmath>
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

// mathutils::R2ypr(Matrix3d).x() (include/utils/math_utils.h:188-203): yaw in degrees
static double R2yaw(const Mat3<double> &R) { return std::atan2(R(1, 0), R(0, 0)) / M_PI * 180.0; }

// mathutils::ypr2R<float> (math_utils.h:205-230): the angle is ypr(i) / 180.0 * M_PI evaluated in double and rounded to float;
// the unqualified cos / sin there resolve to the double ::cos / ::sin (only <cmath> is included), then round to float
static Mat3<float> ypr2R_float(const Vec3<float> &ypr) {
  float y = float(ypr.x / 180.0 * M_PI), p = float(ypr.y / 180.0 * M_PI), r = float(ypr.z / 180.0 * M_PI);
  auto c = [](float v) { return float(std::cos((double)v)); };
  auto s = [](float v) { return float(std::sin((double)v)); };
  Mat3<float> Rz, Ry, Rx;
  Rz(0, 0) = c(y); Rz(0, 1) = -s(y); Rz(1, 0) = s(y); Rz(1, 1) = c(y); Rz(2, 2) = 1;
  Ry(0, 0) = c(p); Ry(0, 2) = s(p); Ry(1, 1) = 1; Ry(2, 0) = -s(p); Ry(2, 2) = c(p);
  Rx(0, 0) = 1; Rx(1, 1) = c(r); Rx(1, 2) = -s(r); Rx(2, 1) = s(r); Rx(2, 2) = c(r);
  return Rz * Ry * Rx;
}

static Transform tf_of(const float *a) { return Transform(Quat<float>(a[3], a[0], a[1], a[2]), Vec3<float>(a[4], a[5], a[6])); }
static void tf_out(const Transform &t, float *o) {
  o[0] = t.rot.x; o[1] = t.rot.y; o[2] = t.rot.z; o[3] = t.rot.w; o[4] = t.pos.x; o[5] = t.pos.y; o[6] = t.pos.z;
}

struct MapBuilderOracle {
  void *map = nullptr;                   // o_cubemap.cc CubeMap
  int centre[3] = {10, 10, 5};           // laser_cloud_cen_length_ / width_ / height_ after the last re-centring
  Transform sum, bef, aft, tobe;
  StageBConfig cfg;
  float corner_leaf = 0.2f, surf_leaf = 0.4f, map_filter_size = 0.2f;
  bool enable_4d = true;
  int skip_count = 2;
  bool system_init = false;
  int odom_count = 0;
  static constexpr int num_map_frames = 5;
  int map_frame_count = num_map_frames - 1;   // PointMapping's constructor (PointMapping.cc:104): the first frame publishes
  int last_iters = 0, last_gate = 0, last_published = 0;
  size_t last_corner_from_map = 0, last_surf_from_map = 0;
  Cloud surround, full_registered;

  MapBuilderOracle() : map(orc_cm_create()) {}
  ~MapBuilderOracle() { orc_cm_destroy(map); }

  Cloud Cube(size_t index, int which) const {
    Cloud c((size_t)orc_cm_cube_size(map, (long long)index, which));
    if (!c.empty()) orc_cm_cube_copy(map, (long long)index, which, (float *)c.data());
    return c;
  }

  // :55-75.  tobe.rot = rot_diff * sum.rot.normalized() is a Matrix3f (RotationBase's matrix * rotation is the product with
  // toRotationMatrix()) assigned to a Quaternionf: Eigen 3.3 quaternionbase_assign_impl<Other, 3, 3>, restated as
  // Quat::fromRotationMatrix in o_linalg.h (trace branch, else the largest-diagonal branch; no normalisation).
  static void Transform4DAssociateToMap(Transform &tobe, const Transform &bef, const Transform &sum) {
    Transform transform_incre = bef.inverse() * sum;
    Transform full_transform = tobe * transform_incre;
    double y_diff = R2yaw(full_transform.rot.normalized().toRotationMatrix().cast<double>()) -
                    R2yaw(sum.rot.normalized().toRotationMatrix().cast<double>());
    Mat3<float> rot_diff = ypr2R_float(Vec3<float>((float)y_diff, 0.f, 0.f));
    tobe.pos = full_transform.pos;
    tobe.rot = Quat<float>::fromRotationMatrix(rot_diff * sum.rot.normalized().toRotationMatrix());
  }

  static void PointAssociateTobeMapped(const PointXYZI &pi, PointXYZI &po, const Transform &t) {   // PointMapping.cc:316-323
    Vec3<float> v(pi.x - t.pos.x, pi.y - t.pos.y, pi.z - t.pos.z);
    Vec3<float> o = t.rot.conjugate() * v;
    po.x = o.x; po.y = o.y; po.z = o.z; po.intensity = pi.intensity;
  }

  void ProcessMap(const Cloud &corner_last, const Cloud &surf_last, const Cloud &full_cloud, const Transform &transform_sum) {
    sum = transform_sum;
    if (!system_init) { system_init = true; bef = sum; tobe = sum; aft = tobe; }   // :227-232
    if (enable_4d) Transform4DAssociateToMap(tobe, bef, sum);
    else tobe = tobe * (bef.inverse() * sum);                                      // TransformAssociateToMap (PointMapping.cc:755-758)
    Cloud corner_stack, surf_stack;
    PointXYZI point_sel;
    for (const PointXYZI &p : corner_last) { PointAssociateToMap(p, point_sel, tobe); corner_stack.push_back(point_sel); }
    for (const PointXYZI &p : surf_last) { PointAssociateToMap(p, point_sel, tobe); surf_stack.push_back(point_sel); }
    PointXYZI point_on_z_axis;
    point_on_z_axis.x = 0.0f; point_on_z_axis.y = 0.0f; point_on_z_axis.z = 10.0f; point_on_z_axis.intensity = 0.f;
    PointAssociateToMap(point_on_z_axis, point_on_z_axis, tobe);
    // re-centring (:307-419), cube selection (:424-486)
    const float pos3[3] = {tobe.pos.x, tobe.pos.y, tobe.pos.z}, z3[3] = {point_on_z_axis.x, point_on_z_axis.y, point_on_z_axis.z};
    int out6[6];
    orc_cm_recentre(map, pos3, out6);
    centre[0] = out6[3]; centre[1] = out6[4]; centre[2] = out6[5];
    long long valid[125], surround_idx[125];
    int n2[2];
    orc_cm_select(map, pos3, z3, out6, valid, surround_idx, n2);
    // laser_cloud_*_from_map_ (:488-495)
    Cloud corner_from_map, surf_from_map;
    for (int i = 0; i < n2[0]; ++i) {
      Cloud c = Cube((size_t)valid[i], 0), s = Cube((size_t)valid[i], 1);
      corner_from_map.insert(corner_from_map.end(), c.begin(), c.end());
      surf_from_map.insert(surf_from_map.end(), s.begin(), s.end());
    }
    last_corner_from_map = corner_from_map.size(); last_surf_from_map = surf_from_map.size();
    for (PointXYZI &p : corner_stack) PointAssociateTobeMapped(p, p, tobe);
    for (PointXYZI &p : surf_stack) PointAssociateTobeMapped(p, p, tobe);
    Cloud corner_ds, surf_ds;
    VoxelGridFilter(corner_stack, corner_leaf, corner_ds);
    VoxelGridFilter(surf_stack, surf_leaf, surf_ds);
    // :529-544.  OptimizeMap (variant 1) / OptimizeTransformTobeMapped end with the update behind their early return (:625-628, :1013)
    last_iters = 0;
    last_gate = odom_count % skip_count == 0;
    if (last_gate) {
      OptimizeTransformTobeMapped(corner_from_map, surf_from_map, corner_ds, surf_ds, tobe, cfg, &last_iters, nullptr, enable_4d ? 1 : 0);
      if (!(corner_from_map.size() <= 10 || surf_from_map.size() <= 100)) { bef = sum; aft = tobe; }
    } else {
      bef = sum; aft = tobe;   // Transform4DUpdate :77-90 / TransformUpdate
    }
    ++odom_count;
    // UpdateMapDatabase (:546-557) with margin centre == the centre the valid indices were computed with
    float tf7[7];
    tf_out(tobe, tf7);
    orc_cm_update(map, (const float *)corner_ds.data(), (int)corner_ds.size(), (const float *)surf_ds.data(), (int)surf_ds.size(), valid, n2[0],
                  tf7, centre);
    // PublishMapBuilderResults :144-218
    last_published = 0;
    if (++map_frame_count >= num_map_frames) {
      map_frame_count = 0;
      last_published = 1;
      Cloud acc;
      for (int i = 0; i < n2[1]; ++i) {
        Cloud c = Cube((size_t)surround_idx[i], 0), s = Cube((size_t)surround_idx[i], 1);
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
// cfg: {map_filter_size, min_match_sq_dis, min_plane_dis, enable_4d, skip_count, max_iterations}
void *orc_mb_create(const float *cfg6) {
  MapBuilderOracle *m = new MapBuilderOracle();
  m->map_filter_size = cfg6[0]; m->cfg.min_match_sq_dis = cfg6[1]; m->cfg.min_plane_dis = cfg6[2];
  m->enable_4d = cfg6[3] != 0.f; m->skip_count = (int)cfg6[4]; m->cfg.num_max_iterations = (int)cfg6[5];
  return m;
}
void orc_mb_destroy(void *h) { delete (MapBuilderOracle *)h; }
// out: tobe tf7, aft tf7, info6 = {iterations, gate optimised, corner_from_map, surf_from_map, surround published, surround size}
void orc_mb_process(void *h, const float *corner, int nc, const float *surf, int ns, const float *full, int nf, const float *sum7, float *tobe7,
                    float *aft7, int *info6) {
  MapBuilderOracle *m = (MapBuilderOracle *)h;
  Cloud c((const PointXYZI *)corner, (const PointXYZI *)corner + nc), s((const PointXYZI *)surf, (const PointXYZI *)surf + ns),
      f((const PointXYZI *)full, (const PointXYZI *)full + nf);
  m->ProcessMap(c, s, f, tf_of(sum7));
  tf_out(m->tobe, tobe7);
  tf_out(m->aft, aft7);
  info6[0] = m->last_iters; info6[1] = m->last_gate; info6[2] = (int)m->last_corner_from_map; info6[3] = (int)m->last_surf_from_map;
  info6[4] = m->last_published; info6[5] = (int)m->surround.size();
}
// which: 0 surround map (last published), 1 registered full cloud (last frame)
int orc_mb_cloud_size(void *h, int which) {
  MapBuilderOracle *m = (MapBuilderOracle *)h;
  return (int)(which == 0 ? m->surround : m->full_registered).size();
}
void orc_mb_cloud_copy(void *h, int which, float *out) {
  MapBuilderOracle *m = (MapBuilderOracle *)h;
  const Cloud &c = which == 0 ? m->surround : m->full_registered;
  std::memcpy(out, c.data(), sizeof(PointXYZI) * c.size());
}
int orc_mb_cube_size(void *h, long long index, int which) { return orc_cm_cube_size(((MapBuilderOracle *)h)->map, index, which); }
void orc_mb_cube_copy(void *h, long long index, int which, float *out) { orc_cm_cube_copy(((MapBuilderOracle *)h)->map, index, which, out); }
void orc_mb_centre(void *h, int *out3) { std::memcpy(out3, ((MapBuilderOracle *)h)->centre, sizeof(int) * 3); }
// Transform4DAssociateToMap (enable_4d) or TransformAssociateToMap alone on explicit transforms (tf7 each); writes the new tobe
void orc_mb_associate(const float *tobe7, const float *bef7, const float *sum7, int enable_4d, float *out7) {
  Transform tobe = tf_of(tobe7);
  if (enable_4d) MapBuilderOracle::Transform4DAssociateToMap(tobe, tf_of(bef7), tf_of(sum7));
  else tobe = tobe * (tf_of(bef7).inverse() * tf_of(sum7));
  tf_out(tobe, out7);
}
// Quat::fromRotationMatrix (Eigen's Matrix3 -> Quaternion assignment) on a row-major 3 x 3; q = (x, y, z, w)
void orc_matrix_to_quat(const float *m9, float *q4) {
  Mat3<float> M;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) M(i, j) = m9[3 * i + j];
  Quat<float> q = Quat<float>::fromRotationMatrix(M);
  q4[0] = q.x; q4[1] = q.y; q4[2] = q.z; q4[3] = q.w;
}
}
