"""The node's odometry topics without a device: the float64 restatement of the lidar poses that ProcessLaserOdom publishes
(Estimator.cc:725-758), which tests/test_lio_node_odometry_gpu.py holds /predict_laser_odom and /local_laser_odom to, pinned here against
scipy.spatial.transform.Rotation; and write_tum's file layout."""
import numpy as np
from scipy.spatial.transform import Rotation

from lio_mapping_b200.node import TOPICS, write_tum


def quat_from_matrix(m):
    """Eigen::Quaterniond(const Matrix3d &) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl): the trace branch, else the
    largest diagonal entry.  Returns x y z w."""
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if t > 0:
        t = np.sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        return np.array([(m[2, 1] - m[1, 2]) * t, (m[0, 2] - m[2, 0]) * t, (m[1, 0] - m[0, 1]) * t, w])
    i = 0
    if m[1, 1] > m[0, 0]:
        i = 1
    if m[2, 2] > m[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    t = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
    q = np.zeros(4)
    q[i] = 0.5 * t
    t = 0.5 / t
    q[3] = (m[k, j] - m[j, k]) * t
    q[j] = (m[j, i] + m[i, j]) * t
    q[k] = (m[k, i] + m[i, k]) * t
    return q


def quat_to_matrix(q):
    """QuaternionBase::toRotationMatrix of x y z w."""
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def quat_rotate(q, v):
    """Quaternion * Vector3 (Eigen's _transformVector): uv = 2 q.vec x v, v + w uv + q.vec x uv."""
    u = np.cross(q[:3], v)
    u = u + u
    return v + q[3] * u + np.cross(q[:3], u)


def quat_inverse(q):
    n2 = q @ q
    return np.array([-q[0] / n2, -q[1] / n2, -q[2] / n2, q[3] / n2])


def lidar_pose(P, R, tlb7):
    """Estimator.cc:729-733 (/local_laser_odom at the pivot) and :746-750 (/predict_laser_odom at W): transform_lb =
    transform_lb_.cast<double>(), rot = Quaterniond(R * transform_lb.rot.inverse()), pos = P - rot * transform_lb.pos.  tlb7 is
    transform_lb_ (float32, widened exactly) or any float64 tf7; returns tf7 float64."""
    lb = np.asarray(tlb7).astype(np.float64)
    rot = quat_from_matrix(np.asarray(R, np.float64) @ quat_to_matrix(quat_inverse(lb[:4])))
    return np.r_[rot, np.asarray(P, np.float64) - quat_rotate(rot, lb[4:])]


def _rotations():
    """Random rotations plus the ones that take each branch of quat_from_matrix: angles near pi about each axis (trace <= 0)."""
    rng = np.random.default_rng(7)
    out = list(Rotation.random(200, random_state=11))
    for axis in np.eye(3):
        for a in (np.pi, np.pi - 1e-3, 0.75 * np.pi, 2.2):
            out.append(Rotation.from_rotvec(a * (axis + 0.05 * rng.standard_normal(3))))
    return out


def _same_sign(q, ref):
    return q if q @ ref >= 0 else -q


def test_quaternion_restatement_against_scipy():
    """quat_from_matrix, quat_to_matrix and quat_rotate against Rotation, every branch of quat_from_matrix taken."""
    rng = np.random.default_rng(3)
    branches = set()
    for r in _rotations():
        m = r.as_matrix()
        q = quat_from_matrix(m)
        tr = np.trace(m)
        branches.add(-1 if tr > 0 else int(np.argmax(np.diag(m))))
        assert abs(np.linalg.norm(q) - 1) < 1e-14
        assert np.abs(_same_sign(q, r.as_quat()) - r.as_quat()).max() < 1e-14
        assert np.abs(quat_to_matrix(r.as_quat()) - m).max() < 1e-14
        v = rng.standard_normal(3) * 50
        assert np.abs(quat_rotate(r.as_quat(), v) - r.apply(v)).max() < 1e-12
    assert branches == {-1, 0, 1, 2}


def test_lidar_pose_restatement_against_scipy():
    """lidar_pose against the same composition in Rotation: R_l = R_b * R_lb^-1, p_l = P - R_l p_lb.  The extrinsic's quaternion is
    a unit one in float64 here: Rotation normalises a quaternion, Eigen does not, so a float32 one would differ by its rounding."""
    rng = np.random.default_rng(5)
    for r in _rotations():
        lb = Rotation.random(random_state=int(rng.integers(1 << 30)))
        tlb7 = np.r_[lb.as_quat(), rng.standard_normal(3)]
        P = rng.standard_normal(3) * 100
        got = lidar_pose(P, r.as_matrix(), tlb7)
        want = r * lb.inv()
        assert np.abs(_same_sign(got[:4], want.as_quat()) - want.as_quat()).max() < 1e-13
        assert np.abs(got[4:] - (P - want.apply(tlb7[4:]))).max() < 1e-12


def test_write_tum_round_trip(tmp_path):
    """stamp tx ty tz qx qy qz qw per line, read back by np.loadtxt at full precision of the stamps used by a drive."""
    rng = np.random.default_rng(9)
    stamp = 1.0 + 0.1 * np.arange(12)
    q = Rotation.random(12, random_state=2).as_quat()
    p = rng.standard_normal((12, 3)) * 20
    tf7 = np.column_stack([q, p])
    path = tmp_path / "traj.tum"
    write_tum(path, stamp, tf7)
    back = np.loadtxt(path)
    assert back.shape == (12, 8)
    assert np.abs(back[:, 0] - stamp).max() < 1e-9
    assert np.abs(back[:, 1:4] - p).max() < 1e-8      # tx ty tz
    assert np.abs(back[:, 4:8] - q).max() < 1e-8      # qx qy qz qw
    write_tum(tmp_path / "empty.tum", np.zeros(0), np.zeros((0, 7)))
    assert (tmp_path / "empty.tum").read_text() == ""


def test_topic_ids():
    """The ids of include/lio_b200.h's LIO_NODE_ODOM_* enum, in its order."""
    assert TOPICS == {"/laser_odom_to_init": 0, "/aft_mapped_to_init": 1, "/predict_odom": 2, "/predict_laser_odom": 3,
                      "/local_laser_odom": 4, "/extrinsic_lb": 5}
