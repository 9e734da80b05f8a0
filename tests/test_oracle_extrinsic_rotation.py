"""ImuInitializer::EstimateExtrinsicRotation (ImuInitializer.cc:353-419), the calibration of the lidar-IMU extrinsic rotation that the
estimator runs before RunInitialization with estimate_extrinsic = 2: the oracle (o_extrinsic_rotation.cc, one-sided Jacobi SVD of A)
against an independent NumPy statement (numpy.linalg.svd of the same A), and the library's host seam
(lio_imu_estimate_extrinsic_rotation_host, eigen-decomposition of A^T A) against the oracle.  No GPU needed."""
import dataclasses

import numpy as np
import pytest

from lio_mapping_b200 import estimator as E
from lio_mapping_b200 import synth
from oracle import extrinsic_rotation_py as ER

NOISE = dict(acc_n=0.2, gyr_n=0.02, acc_w=2e-4, gyr_w=2e-5, g_norm=9.805)
T_LB = np.array([0.0, 0.0, -0.1])
BIAS = np.array([0.02, -0.03, 0.025])   # rad/s


def rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def rot_z(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


TRUTHS = {"identity": np.eye(3), "rot_x": rot_x(0.15), "general": rot_z(0.4) @ rot_y(-0.2) @ rot_x(0.15)}


def qmul(a, b):
    """Hamilton product, x y z w, evaluated in the dtype of a and b."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def conj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]], q.dtype)


def R_of_q(q):
    """Eigen's toRotationMatrix (no normalisation), in the dtype of q."""
    x, y, z, w = q
    two = q.dtype.type(2)
    one = q.dtype.type(1)
    tx, ty, tz = two * x, two * y, two * z
    return np.array([[one - (ty * y + tz * z), ty * x - tz * w, tz * x + ty * w],
                     [ty * x + tz * w, one - (tx * x + tz * z), tz * y - tx * w],
                     [tz * x - ty * w, tz * y + tx * w, one - (tx * x + ty * y)]], q.dtype)


def window(W, k, R_lb, t0=1.0, spacing=0.2, bias=np.zeros(3), kick=None):
    """W + 1 pushes of the HDL-64 drive with roll / pitch amplitude k, spacing s apart: the laser tf7s (T_l = T_b T_lb^-1), and per
    frame the IMU samples (dt, acc, gyr + bias) since the previous push with the first sample of its pre-integration.  kick = (frame,
    rotation): that frame's laser rotation is turned further, so that its two pairs disagree with the IMU."""
    _, _, traj = synth.default_config("hdl64")
    traj = dataclasses.replace(traj, k_roll=k, k_pitch=k)
    t = t0 + spacing * np.arange(W + 1)
    p, R, _, gyro, acc = traj.state(t)
    tfs = []
    for i in range(W + 1):
        Rl = R[i] @ R_lb.T
        if kick is not None and kick[0] == i:
            Rl = Rl @ kick[1]
        pl = p[i] - Rl @ T_LB
        tfs.append(np.r_[synth.rot_to_quat(Rl), pl].astype(np.float32))
    frames = [None]
    for i in range(1, W + 1):
        tt, a, g = synth.make_imu(traj, float(t[i - 1]), float(t[i]), 200.0)
        last, ss = t[i - 1], []
        for j in range(len(tt)):
            ss.append((tt[j] - last, a[j], g[j] + bias))
            last = tt[j]
        frames.append(((acc[i - 1], gyro[i - 1] + bias), ss))
    return np.array(tfs), frames


def make_pims(cls, frames):
    out = [cls(np.zeros(3), np.zeros(3), np.zeros(3), np.zeros(3), **NOISE)]   # frame 0's is never read
    for first, ss in frames[1:]:
        p = cls(first[0], first[1], np.zeros(3), np.zeros(3), **NOISE)
        for dt, a, g in ss:
            p.push_back(dt, a, g)
        out.append(p)
    return out


def numpy_statement(tfs, dqs, tlb7):
    """The same calibration stated with NumPy: A block by block, numpy.linalg.svd, x = V's last column."""
    W = len(tfs) - 1
    # transform_lb.inverse(): the float rotation matrix transposed, back to a quaternion (Shepperd) - the inverse rotation
    q_lb = tlb7[:4].astype(np.float64)
    rot_bl = conj(q_lb / np.linalg.norm(q_lb))
    A = np.zeros((4 * W, 4))
    for i in range(W):
        q_imu = dqs[i + 1]
        q_laser = qmul(conj(tfs[i][:4]), tfs[i + 1][:4]).astype(np.float64)
        q_from_imu = qmul(qmul(conj(rot_bl), q_imu), rot_bl)
        d = qmul(q_laser, conj(q_from_imu))
        deg = np.degrees(2 * np.arctan2(np.linalg.norm(d[:3]), abs(d[3])))
        huber = 5.0 / deg if deg > 5.0 else 1.0

        def skew(v):
            return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])

        def border(q, top):   # LeftQuatMatrix / RightQuatMatrix (math_utils.h:140-161)
            m = np.zeros((4, 4))
            m[:3, :3] = top
            m[3, :3] = -q[:3]; m[:3, 3] = q[:3]; m[3, 3] = q[3]
            return m
        left = border(q_laser, q_laser[3] * np.eye(3) + skew(q_laser[:3]))
        right = border(q_imu, q_imu[3] * np.eye(3) - skew(q_imu[:3]))
        A[4 * i:4 * i + 4] = huber * (left - right)
    _, s, Vt = np.linalg.svd(A)
    x = Vt[3]
    return s, x, bool(s[2] > 0.25)


def _rot(q):
    q = np.asarray(q, np.float64)
    return R_of_q(q / np.linalg.norm(q))


def _dqs(pims):
    return [None] + [p.get()["delta_q"] for p in pims[1:]]


def _determined(sv):
    """x is V's column of the smallest singular value: a rotation is defined only where that one is apart from the next (a yaw-only
    window has two zero singular values, and any unit vector of their plane is a solution)."""
    return sv[2] - sv[3] > 1e-4


def _check_oracle(tfs, frames, tlb7):
    from oracle import oracle_py as O
    pims = make_pims(O.Pim, frames)
    ok, t_out, sv = ER.estimate_extrinsic_rotation(tfs, pims, tlb7)
    s_ref, x, ok_ref = numpy_statement(tfs, _dqs(pims), tlb7)
    np.testing.assert_allclose(sv, s_ref, rtol=1e-10, atol=1e-7)
    assert ok == ok_ref
    if _determined(s_ref):
        np.testing.assert_allclose(_rot(t_out[:4]), _rot(x), rtol=0, atol=1e-6)
    np.testing.assert_array_equal(t_out[4:], tlb7[4:])
    return ok, t_out, sv


def _check_seam(tfs, frames, tlb7):
    from oracle import oracle_py as O
    ok_o, t_o, sv_o = ER.estimate_extrinsic_rotation(tfs, make_pims(O.Pim, frames), tlb7)
    ok_d, t_d, sv_d = E.estimate_extrinsic_rotation(tfs, make_pims(E.Pim, frames), tlb7)
    assert ok_d == ok_o
    np.testing.assert_allclose(sv_d, sv_o, rtol=1e-10, atol=1e-7)
    qd, qo = t_d[:4], t_o[:4] * (1 if np.dot(t_d[:4], t_o[:4]) >= 0 else -1)
    assert not _determined(sv_o) or np.all(np.abs(qd - qo) <= 2 * np.spacing(np.maximum(np.abs(qd), np.abs(qo)))), (qd, qo)   # 2 ulp per coefficient
    np.testing.assert_array_equal(t_d[4:], tlb7[4:])
    return ok_d, t_d, sv_d


GUESS = np.r_[0.0, 0.0, 0.0, 1.0, T_LB].astype(np.float32)   # the identity rotation the indoor configuration starts from


@pytest.mark.parametrize("W", [5, 7, 12])
@pytest.mark.parametrize("truth", list(TRUTHS))
def test_oracle_and_seam_on_excited_windows(oracle, W, truth):
    """k = 0.75 at W 5, 7 and 12: noise-free inputs are calibrated to the truth; both implementations agree with the NumPy statement."""
    tfs, frames = window(W, 0.75, TRUTHS[truth])
    ok, t_out, sv = _check_oracle(tfs, frames, GUESS)
    _check_seam(tfs, frames, GUESS)
    err = np.degrees(np.arccos(np.clip((np.trace(_rot(t_out[:4]).T @ TRUTHS[truth]) - 1) / 2, -1, 1)))
    print(f"W={W} truth={truth}: singular values {np.array2string(sv, precision=4)}, ok={ok}, error {err:.2e} deg")
    if ok:
        assert err < 0.05


@pytest.mark.parametrize("k,expect", [(0.25, False), (0.75, True)], ids=["k0.25-fails", "k0.75-succeeds"])
def test_drive_windows(oracle, k, expect):
    """W 12 windows of pushes 0.2 s apart (init_window_factor 2), truth rot_x(0.15), with and without the test gyro bias: k = 0.25 stays
    below the 0.25 threshold on sigma_2, k = 0.75 passes it."""
    for bias in (np.zeros(3), BIAS):
        tfs, frames = window(12, k, rot_x(0.15), bias=bias)
        ok, t_out, sv = _check_oracle(tfs, frames, GUESS)
        _check_seam(tfs, frames, GUESS)
        err = np.degrees(np.arccos(np.clip((np.trace(_rot(t_out[:4]).T @ rot_x(0.15)) - 1) / 2, -1, 1)))
        print(f"k={k} bias={bias.any()}: singular values {np.array2string(sv, precision=4)}, ok={ok}, error {err:.3f} deg")
        assert ok == expect


def test_yaw_only_window_fails(oracle):
    """Rotations about one axis leave two directions of the quaternion unobserved: sigma_2 is about zero."""
    tfs, frames = window(7, 0.0, rot_x(0.15))
    ok, _, sv = _check_oracle(tfs, frames, GUESS)
    _check_seam(tfs, frames, GUESS)
    assert not ok and sv[2] < 1e-3, sv


def test_huber_branch(oracle):
    """One laser pose turned 8.6 degrees further: its two pairs are more than 5 degrees from the IMU and are down-weighted."""
    tfs, frames = window(7, 0.75, rot_x(0.15), kick=(3, rot_y(0.15)))
    from oracle import oracle_py as O
    pims = make_pims(O.Pim, frames)
    dqs = _dqs(pims)
    degs = []
    for i in range(7):
        q_laser = qmul(conj(tfs[i][:4]), tfs[i + 1][:4]).astype(np.float64)
        d = qmul(q_laser, conj(dqs[i + 1]))
        degs.append(np.degrees(2 * np.arctan2(np.linalg.norm(d[:3]), abs(d[3]))))
    assert sum(x > 5.0 for x in degs) == 2, degs
    _check_oracle(tfs, frames, GUESS)
    _check_seam(tfs, frames, GUESS)


def test_failure_overwrites_the_rotation(oracle):
    """A failed call still replaces the rotation (the reference assigns transform_lb.rot before the test); the position never moves."""
    from oracle import oracle_py as O
    tfs, frames = window(12, 0.25, rot_x(0.15))
    guess = np.r_[synth.rot_to_quat(rot_z(0.3)), 0.05, -0.02, -0.1].astype(np.float32)
    for mod, cls in ((E, E.Pim), (ER, O.Pim)):
        ok, t_out, _ = mod.estimate_extrinsic_rotation(tfs, make_pims(cls, frames), guess)
        assert not ok
        assert not np.array_equal(t_out[:4], guess[:4])
        np.testing.assert_array_equal(t_out[4:], guess[4:])


def test_seam_refusals():
    from lio_mapping_b200 import _lib
    import ctypes as C
    tfs, frames = window(5, 0.75, np.eye(3))
    pims = make_pims(E.Pim, frames)
    sv, ok, t = np.zeros(4), C.c_int(-1), GUESS.copy()
    handles = (C.c_void_p * 6)(*[p.h.value for p in pims])
    assert _lib.lib().lio_imu_estimate_extrinsic_rotation_host(0, tfs, handles, t, sv, C.byref(ok)) == -2
    handles[2] = None
    assert _lib.lib().lio_imu_estimate_extrinsic_rotation_host(5, tfs, handles, t, sv, C.byref(ok)) == -2
    np.testing.assert_array_equal(t, GUESS)
