"""RunInitialization / ImuInitializer::Initialization (Estimator.cc:858-958, ImuInitializer.cc:35-308, :421-452): the oracle
(o_imu_init.cc) against an independent NumPy float64 statement, the library's host seam (lio_imu_run_initialization_host) against
the oracle, and the three outcomes on synthetic windows.  No GPU needed."""
import numpy as np
import pytest

from lio_mapping_b200 import estimator as E
from oracle import imu_init_py as II

G = 9.805
NOISE = dict(acc_n=0.2, gyr_n=0.02, acc_w=2e-4, gyr_w=2e-5)
TLB = np.array([0, 0, 0, 1, 0.05, -0.02, -0.1], np.float32)   # transform_lb_: x y z w, p


def rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def rot_z(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def quat_of(R):
    w = np.sqrt(max(1e-12, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    return np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])


def R_of_q(q):   # x y z w, Eigen's toRotationMatrix
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def drive(W, k_roll=0.25, k_pitch=0.2, k_acc=1.5, bias_g=(0.01, -0.02, 0.015), tilt=(0.1, -0.05, 0.3), rate=200, step=20):
    """A window of W + 1 laser frames at rate / step Hz: body pose in a gravity-aligned world, laser poses in a lidar world tilted by
    `tilt` (roll, pitch, yaw), IMU samples at `rate` Hz with a constant gyro bias.  Returns laser tf7s, per-frame sample lists and
    the lidar world's gravity."""
    dt = 1.0 / rate
    n = W * step + 1
    t = np.arange(n) * dt

    def pose(tt):
        R = rot_z(0.3 * tt + 0.2 * np.sin(1.3 * tt)) @ rot_y(k_pitch * np.sin(2.1 * tt)) @ rot_x(k_roll * np.sin(2.7 * tt + 0.4))
        p = np.array([2.0 * tt + k_acc * np.sin(1.7 * tt), k_acc * np.cos(1.1 * tt), 0.3 * k_acc * np.sin(2.3 * tt)])
        return R, p

    h = 1e-4
    acc, gyr = [], []
    for tt in t:
        R, p = pose(tt)
        Rp, pp = pose(tt + h)
        Rm, pm = pose(tt - h)
        a_w = (pp - 2 * p + pm) / (h * h)
        dR = (Rp - Rm) / (2 * h)
        Om = R.T @ dR
        w_b = np.array([Om[2, 1] - Om[1, 2], Om[0, 2] - Om[2, 0], Om[1, 0] - Om[0, 1]]) / 2
        acc.append(R.T @ (a_w - np.array([0, 0, -G])))
        gyr.append(w_b + np.asarray(bias_g))
    R_lw = rot_z(tilt[2]) @ rot_y(tilt[1]) @ rot_x(tilt[0])
    R_lb, p_lb = R_of_q(TLB[:4].astype(np.float64)), TLB[4:].astype(np.float64)
    tfs = []
    for k in range(W + 1):
        R, p = pose(t[k * step])
        Rl = R_lw @ R @ R_lb.T   # T_li = T_wi * T_lb^-1 in the lidar world
        pl = R_lw @ p - Rl @ p_lb
        tfs.append(np.concatenate([quat_of(Rl), pl]).astype(np.float32))
    samples = [[] for _ in range(W + 1)]
    for k in range(1, W + 1):
        for s in range((k - 1) * step + 1, k * step + 1):
            samples[k].append((dt, acc[s], gyr[s]))
    first = [(acc[(k - 1) * step] if k else acc[0], gyr[(k - 1) * step] if k else gyr[0]) for k in range(W + 1)]
    return np.array(tfs), samples, first, R_lw @ np.array([0, 0, -G])


def make_pims(cls, samples, first, bgs):
    out = []
    for k, ss in enumerate(samples):
        p = cls(first[k][0], first[k][1], np.zeros(3), bgs[k], g_norm=G, **NOISE)
        for dt, a, g in ss:
            p.push_back(dt, a, g)
        out.append(p)
    return out


def numpy_initializer(tfs, pims, repro, bgs0, g_norm):
    """ImuInitializer::Initialization and the yaw removal of RunInitialization, stated with NumPy (np.linalg.solve for Eigen's LDLT).
    pims: the window's pre-integrations as read before the attempt; repro(bg): the same re-propagated with (0, bg)."""
    W = len(tfs) - 1
    Rq = lambda q: R_of_q(np.asarray(q, np.float64))
    A = np.zeros((3, 3)); b = np.zeros(3)
    for i in range(W):
        q_ij = qmul(tfs[i][:4] * np.array([-1, -1, -1, 1], np.float32), tfs[i + 1][:4]).astype(np.float64)
        d = pims[i + 1]
        dq = d["delta_q"] * np.array([-1, -1, -1, 1])
        J = d["jacobian"][3:6, 12:15]
        A += J.T @ J
        b += J.T @ (2 * qmul(dq, q_ij)[:3])
    bgs = bgs0 + np.linalg.solve(A, b)
    P = repro(bgs[0])
    plb, rlb = TLB[4:].astype(np.float64), Rq(TLB[:4])
    a = 0.0; bv = np.zeros(3)
    for i in range(W - 1):
        dt12, dt23 = P[i + 1]["sum_dt"], P[i + 2]["sum_dt"]
        pl = [tfs[i + k][4:].astype(np.float64) for k in range(3)]
        rl = [Rq(tfs[i + k][:4]) for k in range(3)]
        ta = 0.5 * (dt12 * dt12 * dt23 + dt23 * dt23 * dt12)
        tb = ((pl[1] - pl[0]) * dt23 - (pl[2] - pl[1]) * dt12 + (rl[1] - rl[0]) @ plb * dt23 - (rl[2] - rl[1]) @ plb * dt12
              + rl[1] @ rlb @ P[i + 2]["delta_p"] * dt12 + rl[0] @ rlb @ P[i + 1]["delta_v"] * dt12 * dt23 - rl[0] @ rlb @ P[i + 1]["delta_p"] * dt23)
        a += ta * ta; bv -= ta * tb
    g = bv / a
    approx = g.copy()
    if abs(np.linalg.norm(g) - g_norm) > 1.0:
        return dict(bgs=bgs, g_approx=approx, ok=False)
    n = 3 * (W + 1) + 2
    A = np.zeros((n, n)); b = np.zeros(n)
    g = g / np.linalg.norm(g) * g_norm
    for _ in range(5):
        an = g / np.linalg.norm(g)
        tmp = np.array([0.0, 0, 1]) if not np.array_equal(an, [0, 0, 1]) else np.array([1.0, 0, 0])
        bb = tmp - an * (an @ tmp); bb /= np.linalg.norm(bb)
        lxly = np.stack([bb, np.cross(an, bb)], 1)
        for i in range(W):
            dt = P[i + 1]["sum_dt"]
            pl1, pl2 = tfs[i][4:].astype(np.float64), tfs[i + 1][4:].astype(np.float64)
            n1 = tfs[i][:4] / np.sqrt(np.sum(tfs[i][:4] * tfs[i][:4], dtype=np.float32), dtype=np.float32)
            n2 = tfs[i + 1][:4] / np.sqrt(np.sum(tfs[i + 1][:4] * tfs[i + 1][:4], dtype=np.float32), dtype=np.float32)
            rl1, rl2 = Rq(n1), Rq(n2)
            tA = np.zeros((6, 8)); tb = np.zeros(6)
            tA[:3, :3] = dt * np.eye(3); tA[:3, 6:] = 0.5 * lxly * dt * dt
            tb[:3] = pl2 - pl1 - rl1 @ rlb @ P[i + 1]["delta_p"] - (rl1 - rl2) @ plb - 0.5 * g * dt * dt
            tA[3:, :3] = np.eye(3); tA[3:, 3:6] = -np.eye(3); tA[3:, 6:] = lxly * dt
            tb[3:] = -rl1 @ rlb @ P[i + 1]["delta_v"] - g * dt
            rA, rb = tA.T @ tA, tA.T @ tb
            o = 3 * i
            A[o:o + 6, o:o + 6] += rA[:6, :6]; b[o:o + 6] += rb[:6]
            A[-2:, -2:] += rA[6:, 6:]; b[-2:] += rb[6:]
            A[o:o + 6, -2:] += rA[:6, 6:]; A[-2:, o:o + 6] += rA[6:, :6]
        A *= 1000.0; b *= 1000.0
        x = np.linalg.solve(A, b)
        g = g + lxly @ x[-2:]
        g = g / np.linalg.norm(g) * g_norm
    gI = np.array([0, 0, -1.0]); gW = g / np.linalg.norm(g)
    c = np.cross(gI, gW)
    w = c / np.linalg.norm(c) * np.arctan2(np.linalg.norm(c), gI @ gW)
    th = np.linalg.norm(w)
    q = np.concatenate([np.sin(th / 2) / th * w, [np.cos(th / 2)]])
    R_WI = R_of_q(q)
    return dict(bgs=bgs, g_in_laser=g, R_WI_refined=R_WI, Vs=x[:3 * (W + 1)].reshape(-1, 3), ok=True)


def yaw_removal(R_WI, Rs0, g_in_laser):
    R0 = R_WI.T
    M = R0 @ Rs0
    yaw = np.arctan2(M[1, 0], M[0, 0])
    R0 = rot_z(-yaw) @ R0
    return R0, R0 @ g_in_laser


def _read(pims):
    return [p.get() for p in pims]


def _window(W, **kw):
    tfs, samples, first, g_l = drive(W, **kw)
    return tfs, samples, first, g_l


def _run(mod, tfs, samples, first, g_norm=G, R_WI=np.eye(3), bgs=None):
    W = len(tfs) - 1
    bgs = np.zeros((W + 1, 3)) if bgs is None else bgs
    cls = E.Pim if mod is E else __import__("oracle.oracle_py", fromlist=["Pim"]).Pim
    pims = make_pims(cls, samples, first, bgs)
    before = _read(pims)
    r = mod.run_initialization(tfs, pims, TLB, g_norm, np.zeros((W + 1, 3)), bgs, np.ones((W + 1, 3)), R_WI)
    return r, before, _read(pims)


@pytest.mark.parametrize("W", [5, 7, 10])
def test_oracle_against_numpy(oracle, W):
    from oracle import oracle_py as O
    tfs, samples, first, _ = _window(W)
    r, before, after = _run(II, tfs, samples, first)
    assert r["outcome"] == 2
    repro = lambda bg: _read(make_pims(O.Pim, samples, first, np.tile(bg, (W + 1, 1))))
    ref = numpy_initializer(tfs, before, repro, np.zeros((W + 1, 3)), G)
    assert ref["ok"]
    np.testing.assert_allclose(r["Bgs"], ref["bgs"], rtol=1e-9, atol=1e-12)
    # R0 = ypr2R(-yaw, 0, 0) R_WI^T, with Rs[0] the unrotated laser-to-body pose of frame 0
    Rs0 = r["R_WI"] @ r["Rs"][0]
    R0, g_vec = yaw_removal(ref["R_WI_refined"], Rs0, ref["g_in_laser"])
    np.testing.assert_allclose(r["R_WI"], R0.T, rtol=0, atol=1e-9)
    np.testing.assert_allclose(r["g_vec"], g_vec, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(r["Vs"], ref["Vs"] @ R0.T, rtol=1e-7, atol=1e-8)
    # the pre-integrations end re-propagated with (Bas[i], Bgs[i])
    fresh = _read(make_pims(O.Pim, samples, first, ref["bgs"]))
    for a, f in zip(after, fresh):
        np.testing.assert_allclose(a["delta_p"], f["delta_p"], rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(a["delta_v"], f["delta_v"], rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("W", [5, 7])
def test_seam_equals_oracle(oracle, W):
    tfs, samples, first, _ = _window(W)
    R_prev = rot_x(0.02) @ rot_z(0.4)   # R0 is built from whatever R_WI_ holds
    for g_norm in (G, G + 3.0):
        ro, _, ao = _run(II, tfs, samples, first, g_norm=g_norm, R_WI=R_prev)
        rd, _, ad = _run(E, tfs, samples, first, g_norm=g_norm, R_WI=R_prev)
        assert ro["outcome"] == rd["outcome"] == (2 if g_norm == G else 1)
        for k in ("Ps", "Rs", "Vs", "Bgs", "g_vec", "R_WI"):
            np.testing.assert_allclose(rd[k], ro[k], rtol=1e-12, atol=1e-13, err_msg=k)
        for a, b in zip(ad, ao):
            for k in ("delta_p", "delta_q", "delta_v", "sum_dt", "jacobian", "covariance"):
                np.testing.assert_allclose(a[k], b[k], rtol=1e-12, atol=1e-15, err_msg=k)


def test_low_excitation_changes_nothing(oracle):
    """Outcome 0 returns before any side effect: the C entry is called directly with every in / out array filled with sentinels,
    and none of them, nor the pre-integrations, changes."""
    import ctypes as C
    from lio_mapping_b200 import _lib
    W = 7
    tfs, samples, first, _ = _window(W, k_roll=0.0, k_pitch=0.0, k_acc=0.0)
    bgs0 = np.full((W + 1, 3), 0.003)
    pims = make_pims(E.Pim, samples, first, bgs0)
    before = _read(pims)
    outs = dict(bgs=bgs0.copy(), vs=np.full((W + 1, 3), 7.0), R=np.full(9, 5.0), ps=np.full((W + 1, 3), -3.0), rs=np.full((W + 1, 9), -4.0),
                g=np.full(3, -6.0))
    ref = {k: v.copy() for k, v in outs.items()}
    outcome = C.c_int(-7)
    handles = (C.c_void_p * (W + 1))(*[p.h.value for p in pims])
    rc = _lib.lib().lio_imu_run_initialization_host(W, np.ascontiguousarray(tfs, np.float32), handles, TLB, G, np.zeros((W + 1, 3)),
                                                    outs["bgs"], outs["vs"], outs["R"], outs["ps"], outs["rs"], outs["g"], C.byref(outcome))
    assert rc == 0 and outcome.value == 0
    for k in outs:
        np.testing.assert_array_equal(outs[k], ref[k], err_msg=k)
    for a, b in zip(before, _read(pims)):
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    r, before, after = _run(II, tfs, samples, first, bgs=bgs0)
    assert r["outcome"] == 0
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a["delta_p"], b["delta_p"])


def test_wrong_gravity_norm_keeps_side_effects(oracle):
    W = 7
    tfs, samples, first, _ = _window(W)
    R_prev = rot_z(0.7)
    for mod in (II, E):
        ok, _, _ = _run(mod, tfs, samples, first, R_WI=R_prev)
        r, before, after = _run(mod, tfs, samples, first, g_norm=G + 3.0, R_WI=R_prev)
        assert r["outcome"] == 1
        np.testing.assert_array_equal(r["Bgs"], ok["Bgs"])             # EstimateGyroBias ran
        assert not np.array_equal(r["Vs"], np.ones((W + 1, 3)))        # rotated by R0 ...
        R0 = r["R_WI"].T
        np.testing.assert_allclose(r["Vs"], np.ones((W + 1, 3)) @ R0.T, rtol=1e-12)   # ... but not refined
        # R0 came from the previous R_WI_: ypr2R(-yaw) R_prev^T, so R_WI_ R_prev^T is a pure yaw
        D = r["R_WI"].T @ R_prev.T
        np.testing.assert_allclose(D[2], [0, 0, 1], atol=1e-12)
        for a, b in zip(after, before):
            assert not np.array_equal(a["delta_p"], b["delta_p"]) or a["sum_dt"] == 0


def test_excited_window_recovers_bias_and_gravity(oracle):
    W = 10
    bias = np.array([0.01, -0.02, 0.015])
    tfs, samples, first, g_l = _window(W, bias_g=bias)
    r, _, _ = _run(II, tfs, samples, first)
    assert r["outcome"] == 2
    err_bg = np.abs(r["Bgs"] - bias).max()
    g_in_laser = r["R_WI"] @ r["g_vec"]   # g_vec_ = R0 g_in_laser with R0 = R_WI_^T
    err_g = np.degrees(np.arccos(np.clip(g_in_laser @ g_l / (np.linalg.norm(g_in_laser) * np.linalg.norm(g_l)), -1, 1)))
    print(f"oracle on the synthetic W = {W} drive: gyro bias error {err_bg:.3e} rad/s, gravity direction error {err_g:.3e} deg")
    assert err_bg < 2e-3
    assert err_g < 0.5
    np.testing.assert_allclose(np.linalg.norm(r["g_vec"]), G, rtol=1e-12)
