"""The oracle's restatement of the estimator's global cube map after initialisation (oracle/o_global_map.cc) on the CPU: the split
scan equals orc::Estimator's own ProcessScan, no insert on the first O scans, the clouds the aliased opt_*_stack_ entries hold at
the insert, the prediction against float64, and PublishResults' count carrying on from the pre-initialisation calls."""
import numpy as np
import pytest

from tests import helpers


def _quat_R(q):
    x, y, z, w = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _T(tf7):
    T = np.eye(4)
    T[:3, :3] = _quat_R(tf7[:4]); T[:3, 3] = np.asarray(tf7[4:], np.float64)
    return T


def _T_state(s16):
    return _T(np.r_[s16[3:7], s16[0:3]])


class _Staging:
    def __init__(self, est, clouds):
        self.est, self.clouds = est, clouds

    def __getattr__(self, name):
        return getattr(self.est, name)

    def init_frame(self, k, *args):
        self.est.set_scan_clouds(*self.clouds(k))
        self.est.init_frame(k, *args)


def pre_init_sum7(seq, k):
    """The ground-truth lidar pose of sweep k, fed to the pre-initialisation mapper as /laser_odom_to_init."""
    T = _T_state(seq.state16(k, None)) @ np.linalg.inv(_T(seq.tf_lb7()))
    return np.r_[helpers.synth.rot_to_quat(T[:3, :3]), T[:3, 3]].astype(np.float32)


CONFIGS = [
    pytest.param(4, 3, {}, id="W4O3-cutoff_deskew"),
    pytest.param(3, 3, {}, id="W3O3-cutoff_deskew"),
    pytest.param(4, 3, dict(cutoff_deskew=0), id="W4O3-enable_deskew"),
    pytest.param(3, 3, dict(cutoff_deskew=0), id="W3O3-enable_deskew"),
    pytest.param(4, 3, dict(enable_deskew=0, cutoff_deskew=0), id="W4O3-no_deskew"),
    pytest.param(3, 3, dict(enable_deskew=0, cutoff_deskew=0), id="W3O3-no_deskew"),
]


@pytest.mark.parametrize("W,O,extra", CONFIGS)
def test_global_map_oracle(oracle, W, O, extra):
    """VLP-16, O + 4 scans after the warm start, beside an unchanged LocalCloudsEstimator on the same inputs:
    - the estimator inside the restatement ends every scan in the same state, bit for bit (its ProcessScan is split, not changed);
    - no insert on the first O scans, then one per scan;
    - with a de-skew flag the insert takes the PREVIOUS frame's clouds: for W > O its surf slot as SlideWindow accumulated it (more
      points than its own cloud), for W == O its own cloud (it has left the window); without de-skew the frame's own accumulated
      slot; the corner cloud is the one pushed for that frame (the /local corner cloud it was published with);
    - tobe follows tobe * lb * (prev^-1 * curr) * lb^-1 within float rounding of a float64 restatement;
    - the surround map on calls 1, 6, 11, ... counting the W pre-initialisation calls, /cloud_registered bit-equal to
      PointAssociateToMap of the raw staged full cloud, aft frozen."""
    from oracle import global_map_py as gm
    from oracle import local_clouds_py as lc
    from oracle import pm_publish_py as pmp
    cfg = dict(window_size=W, opt_window_size=O, opt_extrinsic=0, **extra)
    seq = helpers.Sequence(oracle, "vlp16", n_total=W + O + 4)
    st_a = [oracle.stage_a(sw, seq.sensor.lower_deg, seq.sensor.upper_deg, seq.sensor.rings) for sw in seq.raw]
    corner = [r["less_sharp"] for r in st_a]
    full = [r["cloud_in_rings"] for r in st_a]
    corner_ds = [oracle.voxel_grid(c, 0.2) for c in corner]
    g = gm.GlobalMapEstimator(corner_filter_size=0.2, **cfg)
    ref = lc.LocalCloudsEstimator(corner_filter_size=0.2, **cfg)
    for k in range(W):
        g.pre_init_process(corner[k], seq.less_flat[k], full[k], pre_init_sum7(seq, k))
    for e in (g, ref):
        helpers.warm_start(_Staging(e, lambda k: (corner_ds[k], full[k])), seq, oracle, W, pose_noise=0.01, seed=1,
                           make_pim=lambda a, g_: oracle.Pim(a, g_, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    tobe, aft0, _, _ = g.map_poses()
    deskew = bool(extra.get("enable_deskew", 1) or extra.get("cutoff_deskew", 1))
    pivot = W - O
    pub_corner = {f: corner_ds[f] for f in range(W)}   # warm-start corner clouds are stored as staged
    pub_surf = {f: oracle.voxel_grid(seq.less_flat[f], 0.4) for f in range(W)}   # each frame's own surf cloud
    tlb = seq.tf_lb7().astype(np.float64)
    n_inserts = 0
    for i in range(O + 4):
        k = W + i
        for e in (g, ref):
            e.set_scan_clouds(corner[k], full[k])
        st_before = None
        for e in (g, ref):
            tt, acc, gyr = seq.imu[k]
            last = seq.t[k - 1]
            for j in range(len(tt)):
                e.process_imu(tt[j] - last, acc[j], gyr[j], tt[j])
                last = tt[j]
            if st_before is None:
                st_before = e.states()
            e.process_scan(seq.less_flat[k])
        assert np.array_equal(g.states(), ref.states()), i
        for q in range(W + 1):
            assert np.array_equal(g.frame(q), ref.frame(q)), (i, q)
        pub = ref.local_clouds()
        pub_corner[i + pivot + 1] = pub["corner"]
        pub_surf[i + pivot + 1] = pub["surf"]
        tobe_prev = tobe.astype(np.float64)
        tobe, aft, ins, info = g.map_poses()
        # prediction
        d = np.linalg.inv(_T_state(st_before[W - 1])) @ _T_state(st_before[W])
        want = _T(tobe_prev) @ _T(tlb) @ d @ np.linalg.inv(_T(tlb))
        got = _T(tobe.astype(np.float64))
        assert np.abs(got[:3, :3] - want[:3, :3]).max() < 1e-5 and np.abs(got[:3, 3] - want[:3, 3]).max() < 1e-5 * (1 + np.abs(want[:3, 3]).max()), i
        assert np.array_equal(tobe, gm.predict(tobe_prev.astype(np.float32), st_before[W - 1], st_before[W], seq.tf_lb7()))
        assert np.array_equal(aft, aft0)
        # the insert
        assert info["inserted"] == (i >= O), i
        if info["inserted"]:
            n_inserts += 1
            f = i + pivot - 1 if deskew else i + pivot    # frame id: warm-start frames 0..W-1, scan i is frame W + i
            own = pub_surf[f]
            if deskew and pivot == 0:
                assert np.array_equal(g.cloud("surf"), own), i
            else:
                slot = g.frame(pivot - 1 if deskew else pivot)
                assert np.array_equal(g.cloud("surf"), slot), i
                if pivot > 0 and f >= W - pivot:          # accumulated: the own cloud at the end, pivot clouds before it
                    assert slot.shape[0] > own.shape[0] and np.array_equal(slot[-own.shape[0]:], own), i
            assert np.array_equal(g.cloud("corner"), pub_corner[f]), i
            assert info["points"] == g.cloud("corner").shape[0] + g.cloud("surf").shape[0]
        # publication
        assert info["surround_published"] == ((W + i + 1) % 5 == 1), i
        assert np.array_equal(g.cloud("registered"), pmp.associate_to_map(full[k], tobe)), i
    assert n_inserts == 4
