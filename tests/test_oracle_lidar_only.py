"""The oracle of the estimator with imu_factor = 0 fed /compact_data messages (oracle/o_lidar_only.cc around the unchanged
orc::Estimator): the reference's ordering of pushes, decimation, start-up, inserts and publications (Estimator.cc:430-856), the
start-up states, the state-W overwrite (:1670-1676) against a float64 statement, and the drift of the optimised window."""
import numpy as np
import pytest

from tests import helpers
from tests.test_global_map_gpu import _T, _T_state


class Drive:
    """A drive with its stage-A clouds (less-sharp corner, less-flat surf, cloud_in_rings full), the ground-truth lidar pose relative
    to the first sweep as transform_sum_ (it starts at identity like the odometry's), and the ground-truth body positions."""

    def __init__(self, oracle, kind, n):
        self.seq = seq = helpers.Sequence(oracle, kind, n_total=n)
        self.corner, self.full = [], []
        for sw in seq.raw:
            r = oracle.stage_a(sw, seq.sensor.lower_deg, seq.sensor.upper_deg, seq.sensor.rings)
            self.corner.append(r["less_sharp"]); self.full.append(r["cloud_in_rings"])
        self.max_full = max(f.shape[0] for f in self.full)
        tlb = _T(seq.tf_lb7())
        T0inv = np.linalg.inv(_T_state(seq.state16(0, None)) @ np.linalg.inv(tlb))
        self.sum7, self.gt_p = [], []
        for k in range(n):
            Tb = T0inv @ _T_state(seq.state16(k, None))
            T = Tb @ np.linalg.inv(tlb)
            self.sum7.append(np.r_[helpers.synth.rot_to_quat(T[:3, :3]), T[:3, 3]].astype(np.float32))
            self.gt_p.append(Tb[:3, 3])

    def clouds(self, k):
        return self.corner[k], self.seq.less_flat[k], self.full[k]


def n_messages(W, O, f, n_inited):
    return f * (W + 1) + n_inited


def _R(q):
    x, y, z, w = np.asarray(q, np.float64) / np.linalg.norm(np.asarray(q, np.float64))
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _R_unnorm(q):   # Eigen's toRotationMatrix of a (not re-normalised) quaternion, float64
    x, y, z, w = (float(v) for v in q)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]])


CONFIGS = [
    pytest.param("vlp16", 5, 4, 1, dict(enable_deskew=0, cutoff_deskew=0), id="vlp16-W5O4-f1-no_deskew"),
    pytest.param("vlp16", 4, 4, 2, dict(enable_deskew=0, cutoff_deskew=0), id="vlp16-W4O4-f2-no_deskew"),
    pytest.param("vlp16", 4, 4, 1, dict(cutoff_deskew=0), id="vlp16-W4O4-f1-enable_deskew"),
    pytest.param("hdl64", 5, 4, 2, {}, id="hdl64-W5O4-f2-cutoff_deskew"),
]


@pytest.mark.parametrize("kind,W,O,f,extra", CONFIGS)
def test_oracle_lidar_only_follows_the_reference(oracle, kind, W, O, f, extra):
    from oracle import lidar_only_py as lo
    n_inited = O + 3
    n = n_messages(W, O, f, n_inited)
    drive = Drive(oracle, kind, n)
    e = lo.LidarOnlyEstimator(init_window_factor=f, window_size=W, opt_window_size=O, opt_extrinsic=0, **extra)
    tlb7 = drive.seq.tf_lb7()
    e.set_extrinsic(tlb7)
    laser, pushes, inited = [], 0, 0
    for k in range(n):
        st = e.process_compact(*drive.clouds(k), drive.sum7[k])
        tobe, aft, ins, info = e.map_poses()
        m = k + 1
        if inited == 0:
            # the first W * f messages push nothing but Process work; the (W+1)-th push starts the window
            push = m % f == 0
            assert st["pushed"] == push and info["process_published"] == (m % 5 == 1), k
            assert not info["inserted"] and not info["surround_published"]
            if push:
                pushes += 1
                laser.append(aft.copy())
            assert st["solved"] == (pushes == W + 1) and st["inited"] == st["solved"], k
            assert st["cir_buf_count"] == min(pushes, W), k
            if not st["solved"]:
                continue
            assert m == f * (W + 1)
            # start-up states: trans_li * lb in float, cast to double
            S = e.startup_states()
            assert np.array_equal(S[:, :3], S[:, :3].astype(np.float32).astype(np.float64))
            for i in range(W + 1):
                Tb = _T(laser[i].astype(np.float64)) @ _T(tlb7.astype(np.float64))
                assert np.abs(S[i, :3] - Tb[:3, 3]).max() < 1e-5 * (1 + np.abs(Tb[:3, 3]).max()), i
                assert np.abs(_R(S[i, 3:7]) - Tb[:3, :3]).max() < 1e-6, i
        else:
            assert st["pushed"] and st["solved"] and st["inited"] and st["cir_buf_count"] == W, k
            assert not info["process_published"]
            laser.append(aft.copy())
            i = inited - 1
            # no estimator insert before the (O+1)-th INITED message: the first opt entries are the pre-initialisation frames
            assert info["inserted"] == (i >= O), k
            assert info["surround_published"] == (m % 5 == 1), k
        inited += 1
        # the state-W overwrite against a float64 statement of :1670-1676 on the oracle's own inputs
        P0, R0, inc, Pw, Rw = e.prediction()
        assert np.abs(Pw - (R0 @ inc[4:].astype(np.float64) + P0)).max() < 1e-12 * (1 + np.abs(Pw).max())
        assert np.abs(Rw - R0 @ _R_unnorm(inc[:4])).max() < 1e-12
        Tinc = np.linalg.inv(_T(tlb7)) @ np.linalg.inv(_T(laser[-2].astype(np.float64))) @ _T(laser[-1].astype(np.float64)) @ _T(tlb7)
        assert np.abs(inc[4:] - Tinc[:3, 3]).max() < 1e-5 and np.abs(_R(inc[:4]) - Tinc[:3, :3]).max() < 1e-5
        p2, r2 = lo.predict(laser[-2], laser[-1], tlb7, P0, R0)
        assert np.array_equal(p2, Pw) and np.array_equal(r2, Rw)
    assert inited == n_inited + 1
    # drift of the optimised window against ground truth: logical frame j < W holds message n - W + j
    s = e.states()
    err = np.abs(s[:W, :3] - np.array([drive.gt_p[n - W + j] for j in range(W)])).max()
    assert err < 0.2, err
