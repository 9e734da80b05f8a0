"""Opt windows 14..16 on the device solver: the two-CTA cluster form of the tiled Cholesky and of the step kernel
(k_chol_test_x2 / k_step_x2) against LAPACK and against the host controller.  Every case runs twice and must repeat
bit for bit."""
import ctypes as C

import numpy as np
import pytest

from lio_mapping_b200 import _lib
from tests import helpers

pytestmark = pytest.mark.gpu


def _solve_rc(A, b):
    n = A.shape[0]
    x = np.zeros(n)
    ok = C.c_int(-1)
    rc = _lib.lib().lio_dev_cholesky_solve_host(np.ascontiguousarray(A), np.ascontiguousarray(b), n, x, C.byref(ok), None, 0)
    return rc, x, ok.value


def _solve_twice(A, b):
    rc1, x1, ok1 = _solve_rc(A, b)
    rc2, x2, ok2 = _solve_rc(A, b)
    assert rc1 == 0 and rc2 == 0, (rc1, rc2)
    assert ok1 == ok2 and np.array_equal(x1, x2)
    return x1, ok1


def _scaled_spd(n, rng, rows):
    J = rng.normal(size=(rows, n))
    A = J.T @ J
    d = 1.0 / (1.0 + np.sqrt(np.diag(A)))
    return A * d[:, None] * d[None, :]


@pytest.mark.parametrize("n", [217, 224, 231, 232, 246, 253, 261])
def test_cluster_cholesky_vs_lapack(n):
    rng = np.random.default_rng(n)
    A = _scaled_spd(n, rng, 3 * n + 5)
    b = rng.normal(size=n)
    x, ok = _solve_twice(A, b)
    assert ok == 1
    xr = np.linalg.solve(A, b)
    assert np.abs(x - xr).max() <= 1e-10 * max(1.0, np.abs(xr).max()) * np.linalg.cond(A) ** 0.5


def test_cluster_cholesky_ill_conditioned_window_like():
    rng = np.random.default_rng(7)
    n = 246
    s = 10.0 ** rng.uniform(-3, 3.5, n)
    J = rng.normal(size=(4 * n, n)) * s[None, :]
    A = J.T @ J
    d = 1.0 / (1.0 + np.sqrt(np.diag(A)))
    A = A * d[:, None] * d[None, :] + 1e-8 * np.eye(n)
    b = rng.normal(size=n)
    x, ok = _solve_twice(A, b)
    assert ok == 1
    r = A @ x - b
    assert np.abs(r).max() <= 1e-9 * max(1.0, np.abs(b).max(), np.abs(A).max() * np.abs(x).max())


# Tile row 25 (odd) is held by rank 0 itself, tile row 30 (even) by rank 1.  The pivot only turns negative through the
# elimination of the columns before it, i.e. through the off-diagonal tiles of its row.  Its coupling to the later columns is
# chosen so that it vanishes once the leading block is eliminated: the pivot alone then decides definiteness.
@pytest.mark.parametrize("col", [8 * 25 + 3, 8 * 30 + 5])
def test_cluster_cholesky_reports_indefinite(col):
    n = 261
    rng = np.random.default_rng(col)
    A = _scaled_spd(n, rng, 3 * n)
    a = A[col, :col]
    w = np.linalg.solve(A[:col, :col], a)
    A[col, col + 1:] = A[col + 1:, :col] @ w
    A[col + 1:, col] = A[col, col + 1:]
    A[col, col] = a @ w - 1e-3                                     # Schur complement of the leading block: -1e-3
    x, ok = _solve_twice(A, np.ones(n))
    assert ok == 0
    A[col, col] += 2e-3                                           # +1e-3: positive definite again
    _, ok = _solve_twice(A, np.ones(n))
    assert ok == 1


def test_cluster_cholesky_refuses_n_262():
    rc, _, _ = _solve_rc(np.eye(262), np.ones(262))
    assert _lib.STATUS[rc] == "LIO_ERR_INVALID"


# ---- the window solver ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def seq16(oracle):
    return helpers.Sequence(oracle, "vlp16", n_total=20, distort=False)


def _est(seq, oracle, O, **cfg):
    from lio_mapping_b200 import estimator
    cfg = dict(dict(odom_max_iterations=1, opt_extrinsic=0), **cfg)
    e = estimator.Estimator(window_size=O, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
    helpers.warm_start(e, seq, oracle, O, pose_noise=0.01, seed=1,
                       make_pim=lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    return e


def _trace(e):
    """lio_est_solver_trace: the (24, 16) timeline, then the Cholesky profile; all zero under the host controller."""
    return np.concatenate([e.solver_trace().ravel(), e.chol_profile])


_SOLVE_KEYS = ["iterations", "successful", "termination", "initial_cost", "final_cost", "cost_pim", "cost_ppp", "cost_marg",
               "has_prior", "linearizations", "cost_evals", "launches"]


def _solve_summary(e):
    s = e.summary()
    return {k: s[k] for k in _SOLVE_KEYS}


@pytest.mark.parametrize("O", [14, 15, 16])
def test_cluster_device_solver_equals_host_solver(oracle, seq16, O):
    """Warm start as test_device_solver_equals_host_solver; two device contexts (bit-identical) against the host controller."""
    dev = [_est(seq16, oracle, O, device_solver=1) for _ in range(2)]
    host = _est(seq16, oracle, O, device_solver=0)
    for k in range(O, O + 3):
        for e in dev + [host]:
            helpers.feed_scan(e, seq16, k)
        s1, s0 = dev[0].summary(), host.summary()
        assert _solve_summary(dev[0]) == _solve_summary(dev[1]) and np.array_equal(dev[0].states(), dev[1].states()), k
        x1, x0 = dev[0].states(), host.states()
        # The marginalisation prior of scan O first enters the window of scan O + 1; its host / device rounding then moves g by
        # ~1e-8 relative (as much at O = 13, on the one-CTA kernel) while the steps and costs still agree to 1e-9.
        if k <= O + 1:
            assert s1["iterations"] == s0["iterations"] and s1["successful"] == s0["successful"], (k, s1, s0)
            assert abs(s1["initial_cost"] - s0["initial_cost"]) <= 1e-9 * s0["initial_cost"], (k, s1["initial_cost"], s0["initial_cost"])
            assert abs(s1["final_cost"] - s0["final_cost"]) <= 1e-9 * s0["final_cost"], (k, s1["final_cost"], s0["final_cost"])
        if k == O:
            H1, g1, c1 = dev[0].normal_equations()
            H0, g0, c0 = host.normal_equations()
            assert H1.shape == H0.shape
            assert np.abs(H1 - H0).max() <= 1e-9 * np.abs(H0).max()
            assert np.abs(g1 - g0).max() <= 1e-9 * max(1.0, np.abs(g0).max())
            assert abs(c1 - c0) <= 1e-9 * c0
        assert np.abs(x1[:, :3] - x0[:, :3]).max() <= 1e-5 * max(1.0, np.abs(x0[:, :3]).max()), k
        tr = _trace(dev[0])
        assert np.any(tr[:24 * 16] != 0), k                 # the device path ran
        assert not np.any(_trace(host) != 0)


def test_cluster_host_controller_when_asked(oracle, seq16):
    e = _est(seq16, oracle, 15, device_solver=0)
    helpers.feed_scan(e, seq16, 15)
    assert not np.any(_trace(e) != 0)


def test_cluster_solver_graph_equals_stream_launches(oracle, seq16):
    es = [_est(seq16, oracle, 15, solver_graph=g) for g in (1, 0, 1, 0)]
    for k in range(15, 18):
        for e in es:
            helpers.feed_scan(e, seq16, k)
        x = es[0].states()
        for e in es[1:]:
            assert np.array_equal(e.states(), x), k
            assert _solve_summary(e) == _solve_summary(es[0]), k
        assert np.any(_trace(es[1])[:24 * 16] != 0)


def test_cluster_stepwise_equals_process_scan(oracle, seq16):
    O = 15
    runs = []
    for _ in range(2):
        a, b = _est(seq16, oracle, O), _est(seq16, oracle, O)
        for k in range(O, O + 3):
            helpers.feed_scan(a, seq16, k)
            tt, acc, gyr = seq16.imu[k]
            last = seq16.t[k - 1]
            for j in range(len(tt)):
                b.process_imu(tt[j] - last, acc[j], gyr[j], tt[j]); last = tt[j]
            b.open_scan(seq16.less_flat[k])
            pose, sb, ex = b.parameters()
            H, g, cost = b.assemble(pose, sb, ex)
            Ha, ga, ca = a.normal_equations()
            if Ha.shape == H.shape:
                assert np.abs(H - Ha).max() <= 1e-12 * np.abs(Ha).max() and abs(cost - ca) <= 1e-12 * ca
            pose, sb, ex, summ = b.solve(pose, sb, ex)
            b.close_scan(pose, sb, ex)
            sa = a.summary()
            assert summ["iterations"] == sa["iterations"] and summ["final_cost"] == sa["final_cost"]
            assert np.array_equal(b.states(), a.states()), k
        assert np.any(_trace(a)[:24 * 16] != 0)
        runs.append(a.states())
    assert np.array_equal(runs[0], runs[1])


def test_cluster_feature_exchange_pair_equals_single(oracle, seq16):
    import threading
    import torch
    from lio_mapping_b200 import estimator
    O = 15
    cfg = dict(odom_max_iterations=3, prior_factor=1)
    mk = lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    runs = []
    for _ in range(2):
        ref = estimator.Estimator(window_size=O, opt_window_size=O, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
        streams = [torch.cuda.Stream() for _ in range(2)]
        ranks = [estimator.Estimator(stream=streams[r].cuda_stream, window_size=O, opt_window_size=O, max_frame_points=1 << 15,
                                     max_scan_points=1 << 17, **cfg) for r in range(2)]
        for e in [ref] + ranks:
            helpers.warm_start(e, seq16, oracle, O, pose_noise=0.01, seed=1, make_pim=mk)
        torch.cuda.synchronize()
        slabs = [e.feature_slab() for e in ranks]
        for r, e in enumerate(ranks):
            e.set_feature_peers(r, 2, ptrs=slabs)
        errs = []

        def run(r):
            try:
                for k in range(O, O + 3):
                    helpers.feed_scan(ranks[r], seq16, k)
            except Exception as exc:   # pragma: no cover
                errs.append(exc)
        th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
        for t_ in th:
            t_.start()
        for k in range(O, O + 3):
            helpers.feed_scan(ref, seq16, k)
        for t_ in th:
            t_.join(timeout=300)
        assert not errs, errs
        x = ref.states()
        for e in ranks:
            assert np.array_equal(e.states(), x)
            assert e.summary()["iterations"] == ref.summary()["iterations"]
        assert np.any(_trace(ref)[:24 * 16] != 0)
        runs.append(x)
    assert np.array_equal(runs[0], runs[1])
