"""Stages B+C+D parity through the C-ABI: product estimator vs the CPU oracle on the same synthetic
scans + IMU.  Exact where the data are fp32 / index sets, stated tolerances where fp64 is summed."""
import numpy as np
import pytest

from lio_mapping_b200 import synth
from tests import helpers

pytestmark = pytest.mark.gpu


def rand_pose(rng, scale=5.0):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    return np.concatenate([rng.uniform(-scale, scale, 3), q])


def test_ppp_rows_device_vs_oracle(oracle):
    """a10: per-factor residual + 1x18 Jacobian row from the kernel's rank-6 form vs PivotPointPlaneFactor::Evaluate."""
    from lio_mapping_b200 import estimator
    rng = np.random.default_rng(4)
    x0, xi, xe = rand_pose(rng, 30), rand_pose(rng, 30), rand_pose(rng, 0.5)
    n = 500
    pts = np.concatenate([rng.uniform(-50, 50, (n, 3)), rng.uniform(0, 1, (n, 1))], 1).astype(np.float32)
    w = rng.normal(size=(n, 3)); w /= np.linalg.norm(w, axis=1, keepdims=True)
    coef = np.concatenate([w * rng.uniform(0.1, 1, (n, 1)), rng.normal(0, 5, (n, 1))], 1).astype(np.float32)
    r, J = estimator.ppp_evaluate_batch(pts, coef, x0, xi, xe)
    for k in range(n):
        ro, Jo = oracle.ppp_evaluate(pts[k, :3].astype(np.float64), coef[k].astype(np.float64), x0, xi, xe)
        Jo = np.concatenate([j[:6] for j in Jo])
        assert abs(r[k] - ro) <= 1e-12 * max(1.0, abs(ro), np.abs(pts[k, :3]).max())
        assert np.abs(J[k] - Jo).max() <= 1e-12 * max(1.0, np.abs(Jo).max())


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 5000, 300001])
def test_asm_ppp_kernel_vs_numpy(n):
    """The fused reduction (28 sym entries + cost) vs a float64 numpy statement of the same sums."""
    from lio_mapping_b200 import estimator
    from tests.test_shard_gloo import s_blocks
    rng = np.random.default_rng(n)
    p = rng.uniform(-60, 60, (n, 4)).astype(np.float32)
    w = rng.normal(size=(n, 3)); w /= np.maximum(np.linalg.norm(w, axis=1, keepdims=True), 1e-9)
    c = np.concatenate([w * rng.uniform(0.2, 1, (n, 1)), rng.normal(0, 0.3, (n, 1))], 1).astype(np.float32)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    R = synth.quat_to_rot(q); t = rng.normal(size=3)
    S, cost = estimator.asm_ppp(p, c, R, t)
    Sr, cr = s_blocks((p.astype(np.float64), c.astype(np.float64)), R, t)
    assert np.abs(S - Sr).max() <= 1e-11 * max(1.0, np.abs(Sr).max())
    assert abs(cost - cr) <= 1e-11 * max(1.0, cr)


def test_asm_ppp_product_fold_and_large_residuals():
    """The cost is accumulated as a per-thread running product of (1 + r^2) that is folded into a log every few stages;
    residuals with r^2 >= 1/16 bypass the product.  Force one fold per stage and mix both regimes."""
    from lio_mapping_b200 import estimator, synth, _lib
    from tests.test_shard_gloo import s_blocks
    rng = np.random.default_rng(11)
    n = 1500000                                            # 6 stages per tile on 132 SMs: several folds per thread
    p = rng.uniform(-30, 30, (n, 4)).astype(np.float32)
    w = rng.normal(size=(n, 3)); w /= np.linalg.norm(w, axis=1, keepdims=True)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    R = synth.quat_to_rot(q); t = rng.normal(size=3)
    a = w @ R                                              # rows: R^T w
    r_target = np.where(rng.uniform(size=n) < 0.9, rng.normal(0, 0.03, n), rng.normal(0, 3.0, n))   # 10 % outliers
    b = r_target - np.einsum("ij,ij->i", a, p[:, :3].astype(np.float64) + t)
    c = np.concatenate([w, b[:, None]], 1).astype(np.float32)
    Sr, cr = s_blocks((p.astype(np.float64), c.astype(np.float64)), R, t)
    try:
        for fold in (1, 2, 1024):
            _lib.check(_lib.lib().lio_asm_set_fold_chunks(fold), "fold")
            S, cost = estimator.asm_ppp(p, c, R, t)
            assert np.abs(S - Sr).max() <= 1e-11 * max(1.0, np.abs(Sr).max())
            assert abs(cost - cr) <= 1e-11 * max(1.0, cr), (fold, cost, cr)
    finally:
        _lib.lib().lio_asm_set_fold_chunks(1024)


@pytest.fixture(scope="module")
def vlp_seq(oracle):
    return helpers.Sequence(oracle, "vlp16", n_total=10, distort=False)


def _mk(oracle, seq, W, gpu_extra=None, **cfg):
    from lio_mapping_b200 import estimator
    eo = oracle.Estimator(window_size=W, opt_window_size=W, **cfg)
    eg = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17,
                             **dict(cfg, **(gpu_extra or {})))
    helpers.warm_start(eo, seq, oracle, W, pose_noise=0.01, seed=1,
                       make_pim=lambda a, g: oracle.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    helpers.warm_start(eg, seq, oracle, W, pose_noise=0.01, seed=1,
                       make_pim=lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    return eo, eg


@pytest.mark.parametrize("device_solver", [1, 0])
def test_window_solve_parity_exact_features(oracle, vlp_seq, device_solver):
    """odom_max_iterations = 1 keeps the newest frame's features a pure CalculateFeatures call, so the
    whole fp32 front of the solve is bit-identical and the fp64 normal equations agree to round-off.
    Run with the GPU-resident dogleg loop (default) and with the host controller."""
    W = 5
    eo, eg = _mk(oracle, vlp_seq, W, gpu_extra=dict(device_solver=device_solver), odom_max_iterations=1, opt_extrinsic=0)
    for k in range(W, 10):
        helpers.feed_scan(eo, vlp_seq, k)
        helpers.feed_scan(eg, vlp_seq, k)
        so, sg = eo.summary(), eg.summary()
        if k == W:   # first solve: identical inputs by construction
            assert np.array_equal(eg.local_map(), eo.local_map())
            for f in range(1, W + 1):
                # SlideWindow already ran: features are stored per pre-slide frame index
                po, co, io = eo.features(f)
                pg, cg, ig = eg.features(f)
                assert np.array_equal(ig, io) and np.array_equal(cg, co) and np.array_equal(pg, po), f
            Ho, go = eo.normal_equations()
            Hg, gg, cg0 = eg.normal_equations()
            assert Hg.shape == Ho.shape
            assert np.abs(Hg - Ho).max() <= 1e-9 * np.abs(Ho).max()
            assert np.abs(gg - go).max() <= 1e-9 * max(1.0, np.abs(go).max())
            assert abs(sg["initial_cost"] - so["initial_cost"]) <= 1e-9 * so["initial_cost"]
        assert sg["map_size"] == so["map_size"]
        assert abs(sg["num_features"] - so["num_features"]) <= 0.001 * so["num_features"]
        assert sg["iterations"] == so["iterations"]
        xo, xg = eo.states(), eg.states()
        scale = max(1.0, np.abs(xo[:, :3]).max())
        if k <= W + 1:
            # no prior yet in the problem: both sides solve the same well-posed system -> round-off agreement
            assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-9 * so["final_cost"]
            assert np.abs(xg[:, :3] - xo[:, :3]).max() <= 1e-9 * scale
            assert np.abs(xg[:, 3:7] - xo[:, 3:7]).max() <= 1e-10
        if k == W + 1:
            # first marginalisation (Schur complement + eigen square root) from identical inputs.  The information
            # matrix has entries ~1e13 (gyro-bias random walk), i.e. an absolute noise floor ~1e-3 in its spectrum.
            Hg_p, bg_p = eg.prior()
            Ho_p, bo_p = eo.prior_canonical(W)
            assert Hg_p.shape == Ho_p.shape
            # (Schur complement A_rr - A_rm A_mm^+ A_mr cancels ~1e13-sized terms: ~1e-3 absolute / 1e-7 relative noise)
            assert np.abs(Hg_p - Ho_p).max() <= 1e-6 * np.abs(Ho_p).max()
            assert np.abs(bg_p - bo_p).max() <= 1e-5 * max(1.0, np.abs(bo_p).max())
        # later windows carry the prior: the reference's pseudo-inverse threshold (1e-8, MarginalizationFactor.h)
        # sits far below that noise floor, so near-null gauge directions are kept or dropped by round-off on
        # either side; parity is then the north_star bound: pose error <= 1e-4 relative.
        assert abs(sg["final_cost"] - so["final_cost"]) <= 5e-3 * so["final_cost"], (k, sg, so)
        assert np.abs(xg[:, :3] - xo[:, :3]).max() <= 1e-4 * scale
        assert np.abs(xg[:, 3:7] - xo[:, 3:7]).max() <= 1e-4
        assert np.abs(xg[:, 7:10] - xo[:, 7:10]).max() <= 1e-3
        assert sg["has_prior"] == so["has_prior"]


def test_window_solve_parity_full_odom(oracle, vlp_seq):
    """Default 10 LaserOdom iterations on the newest frame (fp32 reductions differ in order): tolerance parity."""
    W = 5
    # fixed extrinsic: with only 5 frames of a smooth trajectory the lidar-IMU rotation is barely observable and the
    # free-extrinsic problem amplifies round-off (both sides drift, see test_oracle_factors); the fixed one is well posed
    eo, eg = _mk(oracle, vlp_seq, W, opt_extrinsic=0)
    for k in range(W, 10):
        helpers.feed_scan(eo, vlp_seq, k)
        helpers.feed_scan(eg, vlp_seq, k)
        so, sg = eo.summary(), eg.summary()
        assert sg["map_size"] == so["map_size"] or abs(sg["map_size"] - so["map_size"]) <= 2
        assert abs(sg["num_features"] - so["num_features"]) <= 0.005 * so["num_features"]
        assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-3 * so["final_cost"]
        xo, xg = eo.states(), eg.states()
        scale = max(1.0, np.abs(xo[:, :3]).max())
        assert np.abs(xg[:, :3] - xo[:, :3]).max() <= 1e-4 * scale      # north_star: pose error <= 1e-4 rel
        assert np.abs(xg[:, 3:7] - xo[:, 3:7]).max() <= 1e-4


def test_two_rank_shard_equals_single(oracle, vlp_seq, device_solver=1):
    """Frame sharding with an allreduce of the S blocks reproduces the single-rank solve (two estimator instances on
    one GPU, driven by two threads; the callback sums through the host with a barrier)."""
    import ctypes as C
    import threading
    from lio_mapping_b200 import estimator
    W = 5
    cfg = dict(odom_max_iterations=1, prior_factor=1, device_solver=device_solver)
    ref = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
    ranks = [estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
             for _ in range(2)]
    mk = lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    for e in [ref] + ranks:
        helpers.warm_start(e, vlp_seq, oracle, W, pose_noise=0.01, seed=1, make_pim=mk)
    cudart = C.CDLL("libcudart.so.12") if False else None
    import torch
    bar = threading.Barrier(2)
    stage = [None, None]

    def make_cb(r):
        def cb(ptr, count):
            class _Arr:
                __cuda_array_interface__ = {"shape": (count,), "typestr": "<f8", "data": (ptr, False), "version": 3}
            t = torch.as_tensor(_Arr(), device="cuda")
            torch.cuda.synchronize()
            stage[r] = t.cpu().numpy().copy()
            bar.wait()
            t.copy_(torch.from_numpy(stage[0] + stage[1]))
            torch.cuda.synchronize()
            bar.wait()
            return 0
        return cb
    for r, e in enumerate(ranks):
        e.set_shard(r, 2, make_cb(r))
    errs = []

    def run(r):
        try:
            for k in range(W, 8):
                helpers.feed_scan(ranks[r], vlp_seq, k)
        except Exception as exc:   # pragma: no cover
            errs.append(exc)
            bar.abort()
    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t_ in th:
        t_.start()
    for k in range(W, 8):
        helpers.feed_scan(ref, vlp_seq, k)
    for t_ in th:
        t_.join(timeout=300)
    assert not errs, errs
    x = ref.states()
    for e in ranks:
        assert np.abs(e.states() - x).max() <= 1e-9 * max(1.0, np.abs(x).max())


def test_two_rank_shard_equals_single_host_controller(oracle, vlp_seq):
    """The same with the host dogleg controller."""
    test_two_rank_shard_equals_single(oracle, vlp_seq, device_solver=0)


def test_two_rank_peer_exchange_equals_single(oracle, vlp_seq, device_solver=1):
    """The fused peer-memory exchange (owned S rows stored into every rank's buffer by the stage-C kernel tail, epoch
    flags with system-scope release / acquire): two estimator contexts of one process exchange through raw device
    pointers on one GPU and reproduce the single-rank solve."""
    import threading
    from lio_mapping_b200 import estimator
    W = 5
    cfg = dict(odom_max_iterations=1, prior_factor=1, device_solver=device_solver)
    import torch
    ref = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
    # each rank on its own non-blocking stream: a rank's flag-wait kernel must not serialise with its peer's kernels
    streams = [torch.cuda.Stream() for _ in range(2)]
    ranks = [estimator.Estimator(stream=streams[r].cuda_stream, window_size=W, opt_window_size=W, max_frame_points=1 << 15,
                                 max_scan_points=1 << 17, **cfg) for r in range(2)]
    mk = lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    for e in [ref] + ranks:
        helpers.warm_start(e, vlp_seq, oracle, W, pose_noise=0.01, seed=1, make_pim=mk)
    torch.cuda.synchronize()
    ptrs = [e.exchange_buffer() for e in ranks]
    for r, e in enumerate(ranks):
        e.set_peers(r, 2, ptrs=ptrs)
    errs = []

    def run(r):
        try:
            for k in range(W, 9):
                helpers.feed_scan(ranks[r], vlp_seq, k)
        except Exception as exc:   # pragma: no cover
            errs.append(exc)
    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t_ in th:
        t_.start()
    for k in range(W, 9):
        helpers.feed_scan(ref, vlp_seq, k)
    for t_ in th:
        t_.join(timeout=300)
    assert not errs, errs
    x = ref.states()
    for e in ranks:
        assert np.abs(e.states() - x).max() <= 1e-9 * max(1.0, np.abs(x).max())


def test_two_rank_peer_exchange_equals_single_host_controller(oracle, vlp_seq):
    """The same with the host dogleg controller."""
    test_two_rank_peer_exchange_equals_single(oracle, vlp_seq, device_solver=0)


def test_two_rank_feature_exchange_equals_single(oracle, vlp_seq, device_solver=1):
    """Sharded matching with the per-scan exchange of the features themselves (lio_est_set_feature_peers): each of two contexts
    matches half of the frames, copies its features into the peer's slab and then runs the complete single-GPU solve (graph
    included with the device solver) - the window states are those of an unsharded context, bit for bit."""
    import threading
    import torch
    from lio_mapping_b200 import estimator
    W = 5
    cfg = dict(odom_max_iterations=3, prior_factor=1, device_solver=device_solver)
    ref = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17, **cfg)
    streams = [torch.cuda.Stream() for _ in range(2)]
    ranks = [estimator.Estimator(stream=streams[r].cuda_stream, window_size=W, opt_window_size=W, max_frame_points=1 << 15,
                                 max_scan_points=1 << 17, **cfg) for r in range(2)]
    mk = lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    for e in [ref] + ranks:
        helpers.warm_start(e, vlp_seq, oracle, W, pose_noise=0.01, seed=1, make_pim=mk)
    torch.cuda.synchronize()
    slabs = [e.feature_slab() for e in ranks]
    for r, e in enumerate(ranks):
        e.set_feature_peers(r, 2, ptrs=slabs)
    errs = []

    def run(r):
        try:
            for k in range(W, 10):
                helpers.feed_scan(ranks[r], vlp_seq, k)
        except Exception as exc:   # pragma: no cover
            errs.append(exc)
    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t_ in th:
        t_.start()
    for k in range(W, 10):
        helpers.feed_scan(ref, vlp_seq, k)
    for t_ in th:
        t_.join(timeout=300)
    assert not errs, errs
    x = ref.states()
    for e in ranks:
        assert np.array_equal(e.states(), x)
        assert e.summary()["iterations"] == ref.summary()["iterations"]


def test_two_rank_feature_exchange_equals_single_host_controller(oracle, vlp_seq):
    """The same with the host dogleg controller."""
    test_two_rank_feature_exchange_equals_single(oracle, vlp_seq, device_solver=0)


def _sharded_after_warm_start(oracle, vlp_seq, device_solver, fn):
    """One context of a two-rank shard (rank 0) after warm start, with the allreduce callback fn (None: no exchange)."""
    from lio_mapping_b200 import estimator
    W = 5
    e = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17,
                            odom_max_iterations=1, device_solver=device_solver)
    helpers.warm_start(e, vlp_seq, oracle, W, pose_noise=0.01, seed=1,
                       make_pim=lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    e.set_shard(0, 2, fn)
    return e, W


@pytest.mark.parametrize("device_solver", [1, 0])
def test_sharded_context_without_exchange_is_invalid(oracle, vlp_seq, device_solver):
    """A sharded context with neither a peer exchange nor a callback fails its scan with LIO_ERR_INVALID in both controllers."""
    from lio_mapping_b200 import _lib
    e, W = _sharded_after_warm_start(oracle, vlp_seq, device_solver, None)
    with pytest.raises(_lib.LioError, match="LIO_ERR_INVALID.*without an exchange"):
        helpers.feed_scan(e, vlp_seq, W)


@pytest.mark.parametrize("device_solver", [1, 0])
def test_allreduce_failure_inside_the_solve_fails_the_scan(oracle, vlp_seq, device_solver):
    """The callback fails once, on the scan's second call (the first candidate evaluation of the dogleg loop): the scan fails
    with that error in both controllers (not as a rejected step), and nothing is evaluated after it."""
    from lio_mapping_b200 import _lib
    calls = []

    def cb(ptr, count):
        calls.append(count)
        return 1 if len(calls) == 2 else 0
    e, W = _sharded_after_warm_start(oracle, vlp_seq, device_solver, cb)
    with pytest.raises(_lib.LioError, match="LIO_ERR_CUDA.*allreduce callback failed"):
        helpers.feed_scan(e, vlp_seq, W)
    assert len(calls) == 2


def test_device_solver_equals_host_solver(oracle, vlp_seq):
    """The GPU-resident dogleg loop and the host controller take the same steps."""
    from lio_mapping_b200 import estimator
    W = 5
    cfg = dict(odom_max_iterations=1, opt_extrinsic=0)
    mk = lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    es = []
    for dsol in (1, 0):
        e = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17,
                                device_solver=dsol, **cfg)
        helpers.warm_start(e, vlp_seq, oracle, W, pose_noise=0.01, seed=1, make_pim=mk)
        es.append(e)
    for k in range(W, 10):
        for e in es:
            helpers.feed_scan(e, vlp_seq, k)
        s1, s0 = es[0].summary(), es[1].summary()
        if k <= W + 1:
            assert s1["iterations"] == s0["iterations"] and s1["successful"] == s0["successful"], (k, s1, s0)
        tol = 1e-9 if k <= W + 1 else 1e-3   # once a prior exists its ~1e-7 round-off enters the later windows
        assert abs(s1["initial_cost"] - s0["initial_cost"]) <= tol * s0["initial_cost"], (k, s1["initial_cost"], s0["initial_cost"])
        assert abs(s1["final_cost"] - s0["final_cost"]) <= 5 * tol * s0["final_cost"], (k, s1["final_cost"], s0["final_cost"])
        x1, x0 = es[0].states(), es[1].states()
        assert np.abs(x1[:, :3] - x0[:, :3]).max() <= 1e-5 * max(1.0, np.abs(x0[:, :3]).max())


def test_benchmark_configuration_parity(oracle):
    """The benchmark's configuration (outdoor_test_config_64: free extrinsic + PriorFactor, window 10/10, 10 LaserOdom
    iterations) on VLP-16 sweeps: pose error <= 1e-4 relative against the oracle, scan after scan."""
    W = 10
    seq = helpers.Sequence(oracle, "vlp16", n_total=W + 4, distort=False)
    eo, eg = _mk(oracle, seq, W, prior_factor=1)
    for k in range(W, W + 4):
        helpers.feed_scan(eo, seq, k)
        helpers.feed_scan(eg, seq, k)
        so, sg = eo.summary(), eg.summary()
        assert abs(sg["num_features"] - so["num_features"]) <= 0.005 * so["num_features"]
        xo, xg = eo.states(), eg.states()
        scale = max(1.0, np.abs(xo[:, :3]).max())
        assert np.abs(xg[:, :3] - xo[:, :3]).max() <= 1e-4 * scale, (k, np.abs(xg[:, :3] - xo[:, :3]).max())
        assert np.abs(xg[:, 3:7] - xo[:, 3:7]).max() <= 1e-4
        assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-2 * so["final_cost"], (k, sg["final_cost"], so["final_cost"])


def test_window_solve_parity_with_deskew(oracle):
    """enable_deskew && !cutoff_deskew: the incoming less-flat cloud goes through TransformToEnd (k_deskew on the
    device, float sinf/acosf vs libm) before the 0.4 m voxel grid.  A last-ulp coordinate change can move a point
    across a voxel face, so frame sizes agree within a handful of points and states at the north-star bound."""
    seq = helpers.Sequence(oracle, "vlp16", n_total=9, distort=True)
    W = 5
    eo, eg = _mk(oracle, seq, W, opt_extrinsic=0, enable_deskew=1, cutoff_deskew=0)
    for k in range(W, 9):
        helpers.feed_scan(eo, seq, k)
        helpers.feed_scan(eg, seq, k)
        so, sg = eo.summary(), eg.summary()
        fo, fg = eo.frame(W), eg.frame(W)     # newest frame (pushed at ProcessScan entry)
        assert abs(fg.shape[0] - fo.shape[0]) <= 3
        if fg.shape[0] == fo.shape[0]:
            assert np.abs(fg[:, :3] - fo[:, :3]).max() < 0.4    # same voxel population (centroids may shift by one member)
            assert np.median(np.abs(fg[:, :3] - fo[:, :3]).max(axis=1)) < 1e-5
        assert abs(sg["num_features"] - so["num_features"]) <= 0.005 * so["num_features"]
        xo, xg = eo.states(), eg.states()
        scale = max(1.0, np.abs(xo[:, :3]).max())
        assert np.abs(xg[:, :3] - xo[:, :3]).max() <= 1e-4 * scale
        assert np.abs(xg[:, 3:7] - xo[:, 3:7]).max() <= 1e-4


def test_overlapped_marginalization_is_identical(oracle, vlp_seq):
    """overlap_marginalization only moves the Schur/eigen algebra to a worker thread: bit-identical states and prior."""
    from lio_mapping_b200 import estimator
    W = 5
    mk = lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    es = []
    for ov in (1, 0):
        e = estimator.Estimator(window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 17,
                                overlap_marginalization=ov, opt_extrinsic=0)
        helpers.warm_start(e, vlp_seq, oracle, W, pose_noise=0.01, seed=1, make_pim=mk)
        es.append(e)
    for k in range(W, 10):
        for e in es:
            helpers.feed_scan(e, vlp_seq, k)
        s1, s0 = es[0].summary(), es[1].summary()
        assert s1["has_prior"] == s0["has_prior"]
        assert np.array_equal(es[0].states(), es[1].states())
        if k in (W + 1, 9):
            H1, b1 = es[0].prior()
            H0, b0 = es[1].prior()
            assert np.array_equal(H1, H0) and np.array_equal(b1, b0)
