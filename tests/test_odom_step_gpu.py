"""The 6-DoF Gauss-Newton step of CalculateLaserOdom, PointMapping, MapBuilder and PointOdometry (odom_solve_step and the
reductions in front of it, csrc/odom.cu / odom.cuh) against the float64 statement in tests/odom_ref.py: the normal equations at the
unroll and last-block edges, the column-pivoted QR solve, the degeneracy mask and its round rules, the quaternion updates and the
convergence test, and the whole loops on a corridor whose first round is degenerate."""
import math

import numpy as np
import pytest

from tests import odom_ref as R

pytestmark = pytest.mark.gpu

EPS = R.EPS32
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
NS = [0, 1, 255, 256, 257, 511, 512, 513, 2047, 2048, 2049, 8193, 300001]
# (kernel, blocks): k_odom_reduce mode 0..2 on the callers' grid, one CTA and 7 CTAs; the fused single-CTA k_odom_round
GRIDS = [(m, b) for m in range(3) for b in (0, 1, 7)] + [(3, 0)]


def _x_from_identity(tf):
    """The step taken from the identity pose, read back exactly: q.xyz = X[:3] / 2, pos = X[3:]."""
    tf = np.asarray(tf, np.float64)
    return np.concatenate([2 * tf[:3], tf[4:]])


def _spd(E, seed, diagonal=False):
    E = np.asarray(E, np.float64)
    if diagonal:
        return np.diag(E)
    Q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(6, 6)))
    return (Q * E) @ Q.T


# ---- normal equations ---------------------------------------------------------------------------------------------------------

def _int_features(n, seed):
    rng = np.random.default_rng(seed)
    pts = np.concatenate([rng.integers(-3, 4, (n, 3)), rng.integers(0, 9, (n, 1))], 1).astype(np.float32)
    coef = np.concatenate([rng.integers(-2, 3, (n, 3)), rng.integers(-3, 4, (n, 1))], 1).astype(np.float32)
    tf = IDENT.copy()
    tf[4:] = rng.integers(-2, 3, 3)
    return pts, coef, tf


def _exact_normal_equations(pts, coef, tf, kernel):
    """Small integers and the identity rotation: every row element is an exact float32 integer and every product of two is
    exact, except MapBuilder's 5e-3 weights, which are applied with float32 rounding as the kernel does.  All products are
    multiples of 2^-40 and their sums stay far below 2^13, so the float64 sums are exact in any order."""
    J, b = R.rows(pts, coef, tf, 0 if kernel in (0, 3) else 1)
    if kernel == 2:
        J[:, :2] = (J[:, :2].astype(np.float32) * np.float32(5e-3)).astype(np.float64)
    prod = lambda u, v: (u.astype(np.float32) * v.astype(np.float32)).astype(np.float64)
    AtA = np.array([[prod(J[:, a], J[:, c]).sum() for c in range(6)] for a in range(6)])
    AtB = np.array([prod(J[:, a], b).sum() for a in range(6)])
    return AtA, AtB


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("kernel,blocks", GRIDS)
def test_normal_equations_exact_on_integers(n, kernel, blocks):
    """A dropped or doubled feature at the i0 + u * 512 unroll edges or in the last-block sum changes an exact integer sum."""
    from lio_mapping_b200 import ops
    pts, coef, tf = _int_features(n, seed=n)
    AtA, AtB = ops.odom_normal_equations(pts, coef, tf, kernel, blocks)
    eA, eB = _exact_normal_equations(pts, coef, tf, kernel)
    assert np.array_equal(AtA, eA) and np.array_equal(AtB, eB), (np.abs(AtA - eA).max(), np.abs(AtB - eB).max())
    A2, B2 = ops.odom_normal_equations(pts, coef, tf, kernel, blocks)
    assert np.array_equal(AtA.view(np.uint64), A2.view(np.uint64)) and np.array_equal(AtB.view(np.uint64), B2.view(np.uint64))


@pytest.mark.parametrize("n", [1, 513, 2049, 300001])
@pytest.mark.parametrize("kernel,blocks", GRIDS)
def test_normal_equations_random(n, kernel, blocks):
    """Float features and a non-unit quaternion: within gamma (sum |J_a| |J_b|) of the float64 statement, gamma from eps32;
    bit-identical between two runs."""
    from lio_mapping_b200 import ops
    rng = np.random.default_rng(1000 + n)
    pts = np.concatenate([rng.uniform(-30, 30, (n, 3)), rng.uniform(0, 9, (n, 1))], 1).astype(np.float32)
    w = rng.normal(size=(n, 3))
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    coef = np.concatenate([w, rng.uniform(-0.3, 0.3, (n, 1))], 1).astype(np.float32)
    q = rng.normal(size=4)
    q *= 1.07 / np.linalg.norm(q)
    tf = np.concatenate([q, rng.uniform(-2, 2, 3)]).astype(np.float32)
    mode = 0 if kernel == 3 else kernel
    AtA, AtB = ops.odom_normal_equations(pts, coef, tf, kernel, blocks)
    eA, eB, M, m = R.normal_equations(pts, coef, tf, mode)
    g = R.gamma_device(n)
    assert np.all(np.abs(AtA - eA) <= g * M) and np.all(np.abs(AtB - eB) <= g * m)
    A2, B2 = ops.odom_normal_equations(pts, coef, tf, kernel, blocks)
    assert np.array_equal(AtA.view(np.uint64), A2.view(np.uint64)) and np.array_equal(AtB.view(np.uint64), B2.view(np.uint64))


# ---- the solve ----------------------------------------------------------------------------------------------------------------

def _unmasked_step(A, b, variant=1):
    """The step of a PointMapping-style chain whose round 0 is skipped (too few matches): no round is ever masked, so round 1
    is the bare QR solve."""
    from lio_mapping_b200 import ops
    nmin = R.VARIANTS[variant][0]
    tf, per, st, _ = ops.odom_step(np.stack([np.zeros(36), np.ravel(A)]), np.stack([np.zeros(6), b]), [0, nmin], IDENT, variant, 0.0, 0.0)
    assert st["degenerate"] == 0 and st["iter"] == 2 and np.array_equal(per[0], IDENT)
    return _x_from_identity(tf)


@pytest.mark.parametrize("cond", [1.0, 10.0, 1e2, 1e3, 1e4])
def test_solve_backward_and_forward_error(cond):
    """All eigenvalues above 100: the backward error |A32 x - b32| is a few eps32 (|A| |x| + |b|), the forward error is at most
    the condition number times that.  c = 36 covers the 6 x 6 Householder QR (n^2 eps)."""
    from lio_mapping_b200 import ops
    for seed in range(4):
        E = 150.0 * np.geomspace(1.0, cond, 6)
        A = _spd(E, seed)
        b = np.random.default_rng(seed).normal(size=6) * 150.0
        A32, b32 = R.f32(A), R.f32(b)
        x64 = np.linalg.solve(A32, b32)
        for variant in (0, 1):
            if variant == 0:
                tf, _, st, _ = ops.odom_step(A, b, [1000], IDENT, 0, 0.0, 0.0)
                assert st["degenerate"] == 0
                x = _x_from_identity(tf)
            else:
                x = _unmasked_step(A, b)
            nx = np.linalg.norm(x)
            assert np.linalg.norm(A32 @ x - b32) <= 36 * EPS * (np.linalg.norm(A32, 2) * nx + np.linalg.norm(b32))
            kappa = np.linalg.cond(A32)
            assert np.linalg.norm(x - x64) <= 36 * EPS * kappa * np.linalg.norm(x64) * 2


@pytest.mark.parametrize("j", range(6))
def test_solve_zero_row_and_column(j):
    """An exact zero row and column j: QR's rank cut-off leaves x[j] = 0 and the other coordinates solve the 5 x 5 system."""
    A = _spd(150.0 * np.geomspace(1, 100, 6), 30 + j)
    A[j, :] = 0.0
    A[:, j] = 0.0
    b = np.random.default_rng(j).normal(size=6) * 100.0
    x = _unmasked_step(A, b)
    assert x[j] == 0.0
    keep = [i for i in range(6) if i != j]
    As, bs = R.f32(A[np.ix_(keep, keep)]), R.f32(b[keep])
    xs = np.linalg.solve(As, bs)
    assert np.linalg.norm(x[keep] - xs) <= 72 * EPS * np.linalg.cond(As) * np.linalg.norm(xs)


def test_zero_normal_equations():
    """A^T A = 0, A^T b = 0: x = 0 (every direction is degenerate and the solve has no pivot), so the chain is done in round 0."""
    from lio_mapping_b200 import ops
    tf0 = np.array([0.1, -0.2, 0.3, 0.9, 1.0, 2.0, 3.0], np.float32)
    for variant in range(4):
        tf, per, st, _ = ops.odom_step(np.zeros((3, 36)), np.zeros((3, 6)), [100, 100, 100], tf0, variant)
        assert np.array_equal(tf, tf0) and st["done"] == 1 and st["iter"] == 1, (variant, st)


# ---- the degeneracy mask ------------------------------------------------------------------------------------------------------

def _spectrum(k, thre, seed, mult=1, lmax=1e5):
    """k eigenvalues under thre (at most thre / 1.1), 6 - k above (at least 1.1 thre), the top one lmax; `mult` repeats the
    smallest and the largest values."""
    rng = np.random.default_rng(seed)
    lo = np.sort(rng.uniform(0.05, 1 / 1.1, k)) * thre
    hi = np.sort(np.concatenate([rng.uniform(1.1 * thre, lmax, 5 - k), [lmax]]))[-(6 - k):] if k < 6 else np.zeros(0)
    E = np.concatenate([lo, hi])
    if mult > 1:
        if k >= mult:
            E[1:mult] = E[0]
        if 6 - k >= mult:
            E[6 - mult:] = E[-1]
    return E


CASES = [(k, mult, diag, lmax) for k in range(7) for mult, diag, lmax in ((1, False, 1e5), (2, False, 1e5), (3, False, 1e5),
                                                                           (1, True, 1e5), (1, False, 1e7))]


@pytest.mark.parametrize("k,mult,diagonal,lmax", CASES)
def test_mask_zeroes_the_leading_coordinates(k, mult, diagonal, lmax):
    """k leading eigenvalues under 100: X[:k] is exactly 0 and X[k:] is the QR step's, up to matP = V2 V^T being the coordinate
    mask to within the orthogonality of the Jacobi vectors (a few eps32 per rotation: 1e-5 |X|)."""
    from lio_mapping_b200 import ops
    for seed in range(3):
        E = _spectrum(k, 100.0, 100 * k + 10 * mult + seed, mult, lmax)
        if diagonal:
            E = np.random.default_rng(seed).permutation(E)
        A = _spd(E, 7 * k + seed, diagonal)
        b = (np.random.default_rng(seed + 50).normal(size=6) * 20.0)
        assert R.degenerate_count(A, 100.0) == k
        tf, _, st, P = ops.odom_step(A, b, [1000], IDENT, 0, 0.0, 0.0)
        X = _x_from_identity(tf)
        xq = _unmasked_step(A, b)
        assert st["degenerate"] == int(k > 0)
        assert np.all(X[:k] == 0.0), X
        if k < 6:
            assert np.abs(X[k:] - xq[k:]).max() <= 1e-5 * np.linalg.norm(xq), (X, xq)
        if k > 0:
            assert np.abs(P - np.diag([0.0] * k + [1.0] * (6 - k))).max() <= 1e-5


def test_threshold_per_variant():
    """An eigenvalue of 50 is degenerate under CalculateLaserOdom's, PointMapping's and MapBuilder's threshold of 100 and not
    under PointOdometry's 10."""
    from lio_mapping_b200 import ops
    A = _spd([50.0, 400.0, 900.0, 2e3, 5e3, 1e4], 3)
    b = np.random.default_rng(3).normal(size=6) * 20.0
    xq = _unmasked_step(A, b)
    for variant, expect in ((0, 1), (1, 1), (2, 1), (3, 0)):
        tf, _, st, _ = ops.odom_step(A, b, [1000], IDENT, variant, 0.0, 0.0)
        X = _x_from_identity(tf)
        assert st["degenerate"] == expect, variant
        if expect:
            assert X[0] == 0.0 and abs(xq[0]) > 1e-3
        else:
            assert np.abs(X - xq).max() <= 1e-5 * np.linalg.norm(xq)


# ---- round rules --------------------------------------------------------------------------------------------------------------

def _chain_check(As, bs, ns, tf0, variant, dr=0.0, dt=0.0):
    from lio_mapping_b200 import ops
    tf, per, st, _ = ops.odom_step(np.array([np.ravel(a) for a in As]), np.array(bs), ns, tf0, variant, dr, dt)
    poses, est = R.chain(As, bs, ns, tf0, variant, dr, dt)
    assert st == est, (st, est)
    # each round's float32 solve is off by at most 36 eps32 cond(A) |x|; the errors of the rounds add up
    err = sum(36 * EPS * np.linalg.cond(R.f32(a)) * np.linalg.norm(R.solve(a, b)) for a, b in zip(As, bs)) + 8 * EPS * (1 + np.abs(tf0).max())
    for r, (g, e) in enumerate(zip(per, poses)):
        dp, dq = R.pose_distance(g, e)
        assert dp <= err and dq <= err, (r, g, e, err)
    return per, st


A_DEG = _spd([5.0, 500.0, 900.0, 2e3, 5e3, 1e4], 11)
A_WELL = _spd([300.0, 500.0, 900.0, 2e3, 5e3, 1e4], 12)
B0 = np.array([3.0, -2.0, 1.5, 4.0, -3.0, 2.0])


def test_laser_odom_keeps_the_first_rounds_mask():
    """CalculateLaserOdom analyses its first round only: a degenerate round 0 keeps masking the well-conditioned later rounds;
    a well-conditioned round 0 masks nothing later, however degenerate."""
    per, st = _chain_check([A_DEG, A_WELL, A_WELL], [B0, B0, -B0], [500] * 3, IDENT, 0)
    assert st["degenerate"] == 1
    per, st = _chain_check([A_WELL, A_DEG, A_DEG], [B0, B0, -B0], [500] * 3, IDENT, 0)
    assert st["degenerate"] == 0


@pytest.mark.parametrize("variant", [1, 2, 3])
def test_skipped_first_round_never_masks(variant):
    """PointMapping, MapBuilder, PointOdometry: the analysis belongs to loop index 0.  When round 0 has too few matches it is
    skipped (pose untouched, still counted) and no round is ever masked; a skipped later round changes nothing either."""
    nmin = R.VARIANTS[variant][0]
    tf0 = np.array([0.05, -0.02, 0.1, 0.99, 1.0, -2.0, 0.5], np.float32)
    per, st = _chain_check([A_DEG, A_DEG, A_DEG, A_WELL], [B0, B0, -B0, B0], [nmin - 1, nmin, nmin - 1, nmin], tf0, variant)
    assert np.array_equal(per[0], tf0) and np.array_equal(per[2], per[1]) and st["degenerate"] == 0 and st["iter"] == 4
    per, st = _chain_check([A_DEG, A_WELL, A_WELL], [B0, B0, -B0], [nmin, nmin, nmin], tf0, variant)
    assert st["degenerate"] == 1


@pytest.mark.parametrize("variant", range(4))
def test_rounds_after_done_are_no_ops(variant):
    per, st = _chain_check([A_WELL, A_DEG, A_WELL], [B0, 10 * B0, -B0], [500] * 3, IDENT, variant, 1e9, 1e9)
    assert st["done"] == 1 and st["iter"] == 1 and np.array_equal(per[1], per[0]) and np.array_equal(per[2], per[0])


# ---- update and convergence ---------------------------------------------------------------------------------------------------

def test_right_and_left_update():
    """From a 40-degree yaw, a roll step: rot * DeltaQ (PointMapping, PointOdometry) and DeltaQ * rot (MapBuilder) differ, and
    each equals the statement to float32 round-off."""
    from lio_mapping_b200 import ops
    h = math.radians(20.0)
    tf0 = np.array([0, 0, math.sin(h), math.cos(h), 0.3, 0.2, 0.1], np.float32)
    A = 1000.0 * np.eye(6)
    x = np.array([0.2, 0.0, 0.0, 0.01, 0.02, 0.03])
    out = {}
    for variant in (1, 2):
        tf, _, _, _ = ops.odom_step(A, A @ x, [100], tf0, variant, 0.0, 0.0)
        e = R.update(tf0, R.f32(x), left=(variant == 2))
        assert np.abs(tf - e).max() <= 8 * EPS, (variant, tf, e)
        out[variant] = tf
    assert np.abs(out[1][:4] - out[2][:4]).max() > 0.01


def test_infinite_translation_resets_the_position():
    """A step whose translation overflows float32 leaves a non-finite position coordinate, which the update resets to 0."""
    from lio_mapping_b200 import ops
    tf0 = np.array([0, 0, 0, 1, 1.0, 2.0, 3.0], np.float32)
    A = 0.5 * np.eye(6)
    b = np.array([0.0, 0.0, 0.0, 3e38, 0.01, 0.0])
    tf, per, st, _ = ops.odom_step(np.stack([np.zeros(36), A.ravel()]), np.stack([np.zeros(6), b]), [0, 50], tf0, 1, 0.05, 0.05)
    assert tf[4] == 0.0 and abs(tf[5] - 2.02) < 1e-6 and tf[6] == 3.0 and st["done"] == 0
    assert np.array_equal(R.update(tf0, np.array([0, 0, 0, np.inf, 0.02, 0]))[4:], [0.0, 2.02, 3.0])


@pytest.mark.parametrize("what", ["rotation", "translation"])
@pytest.mark.parametrize("factor,done_round", [(1.1, 2), (0.9, 3)])
def test_abort_thresholds(what, factor, done_round):
    """Steps halving every round; with the abort value at 1.1x the round-2 step the chain is done after round 2, at 0.9x one
    round later.  The 10 % margins are far above float32 round-off."""
    from lio_mapping_b200 import ops
    A = 1000.0 * np.eye(6)
    x0 = np.array([0.02, -0.01, 0.015, 0, 0, 0]) if what == "rotation" else np.array([0, 0, 0, 0.004, -0.003, 0.002])
    xs = [x0 * 0.5 ** r for r in range(5)]
    tf = R.f32(IDENT)
    deltas = []
    for x in xs:
        new = R.update(tf, x)
        deltas.append(R.deltas(tf, new, x))
        tf = new
    d = deltas[2][0 if what == "rotation" else 1] * factor
    dr, dt = (d, 1.0) if what == "rotation" else (1.0, d)
    tfg, per, st, _ = ops.odom_step([A.ravel()] * 5, [A @ x for x in xs], [100] * 5, IDENT, 0, dr, dt)
    assert st["done"] == 1 and st["iter"] == done_round + 1, st
    assert np.array_equal(per[-1], per[done_round])


# ---- the corridor end to end --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def corridor(oracle):
    return R.scan_to_map_inputs(oracle, "corridor")


def _round_matches_statement(tf_out, pts, coef, tf0, mode, variant):
    A, b, M, m = R.normal_equations(pts, coef, tf0, mode)
    _, thre, left, _ = R.VARIANTS[variant]
    tf_m, x, k, P = R.step(A, b, tf0, thre=thre, left=left)
    assert k > 0
    tol_p, tol_q = R.pose_bound(tf0, R.step_error_bound(A, x, M, m, R.gamma_device(pts.shape[0]), P))
    dp, dq = R.pose_distance(tf_out, tf_m)
    assert dp <= tol_p and dq <= tol_q, (dp, tol_p, dq, tol_q)
    tf_u, _, _, _ = R.step(A, b, tf0, thre=thre, left=left, masked=False)
    dp, dq = R.pose_distance(tf_out, tf_u)
    assert dp > tol_p or dq > tol_q
    return A, x


@pytest.mark.parametrize("keep", [False, True])
def test_corridor_laser_odom(oracle, corridor, keep):
    """One round of the device's CalculateLaserOdom on a degenerate corridor equals the masked statement on its own features;
    the full loop stays with the oracle.  Along the corridor A^T A has an eigenvalue near 27: a last-bit difference in the
    reduction order (double tree vs float sum) is amplified by 1 / lambda_min, so the loop is held to the existing 2e-5 plus the
    oracle's own per-round error bound."""
    from lio_mapping_b200 import ops
    smap, cmap, surf, corner, tf0 = corridor
    tg, pg, cg, sg, itg = ops.laser_odom(smap, surf, tf0, keep_features=keep, max_iter=1)
    assert itg == 1
    _round_matches_statement(tg, pg, cg, tf0, 0, 0)
    to, po, co, so, ito = oracle.laser_odom(smap, surf, tf0, keep_features=int(keep))
    tg, pg, cg, sg, itg = ops.laser_odom(smap, surf, tf0, keep_features=keep)
    assert itg == ito
    A, b, M, m = R.normal_equations(po, co, to, 0)
    dx = R.step_error_bound(A, R.solve(A, b), M, m, R.gamma_oracle(po.shape[0]))
    tp, tq = R.pose_bound(to, dx)
    dp, dq = R.pose_distance(tg, to)
    assert dp <= 2e-5 + ito * tp and dq <= 2e-5 + ito * tq, (dp, tp, dq, tq)


@pytest.mark.parametrize("variant", [0, 1])
def test_corridor_scan_to_map(oracle, corridor, variant):
    from lio_mapping_b200 import ops
    smap, cmap, surf, corner, tf0 = corridor
    tg, pg, cg, sg, itg = ops.scan_to_map(cmap, smap, corner, surf, tf0, max_iter=1, variant=variant)
    assert itg == 1
    _round_matches_statement(tg, pg, cg, tf0, 1 + variant, 1 + variant)
    to, po, co, so, ito = oracle.scan_to_map(cmap, smap, corner, surf, tf0, variant=variant)
    tg, pg, cg, sg, itg = ops.scan_to_map(cmap, smap, corner, surf, tf0, variant=variant)
    assert itg == ito
    A, b, M, m = R.normal_equations(po, co, to, 1 + variant)
    _, thre, left, _ = R.VARIANTS[1 + variant]
    _, x, k, P = R.step(A, b, to, thre=thre, left=left)
    tp, tq = R.pose_bound(to, R.step_error_bound(A, x, M, m, R.gamma_oracle(po.shape[0]), P if k else None))
    dp, dq = R.pose_distance(tg, to)
    assert dp <= 2e-5 + ito * tp and dq <= 2e-5 + ito * tq, (dp, tp, dq, tq)


def test_corridor_point_odometry(oracle):
    """PointOdometry over corridor sweeps against the oracle, with the tolerances of its drive test.  It returns no features, so
    only the oracle comparison is made here; its threshold of 10 is covered by the step entry."""
    from lio_mapping_b200 import synth
    from lio_mapping_b200.point_odometry import PointOdometry
    sensor, _, traj = synth.default_config("vlp16")
    scene = R.corridor_scene()
    po = oracle.PointOdometryOracle(0.1, 2, 25)
    pg = PointOdometry(0.1, 2, 25)
    keys = ("sharp", "less_sharp", "flat", "less_flat", "full")
    for f in range(4):
        sw = synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * f, seed=70 + f, distort=True)
        r = oracle.stage_a(sw, sensor.lower_deg, sensor.upper_deg, sensor.rings)
        s = dict(sharp=r["sharp"], less_sharp=r["less_sharp"], flat=r["flat"], less_flat=r["less_flat"], full=r["laser_scans"])
        to, eo, io = po.process(*[s[k] for k in keys])
        tg, eg, ig = pg.Process(*[s[k] for k in keys])
        if f == 0:
            continue
        assert abs(ig["iterations"] - io["iterations"]) <= 1 and abs(ig["matches"] - io["matches"]) <= 2 + 0.01 * io["matches"]
        scale = max(1.0, float(np.abs(to[4:]).max()))
        assert np.abs(eg[4:] - eo[4:]).max() <= 2e-4, (f, eg, eo)
        assert R.pose_distance(eg, eo)[1] <= 2e-5, (f, eg, eo)
        assert np.abs(tg[4:] - to[4:]).max() <= 3e-4 * scale and R.pose_distance(tg, to)[1] <= 5e-5, (f, tg, to)
