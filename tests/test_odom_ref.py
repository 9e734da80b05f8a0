"""The CPU oracle's Gauss-Newton rounds against the float64 statement of the step (tests/odom_ref.py), on the default vlp16 scene
and on a corridor whose first-round A^T A is degenerate.  The oracle and the device were written in the same operation order;
this checks the oracle against an independent statement, so a misreading the two share cannot hide behind their agreement."""
import numpy as np
import pytest

from tests import odom_ref as R


@pytest.fixture(scope="module", params=["vlp16", "corridor"])
def scene(request, oracle):
    return request.param, R.scan_to_map_inputs(oracle, request.param)


def _check_round(tf_out, pts, coef, tf0, mode, variant, expect_k):
    """tf_out is one round of `variant` on the features (pts, coef) from tf0: compare with the masked statement within the
    oracle's error bound, and return that bound with the unmasked statement's pose."""
    A, b, M, m = R.normal_equations(pts, coef, tf0, mode)
    _, thre, left, _ = R.VARIANTS[variant]
    tf_m, x, k, P = R.step(A, b, tf0, thre=thre, left=left)
    if expect_k is not None:
        assert (k > 0) == expect_k, (k, R.eigen(A)[0])
    dx = R.step_error_bound(A, x, M, m, R.gamma_oracle(pts.shape[0]), P if k else None)
    tol_p, tol_q = R.pose_bound(tf0, dx)
    dp, dq = R.pose_distance(tf_out, tf_m)
    assert dp <= tol_p and dq <= tol_q, (dp, tol_p, dq, tol_q)
    tf_u, _, _, _ = R.step(A, b, tf0, thre=thre, left=left, masked=False)
    return k, (tol_p, tol_q), R.pose_distance(tf_out, tf_u)


def test_laser_odom_round_equals_the_statement(oracle, scene):
    name, (smap, cmap, surf, corner, tf0) = scene
    to, po, co, so, it = oracle.laser_odom(smap, surf, tf0, max_iter=1)
    assert it == 1 and po.shape[0] > 1000
    k, (tol_p, tol_q), (dp_u, dq_u) = _check_round(to, po, co, tf0, 0, 0, expect_k=(name == "corridor"))
    if name == "corridor":
        # the degenerate branch changes the answer: the unmasked step is outside the bound
        assert k == 1 and (dp_u > tol_p or dq_u > tol_q), (dp_u, tol_p, dq_u, tol_q)


@pytest.mark.parametrize("variant", [0, 1])
def test_scan_to_map_round_equals_the_statement(oracle, scene, variant):
    """variant 0 PointMapping (mode 1, right update), 1 MapBuilder (mode 2: its 5e-3 rotation weights put two or three
    eigenvalues under 100 in every scene, so its first round is always masked)."""
    name, (smap, cmap, surf, corner, tf0) = scene
    to, po, co, so, it = oracle.scan_to_map(cmap, smap, corner, surf, tf0, max_iter=1, variant=variant)
    assert it == 1 and po.shape[0] >= 50
    expect = True if (variant == 1 or name == "corridor") else False
    k, (tol_p, tol_q), (dp_u, dq_u) = _check_round(to, po, co, tf0, 1 + variant, 1 + variant, expect_k=expect)
    if expect:
        assert dp_u > tol_p or dq_u > tol_q, (dp_u, tol_p, dq_u, tol_q)


def test_statement_mask_is_the_coordinate_mask():
    """matP = V2 V^-1 with leading rows of V2 zeroed is diag(0 x k, 1 x (6 - k)): it zeroes step coordinates, not the
    degenerate eigen-direction."""
    rng = np.random.default_rng(0)
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    for k in range(7):
        E = np.concatenate([np.linspace(20, 80, k), np.linspace(300, 1e5, 6 - k)])
        A = (Q * E) @ Q.T
        P, kk = R.mask_matrix(A, 100.0)
        assert kk == k
        D = np.diag([0.0] * k + [1.0] * (6 - k))
        assert np.abs(P - D).max() < 1e-12


def test_laser_odom_without_matches_takes_a_zero_step(oracle, scene):
    """No matches: A^T A = 0 and A^T b = 0.  The QR solve divides only nonzero right-hand sides, as Eigen's triangular solve does,
    so the step is 0 (not 0 / 0), the pose is kept and the loop stops after one round."""
    name, (smap, cmap, surf, corner, tf0) = scene
    far = surf.copy()
    far[:, :3] += 500.0
    to, po, co, so, it = oracle.laser_odom(smap, far, tf0)
    assert po.shape[0] == 0 and it == 1 and np.array_equal(to, tf0)
