"""A plain float64 statement of the 6-DoF Gauss-Newton step shared by CalculateLaserOdom, PointMapping, MapBuilder and
PointOdometry (odom_solve_step in lio_mapping_b200/csrc/odom.cuh), and the error bounds the float32 implementations are held to.

One round: the features' Jacobian rows give A^T A / A^T b; the step x solves float32(A^T A) x = float32(A^T b); on the round that
analyses degeneracy the leading eigenvalues of A^T A under the threshold are counted (k) and the step becomes matP x with
matP = V2 V^-1, V the eigenvectors in columns (ascending eigenvalues) and V2 = V with its first k ROWS zeroed.  For an orthogonal V
that is D V V^T = D = diag(0 x k, 1 x (6 - k)): the first k coordinates of the step, rotation components, are zeroed, whatever the
degenerate direction is.  That is the reference's formula (Estimator.cc:1308-1339, PointMapping.cc:652-681, MapBuilder.cc:933-960,
PointOdometry.cc:584-615) and the statement keeps it.  The matP of the analysing round is kept for the later rounds of the chain.
"""
import math

import numpy as np

EPS32 = float(np.finfo(np.float32).eps)

# variant -> (match minimum, eigenvalue threshold, left update, loop index decides the analysing round)
VARIANTS = {0: (0, 100.0, False, False),    # CalculateLaserOdom: the first executed round analyses
            1: (50, 100.0, False, True),    # PointMapping::OptimizeTransformTobeMapped
            2: (50, 100.0, True, True),     # MapBuilder::OptimizeMap
            3: (10, 10.0, False, True)}     # PointOdometry


def rotation(q):
    """Eigen's toRotationMatrix of the (possibly non-unit) quaternion (x, y, z, w)."""
    x, y, z, w = (float(v) for v in q)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def _r_skew(R, p, absolute=False):
    """R [p]x for every point (n, 3, 3); absolute: R |[p]x|."""
    n = p.shape[0]
    S = np.zeros((n, 3, 3))
    S[:, 0, 1], S[:, 0, 2], S[:, 1, 2] = -p[:, 2], p[:, 1], -p[:, 0]
    S[:, 1, 0], S[:, 2, 0], S[:, 2, 1] = p[:, 2], -p[:, 1], p[:, 0]
    if absolute:
        S = np.abs(S)
    return np.einsum("ij,njk->nik", R, S)


def rows(pts, coef, tf7, mode):
    """Jacobian rows J (n, 6) and right-hand sides b = -d2 (n,) of the features.
    mode 0 (CalculateLaserOdom): J = [-w^T R [p]x | w^T], d2 = w . (R p + t) + coef.w;  mode 1 (scan-to-map): d2 = coef.w;
    mode 2 (MapBuilder): as 1 with the rotation part post-multiplied by R(q^-1) diag(5e-3, 5e-3, 1).  R is the raw quaternion's
    toRotationMatrix (the quaternion-vector product equals it for any quaternion)."""
    tf = np.asarray(tf7, np.float64)
    p = np.asarray(pts, np.float64).reshape(-1, 4)[:, :3]
    c = np.asarray(coef, np.float64).reshape(-1, 4)
    R = rotation(tf[:4])
    w = c[:, :3]
    J = np.zeros((p.shape[0], 6))
    J[:, :3] = -np.einsum("ni,nij->nj", w, _r_skew(R, p))
    J[:, 3:] = w
    d2 = c[:, 3].copy()
    if mode == 0:
        d2 += np.einsum("ni,ni->n", w, p @ R.T + tf[4:])
    if mode == 2:
        n2 = float(tf[:4] @ tf[:4])
        Ri = rotation(np.array([-tf[0], -tf[1], -tf[2], tf[3]]) / n2)
        J[:, :3] = (J[:, :3] @ Ri) * np.array([5e-3, 5e-3, 1.0])
    return J, -d2


def row_bounds(pts, coef, tf7, mode):
    """Magnitude bounds of the same rows: `rows` with every factor replaced by its absolute value.  A float32 evaluation of a row
    element, a few roundings deep, is off by at most a small multiple of eps32 times this bound."""
    tf = np.asarray(tf7, np.float64)
    p = np.abs(np.asarray(pts, np.float64).reshape(-1, 4)[:, :3])
    c = np.abs(np.asarray(coef, np.float64).reshape(-1, 4))
    Ra = np.abs(rotation(tf[:4])) + 4.0 * float(tf[:4] @ tf[:4]) * EPS32
    w = c[:, :3]
    J = np.zeros((p.shape[0], 6))
    J[:, :3] = np.einsum("ni,nij->nj", w, _r_skew(Ra, p, absolute=True))
    J[:, 3:] = w
    d2 = c[:, 3] + (np.einsum("ni,ni->n", w, p @ Ra.T + np.abs(tf[4:])) if mode == 0 else 0.0)
    if mode == 2:
        n2 = float(tf[:4] @ tf[:4])
        Ri = np.abs(rotation(np.array([-tf[0], -tf[1], -tf[2], tf[3]]) / n2)) + 4.0 / n2 * EPS32
        J[:, :3] = (J[:, :3] @ Ri) * np.array([5e-3, 5e-3, 1.0])
    return J, d2


def normal_equations(pts, coef, tf7, mode):
    """A^T A, A^T b in float64 and the matrices of magnitude sums M = sum |J_a| |J_b|, m = sum |J_a| |b| of the bounds."""
    J, b = rows(pts, coef, tf7, mode)
    Jb, bb = row_bounds(pts, coef, tf7, mode)
    return J.T @ J, J.T @ b, Jb.T @ Jb, Jb.T @ bb


def f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def solve(AtA, AtB):
    """The undamped step: float32(A^T A) x = float32(A^T b), solved in float64."""
    return np.linalg.solve(f32(AtA), f32(AtB))


def eigen(AtA):
    """Ascending eigenvalues and eigenvectors (columns) of float32(A^T A)."""
    return np.linalg.eigh(f32(AtA))


def degenerate_count(AtA, thre):
    """k: the number of LEADING (ascending) eigenvalues under the threshold; the count stops at the first one that is not."""
    E, _ = eigen(AtA)
    k = 0
    while k < 6 and E[k] < thre:
        k += 1
    return k


def mask_matrix(AtA, thre):
    """matP = V2 V^-1 (V2 = V with rows [0, k) zeroed) and k."""
    E, V = eigen(AtA)
    k = degenerate_count(AtA, thre)
    V2 = V.copy()
    V2[:k, :] = 0.0
    return V2 @ np.linalg.inv(V), k


def qmul(a, b):
    """Hamilton product of (x, y, z, w) quaternions."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx,
                     aw * bw - ax * bx - ay * by - az * bz])


def update(tf7, x, left=False):
    """pos += x[3:];  rot = rot * DeltaQ(x[:3]) (right) or DeltaQ(x[:3]) * rot (left), DeltaQ = (x/2, 1) not normalised;
    a non-finite position coordinate is reset to 0."""
    tf = np.asarray(tf7, np.float64).copy()
    dq = np.array([x[0] / 2, x[1] / 2, x[2] / 2, 1.0])
    tf[:4] = qmul(dq, tf[:4]) if left else qmul(tf[:4], dq)
    with np.errstate(invalid="ignore"):
        tf[4:] = tf[4:] + x[3:]
    tf[4:][~np.isfinite(tf[4:])] = 0.0
    return tf


def deltas(tf_old, tf_new, x):
    """delta_r: angularDistance(normalised old rotation, new rotation) in degrees; delta_t = |100 x[3:]|."""
    a = np.asarray(tf_old, np.float64)[:4]
    a = a / np.linalg.norm(a)
    b = np.asarray(tf_new, np.float64)[:4]
    bc = np.array([-b[0], -b[1], -b[2], b[3]])
    d = qmul(a, bc)
    dr = math.degrees(2 * math.atan2(np.linalg.norm(d[:3]), abs(d[3])))
    with np.errstate(invalid="ignore", over="ignore"):
        dt = float(np.linalg.norm(100.0 * np.asarray(x[3:], np.float64)))
    return dr, dt


def step(AtA, AtB, tf7, thre=100.0, left=False, masked=True, matP=None):
    """One analysing round (matP None: computed here) or a later round with a kept matP.  Returns (tf, x, k, matP)."""
    x = solve(AtA, AtB)
    k = None
    if matP is None:
        matP, k = mask_matrix(AtA, thre)
    if masked and (k is None or k > 0):
        x = matP @ x
    return update(tf7, x, left), x, k, matP


def chain(AtAs, AtBs, n_feats, tf7, variant, dr_abort=0.05, dt_abort=0.05):
    """The round rules of the four loops around the step.  A round after convergence does nothing; a round under the match
    minimum leaves the pose alone and still counts; the analysing round is the first executed one (variant 0) or loop index 0
    (variants 1-3: when that round is skipped, no round is ever masked).  Returns (poses after each round, state dict)."""
    nmin, thre, left, by_index = VARIANTS[variant]
    tf = np.asarray(tf7, np.float64).copy()
    st = dict(degenerate=0, done=0, iter=0)
    matP = None
    poses = []
    for r, (A, b, n) in enumerate(zip(AtAs, AtBs, n_feats)):
        if st["done"]:
            poses.append(tf.copy())
            continue
        if n < nmin:
            st["iter"] += 1
            poses.append(tf.copy())
            continue
        first = (r == 0) if by_index else (st["iter"] == 0)
        x = solve(A, b)
        if first:
            matP, k = mask_matrix(A, thre)
            st["degenerate"] = int(k > 0)
        if st["degenerate"]:
            x = matP @ x
        new = update(tf, x, left)
        dr, dt = deltas(tf, new, x)
        tf = new
        st["iter"] += 1
        if dr < dr_abort and dt < dt_abort:
            st["done"] = 1
        poses.append(tf.copy())
    return poses, st


# ---- error bounds ---------------------------------------------------------------------------------------------------------------

def step_error_bound(AtA, x, M, m, gamma, matP=None):
    """Componentwise first-order bound on the error of the (masked) step when every element of A^T A and A^T b is off by at
    most gamma times its magnitude sum (M, m from normal_equations) and the 6 x 6 float32 solve adds a backward error of
    6 eps32 |A| |x|:  |dx| <= |matP| |A^-1| (gamma (M |x| + m) + 6 eps32 |A| |x|).  |A^-1| carries the condition of the problem:
    an error along a weak direction is amplified by 1 / lambda_min."""
    A = f32(AtA)
    ax = np.abs(x)
    dx = np.abs(np.linalg.inv(A)) @ (gamma * (M @ ax + m) + 6 * EPS32 * (np.abs(A) @ ax))
    return dx if matP is None else np.abs(matP) @ dx


def pose_bound(tf7, dx):
    """(position, quaternion) bounds of a pose updated by a step that is off by dx, plus the float32 rounding of the pose."""
    tf = np.abs(np.asarray(tf7, np.float64))
    qn = float(np.linalg.norm(tf[:4]))
    return float(dx[3:].max() + 2 * EPS32 * (tf[4:].max() + 1.0)), float(qn * dx[:3].max() + 4 * EPS32 * qn)


def pose_distance(a, b):
    """max |position difference| and max |quaternion difference| (sign-insensitive)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a[4:] - b[4:]).max()), float(min(np.abs(a[:4] - b[:4]).max(), np.abs(a[:4] + b[:4]).max()))


# ---- error models of the two implementations ------------------------------------------------------------------------------------
# A float32 row element is about five roundings deep and a product of two adds one: 16 eps32 of the magnitude sums covers both.
GAMMA_ROWS = 16 * EPS32


def gamma_device(n):
    """The device rounds each product to float32 and sums in double: the sum adds n eps64."""
    return GAMMA_ROWS + n * float(np.finfo(np.float64).eps)


def gamma_oracle(n):
    """The CPU oracle sums n float32 products in float32, in order: sqrt(n) eps32 (the probabilistic bound of a recursive sum)."""
    return GAMMA_ROWS + math.sqrt(max(n, 1)) * EPS32


# ---- scenes ---------------------------------------------------------------------------------------------------------------------

def corridor_scene():
    """A 600 m x 4 m x 3 m corridor along x with nothing in it: its planes constrain everything but the motion along x (and
    weakly the roll about it), so the first-round A^T A of a VLP-16 sweep has an eigenvalue under 100."""
    from lio_mapping_b200 import synth
    return synth.Scene(np.zeros((0, 6)), np.array([-300.0, -2.0, -1.0, 300.0, 2.0, 2.0]), False)


def scan_to_map_inputs(oracle, scene_name, n_frames=4):
    """Voxel-filtered less_flat (0.4 m) and less_sharp (0.2 m) clouds of VLP-16 sweeps at t = 1.0, 1.1, ... on the default vlp16
    trajectory, their maps from frames 0..n-2 and the perturbed start of the last frame, as the stage-B parity tests build them.
    Returns (surf map, corner map, surf, corner, tf0)."""
    from lio_mapping_b200 import synth
    from tests import helpers
    sensor, scene, traj = synth.default_config("vlp16")
    if scene_name == "corridor":
        scene = corridor_scene()
    sc, cc, poses = [], [], []
    for f in range(n_frames):
        t = 1.0 + 0.1 * f
        sw = synth.make_sweep(sensor, scene, traj, t, seed=10 + f, distort=False)
        r = oracle.stage_a(sw, sensor.lower_deg, sensor.upper_deg, sensor.rings)
        sc.append(oracle.voxel_grid(r["less_flat"], 0.4))
        cc.append(oracle.voxel_grid(r["less_sharp"], 0.2))
        p, R, _, _, _ = traj.state(np.array(t))
        poses.append((R, p))
    smap = helpers.build_map(oracle, sc, poses)
    cmap = helpers.build_map(oracle, cc, poses, leaf=0.2)
    _, _, tf7 = helpers.rel_transform(poses[0], poses[-1])
    tf0 = tf7.copy()
    tf0[4:] += np.array([0.05, -0.04, 0.02], np.float32)
    return smap, cmap, sc[-1], cc[-1], tf0
