"""Plain numpy statement of lio::PointProcessor's PointToRing and ExtractFeaturePoints (PointProcessor.cc:185-783,
PointProcessor.h:104-156), written from the reference source and importing nothing from the package or the oracle.  It is the
independent yardstick stage A's kernels and the oracle are compared with, over every field of lio_pp_config.

Arithmetic, as the reference writes it:
  dis = sqrt(x*x + y*y), the squared differences, depths and curvatures are float32 in source order; the comparisons against
  0.1, 0.0002 * dis2 and 0.05 are made in double; RadToDeg<float> is double arithmetic rounded to float; ElevationToRing is
  float (deg - lower) * factor, + 0.5 in double, truncated toward zero; factor = float(num_rings - 1) / (upper - lower).
  The azimuth is float(2 pi - atan2(y, x)) with the >= 2 pi wrap in double; rel_time = float(scan_period * rel / (2 pi)).
Rounding contract of the angles: atan2 is evaluated as float32(atan2 in float64), the device's documented choice.  The
reference's atan2f need not be correctly rounded, so every point also carries the results it would have with each angle one
float32 ulp either side (point_alternatives), and an `ambiguous` flag: its float64 angle lies within AMBIG_ULPS float64 ulps of a float32
rounding midpoint, or its ring id changes when the elevation moves one float32 ulp.
"""
from __future__ import annotations

import numpy as np

from tests.pcl_voxel_ref import less_flat_cloud

TWO_PI = 2.0 * np.pi
AMBIG_ULPS = 8
F32, F64 = np.float32, np.float64

DEFAULT = dict(lower_bound=-15.0, upper_bound=15.0, num_rings=16, scan_period=0.1, num_scan_subregions=8,
               num_curvature_regions=5, surf_curv_th=0.1, max_corner_sharp=2, max_corner_less_sharp=20, max_surf_flat=4,
               less_flat_filter_size=0.2)
# (lower, upper, rings) of the sensors the node ships (VLP-16, HDL-32, HDL-64 and the 128-ring stress preset)
PRESETS = {16: (-15.0, 15.0, 16), 32: (-30.67, 10.67, 32), 64: (-24.9, 2.0, 64), 128: (-25.0, 15.0, 128)}


def config(**kw) -> dict:
    c = dict(DEFAULT)
    for k in kw:
        if k not in c:
            raise KeyError(k)
    c.update(kw)
    return c


def preset_config(rings: int, **kw) -> dict:
    lo, hi, r = PRESETS[rings]
    return config(lower_bound=lo, upper_bound=hi, num_rings=r, **kw)


# ---- angles -------------------------------------------------------------------------------------------------------------
def _ulp_shift(a: np.ndarray, k: int) -> np.ndarray:
    a = np.asarray(a, F32)
    for _ in range(abs(k)):
        a = np.nextafter(a, F32(np.inf) if k > 0 else F32(-np.inf))
    return a


def _near_midpoint(d64: np.ndarray) -> np.ndarray:
    """float64 values within AMBIG_ULPS float64 ulps of a float32 rounding midpoint (either neighbour)."""
    f = d64.astype(F32)
    lo = np.nextafter(f, F32(-np.inf)).astype(F64)
    hi = np.nextafter(f, F32(np.inf)).astype(F64)
    mid_lo, mid_hi = (f.astype(F64) + lo) / 2, (f.astype(F64) + hi) / 2
    tol = AMBIG_ULPS * np.spacing(np.abs(d64))
    return (np.abs(d64 - mid_lo) <= tol) | (np.abs(d64 - mid_hi) <= tol)


def raw_angles(xyz: np.ndarray):
    """float64 atan2 of the elevation (z over float32 dis) and of the azimuth (y over x)."""
    x, y, z = (np.asarray(xyz[:, a], F32) for a in range(3))
    dis = np.sqrt(x * x + y * y)
    return np.arctan2(z.astype(F64), dis.astype(F64)), np.arctan2(y.astype(F64), x.astype(F64))


def azimuth(atan_yx: np.ndarray) -> np.ndarray:
    """PointProcessor.cc:248-254 from the float atan2(y, x)."""
    azi = (TWO_PI - np.asarray(atan_yx, F32).astype(F64)).astype(F32)
    return np.where(azi.astype(F64) >= TWO_PI, (azi.astype(F64) - TWO_PI).astype(F32), azi)


def elevation_to_ring(ele: np.ndarray, cfg: dict) -> np.ndarray:
    """PointProcessor.h:153-156 with RadToDeg<float> (math_utils.h:38-41); int() truncates toward zero."""
    factor = F32(cfg["num_rings"] - 1) / (F32(cfg["upper_bound"]) - F32(cfg["lower_bound"]))
    deg = (np.asarray(ele, F32).astype(F64) * 180.0 / np.pi).astype(F32)
    v = ((deg - F32(cfg["lower_bound"])) * factor).astype(F64) + 0.5
    with np.errstate(invalid="ignore"):
        return np.trunc(v).astype(np.int64)


def rel_time(azi: np.ndarray, start_ori, scan_period: float) -> np.ndarray:
    """PointProcessor.cc:403-408."""
    rel = np.asarray(azi, F32) - F32(start_ori)
    rel = np.where(rel < 0, (rel.astype(F64) + TWO_PI).astype(F32), rel)
    return (scan_period * rel.astype(F64) / TWO_PI).astype(F32)


def encode(ring, rt, intensity):
    """The two intensity encodings, ring + rel_time and int(I) + rel_time (:414-415)."""
    laser = np.asarray(ring).astype(F32) + rt
    full = np.trunc(np.asarray(intensity, F32)).astype(F32) + rt
    return laser.astype(F32), full.astype(F32)


# ---- PointToRing ----------------------------------------------------------------------------------------------------------
def _finalise(xyzi, ring, accepted, point_azi, cfg, start_ori, rts, extra):
    R = cfg["num_rings"]
    idx = np.flatnonzero(accepted)
    order = idx[np.argsort(ring[idx], kind="stable")]         # stable: input order inside a ring
    counts = np.bincount(ring[idx], minlength=R)[:R]
    laser_i, full_i = encode(ring[order], rts[order], xyzi[order, 3])
    laser = np.concatenate([xyzi[order, :3], laser_i[:, None]], 1).astype(F32)
    full = np.concatenate([xyzi[order, :3], full_i[:, None]], 1).astype(F32)
    cs = np.cumsum(counts)
    scan_ranges = np.stack([cs - counts, np.where(cs > 0, cs - 1, 0)], 1).astype(np.int64)   # :196-200
    out = dict(laser_scans=laser, cloud_in_rings=full, idx_orig_index=order.astype(np.int64), scan_ranges=scan_ranges,
               start_ori=F32(start_ori), ring=ring, accepted=accepted, azi=point_azi)
    out.update(extra)
    return out


def point_to_ring(xyzi: np.ndarray, cfg: dict, shift=(0, 0)) -> dict:
    """PointToRing, elevation variant (PointProcessor.cc:207-426, non-DEBUG_ORIGIN).  shift = (elevation, azimuth) float32
    ulps added to the float atan2 results.  Per input point: ring (-1 when rejected), azimuth; ring-ordered clouds, orig,
    scan_ranges and start_ori."""
    xyzi = np.ascontiguousarray(xyzi, F32).reshape(-1, 4)
    n = xyzi.shape[0]
    finite = np.all(np.isfinite(xyzi[:, :3]), 1)
    safe = np.where(finite[:, None], xyzi[:, :3], F32(1))
    with np.errstate(invalid="ignore", over="ignore"):
        e64, a64 = raw_angles(safe)
    ele, atan = _ulp_shift(e64.astype(F32), shift[0]), _ulp_shift(a64.astype(F32), shift[1])
    ring = np.where(finite, elevation_to_ring(ele, cfg), -1)
    accepted = finite & (ring >= 0) & (ring < cfg["num_rings"])
    ring = np.where(accepted, ring, -1)
    azi = azimuth(atan)
    first = np.flatnonzero(accepted)
    start_ori = azi[first[0]] if first.size else F32(0)                      # :264-267
    rts = rel_time(azi, start_ori, cfg["scan_period"]) if n else np.zeros(0, F32)
    amb = finite & (_near_midpoint(e64) | _near_midpoint(a64))
    for k in (-1, 1):
        amb |= finite & (elevation_to_ring(_ulp_shift(e64.astype(F32), k), cfg) != elevation_to_ring(e64.astype(F32), cfg))
    return _finalise(xyzi, ring, accepted, azi, cfg, start_ori, rts, dict(ambiguous_in=amb))


def point_alternatives(xyzi: np.ndarray, cfg: dict, start_ori, rings=None, end_ori=None) -> dict:
    """For every input point and every (elevation, azimuth) shift in {-1, 0, 1}^2 float32 ulps: its ring and both intensity
    encodings against the given start_ori (and, for the ring-field variant, end_ori).  Arrays of shape (9, n)."""
    xyzi = np.ascontiguousarray(xyzi, F32).reshape(-1, 4)
    finite = np.all(np.isfinite(xyzi[:, :3]), 1)
    safe = np.where(finite[:, None], xyzi[:, :3], F32(1))
    e64, a64 = raw_angles(safe)
    ring_alt, lasers, fulls = [], [], []
    for de in (-1, 0, 1):
        for da in (-1, 0, 1):
            r = np.where(finite, elevation_to_ring(_ulp_shift(e64.astype(F32), de), cfg) if rings is None else rings, -1)
            r = np.where((r >= 0) & (r < cfg["num_rings"]), r, -1)
            azi = azimuth(_ulp_shift(a64.astype(F32), da))
            if rings is None:
                rt = rel_time(azi, start_ori, cfg["scan_period"])
            else:
                adj = np.where(azi - F32(start_ori) < 0, (azi.astype(F64) + TWO_PI).astype(F32), azi)
                with np.errstate(invalid="ignore", divide="ignore"):
                    rt = (cfg["scan_period"] * (adj - F32(start_ori)).astype(F64)
                          / F64(F32(end_ori) - F32(start_ori))).astype(F32)
            la, fu = encode(r, rt, xyzi[:, 3])
            ring_alt.append(r)
            lasers.append(la)
            fulls.append(fu)
    return dict(ring=np.stack(ring_alt), laser=np.stack(lasers), full=np.stack(fulls))


def point_to_ring_field(xyzi: np.ndarray, rings: np.ndarray, cfg: dict) -> dict:
    """PointToRing for PointXYZIR input (PointProcessor.cc:428-536).  The ring comes from the field and ids >= num_rings are
    dropped; an azimuth before start_ori_ gets + 2 pi (the half_passed branch needs i > 3 * cloud_size / 2, which no i
    reaches); end_ori_ is the largest adjusted azimuth, from 0; rel_time = scan_period * (azi - start_ori_) / range_ori.  When
    every azimuth equals start_ori_ the range is 0 and rel_time is 0 / 0, as in the reference."""
    xyzi = np.ascontiguousarray(xyzi, F32).reshape(-1, 4)
    rings = np.asarray(rings, np.int64)
    finite = np.all(np.isfinite(xyzi[:, :3]), 1)
    safe = np.where(finite[:, None], xyzi[:, :3], F32(1))
    e64, a64 = raw_angles(safe)
    azi = azimuth(a64.astype(F32))
    accepted = finite & (rings >= 0) & (rings < cfg["num_rings"])
    ring = np.where(accepted, rings, -1)
    first = np.flatnonzero(accepted)
    start_ori = azi[first[0]] if first.size else F32(0)
    adj = np.where(azi - F32(start_ori) < 0, (azi.astype(F64) + TWO_PI).astype(F32), azi)     # :481-488
    end_ori = F32(0)
    if first.size:
        end_ori = max(end_ori, adj[accepted].max())                                          # :497-499
    range_ori = F32(end_ori) - F32(start_ori)
    with np.errstate(invalid="ignore", divide="ignore"):
        rts = (cfg["scan_period"] * (adj - F32(start_ori)).astype(F64) / F64(range_ori)).astype(F32)
    amb = finite & _near_midpoint(a64)
    return _finalise(xyzi, ring, accepted, azi, cfg, start_ori, rts, dict(ambiguous_in=amb, end_ori=F32(end_ori)))


# ---- ExtractFeaturePoints --------------------------------------------------------------------------------------------------
def _sqdiff(a, b, wb=None):
    if wb is None:
        d = a - b
    else:
        d = a - b * wb[:, None]
    return d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]


def _sq_dist(p):
    return p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]


def prepare_ring(p: np.ndarray, d: int) -> np.ndarray:
    """PrepareRing (:542-585) for i in [d, n - d).  Returns n + 1 mask slots: the reference's fill for i = n - d - 1 in the
    far-point branch reaches one past the ring."""
    n = p.shape[0]
    mask = np.zeros(n + 1, np.uint8)
    i = np.arange(d, n - d)
    cur, nxt, prv = p[i], p[i + 1], p[i - 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        dn2 = _sqdiff(cur, nxt)
        depth, depth_next = np.sqrt(_sq_dist(cur)), np.sqrt(_sq_dist(nxt))
        closer = depth > depth_next
        wd_a = np.sqrt(_sqdiff(nxt, cur, depth_next / depth)) / depth_next
        wd_b = np.sqrt(_sqdiff(cur, nxt, depth / depth_next)) / depth
        far = dn2.astype(F64) > 0.1
        occl_a = far & closer & (wd_a.astype(F64) < 0.1)
        occl_b = far & ~closer & (wd_b.astype(F64) < 0.1)
        dp2 = _sqdiff(cur, prv)
        dis2 = _sq_dist(cur).astype(F64)
        par = ~occl_a & ~occl_b & (dn2.astype(F64) > 0.0002 * dis2) & (dp2.astype(F64) > 0.0002 * dis2)
    for k in range(d + 1):
        mask[i[occl_a] - d + k] = 1
        mask[i[occl_b] + 1 + k] = 1
    mask[i[par]] = 1
    return mask


def curvature(p: np.ndarray, d: int) -> np.ndarray:
    """PrepareSubregion's curvature (:598-609) for every i in [d, n - d): -2d * x, then + (x[i+j] + x[i-j]) for j = 1..d."""
    n = p.shape[0]
    i = np.arange(d, n - d)
    acc = F32(-2 * d) * p[i, :3]
    for j in range(1, d + 1):
        acc = acc + (p[i + j, :3] + p[i - j, :3])
    c = np.zeros(n, F32)
    c[i] = acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1] + acc[:, 2] * acc[:, 2]
    return c


def mask_picked(p: np.ndarray, mask: np.ndarray, idx: int, d: int) -> None:
    """MaskPickedInRing (:624-645)."""
    mask[idx] = 1
    for s in (1, -1):
        for k in range(1, d + 1):
            a, b = p[idx + s * k], p[idx + s * (k - 1)]
            dd = a[:3] - b[:3]
            if F64(dd[0] * dd[0] + dd[1] * dd[1] + dd[2] * dd[2]) > 0.05:
                break
            mask[idx + s * k] = 1


def extract_features(pr: dict, cfg: dict) -> dict:
    """ExtractFeaturePoints (:647-783) on the output of point_to_ring / point_to_ring_field.  Adds mask, labels, the three
    index sets and their clouds, the less-flat cloud and `picks`: one record per pick (ring, subregion, kind, position in the
    walk order of the sorted subregion, position just after the previous pick) and per walk its first position failing
    the curvature test (`stop`), or None."""
    laser = pr["laser_scans"]
    N = laser.shape[0]
    d, S = cfg["num_curvature_regions"], cfg["num_scan_subregions"]
    th = F32(cfg["surf_curv_th"])
    mask_all = np.zeros(N, np.uint8)
    labels = np.zeros(N, np.int8)
    sharp, less, flat, picks, walks = [], [], [], [], []
    for r, (start, end) in enumerate(pr["scan_ranges"]):
        if end <= start + 2 * d:                                   # :660
            continue
        p = laser[start:end + 1]
        n = p.shape[0]
        mask = prepare_ring(p, d)
        curv = curvature(p, d)
        for j in range(S):
            sp, ep = _sub(n, d, S, j)
            if ep <= sp:
                continue
            ids = np.arange(sp, ep + 1)
            srt = ids[np.lexsort((ids, curv[ids]))]                # std::sort of pair<float, size_t>
            lab = np.zeros(ep - sp + 1, np.int8)
            for kind in ("corner", "flat"):
                walk = srt[::-1] if kind == "corner" else srt
                cap = cfg["max_corner_less_sharp"] if kind == "corner" else cfg["max_surf_flat"]
                got, prev, stop = 0, 0, None
                for pos, idx in enumerate(walk):
                    if got >= cap:
                        break
                    c = curv[idx]
                    passes = c > th if kind == "corner" else c < th
                    if not passes and stop is None:
                        stop = pos
                    if mask[idx] == 0 and passes:
                        got += 1
                        if kind == "corner":
                            lab[idx - sp] = 2 if got <= cfg["max_corner_sharp"] else 1
                            if got <= cfg["max_corner_sharp"]:
                                sharp.append(start + idx)
                            less.append(start + idx)
                        else:
                            lab[idx - sp] = -1
                            flat.append(start + idx)
                        picks.append(dict(ring=r, sub=j, kind=kind, pos=pos, after=prev))
                        prev = pos + 1
                        mask_picked(p, mask, idx, d)
                walks.append(dict(ring=r, sub=j, kind=kind, picked=got, stop=stop, size=ep - sp + 1))
            labels[start + sp:start + ep + 1] = lab
        mask_all[start:end + 1] = mask[:n]
    out = dict(pr)
    out.update(mask=mask_all, labels=labels, picks=picks, walks=walks)
    for name, ids in (("sharp", sharp), ("less_sharp", less), ("flat", flat)):
        ids = np.asarray(ids, np.int64)
        out["idx_" + name] = ids
        out[name] = laser[ids]
    out["less_flat"], _ = less_flat_cloud(laser, pr["scan_ranges"], labels, d, S, cfg["less_flat_filter_size"],
                                          pr["start_ori"], cfg["scan_period"])
    return out


def _sub(n: int, d: int, S: int, j: int):
    """Subregion j's (sp, ep) in the reference's size_t arithmetic (:672-675); ep <= sp means skipped."""
    sp = (d * (S - j) + (n - d) * j) // S
    ep = (d * (S - 1 - j) + (n - d) * (j + 1)) // S - 1
    return sp, ep


def process(xyzi: np.ndarray, cfg: dict | None = None, rings: np.ndarray | None = None) -> dict:
    """PointToRing (elevation or ring-field variant) + ExtractFeaturePoints.  `ambiguous` is ring-ordered."""
    cfg = cfg or config()
    pr = point_to_ring(xyzi, cfg) if rings is None else point_to_ring_field(xyzi, rings, cfg)
    out = extract_features(pr, cfg)
    out["ambiguous"] = pr["ambiguous_in"][pr["idx_orig_index"]]
    return out


def chunk_skips(out: dict, kind: str):
    """Picks reached only after a full 32-candidate chunk of masked candidates that still pass the curvature test."""
    return [p for p in out["picks"] if p["kind"] == kind and p["pos"] - p["after"] >= 32]


def stop_breaks(out: dict, kind: str):
    """Walks that meet a candidate failing the curvature test before they run out of their pick budget."""
    return [w for w in out["walks"] if w["kind"] == kind and w["stop"] is not None]


# ---- edge inputs ------------------------------------------------------------------------------------------------------------
def _factor(cfg):
    return F32(cfg["num_rings"] - 1) / (F32(cfg["upper_bound"]) - F32(cfg["lower_bound"]))


def ring_elevation(cfg: dict, ring: int) -> float:
    """Elevation (rad) at the centre of a ring's bucket."""
    return float(np.radians(cfg["lower_bound"] + ring / float(_factor(cfg))))


def _points_at(ele32: np.ndarray, azi: np.ndarray, dis: np.ndarray) -> np.ndarray:
    """float32 points whose float32 elevation angle equals ele32 where a z within 16 float32 ulps reaches it (else the
    nearest), at the given azimuths and horizontal distances."""
    x = (dis * np.cos(azi)).astype(F32)
    y = (dis * np.sin(azi)).astype(F32)
    d32 = np.sqrt(x * x + y * y)
    z0 = (d32.astype(F64) * np.tan(ele32.astype(F64))).astype(F32)
    best, err = z0.copy(), np.full(z0.shape, np.inf)
    for k in range(-16, 17):
        z = _ulp_shift(z0, k)
        e = np.arctan2(z.astype(F64), d32.astype(F64))
        cand = np.abs(e - ele32.astype(F64))
        better = cand < err
        best, err = np.where(better, z, best), np.where(better, cand, err)
    return np.stack([x, y, best], 1)


def bucket_edges(cfg: dict):
    """Every float32 elevation where the ring id changes (ring k - 1 to k for k = -1 .. num_rings + 1 in v terms), found
    by walking float32 values around the nominal edge."""
    factor = float(_factor(cfg))
    out = []
    for k in range(-1, cfg["num_rings"] + 1):
        e = F32(np.radians(cfg["lower_bound"] + (k - 0.5) / factor))
        walk = np.array([_ulp_shift(e, s) for s in range(-96, 97)], F32)
        r = elevation_to_ring(walk, cfg)
        for t in np.flatnonzero(r[1:] != r[:-1]):
            out.append(walk[t + 1])
    return np.unique(np.asarray(out, F32))


def _with_intensity(xyz, rng, lo=0.0, hi=100.0):
    return np.concatenate([np.asarray(xyz, F32), rng.uniform(lo, hi, (len(xyz), 1)).astype(F32)], 1)


def bucket_edge_cloud(rings: int, seed: int = 0) -> np.ndarray:
    """Points on, and 1 and 2 float32 ulps either side of, every bucket edge of a preset (below ring 0 down to the last
    accepted value, and just above the top ring), at several azimuths and ranges, plus ring-centre points so that every
    ring also holds ordinary points; input order shuffled."""
    cfg = preset_config(rings)
    rng = np.random.default_rng(seed)
    eles = np.concatenate([_ulp_shift(e, s)[None] for e in bucket_edges(cfg) for s in (-2, -1, 0, 1, 2)])
    eles = np.repeat(eles, 3)
    centre = np.repeat(np.array([ring_elevation(cfg, r) for r in range(rings)], F32), 4)
    # half a bucket below ring 0: accepted by the truncation toward zero
    below = np.array([ring_elevation(cfg, 0) - np.radians(f / float(_factor(cfg))) for f in (0.75, 1.0, 1.25, 1.45)], F32)
    eles = np.concatenate([eles, centre, np.repeat(below, 3)])
    azi = rng.uniform(-np.pi, np.pi, eles.shape[0])
    dis = rng.uniform(2.0, 60.0, eles.shape[0])
    xyz = _points_at(eles, azi, dis)
    return _with_intensity(xyz[rng.permutation(xyz.shape[0])], rng)


def azimuth_wrap_cloud(rings: int, seed: int = 0) -> np.ndarray:
    """Points whose azimuth sits on its special values, all at a ring centre: y = +-0 with x < 0 and x > 0, x = +-0, y one
    float32 step either side of 0 (2 pi - atan2 rounds to 2 pi and wraps), and the first point at an azimuth just below
    2 pi, so that later points fall on both sides of start_ori."""
    cfg = preset_config(rings)
    rng = np.random.default_rng(seed)
    e = ring_elevation(cfg, rings // 2)
    t = np.float32(np.tan(e))
    tiny = np.float32(1e-30)
    xy = [(1.0, -1e-3), (-3.0, 0.0), (-3.0, -0.0), (3.0, 0.0), (3.0, -0.0), (0.0, 2.0), (-0.0, 2.0), (0.0, -2.0), (-0.0, -2.0),
          (5.0, tiny), (5.0, -tiny), (5.0, np.float32(1e-7)), (5.0, np.float32(-1e-7)), (-5.0, tiny), (-5.0, -tiny)]
    xy = xy + [(float(np.cos(a) * 7), float(np.sin(a) * 7)) for a in rng.uniform(-np.pi, np.pi, 40)]
    xy = np.asarray(xy, F32)
    dis = np.sqrt(xy[:, 0] * xy[:, 0] + xy[:, 1] * xy[:, 1])
    z = (dis * t).astype(F32)
    return _with_intensity(np.concatenate([xy, z[:, None]], 1), rng)


def first_point_cases(rings: int, seed: int = 0):
    """(name, cloud): a ring-centre cloud whose first point is NaN, or is finite but outside every ring, so that
    start_ori_ comes from a later point."""
    cfg = preset_config(rings)
    rng = np.random.default_rng(seed)
    n = 64 * rings
    ring = rng.integers(0, rings, n)
    eles = np.array([ring_elevation(cfg, r) for r in ring], F32)
    xyz = _points_at(eles, rng.uniform(-np.pi, np.pi, n), rng.uniform(3.0, 40.0, n))
    base = _with_intensity(xyz, rng)
    nan = base.copy()
    nan[0, 1] = np.nan
    high = base.copy()
    high[0, :3] = _points_at(np.array([np.radians(cfg["upper_bound"] + 20.0)], F32), np.array([1.0]), np.array([5.0]))[0]
    low = base.copy()
    low[:2, :3] = _points_at(np.array([np.radians(cfg["lower_bound"] - 20.0)] * 2, F32), np.array([2.0, -2.0]), np.array([5.0, 6.0]))
    return [("first_nan", nan), ("first_above", high), ("first_two_below", low)]


# A ring in the z = 0 plane: the elevation is exactly 0, which is ring 8 of the 16-ring preset (v = 8 exactly) whatever the
# atan2's rounding.  Coordinates are multiples of 1/64 so that straight runs are exactly collinear and equally spaced.
def _zigzag(n, x0, y0, step=0.0625, amp=0.25):
    i = np.arange(n)
    return np.stack([x0 + amp * (i % 2), y0 + step * i], 1)


def _line(n, x0, y0, dx, dy):
    i = np.arange(n)
    return np.stack([x0 + dx * i, y0 + dy * i], 1)


def pick_block(y0: float) -> np.ndarray:
    """One block of the pick ring (x, y), in ring order:
       radial   48 points on a radial line 0.375 m apart: curvature exactly 0 and masked by PrepareRing's 0.0002 * dis^2 test
       zigzag   40 points with 0.25 m radial saw-teeth: high curvature, every point masked by the same test
       kink     a tangential line that bends by 90 degrees: the corner candidates left once the zig-zag is masked
       dup      12 copies of one point
       tangent  40 points on a tangential line 1/16 m apart: curvature exactly 0 and unmasked (flat candidates tied at 0)"""
    rad = _line(48, 6.0, y0, 0.375, 0.0)
    z = _zigzag(40, 10.0, y0 + 0.5)
    k1 = _line(12, 10.0, y0 + 3.0, 0.0, 0.0625)
    k2 = _line(12, 10.0 - 0.0625, y0 + 3.0 + 11 * 0.0625, -0.0625, 0.0)
    dup = np.repeat([[10.0, y0 + 5.0]], 12, 0)
    tan = _line(40, 10.0, y0 + 5.5, 0.0, 0.0625)
    return np.concatenate([rad, z, k1, k2, dup, tan])


def pick_ring(blocks: int, seed: int = 0, intensity=(0.0, 100.0)) -> np.ndarray:
    """`blocks` pick blocks one after another, as a z = 0 ring (ring 8 of the 16-ring preset).  Blocks alternate between two
    lateral offsets and turn by 90 degrees every second block (exact in float32), so every point stays within 26 m."""
    rng = np.random.default_rng(seed)
    parts = []
    for b in range(blocks):
        xy = pick_block(-8.0 if b % 2 == 0 else 0.0)
        for _ in range((b // 2) % 4):
            xy = np.stack([-xy[:, 1], xy[:, 0]], 1)
        parts.append(xy)
    xy = np.concatenate(parts)
    xyz = np.concatenate([xy, np.zeros((xy.shape[0], 1))], 1)
    return _with_intensity(xyz, rng, *intensity)


def plane_ring(n: int, seed: int = 0, occlusion: bool = True) -> np.ndarray:
    """n points of a z = 0 ring along a wavy wall with occlusion steps towards and away from the sensor, and intensities
    that are negative and fractional."""
    rng = np.random.default_rng(seed)
    a = np.linspace(-2.5, 2.5, n)
    r = 8.0 + 0.3 * np.sin(7 * a) + 0.02 * rng.standard_normal(n)
    if occlusion:
        r = r + np.where((np.arange(n) // 97) % 3 == 1, -3.0, 0.0)
    xyz = np.stack([r * np.cos(a), r * np.sin(a), np.zeros(n)], 1)
    return _with_intensity(xyz, rng, -50.0, 50.0)


def centre_ring_cloud(cfg: dict, ring: int, n: int, seed: int = 0) -> np.ndarray:
    """n points of one ring at its bucket centre, azimuth in order, on a wavy wall."""
    rng = np.random.default_rng(seed)
    a = np.linspace(-3.0, 3.0, n)
    r = 12.0 + 0.5 * np.sin(5 * a) + 0.05 * rng.standard_normal(n)
    return _with_intensity(_points_at(np.full(n, ring_elevation(cfg, ring), F32), a, r), rng)


def interleaved_rings(cfg: dict, per_ring: np.ndarray, seed: int = 0) -> np.ndarray:
    """Every ring r holds per_ring[r] points in azimuth order on a wavy wall; the rings' points are interleaved in a
    random sequence (each ring keeps its own order), so that every classify / scatter block holds many rings."""
    rng = np.random.default_rng(seed)
    R = len(per_ring)
    seq = rng.permutation(np.repeat(np.arange(R), per_ring))
    rank = np.zeros_like(seq)
    for r in range(R):
        rank[seq == r] = np.arange(per_ring[r])
    frac = (rank + rng.uniform(0.0, 0.5, seq.shape[0])) / np.maximum(np.asarray(per_ring)[seq], 1)
    a = -np.pi + 2 * np.pi * frac
    rr = 15.0 + 2.0 * np.sin(4 * a + seq) + 0.05 * rng.standard_normal(seq.shape[0])
    eles = np.array([ring_elevation(cfg, r) for r in range(R)], F32)[seq]
    return _with_intensity(_points_at(eles, a, rr), rng, -20.0, 120.0)


def ring_field_cases(seed: int = 0):
    """(name, cloud, ring field) of the 16-ring preset: ids 0, 15, 16 and 65535 in one cloud; the first point at an azimuth
    just below 2 pi (every later point is adjusted by + 2 pi); every azimuth equal (range_ori = 0)."""
    cfg = preset_config(16)
    rng = np.random.default_rng(seed)
    per = np.full(16, 60)
    cloud = interleaved_rings(cfg, per, seed)
    ids = elevation_to_ring(raw_angles(cloud)[0].astype(F32), cfg).astype(np.int64)
    ids[::37] = 16
    ids[5::41] = 65535
    out = [("ids", cloud, ids.astype(np.uint16))]
    near = cloud.copy()
    near[0, :3] = [9.0, 1e-6, 1.0]
    near_ids = ids.copy()
    near_ids[0] = 3
    out.append(("start_near_2pi", near, near_ids.astype(np.uint16)))
    k = rng.integers(0, 6, 400)
    xy = np.stack([np.ldexp(1.0, k), np.ldexp(1.0, k - 1)], 1)
    z = rng.uniform(-1.0, 1.0, (400, 1))
    eq = _with_intensity(np.concatenate([xy, z], 1), rng, -5.0, 5.0)
    out.append(("equal_azimuths", eq, rng.integers(0, 16, 400).astype(np.uint16)))
    return out
