"""The map of a whole drive in HBM (csrc/regmap.cu, lio_rm_*; src/save_bag_to_pcd.cc): raw mode bit-equal to np.concatenate,
voxel mode bit-equal to a NumPy statement (float32 keys, np.add.at on float64 sums, first-seen ids), the capacity rule, inserts
without host waits and with a fixed launch count, the lidar chain, the map builder and the estimator's attached map feeding it
from HBM, and the PCD file it writes."""
import numpy as np
import pytest

from lio_mapping_b200 import synth
from lio_mapping_b200.registered_map import RegisteredMap

pytestmark = pytest.mark.gpu

RANGE = 1 << 20
VOXEL_LAUNCHES = 17


def voxel_statement(clouds, leaf):
    """The voxel-mode map of these inserts in arrival order: keys floor(c * (1 / leaf)) in float32, points with a non-finite
    coordinate or a key outside [-2^20, 2^20) dropped, ids in first-seen order, sums by np.add.at in float64."""
    pts = np.concatenate([np.asarray(c, np.float32).reshape(-1, 4) for c in clouds] + [np.zeros((0, 4), np.float32)])
    inv = np.float32(1) / np.float32(leaf)
    with np.errstate(invalid="ignore", over="ignore"):
        v = np.floor(pts[:, :3] * inv)
        ok = np.isfinite(pts[:, :3]).all(1) & (v >= -RANGE).all(1) & (v < RANGE).all(1)
    p, key = pts[ok], v[ok].astype(np.int64)
    if p.shape[0] == 0:
        return np.zeros((0, 4), np.float32)
    _, first, inverse = np.unique(key, axis=0, return_index=True, return_inverse=True)
    rank = np.empty(first.shape[0], np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(first.shape[0])
    ids = rank[inverse.reshape(-1)]
    sums = np.zeros((first.shape[0], 4), np.float64)
    np.add.at(sums, ids, p.astype(np.float64))
    cnt = np.bincount(ids).astype(np.float64)
    return (sums / cnt[:, None]).astype(np.float32)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def to_dev(cloud):
    import torch
    return torch.from_numpy(np.ascontiguousarray(cloud, np.float32).reshape(-1, 4).copy()).cuda()


def insert_all(rm, clouds, dev=True):
    keep = []
    for c in clouds:
        if dev:
            t = to_dev(c)
            keep.append(t)
            rm.insert_dev(t.data_ptr(), t.shape[0])
        else:
            rm.insert(c)
    return keep


def random_cloud(rng, n, scale=50.0):
    c = np.empty((n, 4), np.float32)
    c[:, :3] = rng.uniform(-scale, scale, (n, 3))
    c[:, 3] = rng.uniform(0, 100, n)
    return c


def test_raw_mode_is_the_concatenation():
    rng = np.random.default_rng(1)
    sizes = [0, 17, 3000, 1, 0, 5000, 2000]   # 8018 of 10000, then one cloud larger than what is left
    clouds = [random_cloud(rng, n) for n in sizes]
    clouds[2][5] = [np.nan, 1, 2, 3]; clouds[2][6] = [np.inf, -np.inf, 0, np.nan]   # kept, as the reference tool keeps them
    for dev in (True, False):
        rm = RegisteredMap(0.0, 10000)
        insert_all(rm, clouds[:6], dev)
        s = rm.stats()
        assert s["size"] == 8018 and s["overflow"] == 0 and s["inserts"] == 6 and s["offered"] == 8018
        assert same_bits(rm.download(), np.concatenate(clouds[:6]))
        insert_all(rm, clouds[6:], dev)   # refused: changes nothing, sets the flag
        insert_all(rm, [clouds[1]], dev)  # blocked
        s = rm.stats()
        assert s["size"] == 8018 and s["overflow"] == 1 and s["inserts"] == 8
        out = rm.download()
        assert same_bits(out, np.concatenate(clouds[:6]))
        if dev:
            ref = out
        else:
            assert same_bits(out, ref)   # _dev and _host give the same map
        rm.reset()
        s = rm.stats()
        assert s["size"] == 0 and s["overflow"] == 0
        insert_all(rm, clouds[6:], dev)
        assert same_bits(rm.download(), clouds[6])
        rm.close()


def _voxel_inputs():
    rng = np.random.default_rng(7)
    random = [random_cloud(rng, n) for n in (1000, 0, 25000, 7)]
    dense = [random_cloud(rng, 20000, 3.0) for _ in range(3)]     # ~hundreds of points per 0.2 m ... 1 m voxel
    # points on voxel boundaries and at negative coordinates: multiples of the leaf in float32 and their neighbours
    g = (np.arange(-40, 40, dtype=np.float32) * np.float32(0.2)).astype(np.float32)
    edge = np.stack(np.meshgrid(g, g[::3], g[::7], indexing="ij"), -1).reshape(-1, 3)
    edge = np.concatenate([edge, np.nextafter(edge, np.float32(-np.inf)), np.nextafter(edge, np.float32(np.inf))])
    edge = np.c_[edge, rng.uniform(0, 1, edge.shape[0]).astype(np.float32)].astype(np.float32)
    bad = random_cloud(rng, 3000)
    bad[::7, 0] = np.nan; bad[1::11, 1] = np.inf; bad[2::13, 2] = -np.inf; bad[3::17, 3] = np.nan   # a NaN intensity is kept
    return random, dense, [edge], [bad]


@pytest.mark.parametrize("leaf", [0.2, 1.0, 0.05])
def test_voxel_mode_equals_the_numpy_statement(leaf):
    random, dense, edge, bad = _voxel_inputs()
    for clouds in (random, dense, edge, bad, random + dense + edge + bad):
        for dev in (True, False):
            rm = RegisteredMap(leaf, 1 << 20)
            insert_all(rm, clouds, dev)
            ref = voxel_statement(clouds, leaf)
            got = rm.download()
            assert same_bits(got, ref), (leaf, len(clouds), got.shape, ref.shape)
            s = rm.stats()
            offered = sum(c.shape[0] for c in clouds)
            assert s["size"] == ref.shape[0] and s["offered"] == offered and s["accepted"] + s["dropped"] == offered
            rm.close()


def test_voxel_keys_beyond_the_range_are_dropped():
    leaf = 1.0
    r = float(RANGE)
    c = np.array([[-r, 0, 0, 1], [-r - 1, 0, 0, 2], [r - 0.5, 0, 0, 3], [r, 0, 0, 4], [0, r - 1, -r, 5], [0, 0, r + 8, 6],
                  [0, 3e30, 0, 7], [-5e9, 1, 1, 8], [1.5, -0.5, -r, 9]], np.float32)
    rm = RegisteredMap(leaf, 100)
    insert_all(rm, [c])
    assert same_bits(rm.download(), voxel_statement([c], leaf))
    s = rm.stats()
    assert s["size"] == 4 and s["accepted"] == 4 and s["dropped"] == 5
    # 0.1 m leaf over a 120 km extent: keys up to 1.2e6 per axis, where PCL's 32-bit index has long overflowed
    rng = np.random.default_rng(3)
    far = random_cloud(rng, 20000, 1.2e5)
    rm2 = RegisteredMap(0.1, 1 << 16)
    insert_all(rm2, [far])
    assert same_bits(rm2.download(), voxel_statement([far], 0.1))
    assert 0 < rm2.stats()["dropped"] < 20000


def test_one_voxel_across_many_inserts_sums_in_arrival_order():
    """Intensities of +-1e15 between small ones in one voxel: the float64 sums cancel, so another order of the additions gives
    another mean."""
    rng = np.random.default_rng(11)
    clouds = []
    for k in range(40):
        n = 3 * int(rng.integers(1, 100))
        c = np.zeros((n, 4), np.float32)
        c[:, :3] = rng.uniform(0.0, 0.19, (n, 3)).astype(np.float32) * rng.choice([1e-7, 1.0, 1e-3], (n, 1)).astype(np.float32)
        big = np.where(np.arange(n) % 3 == 0, 1e15, np.where(np.arange(n) % 3 == 1, -1e15, 0.0))
        c[:, 3] = np.where(np.arange(n) % 3 == 2, rng.uniform(0.0, 1.0, n), big)
        clouds.append(c)
    rm = RegisteredMap(0.2, 16)
    insert_all(rm, clouds)
    got = rm.download()
    assert got.shape == (1, 4) and same_bits(got, voxel_statement(clouds, 0.2))
    assert not same_bits(voxel_statement([np.concatenate(clouds)[::-1]], 0.2), got)   # the inputs tell the orders apart


def test_repeatable():
    random, dense, edge, bad = _voxel_inputs()
    clouds = dense + random + bad + edge + dense
    out = []
    for _ in range(2):
        rm = RegisteredMap(0.2, 1 << 20)
        insert_all(rm, clouds)
        out.append(rm.download())
        rm.close()
    assert same_bits(out[0], out[1])


def test_capacity_refuses_the_whole_insert():
    rng = np.random.default_rng(5)
    a = random_cloud(rng, 4000, 2.0)    # 4 x 4 x 4 voxels of 1 m
    b = random_cloud(rng, 4000, 2.0) + np.array([10, 0, 0, 0], np.float32)   # 64 new voxels
    rm = RegisteredMap(1.0, 100)
    insert_all(rm, [a])
    before = rm.download()
    assert before.shape[0] == 64 and rm.stats()["overflow"] == 0
    insert_all(rm, [b])                  # 64 + 64 > 100: nothing changes
    s = rm.stats()
    assert s["overflow"] == 1 and s["size"] == 64 and s["accepted"] == 4000
    insert_all(rm, [a[:10]])             # only old voxels, but the flag blocks it
    assert rm.stats()["accepted"] == 4000 and same_bits(rm.download(), before)
    rm.reset()
    s = rm.stats()
    assert s["overflow"] == 0 and s["size"] == 0 and rm.download().shape == (0, 4)
    insert_all(rm, [b, a[:10]])
    assert same_bits(rm.download(), voxel_statement([b, a[:10]], 1.0))
    exact = RegisteredMap(1.0, 64)       # size + misses == capacity is accepted
    insert_all(exact, [a, a])
    assert exact.stats()["overflow"] == 0 and same_bits(exact.download(), voxel_statement([a, a], 1.0))


@pytest.mark.parametrize("leaf", [0.0, 0.2])
def test_inserts_never_wait_and_launch_a_fixed_count(leaf):
    import torch
    rng = np.random.default_rng(9)
    sizes = [0, 1, 5000, 130000, 300000, 7, 0, 65536, 2048, 2049]   # the scratch grows twice on the way
    clouds = [to_dev(random_cloud(rng, n)) for n in sizes]
    torch.cuda.synchronize()
    rm = RegisteredMap(leaf, 1 << 21)
    w0 = rm.stats()["waits"]
    for t in clouds:
        rm.insert_dev(t.data_ptr(), t.shape[0])
    assert rm.stats()["waits"] == w0 + 1      # the stats call's own wait only
    for t in clouds:
        rm.insert_dev(t.data_ptr(), t.shape[0])
        assert rm.stats()["launches"] == (VOXEL_LAUNCHES if leaf else 1)
    host = [t.cpu().numpy() for t in clouds]
    ref = np.concatenate(host + host) if leaf == 0 else voxel_statement(host + host, leaf)
    assert same_bits(rm.download(), ref)


def test_errors():
    from lio_mapping_b200 import _lib
    L = _lib.lib()
    import ctypes as C
    h = C.c_void_p()
    for leaf, cap in ((-0.1, 10), (float("nan"), 10), (0.2, 0), (0.0, -5), (0.2, (1 << 30) + 1), (1e-45, 10)):
        assert L.lio_rm_create(leaf, cap, 0, None, C.byref(h)) == -2, (leaf, cap)
    rm = RegisteredMap(0.2, 10)
    assert L.lio_rm_insert_dev(rm.h, None, 5) == -2 and L.lio_rm_insert_dev(rm.h, None, -1) == -2
    n = C.c_longlong()
    assert L.lio_rm_download(rm.h, np.zeros((1, 4), np.float32), -1, C.byref(n)) == -2
    rm.insert(np.ones((3, 4), np.float32) * np.arange(3, dtype=np.float32)[:, None])
    assert L.lio_rm_download(rm.h, np.zeros((1, 4), np.float32), 1, C.byref(n)) == -3 and n.value == 3


# ---- the registered clouds of the device pipelines -------------------------------------------------------------------------

STAGE_A = ("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat", "surface_points_less_flat", "cloud_in_rings")


def _check_chain(maps, acc):
    raw, vox = maps
    assert raw.stats()["waits"] == 1 and vox.stats()["waits"] == 1   # no insert waited: this stats call is the first wait
    assert sum(a.shape[0] for a in acc) > 0
    assert same_bits(raw.download(), np.concatenate(acc))
    assert same_bits(vox.download(), voxel_statement(acc, 0.2))
    s = vox.stats()
    assert s["launches"] == VOXEL_LAUNCHES and s["overflow"] == 0


def test_lidar_chain_registered_clouds():
    """Stage A -> PointOdometry -> publishing PointMapping in HBM over 20 HDL-64 sweeps: inserting lio_mb_full_dev after every
    mapped sweep equals accumulating lio_mb_full_download on the host."""
    import torch
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    from lio_mapping_b200.point_processor import PointProcessor
    sensor, scene, traj = synth.default_config("hdl64")
    raw = [np.ascontiguousarray(synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * f, seed=70 + f, distort=True), np.float32)
           for f in range(20)]
    max_raw = max(r.shape[0] for r in raw)
    pp = PointProcessor(sensor.lower_deg, sensor.upper_deg, sensor.rings, max_points=max_raw)
    n_dev = [pp.cloud_count_dev(name) for name in STAGE_A]
    od = PointOdometry(0.1, 1, 25, max_full_points=max_raw)
    pm = PointMapping(max_points=1 << 17)
    pm.EnablePublish(0.6, max_raw)
    maps = (RegisteredMap(0.0, 20 * max_raw), RegisteredMap(0.2, 1 << 22))
    acc = []
    for r in raw:
        t = torch.from_numpy(r).cuda()
        pp.process_device(t.data_ptr(), t.shape[0])
        ts, _, info = od.ProcessDev([pp.cloud_dev(name) for name in STAGE_A], n_dev, [1 << 17] * 4 + [max_raw])
        if not info["published"]:
            continue
        ptrs, cn_dev, cn = od.clouds_dev()
        pm.ProcessDev(ptrs, cn_dev, cn, ts)
        for m in maps:
            m.insert_dev(*pm.registered_full_cloud_dev())
        acc.append(pm.registered_full_cloud())
    assert len(acc) >= 10
    _check_chain(maps, acc)


def test_map_builder_registered_clouds(oracle):
    from lio_mapping_b200.map_builder import MapBuilder
    from tests.test_oracle_map_builder import mapping_frames
    frames = mapping_frames(oracle, "hdl64", 12)
    mb = MapBuilder(max_points=1 << 17, max_full_points=max(fr[2].shape[0] for fr in frames))
    maps = (RegisteredMap(0.0, 1 << 22), RegisteredMap(0.2, 1 << 22))
    acc = []
    for corner, surf, full, tf_odom, _ in frames:
        mb.ProcessMap(corner, surf, full, tf_odom)
        for m in maps:
            m.insert_dev(*mb.registered_full_cloud_dev())
        acc.append(mb.registered_full_cloud())
    _check_chain(maps, acc)


def test_estimator_attached_map_registered_clouds(oracle):
    from tests.test_global_map_gpu import _Setup
    W, O = 5, 4
    s = _Setup(oracle, W, O, O + 5, opt_extrinsic=0)
    s.eg.attach_map(s.pm)
    maps = (RegisteredMap(0.0, 1 << 22), RegisteredMap(0.2, 1 << 22))
    acc = []
    for i in range(O + 5):
        k = W + i
        s.eg.set_scan_clouds(s.corner[k], s.full[k])
        s.imu(s.eg, k)
        s.eg.process_scan(s.less_flat(k))
        for m in maps:
            m.insert_dev(*s.pm.registered_full_cloud_dev())
        acc.append(s.pm.registered_full_cloud())
    _check_chain(maps, acc)


# ---- PCD -----------------------------------------------------------------------------------------------------------------

def read_pcd(path):
    """A small binary PCD reader: the header as a dict of its lines (and their order), then the records."""
    data = open(path, "rb").read()
    lines, pos = [], 0
    while True:
        end = data.index(b"\n", pos)
        lines.append(data[pos:end].decode())
        pos = end + 1
        if lines[-1].startswith("DATA"):
            break
    head = {ln.split(" ", 1)[0]: ln.split(" ", 1)[1] for ln in lines[1:]}
    n = int(head["POINTS"])
    fields = head["FIELDS"].split()
    rec = np.dtype([(f, "<f4") for f in fields])
    assert len(data) - pos == n * rec.itemsize
    arr = np.frombuffer(data, rec, n, pos)
    return lines, head, np.stack([arr[f] for f in fields], 1).astype(np.float32).reshape(-1, 4)


@pytest.mark.parametrize("leaf", [0.0, 0.2])
def test_pcd_round_trip(tmp_path, leaf):
    rng = np.random.default_rng(2)
    clouds = [random_cloud(rng, n) for n in (5000, 3, 12000)]
    rm = RegisteredMap(leaf, 1 << 20)
    insert_all(rm, clouds)
    path = tmp_path / "map.pcd"
    rm.write_pcd(path)
    lines, head, pts = read_pcd(path)
    n = rm.stats()["size"]
    assert lines == ["# .PCD v0.7 - Point Cloud Data file format", "VERSION 0.7", "FIELDS x y z intensity", "SIZE 4 4 4 4",
                     "TYPE F F F F", "COUNT 1 1 1 1", f"WIDTH {n}", "HEIGHT 1", "VIEWPOINT 0 0 0 1 0 0 0", f"POINTS {n}", "DATA binary"]
    assert same_bits(pts, rm.download())
    rm.reset()
    rm.write_pcd(path)
    assert read_pcd(path)[2].shape == (0, 4)
