"""Entries of the handle types (lio_pp, lio_po, lio_pm, lio_rm, lio_est, lio_node): a null handle is refused with text naming the
entry, and a handle on device 1 gives the same results when device 0 is current at each of its calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from lio_mapping_b200 import _lib

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "lio_b200.h")
HANDLES = ("lio_pp", "lio_po", "lio_pm", "lio_rm", "lio_est", "lio_node")
# entries that return a count or text rather than a status
NOT_STATUS = {"lio_pp_last_launches", "lio_po_last_launches", "lio_est_last_launches", "lio_est_last_error"}


def handle_entries():
    """(name, ctypes argtypes) of every header function whose first parameter is a handle, destroy entries excluded."""
    with open(HEADER) as f:
        text = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    out = []
    for name, params in re.findall(r"\b(lio_\w+)\s*\(([^()]*)\)\s*;", text):
        params = [p.strip() for p in params.split(",")]
        first = re.match(r"(?:const\s+)?(\w+)\s*\*", params[0])
        if not first or first.group(1) not in HANDLES or name.endswith("_destroy") or name in NOT_STATUS:
            continue
        types = []
        for p in params:
            if "*" in p or "[" in p or p.startswith("lio_allreduce_fn"):
                types.append(C.c_void_p)
            elif p.startswith("double"):
                types.append(C.c_double)
            elif p.startswith("float"):
                types.append(C.c_float)
            elif p.startswith(("long long", "size_t")):
                types.append(C.c_longlong)
            else:
                assert re.match(r"(const\s+)?(int|uint\w+|int\w+)\s+\w+$", p), (name, p)
                types.append(C.c_int)
        out.append((name, types))
    return out


def test_header_lists_the_handle_entries():
    names = {n for n, _ in handle_entries()}
    assert len(names) > 100
    assert {"lio_pp_download_cloud", "lio_mb_surround_download", "lio_rm_write_pcd", "lio_est_get_frame", "lio_node_status"} <= names


@pytest.mark.parametrize("name,types", handle_entries(), ids=[n for n, _ in handle_entries()])
def test_null_handle_is_refused_by_name(name, types):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("liblio_b200.so not built")
    f = getattr(C.CDLL(_lib.LIB_PATH), name)   # a CDLL of its own: the package's prototypes stay as they are
    f.restype, f.argtypes = C.c_int, types
    assert f(*[t() for t in types]) == -2
    assert re.search(r"\b%s:" % name, _lib.lib().lio_last_error().decode())


class Interleaved:
    """Calls between() before every method call on the wrapped handle object."""

    def __init__(self, obj, between):
        self._obj, self._between = obj, between

    def __getattr__(self, name):
        attr = getattr(self._obj, name)
        if not callable(attr):
            return attr

        def call(*args, **kwargs):
            self._between()
            return attr(*args, **kwargs)
        return call


def run_processor(dev, wrap, sweeps):
    import torch
    from lio_mapping_b200.point_processor import PointProcessor
    pp = wrap(PointProcessor(-15.0, 15.0, 16, max_points=max(s.shape[0] for s in sweeps), device=dev))
    out = {}
    for k, s in enumerate(sweeps):
        if k % 2:
            pp.SetInputCloud(s)
            pp.Process()
        else:
            t = torch.from_numpy(s).to("cuda:%d" % dev)
            pp.process_device(t.data_ptr(), t.shape[0])
        out.update({"%d_size_%s" % (k, n): v for n, v in pp.sizes().items()})
        for name in ("laser_scans", "corner_points_sharp", "surface_points_flat", "surface_points_less_flat"):
            out["%d_%s" % (k, name)] = pp.cloud(name)
        for name in ("sharp", "flat", "orig"):
            out["%d_idx_%s" % (k, name)] = pp.index(name)
        out["%d_ranges" % k] = pp.scan_ranges()
        out["%d_mask" % k], out["%d_labels" % k] = pp.mask_labels()
        out["%d_start_ori" % k] = np.float32(pp.start_ori())
    return out


def run_lidar_chain(dev, wrap, sweeps):
    import torch
    from lio_mapping_b200.point_mapping import PointMapping
    from lio_mapping_b200.point_odometry import PointOdometry
    from lio_mapping_b200.point_processor import PointProcessor
    names = ("corner_points_sharp", "corner_points_less_sharp", "surface_points_flat", "surface_points_less_flat", "cloud_in_rings")
    max_raw = max(s.shape[0] for s in sweeps)
    pp = wrap(PointProcessor(-15.0, 15.0, 16, max_points=max_raw, device=dev))
    od = wrap(PointOdometry(0.1, 1, 25, max_full_points=max_raw, device=dev))
    pm = wrap(PointMapping(max_points=1 << 17, device=dev))
    pm.EnablePublish(0.6, max_raw)
    n_dev = [pp.cloud_count_dev(n) for n in names]
    out = {}
    for k, s in enumerate(sweeps):
        t = torch.from_numpy(s).to("cuda:%d" % dev)
        pp.process_device(t.data_ptr(), t.shape[0])
        ts, es, info = od.ProcessDev([pp.cloud_dev(n) for n in names], n_dev, [1 << 17] * 4 + [max_raw])
        out["%d_sum" % k], out["%d_es" % k] = ts, es
        if not info["published"]:
            continue
        out["%d_compact" % k] = od.compact_data()
        for which in ("last_corner", "last_surf", "full"):
            out["%d_po_%s" % (k, which)] = od.cloud(which)
        ptrs, cn_dev, cn = od.clouds_dev()
        out["%d_pm" % k] = pm.ProcessDev(ptrs, cn_dev, cn, ts)
        out["%d_registered" % k] = pm.registered_full_cloud()
        out["%d_surround" % k] = pm.surround_map()
        out["%d_centre" % k] = pm.centre()
        valid, _ = pm.cube_lists()
        for which in ("corner", "surf"):
            out["%d_cube_sizes_%s" % (k, which)] = pm.cube_sizes(which)
            for v in valid[:3]:
                out["%d_cube_%s_%d" % (k, which, v)] = pm.cube(int(v), which)
    return out


def run_estimator(dev, wrap, scn, W, surf_ds):
    from lio_mapping_b200 import estimator, scenario
    est = wrap(estimator.Estimator(device=dev, window_size=W, opt_window_size=W, max_frame_points=1 << 15, max_scan_points=1 << 16,
                                   **scenario.EST_CFG["vlp16"]))
    scenario.warm_start(est, scn, W, lambda k: surf_ds[k],
                        lambda a, g: estimator.Pim(a, g, np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02))
    out = {}
    for k in range(W, len(surf_ds)):
        scenario.feed_imu(est, scn, k)
        est.process_scan(surf_ds[k])
        sm = est.summary()
        out.update({"%d_%s" % (k, n): sm[n] for n in ("iterations", "final_cost", "map_size", "num_features")})
        out["%d_states" % k] = est.states()
        out["%d_features" % k] = est.features(W)
        out["%d_map" % k] = est.local_map()
        out["%d_frame" % k] = est.frame(W)
        out["%d_extrinsic" % k] = est.extrinsic()
    return out


def run_registered_map(dev, wrap, clouds):
    import torch
    from lio_mapping_b200.registered_map import RegisteredMap
    rm = wrap(RegisteredMap(0.2, 1 << 20, device=dev))
    out = {}
    for k, c in enumerate(clouds):
        if k % 2:
            rm.insert(c)
        else:
            t = torch.from_numpy(c).to("cuda:%d" % dev)
            rm.insert_dev(t.data_ptr(), t.shape[0])
        out["%d_stats" % k] = rm.stats()
        out["%d_map" % k] = rm.download()
    rm.reset()
    out["reset"] = rm.download()
    return out


def assert_same(a, b, key="out"):
    """Bit-equal nested dicts, tuples and arrays."""
    if isinstance(a, dict):
        assert a.keys() == b.keys(), key
        for k in a:
            assert_same(a[k], b[k], "%s.%s" % (key, k))
    elif isinstance(a, tuple):
        assert isinstance(b, tuple) and len(a) == len(b), key
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, "%s[%d]" % (key, i))
    else:
        assert np.array_equal(np.asarray(a), np.asarray(b)), key


@pytest.mark.gpu
def test_handles_on_device_1_ignore_the_current_device():
    """Each handle on device 1 gives the same getter output alone and with a device-0 twin called between every two of its calls."""
    import torch
    if torch.cuda.device_count() < 2 or _lib.lib().lio_device_count() < 2:
        pytest.skip("needs two CUDA devices")
    check_interleaved(1, 0)


def check_interleaved(dev, twin_dev):
    import torch
    from lio_mapping_b200 import ops, scenario, synth
    from lio_mapping_b200.point_processor import PointProcessor
    sensor, scene, traj = synth.default_config("vlp16")
    sweeps = [np.ascontiguousarray(synth.make_sweep(sensor, scene, traj, 1.0 + 0.1 * f, seed=30 + f, distort=True), np.float32)
              for f in range(6)]
    W = 4
    scn = scenario.Scenario("vlp16", n_total=W + 3)
    twin = PointProcessor(-15.0, 15.0, 16, max_points=max(s.shape[0] for s in sweeps + list(scn.raw)), device=twin_dev)
    surf_ds = []
    for raw in scn.raw[:W + 2]:
        twin.SetInputCloud(raw)
        twin.Process()
        surf_ds.append(ops.voxel_grid(twin.cloud("surface_points_less_flat"), 0.4, device=twin_dev))
    registered = [np.ascontiguousarray(s[::3], np.float32) for s in sweeps]

    def between():
        twin.start_ori()   # a device entry of the twin: its device is current when the next call on a handle arrives
        assert torch.cuda.current_device() == twin_dev

    def alone(obj):
        return obj

    def interleaved(obj):
        return Interleaved(obj, between)

    for run, args in ((run_processor, (sweeps,)), (run_lidar_chain, (sweeps,)), (run_estimator, (scn, W, surf_ds)),
                      (run_registered_map, (registered,))):
        assert_same(run(dev, alone, *args), run(dev, interleaved, *args))
