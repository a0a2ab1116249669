"""GPU: layer values at points (ElevationMap.values_at / emap_grid_values_at, emap_map_values_at).  The device equals the
header's host build (tests/native/values_at_host.cpp) and the Python-float oracle (tests/values_at_oracle.py) bit for
bit, for each method, on a get_submaps window of a LiDAR map, the planar terrain's layers, a NaN-holed window and the
2047^2 window with 10^6 points.  Every host/device combination of grid, positions and output gives the same bits.  The
live map equals emap_grid_values_at on get_maps_with_names_ref's planes at the map centre, bit for bit, for every basic
export name, plugin layers with fill_nan / is_height_layer, a semantic layer and 24 layers in one call, and equals the
whole-map get_submaps window.  A captured call replayed after a frame at the capture centre equals an eager call.  One
launch per call, none for no points, and none for a rejected call, which leaves the output untouched."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import values_at_oracle as O                                         # noqa: E402
from test_values_at_cpu import host_values_at, native               # noqa: E402,F401
from test_gpu_grid_lookup import _scene                              # noqa: E402
from test_gpu_submap import NAMES, _make                             # noqa: E402

pytestmark = pytest.mark.gpu

METHODS = ("nearest", "linear", "cubic")
CODE = {"nearest": O.NEAREST, "linear": O.LINEAR, "cubic": O.CUBIC}


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _geom(em, grid):
    return np.asarray(_host(grid["centre"]), np.float64), float(grid.get("resolution", em.resolution))


def _points(shape, centre, res, n, seed, margin=1.2):
    rng = np.random.default_rng(seed)
    h = 0.5 * np.asarray(shape, np.float64) * res * margin
    pts = rng.uniform(centre - h, centre + h, (n, 2))
    # a share of exact cell centres and cell boundaries
    k = n // 10
    ij = rng.integers(0, shape, (k, 2))
    top = centre + 0.5 * np.asarray(shape) * res
    pts[:k] = (top - 0.5 * res) - res * ij
    pts[k:2 * k] = top - res * ij
    return pts


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    bad = np.nonzero(a.view(np.uint32 if a.dtype == np.float32 else a.dtype) !=
                     b.view(np.uint32 if b.dtype == np.float32 else b.dtype))
    assert bad[0].size == 0, (bad[0][:5], a[bad][:5], b[bad][:5])


def _got(r, names):
    return np.stack([_host(r["values"][n]) for n in names]), _host(r["status"])


@pytest.mark.parametrize("name", ["lidar", "terrain", "holes", "big"])
def test_device_equals_host_build_and_oracle(native, name):
    import torch
    em, grid, layers = _scene(name)
    if name == "holes":
        # the holed terrain's layers with seeded NaN blobs punched into them, as the caller's own device grid
        rng = np.random.default_rng(4)
        holed = {}
        for k in layers:
            a = _host(grid["layers"][k]).copy()
            for r, c in rng.integers(0, a.shape, (12, 2)):
                a[max(r - 2, 0):r + 3, max(c - 3, 0):c + 2] = np.nan
            holed[k] = torch.as_tensor(a, device="cuda")
        grid = dict(grid, layers=holed)
    centre, res = _geom(em, grid)
    host_layers = [_host(grid["layers"][k]) for k in layers]
    shape = host_layers[0].shape
    n = 10 ** 6 if name == "big" else 50000
    pts = _points(shape, centre, res, n, seed=len(name))
    qd = torch.as_tensor(pts, device="cuda")
    for method in METHODS:
        r = em.values_at(qd, layers, method, grid=grid)
        assert r["status"].is_cuda
        got = _got(r, layers)
        want = host_values_at(native, host_layers, centre, res, CODE[method], pts)
        _same(got[0], want[0])
        _same(got[1], want[1])
        assert (got[1] == CODE[method] + 1).sum() > n // 2
        sub = np.arange(0, n, max(1, n // 3000))
        ov, os_ = O.values_at(host_layers, centre, res, CODE[method], pts[sub])
        _same(got[0][:, sub], ov)
        _same(got[1][sub], os_)
        if name == "holes":
            assert np.isnan(got[0]).any() and np.isfinite(got[0]).any()


def test_host_and_device_arguments_give_the_same_bits():
    import torch
    em, grid, layers = _scene("lidar")
    centre, res = _geom(em, grid)
    host_grid = dict(grid, layers={k: np.ascontiguousarray(_host(v)) for k, v in grid["layers"].items()})
    dev_grid = dict(grid, layers={k: torch.as_tensor(v, device="cuda").contiguous() for k, v in host_grid["layers"].items()})
    pts = _points(host_grid["layers"][layers[0]].shape, centre, res, 20000, seed=3)
    for method in METHODS:
        results = []
        for g in (host_grid, dev_grid):
            for q in (pts, torch.as_tensor(pts, device="cuda")):
                for out_dev in (False, True):
                    out = None
                    if out_dev:
                        out = {"values": torch.full((len(layers), len(pts)), 7.0, device="cuda"),
                               "status": torch.full((len(pts),), 9, dtype=torch.int32, device="cuda")}
                    r = em.values_at(q, layers, method, grid=g, out=out)
                    torch.cuda.synchronize()
                    results.append(_got(r, layers))
        for got in results[1:]:
            _same(got[0], results[0][0])
            _same(got[1], results[0][1])


@pytest.fixture(scope="module")
def live(tmp_path_factory):
    """A 202^2 map after LiDAR frames and a move off the cell grid, with plugin layers and a semantic layer; its full
    export of every name."""
    from elevation_mapping_cupy_b200.elevation_mapping import EXPORT_NAMES
    em = _make(202, str(tmp_path_factory.mktemp("values_at")))
    names = list(EXPORT_NAMES) + [n for n in NAMES if n not in EXPORT_NAMES]
    full = np.zeros((len(names), 200, 200), np.float32)
    em.get_maps_with_names_ref(names, full)
    grid = {"layers": dict(zip(names, full)), "centre": em.center[:2].astype(np.float64),
            "resolution": em.resolution}
    return em, names, grid


def test_live_map_equals_its_full_export(native, live):
    import torch
    em, names, grid = live
    assert "normal_color" in names and "min_filter" in names and "feat" in names
    centre, res = _geom(em, grid)
    pts = _points((200, 200), centre, res, 30000, seed=5)
    for method in METHODS:
        r = em.values_at(pts, names, method)
        got = _got(r, names)
        want = _got(em.values_at(pts, names, method, grid=grid), names)
        _same(got[0], want[0])
        _same(got[1], want[1])
        hv, hs = host_values_at(native, [grid["layers"][n] for n in names], centre, res, CODE[method], pts)
        _same(got[0], hv)
        _same(got[1], hs)
        assert np.isnan(got[0][0]).any() and np.isfinite(got[0][0]).any()
    # 24 layers in one call, device positions and output
    many = (names * 3)[:24]
    qd = torch.as_tensor(pts, device="cuda")
    r = em.values_at(qd, many, "cubic")
    got = _got(r, many)
    hv, hs = host_values_at(native, [grid["layers"][n] for n in many], centre, res, O.CUBIC, pts)
    _same(got[0], hv)
    _same(got[1], hs)


def test_live_map_equals_the_whole_map_window(live):
    em, names, _ = live
    c = em.center[:2].astype(np.float64)
    win = em.get_submap(c, (1000.0, 1000.0), ["elevation", "feat"])
    assert win["size"] == (200, 200) and np.array_equal(win["centre"], c)
    pts = _points((200, 200), c, em.resolution, 20000, seed=6)
    for method in METHODS:
        got = _got(em.values_at(pts, ["elevation", "feat"], method), ["elevation", "feat"])
        want = _got(em.values_at(pts, ["elevation", "feat"], method, grid=win), ["elevation", "feat"])
        _same(got[0], want[0])
        _same(got[1], want[1])


def test_graph_replay_after_a_frame_equals_an_eager_call():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    em = ElevationMap(core_parameter(202))
    pts0, R, t = wl.lidar_cloud(1, 0, n_rings=32, n_az=1250, max_range=4.0)
    em.move_to(t, R)
    em.input_pointcloud(pts0, ["x", "y", "z"], R, t, 0.02, 0.02)
    names = ["elevation", "variance", "normal_color"]
    n = 50000
    pts = _points((200, 200), em.center[:2].astype(np.float64), em.resolution, n, seed=8)
    qd = torch.as_tensor(pts, device="cuda")
    vals = torch.empty((len(names), n), device="cuda")
    st = torch.empty(n, dtype=torch.int32, device="cuda")
    o = _lib.EmapValuesOut(vals.data_ptr(), st.data_ptr())
    c_names = (C.c_char_p * len(names))(*[s.encode() for s in names])
    planes = (C.c_void_p * len(names))()
    flags = (C.c_int32 * len(names))()
    em.values_at(qd, names, "cubic", out={"values": vals, "status": st})      # eager, the largest size
    cs = torch.cuda.Stream()
    torch.cuda.synchronize()
    em.set_stream(cs.cuda_stream)
    try:
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=cs):
            rc = em._L.emap_map_values_at(em._h, len(names), c_names, planes, flags, n, qd.data_ptr(), 1, O.CUBIC,
                                          C.byref(o), 1)
            assert rc == 0, em._L.emap_last_error(em._h)
    finally:
        em.set_stream(None)
    # a frame at the capture centre, then the replay
    pts1, _, _ = wl.lidar_cloud(1, 1, n_rings=32, n_az=1250, max_range=4.0)
    em.input_pointcloud(pts1, ["x", "y", "z"], R, t, 0.02, 0.02)
    em.synchronize()
    vals.fill_(7.0)
    gr.replay()
    torch.cuda.synchronize()
    got = (vals.cpu().numpy(), st.cpu().numpy())
    want = _got(em.values_at(pts, names, "cubic"), names)
    _same(got[0], want[0])
    _same(got[1], want[1])


@pytest.mark.parametrize("live_map", [False, True])
def test_launch_count_and_rejections(live_map):
    import torch
    from elevation_mapping_cupy_b200 import _lib
    em, grid, layers = _scene("lidar")
    centre, res = _geom(em, grid)
    data = [torch.as_tensor(_host(grid["layers"][k]), device="cuda").contiguous() for k in layers]
    rows, cols = data[0].shape
    n = 1000
    q = torch.as_tensor(_points((rows, cols), centre, res, n, seed=9), device="cuda")
    vals = torch.full((24, n), 7.0, device="cuda")
    st = torch.full((n,), 9, dtype=torch.int32, device="cuda")
    o = _lib.EmapValuesOut(vals.data_ptr(), st.data_ptr())
    null_out = _lib.EmapValuesOut(None, st.data_ptr())

    def grids(k=2, **change):
        gs = []
        for i in range(k):
            d = data[i % len(data)]
            g = dict(data=d.data_ptr(), rows=rows, cols=cols, position=list(centre), resolution=res)
            if i == 1:
                g.update(change)
            gs.append(_lib.EmapGrid(g["data"], g["rows"], g["cols"], (C.c_double * 2)(*g["position"]),
                                    g["resolution"]))
        return (_lib.EmapGrid * max(k, 1))(*gs)

    def call(k=2, method=1, npts=n, out=o, q_ptr=q.data_ptr(), names=None, **change):
        if live_map:
            nm = names or ["elevation", "variance"] * 13
            c_names = (C.c_char_p * len(nm))(*[s.encode() for s in nm])
            return em._L.emap_map_values_at(em._h, k, c_names, None, None, npts, q_ptr, 1, method, C.byref(out), 1)
        return em._L.emap_grid_values_at(em._h, k, grids(k, **change), 1, npts, q_ptr, 1, method, C.byref(out), 1)

    for k in (1, 2, 24):
        for method in (0, 1, 2):
            n0 = em.launch_count()
            assert call(k, method) == 0, em._L.emap_last_error(em._h)
            assert em.launch_count() == n0 + 1
    n0 = em.launch_count()
    assert call(npts=0) == 0 and em.launch_count() == n0
    torch.cuda.synchronize()
    vals.fill_(7.0)
    st.fill_(9)
    bad = [dict(k=0), dict(k=25), dict(method=3), dict(method=-1), dict(npts=-1), dict(q_ptr=None),
           dict(out=null_out)]
    if live_map:
        bad.append(dict(names=["elevation", "no_such_layer"]))
    else:
        bad += [dict(rows=rows - 1), dict(cols=cols + 1), dict(position=[centre[0] + res, centre[1]]),
                dict(resolution=2 * res), dict(data=None), dict(resolution=float("nan"))]
    for b in bad:
        n0 = em.launch_count()
        assert call(**b) != 0, b
        assert em.launch_count() == n0, b
    torch.cuda.synchronize()
    assert (vals == 7.0).all() and (st == 9).all()
