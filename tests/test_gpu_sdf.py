"""GPU: the signed distance field and its queries (ElevationMap.signed_distance_field and sdf_values /
emap_signed_distance_field and emap_sdf_values) against the NumPy oracle and the Python-float restatement
(tests/sdf_oracle.py), bit for bit: the five demo terrains with host and device input and output, the planar terrain's
smooth_planar and elevation layers for the node's window, a get_submap window of the LiDAR map with NaN cells, a 2047^2
window with about 32 slices, 1 x 1, 1 x N and N x 1 grids and one slice, ranges below and above the terrain, an all-NaN
layer and the largest accepted d2; 10^5 queries of every kind.  Also: two calls give the same bytes, a build and a query
captured into one CUDA graph replay to the eager result, the launch counts, and every rejection writes and launches
nothing."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import plane_scenes as S                                          # noqa: E402
import sdf_oracle as O                                            # noqa: E402
from test_sdf_cpu import assert_same_bits, query_points           # noqa: E402

pytestmark = pytest.mark.gpu

_MAPS = {}


def _map(cell_n):
    if cell_n not in _MAPS:
        from elevation_mapping_cupy_b200.parameter import core_parameter
        from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
        _MAPS.clear()
        _MAPS[cell_n] = ElevationMap(core_parameter(cell_n))
    return _MAPS[cell_n]


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _dev(x):
    import torch
    return torch.as_tensor(np.ascontiguousarray(x), device="cuda")


def _grid(layer, centre=(0.0, 0.0), res=S.RES):
    return {"layers": {"elevation": layer}, "centre": np.array(centre, np.float64), "resolution": res}


def _terrain(name):
    png, scale, _, _ = S.TERRAINS[name]
    return S.terrain_image(np.load(S.GOLDEN)["grey__" + name], scale, seed=5 if name == "holes" else None)


def _want(layer, res, clearance=0.1, z_range=None):
    layer = _host(layer)
    if z_range is None:
        z_min, n_z = O.default_range(layer, res, clearance)
    else:
        z_min, n_z = float(z_range[0]), int(math.floor((float(z_range[1]) - float(z_range[0])) / res)) + 1
    return O.field(layer, z_min, n_z, res), z_min, n_z


def _check(em, grid, layer="elevation", z_range=None, res=None, sides=("hh", "dd")):
    """The field of every requested side (input, output: h host, d device) equals the oracle, bit for bit."""
    import torch
    res = grid.get("resolution", em.resolution) if res is None else res
    data = _host(grid["layers"][layer])
    want, z_min, n_z = _want(data, res, z_range=z_range)
    for side in sides:
        g = dict(grid, layers={layer: _dev(data) if side[0] == "d" else data})
        out = torch.full(want.shape, 7.0, device="cuda") if side == "hd" else None
        f = em.signed_distance_field(g, layer, z_range=z_range, out=out)
        assert f["z_min"] == z_min and f["n_z"] == n_z and f["resolution"] == res
        assert (side[1] == "d") == hasattr(f["volume"], "is_cuda")
        assert_same_bits(_host(f["volume"]), want)
    return f, want


@pytest.mark.parametrize("name", ["terrain", "slope", "straight_stairs", "real_stairs", "holes"])
def test_demo_terrains(name):
    em = _map(S.LIDAR_W)
    _check(em, _grid(_terrain(name)), sides=("hh", "dd", "hd"))


def test_planar_terrain_layers():
    import torch
    png, scale, pos, ln = S.TERRAINS["terrain"]
    img = _terrain("terrain")
    em = _map(img.shape[0] + 2)
    S.set_image(em, img)
    res = em.planar_terrain(pos, ln, S.params(), out=torch.zeros(10 * img.shape[0] ** 2, dtype=torch.float32,
                                                                 device="cuda"))
    for layer in ("smooth_planar", "elevation"):
        _check(em, res, layer)


def test_submap_window_with_nan_cells():
    _MAPS.pop(S.LIDAR_W, None)
    em = _map(S.LIDAR_W)
    S.lidar_frames(em)
    grid = em.get_submap(S.lidar_window(em.center), (5.0, 4.0), ["elevation"])
    assert np.isnan(grid["layers"]["elevation"]).any() and np.isfinite(grid["layers"]["elevation"]).any()
    _check(em, grid)


def test_2047_window():
    e = S.big_image()
    assert e.shape == (2047, 2047)
    em = _map(S.LIDAR_W)
    f, want = _check(em, _grid(e), z_range=(0.3, 0.3 + 31.5 * S.RES), sides=("dd",))
    assert f["n_z"] == 32


@pytest.mark.parametrize("shape", [(1, 1), (1, 37), (29, 1), (5, 6)])
@pytest.mark.parametrize("one_slice", [True, False])
def test_degenerate_shapes(shape, one_slice):
    rng = np.random.default_rng(shape[0] * 100 + shape[1])
    e = (rng.random(shape) * 0.4).astype(np.float32)
    z_range = (0.1, 0.1) if one_slice else None
    _check(_map(S.LIDAR_W), _grid(e, (0.2, -0.3), 0.05), z_range=z_range, sides=("hh", "dd"))


def test_ranges_below_and_above_the_terrain():
    em = _map(S.LIDAR_W)
    e = _terrain("slope")
    lo, hi = float(np.nanmin(e)), float(np.nanmax(e))
    f, _ = _check(em, _grid(e), z_range=(lo - 2.0, lo - 1.0))
    assert bool((f["volume"] == -math.inf).all())
    f, _ = _check(em, _grid(e), z_range=(hi + 0.01, hi + 0.5))
    assert bool((f["volume"] == math.inf).all())


def test_all_nan_layer():
    em = _map(S.LIDAR_W)
    e = np.full((20, 30), np.nan, np.float32)
    with pytest.raises(ValueError):
        em.signed_distance_field(_grid(e))
    with pytest.raises(ValueError):
        em.signed_distance_field(_grid(_dev(e)))
    f, _ = _check(em, _grid(e), z_range=(0.0, 0.5))
    assert bool((f["volume"] == math.inf).all())


def test_largest_d2():
    from elevation_mapping_cupy_b200 import _lib
    em = _map(S.LIDAR_W)
    rows, cols = 3000, 2
    n_z = 1
    while (rows - 1) ** 2 + (cols - 1) ** 2 + n_z ** 2 < O.MAX_D2:
        n_z += 1
    e = np.full((rows, cols), -1.0, np.float32)
    e[0, 0] = 0.0
    f, want = _check(em, _grid(e, (0.0, 0.0), 1.0), z_range=(0.0, n_z - 1.0), sides=("dd",))
    d2 = (rows - 1) ** 2 + (cols - 1) ** 2 + (n_z - 1) ** 2
    assert _host(f["volume"])[-1, -1, -1] == np.sqrt(np.float32(d2))
    g = _lib.EmapGrid(e.ctypes.data, rows, cols, (C.c_double * 2)(0.0, 0.0), 1.0)
    out = np.zeros(rows * cols * (n_z + 1), np.float32)
    assert em._L.emap_signed_distance_field(em._h, C.byref(g), 0, 0.0, n_z + 1, out.ctypes.data, out.size, 0) != 0


def test_queries():
    import torch
    em = _map(S.LIDAR_W)
    f, vol = _check(em, _grid(_terrain("terrain"), (0.4, -0.2)), sides=("dd",))
    pos, res, z_min = f["position"], f["resolution"], f["z_min"]
    pts = query_points(vol.shape, pos, res, z_min, n=100_000, seed=3)
    assert len(pts) >= 100_000
    want = O.values(vol, pos, res, z_min, pts)
    hf = dict(f, volume=vol)
    got = [em.sdf_values(f, pts), em.sdf_values(f, _dev(pts)), em.sdf_values(hf, pts), em.sdf_values(hf, _dev(pts)),
           em.sdf_values(f, pts, out=torch.zeros((len(pts), 4), dtype=torch.float64, device="cuda"))]
    assert [hasattr(g, "is_cuda") for g in got] == [False, True, False, True, True]
    for g in got:
        assert_same_bits(_host(g), want)
    assert em.sdf_values(f, np.zeros((0, 3))).shape == (0, 4)


def test_repeatable_and_graph_replay():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    em = _map(S.LIDAR_W)
    e = _dev(_terrain("holes"))
    grid = _grid(e)
    f1 = em.signed_distance_field(grid)
    f2 = em.signed_distance_field(grid)
    assert_same_bits(_host(f1["volume"]), _host(f2["volume"]))
    pts = _dev(query_points(tuple(f1["volume"].shape), f1["position"], f1["resolution"], f1["z_min"], n=5000))
    want_q = _host(em.sdf_values(f1, pts))
    # build and query captured into one graph, from a layer written just before replay
    rows, cols = e.shape
    n_z, z_min = f1["n_z"], f1["z_min"]
    src = torch.zeros_like(e)
    vol = torch.full((n_z, rows, cols), 3.0, device="cuda")
    out = torch.zeros((len(pts), 4), dtype=torch.float64, device="cuda")
    g = _lib.EmapGrid(src.data_ptr(), rows, cols, (C.c_double * 2)(0.0, 0.0), S.RES)
    sf = _lib.EmapSdf(vol.data_ptr(), rows, cols, n_z, (C.c_double * 2)(0.0, 0.0), S.RES, z_min)
    cs = torch.cuda.Stream()
    torch.cuda.synchronize()
    em.set_stream(cs.cuda_stream)
    try:
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=cs):
            rc = em._L.emap_signed_distance_field(em._h, C.byref(g), 1, z_min, n_z, vol.data_ptr(), vol.numel(), 1)
            assert rc == 0, em._L.emap_last_error(em._h)
            rc = em._L.emap_sdf_values(em._h, C.byref(sf), 1, len(pts), pts.data_ptr(), 1, out.data_ptr(), 1)
            assert rc == 0, em._L.emap_last_error(em._h)
        src.copy_(e)
        gr.replay()
        torch.cuda.synchronize()
    finally:
        em.set_stream(None)
    assert_same_bits(_host(vol), _host(f1["volume"]))
    assert_same_bits(_host(out), want_q)


def test_launch_counts():
    em = _map(S.LIDAR_W)
    counts = set()
    for e in (_terrain("terrain"), np.zeros((1, 1), np.float32), S.big_image()[:300, :500]):
        n0 = em.launch_count()
        f = em.signed_distance_field(_grid(e), z_range=(0.0, 0.4))
        n1 = em.launch_count()
        em.sdf_values(f, np.zeros((10, 3)))
        n2 = em.launch_count()
        em.sdf_values(f, np.zeros((0, 3)))
        counts.add((n1 - n0, n2 - n1, em.launch_count() - n2))
    assert counts == {(3, 1, 0)}


_REJECT = ["null grid", "null data", "rows 0", "cols 0", "bad resolution", "tiny resolution", "nan position",
           "extent", "n_z 0", "nan z_min", "inf z_min", "d2 limit", "long line", "capacity", "null out",
           "q null field", "q null data", "q n_z 0", "q nan z_min", "q d2 limit", "q negative n", "q null points",
           "q null out"]


@pytest.mark.parametrize("why", _REJECT)
def test_rejections_write_and_launch_nothing(why):
    from elevation_mapping_cupy_b200 import _lib
    em = _map(S.LIDAR_W)
    e = np.zeros((20, 30), np.float32)
    rows, cols, n_z, z_min, res, pos = 20, 30, 4, 0.0, 0.05, [0.0, 0.0]
    data, cap = e.ctypes.data, 20 * 30 * 4
    out = np.zeros(cap + 100, np.float32)
    optr = out.ctypes.data
    pts = np.zeros((5, 3))
    qout = np.zeros((5, 4))
    n, pptr, qptr = 5, pts.ctypes.data, qout.ctypes.data
    grid_null = field_null = False
    w = why[2:] if why.startswith("q ") else why
    if w == "null grid":
        grid_null = True
    elif w == "null field":
        field_null = True
    elif w == "null data":
        data = None
    elif w == "rows 0":
        rows = 0
    elif w == "cols 0":
        cols = 0
    elif w == "bad resolution":
        res = float("nan")
    elif w == "tiny resolution":
        res = 2.0 ** -21
    elif w == "nan position":
        pos = [float("nan"), 0.0]
    elif w == "extent":
        pos = [2.0 ** 20, 0.0]
    elif w == "n_z 0":
        n_z = 0
    elif w in ("nan z_min", "inf z_min"):
        z_min = float("nan") if w.startswith("nan") else float("inf")
    elif w == "d2 limit":                  # 199^2 + 29^2 + 4095^2 >= 2^24, with room for the volume
        rows, n_z = 200, 4096
        cap = rows * cols * n_z
    elif w == "long line":
        rows, cols, n_z = 4097, 1, 1
    elif w == "capacity":
        cap -= 1
    elif w == "null out":
        optr = None
    elif w == "negative n":
        n = -1
    elif w == "null points":
        pptr = None
    g = _lib.EmapGrid(data, rows, cols, (C.c_double * 2)(*pos), res)
    n0 = em.launch_count()
    if why.startswith("q "):
        if w == "null out":
            qptr = None
        f = _lib.EmapSdf(data, rows, cols, n_z, (C.c_double * 2)(*pos), res, z_min)
        rc = em._L.emap_sdf_values(em._h, None if field_null else C.byref(f), 0, n, pptr, 0, qptr, 0)
        name = b"emap_sdf_values"
    else:
        rc = em._L.emap_signed_distance_field(em._h, None if grid_null else C.byref(g), 0, z_min, n_z, optr, cap, 0)
        name = b"emap_signed_distance_field"
    assert rc != 0
    assert name in em._L.emap_last_error(em._h)
    if w in ("d2 limit", "long line"):
        assert b"2^24" in em._L.emap_last_error(em._h)
    assert em.launch_count() == n0
    assert not out.any() and not qout.any()
