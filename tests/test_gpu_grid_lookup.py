"""GPU: lookups along lines and derivatives at points (ElevationMap.max_value_between_locations,
values_between_locations and grid_derivatives / emap_max_values_between, emap_values_between, emap_grid_derivatives)
against the header's host build (tests/native/lookup_host.cpp) and the Python-float oracle (tests/grid_lookup_oracle.py),
bit for bit, on the planar terrain's smooth_planar and elevation layers (device output), a get_submaps window of the
LiDAR map and the 2047^2 window.  Also: host and device grids, queries and outputs give the same bits; a device call is
ordered after the caller's stream and can be captured into a CUDA graph and replayed with new queries; the launch count
depends on the number of queries only; too small a capacity and its retry; empty batches; and every rejected argument
launches nothing."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import grid_lookup_oracle as O              # noqa: E402
import plane_scenes as S                    # noqa: E402
from test_grid_lookup_cpu import (assert_same_bits, host_derivatives, host_max, host_values,  # noqa: E402,F401
                                  native)

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


def _oracle_grid(em, grid, layer):
    return O.Grid(_host(grid["layers"][layer]), _host(grid["centre"]), grid.get("resolution", em.resolution))


def _scene(name):
    """(map, grid dict, layer names) for a scene."""
    import torch
    if name == "lidar":
        _MAPS.pop(S.LIDAR_W, None)
        em = _map(S.LIDAR_W)
        S.lidar_frames(em)
        grid = em.get_submap(S.lidar_window(em.center), (5.0, 4.0), ["elevation", "variance"])
        return em, grid, ["elevation", "variance"]
    if name == "big":
        em = _map(S.BIG_W)
        S.set_image(em, S.big_image())
        out = torch.zeros(S.BIG_W ** 2, dtype=torch.float32, device="cuda")
        return em, em.get_submap((0.0, 0.0), (100.0, 100.0), ["elevation"], out=out), ["elevation"]
    png, scale, pos, ln = S.TERRAINS[name]
    img = S.terrain_image(np.load(S.GOLDEN)["grey__" + name], scale, seed=5 if name == "holes" else None)
    em = _map(img.shape[0] + 2)
    S.set_image(em, img)
    n = img.shape[0] ** 2
    res = em.planar_terrain(pos, ln, S.params(), out=torch.zeros(10 * n, dtype=torch.float32, device="cuda"))
    assert res["complete"] and res["layers"]["smooth_planar"].is_cuda
    return em, res, ["smooth_planar", "elevation"]


def _max(em, grid, layer, lines, **kw):
    r = em.max_value_between_locations(grid, layer, lines[:, :2], lines[:, 2:], **kw)
    index = np.concatenate([_host(r["valid"]).astype(np.int32)[:, None], _host(r["index"])], 1)
    value = np.concatenate([_host(r["value"])[:, None], _host(r["position"])], 1)
    return np.ascontiguousarray(index, np.int32), np.ascontiguousarray(value)


def _values(em, grid, layer, lines, **kw):
    r = em.values_between_locations(grid, layer, lines[:, :2], lines[:, 2:], **kw)
    return _host(r["counts"]), _host(r["first"]), _host(r["rows"])


def _deriv(em, grid, layer, pos, curvature, **kw):
    r = em.grid_derivatives(grid, layer, pos, curvature, **kw)
    value = _host(r["gradient"])
    if curvature:
        value = np.concatenate([value, _host(r["curvature"])], 1)
    index = np.concatenate([_host(r["status"])[:, None], _host(r["index"])], 1)
    return np.ascontiguousarray(index, np.int32), np.ascontiguousarray(value)


def _across(g, n, seed):
    """Lines between random points on opposite edges: each crosses the whole window."""
    rng = np.random.default_rng(seed)
    hx, hy = 0.5 * g.len[0], 0.5 * g.len[1]
    t = rng.random((n, 2)) * 2 - 1
    a = np.stack([g.pos[0] + hx * np.ones(n), g.pos[1] + hy * t[:, 0]], 1)
    b = np.stack([g.pos[0] - hx * np.ones(n), g.pos[1] + hy * t[:, 1]], 1)
    c = np.stack([g.pos[0] + hx * t[:, 0], g.pos[1] + hy * np.ones(n)], 1)
    d = np.stack([g.pos[0] + hx * t[:, 1], g.pos[1] - hy * np.ones(n)], 1)
    return np.concatenate([np.concatenate([a, b], 1), np.concatenate([c, d], 1)])


SCENES = ["terrain", "holes", "lidar", "big"]


@pytest.mark.parametrize("name", SCENES)
def test_device_equals_host_build_and_oracle(native, name):
    em, grid, layers = _scene(name)
    big = name == "big"
    for li, layer in enumerate(layers):
        g = _oracle_grid(em, grid, layer)
        lines = np.concatenate([O.random_lines(g, 20000, seed=li, lo=0.5, hi=3.0), O.edge_lines(g)]
                               + ([_across(g, 200, seed=li)] if big else []))
        pos = O.random_positions(g, 20000, seed=li)
        got_max, got_val = _max(em, grid, layer, lines), _values(em, grid, layer, lines)
        assert_same_bits(got_max, host_max(native, g, lines))
        assert_same_bits(got_val, host_values(native, g, lines))
        for curv in (False, True):
            got = _deriv(em, grid, layer, pos, curv)
            assert_same_bits(got, host_derivatives(native, g, pos, curv))
            sub = pos[:: 97]
            assert_same_bits(_deriv(em, grid, layer, sub, curv), O.derivative_batch(g, sub, curv))
        sub = np.concatenate([lines[:: 401], lines[-20:]])
        assert_same_bits(_max(em, grid, layer, sub), O.max_batch(g, sub))
        assert_same_bits(_values(em, grid, layer, sub), O.values_batch(g, sub))
        assert got_max[0][:, 0].sum() > len(lines) // 10          # the LiDAR window is sparse
        if big:
            assert (got_val[0][-400:] < 2047).any()        # crossing lines through NaN regions


def test_grid_query_and_output_sources_agree():
    import torch
    em, grid, _ = _scene("holes")
    hgrid = dict(grid, layers={k: _host(v) for k, v in grid["layers"].items()})
    g = _oracle_grid(em, grid, "smooth_planar")
    lines = O.random_lines(g, 3000, seed=9)
    pos = O.random_positions(g, 3000, seed=9)[:3000]
    want = (_max(em, hgrid, "smooth_planar", lines), _values(em, hgrid, "smooth_planar", lines),
            _deriv(em, hgrid, "smooth_planar", pos, True))
    ld, pd = torch.as_tensor(lines, device="cuda"), torch.as_tensor(pos, device="cuda")
    for gr in (grid, hgrid):
        for q_lines, q_pos in ((lines, pos), (ld, pd)):
            assert_same_bits(_max(em, gr, "smooth_planar", q_lines), want[0])
            assert_same_bits(_values(em, gr, "smooth_planar", q_lines), want[1])
            assert_same_bits(_deriv(em, gr, "smooth_planar", q_pos, True), want[2])
    r = em.max_value_between_locations(grid, "smooth_planar", ld[:, :2], ld[:, 2:])
    assert r["value"].is_cuda
    r = em.values_between_locations(grid, "smooth_planar", lines[:, :2], lines[:, 2:])
    assert r["rows"].is_cuda                                  # a device layer keeps the rows on the device
    out = {"index": torch.empty((3000, 3), dtype=torch.int32, device="cuda"),
           "value": torch.empty((3000, 5), dtype=torch.float64, device="cuda")}
    em.grid_derivatives(hgrid, "smooth_planar", pos, True, out=out)          # host grid and queries, device output
    assert_same_bits((out["index"].cpu().numpy(), out["value"].cpu().numpy()), want[2])


def test_stream_order_and_graph_replay():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    em, grid, _ = _scene("terrain")
    g = _oracle_grid(em, grid, "elevation")
    n = 4000
    l1, l2 = O.random_lines(g, n, seed=1), O.random_lines(g, n, seed=2)
    want1, want2 = _values(em, grid, "elevation", l1), _values(em, grid, "elevation", l2)
    wmax2 = _max(em, grid, "elevation", l2)
    # stream order: the queries are written by a long kernel chain on the caller's stream just before the call
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        qd = torch.zeros((n, 4), dtype=torch.float64, device="cuda")
        big = torch.ones((4096, 4096), device="cuda")
        for _ in range(20):
            big = big @ big / 4096.0
        qd += torch.as_tensor(l1, device="cuda") + big[0, 0].double() * 0
        r = em.values_between_locations(grid, "elevation", qd[:, :2], qd[:, 2:], capacity=int(want1[2].shape[0]))
        got = r["rows"].clone()
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy(), want1[2])
    # capture with a device grid, queries and output, then replay with new queries in the same buffer
    data = grid["layers"]["elevation"]
    eg = _lib.EmapGrid(data.data_ptr(), data.shape[0], data.shape[1], (C.c_double * 2)(*grid["centre"].tolist()),
                       grid["resolution"])
    cap = 3 * max(len(want1[2]), len(want2[2]))
    rows = torch.empty((cap, 3), dtype=torch.float64, device="cuda")
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    first = torch.empty(n, dtype=torch.int64, device="cuda")
    info = torch.empty(2, dtype=torch.int64, device="cuda")
    mx = [torch.empty((n, 3), dtype=torch.int32, device="cuda"), torch.empty((n, 3), dtype=torch.float64, device="cuda")]
    vo = _lib.EmapLineValuesOut(rows.data_ptr(), cap, counts.data_ptr(), first.data_ptr(), info.data_ptr())
    mo = _lib.EmapLineMaxOut(mx[0].data_ptr(), mx[1].data_ptr())
    qd = torch.as_tensor(l1, device="cuda")
    cs = torch.cuda.Stream()
    torch.cuda.synchronize()
    em.set_stream(cs.cuda_stream)
    try:
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=cs):
            rc = em._L.emap_values_between(em._h, C.byref(eg), 1, n, qd.data_ptr(), 1, C.byref(vo), 1)
            assert rc == 0, em._L.emap_last_error(em._h)
            rc = em._L.emap_max_values_between(em._h, C.byref(eg), 1, n, qd.data_ptr(), 1, C.byref(mo), 1)
            assert rc == 0, em._L.emap_last_error(em._h)
        gr.replay()
        torch.cuda.synchronize()
        assert info.tolist() == [len(want1[2]), 1]
        assert np.array_equal(rows[:len(want1[2])].cpu().numpy(), want1[2])
        qd.copy_(torch.as_tensor(l2, device="cuda"))
        gr.replay()
        torch.cuda.synchronize()
    finally:
        em.set_stream(None)
    assert info.tolist() == [len(want2[2]), 1]
    assert np.array_equal(counts.cpu().numpy(), want2[0]) and np.array_equal(first.cpu().numpy(), want2[1])
    assert np.array_equal(rows[:len(want2[2])].cpu().numpy(), want2[2])
    assert_same_bits((mx[0].cpu().numpy(), mx[1].cpu().numpy()), wmax2)


def test_launch_count_depends_on_queries_only():
    counts = {}
    for name in ("terrain", "lidar"):
        em, grid, layers = _scene(name)
        g = _oracle_grid(em, grid, layers[0])
        lines = O.random_lines(g, 300, seed=3)
        for m in (0, 1, 300):
            for call in ("max", "values", "deriv"):
                n0 = em.launch_count()
                if call == "max":
                    em.max_value_between_locations(grid, layers[0], lines[:m, :2], lines[:m, 2:])
                elif call == "values":
                    em.values_between_locations(grid, layers[0], lines[:m, :2], lines[:m, 2:], capacity=10 ** 6)
                else:
                    em.grid_derivatives(grid, layers[0], lines[:m, :2], True)
                counts.setdefault((call, m > 0), set()).add(em.launch_count() - n0)
    assert counts == {("max", False): {0}, ("max", True): {1}, ("values", False): {0}, ("values", True): {3},
                      ("deriv", False): {0}, ("deriv", True): {1}}


def test_too_small_capacity_and_retry():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    em, grid, _ = _scene("lidar")
    g = _oracle_grid(em, grid, "elevation")
    lines = O.random_lines(g, 500, seed=4)
    want = O.values_batch(g, lines)
    total = len(want[2])
    r = em.values_between_locations(grid, "elevation", lines[:, :2], lines[:, 2:], capacity=total - 1)
    assert r["retried"] and r["rows"].shape == (total, 3)
    assert_same_bits((r["counts"], r["first"], r["rows"]), want)
    assert not em.values_between_locations(grid, "elevation", lines[:, :2], lines[:, 2:], capacity=total)["retried"]
    for device in (False, True):        # the raw call: complete = 0 and no row written
        data = np.ascontiguousarray(grid["layers"]["elevation"])
        mk = (lambda s, dt: torch.full(s, 7, dtype=getattr(torch, dt), device="cuda")) if device else (
            lambda s, dt: np.full(s, 7, dt))
        rows, counts, first, info = mk((total, 3), "float64"), mk((500,), "int32"), mk((500,), "int64"), mk((2,), "int64")
        ptr = (lambda a: a.data_ptr()) if device else (lambda a: a.ctypes.data)
        eg = _lib.EmapGrid(data.ctypes.data, data.shape[0], data.shape[1], (C.c_double * 2)(*grid["centre"].tolist()),
                           em.resolution)
        vo = _lib.EmapLineValuesOut(ptr(rows), total - 1, ptr(counts), ptr(first), ptr(info))
        q = np.ascontiguousarray(lines)
        assert em._L.emap_values_between(em._h, C.byref(eg), 0, 500, q.ctypes.data, 0, C.byref(vo), int(device)) == 0
        em.synchronize()
        assert _host(info).tolist() == [total, 0]
        assert (_host(rows) == 7).all()
        assert np.array_equal(_host(counts), want[0]) and np.array_equal(_host(first), want[1])


def test_empty_batches():
    import torch
    em, grid, layers = _scene("lidar")
    z = np.zeros((0, 2))
    r = em.max_value_between_locations(grid, "elevation", z, z)
    assert r["value"].shape == (0,)
    r = em.values_between_locations(grid, "elevation", z, z)
    assert r["rows"].shape == (0, 3) and not r["retried"]
    zd = torch.zeros((0, 2), dtype=torch.float64, device="cuda")
    r = em.values_between_locations(grid, "elevation", zd, zd)
    assert r["rows"].shape == (0, 3) and r["rows"].is_cuda
    assert em.grid_derivatives(grid, "elevation", z, True)["curvature"].shape == (0, 3)


WHY = ["null grid", "null out", "null data", "rows 0", "cols 0", "deriv rows 4", "too many cells", "res nan",
       "res tiny", "position inf", "extent", "negative queries", "null queries", "null output", "values null info",
       "values capacity negative", "values null rows"]


@pytest.mark.parametrize("why", WHY)
def test_rejections_launch_nothing(why):
    from elevation_mapping_cupy_b200 import _lib
    em, grid, _ = _scene("lidar")
    data = np.ascontiguousarray(grid["layers"]["elevation"])
    eg = _lib.EmapGrid(data.ctypes.data, data.shape[0], data.shape[1], (C.c_double * 2)(*grid["centre"].tolist()),
                       em.resolution)
    n = 4
    q = np.zeros((n, 4))
    index, value = np.zeros((n, 3), np.int32), np.zeros((n, 5))
    rows, counts, first, info = np.zeros((8, 3)), np.zeros(n, np.int32), np.zeros(n, np.int64), np.zeros(2, np.int64)
    mo = _lib.EmapLineMaxOut(index.ctypes.data, value.ctypes.data)
    vo = _lib.EmapLineValuesOut(rows.ctypes.data, 8, counts.ctypes.data, first.ctypes.data, info.ctypes.data)
    do = _lib.EmapDerivativeOut(index.ctypes.data, value.ctypes.data)
    gp, qp, nq = C.byref(eg), q.ctypes.data, n
    outs = [C.byref(mo), C.byref(vo), C.byref(do)]
    calls = ["max", "values", "deriv"]
    if why == "null grid":
        gp = None
    elif why == "null out":
        outs = [None, None, None]
    elif why == "null data":
        eg.data = None
    elif why == "rows 0":
        eg.rows = 0
    elif why == "cols 0":
        eg.cols = 0
    elif why == "deriv rows 4":
        eg.rows, calls = 4, ["deriv"]
    elif why == "too many cells":
        eg.rows, eg.cols, eg.resolution = 1 << 16, 1 << 15, 2.0 ** -20
    elif why == "res nan":
        eg.resolution = float("nan")
    elif why == "res tiny":
        eg.resolution = 2.0 ** -21
    elif why == "position inf":
        eg.position[1] = float("inf")
    elif why == "extent":
        eg.position[0] = 2.0 ** 20
    elif why == "negative queries":
        nq = -1
    elif why == "null queries":
        qp = None
    elif why == "null output":
        mo.value, vo.first, do.index = None, None, None
    elif why == "values null info":
        vo.info, calls = None, ["values"]
    elif why == "values capacity negative":
        vo.capacity, calls = -1, ["values"]
    elif why == "values null rows":
        vo.rows, calls = None, ["values"]
    fns = {"max": (em._L.emap_max_values_between, outs[0], "emap_max_values_between"),
           "values": (em._L.emap_values_between, outs[1], "emap_values_between"),
           "deriv": (em._L.emap_grid_derivatives, outs[2], "emap_grid_derivatives")}
    for call in calls:
        fn, o, name = fns[call]
        n0 = em.launch_count()
        if call == "deriv":
            rc = fn(em._h, gp, 0, nq, qp, 0, 1, o, 0)
        else:
            rc = fn(em._h, gp, 0, nq, qp, 0, o, 0)
        assert rc == -1, call
        assert name.encode() in em._L.emap_last_error(em._h)
        assert em.launch_count() == n0
    assert not index.any() and not value.any() and not rows.any() and not counts.any() and not first.any()
    assert not info.any()
