"""GPU: projection onto the planar regions and convex growth (ElevationMap.project_to_planar_regions /
emap_project_to_planar_regions) against the header's host build (tests/native/projection_host.cpp) and the Python-float
oracle (tests/planar_projection_oracle.py), bit for bit, on the regions planar_terrain returns for the demo terrains,
the LiDAR map and a 2047^2 window, with and without growth.  Also: host and device tables, queries and outputs give the
same bits; a device call is ordered after the caller's stream and can be captured into a CUDA graph and replayed with
new queries; the launch count depends on the number of queries and the growth only; zero regions, zero queries and a
window without planes; and every rejected argument launches nothing."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import plane_scenes as S                    # noqa: E402
import planar_projection_oracle as PP       # noqa: E402
from test_planar_projection_cpu import assert_same_bits, host_project, native   # noqa: E402,F401

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

_MAPS = {}
_TERRAIN = {}


def _map(cell_n):
    if cell_n not in _MAPS:
        from elevation_mapping_cupy_b200.parameter import core_parameter
        from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
        _MAPS.clear()
        _MAPS[cell_n] = ElevationMap(core_parameter(cell_n))
    return _MAPS[cell_n]


def _scene(name):
    """(map, planar_terrain result with host tables) for a golden scene."""
    if name == "lidar":
        _MAPS.pop(S.LIDAR_W, None)
        em = _map(S.LIDAR_W)
        S.lidar_frames(em)
        pos, ln = S.lidar_window(em.center), (3.0, 3.0)
    elif name == "big":
        em = _map(S.BIG_W)
        S.set_image(em, S.big_image())
        pos, ln = (0.0, 0.0), (100.0, 100.0)
    else:
        png, scale, pos, ln = S.TERRAINS[name]
        img = S.terrain_image(np.load(S.GOLDEN)["grey__" + name], scale, seed=5 if name == "holes" else None)
        em = _map(img.shape[0] + 2)
        S.set_image(em, img)
    return em, em.planar_terrain(pos, ln, S.params()), pos, ln


def _tables(res):
    t = res["tables"]
    return t["regions"], t["polygons"], t["vertices"]


def _device_result(r):
    return tuple(np.ascontiguousarray(a) for a in (
        np.stack([r["region"], r["status"], r["iterations"]], 1).astype(np.int32),
        np.concatenate([r["cost"][:, None], r["position_plane"], r["position_world"]], 1)))


def _call(em, res, q, wz=0.0, n=0, g=1.05):
    r = em.project_to_planar_regions(res, q, wz, n, g)
    index, point = _device_result(r)
    convex = np.concatenate([r["convex_plane"], r["convex_world"]], 2) if n else np.zeros((len(q), 0, 5))
    return index, point, np.ascontiguousarray(convex)


SCENES = list(S.TERRAINS) + ["lidar", "big"]


@pytest.mark.parametrize("name", SCENES)
def test_device_equals_host_build_and_oracle(native, name):
    em, res, _, _ = _scene(name)
    tables = _tables(res)
    regions = PP.regions_from_tables(*tables)
    assert len(regions) > 0
    big = name == "big"
    q = PP.queries_for(regions, 2000 if big else 10000, seed=SCENES.index(name))
    for wz in (0.0, 0.1):
        got = _call(em, res, q, wz)
        assert_same_bits(got[:2], host_project(native, tables, q, wz)[:2])
        sub = np.concatenate([q[:: max(len(q) // (8 if big else 150), 1)], q[-3:]])
        assert_same_bits(_call(em, res, sub, wz)[:2], PP.project(regions, sub, wz)[:2])
    assert (got[0][:, 0] >= 0).sum() > len(q) // 2
    assert set(got[0][:, 1].tolist()) >= {PP.GROWN, PP.INVALID_QUERY}
    qg = q[:: max(len(q) // (300 if big else 1500), 1)]
    for n, g in ((6, 1.05), (16, 1.11)):
        got = _call(em, res, qg, 0.1, n, g)
        assert_same_bits(got, host_project(native, tables, qg, 0.1, n, g))
        sub = np.concatenate([qg[:: max(len(qg) // (2 if big else 12), 1)], qg[-1:]])
        assert_same_bits(_call(em, res, sub, 0.1, n, g), PP.project(regions, sub, 0.1, n, g))
        assert (got[0][:, 2] > 1).sum() > len(qg) // 4


def test_table_query_and_output_sources_agree():
    import torch
    em, res, pos, ln = _scene("holes")
    dev = em.planar_terrain(pos, ln, S.params(), out=torch.zeros(10 * res["size"][0] * res["size"][1],
                                                                  dtype=torch.float32, device="cuda"))
    assert dev["complete"] and isinstance(dev["tables"]["regions"], torch.Tensor)
    for k in ("regions", "polygons", "vertices"):
        assert np.array_equal(dev["tables"][k].cpu().numpy(), res["tables"][k])
    q = PP.queries_for(PP.regions_from_tables(*_tables(res)), 3000, seed=7)
    want = _call(em, res, q, 0.1, 8, 1.05)
    assert_same_bits(_call(em, dev, q, 0.1, 8, 1.05), want)                         # device tables, host queries
    qd = torch.as_tensor(q, device="cuda")
    r = em.project_to_planar_regions(dev, qd, 0.1, 8, 1.05)                          # all on the device
    assert r["cost"].is_cuda
    assert_same_bits(_device_result({k: v.cpu().numpy() for k, v in r.items()}), want[:2])
    assert np.array_equal(torch.cat([r["convex_plane"], r["convex_world"]], 2).cpu().numpy(), want[2], equal_nan=True)
    r = em.project_to_planar_regions(res, qd, 0.1, 8, 1.05)                          # host tables, device queries
    assert_same_bits(_device_result({k: v.cpu().numpy() for k, v in r.items()}), want[:2])
    out = {"index": torch.empty((len(q), 3), dtype=torch.int32, device="cuda"),
           "point": torch.empty((len(q), 6), dtype=torch.float64, device="cuda"),
           "convex": torch.empty((len(q), 8, 5), dtype=torch.float64, device="cuda")}
    em.project_to_planar_regions(res, q, 0.1, 8, 1.05, out=out)                      # host queries, device output
    assert np.array_equal(out["point"].cpu().numpy(), want[1], equal_nan=True)
    assert np.array_equal(out["index"].cpu().numpy(), want[0])
    r = em.project_to_planar_regions(dev, qd, 0.1)
    lab = res["tables"]["regions"][want[0][:, 0].clip(0), 0]
    assert np.array_equal(r["label"].cpu().numpy(), np.where(want[0][:, 0] >= 0, lab, np.nan), equal_nan=True)


def test_stream_order_and_graph_replay():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    em, res, pos, ln = _scene("terrain")
    regions = PP.regions_from_tables(*_tables(res))
    q1 = PP.queries_for(regions, 2000, seed=1)[:2000]
    q2 = PP.queries_for(regions, 2000, seed=2)[:2000]
    want1, want2 = _call(em, res, q1, 0.0, 6, 1.05), _call(em, res, q2, 0.0, 6, 1.05)
    tabs = [torch.as_tensor(a, device="cuda") for a in _tables(res)]
    # stream order: the queries are written by a long kernel chain on the caller's stream just before the call
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        qd = torch.zeros((2000, 3), dtype=torch.float64, device="cuda")
        big = torch.ones((4096, 4096), device="cuda")
        for _ in range(20):
            big = big @ big / 4096.0
        qd += torch.as_tensor(q1, device="cuda") + big[0, 0].double() * 0
        terrain = {"tables": {"regions": tabs[0], "polygons": tabs[1], "vertices": tabs[2]}}
        r = em.project_to_planar_regions(terrain, qd, 0.0, 6, 1.05)
        got = r["cost"].clone()
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy(), want1[1][:, 0], equal_nan=True)
    # capture with device tables, queries and output, then replay with new queries in the same buffer
    n = 2000
    out = [torch.empty((n, 3), dtype=torch.int32, device="cuda"), torch.empty((n, 6), dtype=torch.float64, device="cuda"),
           torch.empty((n, 6, 5), dtype=torch.float64, device="cuda")]
    t = _lib.EmapRegionTables(tabs[0].data_ptr(), len(tabs[0]), tabs[1].data_ptr(), len(tabs[1]), tabs[2].data_ptr(),
                              len(tabs[2]))
    o = _lib.EmapProjectionOut(*[a.data_ptr() for a in out])
    qd = torch.as_tensor(q1, device="cuda")
    cs = torch.cuda.Stream()
    torch.cuda.synchronize()
    em.set_stream(cs.cuda_stream)
    try:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=cs):
            rc = em._L.emap_project_to_planar_regions(em._h, C.byref(t), 1, n, qd.data_ptr(), 1, 0.0, 6, 1.05,
                                                      C.byref(o), 1)
        assert rc == 0, em._L.emap_last_error(em._h)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out[1].cpu().numpy(), want1[1], equal_nan=True)
        qd.copy_(torch.as_tensor(q2, device="cuda"))
        g.replay()
        torch.cuda.synchronize()
    finally:
        em.set_stream(None)
    assert np.array_equal(out[0].cpu().numpy(), want2[0])
    assert np.array_equal(out[1].cpu().numpy(), want2[1], equal_nan=True)
    assert np.array_equal(out[2].cpu().numpy(), want2[2], equal_nan=True)


def test_launch_count_depends_on_queries_and_growth_only():
    counts = {}
    for name in ("terrain", "holes"):
        em, res, _, _ = _scene(name)
        q = PP.queries_for(PP.regions_from_tables(*_tables(res)), 50, seed=3)
        for n_conv in (0, 5):
            for m in (0, 1, len(q)):
                n0 = em.launch_count()
                em.project_to_planar_regions(res, q[:m], 0.0, n_conv)
                counts.setdefault((n_conv, m > 0), set()).add(em.launch_count() - n0)
    assert counts == {(0, False): {0}, (0, True): {2}, (5, False): {0}, (5, True): {3}}


def test_empty_cases():
    em, res, _, _ = _scene("terrain")
    q = np.array([[0.0, 0.0, 0.0], [1.0, 2.0, 3.0], [np.nan, 0.0, 0.0]])
    empty = {"tables": {"regions": np.zeros((0, 17)), "polygons": np.zeros((0, 5), np.int32),
                        "vertices": np.zeros((0, 2))}}
    r = em.project_to_planar_regions(empty, q, 0.0, 4)
    assert r["status"].tolist() == [PP.NO_REGION, PP.NO_REGION, PP.INVALID_QUERY]
    assert r["region"].tolist() == [-1, -1, -1] and np.isinf(r["cost"]).all()
    assert np.isnan(r["position_world"]).all() and np.isnan(r["convex_world"]).all()
    r = em.project_to_planar_regions(res, np.zeros((0, 3)), 0.0, 4)
    assert r["cost"].shape == (0,) and r["convex_plane"].shape == (0, 4, 2)
    em2 = _map(102)
    S.set_image(em2, S.synthetic("empty", 100, 0))
    none = em2.planar_terrain((0.0, 0.0), (3.0, 3.0), S.params())
    assert len(none["tables"]["regions"]) == 0
    r = em2.project_to_planar_regions(none, q)
    assert r["status"].tolist() == [PP.NO_REGION, PP.NO_REGION, PP.INVALID_QUERY]


@pytest.mark.parametrize("why", ["null tables", "null out", "null queries", "null index", "null convex",
                                 "negative queries", "negative regions", "null regions", "n_convex 2", "n_convex 65",
                                 "growth 1", "growth nan", "penalty negative", "penalty inf", "bad host table"])
def test_rejections_launch_nothing(why):
    from elevation_mapping_cupy_b200 import _lib
    em, res, _, _ = _scene("terrain")
    reg, poly, vert = (np.ascontiguousarray(a) for a in _tables(res))
    if why == "bad host table":
        poly = poly.copy()
        poly[0, 1] = 2
    q = np.zeros((4, 3))
    index, point, convex = np.zeros((4, 3), np.int32), np.zeros((4, 6)), np.zeros((4, 4, 5))
    t = _lib.EmapRegionTables(reg.ctypes.data, len(reg), poly.ctypes.data, len(poly), vert.ctypes.data, len(vert))
    o = _lib.EmapProjectionOut(index.ctypes.data, point.ctypes.data, convex.ctypes.data)
    args = dict(tables=C.byref(t), n=4, q=q.ctypes.data, wz=0.0, nc=4, g=1.05, out=C.byref(o))
    if why == "null tables":
        args["tables"] = None
    elif why == "null out":
        args["out"] = None
    elif why == "null queries":
        args["q"] = None
    elif why == "null index":
        o.index = None
    elif why == "null convex":
        o.convex = None
    elif why == "negative queries":
        args["n"] = -1
    elif why == "negative regions":
        t.n_regions = -1
    elif why == "null regions":
        t.regions = None
    elif why == "n_convex 2":
        args["nc"] = 2
    elif why == "n_convex 65":
        args["nc"] = 65
    elif why == "growth 1":
        args["g"] = 1.0
    elif why == "growth nan":
        args["g"] = float("nan")
    elif why == "penalty negative":
        args["wz"] = -0.1
    elif why == "penalty inf":
        args["wz"] = float("inf")
    n0 = em.launch_count()
    rc = em._L.emap_project_to_planar_regions(em._h, args["tables"], 0, args["n"], args["q"], 0, args["wz"],
                                              args["nc"], args["g"], args["out"], 0)
    assert rc == -1
    assert b"emap_project_to_planar_regions" in em._L.emap_last_error(em._h)
    assert em.launch_count() == n0
    assert not index.any() and not point.any() and not convex.any()
