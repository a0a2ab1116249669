"""GPU: get_polygon_traversability / emap_polygon_traversability against tests/polygon_oracle.py (whose mask is pinned to
the reference's own kernel source by tests/test_polygon_cpu.py) and the stored reference masks."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import polygon_oracle as PO          # noqa: E402

pytestmark = pytest.mark.gpu


def _mk(param):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    return ElevationMap(param)


def _check(em, poly, checker=None):
    """One call of the engine against the oracle on the map's current state; returns the oracle's dict."""
    state, _ = em.get_state()
    p = em.param
    chk = state[3] if checker is None else checker
    ref = PO.polygon_traversability(poly, em.center, em.cell_n, em.resolution, state[2], chk, p.safe_thresh,
                                    p.safe_min_thresh, p.max_unsafe_n)
    out = np.zeros(3)
    n = em.get_polygon_traversability(poly, out)
    assert np.array_equal(em.mask.cpu().numpy(), ref["mask"].astype(np.float32))
    assert out[0] == ref["result"][0] and out[2] == ref["result"][2]
    t64 = ref["t64"]
    if np.isnan(t64):
        assert np.isnan(out[1])
    else:
        assert abs(out[1] - t64) <= 1e-6 * abs(t64), (out[1], t64)
    assert n == len(ref["ring"])
    ring = np.zeros((n, 2))
    em.get_untraversable_polygon(ring)
    assert PO.same_ring(ring, ref["ring"]), (ring, ref["ring"])
    if n:   # the documented convention: smallest (row, col) first, counter-clockwise in (row, col)
        assert np.array_equal(ring, ref["ring"])
    again = np.zeros(3)
    assert em.get_polygon_traversability(poly, again) == n
    assert np.array_equal(np.nan_to_num(again, nan=-1), np.nan_to_num(out, nan=-1))      # deterministic t
    return ref


@pytest.mark.parametrize("W", [130, 202, 1024, 2048])
def test_polygons_after_frames_match_oracle(W):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(W)
    em = _mk(p)
    for f in range(3):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=625, max_range=6.0)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    c = em.center
    n_over = 0
    for name, poly, pc in PO.mask_cases(W, p.resolution):
        if name.startswith("moved"):
            continue
        ref = _check(em, (poly - pc[:2] + c[:2]).astype(np.float32))
        n_over += ref["over"]
    # the whole map, so that the statistics see the cells the frames made valid (the nearest ground returns of a
    # sensor 1.5 m up lie about 3.2 m away)
    L = 0.5 * (W - 2) * p.resolution
    ref = _check(em, (np.array([[-1, -1], [1, -1], [1, 1], [-1, 1]], np.float32) * L + c[:2]))
    assert (ref["mask"][1:-1, 1:-1] * (em.get_state()[0][2][1:-1, 1:-1] > 0.5)).sum() > 0


def test_golden_reference_masks():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 130
    p = core_parameter(W)
    em = _mk(p)
    gold = np.load(os.path.join(HERE, "golden", "polygon_core130.npz"))
    st = np.zeros((7, W, W), np.float32)
    st[2] = 1.0; st[3] = 1.0
    for name, poly, center in PO.mask_cases(W, p.resolution):
        em.set_state(st, center=center.astype(np.float64))
        out = np.zeros(3)
        em.get_polygon_traversability(poly, out)
        ref = np.unpackbits(gold[name])[:W * W].reshape(W, W).astype(np.float32)
        assert np.array_equal(em.mask.cpu().numpy(), ref), name
        _check(em, poly)


def _designed(W, seed):
    rng = np.random.default_rng(seed)
    st = np.zeros((7, W, W), np.float32)
    st[2] = (rng.random((W, W)) < 0.9).astype(np.float32)
    st[3] = 1.0
    return st, rng


def test_designed_maps_decide_each_rule():
    """core parameters: safe_thresh 0.7 (a cell is over at untraversability > 0.3), safe_min_thresh 0.4 (max 0.6),
    max_unsafe_n 10."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    big = np.array([[-3.5, -3.5], [3.6, -3.2], [3.4, 3.7], [-3.3, 3.1]], np.float32)
    st, rng = _designed(W, 1)
    st[2] = 1.0
    em.set_state(st)
    ref = _check(em, big)                                             # nothing over: safe, no polygon
    assert ref["result"][0] == 1.0 and len(ref["ring"]) == 0 and ref["over"] == 0
    st[3, 100, 90] = 0.5                                              # one over cell: a point, no polygon
    em.set_state(st)
    ref = _check(em, big)
    assert ref["over"] == 1 and len(ref["ring"]) == 0 and ref["result"][0] == 1.0
    st[3, 60:70, 90] = 0.5                                            # collinear over cells: a line, no polygon
    st[3, 100, 90] = 1.0
    em.set_state(st)
    ref = _check(em, big)
    assert ref["over"] == 10 and len(ref["ring"]) == 0 and ref["result"][0] == 1.0
    st[3, 80, 95] = 0.5                                               # 11 cells at 0.5: the count decides
    em.set_state(st)
    ref = _check(em, big)
    assert ref["over"] == 11 and len(ref["ring"]) == 4 and ref["result"][0] == 0.0
    st[3, 60:70, 90] = 1.0
    st[3, 80, 95] = 0.3                                               # one cell at 0.7 untraversable: the maximum decides
    st[3, 81, 97] = 0.5
    em.set_state(st)
    ref = _check(em, big)
    assert ref["over"] == 2 and ref["result"][0] == 0.0
    st, rng = _designed(W, 2)                                         # random untraversable blobs: a real hull
    st[3] = np.where(rng.random((W, W)) < 0.02, rng.random((W, W)) * 0.6, 1.0).astype(np.float32)
    em.set_state(st)
    ref = _check(em, big)
    assert len(ref["ring"]) > 4
    st[2, 100, 100] = 1.0
    st[3, 100, 100] = np.nan                                          # NaN inside: t NaN, the maximum test fails
    em.set_state(st)
    ref = _check(em, big)
    assert np.isnan(ref["t64"])
    st[3, 100, 100] = 1.0
    st[2, 5, 5] = 1.0
    st[3, 5, 5] = np.nan                                              # NaN on a valid cell outside the polygon (NaN * 0)
    em.set_state(st)
    ref = _check(em, np.array([[0, 0], [2, 0], [0, 2]], np.float32))
    assert np.isnan(ref["t64"])
    for name, poly, center in PO.mask_cases(W, p.resolution):        # moved maps: large coordinates through fp16
        em.set_state(st, center=center.astype(np.float64))
        _check(em, poly)


def test_plugin_and_semantic_checker_layers():
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import Parameter
    p = Parameter(); p.update()
    em = _mk(p)
    pts, R, t = wl.reference_test_cloud(0, n_ch=5)
    em.input_pointcloud(torch.from_numpy(pts).cuda(), ["x", "y", "z", "a", "b"], R, t, 0, 0)
    poly = np.array([[-3.0, -2.5], [3.1, -2.8], [2.7, 3.3], [-2.6, 2.9]], np.float32)
    sem = em.semantic_map.layer_names
    assert sem, "the reference cloud's extra channels make semantic layers"
    for layer in ["smooth", sem[0]]:
        p.checker_layer = layer
        plane = em.get_layer(layer)
        _check(em, poly, checker=plane.detach().cpu().numpy().astype(np.float32))
    p.checker_layer = "traversability"


def test_c_abi_argument_checks():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 130
    em = _mk(core_parameter(W))
    st = np.zeros((7, W, W), np.float32)
    st[2] = 1.0; st[3] = np.where(np.random.default_rng(0).random((W, W)) < 0.1, 0.0, 1.0)
    em.set_state(st)
    L, h = em._L, em._h
    res = np.zeros(3)
    hull = np.zeros((4, 2))
    poly = np.array([[-2, -2], [2, -2], [2, 2], [-2, 2]], np.float32)
    cap = C.c_int32(4)
    assert L.emap_polygon_traversability(h, poly.ctypes.data, 2, None, 0.7, 0.4, 10, res.ctypes.data, hull.ctypes.data,
                                         C.byref(cap), None) == -1
    big = np.zeros((1025, 2), np.float32)
    assert L.emap_polygon_traversability(h, big.ctypes.data, 1025, None, 0.7, 0.4, 10, res.ctypes.data,
                                         hull.ctypes.data, C.byref(cap), None) == -1
    rc = L.emap_polygon_traversability(h, poly.ctypes.data, 4, None, 0.7, 0.4, 10, res.ctypes.data, hull.ctypes.data,
                                       C.byref(cap), None)
    assert rc == -1 and cap.value > 4                                  # the needed ring length comes back
    need = cap.value
    hull = np.zeros((need, 2))
    assert L.emap_polygon_traversability(h, poly.ctypes.data, 4, None, 0.7, 0.4, 10, res.ctypes.data, hull.ctypes.data,
                                         C.byref(cap), None) == 0
    assert cap.value == need and np.array_equal(hull[0], hull[-1])


def test_reference_smoke_sequence_with_polygon():
    """test_elevation_mapping.py:46-118 in order, the polygon call included (its result array is an int array there)."""
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import Parameter
    p = Parameter(); p.update()
    em = _mk(p)
    assert em.untraversable_polygon.shape == (1, 2)                    # EM.py:110
    pts, R, t = wl.reference_test_cloud(0, n_ch=5)
    em.input_pointcloud(torch.from_numpy(pts).cuda(), ["x", "y", "z", "a", "b"], R, t, 0, 0)
    em.update_normal(em.elevation_map[0].contiguous())
    for i in range(20):
        em.move_to(np.array([i * 0.01, i * 0.02, i * 0.01]), np.random.rand(3, 3))
    polygon = torch.tensor([[0, 0], [2, 0], [0, 2]], dtype=torch.float64, device="cuda")
    result = np.array([0, 0, 0])
    number_polygons = em.get_polygon_traversability(polygon, result)
    untraversable_polygon = np.zeros((number_polygons, 2))
    em.get_untraversable_polygon(untraversable_polygon)
    assert result[2] == 2                                              # area 2 m^2, truncated into the int array
    assert int(em.mask.sum().item()) > 0
    em.clear()
