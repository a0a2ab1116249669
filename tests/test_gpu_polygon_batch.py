"""GPU: get_polygons_traversability / emap_polygon_traversability_batch.  Every entry of a batch must be what the single
call (get_polygon_traversability, itself pinned to tests/polygon_oracle.py by test_gpu_polygon.py) returns for that
polygon on the same map: is_safe, the area and the ring exactly, t bit for bit.  Some cases also check the oracle."""
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


def _same_t(a, b):
    """t bit for bit (any NaN matches any NaN)."""
    if np.isnan(a) or np.isnan(b):
        return bool(np.isnan(a) and np.isnan(b))
    return np.float64(a).view(np.int64) == np.float64(b).view(np.int64)


def _batch(em, polys, hulls=True):
    res = np.full((len(polys), 3), -7.0)
    rings = em.get_polygons_traversability(polys, res, compute_untraversable_polygon=hulls)
    assert len(rings) == len(polys)
    return res, rings


def _check(em, polys, oracle=False, checker=None):
    """One batch against one single call per polygon on the same map state; returns (results, rings)."""
    res, rings = _batch(em, polys)
    again, rings2 = _batch(em, polys)                                 # run to run: identical
    assert np.array_equal(np.nan_to_num(res, nan=-1), np.nan_to_num(again, nan=-1))
    assert all(np.array_equal(a, b) for a, b in zip(rings, rings2))
    state = em.get_state()[0] if oracle else None
    p = em.param
    for i, poly in enumerate(polys):
        out = np.zeros(3)
        n = em.get_polygon_traversability(poly, out)
        ring = em.untraversable_polygon
        assert res[i, 0] == out[0] and res[i, 2] == out[2], (i, res[i], out)
        assert _same_t(res[i, 1], out[1]), (i, res[i, 1], out[1])
        assert rings[i].dtype == np.float64 and rings[i].shape == (n, 2), (i, rings[i].shape, n)
        assert np.array_equal(rings[i], ring), i
        if oracle:
            chk = state[3] if checker is None else checker
            ref = PO.polygon_traversability(poly, em.center, em.cell_n, em.resolution, state[2], chk, p.safe_thresh,
                                            p.safe_min_thresh, p.max_unsafe_n)
            assert res[i, 0] == ref["result"][0] and res[i, 2] == ref["result"][2], i
            t64 = ref["t64"]
            if np.isfinite(t64):
                assert abs(res[i, 1] - t64) <= 1e-6 * abs(t64), (i, res[i, 1], t64)
            else:
                assert _same_t(res[i, 1], t64), (i, res[i, 1], t64)
            assert np.array_equal(rings[i], ref["ring"]), i
    return res, rings


def _polygons(W, res, c, rng):
    """mask_cases moved to the map centre c, seeded stars and footprints, 3- and 1024-vertex polygons, polygons partly or
    fully outside the map, on cell boundaries, and the whole-map square."""
    L = 0.5 * (W - 2) * res
    out = [(poly - pc[:2] + c[:2]).astype(np.float32) for name, poly, pc in PO.mask_cases(W, res)]
    for _ in range(6):
        o = rng.uniform(-0.8 * L, 0.8 * L, 2)
        out.append(PO.star(rng, int(rng.integers(3, 40)), 0.02 * L, rng.uniform(0.05, 0.5) * L, c[0] + o[0], c[1] + o[1]))
    for _ in range(6):                                                # footprints of 0.5 to 1 m
        o = rng.uniform(-0.9 * L, 0.9 * L, 2)
        out.append(PO.star(rng, 8, 0.25, 0.5, c[0] + o[0], c[1] + o[1]))
    out.append(np.array([[0, 0], [0.3, 0], [0, 0.3]], np.float32) + c[:2].astype(np.float32))
    out.append(PO.star(rng, 1024, 0.2 * L, 0.9 * L, c[0], c[1]))
    out.append(np.array([[0.9 * L, 0.9 * L], [1.3 * L, 0.9 * L], [1.3 * L, 1.4 * L]], np.float32) + c[:2])
    out.append(np.array([[-3 * L, -3 * L], [-2 * L, -3 * L], [-2 * L, -2 * L]], np.float32) + c[:2])
    # vertices on cell boundaries and on the tile grid's lines
    k = np.array([[-64, -32], [64, -32], [64, 32], [-64, 32]], np.float64) * res
    out.append((k + c[:2]).astype(np.float32))
    out.append((np.array([[-1, -1], [1, -1], [1, 1], [-1, 1]], np.float32) * L + c[:2]).astype(np.float32))
    return [np.asarray(p, np.float32) for p in out]


@pytest.mark.parametrize("W", [130, 202, 1024, 2048, 2049])
def test_batch_after_frames_matches_single_calls(W):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(W)
    em = _mk(p)
    for f in range(3):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=625, max_range=6.0)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    polys = _polygons(W, p.resolution, em.center, np.random.default_rng(W))
    res, rings = _check(em, polys, oracle=W <= 1024)
    assert (res[:, 0] == 0).any() and (res[:, 0] == 1).any()


def _designed(W, seed):
    rng = np.random.default_rng(seed)
    st = np.zeros((7, W, W), np.float32)
    st[2] = (rng.random((W, W)) < 0.9).astype(np.float32)
    st[3] = np.where(rng.random((W, W)) < 0.02, rng.random((W, W)) * 0.6, 1.0).astype(np.float32)
    return st, rng


def test_order_and_duplicates():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    st, rng = _designed(W, 3)
    em.set_state(st)
    polys = _polygons(W, p.resolution, em.center, rng)
    res, rings = _check(em, polys)
    perm = rng.permutation(len(polys))
    res_p, rings_p = _batch(em, [polys[i] for i in perm])
    assert np.array_equal(res_p, res[perm])
    assert all(np.array_equal(rings_p[j], rings[i]) for j, i in enumerate(perm))
    dup = [polys[3]] * 5 + [polys[0], polys[3]]
    res_d, rings_d = _batch(em, dup)
    assert all(np.array_equal(res_d[k], res[3]) for k in (0, 1, 2, 3, 4, 6))
    assert all(np.array_equal(rings_d[k], rings[3]) for k in (0, 1, 2, 3, 4, 6))


def _three(W, res):
    """Three small polygons far apart and one overlapping the first, in metres about the map centre (0, 0)."""
    a = np.array([[-2.0, -2.0], [-1.0, -2.0], [-1.0, -1.0], [-2.0, -1.0]], np.float32)
    b = np.array([[1.0, 1.0], [2.0, 1.0], [2.0, 2.0], [1.0, 2.0]], np.float32)
    c = np.array([[1.0, -2.0], [2.0, -2.0], [1.5, -1.0]], np.float32)
    d = a + np.float32(0.5)
    return [a, b, c, d]


def _cell(em, x, y):
    """(row, col) of the map cell under the point (x, y) of a map centred at (0, 0)."""
    return int(x / em.resolution + em.cell_n / 2), int(y / em.resolution + em.cell_n / 2)


def test_non_finite_cells():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    polys = _three(W, p.resolution)
    base, _ = _designed(W, 4)
    base[2] = 1.0
    inside = _cell(em, -1.5, -1.8)                                   # inside polygon 0 only (not the overlap)
    overlap = _cell(em, -1.2, -1.2)                                  # inside polygons 0 and 3
    outside = (10, 190)                                              # outside every polygon and its tiles
    # a NaN checker value inside one polygon only: it lies outside the others, so it poisons them too (NaN * 0)
    st = base.copy(); st[3][inside] = np.nan
    em.set_state(st)
    res, _ = _check(em, polys, oracle=True)
    assert np.isnan(res[:, 1]).all()
    # a NaN checker value outside every polygon poisons every entry (NaN * 0)
    st = base.copy(); st[3][outside] = np.nan
    em.set_state(st)
    res, _ = _check(em, polys, oracle=True)
    assert np.isnan(res[:, 1]).all()
    # -inf inside polygon 1 (untraversability +inf there) and outside the others (inf * 0 = NaN)
    st = base.copy(); st[3][_cell(em, 1.5, 1.5)] = -np.inf
    em.set_state(st)
    res, _ = _check(em, polys, oracle=True)
    assert res[1, 1] == np.inf or np.isnan(res[1, 1])
    assert np.isnan(res[0, 1]) and np.isnan(res[2, 1])
    # a non-finite is_valid outside every polygon: Σvalid is NaN, so t = 0
    st = base.copy(); st[2][outside] = np.inf
    em.set_state(st)
    res, _ = _check(em, polys, oracle=True)
    assert (res[:, 1] == 0).all()
    st = base.copy(); st[2][outside] = np.nan
    em.set_state(st)
    res, _ = _check(em, polys, oracle=True)
    assert (res[:, 1] == 0).all()
    # an untraversable cell in the overlap of polygons 0 and 3 counts for both
    st = base.copy(); st[3] = 1.0; st[3][overlap] = 0.0
    em.set_state(st)
    res, _ = _check(em, polys, oracle=True)
    assert res[0, 1] > 0 and res[3, 1] > 0 and res[1, 1] == 0 and res[2, 1] == 0
    # on a map with an outside cell at +inf checker (untraversability -inf outside: NaN * 0 as well)
    st = base.copy(); st[3][outside] = np.inf
    em.set_state(st)
    res, _ = _check(em, polys, oracle=True)
    assert np.isnan(res[:, 1]).all()


def test_each_rule_decides_an_entry_and_rings():
    """core parameters: a cell is over at untraversability > 0.3, the maximum test at > 0.6, max_unsafe_n 10."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    st = np.zeros((7, W, W), np.float32)
    st[2] = 1.0; st[3] = 1.0
    sq = lambda x, y, h: np.array([[x - h, y - h], [x + h, y - h], [x + h, y + h], [x - h, y + h]], np.float32)
    polys = [sq(-3, -3, 0.5), sq(-3, 0, 0.5), sq(-3, 3, 0.5), sq(0, -3, 0.5), sq(0, 0, 0.5), sq(3, 3, 1.5),
             np.array([[50, 50], [60, 50], [60, 60]], np.float32), sq(0, 3, 0.5)]
    r, c = _cell(em, -3, 0)
    st[3, r, c] = 0.5                                                 # polygon 1: one over cell, a point, safe
    r, c = _cell(em, -3, 3)
    st[3, r - 3:r + 3, c] = 0.5                                       # polygon 2: collinear over cells, a line, safe
    r, c = _cell(em, 0, -3)
    st[3, r - 5:r + 1, c - 1:c + 1] = 0.5                             # polygon 3: 12 over cells, the count decides
    r, c = _cell(em, 0, 0)
    st[3, r, c] = 0.3                                                 # polygon 4: one cell at 0.7: the maximum decides
    blob = np.random.default_rng(5).random((40, 40)) < 0.1            # polygon 5: a large ring
    r, c = _cell(em, 3, 3)
    st[3, r - 20:r + 20, c - 20:c + 20][blob] = 0.2
    em.set_state(st)
    res, rings = _check(em, polys, oracle=True)
    assert res[0, 0] == 1 and len(rings[0]) == 0
    assert res[1, 0] == 1 and len(rings[1]) == 0
    assert res[2, 0] == 1 and len(rings[2]) == 0
    assert res[3, 0] == 0 and len(rings[3]) == 5
    assert res[4, 0] == 0
    assert res[5, 0] == 0 and len(rings[5]) > 6
    assert res[6, 0] == 0                                             # outside the map: the clipped-area rule
    assert res[7, 0] == 1


def test_no_hulls_and_capacity():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    st, rng = _designed(W, 6)
    em.set_state(st)
    polys = _polygons(W, p.resolution, em.center, rng)
    res, rings = _batch(em, polys)
    res_n, rings_n = _batch(em, polys, hulls=False)
    assert np.array_equal(res, res_n)
    assert all(r.shape == (0, 2) for r in rings_n) and any(len(r) for r in rings)
    # the C ABI: a capacity below the total gives EMAP_ERR_INVALID, the total, the results and the offsets
    L, h = em._L, em._h
    n = np.array([len(q) for q in polys], np.int32)
    xy = np.ascontiguousarray(np.concatenate(polys))
    total = sum(len(r) for r in rings)
    out = np.zeros((len(polys), 3))
    off = np.full(len(polys) + 1, -5, np.int64)
    hull = np.zeros((total, 2))
    rows = C.c_int64(total - 1)
    assert L.emap_polygon_traversability_batch(h, len(polys), n.ctypes.data, xy.ctypes.data, None, p.safe_thresh,
                                               p.safe_min_thresh, p.max_unsafe_n, out.ctypes.data, hull.ctypes.data,
                                               off.ctypes.data, C.byref(rows)) == -1
    assert rows.value == total and np.array_equal(out, res)
    assert np.array_equal(np.diff(off), [len(r) for r in rings]) and off[0] == 0
    rows = C.c_int64(total)
    assert L.emap_polygon_traversability_batch(h, len(polys), n.ctypes.data, xy.ctypes.data, None, p.safe_thresh,
                                               p.safe_min_thresh, p.max_unsafe_n, out.ctypes.data, hull.ctypes.data,
                                               off.ctypes.data, C.byref(rows)) == 0
    assert rows.value == total and np.array_equal(hull, np.concatenate(rings))
    # no hulls: the offsets and the row count come back zero
    assert L.emap_polygon_traversability_batch(h, len(polys), n.ctypes.data, xy.ctypes.data, None, p.safe_thresh,
                                               p.safe_min_thresh, p.max_unsafe_n, out.ctypes.data, None,
                                               off.ctypes.data, C.byref(rows)) == 0
    assert rows.value == 0 and not off.any() and np.array_equal(out, res)


def test_c_abi_argument_checks():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 130
    p = core_parameter(W)
    em = _mk(p)
    L, h = em._L, em._h
    sq = np.array([[-1, -1], [1, -1], [1, 1], [-1, 1]], np.float32)
    out = np.zeros((4097, 3))
    off = np.zeros(4098, np.int64)
    hull = np.zeros((16, 2))

    def call(B, n, xy, res=out, hl=hull, offs=off, rows=16):
        r = C.c_int64(rows)
        n = np.asarray(n, np.int32)
        return L.emap_polygon_traversability_batch(
            h, B, None if n is None else n.ctypes.data, None if xy is None else xy.ctypes.data, None, 0.7, 0.4, 10,
            None if res is None else res.ctypes.data, None if hl is None else hl.ctypes.data,
            None if offs is None else offs.ctypes.data, C.byref(r))

    xy = np.ascontiguousarray(np.tile(sq, (4097, 1)))
    assert call(1, [4], xy) == 0
    assert call(0, [4], xy) == -1
    assert call(-1, [4], xy) == -1
    assert call(4097, [4] * 4097, xy) == -1
    assert call(4096, [4] * 4096, xy, hl=None) == 0
    assert call(2, [4, 2], xy) == -1
    assert call(2, [4, 1025], np.zeros((1029, 2), np.float32)) == -1
    assert call(1, [4], None) == -1
    assert call(1, [4], xy, res=None) == -1
    assert call(1, [4], xy, offs=None) == -1
    assert call(1, [4], xy, rows=-1) == -1
    assert L.emap_polygon_traversability_batch(h, 1, None, xy.ctypes.data, None, 0.7, 0.4, 10, out.ctypes.data,
                                               None, None, None) == -1
    assert L.emap_polygon_traversability_batch(h, 1, np.array([4], np.int32).ctypes.data, xy.ctypes.data, None, 0.7,
                                               0.4, 10, out.ctypes.data, None, None, None) == 0


def test_checker_layers_streams_and_single_call_state():
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import Parameter
    p = Parameter(); p.update()
    em = _mk(p)
    pts, R, t = wl.reference_test_cloud(0, n_ch=5)
    em.input_pointcloud(torch.from_numpy(pts).cuda(), ["x", "y", "z", "a", "b"], R, t, 0, 0)
    polys = [np.array([[-3.0, -2.5], [3.1, -2.8], [2.7, 3.3], [-2.6, 2.9]], np.float32),
             np.array([[0.1, 0.1], [0.6, 0.1], [0.4, 0.5]], np.float32),
             np.array([[-1.0, 0.2], [-0.4, 0.3], [-0.6, 0.9], [-1.1, 0.8]], np.float32)]
    sem = em.semantic_map.layer_names
    assert sem, "the reference cloud's extra channels make semantic layers"
    for layer in ["smooth", sem[0]]:
        p.checker_layer = layer
        plane = em.get_layer(layer).detach().cpu().numpy().astype(np.float32)
        _check(em, polys, oracle=True, checker=plane)
    p.checker_layer = "traversability"
    # the single call's mask and ring stay as they were
    out = np.zeros(3)
    n = em.get_polygon_traversability(polys[0], out)
    mask = em.mask.clone()
    ring = np.zeros((n, 2)); em.get_untraversable_polygon(ring)
    _batch(em, polys[1:])
    assert torch.equal(em.mask, mask)
    ring2 = np.zeros((n, 2)); em.get_untraversable_polygon(ring2)
    assert np.array_equal(ring, ring2)
    # a state written on a non-default torch stream just before the call
    st, _ = _designed(em.cell_n, 8)
    st[3][100:140, 100:140] = 0.0
    want = _mk(p)
    want.set_state(st, center=em.center.astype(np.float64))
    res_w, rings_w = _batch(want, polys)
    s = torch.cuda.Stream()
    dev = torch.from_numpy(st).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        em.elevation_map.copy_(dev)
        res, rings = _batch(em, polys)
    torch.cuda.synchronize()
    assert np.array_equal(np.nan_to_num(res, nan=-1), np.nan_to_num(res_w, nan=-1))
    assert all(np.array_equal(a, b) for a, b in zip(rings, rings_w))


def test_full_batch_2048():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 2048
    p = core_parameter(W)
    em = _mk(p)
    st, rng = _designed(W, 9)
    em.set_state(st)
    L = 0.5 * (W - 2) * p.resolution
    s = np.linspace(-0.95, 0.95, 4096)
    path = np.stack([s * L, 0.6 * L * np.sin(3 * s)], 1)
    polys = [PO.star(rng, 8, 0.25, 0.5, x, y) for x, y in path]
    res, rings = _check(em, polys)
    assert (res[:, 0] == 0).any() and (res[:, 0] == 1).any()


def test_threshold_above_one_then_normal():
    """safe_thresh > 1: fp32(1 - safe_thresh) < 0, so the masked 0 of every cell outside a polygon is over as well
    (traversability_polygon.py:25 compares the whole interior), and each polygon's count and ring take the whole map.
    The batch must still equal the single call, and the column extremes it leaves must not disturb the calls that
    follow at the usual threshold."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    st, rng = _designed(W, 11)
    em.set_state(st)
    polys = _polygons(W, p.resolution, em.center, rng)
    p.safe_thresh = 1.2
    res, rings = _check(em, polys, oracle=True)
    assert (res[:, 0] == 0).all() and all(len(r) > 0 for r in rings)
    res_n, rings_n = _batch(em, polys, hulls=False)
    assert np.array_equal(np.nan_to_num(res_n, nan=-1), np.nan_to_num(res, nan=-1))
    p.safe_thresh = 0.7
    _check(em, polys, oracle=True)
    _check(em, polys[::-1], oracle=True)
