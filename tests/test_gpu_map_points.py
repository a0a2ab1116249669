"""GPU: the exported map as a point cloud (get_map_points / emap_get_map_points), as normal arrows (get_normal_arrows /
emap_get_normal_arrows), the normal colour layer (`normal_color`) and the normal maps (get_normal_maps / get_normal_ref).
Every row must be, bit for bit, what tests/map_points_oracle.py computes from a full get_maps_with_names_ref export of
the same state, on maps built from seeded LiDAR frames and moved off the cell grid, at W = 202, 301 (odd), 1024 and
2048.  Also: capacity and argument rejections, the all-invalid map, repeatability, and an unchanged map state."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import map_points_oracle as MO      # noqa: E402
import submap_oracle as SO          # noqa: E402

pytestmark = pytest.mark.gpu

NAMES = ["elevation", "normal_x", "normal_y", "normal_z", "normal_color"]
_MAPS = {}


def _frames(em, W, n_frames, seed):
    from elevation_mapping_cupy_b200 import workloads as wl
    for f in range(n_frames):
        pts, R, t = wl.lidar_cloud(seed, f, n_rings=64 if W > 500 else 32, n_az=1250, max_range=0.45 * W * 0.04)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    return R, t


def _make(W, seed=3):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    em = ElevationMap(core_parameter(W))
    R, t = _frames(em, W, 3, seed)
    em.move_to(np.asarray(t, np.float64) + [0.37, -0.53, 0.0], R)              # a moved centre, off the cell grid
    return em


def _map(W):
    """(map, full export of NAMES) of a W x W map after seeded LiDAR frames and a move_to, made once per W."""
    if W not in _MAPS:
        em = _make(W)
        full = np.zeros((len(NAMES), W - 2, W - 2), np.float32)
        em.get_maps_with_names_ref(NAMES, full)
        assert np.isfinite(full[0]).sum() > 1000 and np.isnan(full[0]).sum() > 1000
        _MAPS[W] = (em, full)
    return _MAPS[W]


def _eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("W", [202, 301, 1024, 2048])
def test_points_arrows_and_colour_match_the_oracle(W):
    em, full = _map(W)
    res, c = em.resolution, em.center
    pts = em.get_map_points()
    assert _eq(pts, MO.map_points(full[0], res, c))
    assert len(pts) == np.isfinite(full[0]).sum()
    ids, seg = em.get_normal_arrows()
    want_ids, want_seg = MO.normal_arrows(full[0], full[1], full[2], full[3], res, c)
    assert _eq(ids, want_ids) and _eq(seg, want_seg)
    assert len(ids) > 1000
    assert _eq(full[4], MO.normal_color(full[1], full[2], full[3]))


@pytest.mark.parametrize("W", [202, 301, 2048])
def test_normal_maps_are_the_normal_export(W):
    em, full = _map(W)
    maps = em.get_normal_maps()
    assert _eq(maps, full[1:4])
    outs = [np.full((W - 2, W - 2), -7.0, np.float32) for _ in range(3)]
    em.get_normal_ref(*outs)
    for k in range(3):
        assert _eq(outs[k], full[1 + k])


@pytest.mark.parametrize("W", [202, 1024])
def test_normal_color_through_submaps(W):
    em, full = _map(W)
    half = 0.5 * (W - 2) * em.resolution
    c = em.center.astype(np.float64)
    reqs = [(c[:2], (2.0, 2.0)), (c[:2] + (half - 0.3, -half + 0.3), (3.0, 1.0)), (c[:2], (4 * half, 4 * half))]
    res = em.get_submaps(reqs, ["normal_color", "elevation"])
    for (pos, ln), r in zip(reqs, res):
        want, _ = SO.window(W, em.resolution, c, np.array([pos[0], pos[1], ln[0], ln[1]], np.float64))
        crop = SO.crop(full[[4, 0]], want)
        assert r["success"] and _eq(r["layers"]["normal_color"], crop[0]) and _eq(r["layers"]["elevation"], crop[1])


def test_all_invalid_map_returns_no_rows():
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    em = ElevationMap(core_parameter(202))
    assert em.get_map_points().shape == (0, 3)
    ids, seg = em.get_normal_arrows()
    assert ids.shape == (0,) and seg.shape == (0, 6)
    n = C.c_int64(0)
    assert em._L.emap_get_map_points(em._h, None, C.byref(n)) == 0 and n.value == 0
    assert em._L.emap_get_normal_arrows(em._h, None, None, C.byref(n)) == 0 and n.value == 0


def test_capacity_and_argument_rejections():
    em, full = _map(202)
    L, h = em._L, em._h
    need_p = int(np.isfinite(full[0]).sum())
    need_a = len(em.get_normal_arrows()[0])
    xyz = np.full((need_p, 3), -7.0, np.float32)
    ids = np.full(need_a, -7, np.int32)
    seg = np.full((need_a, 6), -7.0, np.float64)
    for cap in (0, need_p - 1):
        n = C.c_int64(cap)
        assert L.emap_get_map_points(h, xyz.ctypes.data, C.byref(n)) == -1 and n.value == need_p
        assert (xyz == -7.0).all()
    for cap in (0, need_a - 1):
        n = C.c_int64(cap)
        assert L.emap_get_normal_arrows(h, ids.ctypes.data, seg.ctypes.data, C.byref(n)) == -1 and n.value == need_a
        assert (ids == -7).all() and (seg == -7.0).all()
    for n0, p in ((5, None), (-1, xyz.ctypes.data)):
        n = C.c_int64(n0)
        assert L.emap_get_map_points(h, p, C.byref(n)) == -1 and n.value == n0
    assert L.emap_get_map_points(h, xyz.ctypes.data, None) == -1
    for a, b in ((None, seg.ctypes.data), (ids.ctypes.data, None)):
        n = C.c_int64(need_a)
        assert L.emap_get_normal_arrows(h, a, b, C.byref(n)) == -1 and n.value == need_a
    assert L.emap_get_normal_arrows(h, ids.ctypes.data, seg.ctypes.data, None) == -1
    assert (xyz == -7.0).all() and (ids == -7).all() and (seg == -7.0).all()
    n = C.c_int64(need_p)                                   # an exact capacity fills every row
    assert L.emap_get_map_points(h, xyz.ctypes.data, C.byref(n)) == 0 and n.value == need_p
    assert _eq(xyz, MO.map_points(full[0], em.resolution, em.center))


def test_repeatable_and_state_unchanged():
    em, _ = _map(202)
    s0, n0 = em.get_state()
    a = em.get_map_points(), em.get_normal_arrows()
    b = em.get_map_points(), em.get_normal_arrows()
    assert _eq(a[0], b[0]) and _eq(a[1][0], b[1][0]) and _eq(a[1][1], b[1][1])
    s1, n1 = em.get_state()
    assert _eq(s0, s1) and _eq(n0, n1)


def test_get_grid_map_with_normal_color():
    """A stand-in for the C++ bridge's get_grid_map with enable_normal_color (WRAP:213-252): the layers that exist, then
    get_normal_ref into three (cell_n-2)^2 arrays and the colour layer, here the `normal_color` export."""
    em, full = _map(202)
    n = em.cell_n - 2
    layers = {}
    for name in ["elevation", "traversability", "variance"]:
        if em.exists_layer(name):
            m = np.zeros((n, n), np.float32)
            em.get_map_with_name_ref(name, m)
            layers[name] = m
    normals = [np.zeros((n, n), np.float32) for _ in range(3)]
    em.get_normal_ref(*normals)
    color = np.zeros((n, n), np.float32)
    em.get_map_with_name_ref("normal_color", color)
    layers["color"] = color
    assert _eq(layers["elevation"], full[0]) and _eq(color, MO.normal_color(*normals))
