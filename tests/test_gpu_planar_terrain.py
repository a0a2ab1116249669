"""GPU: the planar terrain of a map window (ElevationMap.planar_terrain / emap_planar_terrain).  Layers 0 .. 3, the plane
table, the region tables and the info words are extract_planar_regions' bytes; layers 4 .. 7 and 9 equal the NumPy +
cv2 restatement in tests/planar_terrain_oracle.py as values (NaN positions exact, -0.0 == +0.0); smooth_planar equals
cv2 for 3-tap Gaussians and is within EMAP_POST_GAUSS_ULPS(k) of it otherwise, and equals the library's restatement of its
own arithmetic bit for bit.  Scenes: the synthetic plane scenes, the reference's demo terrains, the LiDAR map and a
2047^2 window, at 0.02, 0.04, 0.05 and 0.1 m, with horizontal offsets 0, 1 and 2 and zero and non-zero height offsets.
Also: host and device output agree, two calls give the same bytes, the map state is untouched, the launch count does
not depend on the scene, a device-output call can be captured into a CUDA graph, windows without a planar cell, without
a finite cell, outside the map and smaller than the dilation kernel, and every rejected argument writes nothing."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import plane_scenes as S   # noqa: E402

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
import planar_terrain_oracle as TO   # noqa: E402

W = 102
EMAP_ERR_INVALID = -1
NAMES = ["elevation_raw", "elevation_before_postprocess", "segmentation", "plane_classification", "elevationWithNaN",
         "elevationWithNaN_i", "elevationWithNaNClosed", "elevationWithNaNClosedDilated", "smooth_planar", "elevation"]
REGION_NAMES = ["elevation_raw", "elevation", "segmentation", "plane_classification"]
_MAPS = {}


def _map(cell_n, res=0.04):
    key = (cell_n, res)
    if key not in _MAPS:
        from elevation_mapping_cupy_b200.parameter import core_parameter
        from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
        _MAPS.clear()
        _MAPS[key] = ElevationMap(core_parameter(cell_n, resolution=res))
    return _MAPS[key]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _params(res=0.04, **kw):
    return S.params(resolution=res, **kw)


def _same_values(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    assert np.array_equal(a, b, equal_nan=True)


def _check(em, pos, ln, p):
    """The call against extract_planar_regions and the oracle; returns the call's result."""
    t = em.planar_terrain(pos, ln, p)
    r = em.extract_planar_regions(pos, ln, p)
    assert t["success"] == r["success"] and t["complete"] and r["complete"]
    assert (t["highest_label"], t["size"]) == (r["highest_label"], r["size"])
    assert t["planes"].tobytes() == r["planes"].tobytes()
    for k in ("regions", "polygons", "vertices"):
        assert t["tables"][k].tobytes() == r["tables"][k].tobytes()
    if not t["success"]:
        return t
    for a, b in zip(NAMES[:4], REGION_NAMES):
        assert np.array_equal(_bits(t["layers"][a]), _bits(r["layers"][b]))
    res = float(em.resolution)
    want = TO.postprocess(r["layers"]["elevation"], r["layers"]["plane_classification"], res, p)
    for name in ("elevationWithNaN", "elevationWithNaN_i", "elevationWithNaNClosed", "elevationWithNaNClosedDilated",
                 "elevation"):
        _same_values(t["layers"][name], want[name])
    _, kb, kg = want["sizes"]
    got, dil = t["layers"]["smooth_planar"], t["layers"]["elevationWithNaNClosedDilated"]
    mine = TO.gauss_restated(TO.box_restated(dil, kb), kg)       # bits, except the payload of a NaN
    assert np.array_equal(np.isnan(got), np.isnan(mine))
    assert np.array_equal(_bits(got)[~np.isnan(got)], _bits(mine)[~np.isnan(mine)])
    if kg <= 3:
        _same_values(got, want["smooth_planar"])
    else:
        assert TO.ulps(got, want["smooth_planar"], np.nanmax(np.abs(dil), initial=0.0)) <= TO.gauss_ulps_bound(kg)
    return t


SCENES = ["ramps", "stairs", "holes", "diagonal", "rough"]
WINDOWS = [("whole", (0.0, 0.0), (4.0, 4.0)), ("node", (0.3, -0.2), (3.0, 3.0)), ("clipped", (1.7, 1.5), (1.5, 1.0))]


@pytest.mark.parametrize("heights", [(0.0, 0.0), (0.03, 0.02), (0.0, -0.05)])
@pytest.mark.parametrize("offset", [0, 1, 2])
@pytest.mark.parametrize("scene", SCENES)
def test_scene_matches_oracle(scene, offset, heights):
    em = _map(W)
    S.set_image(em, S.synthetic(scene, W - 2, SCENES.index(scene)))
    p = _params(nonplanar_horizontal_offset=offset, extracted_planes_height_offset=heights[0],
                nonplanar_height_offset=heights[1])
    for _, pos, ln in WINDOWS:
        assert _check(em, pos, ln, p)["success"]


@pytest.mark.parametrize("res", [0.02, 0.05, 0.1])
@pytest.mark.parametrize("scene", ["ramps", "stairs", "holes"])
def test_resolutions(scene, res):
    em = _map(W, res)
    S.set_image(em, S.synthetic(scene, W - 2, 1))
    for offset in (0, 2):
        p = _params(res, nonplanar_horizontal_offset=offset)
        side = (W - 2) * res
        t = _check(em, (0.0, 0.0), (side, side), p)
        assert t["success"] and (t["layers"]["plane_classification"] == 1).any()


def _golden_map(name):
    if name == "lidar":
        _MAPS.pop((S.LIDAR_W, 0.04), None)
        em = _map(S.LIDAR_W)
        S.lidar_frames(em)
        return em, S.lidar_window(em.center), (3.0, 3.0)
    if name == "big":
        em = _map(S.BIG_W)
        S.set_image(em, S.big_image())
        return em, (0.0, 0.0), (100.0, 100.0)
    png, scale, pos, ln = S.TERRAINS[name]
    g = np.load(S.GOLDEN)
    img = S.terrain_image(g["grey__" + name], scale, seed=5 if name == "holes" else None)
    em = _map(img.shape[0] + 2)
    S.set_image(em, img)
    return em, pos, ln


@pytest.mark.parametrize("name", list(S.TERRAINS) + ["lidar", "big"])
def test_golden_scene(name):
    em, pos, ln = _golden_map(name)
    t = _check(em, pos, ln, _params())
    assert t["success"] and (t["layers"]["plane_classification"] == 1).any()


@pytest.mark.parametrize("name", ["lidar", "big"])
def test_host_device_determinism_and_state(name):
    import torch
    em, pos, ln = _golden_map(name)
    p = _params()
    before = em.get_state()
    a = em.planar_terrain(pos, ln, p)
    b = em.planar_terrain(pos, ln, p)
    after = em.get_state()
    assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(before, after))
    rows, cols = a["size"]
    for k in NAMES:
        assert np.array_equal(_bits(a["layers"][k]), _bits(b["layers"][k]))
    out = torch.empty(10 * rows * cols, dtype=torch.float32, device="cuda")
    d = em.planar_terrain(pos, ln, p, out=out)
    assert d["complete"] and d["regions"] is None
    for k in NAMES:
        assert np.array_equal(_bits(d["layers"][k].cpu().numpy()), _bits(a["layers"][k]))
    for k in ("regions", "polygons", "vertices"):
        assert d["tables"][k].cpu().numpy().tobytes() == a["tables"][k].tobytes()


def _raw_call(em, pos, ln, p, post, caps=(64, 256, 4096), fill=5, out_floats=None, planes_less=0):
    from elevation_mapping_cupy_b200 import _lib
    pc, rp = p.to_c(), p.regions_to_c()
    req = np.array(list(pos) + list(ln), np.float64)
    rows, cols = em.get_submap(pos, ln, ["elevation"])["size"]
    n = rows * cols
    cap = max(int(em._L.emap_plane_capacity(rows, cols, C.byref(pc))), 1)
    out = np.full(max(10 * n, 1), fill, np.float32)
    planes = np.full((cap, 7), fill, np.float64)
    tabs = (np.full((caps[0], 17), fill, np.float64), np.full((caps[1], 5), fill, np.int32),
            np.full((caps[2], 2), fill, np.float64))
    info = np.full(9, fill, np.int32)
    o = _lib.EmapRegionOut(tabs[0].ctypes.data, caps[0], tabs[1].ctypes.data, caps[1], tabs[2].ctypes.data, caps[2])
    n0 = em.launch_count()
    rc = em._L.emap_planar_terrain(em._h, req.ctypes.data, C.byref(pc), C.byref(rp),
                                   None if post is None else C.byref(post), out.ctypes.data, 0,
                                   out.size if out_floats is None else out_floats, planes.ctypes.data,
                                   cap - planes_less, C.byref(o), info.ctypes.data)
    return rc, out, planes, tabs, info, em.launch_count() - n0


def test_no_planar_cell_no_finite_cell_and_outside():
    em = _map(W)
    S.set_image(em, S.synthetic("stairs", W - 2, 0))
    t = _check(em, (0.0, 0.0), (4.0, 4.0), _params(local_plane_inclination_cos=1.0))   # n.z > 1: no planar cell
    assert t["success"] and not (t["layers"]["plane_classification"] == 1).any()
    for k in NAMES[4:9]:
        assert np.isnan(t["layers"][k]).all()
    assert np.isfinite(t["layers"]["elevation"]).all()
    S.set_image(em, S.synthetic("empty", W - 2, 0))
    rc, out, planes, tabs, info, _ = _raw_call(em, (0.0, 0.0), (4.0, 4.0), _params(), _params().postprocess_to_c())
    assert rc == 0 and info[0] == 0 and info[8] == 1 and (out == 5).all()
    t = em.planar_terrain((0.0, 0.0), (4.0, 4.0), _params())
    assert not t["success"] and t["regions"] == []
    t = em.planar_terrain((50.0, 0.0), (4.0, 4.0), _params())
    assert not t["success"] and t["size"] == (0, 0) and t["complete"]


def test_window_smaller_than_the_dilation_kernel():
    em = _map(W)
    S.set_image(em, S.synthetic("stairs", W - 2, 0))
    p = _params()
    rc, out, planes, tabs, info, launches = _raw_call(em, (0.0, 0.0), (0.3, 4.0), p, p.postprocess_to_c())
    assert rc == EMAP_ERR_INVALID and launches == 0
    assert (out == 5).all() and (info == 5).all() and (planes == 5).all()
    # a one-cell dilation kernel takes the same window
    q = _params(smoothing_dilation_size=0.0)
    t = _check(em, (0.0, 0.0), (0.3, 4.0), q)
    assert t["success"] and t["size"][0] < 11


def test_launch_count_does_not_depend_on_the_scene():
    em = _map(W)
    counts = []
    for scene in SCENES + ["empty"]:
        S.set_image(em, S.synthetic(scene, W - 2, 1))
        n0 = em.launch_count()
        em.planar_terrain((0.1, 0.1), (3.0, 3.0), _params())
        counts.append(em.launch_count() - n0)
    assert len(set(counts)) == 1, counts


def test_device_call_captures_into_a_graph():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    em = _map(W)
    S.set_image(em, S.synthetic("stairs", W - 2, 0))
    p = _params()
    ref = em.planar_terrain((0.0, 0.0), (3.0, 3.0), p)
    rows, cols = ref["size"]
    pc, rp, pp = p.to_c(), p.regions_to_c(), p.postprocess_to_c()
    req = np.array([0.0, 0.0, 3.0, 3.0], np.float64)
    cap = int(em._L.emap_plane_capacity(rows, cols, C.byref(pc)))
    caps = [len(ref["tables"][k]) for k in ("regions", "polygons", "vertices")]
    out = torch.zeros(10 * rows * cols, dtype=torch.float32, device="cuda")
    planes = torch.zeros((cap, 7), dtype=torch.float64, device="cuda")
    tabs = (torch.zeros((caps[0], 17), dtype=torch.float64, device="cuda"),
            torch.zeros((caps[1], 5), dtype=torch.int32, device="cuda"),
            torch.zeros((caps[2], 2), dtype=torch.float64, device="cuda"))
    o = _lib.EmapRegionOut(tabs[0].data_ptr(), caps[0], tabs[1].data_ptr(), caps[1], tabs[2].data_ptr(), caps[2])
    info = torch.zeros(9, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    em.set_stream(s.cuda_stream)
    try:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            rc = em._L.emap_planar_terrain(em._h, req.ctypes.data, C.byref(pc), C.byref(rp), C.byref(pp),
                                           out.data_ptr(), 1, out.numel(), planes.data_ptr(), cap, C.byref(o),
                                           info.data_ptr())
        assert rc == 0, em._L.emap_last_error(em._h)
        g.replay()
        torch.cuda.synchronize()
    finally:
        em.set_stream(None)
    assert info.cpu().numpy().tolist() == [1, rows, cols, ref["highest_label"], len(ref["planes"])] + caps + [1]
    got = out.cpu().numpy().reshape(10, rows, cols)
    for k, name in enumerate(NAMES):
        assert np.array_equal(_bits(got[k]), _bits(ref["layers"][name]))


@pytest.mark.parametrize("why", ["null post", "dilation nan", "box negative", "gauss inf", "kernel too big",
                                 "offset negative", "offset too big", "height nan", "out small", "planes small",
                                 "margin", "ransac"])
def test_rejections_write_nothing(why):
    em = _map(W)
    S.set_image(em, S.synthetic("stairs", W - 2, 0))
    kw = {"dilation nan": {"smoothing_dilation_size": float("nan")},
          "box negative": {"smoothing_box_kernel_size": -0.1},
          "gauss inf": {"smoothing_gauss_kernel_size": float("inf")},
          "kernel too big": {"smoothing_box_kernel_size": 32 * 0.04},
          "offset negative": {"nonplanar_horizontal_offset": -1},
          "offset too big": {"nonplanar_horizontal_offset": 32},
          "height nan": {"nonplanar_height_offset": float("nan")},
          "margin": {"margin_size": 5},
          "ransac": {"include_ransac_refinement": True}}.get(why, {})
    p = _params(**kw)
    rows, cols = em.get_submap((0.0, 0.0), (2.0, 2.0), ["elevation"])["size"]
    rc, out, planes, tabs, info, launches = _raw_call(em, (0.0, 0.0), (2.0, 2.0), p,
                                            None if why == "null post" else p.postprocess_to_c(),
                                            out_floats=10 * rows * cols - 1 if why == "out small" else None,
                                            planes_less=1 if why == "planes small" else 0)
    assert rc == EMAP_ERR_INVALID, why
    assert launches == 0
    assert (out == 5).all() and (planes == 5).all() and (info == 5).all()
    assert all((t == 5).all() for t in tabs)
    msg = em._L.emap_last_error(em._h)
    assert (msg.decode() if isinstance(msg, bytes) else str(msg)).startswith("emap_planar_terrain:")
