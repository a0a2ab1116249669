"""GPU: the plane decomposition pipeline on a caller's grid, with the preprocessing's resampling
(ElevationMap.plane_decomposition / emap_plane_decomposition).  Identity: without resampling, a get_submap window fed
back in gives planar_terrain's bytes for that window, for every scene, with host and device output.  Resampled: 0.05 m
to 0.04 m (the node's parameters.yaml), 0.04 to 0.05, an exact 2x (0.02 to 0.04) and 0.08 to 0.04 against the composed
oracle in tests/resample_oracle.py: the resampled elevation, decisions and layers exact, plane parameters to 1e-9,
region geometry to 1e-12, smooth_planar within EMAP_POST_GAUSS_ULPS.  Also a yawed get_transformed_submap grid, host
and device grids giving the same bytes, graph capture with a device grid, the result fed to project_to_planar_regions
and grid_derivatives, an empty grid, and every rejection writing and launching nothing."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import plane_scenes as S   # noqa: E402

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
import planar_regions_oracle as RO   # noqa: E402
import planar_terrain_oracle as TO   # noqa: E402
import resample_oracle as RS   # noqa: E402
import test_gpu_planar_regions as TR   # noqa: E402

W = 102
EMAP_ERR_INVALID = -1
NAMES = ["elevation_raw", "elevation_before_postprocess", "segmentation", "plane_classification", "elevationWithNaN",
         "elevationWithNaN_i", "elevationWithNaNClosed", "elevationWithNaNClosedDilated", "smooth_planar", "elevation"]
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
    if hasattr(a, "cpu"):
        a = a.cpu().numpy()
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


def _device_submap(em, pos, ln):
    import torch
    rows, cols = em.get_submap(pos, ln, ["elevation"])["size"]
    out = torch.empty(max(rows * cols, 1), dtype=torch.float32, device="cuda")
    return em.get_submap(pos, ln, ["elevation"], out=out)


def _same_result(a, b):
    assert (a["success"], a["complete"], a["highest_label"], a["size"]) == \
        (b["success"], b["complete"], b["highest_label"], b["size"])
    assert a["resolution"] == b["resolution"]
    assert np.array_equal(a["origin"], b["origin"]) and np.array_equal(_host(a["centre"]), _host(b["centre"]))
    assert _host(a["planes"]).tobytes() == _host(b["planes"]).tobytes()
    for k in ("regions", "polygons", "vertices"):
        assert _host(a["tables"][k]).tobytes() == _host(b["tables"][k]).tobytes()
    if a["success"]:
        for k in NAMES:
            assert np.array_equal(_bits(a["layers"][k]), _bits(b["layers"][k])), k


def _scene_map(name):
    if name in S.TERRAINS:
        png, scale, pos, ln = S.TERRAINS[name]
        g = np.load(S.GOLDEN)
        img = S.terrain_image(g["grey__" + name], scale, seed=5 if name == "holes" else None)
        em = _map(img.shape[0] + 2)
        S.set_image(em, img)
        return em, pos, ln
    em = _map(W)
    S.set_image(em, S.synthetic(name, W - 2, 3))
    return em, (0.3, -0.2), (3.0, 3.0)


@pytest.mark.parametrize("device_out", [False, True])
@pytest.mark.parametrize("scene", ["ramps", "stairs", "holes", "diagonal", "rough"] + list(S.TERRAINS))
def test_identity_with_planar_terrain(scene, device_out):
    import torch
    em, pos, ln = _scene_map(scene)
    p = S.params()
    grid = _device_submap(em, pos, ln)
    rows, cols = grid["size"]
    outs = [torch.empty(10 * rows * cols, dtype=torch.float32, device="cuda") if device_out else None for _ in range(2)]
    want = em.planar_terrain(pos, ln, p, out=outs[0])
    got = em.plane_decomposition(grid, "elevation", p, out=outs[1])
    assert got["success"]
    _same_result(got, want)


def _resampled_case(res_map, res_new, scene="stairs", side=3.0, pos=(0.1, -0.2), cells=None):
    """A map window as plane_decomposition's grid; `cells` crops it to cells x cells (its centre kept)."""
    em = _map(W, res_map)
    S.set_image(em, S.synthetic(scene, W - 2, 2))
    p = S.params(resolution=res_new)
    grid = em.get_submap(pos, (side, side), ["elevation"])
    if cells is not None:
        layer = np.ascontiguousarray(grid["layers"]["elevation"][:cells, :cells])
        grid = dict(grid, layers={"elevation": layer}, size=layer.shape)
    return em, p, grid


def _check_against_oracle(em, grid, p, res_in, t):
    want = RS.decompose(grid["layers"]["elevation"], res_in, grid["centre"], p)
    assert t["size"] == want["size"] and t["resolution"] == want["resolution"]
    assert np.array_equal(t["origin"], want["origin"])
    seg = want["seg"]
    assert t["success"] == seg["success"]
    L = t["layers"]
    assert np.array_equal(_bits(L["elevation_before_postprocess"]), _bits(seg["elevation"]))
    assert np.array_equal(L["segmentation"].astype(np.int32), seg["segmentation"])
    assert np.array_equal(L["plane_classification"], seg["classification"])
    assert t["highest_label"] == seg["highest_label"]
    assert t["planes"].shape == seg["planes"].shape
    assert np.abs(t["planes"] - seg["planes"]).max(initial=0.0) <= 1e-9
    regions = RO.extract(L["segmentation"], t["planes"], t["origin"], t["resolution"], p.margin_size,
                         p.extracted_planes_height_offset)
    TR._compare(t["regions"], regions)
    post = TO.postprocess(L["elevation_before_postprocess"], L["plane_classification"], t["resolution"], p)
    for name in ("elevationWithNaN", "elevationWithNaN_i", "elevationWithNaNClosed", "elevationWithNaNClosedDilated",
                 "elevation"):
        a, b = np.asarray(L[name], np.float32), np.asarray(post[name], np.float32)
        assert np.array_equal(a, b, equal_nan=True), name
    _, _, kg = post["sizes"]
    dil = L["elevationWithNaNClosedDilated"]
    assert TO.ulps(L["smooth_planar"], post["smooth_planar"], np.nanmax(np.abs(dil), initial=0.0)) <= \
        (0 if kg <= 3 else TO.gauss_ulps_bound(kg))
    assert np.array_equal(_bits(L["elevation_raw"]), _bits(grid["layers"]["elevation"]))
    return want


@pytest.mark.parametrize("res_map,res_new", [(0.05, 0.04), (0.04, 0.05), (0.02, 0.04), (0.08, 0.04)])
@pytest.mark.parametrize("scene", ["ramps", "stairs", "holes"])
def test_resampled_matches_composed_oracle(scene, res_map, res_new):
    cells = 80 if res_map == 0.02 else None        # 80 x 80 cells at 0.02 m: an exact 2x downscale
    em, p, grid = _resampled_case(res_map, res_new, scene, 1.7 if cells else 3.0, cells=cells)
    t = em.plane_decomposition(grid, "elevation", p)
    want = _check_against_oracle(em, grid, p, res_map, t)
    assert t["size"] != grid["size"] and t["success"]
    assert (t["layers"]["plane_classification"] == 1).any()
    if res_map == 0.02:
        assert grid["size"] == (80, 80) and want["size"] == (40, 40)


def test_node_parameters_yaml_on_a_05_map():
    """The node's unmodified parameters.yaml (RANSAC off) on a 0.05 m map: the 3 m x 3 m window is resampled to 75 x 75
    cells at 0.04 m."""
    from elevation_mapping_cupy_b200.plane_segmentation import PlaneSegmentationParams
    p = PlaneSegmentationParams.from_yaml(os.path.join(HERE, "golden", "planes", "parameters.yaml"))
    p.include_ransac_refinement = False
    assert p.resolution == 0.04
    em, _, grid = _resampled_case(0.05, 0.04, "ramps", cells=60)
    t = em.plane_decomposition(grid, "elevation", p)
    assert t["size"] == (75, 75) and t["success"]
    _check_against_oracle(em, grid, p, 0.05, t)


def test_transformed_submap_grid():
    em = _map(W, 0.05)
    S.set_image(em, S.synthetic("ramps", W - 2, 5))
    yaw = 0.3
    T = np.eye(4)
    T[:2, :2] = [[math.cos(yaw), -math.sin(yaw)], [math.sin(yaw), math.cos(yaw)]]
    T[:3, 3] = [0.2, -0.1, 0.05]
    grid = em.get_transformed_submap((0.2, 0.1), (3.0, 3.0), ["elevation"], T)
    assert grid["success"]
    p = S.params(resolution=0.04)
    t = em.plane_decomposition(grid, "elevation", p)
    g = dict(grid, centre=grid["frame_centre"])
    _check_against_oracle(em, g, p, 0.05, t)


def test_host_and_device_grids_give_the_same_bytes():
    import torch
    em, p, grid = _resampled_case(0.05, 0.04)
    dgrid = _device_submap(em, (0.1, -0.2), (3.0, 3.0))
    a = em.plane_decomposition(grid, "elevation", p)
    b = em.plane_decomposition(dgrid, "elevation", p)
    b["layers"]["elevation_raw"] = b["layers"]["elevation_raw"].cpu().numpy()
    _same_result(a, b)
    rows, cols = a["size"]
    out = torch.empty(10 * rows * cols, dtype=torch.float32, device="cuda")
    d = em.plane_decomposition(dgrid, "elevation", p, out=out)
    d["layers"]["elevation_raw"] = d["layers"]["elevation_raw"].cpu().numpy()
    _same_result(d, a)


def _raw(em, grid_arr, res, centre, p, post=True, fill=5, out_floats=None, planes_less=0, caps=(64, 256, 4096),
         on_device=False):
    from elevation_mapping_cupy_b200 import _lib
    pc, rp = p.to_c(), p.regions_to_c()
    pp = p.postprocess_to_c()
    R, Cc = grid_arr.shape if grid_arr is not None else (0, 0)
    size = np.zeros(2, np.int64)
    r = C.c_double(0.0)
    em._L.emap_plane_grid_geometry(max(R, 1), max(Cc, 1), res if res > 0 else 0.04, C.byref(pc), size.ctypes.data,
                                   C.addressof(r))
    n = int(size[0]) * int(size[1])
    cap = max(int(em._L.emap_plane_capacity(int(size[0]), int(size[1]), C.byref(pc))), 1)
    out = np.full(max(10 * n, 1), fill, np.float32)
    planes = np.full((cap, 7), fill, np.float64)
    tabs = (np.full((caps[0], 17), fill, np.float64), np.full((caps[1], 5), fill, np.int32),
            np.full((caps[2], 2), fill, np.float64))
    info = np.full(9, fill, np.int32)
    o = _lib.EmapRegionOut(tabs[0].ctypes.data, caps[0], tabs[1].ctypes.data, caps[1], tabs[2].ctypes.data, caps[2])
    data = None if grid_arr is None else np.ascontiguousarray(grid_arr, np.float32)
    g = _lib.EmapGrid(None if data is None else data.ctypes.data, R, Cc, (C.c_double * 2)(*centre), res)
    n0 = em.launch_count()
    rc = em._L.emap_plane_decomposition(em._h, C.byref(g), 0, C.byref(pc), C.byref(rp),
                                        C.byref(pp) if post else None, out.ctypes.data, 0,
                                        out.size if out_floats is None else out_floats, planes.ctypes.data,
                                        cap - planes_less, C.byref(o), info.ctypes.data)
    return rc, out, planes, tabs, info, em.launch_count() - n0


def test_empty_grid_and_launch_counts():
    em, p, grid = _resampled_case(0.05, 0.04)
    img = np.full((60, 60), np.nan, np.float32)
    rc, out, planes, tabs, info, launches = _raw(em, img, 0.05, (0.0, 0.0), p)
    assert rc == 0 and info[0] == 0 and info[8] == 1 and (out == 5).all()
    rc2, *_, launches2 = _raw(em, np.asarray(grid["layers"]["elevation"]), 0.05, (0.0, 0.0), p)
    assert rc2 == 0 and launches2 == launches
    # one launch more than the window call at the same size (the resampling), the grid's copy replacing k_submap
    em4 = _map(W, 0.04)
    S.set_image(em4, S.synthetic("stairs", W - 2, 2))
    g4 = em4.get_submap((0.0, 0.0), (3.0, 3.0), ["elevation"])
    n0 = em4.launch_count()
    em4.planar_terrain((0.0, 0.0), (3.0, 3.0), S.params())
    window = em4.launch_count() - n0
    n0 = em4.launch_count()
    em4.plane_decomposition(g4, "elevation", S.params())
    assert em4.launch_count() - n0 == window - 1        # no k_submap, no resampling
    n0 = em4.launch_count()
    em4.plane_decomposition(g4, "elevation", S.params(resolution=0.05))
    assert em4.launch_count() - n0 == window


def test_result_feeds_projection_and_lookups():
    import torch
    em, p, grid = _resampled_case(0.05, 0.04)
    t = em.plane_decomposition(grid, "elevation", p)
    assert len(t["tables"]["regions"]) > 0
    rng = np.random.default_rng(3)
    q = np.zeros((64, 3))
    q[:, :2] = t["centre"] + rng.uniform(-1.2, 1.2, (64, 2))
    q[:, 2] = 0.2
    pr = em.project_to_planar_regions(t, q)
    assert (pr["region"] >= 0).all()
    d = em.grid_derivatives(t, "smooth_planar", q[:, :2], curvature=True)
    assert (d["status"] == 0).all()
    gd = em.grid_derivatives(t, "elevation", q[:, :2])
    assert np.isfinite(gd["gradient"]).all()
    # device tables give the same projection
    rows, cols = t["size"]
    out = torch.empty(10 * rows * cols, dtype=torch.float32, device="cuda")
    td = em.plane_decomposition(grid, "elevation", p, out=out)
    pd = em.project_to_planar_regions(td, torch.as_tensor(q, device="cuda"))
    assert np.array_equal(pd["position_world"].cpu().numpy(), pr["position_world"])


def test_device_grid_call_captures_into_a_graph():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    em, p, grid = _resampled_case(0.05, 0.04)
    dgrid = _device_submap(em, (0.1, -0.2), (3.0, 3.0))
    ref = em.plane_decomposition(grid, "elevation", p)
    rows, cols = ref["size"]
    pc, rp, pp = p.to_c(), p.regions_to_c(), p.postprocess_to_c()
    cap = int(em._L.emap_plane_capacity(rows, cols, C.byref(pc)))
    caps = [len(ref["tables"][k]) for k in ("regions", "polygons", "vertices")]
    out = torch.zeros(10 * rows * cols, dtype=torch.float32, device="cuda")
    planes = torch.zeros((cap, 7), dtype=torch.float64, device="cuda")
    tabs = (torch.zeros((caps[0], 17), dtype=torch.float64, device="cuda"),
            torch.zeros((caps[1], 5), dtype=torch.int32, device="cuda"),
            torch.zeros((caps[2], 2), dtype=torch.float64, device="cuda"))
    o = _lib.EmapRegionOut(tabs[0].data_ptr(), caps[0], tabs[1].data_ptr(), caps[1], tabs[2].data_ptr(), caps[2])
    info = torch.zeros(9, dtype=torch.int32, device="cuda")
    data = dgrid["layers"]["elevation"]
    g = _lib.EmapGrid(data.data_ptr(), data.shape[0], data.shape[1], (C.c_double * 2)(*dgrid["centre"].tolist()), 0.05)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    em.set_stream(s.cuda_stream)
    try:
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=s):
            rc = em._L.emap_plane_decomposition(em._h, C.byref(g), 1, C.byref(pc), C.byref(rp), C.byref(pp),
                                                out.data_ptr(), 1, out.numel(), planes.data_ptr(), cap, C.byref(o),
                                                info.data_ptr())
        assert rc == 0, em._L.emap_last_error(em._h)
        cg.replay()
        torch.cuda.synchronize()
    finally:
        em.set_stream(None)
    assert info.cpu().numpy().tolist() == [1, rows, cols, ref["highest_label"], len(ref["planes"])] + caps + [1]
    got = out.cpu().numpy().reshape(10, rows, cols)
    for k, name in enumerate(NAMES[1:], 1):
        assert np.array_equal(_bits(got[k]), _bits(ref["layers"][name]))
    assert (got[0] == 0).all()          # layer 0 is not written


@pytest.mark.parametrize("why", ["null grid data", "rows 0", "res nan", "position inf", "grid too big",
                                 "resampled too big", "resampled to 0", "smaller than dilation", "null post",
                                 "out small", "planes small", "margin", "ransac", "resolution nan", "median"])
def test_rejections_write_nothing(why):
    em, p, grid = _resampled_case(0.05, 0.04)
    img = np.asarray(grid["layers"]["elevation"], np.float32)
    res, centre = 0.05, (0.0, 0.0)
    kw = {"margin": {"margin_size": 5}, "ransac": {"include_ransac_refinement": True},
          "resolution nan": {"resolution": float("nan")}, "median": {"median_kernel": 4},
          "resampled too big": {"resolution": 0.05 / 1.2}, "resampled to 0": {"resolution": 10.0},
          "smaller than dilation": {"resolution": 0.2, "smoothing_dilation_size": 2.0}}.get(why, {})
    q = S.params(**{"resolution": 0.04, **kw})
    if why == "rows 0":
        img = img[:0]
    if why == "res nan":
        res = float("nan")
    if why == "position inf":
        centre = (float("inf"), 0.0)
    if why in ("grid too big", "resampled too big"):
        img = np.zeros((2048 if why == "grid too big" else 1800, 8), np.float32)
        if why == "grid too big":
            q = S.params(resolution=0.0)
    rc, out, planes, tabs, info, launches = _raw(
        em, None if why == "null grid data" else img, res, centre, q, post=why != "null post",
        out_floats=(10 * 75 * 75 - 1) if why == "out small" else None, planes_less=1 if why == "planes small" else 0)
    assert rc == EMAP_ERR_INVALID, why
    assert launches == 0
    assert (out == 5).all() and (planes == 5).all() and (info == 5).all()
    assert all((t == 5).all() for t in tabs)
    msg = em._L.emap_last_error(em._h)
    if why != "null post":
        assert (msg.decode() if isinstance(msg, bytes) else str(msg)).startswith("emap_plane_decomposition:")
