"""GPU: plane segmentation of a map window (ElevationMap.segment_planes / emap_segment_planes).  Per scene: elevation_raw
is get_submaps' window bit for bit; the filled and denoised elevation, the labels, the classification and highest_label
are exact; the plane table has the expected labels in their order, with support and normal within 1e-9.  Expected
values come from the NumPy + cv2 restatement in tests/plane_segmentation_oracle.py when cv2 is importable, and from
tests/golden/planes_golden.npz (the reference's demo terrains, the default map after LiDAR frames, a 2047^2 window)
whether or not it is.  Also: host and device output agree, two calls give the same bytes, the map state is untouched,
the launch count does not depend on the scene, a device-output call can be captured into a CUDA graph (so it makes no
host synchronisation), and every rejected argument writes nothing."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import plane_scenes as S   # noqa: E402

pytestmark = pytest.mark.gpu

W = 102
RES = S.RES
TOL = 1e-9
EMAP_ERR_INVALID = -1
_params = S.params
_set = S.set_image
_MAPS = {}


def _oracle():
    try:
        import cv2  # noqa: F401
    except ImportError:
        return None
    import plane_segmentation_oracle as PO
    return PO


def _scene(name, seed):
    return S.synthetic(name, W - 2, seed)


SCENES = ["ramps", "stairs", "holes", "diagonal", "rough"]
CASES = [("default", {}), ("conn8", {"connectivity": 8}), ("opening", {"planarity_opening_filter": 1}),
         ("median5x2", {"median_kernel": 5, "median_repeats": 2}), ("kernel5", {"kernel_size": 5}),
         ("min_points", {"min_number_points_per_label": 40})]
WINDOWS = [("whole", (0.0, 0.0), (4.0, 4.0)), ("node", (0.3, -0.2), (3.0, 3.0)), ("clipped", (1.7, 1.5), (1.5, 1.0))]


def _map(cell_n):
    if cell_n not in _MAPS:
        from elevation_mapping_cupy_b200.parameter import core_parameter
        from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
        _MAPS.clear()                    # one map alive at a time: the 2049^2 one is large
        _MAPS[cell_n] = ElevationMap(core_parameter(cell_n))
    return _MAPS[cell_n]


@pytest.fixture
def em():
    return _map(W)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _run(em, pos, ln, p):
    res = em.segment_planes(pos, ln, p)
    raw = em.get_submap(pos, ln, ["elevation"])
    assert res["success"] == raw["success"]
    assert np.array_equal(_bits(res["layers"]["elevation_raw"]), _bits(raw["layers"]["elevation"]))
    return res, raw["layers"]["elevation"]


def _same(res, elevation, segmentation, highest, planes):
    L = res["layers"]
    assert np.array_equal(_bits(L["elevation"]), _bits(elevation))
    assert np.array_equal(L["segmentation"], np.asarray(segmentation, np.float32))
    assert np.array_equal(L["plane_classification"], (np.asarray(segmentation) > 0).astype(np.float32))
    assert res["highest_label"] == highest
    assert np.array_equal(res["planes"][:, 0], planes[:, 0])
    assert np.abs(res["planes"][:, 1:] - planes[:, 1:]).max(initial=0.0) < TOL


def _check(em, pos, ln, p):
    """The call against the live oracle (cv2 needed)."""
    PO = _oracle()
    if PO is None:
        pytest.skip("the live oracle needs cv2; the golden scenes cover this machine")
    res, raw = _run(em, pos, ln, p)
    o = PO.segment(raw, RES, res["origin"], p)
    if not o["success"]:
        assert not res["success"]
        return res, o
    assert res["success"]
    assert o["margin"] > TOL, "the scene holds a decision within 1e-9 of its threshold"
    _same(res, o["elevation"], o["segmentation"], o["highest_label"], o["planes"])
    return res, o


@pytest.mark.parametrize("case,kw", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("scene", SCENES)
def test_scene_matches_oracle(em, scene, case, kw):
    _set(em, _scene(scene, SCENES.index(scene)))
    p = _params(**kw)
    for _, pos, ln in WINDOWS:
        _check(em, pos, ln, p)


GOLDEN_SCENES = list(S.TERRAINS) + ["lidar", "big"]


def _golden_map(name):
    """The map of a golden scene, and the window (position, length)."""
    if name == "lidar":
        _MAPS.pop(S.LIDAR_W, None)       # a fresh map: the frames start from an empty one centred at the origin
        em = _map(S.LIDAR_W)
        S.lidar_frames(em)
        return em, S.lidar_window(em.center), (3.0, 3.0)
    if name == "big":
        em = _map(S.BIG_W)
        _set(em, S.big_image())
        return em, (0.0, 0.0), (100.0, 100.0)
    png, scale, pos, ln = S.TERRAINS[name]
    g = np.load(S.GOLDEN)
    img = S.terrain_image(g["grey__" + name], scale, seed=5 if name == "holes" else None)
    em = _map(img.shape[0] + 2)
    _set(em, img)
    return em, pos, ln


@pytest.mark.parametrize("case", ["conn4", "conn8"])
@pytest.mark.parametrize("name", GOLDEN_SCENES)
def test_golden_scene(name, case):
    em, pos, ln = _golden_map(name)
    g = np.load(S.GOLDEN)
    k = f"{name}__{case}__"
    p = _params(connectivity=8 if case == "conn8" else 4)
    res, raw = _run(em, pos, ln, p)
    assert res["success"]
    assert S.digest(raw) == str(g[k + "raw"])
    L = res["layers"]
    assert S.digest(L["elevation"]) == str(g[k + "elevation"])
    seg = L["segmentation"]
    assert S.digest(seg) == str(g[k + "segmentation"])
    assert np.array_equal(L["plane_classification"], (seg > 0).astype(np.float32))
    assert res["highest_label"] == int(g[k + "highest_label"])
    planes = g[k + "planes"]
    assert np.array_equal(res["planes"][:, 0], planes[:, 0])
    assert np.abs(res["planes"][:, 1:] - planes[:, 1:]).max(initial=0.0) < TOL
    PO = _oracle()
    if PO is not None:
        o = PO.segment(raw, RES, res["origin"], p)
        _same(res, o["elevation"], o["segmentation"], o["highest_label"], o["planes"])


@pytest.mark.parametrize("name", ["lidar", "big"])
def test_large_and_lidar_maps_host_device_determinism_state(name):
    import torch
    em, pos, ln = _golden_map(name)
    p = _params()
    before = em.get_state()
    n0 = em.launch_count()
    a = em.segment_planes(pos, ln, p)
    n1 = em.launch_count()
    b = em.segment_planes(pos, ln, p)
    assert em.launch_count() - n1 == n1 - n0
    after = em.get_state()
    assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(before, after))
    rows, cols = a["size"]
    out = torch.empty(4 * rows * cols, dtype=torch.float32, device="cuda")
    d = em.segment_planes(pos, ln, p, out=out)
    for k in a["layers"]:
        assert np.array_equal(_bits(a["layers"][k]), _bits(b["layers"][k]))
        assert np.array_equal(_bits(d["layers"][k].cpu().numpy()), _bits(a["layers"][k]))
    assert a["planes"].tobytes() == b["planes"].tobytes() == d["planes"].cpu().numpy().tobytes()
    assert a["highest_label"] == b["highest_label"] == d["highest_label"]


def test_ramps_one_plane_one_background(em):
    _set(em, _scene("ramps", 0))
    p = _params()
    res, raw = _run(em, (0.0, 0.0), (4.0, 4.0), p)
    seg = res["layers"]["segmentation"]
    steep = (slice(5, 95), slice(73, 97))               # the 32 degree ramp's interior
    assert (seg[steep] == 0).all()
    kept = set(np.unique(seg).tolist()) - {0.0}
    assert res["highest_label"] > len(kept)             # a label was set to background
    gentle = res["planes"][np.isin(res["planes"][:, 0], seg[5:95, 38:62])]
    assert len(gentle) == 1 and abs(gentle[0, 6] - np.cos(np.radians(20))) < 1e-4
    PO = _oracle()
    if PO is not None:
        o = PO.segment(raw, RES, res["origin"], p)
        assert o["planar"][steep].all()                 # locally planar: the per-label test set it to background
        _same(res, o["elevation"], o["segmentation"], o["highest_label"], o["planes"])


def test_small_label_keeps_its_label(em):
    _set(em, _scene("rough", 4))
    res, _ = _run(em, (0.0, 0.0), (4.0, 4.0), _params(min_number_points_per_label=40))
    kept = set(np.unique(res["layers"]["segmentation"]).tolist()) - {0.0}
    with_plane = set(res["planes"][:, 0].tolist())
    assert kept - with_plane, "some labels below min points keep their label without a plane"
    if _oracle() is not None:
        _check(em, (0.0, 0.0), (4.0, 4.0), _params(min_number_points_per_label=40))


def test_no_finite_cell_and_outside(em):
    _set(em, _scene("empty", 0))
    out = np.full(4 * 100 * 100, 7.0, np.float32)
    res = em.segment_planes((0.0, 0.0), (4.0, 4.0), _params(), out=out)
    assert not res["success"] and res["highest_label"] == 0 and len(res["planes"]) == 0
    assert (out == 7.0).all()
    res = em.segment_planes((50.0, 0.0), (4.0, 4.0), _params())
    assert not res["success"] and res["size"] == (0, 0)


def test_launches_state_determinism_and_device_output(em):
    import torch
    counts = []
    for scene in SCENES:
        _set(em, _scene(scene, 1))
        before = em.get_state()
        n0 = em.launch_count()
        a = em.segment_planes((0.1, 0.1), (3.0, 3.0), _params())
        counts.append(em.launch_count() - n0)
        b = em.segment_planes((0.1, 0.1), (3.0, 3.0), _params())
        after = em.get_state()
        assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(before, after))
        for k in a["layers"]:
            assert np.array_equal(_bits(a["layers"][k]), _bits(b["layers"][k]))
        assert a["planes"].tobytes() == b["planes"].tobytes()
        rows, cols = a["size"]
        out = torch.empty(4 * rows * cols, dtype=torch.float32, device="cuda")
        d = em.segment_planes((0.1, 0.1), (3.0, 3.0), _params(), out=out)
        for k in a["layers"]:
            assert np.array_equal(_bits(d["layers"][k].cpu().numpy()), _bits(a["layers"][k]))
        assert d["planes"].cpu().numpy().tobytes() == a["planes"].tobytes()
        assert d["highest_label"] == a["highest_label"]
    assert len(set(counts)) == 1, counts


def test_device_call_captures_into_a_graph(em):
    import torch
    _set(em, _scene("stairs", 0))
    p = _params().to_c()
    req = np.array([0.0, 0.0, 3.0, 3.0], np.float64)
    ref = em.segment_planes((0.0, 0.0), (3.0, 3.0), _params())
    rows, cols = ref["size"]
    cap = int(em._L.emap_plane_capacity(rows, cols, C.byref(p)))
    out = torch.zeros(4 * rows * cols, dtype=torch.float32, device="cuda")
    planes = torch.zeros((cap, 7), dtype=torch.float64, device="cuda")
    info = torch.zeros(5, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    em.set_stream(s.cuda_stream)
    try:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            rc = em._L.emap_segment_planes(em._h, req.ctypes.data, C.byref(p), out.data_ptr(), 1, out.numel(),
                                           planes.data_ptr(), cap, info.data_ptr())
        assert rc == 0, em._L.emap_last_error(em._h)
        g.replay()
        torch.cuda.synchronize()
    finally:
        em.set_stream(None)
    inf = info.cpu().numpy()
    assert inf.tolist() == [1, rows, cols, ref["highest_label"], len(ref["planes"])]
    assert np.array_equal(_bits(out.cpu().numpy()[:rows * cols]), _bits(ref["layers"]["elevation_raw"].reshape(-1)))
    assert planes.cpu().numpy()[:len(ref["planes"])].tobytes() == ref["planes"].tobytes()


@pytest.mark.parametrize("why,kw,size", [
    ("ransac", {"include_ransac_refinement": True}, None),
    ("median even", {"median_kernel": 4}, None),
    ("median 2", {"median_kernel": 2}, None),
    ("kernel even", {"kernel_size": 4}, None),
    ("kernel small", {"kernel_size": 1}, None),
    ("connectivity", {"connectivity": 6}, None),
    ("resolution", {"resolution": 0.05}, None),
    ("out small", {}, "out"),
    ("planes small", {}, "planes"),
    ("null out", {}, "null"),
])
def test_rejections_write_nothing(em, why, kw, size):
    _set(em, _scene("stairs", 0))
    p = _params(**kw).to_c()
    req = np.array([0.0, 0.0, 2.0, 2.0], np.float64)
    rows, cols = em.get_submap((0.0, 0.0), (2.0, 2.0), ["elevation"])["size"]
    n = rows * cols
    out = np.full(4 * n - (1 if size == "out" else 0), 5.0, np.float32)
    cap = n // 4 - (1 if size == "planes" else 0)
    planes = np.full((max(cap, 1), 7), 5.0)
    info = np.full(5, 5, np.int32)
    n0 = em.launch_count()
    rc = em._L.emap_segment_planes(em._h, req.ctypes.data, C.byref(p), None if size == "null" else out.ctypes.data, 0,
                                   out.size, planes.ctypes.data, cap, info.ctypes.data)
    assert rc == EMAP_ERR_INVALID, why
    assert em.launch_count() == n0
    assert (out == 5.0).all() and (planes == 5.0).all() and (info == 5).all()
