"""GPU: planar regions of a map window (ElevationMap.extract_planar_regions / emap_extract_planar_regions) against the
NumPy + cv2 restatement in tests/planar_regions_oracle.py, run on the call's own segmentation and plane table: region
order, polygon roles and vertex counts exactly, coordinates, transforms and bboxes within 1e-12.  Scenes: the
synthetic plane scenes, the reference's demo terrains, the LiDAR map and a 2047^2 window, with connectivity 4 and 8 and
margins 0, 1 and 2, plus a plane nested in another's hole, a scene that needs the fallback erosion and regions on the
window edge.  Also: the layers and plane table equal segment_planes' bytes, host and device output agree, two calls give
the same bytes, the map state is untouched, the launch count does not depend on the scene, a device-output call can be
captured into a CUDA graph, an overflow reports exact counts and the retry succeeds, windows below 2 x 2, without a
finite cell and outside the map, and every rejected argument writes nothing."""
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
import planar_regions_oracle as RO   # noqa: E402

W = 102
TOL = 1e-12
EMAP_ERR_INVALID = -1
_MAPS = {}


def _map(cell_n):
    if cell_n not in _MAPS:
        from elevation_mapping_cupy_b200.parameter import core_parameter
        from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
        _MAPS.clear()
        _MAPS[cell_n] = ElevationMap(core_parameter(cell_n))
    return _MAPS[cell_n]


@pytest.fixture
def em():
    return _map(W)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _params(**kw):
    return S.params(**kw)


def _compare(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a["label"] == b["label"]
        assert np.abs(a["transform"] - b["transform"]).max() <= TOL
        assert np.abs(a["bbox"] - b["bbox"]).max() <= TOL
        assert len(a["boundary"]["holes"]) == len(b["boundary"]["holes"])
        assert len(a["insets"]) == len(b["insets"])
        pa = [a["boundary"]["outer"]] + a["boundary"]["holes"]
        pb = [b["boundary"]["outer"]] + b["boundary"]["holes"]
        for ia, ib in zip(a["insets"], b["insets"]):
            assert len(ia["holes"]) == len(ib["holes"])
            pa += [ia["outer"]] + ia["holes"]
            pb += [ib["outer"]] + ib["holes"]
        assert [len(p) for p in pa] == [len(p) for p in pb]
        for p, q in zip(pa, pb):
            assert np.abs(p - q).max(initial=0.0) <= TOL


def _check(em, pos, ln, p):
    """The call against segment_planes and the oracle; returns the call's result and the oracle's regions."""
    res = em.extract_planar_regions(pos, ln, p)
    seg = em.segment_planes(pos, ln, p)
    assert res["success"] == seg["success"] and res["complete"]
    for k in seg["layers"]:
        assert np.array_equal(_bits(res["layers"][k]), _bits(seg["layers"][k]))
    assert res["planes"].tobytes() == seg["planes"].tobytes()
    assert res["highest_label"] == seg["highest_label"]
    if not res["success"]:
        return res, []
    want = RO.extract(res["layers"]["segmentation"], res["planes"], res["origin"], res["resolution"], p.margin_size,
                      p.extracted_planes_height_offset)
    _compare(res["regions"], want)
    return res, want


SCENES = ["ramps", "stairs", "holes", "diagonal", "rough"]
WINDOWS = [("whole", (0.0, 0.0), (4.0, 4.0)), ("node", (0.3, -0.2), (3.0, 3.0)), ("clipped", (1.7, 1.5), (1.5, 1.0))]


@pytest.mark.parametrize("margin", [0, 1, 2, 4])
@pytest.mark.parametrize("conn", [4, 8])
@pytest.mark.parametrize("scene", SCENES)
def test_scene_matches_oracle(em, scene, conn, margin):
    S.set_image(em, S.synthetic(scene, W - 2, SCENES.index(scene)))
    p = _params(connectivity=conn, margin_size=margin, extracted_planes_height_offset=0.03 * margin)
    total = 0
    for _, pos, ln in WINDOWS:
        _, want = _check(em, pos, ln, p)
        total += len(want)
    assert total > 0


def _golden_map(name):
    if name == "lidar":
        _MAPS.pop(S.LIDAR_W, None)
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


@pytest.mark.parametrize("conn", [4, 8])
@pytest.mark.parametrize("name", list(S.TERRAINS) + ["lidar", "big"])
def test_golden_scene(name, conn):
    em, pos, ln = _golden_map(name)
    for margin in ([1] if name == "big" else [0, 1, 2]):
        _, want = _check(em, pos, ln, _params(connectivity=conn, margin_size=margin))
        assert len(want) > 0


def _nested():
    """A floor with a square moat of rough cells holding a raised plate that holds a rough pit with a floor-level
    plate: planes nested in the holes of other planes."""
    n = W - 2
    rng = np.random.default_rng(3)
    z = np.zeros((n, n), np.float32)
    z[20:80, 20:80] = 0.3 * rng.standard_normal((60, 60))
    z[26:74, 26:74] = 0.2
    z[38:62, 38:62] = 0.3 * rng.standard_normal((24, 24))
    z[44:56, 44:56] = 0.0
    return z


def test_nested_planes(em):
    S.set_image(em, _nested())
    for conn in (4, 8):
        res, want = _check(em, (0.0, 0.0), (4.0, 4.0), _params(connectivity=conn))
        labels = [r["label"] for r in want]
        holed = [r for r in want if r["boundary"]["holes"]]
        assert len(set(labels)) >= 3 and len(holed) >= 2


def test_fallback(em):
    """Planar strips two cells wide: a margin of 2 erodes them away, so each strip's region comes from the cross
    erosion."""
    n = W - 2
    rng = np.random.default_rng(9)
    z = (0.3 * rng.standard_normal((n, n))).astype(np.float32)
    for k in range(5):
        z[10 + 16 * k:12 + 16 * k, 8:90] = 0.1 * k
    S.set_image(em, z)
    p = _params(margin_size=2)
    res, want = _check(em, (0.0, 0.0), (4.0, 4.0), p)
    strict = RO.extract(res["layers"]["segmentation"], res["planes"], res["origin"], res["resolution"], 2)
    assert len(want) >= 5
    # without the fallback (an oracle that stops after the margin erosion) the strips have no region
    lab = res["layers"]["segmentation"]
    up = RO.upsample(lab)
    k = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (7, 7))
    empty = [r["label"] for r in strict
             if not RO.boundary_and_inset(cv2.erode((up == r["label"]).astype(np.uint8), k,
                                                    borderType=cv2.BORDER_REPLICATE))]
    assert len(empty) >= 5


def test_regions_on_the_window_edge(em):
    S.set_image(em, np.zeros((W - 2, W - 2), np.float32))
    res, want = _check(em, (0.0, 0.0), (4.0, 4.0), _params(margin_size=0))
    assert len(want) == 1
    rows, cols = res["size"]
    # one plane over the whole window: the boundary is the upsampled image's frame after the erosion
    assert len(want[0]["boundary"]["outer"]) == 4 and len(want[0]["insets"]) == 1


@pytest.mark.parametrize("name", ["lidar", "big"])
def test_host_device_determinism_state_and_retry(name):
    import torch
    em, pos, ln = _golden_map(name)
    p = _params()
    before = em.get_state()
    a = em.extract_planar_regions(pos, ln, p)
    b = em.extract_planar_regions(pos, ln, p)
    after = em.get_state()
    assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(before, after))
    for k in ("regions", "polygons", "vertices"):
        assert a["tables"][k].tobytes() == b["tables"][k].tobytes()
        assert len(a["tables"][k]) > 0
    rows, cols = a["size"]
    out = torch.empty(4 * rows * cols, dtype=torch.float32, device="cuda")
    d = em.extract_planar_regions(pos, ln, p, out=out)
    assert d["complete"] and d["regions"] is None
    for k in ("regions", "polygons", "vertices"):
        assert d["tables"][k].cpu().numpy().tobytes() == a["tables"][k].tobytes()
    for k in a["layers"]:
        assert np.array_equal(_bits(d["layers"][k].cpu().numpy()), _bits(a["layers"][k]))


def _raw_call(em, pos, ln, p, caps, out_is_device=False, fill=5):
    pc, rp = p.to_c(), p.regions_to_c()
    req = np.array(list(pos) + list(ln), np.float64)
    rows, cols = em.get_submap(pos, ln, ["elevation"])["size"]
    n = rows * cols
    cap = max(int(em._L.emap_plane_capacity(rows, cols, C.byref(pc))), 1)
    out = np.full(max(4 * n, 1), fill, np.float32)
    planes = np.full((cap, 7), fill, np.float64)
    tabs = (np.full((max(caps[0], 1), 17), fill, np.float64), np.full((max(caps[1], 1), 5), fill, np.int32),
            np.full((max(caps[2], 1), 2), fill, np.float64))
    info = np.full(9, fill, np.int32)
    return pc, rp, req, out, planes, cap, tabs, info


def test_overflow_reports_counts_and_retry_succeeds(em):
    S.set_image(em, S.synthetic("stairs", W - 2, 0))
    p = _params()
    full = em.extract_planar_regions((0.0, 0.0), (4.0, 4.0), p)
    nr, npoly, nv = (len(full["tables"][k]) for k in ("regions", "polygons", "vertices"))
    assert nr > 1
    for caps in ((nr - 1, npoly, nv), (nr, npoly - 1, nv), (nr, npoly, nv - 1), (nr, npoly, nv)):
        pc, rp, req, out, planes, cap, tabs, info = _raw_call(em, (0.0, 0.0), (4.0, 4.0), p, caps)
        from elevation_mapping_cupy_b200 import _lib
        o = _lib.EmapRegionOut(tabs[0].ctypes.data, caps[0], tabs[1].ctypes.data, caps[1], tabs[2].ctypes.data, caps[2])
        rc = em._L.emap_extract_planar_regions(em._h, req.ctypes.data, C.byref(pc), C.byref(rp), out.ctypes.data, 0,
                                               out.size, planes.ctypes.data, cap, C.byref(o), info.ctypes.data)
        assert rc == 0
        assert info[5:8].tolist() == [nr, npoly, nv]
        if caps == (nr, npoly, nv):
            assert info[8] == 1
            assert tabs[0].tobytes() == full["tables"]["regions"].tobytes()
            assert tabs[1].tobytes() == full["tables"]["polygons"].tobytes()
            assert tabs[2].tobytes() == full["tables"]["vertices"].tobytes()
        else:
            assert info[8] == 0
            assert (tabs[0] == 5).all() and (tabs[1] == 5).all() and (tabs[2] == 5).all()
    again = em.extract_planar_regions((0.0, 0.0), (4.0, 4.0), p, capacities=(1, 1, 1))
    assert again["retried"] and again["complete"]
    assert not em.extract_planar_regions((0.0, 0.0), (4.0, 4.0), p)["retried"]
    for k in ("regions", "polygons", "vertices"):
        assert again["tables"][k].tobytes() == full["tables"][k].tobytes()


def test_small_empty_and_outside_windows(em):
    S.set_image(em, np.zeros((W - 2, W - 2), np.float32))
    thin = [s for s in (0.0, 0.01, 0.02, 0.03, 0.04) if em.get_submap((0.0, 0.0), (s, 4.0), ["elevation"])["size"][0] == 1]
    assert thin
    for ln in ((thin[0], 4.0), (4.0, thin[0])):
        res = em.extract_planar_regions((0.0, 0.0), ln, _params())
        assert res["success"] and min(res["size"]) == 1 and res["complete"] and res["regions"] == []
        assert res["planes"].tobytes() == em.segment_planes((0.0, 0.0), ln, _params())["planes"].tobytes()
    S.set_image(em, S.synthetic("empty", W - 2, 0))
    res = em.extract_planar_regions((0.0, 0.0), (4.0, 4.0), _params())
    assert not res["success"] and res["complete"] and res["regions"] == []
    res = em.extract_planar_regions((50.0, 0.0), (4.0, 4.0), _params())
    assert not res["success"] and res["size"] == (0, 0) and res["complete"] and res["regions"] == []


def test_launch_count_does_not_depend_on_the_scene(em):
    counts = []
    for scene in SCENES + ["empty"]:
        S.set_image(em, S.synthetic(scene, W - 2, 1))
        n0 = em.launch_count()
        em.extract_planar_regions((0.1, 0.1), (3.0, 3.0), _params())
        counts.append(em.launch_count() - n0)
    assert len(set(counts)) == 1, counts


def test_device_call_captures_into_a_graph(em):
    import torch
    from elevation_mapping_cupy_b200 import _lib
    S.set_image(em, S.synthetic("stairs", W - 2, 0))
    p = _params()
    ref = em.extract_planar_regions((0.0, 0.0), (3.0, 3.0), p)
    rows, cols = ref["size"]
    pc, rp = p.to_c(), p.regions_to_c()
    req = np.array([0.0, 0.0, 3.0, 3.0], np.float64)
    cap = int(em._L.emap_plane_capacity(rows, cols, C.byref(pc)))
    caps = [len(ref["tables"][k]) for k in ("regions", "polygons", "vertices")]
    out = torch.zeros(4 * rows * cols, dtype=torch.float32, device="cuda")
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
            rc = em._L.emap_extract_planar_regions(em._h, req.ctypes.data, C.byref(pc), C.byref(rp), out.data_ptr(), 1,
                                                   out.numel(), planes.data_ptr(), cap, C.byref(o), info.data_ptr())
        assert rc == 0, em._L.emap_last_error(em._h)
        g.replay()
        torch.cuda.synchronize()
    finally:
        em.set_stream(None)
    assert info.cpu().numpy().tolist() == [1, rows, cols, ref["highest_label"], len(ref["planes"])] + caps + [1]
    for t, k in zip(tabs, ("regions", "polygons", "vertices")):
        assert t.cpu().numpy().tobytes() == ref["tables"][k].tobytes()


@pytest.mark.parametrize("why", ["margin", "margin negative", "offset", "negative capacity", "huge capacity",
                                 "null table", "null out", "ransac", "planes small"])
def test_rejections_write_nothing(em, why):
    from elevation_mapping_cupy_b200 import _lib
    S.set_image(em, S.synthetic("stairs", W - 2, 0))
    kw = {"margin": {"margin_size": 5}, "margin negative": {"margin_size": -1},
          "offset": {"extracted_planes_height_offset": float("nan")},
          "ransac": {"include_ransac_refinement": True}}.get(why, {})
    p = _params(**kw)
    caps = (16, 64, 1024)
    pc, rp, req, out, planes, cap, tabs, info = _raw_call(em, (0.0, 0.0), (2.0, 2.0), p, caps)
    o = _lib.EmapRegionOut(None if why == "null table" else tabs[0].ctypes.data, caps[0], tabs[1].ctypes.data,
                           -1 if why == "negative capacity" else caps[1], tabs[2].ctypes.data,
                           2 ** 61 if why == "huge capacity" else caps[2])
    n0 = em.launch_count()
    rc = em._L.emap_extract_planar_regions(em._h, req.ctypes.data, C.byref(pc), C.byref(rp),
                                           None if why == "null out" else out.ctypes.data, 0, out.size,
                                           planes.ctypes.data, cap - (1 if why == "planes small" else 0), C.byref(o),
                                           info.ctypes.data)
    assert rc == EMAP_ERR_INVALID, why
    assert em.launch_count() == n0
    assert (out == 5).all() and (planes == 5).all() and (info == 5).all()
    assert all((t == 5).all() for t in tabs)
    msg = em._L.emap_last_error(em._h)
    assert (msg.decode() if isinstance(msg, bytes) else str(msg)).startswith("emap_extract_planar_regions:")
