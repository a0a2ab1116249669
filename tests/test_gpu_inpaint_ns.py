"""GPU: cv2.inpaint for one 8-bit channel (ElevationMap.inpaint_image / emap_inpaint_image) and grid_map_filters_rsl's
nonlinearInterpolation (ElevationMap.nonlinear_interpolation / emap_nonlinear_interpolation).  Navier-Stokes against
cv2 bit for bit on the reference plugin test's 202^2 states, config D's 2048^2 map, rectangular images up to 2047 on a
side, border-touching holes and no-hole / all-hole images; Telea against cv2 and against emap_inpaint on the same
planes; the grid call on get_submap, get_transformed_submap and planar_terrain grids against the NumPy restatement plus
cv2; host and device sides give the same bytes, device calls do not synchronise with the host, the launch counts, and
every rejection writes and launches nothing."""
import ctypes as C
import os
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ns_inpaint_oracle as O                                     # noqa: E402
import plane_scenes as S                                          # noqa: E402

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

_MAPS = {}


def _map(cell_n=S.LIDAR_W):
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


def _ns(img, mask):
    return cv2.inpaint(img, mask, 1, cv2.INPAINT_NS)


def _check_ns(em, img, mask):
    """NS on host and device inputs equals cv2; returns the device result."""
    want = _ns(img, mask)
    got_h = em.inpaint_image(img, mask)
    got_d = em.inpaint_image(_dev(img), _dev(mask))
    assert isinstance(got_h, np.ndarray) and got_d.is_cuda
    assert np.array_equal(got_h, want), (img.shape, int((got_h != want).sum()))
    assert np.array_equal(_host(got_d), want)
    return got_d


def _telea_replay(img, mask):
    from test_inpaint_cpu import _host_lib, _run_host
    return _run_host(_host_lib(), np.ascontiguousarray(img), np.ascontiguousarray(mask))[0]


def _plugin_planes(h, is_valid):
    """plugins/inpainting.py's 8-bit planes (as oracle.inpaint_cv2 builds them)."""
    mask = (is_valid < 0.5).astype(np.uint8)
    hv = h[mask < 1]
    h_max, h_min = float(hv.max()), float(hv.min())
    q = (h.astype(np.float32) - np.float32(h_min)) * np.float32(255) / np.float32(h_max - h_min)
    return np.clip(np.nan_to_num(np.trunc(q), nan=0.0), 0, 255).astype(np.uint8), mask, h_min, h_max


def test_plugin_test_states_ns_and_telea():
    """The 202^2 randn states of test_gpu_plugins.py's three seeds: NS against cv2; Telea against cv2 and, de-normalised,
    against the inpainting plugin's output (emap_inpaint) on the same planes."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.plugins.inpainting import Inpainting
    em = ElevationMap(core_parameter(202))
    for seed, valid_frac in ((11, 0.31), (12, 0.7), (13, 0.02)):
        rng = np.random.default_rng(seed)
        st = np.zeros((7, 202, 202), np.float32)
        st[0] = rng.standard_normal((202, 202)).astype(np.float32)
        st[1] = 0.05
        st[2] = (rng.random((202, 202)) < valid_frac).astype(np.float32)
        st[3] = 1.0
        st[5] = st[0]
        img, mask, h_min, h_max = _plugin_planes(st[0], st[2])
        _check_ns(em, img, mask)
        tel = em.inpaint_image(img, mask, method="telea")
        assert np.array_equal(tel, cv2.inpaint(img, mask, 1, cv2.INPAINT_TELEA)), seed
        em.set_state(st)
        plug = Inpainting(cell_n=202, method="telea", engine=em)(em.elevation_map, em.layer_names, None, []).cpu().numpy()
        assert np.array_equal(plug, tel.astype(np.float32) * (h_max - h_min) / 255 + h_min), seed


def test_config_d_map():
    """BASELINE config D: the 2048^2 map after a dense depth-camera frame, 98 % holes."""
    from elevation_mapping_cupy_b200 import workloads as wl
    em = _map(2048)
    pts, R, t = wl.depth_camera_cloud(3, 0)
    em.move_to(t, R)
    em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.0, 0.0)
    st, _ = em.get_state()
    img, mask, _, _ = _plugin_planes(st[0], st[2])
    assert mask.mean() > 0.9
    got = _check_ns(em, img, mask)
    assert np.array_equal(_host(em.inpaint_image(got.new_tensor(img), got.new_tensor(mask), method="telea")),
                          cv2.inpaint(img, mask, 1, cv2.INPAINT_TELEA))


@pytest.mark.parametrize("shape", [(2047, 1311), (1500, 2047), (5, 2047), (2047, 2), (63, 64), (1, 2047), (2047, 1)])
def test_rectangular_images(shape):
    from test_inpaint_cpu import _terrain_case
    rng = np.random.default_rng(shape[0] + shape[1])
    em = _map()
    if min(shape) > 100:                                          # terrain with a deep hole and dropouts
        t_img, t_mask = _terrain_case(max(shape), rng)
        img, mask = (np.ascontiguousarray(a[:shape[0], :shape[1]]) for a in (t_img, t_mask))
    elif min(shape) == 1:                                         # holes reaching one end (see below)
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        mask = np.zeros(shape, np.uint8)
        mask.reshape(-1)[700:] = 1
        _check_ns(em, img, mask)
        return
    else:
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        mask = (rng.random(shape) < 0.6).astype(np.uint8)
    _check_ns(em, img, mask)
    # Telea is the replay emap_inpaint runs (tests/native/inpaint_host.cpp replays it on the CPU).  On the 2047 x 1311
    # crop the front is mirror-symmetric about its middle column, where popper chains tie beyond IP_CMP_DEPTH levels: the
    # replay (the host one as well) then orders some events by pixel index and differs from cv2 along that column.
    tel = em.inpaint_image(img, mask, method="telea")
    assert np.array_equal(tel, _telea_replay(img, mask))
    if shape != (2047, 1311):
        assert np.array_equal(tel, cv2.inpaint(img, mask, 1, cv2.INPAINT_TELEA))


def test_border_holes_and_degenerate_masks():
    em = _map()
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (57, 83), dtype=np.uint8)
    for sl in (np.s_[:2, :], np.s_[-2:, :], np.s_[:, :2], np.s_[:, -2:], np.s_[:4, :4], np.s_[-4:, -4:]):
        mask = np.zeros_like(img)
        mask[sl] = rng.random(mask[sl].shape) < 0.8
        _check_ns(em, img, mask)
    for frac in (0.05, 0.5, 0.95, 0.999):
        _check_ns(em, img, ((rng.random(img.shape) < frac) * 255).astype(np.uint8))
    for mask in (np.zeros_like(img), np.ones_like(img)):          # no hole; nothing known: both unchanged
        assert np.array_equal(_check_ns(em, img, mask).cpu().numpy(), img)
        assert np.array_equal(em.inpaint_image(img, mask, method="telea"), img)


def test_one_row_and_one_column_images():
    """cv2 reads outside a one-row image; where its result is defined (holes reaching one end) the device equals it,
    and everywhere the restatement that clamps those reads."""
    em = _map()
    rng = np.random.default_rng(5)
    for n in (1, 2, 7, 2047):
        img = rng.integers(0, 256, (1, n), dtype=np.uint8)
        mask = np.zeros_like(img)
        mask[:, n // 2:] = 1
        for a, m in ((img, mask), (img.T.copy(), mask.T.copy())):
            _check_ns(em, a, m)
        m = (rng.random((1, n)) < 0.5).astype(np.uint8)
        for a, mm in ((img, m), (img.T.copy(), m.T.copy())):
            want = O.ns_inpaint(a, mm) if n < 300 else None
            got = em.inpaint_image(a, mm)
            assert np.array_equal(_host(em.inpaint_image(_dev(a), _dev(mm))), got)
            if want is not None:
                assert np.array_equal(got, want)


def _grids():
    import torch
    em = _map()
    S.lidar_frames(em)
    sub = em.get_submap(S.lidar_window(em.center), (5.0, 4.0), ["elevation"])
    yaw = 0.3
    T = np.eye(4)
    T[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
    T[:3, 3] = [0.2, -0.1, 0.05]
    sub_res = float(sub.get("resolution", em.resolution))
    # a yawed window of the terrain with holes (the LiDAR map's rings are too sparse for a small window)
    _, hscale, _, _ = S.TERRAINS["holes"]
    himg = S.terrain_image(np.load(S.GOLDEN)["grey__holes"], hscale, seed=5)
    em1 = _map(himg.shape[0] + 2)
    S.set_image(em1, himg)
    tsub = em1.get_transformed_submap((0.1, -0.05), (1.5, 1.5), ["elevation"], T)
    tsub_res = float(tsub.get("resolution", em1.resolution))
    png, scale, pos, ln = S.TERRAINS["terrain"]
    timg = S.terrain_image(np.load(S.GOLDEN)["grey__terrain"], scale)
    em2 = _map(timg.shape[0] + 2)
    S.set_image(em2, timg)
    terr = em2.planar_terrain(pos, ln, S.params(), out=torch.zeros(10 * timg.shape[0] ** 2, dtype=torch.float32,
                                                                   device="cuda"))
    return em2, [(sub, "elevation", sub_res), (tsub, "elevation", tsub_res),
                 (terr, "elevationWithNaN", float(terr.get("resolution", em2.resolution)))]


def test_nonlinear_interpolation_grids():
    em, grids = _grids()
    for grid, layer, res in grids:
        h = _host(grid["layers"][layer]).astype(np.float32)
        assert np.isnan(h).any() and np.isfinite(h).any(), layer
        want = O.nonlinear_interpolation(h, res, res, lambda img, m, r: cv2.inpaint(img, m, r, cv2.INPAINT_NS))
        centre = grid["centre"] if "centre" in grid else grid["frame_centre"]     # get_transformed_submap's frame
        hg = {"layers": {layer: h}, "centre": centre, "resolution": res}
        dg = dict(hg, layers={layer: _dev(h)})
        outs = [em.nonlinear_interpolation(hg, layer), em.nonlinear_interpolation(dg, layer),
                em.nonlinear_interpolation(hg, layer, res, out=_dev(np.zeros_like(h))),
                em.nonlinear_interpolation(dg, layer, res, out=np.zeros_like(h))]
        assert [hasattr(o, "is_cuda") for o in outs] == [False, True, True, False]
        for o in outs:
            o = _host(o)
            assert o.view(np.uint32).tobytes() == want.view(np.uint32).tobytes(), layer
            keep = ~np.isnan(h)
            assert np.array_equal(o[keep].view(np.uint32), h[keep].view(np.uint32))
            assert not np.isnan(o).any()


def test_nonlinear_interpolation_edge_cases():
    em = _map()
    h = np.ones((10, 20), np.float32)                             # TestFilters.cpp:26
    h[:3, :3] = np.nan
    h[5:7, :] = np.nan
    g = {"layers": {"elevation": h}, "centre": np.zeros(2), "resolution": 0.1}
    assert np.array_equal(em.nonlinear_interpolation(g, "elevation", 0.1), np.ones_like(h))
    rng = np.random.default_rng(6)
    cases = [np.full((7, 9), np.nan, np.float32),                  # nothing finite: unchanged
             np.where(rng.random((8, 8)) < 0.5, np.nan, -2.5).astype(np.float32),   # lo == hi
             (rng.standard_normal((30, 41)) * 3).astype(np.float32)]
    cases[1][0, 0] = -2.5
    c = cases[2]
    c[rng.random(c.shape) < 0.4] = np.nan
    c[3, 4], c[10, 11], c[0, 0] = np.inf, -np.inf, np.inf          # not masked, copied, quantised to 255 / 0
    for h in cases:
        g = {"layers": {"elevation": h}, "centre": np.zeros(2), "resolution": 0.05}
        want = O.nonlinear_interpolation(h, 0.05, 0.05, lambda img, m, r: cv2.inpaint(img, m, r, cv2.INPAINT_NS))
        for got in (em.nonlinear_interpolation(g, "elevation"),
                    em.nonlinear_interpolation(dict(g, layers={"elevation": _dev(h)}), "elevation")):
            assert _host(got).view(np.uint32).tobytes() == want.view(np.uint32).tobytes()


def test_device_calls_do_not_synchronise_and_launch_counts():
    import torch
    em = _map()
    rng = np.random.default_rng(7)
    img = _dev(rng.integers(0, 256, (300, 200), dtype=np.uint8))
    mask = _dev((rng.random((300, 200)) < 0.5).astype(np.uint8))
    h = rng.standard_normal((300, 200)).astype(np.float32)
    h[rng.random(h.shape) < 0.5] = np.nan
    g = {"layers": {"elevation": _dev(h)}, "centre": np.zeros(2), "resolution": 0.05}
    want_i = _host(em.inpaint_image(img, mask))                    # scratch grown: later calls do not allocate
    want_g = _host(em.nonlinear_interpolation(g, "elevation"))
    n0 = em.launch_count()
    em.inpaint_image(img, mask)
    n1 = em.launch_count()
    em.nonlinear_interpolation(g, "elevation")
    assert (n1 - n0, em.launch_count() - n1) == (4, 6)
    out_i, out_g = torch.zeros_like(img), torch.zeros_like(g["layers"]["elevation"])
    torch.cuda.synchronize()
    torch.cuda._sleep(2_000_000_000)                               # about a second of GPU time queued before the calls
    t0 = time.perf_counter()
    em.inpaint_image(img, mask, out=out_i)
    em.nonlinear_interpolation(g, "elevation", out=out_g)
    dt = time.perf_counter() - t0
    torch.cuda.synchronize()
    assert dt < 0.25, dt
    assert np.array_equal(_host(out_i), want_i)
    assert _host(out_g).view(np.uint32).tobytes() == want_g.view(np.uint32).tobytes()


_REJECT = ["null img", "null mask", "null out", "rows 0", "cols 0", "telea 1 row", "rows max", "method 2",
           "method -1", "radius 2", "radius 1.5", "radius nan", "radius inf",
           "g null grid", "g null data", "g null out", "g rows 0", "g bad resolution", "g nan position", "g rows max",
           "g radius 2 px", "g radius nan"]


@pytest.mark.parametrize("why", _REJECT)
def test_rejections_write_and_launch_nothing(why):
    from elevation_mapping_cupy_b200 import _lib
    em = _map()
    L = em._L
    rows, cols = 12, 17
    img = np.full((rows, cols), 7, np.uint8)
    mask = np.zeros((rows, cols), np.uint8)
    mask[3:6, 4:9] = 1
    out = np.full((rows, cols), 99, np.uint8)
    n0 = em.launch_count()
    if not why.startswith("g "):
        ip, mp, op = img.ctypes.data, mask.ctypes.data, out.ctypes.data
        r, c, radius, method = rows, cols, 1.0, 1
        big = np.zeros(0, np.uint8)
        if why == "null img":
            ip = None
        elif why == "null mask":
            mp = None
        elif why == "null out":
            op = None
        elif why == "rows 0":
            r = 0
        elif why == "cols 0":
            c = 0
        elif why == "telea 1 row":
            r, method = 1, 0
        elif why == "rows max":
            big = np.zeros((8193, 1), np.uint8)
            ip = mp = big.ctypes.data
            r, c = 8193, 1
        elif why == "method 2":
            method = 2
        elif why == "method -1":
            method = -1
        else:
            radius = {"radius 2": 2.0, "radius 1.5": 1.5, "radius nan": float("nan"), "radius inf": float("inf")}[why]
        assert L.emap_inpaint_image(em._h, ip, mp, r, c, radius, method, op, 0) == -1
        assert (out == 99).all()
        if why == "method 2":
            with pytest.raises(ValueError):
                em.inpaint_image(img, mask, method="bogus")
        elif why in ("radius 2", "rows 0"):
            with pytest.raises(_lib.EmapError):
                em.inpaint_image(img if why != "rows 0" else img[:0], mask if why != "rows 0" else mask[:0],
                                 radius=2.0 if why == "radius 2" else 1, method="ns")

    else:
        h = np.full((rows, cols), 1.0, np.float32)
        h[2:5, 3:7] = np.nan
        fout = np.full((rows, cols), 5.0, np.float32)
        res, pos, data, fptr, radius, gr, gc = 0.05, [0.0, 0.0], h.ctypes.data, fout.ctypes.data, 0.05, rows, cols
        big = np.zeros(0, np.float32)
        null_grid = False
        w = why[2:]
        if w == "null grid":
            null_grid = True
        elif w == "null data":
            data = None
        elif w == "null out":
            fptr = None
        elif w == "rows 0":
            gr = 0
        elif w == "bad resolution":
            res = -1.0
        elif w == "nan position":
            pos = [float("nan"), 0.0]
        elif w == "rows max":
            big = np.zeros((8193, 1), np.float32)
            data, gr, gc = big.ctypes.data, 8193, 1
        elif w == "radius 2 px":
            radius = 0.1
        elif w == "radius nan":
            radius = float("nan")
        g = _lib.EmapGrid(data, gr, gc, (C.c_double * 2)(*pos), res)
        assert L.emap_nonlinear_interpolation(em._h, None if null_grid else C.byref(g), 0, radius, fptr, 0) == -1
        assert (fout == 5.0).all()
        if w == "radius 2 px":
            with pytest.raises(_lib.EmapError):
                em.nonlinear_interpolation({"layers": {"e": h}, "centre": np.zeros(2), "resolution": res}, "e", 0.1)
    assert em.launch_count() == n0
