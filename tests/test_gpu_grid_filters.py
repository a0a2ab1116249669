"""GPU: grid_map_filters_rsl's layer filters (ElevationMap.min_values, median, box_blur, gaussian_blur, dilate, erode,
outline / emap_grid_filter) against tests/filters_oracle.py and cv2 at 76^2, 1022^2 and 2047^2; every host/device
combination of grid, mask and output gives the same bytes; the filters on get_submap, get_transformed_submap and
planar_terrain layers; noiseNode's minValues-then-boxBlur chain; device calls do not synchronise with the host and
launch the kernels include/emap.h states; every rejection writes and launches nothing."""
import ctypes as C
import os
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import filters_oracle as F                                         # noqa: E402
from planar_terrain_oracle import gauss_ulps_bound, ulps           # noqa: E402
from test_gpu_inpaint_ns import _dev, _grids, _host, _map          # noqa: E402
from test_grid_filters_cpu import grids, same                      # noqa: E402

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

# (method, kwargs, oracle kwargs): one case per op and path
CASES = [
    ("min_values", {}, dict(op=F.MIN_VALUES)),
    ("median", dict(kernel_size=3), dict(op=F.MEDIAN, kernel=3)),
    ("median", dict(kernel_size=3, number_of_repeats=2), dict(op=F.MEDIAN, kernel=3, repeats=2)),
    ("median", dict(kernel_size=7), dict(op=F.MEDIAN, kernel=7)),
    ("median", dict(kernel_size=5, number_of_repeats=2), dict(op=F.MEDIAN, kernel=5, repeats=2)),
    ("box_blur", dict(kernel_size=3), dict(op=F.BOX_BLUR, kernel=3)),
    ("box_blur", dict(kernel_size=4), dict(op=F.BOX_BLUR, kernel=4)),
    ("box_blur", dict(kernel_size=9, number_of_repeats=2), dict(op=F.BOX_BLUR, kernel=9, repeats=2)),
    ("gaussian_blur", dict(kernel_size=3, sigma=0.0), dict(op=F.GAUSSIAN_BLUR, kernel=3)),
    ("gaussian_blur", dict(kernel_size=7, sigma=1.5), dict(op=F.GAUSSIAN_BLUR, kernel=7, sigma=1.5)),
    ("gaussian_blur", dict(kernel_size=0, sigma=0.9), dict(op=F.GAUSSIAN_BLUR, kernel=0, sigma=0.9)),
    ("dilate", dict(kernel_size=5), dict(op=F.DILATE, kernel=5)),
    ("erode", dict(kernel_size=3, inpaint=False), dict(op=F.ERODE, kernel=3, inpaint=False)),
    ("outline", {}, dict(op=F.OUTLINE)),
]


def _want(a, o, mask=None):
    return F.apply(img=a, mask=mask, **{k: v for k, v in o.items()})


def _check(got, want, o, a, name=""):
    got = _host(got)
    if o["op"] == F.GAUSSIAN_BLUR:
        k, sigma = o["kernel"], o.get("sigma", 0)
        ref = cv2.GaussianBlur(a, (k, k), sigma)
        if k == 3 and sigma <= 0:
            assert same(got, ref), name                # NaN and +-inf included
        elif np.isfinite(a).all():
            assert ulps(got, ref, np.abs(a).max()) <= gauss_ulps_bound(k or F.gauss_kernel_size(sigma)), name
    if o["op"] in (F.DILATE, F.ERODE):
        assert got.tobytes() == want.tobytes(), name   # the sign of a zero included
    assert same(got, want), (name, int((~((got == want) | (np.isnan(got) & np.isnan(want)))).sum()))


def _grid(h, dev=False):
    return {"layers": {"elevation": _dev(h) if dev else h}, "centre": np.zeros(2), "resolution": 0.05}


@pytest.mark.parametrize("size", [76, 1022, 2047])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_filters_equal_the_oracle(size, case):
    method, kw, o = CASES[case]
    em = _map()
    names = ["terrain", "holed", "wide"] if size > 76 else list(grids((8, 8), 0))
    for name, a in grids((size, size - 1), size + case).items():
        if name not in names:
            continue
        want = _want(a, o)
        _check(getattr(em, method)(_grid(a), **kw), want, o, a, name)
        last = o.get("kernel", 3) + (2 * (o.get("repeats", 1) - 1) if o["op"] == F.MEDIAN else 0)
        if o["op"] in (F.BOX_BLUR, F.MEDIAN) and last <= 5 and name in ("random", "terrain", "wide"):
            ref = a
            for r in range(o.get("repeats", 1)):
                k = o["kernel"] + (2 * r if o["op"] == F.MEDIAN else 0)
                ref = cv2.blur(ref, (k, k)) if o["op"] == F.BOX_BLUR else cv2.medianBlur(ref, k)
            assert same(want, ref)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_host_and_device_sides_give_the_same_bytes(case):
    method, kw, o = CASES[case]
    em = _map()
    rng = np.random.default_rng(case)
    a = grids((300, 211), case)["holed"]
    mask = (rng.random(a.shape) < 0.7).astype(np.float32) if o["op"] in (F.DILATE, F.ERODE) else None
    want = _want(a, o, mask)
    outs = []
    for g_dev in (False, True):
        for o_dev in (False, True):
            kwm = dict(kw, mask=(_dev(mask) if g_dev else mask)) if mask is not None else kw
            out = _dev(np.zeros_like(a)) if o_dev else np.zeros_like(a)
            got = getattr(em, method)(_grid(a, g_dev), out=out, **kwm)
            assert got is out
            outs.append(_host(got))
    for got in outs[1:]:
        assert got.tobytes() == outs[0].tobytes()
    _check(outs[0], want, o, a)


def test_filters_on_windows_and_terrain_layers():
    em, gs = _grids()
    for grid, layer, res in gs:
        h = _host(grid["layers"][layer]).astype(np.float32)
        for method, kw, o in CASES:
            if o["op"] == F.OUTLINE and min(h.shape) < 3 or o.get("kernel", 1) > min(h.shape):
                continue
            _check(getattr(em, method)(grid, layer, **kw), _want(h, o), o, h, (layer, method))


@pytest.mark.parametrize("method", ["dilate", "erode"])
def test_windows_without_a_finite_value_fold_as_eigen(method):
    """Windows of only NaN and +-inf: the functor's column-major fold (a NaN first cell keeps the cell, else the
    extreme infinity), and the earliest zero's sign, against the cell-by-cell transliteration."""
    em = _map()
    rng = np.random.default_rng(12)
    for k, shape in ((3, (61, 47)), (4, (40, 9)), (1, (20, 20)), (5, (5, 30))):
        a = np.full(shape, np.nan, np.float32)
        u = rng.random(shape)
        a[u < 0.2] = np.inf
        a[(u >= 0.2) & (u < 0.4)] = -np.inf
        a[u > 0.97] = 1.5
        z = rng.random(shape) < 0.1
        a[z] = np.where(rng.random(shape) < 0.5, np.float32(0.0), np.float32(-0.0))[z]
        mask = np.where(rng.random(shape) < 0.1, np.float32(0.0), np.float32(-1.0)).astype(np.float32)
        for m in (None, mask):
            for inpaint in (True, False):
                want = F.morph_literal(a, k, m, inpaint, method == "dilate")
                for dev in (False, True):
                    mm = None if m is None else (_dev(m) if dev else m)
                    got = getattr(em, method)(_grid(a, dev), kernel_size=k, mask=mm, inpaint=inpaint)
                    assert _host(got).tobytes() == want.tobytes(), (k, shape, m is None, inpaint, dev)


def test_noise_node_chain():
    """noiseNode.cpp: minValues, then boxBlur, on the device from end to end."""
    em = _map()
    a = grids((1022, 1021), 3)["holed"]
    filled = em.min_values(_grid(a, True))
    got = em.box_blur({"layers": {"elevation": filled}, "centre": np.zeros(2), "resolution": 0.05}, kernel_size=5)
    want = F.min_values(a)
    assert same(got.cpu().numpy(), cv2.blur(want, (5, 5)))


def test_device_calls_do_not_synchronise_and_launch_counts():
    import torch
    em = _map()
    a = grids((600, 500), 9)["holed"]
    g = _grid(a, True)
    mask = _dev(np.ones_like(a))
    expect = {"min_values": 5, "median": 1, "box_blur": 2, "gaussian_blur": 2, "dilate": 2, "erode": 2, "outline": 1}
    calls = [("min_values", {}), ("median", dict(kernel_size=3)), ("box_blur", dict(kernel_size=3)),
             ("gaussian_blur", dict(kernel_size=3, sigma=0.0)), ("dilate", dict(kernel_size=3, mask=mask)),
             ("erode", dict(kernel_size=3)), ("outline", {}), ("median", dict(kernel_size=9, number_of_repeats=2)),
             ("median", dict(kernel_size=1, number_of_repeats=2)), ("box_blur", dict(kernel_size=7, number_of_repeats=3))]
    counts = {"median9x2": 3 + 2, "median1x2": 1, "box7x3": 6}
    wants = [_host(getattr(em, m)(g, **kw)) for m, kw in calls]      # scratch grown: later calls do not allocate
    got = []
    for m, kw in calls:
        n0 = em.launch_count()
        getattr(em, m)(g, **kw)
        got.append(em.launch_count() - n0)
    assert got == [expect[m] for m, _ in calls[:7]] + [counts["median9x2"], counts["median1x2"], counts["box7x3"]]
    outs = [torch.zeros_like(g["layers"]["elevation"]) for _ in calls]
    torch.cuda.synchronize()
    torch.cuda._sleep(2_000_000_000)                               # about a second of GPU time queued before the calls
    t0 = time.perf_counter()
    for (m, kw), out in zip(calls, outs):
        getattr(em, m)(g, out=out, **kw)
    dt = time.perf_counter() - t0
    torch.cuda.synchronize()
    assert dt < 0.25, dt
    for w, out in zip(wants, outs):
        assert _host(out).tobytes() == w.tobytes()


_REJECT = [("null grid", {}), ("null out", {}), ("null op", {}), ("op -1", dict(op=-1)), ("op 7", dict(op=7)),
           ("kernel 0", dict(op=2, kernel_size=0)), ("kernel 64", dict(op=2, kernel_size=64)),
           ("median even", dict(op=1, kernel_size=4)), ("median odd delta", dict(op=1, kernel_size=3,
                                                                                   delta_kernel_size=1)),
           ("median float 7", dict(op=1, kernel_size=7, delta_kernel_size=-2, number_of_repeats=2)),
           ("median past max", dict(op=1, kernel_size=61, delta_kernel_size=2, number_of_repeats=3)),
           ("median repeats 0", dict(op=1, kernel_size=3, number_of_repeats=0)),
           ("box repeats -1", dict(op=2, kernel_size=3, number_of_repeats=-1)),
           ("gauss even", dict(op=3, kernel_size=4)), ("gauss sigma nan", dict(op=3, kernel_size=3, sigma=np.nan)),
           ("gauss 0 without sigma", dict(op=3, kernel_size=0, sigma=0.0)),
           ("gauss 0 sigma too wide", dict(op=3, kernel_size=0, sigma=8.0)),
           ("dilate window", dict(op=4, kernel_size=13)), ("erode window", dict(op=5, kernel_size=13)),
           ("outline 2 rows", dict(op=6)), ("bad resolution", dict(op=0))]


@pytest.mark.parametrize("why", [w for w, _ in _REJECT])
def test_rejections_write_and_launch_nothing(why):
    from elevation_mapping_cupy_b200 import _lib
    em = _map()
    kw = dict(_REJECT)[why]
    f = _lib.EmapFilterOp(kw.get("op", 2), kw.get("kernel_size", 3), kw.get("delta_kernel_size", 2),
                          kw.get("number_of_repeats", 1), kw.get("sigma", 0.0), 1)
    rows = 2 if why == "outline 2 rows" else 12
    h = np.ones((rows, 11), np.float32)
    out = np.full_like(h, 99.0)
    g = _lib.EmapGrid(h.ctypes.data, rows, 11, (C.c_double * 2)(0, 0), 0.0 if why == "bad resolution" else 0.05)
    n0 = em.launch_count()
    rc = em._L.emap_grid_filter(em._h, None if why == "null grid" else C.byref(g), 0,
                                None if why == "null op" else C.byref(f), None,
                                None if why == "null out" else out.ctypes.data, 0)
    assert rc == -1
    assert em.launch_count() == n0
    assert (out == 99.0).all()
