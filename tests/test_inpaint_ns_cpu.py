"""Navier-Stokes inpainting and grid_map_filters_rsl's nonlinearInterpolation without a GPU: the sequential restatement
of cv2.inpaint(INPAINT_NS) (tests/ns_inpaint_oracle.py) and the parallel round replay with the device's NS estimate
(csrc/emap_inpaint.cuh, run on the CPU by tests/native/inpaint_ns_host.cpp) are pinned against the cv2 binary bit for
bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from ns_inpaint_oracle import cv_radius, fma_f32, nonlinear_interpolation, ns_inpaint, to_image_u8  # noqa: E402
from test_inpaint_cpu import _terrain_case  # noqa: E402


def _host_lib():
    src = os.path.join(ROOT, "tests", "native", "inpaint_ns_host.cpp")
    out_dir = os.path.join(ROOT, "tests", "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libinpaint_ns_host.so")
    hdr = os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc", "emap_inpaint.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src], check=True)
    return C.CDLL(so)


def _run_host(L, img, mask, cap=4096):
    img, mask = np.ascontiguousarray(img, np.uint8), np.ascontiguousarray(mask, np.uint8)
    H, W = img.shape
    out = np.zeros_like(img)
    r, mj, nc = C.c_int(), C.c_int(), C.c_int()
    L.inpaint_ns_host(img.ctypes.data_as(C.c_void_p), mask.ctypes.data_as(C.c_void_p), H, W,
                      out.ctypes.data_as(C.c_void_p), cap, C.byref(r), C.byref(mj), C.byref(nc))
    assert nc.value == 0
    return out, r.value


def _ns(img, mask, r=1):
    return cv2.inpaint(img, mask, r, cv2.INPAINT_NS)


def _random_cases(rng, n, lo=2, hi=40):
    for _ in range(n):
        H, W = (int(v) for v in rng.integers(lo, hi, 2))
        img = rng.integers(0, 256, (H, W), dtype=np.uint8)
        mask = (rng.random((H, W)) < rng.choice([0.1, 0.4, 0.7, 0.95, 0.999])).astype(np.uint8)
        yield img, mask


def test_restatement_equals_cv2():
    rng = np.random.default_rng(11)
    for img, mask in _random_cases(rng, 12):                       # random, rectangular, border-touching
        assert np.array_equal(ns_inpaint(img, mask), _ns(img, mask)), (img.shape, mask.mean())
    img, mask = _terrain_case(48, rng)                             # smooth data
    assert np.array_equal(ns_inpaint(img, mask), _ns(img, mask))
    for H, W in ((2, 31), (31, 2), (3, 17)):                       # narrow images
        img = rng.integers(0, 256, (H, W), dtype=np.uint8)
        mask = (rng.random((H, W)) < 0.5).astype(np.uint8)
        assert np.array_equal(ns_inpaint(img, mask), _ns(img, mask)), (H, W)
    # holes along each border only: the reference's shifted indices next to the border
    img = rng.integers(0, 256, (19, 23), dtype=np.uint8)
    for sl in (np.s_[:2, :], np.s_[-2:, :], np.s_[:, :2], np.s_[:, -2:], np.s_[:3, :3], np.s_[-3:, -3:]):
        mask = np.zeros_like(img)
        mask[sl] = (rng.random(mask[sl].shape) < 0.7)
        assert np.array_equal(ns_inpaint(img, mask), _ns(img, mask))
    # no hole, all holes (nothing known: unchanged), a mask of 255s
    assert np.array_equal(ns_inpaint(img, np.zeros_like(img)), img)
    assert np.array_equal(_ns(img, np.ones_like(img)), img) and np.array_equal(ns_inpaint(img, np.ones_like(img)), img)
    mask = ((rng.random(img.shape) < 0.5) * 255).astype(np.uint8)
    assert np.array_equal(ns_inpaint(img, mask), _ns(img, mask))


def test_restatement_radius_rounding_and_wider_radii():
    """cv::inpaint rounds the radius half to even and raises it to 1; the restatement also holds at radii 2 and 3 (the
    device provides radius 1 only)."""
    rng = np.random.default_rng(12)
    img = rng.integers(0, 256, (21, 26), dtype=np.uint8)
    mask = (rng.random(img.shape) < 0.5).astype(np.uint8)
    assert [cv_radius(r) for r in (0, 0.2, 0.5, 1.4, 1.5, 2.5, 3.5, -2)] == [1, 1, 1, 1, 2, 2, 4, 1]
    for r in (0, 0.2, 0.5, 1.4):
        assert np.array_equal(_ns(img, mask, r), _ns(img, mask, 1))
    assert np.array_equal(_ns(img, mask, 2.5), _ns(img, mask, 2))
    for r in (2, 3):
        for img, mask in _random_cases(rng, 3, 5, 30):
            assert np.array_equal(ns_inpaint(img, mask, r), _ns(img, mask, r)), r


def test_one_row_and_one_column_images():
    """On a 1 x N (N x 1) image the reference reads outside the image next to its border, so its result is only
    defined where the weights do not matter: a run of holes reaching one end is filled from its single known
    neighbour.  There the restatement (which clamps those reads) equals cv2; everywhere it equals the host replay."""
    rng = np.random.default_rng(13)
    L = _host_lib()
    for n in (1, 2, 5, 40):
        for t in range(4):
            img = rng.integers(0, 256, (1, n), dtype=np.uint8)
            k = int(rng.integers(0, n))
            mask = np.zeros_like(img)
            if t % 2:
                mask[:, :k] = 1
            else:
                mask[:, n - k:] = 1
            for a, m in ((img, mask), (img.T.copy(), mask.T.copy())):
                assert np.array_equal(ns_inpaint(a, m), _ns(a, m)), (n, t)
            m = (rng.random((1, n)) < 0.5).astype(np.uint8)
            for a, mm in ((img, m), (img.T.copy(), m.T.copy())):
                assert np.array_equal(_run_host(L, a, mm)[0], ns_inpaint(a, mm))


def test_host_replay_equals_restatement_and_cv2():
    L = _host_lib()
    rng = np.random.default_rng(14)
    for img, mask in _random_cases(rng, 25, 1, 60):
        want = ns_inpaint(img, mask)
        got, _ = _run_host(L, img, mask)
        generic, _ = _run_host(L, img, mask, -4096)                # the border-aware evaluation everywhere
        assert np.array_equal(got, want) and np.array_equal(generic, want), (img.shape, mask.mean())
        if min(img.shape) > 1:
            assert np.array_equal(got, _ns(img, mask))


def test_host_replay_equals_cv2_on_large_maps():
    L = _host_lib()
    rng = np.random.default_rng(5)
    # the reference's plugin test shape: 202^2 random heights, mask = randn < 0.5
    em = rng.standard_normal((7, 202, 202)).astype(np.float32)
    mask = np.ascontiguousarray((em[2] < 0.5).astype(np.uint8))
    h = em[0]
    hmax, hmin = float(h[mask < 1].max()), float(h[mask < 1].min())
    img = np.ascontiguousarray(np.clip((h - hmin) * 255 / (hmax - hmin), 0, 255).astype(np.uint8))
    assert np.array_equal(_run_host(L, img, mask)[0], _ns(img, mask))
    # a terrain map with one deep hole (many rounds)
    img, mask = _terrain_case(320, rng)
    got, rounds = _run_host(L, img, mask)
    assert rounds > 150 and np.array_equal(got, _ns(img, mask))
    # an expanding front: a small known blob in an empty image (T ties at every level of the popper chains)
    W = 240
    img = np.zeros((W, W + 17), np.uint8); mask = np.ones_like(img)
    yy, xx = np.mgrid[0:W, 0:W + 17]
    blob = (yy - 120) ** 2 + (xx - 110) ** 2 < 20 ** 2
    img[blob] = (128 + 60 * np.sin(xx[blob] / 7.0) + 40 * np.cos(yy[blob] / 5.0)).astype(np.uint8); mask[blob] = 0
    got, rounds = _run_host(L, img, mask)
    assert rounds > 100 and np.array_equal(got, _ns(img, mask))


def test_convert_to_is_fused_on_x86():
    """cv::Mat::convertTo(CV_32F, a, b) of an 8-bit image rounds v * a + b once (cv2.normalize calls it with
    a = (hi - lo) / 255 and b = lo for an image spanning 0 .. 255)."""
    rng = np.random.default_rng(15)
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    for _ in range(20):
        lo = float(rng.standard_normal() * 5)
        hi = lo + float(rng.random() * 3)
        got = cv2.normalize(v, None, lo, hi, cv2.NORM_MINMAX, dtype=cv2.CV_32F)
        assert np.array_equal(got, fma_f32(v, np.float32((hi - lo) / 255.0), np.float32(lo)))


def test_nonlinear_interpolation_testfilters_scenario():
    """TestFilters.cpp:26: a constant 1.0 layer on a 1 m x 2 m grid at 0.1 m with a 3 x 3 NaN corner and two NaN rows,
    radius 0.1 m, gives back the constant exactly."""
    h = np.ones((10, 20), np.float32)
    h[:3, :3] = np.nan
    h[5:7, :] = np.nan
    L = _host_lib()
    host = lambda img, m, r: _run_host(L, img, m)[0]  # noqa: E731
    for fill in (None, lambda img, m, r: _ns(img, m, r), host):
        out = nonlinear_interpolation(h, 0.1, 0.1, fill)
        assert out.dtype == np.float32 and np.array_equal(out, np.ones_like(h))


def test_nonlinear_interpolation_restatement():
    rng = np.random.default_rng(16)
    h = (rng.standard_normal((23, 31)) * 0.3 + 1.0).astype(np.float32)
    h[rng.random(h.shape) < 0.3] = np.nan
    h[2, 3], h[7, 9] = np.inf, -np.inf
    out = nonlinear_interpolation(h, 0.05, 0.05, lambda img, m, r: _ns(img, m, r))
    fin = np.isfinite(h)
    lo, hi = h[fin].min(), h[fin].max()
    img = to_image_u8(h, lo, hi)
    assert img[2, 3] == 255 and img[7, 9] == 0 and (img[np.isnan(h)] == 0).all()
    keep = ~np.isnan(h)
    assert np.array_equal(out[keep].view(np.uint32), h[keep].view(np.uint32))
    assert np.isfinite(out[~keep]).all() and (out[~keep] >= lo).all() and (out[~keep] <= hi).all()
    # edge cases: no finite cell -> unchanged; a single finite value -> the NaN cells take it
    nan = np.full((4, 5), np.nan, np.float32)
    assert np.isnan(nonlinear_interpolation(nan, 0.1, 0.1)).all()
    const = np.where(rng.random((6, 7)) < 0.5, np.float32(np.nan), np.float32(-2.5)).astype(np.float32)
    const[0, 0] = -2.5
    assert (nonlinear_interpolation(const, 0.1, 0.1) == np.float32(-2.5)).all()
