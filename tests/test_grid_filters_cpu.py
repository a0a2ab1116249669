"""grid_map_filters_rsl's layer filters without a GPU: the restatements of tests/filters_oracle.py (which
emap_grid_filter computes on the device) pinned against cv2 4.13 and against literal transliterations of
processing.cpp and inpainting.cpp, on random, terrain, NaN-holed, infinite, wide-range and one-row / one-column grids."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

import filters_oracle as F  # noqa: E402
import plane_segmentation_oracle as PO  # noqa: E402
from planar_terrain_oracle import gauss_ulps_bound, ulps  # noqa: E402

SHAPES = [(12, 12), (37, 53), (1, 29), (29, 1), (3, 2), (64, 7)]


def same(a, b):
    """NaN-aware bit equality: every non-NaN cell bit for bit, NaN at the same cells."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def grids(shape, seed):
    """Random, terrain, NaN-holed, infinite and wide-range grids of `shape`."""
    rng = np.random.default_rng(seed)
    R, C = shape
    x, y = np.meshgrid(np.linspace(0, 3, C), np.linspace(0, 2, R))
    out = {"random": (rng.standard_normal(shape) * 3).astype(np.float32),
           "terrain": (np.sin(x) * np.cos(2 * y) + 0.3 * np.floor(2 * x) + 0.01 * rng.standard_normal(shape))
           .astype(np.float32)}
    holed = out["terrain"].copy()
    holed[rng.random(shape) < 0.25] = np.nan
    out["holed"] = holed
    inf = out["random"].copy()
    inf[rng.random(shape) < 0.05] = np.inf
    inf[rng.random(shape) < 0.05] = -np.inf
    inf[rng.random(shape) < 0.05] = np.nan
    out["inf"] = inf
    wide = out["random"].copy()
    wide[rng.random(shape) < 0.3] *= np.float32(1e-30)
    wide[rng.random(shape) < 0.1] *= np.float32(1e10)
    out["wide"] = wide
    return out


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 7, 9, 15])
def test_box_blur_is_cv2_blur(shape, k):
    for name, a in grids(shape, k).items():
        for repeats in (1, 2):
            ref = a
            for _ in range(repeats):
                ref = cv2.blur(ref, (k, k))
            assert same(F.box_blur(a, k, repeats), ref), (name, repeats)


def test_box_blur_nan_runs_to_the_bottom():
    a = np.ones((12, 12), np.float32)
    a[3, 5] = np.nan
    out = F.box_blur(a, 3)
    assert np.isnan(out[2:, 4:7]).all() and np.isfinite(out[:2]).all() and np.isfinite(out[:, :4]).all()
    assert same(out, cv2.blur(a, (3, 3)))


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("k", [1, 3, 5])
def test_float_median_is_cv2_on_nan_free_windows(shape, k):
    for name, a in grids(shape, 10 + k).items():
        ref = cv2.medianBlur(a, k)
        got = F.median(a, k, 2, 1)
        nan = np.isnan(a)
        assert np.array_equal(np.isnan(got), nan), name        # a NaN cell stays NaN, and only a NaN cell
        from scipy import ndimage
        clean = ~ndimage.maximum_filter(nan, size=k, mode="nearest")
        assert same(got[clean], ref[clean]), name


def test_float_median_keeps_an_isolated_nan():
    rng = np.random.default_rng(3)
    for k in (3, 5):
        a = rng.random((40, 40)).astype(np.float32)
        a[17, 23] = np.nan
        assert np.isnan(cv2.medianBlur(a, k)).sum() == 1      # cv2's network may move it within the window
        assert np.argwhere(np.isnan(F.median(a, k))).tolist() == [[17, 23]]


@pytest.mark.parametrize("kernel,delta,repeats", [(3, 2, 2), (5, 2, 1), (7, 2, 1), (3, 2, 3), (5, 0, 3), (9, 4, 2),
                                                  (21, 2, 1)])
def test_median_switch_at_5_and_7(kernel, delta, repeats):
    for name, a in grids((41, 37), kernel).items():
        got = F.median(a, kernel, delta, repeats)
        if kernel + delta * (repeats - 1) <= 5:
            ref = a
            for r in range(repeats):
                ref = cv2.medianBlur(ref, kernel + delta * r)
            fin = ~np.isnan(a)
            if name != "inf" and name != "holed":
                assert same(got, ref), name
            assert np.isnan(got[~fin]).all()
        else:
            fin = a[np.isfinite(a)]
            lo, hi = fin.min(), fin.max()
            import ns_inpaint_oracle as NS
            u = NS.to_image_u8(a, lo, hi)
            for r in range(repeats):
                u = cv2.medianBlur(u, kernel + delta * r)
            assert np.array_equal(F.median_u8(NS.to_image_u8(a, lo, hi), kernel), cv2.medianBlur(
                NS.to_image_u8(a, lo, hi), kernel))
            ref = NS.fma_f32(u, np.float32((hi - lo) / np.float32(255)), lo)
            assert same(got, ref), name
            assert np.isfinite(got).all(), name        # every cell is written, NaN cells included


@pytest.mark.parametrize("k", [3, 7, 9, 15, 31, 63])
def test_u8_median_is_cv2(k):
    rng = np.random.default_rng(k)
    for shape in [(50, 61), (1, 40), (40, 1), (3, 3)]:
        u = rng.integers(0, 256, shape).astype(np.uint8)
        assert np.array_equal(F.median_u8(u, k), cv2.medianBlur(u, k))


@pytest.mark.parametrize("k", [1, 3, 5, 7, 9, 15, 63])
@pytest.mark.parametrize("sigma", [0.0, 0.6, 1.0, 2.5, 9.0])
def test_gauss_coefficients_are_opencvs(k, sigma):
    assert F.gauss_coeffs(k, sigma).tobytes() == cv2.getGaussianKernel(k, sigma, cv2.CV_32F).ravel().tobytes()


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("k,sigma", [(1, 0.0), (3, 0.0), (3, 0.8), (5, 0.0), (5, 1.5), (7, 2.0), (15, 3.0), (0, 0.9)])
def test_gaussian_blur_against_cv2(shape, k, sigma):
    for name, a in grids(shape, k).items():
        ref = cv2.GaussianBlur(a, (k, k), sigma)
        got = F.gaussian_blur(a, k, sigma)
        if k <= 3 and sigma <= 0:
            assert same(got, ref), name                    # NaN and +-inf included
        elif name not in ("holed", "inf"):
            kk = k or F.gauss_kernel_size(sigma)
            assert ulps(got, ref, np.abs(a).max()) <= gauss_ulps_bound(kk), name


def _native():
    import ctypes
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    src = os.path.join(here, "native", "filters_host.cpp")
    out_dir = os.path.join(here, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libfilters_host.so")
    hdr = os.path.join(here, "..", "elevation_mapping_cupy_b200", "csrc", "emap_postprocess.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                        src], check=True)
    return ctypes.CDLL(so)


@pytest.mark.parametrize("sigma", [0.0, -1.0, 0.6, 1.0, 2.5, 9.0])
def test_library_gauss_coefficients_are_opencvs(sigma):
    """csrc/emap_postprocess.cuh's pp_gauss_coeffs, built for the CPU, against cv2.getGaussianKernel."""
    import ctypes
    L = _native()
    for k in range(1, 64, 2):
        out = np.zeros(k, np.float32)
        L.gf_gauss(k, ctypes.c_double(sigma), out.ctypes.data_as(ctypes.c_void_p))
        assert out.tobytes() == cv2.getGaussianKernel(k, sigma, cv2.CV_32F).ravel().tobytes(), k


@pytest.mark.parametrize("sigma", [0.1, 0.9, 1.0, 1.0625, 3.3, 7.7])
def test_gaussian_size_from_sigma(sigma):
    a = grids((40, 33), 2)["terrain"]
    k = F.gauss_kernel_size(sigma)
    assert same(cv2.GaussianBlur(a, (0, 0), sigma), cv2.GaussianBlur(a, (k, k), sigma))


@pytest.mark.parametrize("k", [1, 2, 3, 5])
@pytest.mark.parametrize("inpaint", [True, False])
@pytest.mark.parametrize("maximum", [True, False])
def test_dilate_erode_are_processing_cpp(k, inpaint, maximum):
    rng = np.random.default_rng(k)
    for shape in [(12, 9), (5, 5), (k, 7), (7, k)]:
        for a in grids(shape, k).values():
            mask = (rng.random(shape) < 0.8).astype(np.float32)
            for m in (None, mask):
                got = F.morph(a, k, m, inpaint, maximum)
                got = F.morph(a, k, m, inpaint, maximum)
                assert got.tobytes() == F.morph_literal(a, k, m, inpaint, maximum).tobytes()   # zero signs too


@pytest.mark.parametrize("maximum", [True, False])
def test_dilate_erode_windows_without_a_finite_value(maximum):
    """Windows of only NaN and +-inf take the functor's column-major fold, as Eigen's redux computes it."""
    rng = np.random.default_rng(11)
    for k in (1, 2, 3, 4):
        for shape in [(14, 11), (k, 9), (9, k)]:
            a = np.full(shape, np.nan, np.float32)
            u = rng.random(shape)
            a[u < 0.2] = np.inf
            a[(u >= 0.2) & (u < 0.4)] = -np.inf
            a[u > 0.97] = 1.5
            z = rng.random(shape) < 0.1
            a[z] = np.where(rng.random(shape) < 0.5, np.float32(0.0), np.float32(-0.0))[z]
            for inpaint in (True, False):
                got = F.morph(a, k, None, inpaint, maximum)
                assert got.tobytes() == F.morph_literal(a, k, None, inpaint, maximum).tobytes()
    # the fold, by hand: a NaN first cell keeps the cell; else the extreme infinity in the window
    a = np.array([[np.nan, -np.inf], [np.inf, np.nan]], np.float32)
    assert same(F.morph(a, 2, None, True, maximum), a)
    b = np.array([[-np.inf, np.nan], [np.inf, np.nan]], np.float32)
    assert same(F.morph(b, 2, None, True, maximum), np.full((2, 2), np.inf if maximum else -np.inf, np.float32))


def test_dilate_keeps_the_earliest_zero():
    a = np.array([[-0.0, 0.0], [0.0, -0.0]], np.float32)
    assert np.signbit(F.morph(a, 2, None, True, True)).all()
    assert not np.signbit(F.morph(a.T.copy() * -1, 2, None, True, False)).all()


def test_outline_is_processing_cpp():
    for shape in [(12, 9), (3, 3), (3, 40)]:
        for a in grids(shape, 5).values():
            R, C = a.shape
            ref = np.empty_like(a)
            for col in range(C):
                for row in range(R):
                    cc, rr = min(max(col - 1, 0), C - 3), min(max(row - 1, 0), R - 3)
                    ref[row, col] = a[row, col] if np.isnan(a[rr:rr + 3, cc:cc + 3]).any() else np.nan
            assert same(F.outline(a), ref)


def test_min_values_is_the_sweeps_fixed_point():
    for shape in [(15, 13), (1, 20), (20, 1)]:
        for a in grids(shape, 7).values():
            assert same(F.min_values(a), PO.fill_min_values_literal(a))
    a = np.full((5, 5), np.nan, np.float32)
    assert same(F.min_values(a), a)
    z = np.array([[0.0, np.nan, -0.0]], np.float32)
    assert np.signbit(F.min_values(z)[0, 1])


def test_noise_node_chain():
    """noiseNode.cpp: minValues, then boxBlur."""
    a = grids((30, 40), 1)["holed"]
    filled = F.min_values(a)
    assert same(F.box_blur(filled, 5, 2), cv2.blur(cv2.blur(filled, (5, 5)), (5, 5)))
