"""CPU: the pieces of the planar terrain's post-processing that need no GPU.  The node's parameters.yaml loads the
post-processing parameters; the kernel sizes follow std::round (the 2.5 tie at 0.04 m gives 7); the library header's
ellipse spans, kernel sizes, Gaussian coefficients and slope offsets (csrc/emap_postprocess.cuh, compiled natively by
tests/native/postprocess_host.cpp) equal cv2's and the oracle's; the oracle's sloped dilation equals a literal loop of
applyKernelFunction on every cell, the border included; the box restatement and the 3-tap Gaussian restatement equal
cv2 bit for bit, and longer Gaussians, alone and after the box filter, stay within EMAP_POST_GAUSS_ULPS(k) units in
the last place of the layer's largest magnitude of it, on wide-range and on planar, narrow-relief images for every odd
k up to EMAP_POST_MAX_KERNEL."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
cv2 = pytest.importorskip("cv2")
import planar_terrain_oracle as TO   # noqa: E402



@pytest.fixture(scope="module")
def native():
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libpostprocess_host.so")
    src = os.path.join(HERE, "native", "postprocess_host.cpp")
    deps = [src] + [os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc", f)
                    for f in ("emap_postprocess.cuh", "emap_planes.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                        src], check=True)
    lib = C.CDLL(so)
    lib.pp_ellipse_spans.argtypes = [C.c_int, C.c_void_p]
    lib.pp_kernel.argtypes = [C.c_double, C.c_double]
    lib.pp_kernel.restype = C.c_int
    lib.pp_gauss.argtypes = [C.c_int, C.c_void_p]
    lib.pp_offsets.argtypes = [C.c_float, C.c_int, C.c_void_p]
    return lib


def test_from_yaml_reads_postprocessing():
    from elevation_mapping_cupy_b200.plane_segmentation import PlaneSegmentationParams
    p = PlaneSegmentationParams.from_yaml(os.path.join(HERE, "golden", "planes", "parameters.yaml"))
    assert (p.extracted_planes_height_offset, p.nonplanar_height_offset, p.nonplanar_horizontal_offset,
            p.smoothing_dilation_size, p.smoothing_box_kernel_size, p.smoothing_gauss_kernel_size) == \
        (0.0, 0.02, 1, 0.2, 0.1, 0.05)
    c = p.postprocess_to_c()
    assert (c.nonplanar_height_offset, c.nonplanar_horizontal_offset, c.smoothing_dilation_size,
            c.smoothing_box_kernel_size, c.smoothing_gauss_kernel_size) == (0.02, 1, 0.2, 0.1, 0.05)
    d = PlaneSegmentationParams()
    assert (d.nonplanar_height_offset, d.nonplanar_horizontal_offset, d.smoothing_dilation_size,
            d.smoothing_box_kernel_size, d.smoothing_gauss_kernel_size) == (0.02, 1, 0.2, 0.1, 0.05)


@pytest.mark.parametrize("res,sizes", [(0.04, (11, 7, 3)), (0.02, (21, 11, 7)), (0.05, (9, 5, 3)), (0.1, (5, 3, 3))])
def test_kernel_sizes(native, res, sizes):
    got = tuple(TO.kernel_size(s, res) for s in (0.2, 0.1, 0.05))
    assert got == sizes
    assert tuple(native.pp_kernel(s, res) for s in (0.2, 0.1, 0.05)) == sizes
    assert round(0.1 / 0.04) == 2 and 0.1 / 0.04 == 2.5          # the tie Python's round would get wrong


def test_kernel_size_rounds_like_std_round(native):
    q = 0.49999999999999994                      # q + 0.5 rounds to 1.0 in double; std::round(q) is 0
    assert q + 0.5 == 1.0
    for size, res in ((q, 1.0), (0.5, 1.0), (1.5, 1.0), (2.5, 1.0), (2.4999999999999996, 1.0), (0.1, 0.04),
                      (0.3, 0.04), (0.06, 0.04), (0.2, 0.08)):
        assert TO.kernel_size(size, res) == native.pp_kernel(size, res), (size, res)
    assert TO.kernel_size(q, 1.0) == 1 and TO.kernel_size(2.5, 1.0) == 7


def test_kernel_size_rejections(native):
    assert native.pp_kernel(0.0, 0.04) == 1
    assert native.pp_kernel(31 * 0.04, 0.04) == 63
    for bad in (32 * 0.04, -0.01, float("nan"), float("inf"), 1e300):
        assert native.pp_kernel(bad, 0.04) == -1


def test_header_ellipse_spans_equal_cv2(native):
    for size in range(1, 42, 2):
        half = np.zeros(size, np.int32)
        native.pp_ellipse_spans(size, half.ctypes.data)
        r = (size - 1) // 2
        mine = np.zeros((size, size), np.uint8)
        for i in range(size):
            mine[i, r - half[i]:r + half[i] + 1] = 1
        assert np.array_equal(mine, cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (size, size))), size


def test_header_gaussian_coefficients_equal_cv2(native):
    for k in range(1, 64, 2):
        mine = np.zeros(k, np.float32)
        native.pp_gauss(k, mine.ctypes.data)
        want = cv2.getGaussianKernel(k, 0, cv2.CV_32F).ravel()
        assert mine.tobytes() == want.tobytes(), k


@pytest.mark.parametrize("res", [0.02, 0.04, 0.05, 0.1])
def test_header_offsets_equal_oracle(native, res):
    for k in (1, 3, 11, 21, 63):
        mine = np.zeros(k * k, np.float32)
        native.pp_offsets(np.float32(res), k, mine.ctypes.data)
        assert mine.tobytes() == TO.slope_offsets(k, res).tobytes()


def _image(seed, shape, nan=0.0):
    rng = np.random.default_rng(seed)
    img = (5.0 * rng.random(shape) - 1.0 + 0.1 * rng.standard_normal(shape)).astype(np.float32)
    if nan:
        img[rng.random(shape) < nan] = np.nan
    return img


@pytest.mark.parametrize("k", [1, 3, 5, 11])
@pytest.mark.parametrize("shape", [(11, 11), (12, 17), (23, 14)])
def test_sloped_dilation_equals_literal_loop(k, shape):
    for seed, nan in ((0, 0.0), (1, 0.3)):
        img = _image(seed + k, shape, nan)
        if nan:
            img[:4, :] = np.nan                      # whole windows without a finite value
        got = TO.sloped_dilation(img, k, 0.04)
        want = TO.sloped_dilation_literal(img, k, 0.04)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)) or \
            np.array_equal(got, want, equal_nan=True)


@pytest.mark.parametrize("k", [1, 3, 5, 7, 9, 11, 21, 41])
def test_box_restatement_equals_cv2(k):
    for seed in range(4):
        img = _image(10 + seed, (20 + 13 * seed, 90 - 11 * seed))
        assert TO.box_restated(img, k).tobytes() == TO.box(img, k).tobytes()


def test_gauss_3_restatement_equals_cv2():
    for seed in range(6):
        img = _image(20 + seed, (17 + 19 * seed, 120 - 13 * seed))
        assert TO.gauss_restated(img, 3).tobytes() == TO.gauss(img, 3).tobytes()


def _narrow_images(seed, shape):
    """Planar layers: an offset with centimetre to decimetre relief, and a tilted plane with centimetre noise."""
    rng = np.random.default_rng(seed)
    r, c = np.meshgrid(np.arange(shape[0]), np.arange(shape[1]), indexing="ij")
    yield (1.9 + 0.1 * rng.random(shape)).astype(np.float32)
    yield (100.0 + 0.3 * rng.random(shape)).astype(np.float32)
    yield (0.7 + 0.002 * r - 0.001 * c + 0.01 * rng.standard_normal(shape)).astype(np.float32)


@pytest.mark.parametrize("k", range(5, 64, 2))
def test_longer_gauss_restatement_within_bound(k):
    worst = 0.0
    for seed in range(100, 104):
        shape = (90 + seed - 100, 110 - seed + 100)
        for img in [_image(seed, shape)] + list(_narrow_images(seed, shape)):
            worst = max(worst, TO.ulps(TO.gauss_restated(img, k), TO.gauss(img, k), np.abs(img).max()))
    assert worst <= TO.gauss_ulps_bound(k), worst
    print(f"k = {k}: {worst} ulps of the largest magnitude")


@pytest.mark.parametrize("kb,kg", [(7, 3), (11, 7), (11, 41), (5, 63), (21, 21)])
def test_box_then_gauss_within_bound(kb, kg):
    """smooth_planar as the library computes it (box, then Gaussian) against cv2's boxFilter and GaussianBlur."""
    for seed in range(100, 103):
        shape = (90 + seed - 100, 110 - seed + 100)
        for img in [_image(seed, shape)] + list(_narrow_images(seed, shape)):
            mine = TO.gauss_restated(TO.box_restated(img, kb), kg)
            want = TO.gauss(TO.box(img, kb), kg)
            if kg == 3:
                assert mine.tobytes() == want.tobytes()
            else:
                assert TO.ulps(mine, want, np.abs(img).max()) <= TO.gauss_ulps_bound(kg)
