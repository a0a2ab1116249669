"""CPU: emap_plane_decomposition's resampling (csrc/emap_resample.cuh, include/emap.h).  The NumPy restatement in
tests/resample_oracle.py against cv2.resize(INTER_LINEAR)'s default path within EMAP_RESAMPLE_ULPS (and
EMAP_RESAMPLE_ULPS_LINE for one-row and one-column sources) over up, down and non-integer scales, odd and even sizes up
to 2047, both sides of the exact 2x switch (bit for bit at 2x) and +-inf; the header's per-cell code, built for the CPU
(tests/native/resample_host.cpp), against the restatement bit for bit; and its geometry against inpainting.cpp's
formula, directly and through the library's emap_plane_grid_geometry."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
cv2 = pytest.importorskip("cv2")
import resample_oracle as RS   # noqa: E402

F32 = np.float32

SIZES = [((60, 60), (75, 75)), ((100, 100), (80, 80)), ((101, 101), (50, 50)), ((100, 100), (50, 50)),
         ((37, 53), (90, 20)), ((300, 200), (299, 201)), ((7, 9), (3, 4)), ((2, 2), (5, 5)), ((5, 5), (2, 2)),
         ((40, 40), (1, 55)), ((40, 40), (55, 1)), ((76, 76), (60, 60)), ((60, 80), (30, 40)),
         ((2047, 2047), (1637, 1637)), ((1637, 1637), (2047, 2047)), ((2047, 1024), (1023, 2047))]
LINES = [((1, 40), (1, 55)), ((40, 1), (55, 1)), ((1, 40), (3, 55)), ((40, 1), (55, 3)), ((1, 2047), (1, 1500)),
         ((2047, 1), (1000, 1)), ((1, 1), (3, 3))]


def _image(shape, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) * 3.0 * scale + 10.0 * scale).astype(F32)


def _cv2(img, rows, cols):
    return cv2.resize(img, (cols, rows), interpolation=cv2.INTER_LINEAR)


@pytest.mark.parametrize("scale", [1.0, 1000.0, 1e-3])
@pytest.mark.parametrize("src,dst", SIZES)
def test_restatement_within_bound_of_cv2(src, dst, scale):
    img = _image(src, sum(src) + sum(dst), scale)
    got, want = RS.resample(img, *dst), _cv2(img, *dst)
    assert RS.ulps(got, want, np.abs(img).max()) <= RS.RESAMPLE_ULPS


@pytest.mark.parametrize("src,dst", LINES)
def test_line_sources_within_line_bound(src, dst):
    img = _image(src, 3)
    got, want = RS.resample(img, *dst), _cv2(img, *dst)
    assert RS.ulps(got, want, np.abs(img).max()) <= RS.resample_ulps_line(max(src))


@pytest.mark.parametrize("src", [(100, 100), (60, 80), (4, 6), (2046, 2046)])
def test_exact_2x_is_cv2_bit_for_bit(src):
    """cv2's default path switches INTER_LINEAR to its area-fast path at an exact 2x downscale in both axes; what it
    computes there is a + 0.5 (b - a) per pass, the general formula with f = 0.5, bit for bit."""
    img = _image(src, 11)
    dst = (src[0] // 2, src[1] // 2)
    assert RS.resample(img, *dst).tobytes() == _cv2(img, *dst).tobytes()
    # the 2 x 2 mean in fp32 is not what cv2 computes there
    a, b, c, d = img[0::2, 0::2], img[0::2, 1::2], img[1::2, 0::2], img[1::2, 1::2]
    mean = ((((a + b).astype(F32) + c).astype(F32) + d).astype(F32) * F32(0.25)).astype(F32)
    if src[0] > 4:
        assert mean.tobytes() != _cv2(img, *dst).tobytes()


def test_101_to_50_is_the_linear_path():
    img = _image((101, 101), 5)
    got, want = RS.resample(img, 50, 50), _cv2(img, 50, 50)
    assert RS.ulps(got, want, np.abs(img).max()) <= RS.RESAMPLE_ULPS


@pytest.mark.parametrize("src,dst", [((20, 20), (25, 25)), ((20, 20), (13, 13)), ((21, 17), (9, 30)),
                                     ((20, 20), (10, 10)), ((9, 9), (20, 20))])
def test_interior_infinities_as_cv2(src, dst):
    """+-inf inside the grid: the NaN and infinite cells are cv2's (inf - inf and 0 * inf are NaN; zero weights are
    not skipped), the finite cells within the bound."""
    img = _image(src, 17)
    img[4, 4], img[4, 5], img[7, 3] = np.inf, -np.inf, np.inf
    got, want = RS.resample(img, *dst), _cv2(img, *dst)
    fin = np.isfinite(img)
    assert RS.ulps(got, want, np.abs(img[fin]).max()) <= RS.RESAMPLE_ULPS
    assert np.isnan(want).any()


@pytest.mark.parametrize("src,dst", [((20, 20), (25, 25)), ((9, 9), (20, 20)), ((21, 17), (9, 30))])
def test_edge_infinities_away_from_the_edge(src, dst):
    """+-inf on the edge rows and columns: cv2's default path mixes single and two-tap evaluation at the edge
    positions, which the restatement does not reproduce; every cell whose taps stay off the edge positions agrees."""
    img = _image(src, 23)
    img[0, 3], img[-1, 4], img[5, 0], img[6, -1] = np.inf, -np.inf, np.inf, -np.inf
    got, want = RS.resample(img, *dst), _cv2(img, *dst)
    sr, _, _, er = RS._axis(src[0], dst[0])
    sc, _, _, ec = RS._axis(src[1], dst[1])
    keep = ~(er[:, None] | ec[None, :])
    fin = np.isfinite(img)
    assert RS.ulps(got[keep], want[keep], np.abs(img[fin]).max()) <= RS.RESAMPLE_ULPS
    assert np.isnan(want[keep]).any() or np.isinf(want[keep]).any()


@pytest.fixture(scope="module")
def host():
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libresample_host.so")
    src = os.path.join(HERE, "native", "resample_host.cpp")
    hdr = os.path.join(HERE, "..", "elevation_mapping_cupy_b200", "csrc", "emap_resample.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so, src], check=True)
    lib = C.CDLL(so)
    lib.resample_geometry.argtypes = [C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
    lib.resample_grid.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    return lib


@pytest.mark.parametrize("src,dst", SIZES[:13] + LINES)
def test_host_build_equals_restatement(host, src, dst):
    img = _image(src, 29)
    img[min(3, src[0] - 1), min(2, src[1] - 1)] = np.inf
    out = np.zeros(dst, F32)
    host.resample_grid(img.ctypes.data, src[0], src[1], out.ctypes.data, dst[0], dst[1])
    want = RS.resample(img, *dst)
    assert np.array_equal(np.isnan(out), np.isnan(want))
    ok = ~np.isnan(want)
    assert out[ok].tobytes() == want[ok].tobytes()


GEOMETRY = [(60, 60, 0.05, 0.04), (75, 75, 0.04, 0.05), (100, 100, 0.02, 0.04), (50, 50, 0.04, 0.02),
            (2047, 2047, 0.02, 0.05), (76, 75, 0.04, 0.04 + 5e-7), (76, 75, 0.04, 0.04 + 2e-6), (76, 75, 0.04, 0.0),
            (76, 75, 0.04, -1.0), (3, 3, 0.04, 1.0), (33, 17, 0.031, 0.047), (2047, 1, 0.05, 0.04)]


@pytest.mark.parametrize("rows,cols,res,new_res", GEOMETRY)
def test_geometry_host_build(host, rows, cols, res, new_res):
    size = np.zeros(2, np.int64)
    r = C.c_double(-1.0)
    host.resample_geometry(rows, cols, res, new_res, size.ctypes.data, C.addressof(r))
    want = RS.geometry(rows, cols, res, new_res)
    assert (int(size[0]), int(size[1])) == want[:2] and r.value == want[2]


@pytest.mark.parametrize("rows,cols,res,new_res", GEOMETRY)
def test_geometry_library(rows, cols, res, new_res):
    from elevation_mapping_cupy_b200 import _lib
    from elevation_mapping_cupy_b200.plane_segmentation import PlaneSegmentationParams
    L = _lib.load()
    p = PlaneSegmentationParams(resolution=new_res).to_c()
    size = np.zeros(2, np.int64)
    r = C.c_double(-1.0)
    assert L.emap_plane_grid_geometry(rows, cols, res, C.byref(p), size.ctypes.data, C.addressof(r)) == 0
    assert (int(size[0]), int(size[1]), r.value) == RS.geometry(rows, cols, res, new_res)


def test_geometry_library_rejects():
    from elevation_mapping_cupy_b200 import _lib
    from elevation_mapping_cupy_b200.plane_segmentation import PlaneSegmentationParams
    L = _lib.load()
    size = np.zeros(2, np.int64)
    r = C.c_double(0.0)
    p = PlaneSegmentationParams().to_c()
    for rows, cols, res in ((0, 5, 0.04), (5, 0, 0.04), (5, 5, 0.0), (5, 5, float("nan")), (5, 5, float("inf"))):
        assert L.emap_plane_grid_geometry(rows, cols, res, C.byref(p), size.ctypes.data, C.addressof(r)) == -1
    assert L.emap_plane_grid_geometry(5, 5, 0.04, None, size.ctypes.data, C.addressof(r)) == -1
    q = PlaneSegmentationParams(resolution=float("nan")).to_c()
    assert L.emap_plane_grid_geometry(5, 5, 0.04, C.byref(q), size.ctypes.data, C.addressof(r)) == -1


def test_node_parameters_map_05_to_04():
    """The node's parameters.yaml resamples a 3 m x 3 m window of a 0.05 m map (60 x 60) to 75 x 75 at 0.04 m."""
    assert RS.geometry(60, 60, 0.05, 0.04) == (75, 75, 0.04)
