"""CPU: the pieces of planar region extraction that need no GPU.  The oracle's upsampling equals a transliteration of
Upsampling.cpp's loops; the cropped oracle equals the uncropped one; the integer point-in-polygon test agrees with a
brute-force one on and off the edges; the library header's upsampling index, margin ellipse, border-start rule, border
following and CHAIN_APPROX_SIMPLE compression (csrc/emap_regions.cuh, compiled natively by tests/native/
regions_host.cpp) reproduce cv2.findContours(RETR_CCOMP, CHAIN_APPROX_SIMPLE) contour for contour, in order, with the
parent links; the node's parameters.yaml loads the contour and postprocessing parameters."""
import ctypes as C
import math
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
import planar_regions_oracle as RO   # noqa: E402


@pytest.fixture(scope="module")
def native():
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libregions_host.so")
    src = os.path.join(HERE, "native", "regions_host.cpp")
    deps = [src] + [os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc", f)
                    for f in ("emap_regions.cuh", "emap_planes.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so, src], check=True)
    lib = C.CDLL(so)
    lib.regions_contours.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_int]
    lib.regions_src.argtypes = [C.c_int, C.c_void_p]
    return lib


def _native_contours(lib, img, margin=0):
    img = np.ascontiguousarray(img, np.uint8)
    cap = img.size + 4
    meta = np.zeros(2 * cap, np.int32)
    xy = np.zeros(16 * cap, np.int32)
    half = np.zeros(32, np.int32)
    n = lib.regions_contours(img.ctypes.data, img.shape[0], img.shape[1], meta.ctypes.data, cap, xy.ctypes.data,
                             xy.size, half.ctypes.data, margin)
    assert n >= 0
    out, k = [], 0
    for c in range(n):
        parent, npt = int(meta[2 * c]), int(meta[2 * c + 1])
        out.append((parent, xy[k:k + 2 * npt].reshape(-1, 2).tolist()))
        k += 2 * npt
    return out, half


def _cv2_contours(img):
    """Every top-level contour of RETR_CCOMP in cv2's order, each followed by its children in link order, with the
    index of the parent in this list (-1 for top level)."""
    contours, hierarchy = cv2.findContours(np.ascontiguousarray(img, np.uint8), cv2.RETR_CCOMP,
                                           cv2.CHAIN_APPROX_SIMPLE)
    out = []
    if hierarchy is None:
        return out
    h = hierarchy[0]
    assert len(contours) == sum(1 for i in range(len(contours)) if h[i][3] < 0) + sum(
        1 for i in range(len(contours)) if h[i][3] >= 0)
    for i, c in enumerate(contours):
        if h[i][3] < 0:
            me = len(out)
            out.append((-1, c.reshape(-1, 2).tolist()))
            child = h[i][2]
            while child >= 0:
                assert h[child][3] == i
                out.append((me, contours[child].reshape(-1, 2).tolist()))
                child = h[child][0]
    assert len(out) == len(contours)
    return out


def _masks(seed, count):
    """Seeded random small masks: noise of every density, thin lines, single pixels, diagonal pinches, rings holding
    islands, and foreground on the image edge."""
    rng = np.random.default_rng(seed)
    for k in range(count):
        R, C_ = (int(v) for v in rng.integers(1, 16, 2))
        kind = k % 5
        if kind == 0:
            m = rng.random((R, C_)) < rng.uniform(0.1, 0.95)
        elif kind == 1:                                   # lines and single pixels
            m = np.zeros((R, C_), bool)
            for _ in range(rng.integers(1, 5)):
                if rng.random() < 0.5:
                    m[rng.integers(0, R), :] = True
                else:
                    m[:, rng.integers(0, C_)] = True
            m ^= rng.random((R, C_)) < 0.1
        elif kind == 2:                                   # diagonal pinches
            m = np.zeros((R, C_), bool)
            m[::2, ::2] = True
            m[1::2, 1::2] = rng.random(m[1::2, 1::2].shape) < 0.7
        elif kind == 3:                                   # rings with islands
            R, C_ = max(R, 7), max(C_, 7)
            m = np.zeros((R, C_), bool)
            m[1:-1, 1:-1] = True
            m[2:-2, 2:-2] = False
            m[3:-3, 3:-3] = rng.random(m[3:-3, 3:-3].shape) < 0.6
        else:                                             # edge foreground
            m = rng.random((R, C_)) < 0.5
            m[0, :] = True
            m[:, -1] = rng.random(R) < 0.8
        yield m.astype(np.uint8)


@pytest.mark.parametrize("seed", range(4))
def test_header_tracing_matches_find_contours(native, seed):
    n = 0
    for m in _masks(seed, 1000):
        got, _ = _native_contours(native, m)
        assert got == _cv2_contours(m), m
        n += len(got)
    assert n > 1000


def test_header_ellipse_and_source_index(native):
    for margin in range(5):
        _, half = _native_contours(native, np.zeros((2, 2), np.uint8), margin)
        r = 1 + margin
        mine = np.zeros((2 * r + 1, 2 * r + 1), np.uint8)
        for i in range(2 * r + 1):
            mine[i, r - half[i]:r + half[i] + 1] = 1
        assert np.array_equal(mine, cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2 * r + 1, 2 * r + 1)))
    for m in (2, 3, 4, 7, 30):
        out = np.zeros(3 * m - 2, np.int32)
        native.regions_src(m, out.ctypes.data)
        assert np.array_equal(out, RO.source_index(m))


@pytest.mark.parametrize("shape", [(2, 2), (2, 5), (3, 3), (7, 4), (13, 11)])
def test_upsampling_equals_literal_loop(shape):
    img = np.random.default_rng(shape[0] * 31 + shape[1]).integers(0, 9, shape).astype(np.float32)
    up = RO.upsample(img)
    assert up.shape == (4 + 3 * (shape[0] - 2), 4 + 3 * (shape[1] - 2))
    assert np.array_equal(up, RO.upsample_literal(img))


def _label_scene(seed, n=24):
    rng = np.random.default_rng(seed)
    lab = np.zeros((n, n), np.float32)
    for k in range(1, 7):
        r, c, h, w = rng.integers(0, n, 4)
        lab[r:r + 2 + h // 2, c:c + 2 + w // 2] = k
    lab[rng.random((n, n)) < 0.08] = 0
    planes = np.array([[k, 0.1 * k, -0.2, 0.3, 0.05 * k, -0.1, 1.0] for k in range(1, 7) if (lab == k).any()])
    planes[:, 4:] /= np.linalg.norm(planes[:, 4:], axis=1)[:, None]
    return lab, planes


def _same_regions(a, b, tol=0.0):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x["label"] == y["label"]
        assert np.abs(x["transform"] - y["transform"]).max() <= tol
        polys_x = [x["boundary"]["outer"]] + x["boundary"]["holes"] + [p for i in x["insets"]
                                                                       for p in [i["outer"]] + i["holes"]]
        polys_y = [y["boundary"]["outer"]] + y["boundary"]["holes"] + [p for i in y["insets"]
                                                                       for p in [i["outer"]] + i["holes"]]
        assert len(x["insets"]) == len(y["insets"]) and len(x["boundary"]["holes"]) == len(y["boundary"]["holes"])
        assert [len(p) for p in polys_x] == [len(p) for p in polys_y]
        for p, q in zip(polys_x, polys_y):
            assert np.abs(p - q).max(initial=0.0) <= tol


@pytest.mark.parametrize("margin", [0, 1, 2])
@pytest.mark.parametrize("seed", range(4))
def test_cropped_oracle_equals_whole_image(seed, margin):
    lab, planes = _label_scene(seed)
    a = RO.extract(lab, planes, (1.0, -0.5), 0.04, margin, 0.1, crop=True)
    b = RO.extract(lab, planes, (1.0, -0.5), 0.04, margin, 0.1, crop=False)
    assert len(a) > 0
    _same_regions(a, b)


def _brute_side(p, poly):
    """On an edge: one of the lattice points of an edge; else the winding number by summed angles."""
    n = len(poly)
    for k in range(n):
        a, b = np.array(poly[k]), np.array(poly[(k + 1) % n])
        d = b - a
        g = math.gcd(int(abs(d[0])), int(abs(d[1])))
        steps = [a + d * t // g for t in range(g + 1)] if g else [a]
        if any(tuple(s) == tuple(p) for s in steps):
            return 0
    ang = 0.0
    for k in range(n):
        a = np.array(poly[k], float) - p
        b = np.array(poly[(k + 1) % n], float) - p
        ang += math.atan2(a[0] * b[1] - a[1] * b[0], a @ b)
    return 1 if abs(ang) > math.pi else -1


def test_bounded_side_matches_brute_force():
    rng = np.random.default_rng(3)
    checked = 0
    for m in _masks(11, 200):
        for outer, holes in RO.polygons(np.pad(m, 1)):
            polys = [outer] + holes
            for poly in polys:
                pts = [tuple(int(v) for v in q) for q in poly]
                for _ in range(8):
                    p = (int(rng.integers(-1, m.shape[1] + 3)), int(rng.integers(-1, m.shape[0] + 3)))
                    assert RO.bounded_side(p, pts) == _brute_side(p, pts)
                    checked += 1
                for q in pts:                                   # every vertex is on the boundary
                    assert RO.bounded_side(q, pts) == 0
    assert checked > 1000


def test_from_yaml_reads_contour_and_postprocessing():
    from elevation_mapping_cupy_b200.plane_segmentation import PlaneSegmentationParams
    p = PlaneSegmentationParams.from_yaml(os.path.join(HERE, "golden", "planes", "parameters.yaml"))
    assert p.margin_size == 1
    assert p.extracted_planes_height_offset == 0.0
    c = p.regions_to_c()
    assert (c.margin_size, c.plane_height_offset) == (1, 0.0)
