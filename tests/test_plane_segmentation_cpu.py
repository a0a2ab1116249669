"""CPU: the pieces of plane segmentation that need no GPU.  The oracle's component-minimum fill equals a literal
transliteration of grid_map_filters_rsl's minValues loop; the vectorised sliding-window fit equals the per-cell loop;
the library header's fit and eigen solver (csrc/emap_planes.cuh, compiled natively by tests/native/planes_host.cpp)
match numpy.linalg.eigh; the node's parameters.yaml loads to the expected cosines."""
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
import plane_segmentation_oracle as PO   # noqa: E402


@pytest.mark.parametrize("seed", range(6))
def test_fill_equals_literal_min_values(seed):
    rng = np.random.default_rng(seed)
    R, C_ = rng.integers(3, 24, 2)
    h = rng.normal(0, 1, (R, C_)).astype(np.float32)
    h[rng.random((R, C_)) < rng.uniform(0.2, 0.8)] = np.nan
    if seed == 0:
        h[1, 1] = np.inf
        h[2, 2] = -np.inf
    a, b = PO.fill_min_values(h), PO.fill_min_values_literal(h)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("k", [3, 5])
def test_vectorised_window_fit_equals_loop(k):
    rng = np.random.default_rng(k)
    img = (0.1 * rng.normal(0, 1, (9, 11))).astype(np.float32)
    img[2, 3] = np.nan
    img[0, 0] = np.inf
    img[4:7, 4:7] = 0.3
    na, ea = PO.window_fits(img.astype(np.float64), k, 0.04)
    nb, eb = PO.window_fits_literal(img, k, 0.04)
    assert np.allclose(ea, eb, rtol=1e-9, atol=1e-15)
    assert np.allclose(na[..., 2], nb[..., 2], atol=1e-9)


@pytest.fixture(scope="module")
def native():
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libplanes_host.so")
    src = os.path.join(HERE, "native", "planes_host.cpp")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(
            os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc", "emap_planes.cuh"))):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                        src], check=True)
    lib = C.CDLL(so)
    lib.planes_window_fit.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p]
    return lib


def _fit(native, img, r, c, k, res):
    img = np.ascontiguousarray(img, np.float32)
    out = np.zeros(4)
    native.planes_window_fit(img.ctypes.data, img.shape[0], img.shape[1], r, c, k, res, out.ctypes.data)
    return out


@pytest.mark.parametrize("case", ["flat", "tilted", "wall", "zflip", "few", "degenerate", "noisy"])
def test_header_fit_matches_eigh(native, case):
    rng = np.random.default_rng(1)
    k, res = 5, 0.04
    r_, c_ = np.meshgrid(np.arange(k), np.arange(k), indexing="ij")
    img = np.zeros((k, k), np.float32)
    if case == "tilted":
        img = (0.3 * r_ * res - 0.1 * c_ * res).astype(np.float32)
    elif case == "wall":               # a vertical step: the normal lies in the xy plane
        img = np.where(c_ < 2, 0.0, 1.0).astype(np.float32)
    elif case == "zflip":
        img = (-0.5 * r_ * res + 0.2 * c_ * res).astype(np.float32)
    elif case == "few":
        img = np.full((k, k), np.nan, np.float32)
        img[0, 0] = img[1, 1] = 0.0
    elif case == "degenerate":         # one column of points: the middle eigenvalue is 0
        img = np.full((k, k), np.nan, np.float32)
        img[:, 2] = 0.1
    elif case == "noisy":
        img = rng.normal(0, 0.05, (k, k)).astype(np.float32)
    got = _fit(native, img, 2, 2, k, res)
    n_ref, e_ref = PO.window_fits_literal(img, k, res)
    n_ref, e_ref = n_ref[2, 2], e_ref[2, 2]
    if e_ref >= 1e29:
        assert got[3] == 1e30 and tuple(got[:3]) == (0.0, 0.0, 1.0)
        return
    assert got[2] >= 0
    assert abs(got[3] - e_ref) < 1e-12
    if abs(n_ref[2]) > 1e-12:
        assert np.abs(got[:3] - n_ref).max() < 1e-9
    else:                              # a vertical normal's sign is not defined
        assert np.abs(np.abs(got[:3]) - np.abs(n_ref)).max() < 1e-9


def test_parameters_yaml_cosines():
    """The node's own parameters.yaml (copied from convex_plane_decomposition_ros/config as data)."""
    from elevation_mapping_cupy_b200.plane_segmentation import PlaneSegmentationParams
    p = PlaneSegmentationParams.from_yaml(os.path.join(HERE, "golden", "planes", "parameters.yaml"))
    assert p.plane_inclination_cos == math.cos(30.0 * math.pi / 180.0)
    assert p.local_plane_inclination_cos == math.cos(35.0 * math.pi / 180.0)
    assert (p.median_kernel, p.median_repeats, p.resolution) == (3, 1, 0.04)
    assert (p.kernel_size, p.planarity_opening_filter, p.plane_patch_error_threshold) == (3, 0, 0.02)
    assert (p.min_number_points_per_label, p.connectivity) == (4, 4)
    assert p.include_ransac_refinement is True          # the node's file turns RANSAC on: segment_planes rejects it
    d = PlaneSegmentationParams()
    assert d.include_ransac_refinement is False and d.plane_inclination_cos == p.plane_inclination_cos


def test_golden_fixtures_hold_the_terrains():
    """The golden file carries the demo terrains and an entry for every scene the GPU test reads."""
    import plane_scenes as S
    g = np.load(S.GOLDEN)
    for name in S.TERRAINS:
        assert g["grey__" + name].dtype == np.uint8
    for name in list(S.TERRAINS) + ["lidar", "big"]:
        for case in ("conn4", "conn8"):
            assert g[f"{name}__{case}__planes"].shape[1] == 7
