"""CPU: the signed distance field without a GPU.  The NumPy oracle (tests/sdf_oracle.py) equals brute force over every
pair of voxels on small volumes; the per-line envelope of csrc/emap_sdf.cuh (compiled natively by
tests/native/sdf_host.cpp) equals brute force on random lines with absent sites, all-zero lines, and lines of 1, 2 and
2047 cells, whole and split as a CTA's threads split them; the top slice agrees with the exact comparison next to slice
boundaries; the header's whole field and its queries equal the oracle bit for bit on the demo terrains, NaN-holed and
degenerate grids, and at every kind of query point."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import plane_scenes as S     # noqa: E402
import sdf_oracle as O       # noqa: E402

P = C.c_void_p
D = C.c_double
I64 = C.c_int64
INF = 2 ** 31 - 1


def load_native():
    """The header's host build (compiled on first use)."""
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libsdf_host.so")
    src = os.path.join(HERE, "native", "sdf_host.cpp")
    csrc = os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc")
    deps = [src, os.path.join(csrc, "emap_sdf.cuh"), os.path.join(csrc, "emap_grid.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                        src], check=True)
    lib = C.CDLL(so)
    lib.sdfh_envelope.argtypes = [P, C.c_int, C.c_int, P]
    lib.sdfh_envelope.restype = C.c_int
    lib.sdfh_line.argtypes = [P, C.c_int, C.c_int, P]
    lib.sdfh_top.argtypes = [C.c_float, D, D, C.c_int]
    lib.sdfh_top.restype = C.c_int
    lib.sdfh_field.argtypes = [P, C.c_int, C.c_int, D, C.c_int, D, P]
    lib.sdfh_values.argtypes = [P, C.c_int, C.c_int, C.c_int, P, D, D, I64, P, P]
    return lib


@pytest.fixture(scope="module")
def native():
    return load_native()


def assert_same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    ia, ib = a.view(u), b.view(u)
    bad = np.flatnonzero(ia.reshape(-1) != ib.reshape(-1))
    assert bad.size == 0, "%d of %d differ, first at %d: %r vs %r" % (bad.size, a.size, bad[0], a.reshape(-1)[bad[0]],
                                                                     b.reshape(-1)[bad[0]])


def host_field(lib, e, z_min, n_z, res):
    e = np.ascontiguousarray(e, np.float32)
    out = np.empty((n_z,) + e.shape, np.float32)
    lib.sdfh_field(e.ctypes.data, e.shape[0], e.shape[1], z_min, n_z, res, out.ctypes.data)
    return out


def host_values(lib, vol, pos, res, z_min, pts):
    vol = np.ascontiguousarray(vol, np.float32)
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    pos = np.asarray(pos, np.float64)
    out = np.empty((len(pts), 4))
    lib.sdfh_values(vol.ctypes.data, vol.shape[1], vol.shape[2], vol.shape[0], pos.ctypes.data, res, z_min, len(pts),
                    pts.ctypes.data, out.ctypes.data)
    return out


def small_layers():
    """(name, layer, z_min, n_z, res) of small volumes with every kind of corner case."""
    rng = np.random.default_rng(3)
    out = []
    for shape in ((1, 1), (1, 7), (6, 1), (5, 6), (9, 4)):
        e = (rng.random(shape) * 0.3).astype(np.float32)
        out.append(("random%dx%d" % shape, e, -0.02, 5, 0.05))
    e = (rng.random((7, 5)) * 0.2).astype(np.float32)
    e[2, 3] = np.nan
    e[0, 0] = np.inf
    e[4, 1] = -np.inf
    out += [("nan", e, 0.0, 6, 0.04), ("one_slice", e, 0.1, 1, 0.04),
            ("below", e, -5.0, 4, 0.04), ("above", e, 5.0, 4, 0.04),
            ("all_nan", np.full((4, 5), np.nan, np.float32), 0.0, 3, 0.1),
            ("flat", np.zeros((6, 6), np.float32), -0.1, 4, 0.05)]
    return out


@pytest.mark.parametrize("case", small_layers(), ids=lambda c: c[0])
def test_oracle_matches_brute_force(case):
    _, e, z_min, n_z, res = case
    occ = O.occupancy(e, z_min, n_z, res)
    assert np.array_equal(O.d2_field(occ), O.brute_d2(occ))


def test_oracle_infinities():
    e = np.full((3, 4), 0.5, np.float32)
    assert np.all(O.field(e, -1.0, 3, 0.1) == -np.inf)
    assert np.all(O.field(e, 2.0, 3, 0.1) == np.inf)
    assert np.all(O.field(np.full((3, 4), np.nan, np.float32), 0.0, 3, 0.1) == np.inf)


def _envelope(lib, f, parts):
    fi = np.array([INF if v is None else v for v in f], np.int32)
    out = np.zeros(len(f), np.int32)
    lib.sdfh_envelope(fi.ctypes.data, len(f), parts, out.ctypes.data)
    return [None if v == INF else int(v) for v in out]


def _lines():
    rng = np.random.default_rng(11)
    lines = [[0], [None], [5], [0, 0], [None, 3], [7, None], [None, None], [0] * 64, [None] * 40, [0] * 2047]
    for n in (2, 3, 17, 100, 2047):
        for p_absent in (0.0, 0.5, 0.95):
            f = rng.integers(0, 3000, n)
            lines.append([None if rng.random() < p_absent else int(v) for v in f])
    lines.append([None if k % 97 else (k * 13) % 50 for k in range(2047)])
    lines.append([int(v) for v in rng.integers(0, 4, 2047) ** 2])
    lines.append([(2046 - k) ** 2 if k % 2 else None for k in range(2047)])
    return lines


@pytest.mark.parametrize("parts", [1, 64])
def test_envelope_equals_brute_force(native, parts):
    for f in _lines():
        assert _envelope(native, f, parts) == O.brute_envelope(f), len(f)


def test_signed_line_equals_brute_force(native):
    rng = np.random.default_rng(5)
    for n in (1, 2, 3, 31, 200, 2047):
        for _ in range(4):
            mag = rng.integers(1, 4000, n)
            sign = np.where(rng.random(n) < rng.random(), -1, 1)
            s = sign * np.where(rng.random(n) < 0.2, INF, mag)
            s = s.astype(np.int32)
            out = np.zeros(n, np.int32)
            native.sdfh_line(s.ctypes.data, n, 64, out.ctypes.data)
            to_occ = O.brute_envelope([None if v == INF else (int(v) if v > 0 else 0) for v in s])
            to_free = O.brute_envelope([None if v == -INF else (-int(v) if v < 0 else 0) for v in s])
            want = [(INF if to_occ[q] is None else to_occ[q]) if s[q] > 0 else
                    -(INF if to_free[q] is None else to_free[q]) for q in range(n)]
            assert out.tolist() == want


def test_top_slice_agrees_with_the_comparison(native):
    rng = np.random.default_rng(9)
    for z_min, res, n_z in ((0.0, 0.04, 40), (-1.3, 0.05, 60), (0.1, 0.1, 7), (123.456, 0.03, 100), (-0.7, 0.02, 1)):
        z = O.slices(z_min, n_z, res)
        cand = [np.float32(v) for v in z] + [np.nextafter(np.float32(v), np.float32(-np.inf)) for v in z]
        cand += [np.nextafter(np.float32(v), np.float32(np.inf)) for v in z]
        cand += list((z_min - 1.0 + rng.random(200) * (n_z * res + 2.0)).astype(np.float32))
        cand += [np.float32(-3e38), np.float32(3e38), np.float32(-np.inf)]
        for e in cand:
            want = int((np.float64(e) >= z).sum()) - 1
            assert native.sdfh_top(float(e), z_min, res, n_z) == want, (e, z_min, res)


def _terrain(name):
    png, scale, _, _ = S.TERRAINS[name]
    return S.terrain_image(np.load(S.GOLDEN)["grey__" + name], scale, seed=5 if name == "holes" else None)


@pytest.mark.parametrize("name", ["terrain", "slope", "straight_stairs", "real_stairs", "holes"])
def test_host_field_equals_oracle_on_demo_terrains(native, name):
    e = _terrain(name)[::4, ::4]    # a coarser copy keeps the oracle fast; the GPU tests take the full size
    res = 0.16
    z_min, n_z = O.default_range(e, res, 0.1)
    assert_same_bits(host_field(native, e, z_min, n_z, res), O.field(e, z_min, n_z, res))


@pytest.mark.parametrize("case", small_layers(), ids=lambda c: c[0])
def test_host_field_equals_oracle_on_small_volumes(native, case):
    _, e, z_min, n_z, res = case
    assert_same_bits(host_field(native, e, z_min, n_z, res), O.field(e, z_min, n_z, res))


def test_host_field_largest_d2(native):
    """The largest n_z below the d2 limit for a 3000 x 2 grid, with one occupied voxel in a corner, so the far corner
    holds the largest accepted d2."""
    rows, cols, n_z = 3000, 2, 4096
    while (rows - 1) ** 2 + (cols - 1) ** 2 + (n_z - 1) ** 2 >= O.MAX_D2:
        n_z -= 1
    e = np.full((rows, cols), -1.0, np.float32)
    e[0, 0] = 0.0
    vol = host_field(native, e, 0.0, n_z, 1.0)
    want = O.field(e, 0.0, n_z, 1.0)
    assert_same_bits(vol, want)
    d2 = (rows - 1) ** 2 + (cols - 1) ** 2 + (n_z - 1) ** 2
    assert d2 < O.MAX_D2 <= d2 + 2 * n_z - 1
    assert vol[-1, -1, -1] == np.sqrt(np.float32(d2))


def query_points(vol_shape, pos, res, z_min, n=4000, seed=0):
    """Points at voxel centres, between them, outside every face, edge and corner of the box, far away, on the box's
    faces, and with NaN and infinite coordinates."""
    n_z, rows, cols = vol_shape
    rng = np.random.default_rng(seed)
    ox = pos[0] + (0.5 * (rows * res) - 0.5 * res)
    oy = pos[1] + (0.5 * (cols * res) - 0.5 * res)
    pts = []
    r, c, k = rng.integers(0, rows, n), rng.integers(0, cols, n), rng.integers(0, n_z, n)
    pts.append(np.stack([ox - res * r, oy - res * c, z_min + k * res], 1))
    fr = rng.uniform(-0.2, rows - 0.8, n)
    fc = rng.uniform(-0.2, cols - 0.8, n)
    fk = rng.uniform(-0.2, n_z - 0.8, n)
    pts.append(np.stack([ox - res * fr, oy - res * fc, z_min + res * fk], 1))
    for sr in (-1, 0, 1):               # every face, edge and corner region outside the box
        for sc in (-1, 0, 1):
            for sk in (-1, 0, 1):
                m = n // 27 + 1
                def axis(s, lo, hi):
                    if s < 0:
                        return lo - rng.uniform(0.01, 5.0, m)
                    if s > 0:
                        return hi + rng.uniform(0.01, 5.0, m)
                    return rng.uniform(lo, hi, m)
                pts.append(np.stack([ox - res * axis(sr, 0.0, rows - 1.0), oy - res * axis(sc, 0.0, cols - 1.0),
                                     z_min + res * axis(sk, 0.0, n_z - 1.0)], 1))
    pts.append(np.array([[np.nan, 0.0, 0.0], [0.0, np.nan, 0.0], [0.0, 0.0, np.nan], [np.inf, 0.0, z_min],
                         [-np.inf, oy, z_min], [ox, np.inf, z_min], [ox, oy, -np.inf], [ox, oy, 1e300],
                         [ox - res * (rows - 1), oy - res * (cols - 1), z_min + res * (n_z - 1)]]))
    return np.ascontiguousarray(np.concatenate(pts), np.float64)


def test_host_values_equal_oracle(native):
    e = _terrain("terrain")[::3, ::3]
    res = 0.12
    z_min, n_z = O.default_range(e, res, 0.1)
    vol = O.field(e, z_min, n_z, res)
    pos = (0.3, -0.7)
    pts = query_points(vol.shape, pos, res, z_min)
    assert_same_bits(host_values(native, vol, pos, res, z_min, pts), O.values(vol, pos, res, z_min, pts))


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 1, 6), (1, 5, 1), (4, 1, 1), (3, 4, 5)])
def test_host_values_degenerate_axes(native, shape):
    n_z, rows, cols = shape
    rng = np.random.default_rng(sum(shape))
    e = (rng.random((rows, cols)) * 0.3).astype(np.float32)
    vol = O.field(e, -0.05, n_z, 0.05)
    pts = query_points(vol.shape, (0.0, 0.0), 0.05, -0.05, n=500)
    got = host_values(native, vol, (0.0, 0.0), 0.05, -0.05, pts)
    assert_same_bits(got, O.values(vol, (0.0, 0.0), 0.05, -0.05, pts))
    for a, n in enumerate((rows, cols, n_z)):
        if n == 1:
            assert np.all(got[~np.isnan(pts).any(1), 1 + a] == 0.0)


def test_values_of_an_infinite_volume(native):
    vol = O.field(np.full((3, 3), 9.0, np.float32), 0.0, 2, 0.1)
    assert np.all(vol == -np.inf)
    pts = query_points(vol.shape, (0.0, 0.0), 0.1, 0.0, n=100)
    got = host_values(native, vol, (0.0, 0.0), 0.1, 0.0, pts)
    assert_same_bits(got, O.values(vol, (0.0, 0.0), 0.1, 0.0, pts))
    assert np.all(np.isnan(got[:, 1:3]) | (got[:, 1:3] == 0.0))


def test_nan_points_give_quiet_nans(native):
    vol = O.field(np.zeros((3, 3), np.float32), -0.1, 3, 0.1)
    got = host_values(native, vol, (0.0, 0.0), 0.1, -0.1, np.array([[np.nan, 0, 0], [0, 0, np.nan]]))
    assert np.all(got.view(np.uint64) == 0x7FF8000000000000)
