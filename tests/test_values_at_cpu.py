"""CPU: layer values at points without a GPU.  The per-point functions of csrc/emap_values_at.cuh, compiled natively by
tests/native/values_at_host.cpp, equal the Python-float restatement of include/emap.h (tests/values_at_oracle.py) bit
for bit, values and statuses, for every method: random points in and around grids, cell centres and cell boundaries,
every edge and corner (where the fallback chain cubic -> linear -> nearest -> outside shows in the status), the
smallest grids, NaN and infinite cells and coordinates, and the extreme accepted grids.  Properties: linear and cubic
return a cell's value at its centre, reproduce an affine layer, and cubic reproduces a quadratic."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import values_at_oracle as O   # noqa: E402

P = C.c_void_p
I64 = C.c_int64
MAX_EXTENT = 1048576.0                  # EMAP_GRID_MAX_EXTENT
MIN_RES = 9.5367431640625e-07           # EMAP_GRID_MIN_RESOLUTION
METHODS = (O.NEAREST, O.LINEAR, O.CUBIC)


def load_native():
    """The header's host build (compiled on first use)."""
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libvalues_at_host.so")
    src = os.path.join(HERE, "native", "values_at_host.cpp")
    csrc = os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc")
    deps = [src, os.path.join(csrc, "emap_values_at.cuh"), os.path.join(csrc, "emap_grid.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                        src], check=True)
    lib = C.CDLL(so)
    lib.vah_values_at.argtypes = [P, C.c_int, I64, I64, P, C.c_double, C.c_int, I64, P, P, P]
    lib.vah_cubic_weights.argtypes = [C.c_double, P]
    return lib


@pytest.fixture(scope="module")
def native():
    return load_native()


def host_values_at(lib, layers, position, res, method, positions):
    data = np.ascontiguousarray(np.stack([np.asarray(a, np.float32) for a in layers]))
    pos = np.array(position, np.float64)
    q = np.ascontiguousarray(np.asarray(positions, np.float64).reshape(-1, 2))
    values = np.zeros((len(layers), len(q)), np.float32)
    status = np.zeros(len(q), np.int32)
    rows, cols = data.shape[1:]
    lib.vah_values_at(data.ctypes.data, len(layers), rows, cols, pos.ctypes.data, float(res), method, len(q),
                      q.ctypes.data, values.ctypes.data, status.ctypes.data)
    return values, status


def check(lib, layers, position, res, positions, methods=METHODS):
    """Host build == oracle, bit for bit, for each method; returns {method: (values, status)}."""
    out = {}
    for m in methods:
        hv, hs = host_values_at(lib, layers, position, res, m, positions)
        ov, os_ = O.values_at(layers, position, res, m, positions)
        np.testing.assert_array_equal(hs, os_)
        bad = np.nonzero(hv.view(np.uint32) != ov.view(np.uint32))
        assert bad[0].size == 0, (m, bad, hv[bad][:5], ov[bad][:5])
        out[m] = (hv, hs)
    return out


def terrain(rows, cols, seed=0):
    rng = np.random.default_rng(seed)
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    return [(np.sin(0.3 * r) * np.cos(0.2 * c) + 0.1 * rng.standard_normal((rows, cols))).astype(np.float32),
            rng.uniform(-5, 5, (rows, cols)).astype(np.float32),
            (0.01 * r * c).astype(np.float32)]


def centres(rows, cols, position, res):
    L = (rows * res, cols * res)
    xs = [O.axis_position(position[0], L[0], res, i) for i in range(rows)]
    ys = [O.axis_position(position[1], L[1], res, j) for j in range(cols)]
    return np.array([(x, y) for x in xs for y in ys], np.float64)


def random_points(rows, cols, position, res, n, seed=1, margin=2.0):
    rng = np.random.default_rng(seed)
    hx, hy = 0.5 * rows * res * margin, 0.5 * cols * res * margin
    return np.stack([rng.uniform(position[0] - hx, position[0] + hx, n),
                     rng.uniform(position[1] - hy, position[1] + hy, n)], 1)


def boundaries(rows, cols, position, res):
    """Every cell edge on both axes (and the map's own edges), crossed with cell centres and edges of the other."""
    L = (rows * res, cols * res)
    ex = [position[0] + 0.5 * L[0] - res * i for i in range(rows + 1)]
    ey = [position[1] + 0.5 * L[1] - res * j for j in range(cols + 1)]
    cx = [O.axis_position(position[0], L[0], res, i) for i in range(rows)]
    cy = [O.axis_position(position[1], L[1], res, j) for j in range(cols)]
    pts = [(x, y) for x in ex for y in ey + cy] + [(x, y) for x in cx for y in ey]
    return np.array(pts, np.float64)


@pytest.mark.parametrize("shape", [(40, 40), (17, 29), (64, 9)])
def test_random_points_match_oracle(native, shape):
    rows, cols = shape
    position, res = (1.25, -0.75), 0.1
    layers = terrain(rows, cols)
    pts = random_points(rows, cols, position, res, 3000)
    out = check(native, layers, position, res, pts)
    for m in METHODS:
        assert (out[m][1] == O.OUTSIDE).any() and (out[m][1] == m + 1).any()


def test_centres_and_boundaries_match_oracle(native):
    rows, cols, position, res = 12, 10, (-3.3, 7.1), 0.2
    layers = terrain(rows, cols, 2)
    check(native, layers, position, res, centres(rows, cols, position, res))
    check(native, layers, position, res, boundaries(rows, cols, position, res))


def test_fallback_chain_at_edges_and_corners(native):
    """Cubic needs two cells on the far side of its corner, linear one neighbour: along the edges and at the corners the
    status steps down cubic -> linear -> nearest, and beyond the map it is outside."""
    rows, cols, position, res = 8, 8, (0.0, 0.0), 1.0
    layers = terrain(rows, cols, 3)
    L = rows * res
    # rows of points at fractions across the grid, 0.1 res apart, from outside the +x edge to outside the -x edge
    xs = np.arange(0.5 * L + 0.35, -0.5 * L - 0.4, -0.1)
    pts = np.array([(x, 0.05) for x in xs] + [(0.05, y) for y in xs] + [(x, x) for x in xs], np.float64)
    out = check(native, layers, position, res, pts)
    st = out[O.CUBIC][1]
    assert set(st.tolist()) == {O.OUTSIDE, O.BY_NEAREST, O.BY_LINEAR, O.BY_CUBIC}
    # walking in from the +x edge along y = 0.05 (an interior column): outside, nearest, linear, cubic
    first = [int(s) for s in st[:len(xs) // 2]]
    seen = [s for i, s in enumerate(first) if i == 0 or s != first[i - 1]]
    assert seen == [O.OUTSIDE, O.BY_NEAREST, O.BY_LINEAR, O.BY_CUBIC], seen
    assert (out[O.LINEAR][1] <= O.BY_LINEAR).all() and (out[O.NEAREST][1] <= O.BY_NEAREST).all()
    # every corner cell: near its outer corner nearest (no neighbour outside), outside beyond it
    for sx in (1, -1):
        for sy in (1, -1):
            p = np.array([[sx * (0.5 * L - 0.1), sy * (0.5 * L - 0.1)], [sx * (0.5 * L + 0.1), sy * (0.5 * L - 0.1)]])
            o = check(native, layers, position, res, p)
            assert o[O.CUBIC][1].tolist() == [O.BY_NEAREST, O.OUTSIDE]


@pytest.mark.parametrize("shape", [(1, 1), (1, 7), (7, 1), (2, 2), (3, 3), (4, 4)])
def test_small_grids(native, shape):
    rows, cols = shape
    position, res = (0.4, -0.2), 0.25
    layers = terrain(rows, cols, 4)
    pts = np.concatenate([random_points(rows, cols, position, res, 500, 5, 1.5), centres(rows, cols, position, res),
                          boundaries(rows, cols, position, res)])
    out = check(native, layers, position, res, pts)
    st = out[O.CUBIC][1]
    assert (st == O.BY_CUBIC).any() == (rows >= 4 and cols >= 4)
    assert (st == O.BY_LINEAR).any() == (rows >= 2 and cols >= 2)


def test_non_finite_cells_and_coordinates(native):
    rows, cols, position, res = 16, 16, (0.0, 0.0), 0.5
    rng = np.random.default_rng(6)
    layers = terrain(rows, cols, 6)
    for a, v in zip(layers, (np.nan, np.inf, -np.inf)):
        idx = rng.integers(0, rows * cols, 20)
        a.reshape(-1)[idx] = v
    # NaNs with a payload, and a negative NaN
    layers[0].reshape(-1)[:4].view(np.uint32)[:] = [0x7FC00001, 0xFFC00000, 0x7F800001, 0xFFFFFFFF]
    pts = np.concatenate([random_points(rows, cols, position, res, 2000, 7, 1.2), centres(rows, cols, position, res),
                          [[np.nan, 0.0], [0.0, np.nan], [np.inf, 0.0], [0.0, -np.inf], [np.nan, np.nan],
                           [-np.inf, np.inf]]])
    out = check(native, layers, position, res, pts)
    for m in METHODS:
        v, st = out[m]
        assert (st[-6:] == O.OUTSIDE).all()
        nan = np.isnan(v)
        assert nan.any() and (v[nan].view(np.uint32) == 0x7FC00000).all()
        assert np.isinf(v).any()


def test_zero_weight_next_to_an_infinite_cell_is_nan(native):
    rows, cols, res = 8, 8, 1.0
    a = np.zeros((rows, cols), np.float32)
    a[3, 4] = np.inf
    # at the centre of cell (3, 3): linear reads (3, 3), (2, 3), (3, 2), (2, 2); cubic reads rows 4..1, cols 4..1
    p = centres(rows, cols, (0.0, 0.0), res).reshape(rows, cols, 2)[3, 3][None]
    out = check(native, [a], (0.0, 0.0), res, p)
    assert out[O.LINEAR][0][0, 0] == 0.0
    assert np.isnan(out[O.CUBIC][0][0, 0])


@pytest.mark.parametrize("case", ["max_extent", "min_resolution"])
def test_extreme_grids(native, case):
    if case == "max_extent":
        rows, cols, res = 64, 48, 1024.0
        position = (MAX_EXTENT - rows * res, -(MAX_EXTENT - cols * res))
    else:
        rows, cols, res = 64, 48, MIN_RES
        position = (1000.0, -1000.0)
    layers = terrain(rows, cols, 8)
    pts = np.concatenate([random_points(rows, cols, position, res, 2000, 9, 1.1), centres(rows, cols, position, res),
                          boundaries(rows, cols, position, res)])
    out = check(native, layers, position, res, pts)
    for m in METHODS:
        assert (out[m][1] == m + 1).any()


def test_value_at_a_cell_centre(native):
    """Linear and cubic return the cell's own value at its centre when the cells they read are finite."""
    rows, cols, position, res = 20, 24, (2.0, 3.0), 0.05
    layers = terrain(rows, cols, 10)
    pts = centres(rows, cols, position, res)
    out = check(native, layers, position, res, pts)
    rc = np.array([(i, j) for i in range(rows) for j in range(cols)])
    for m in (O.LINEAR, O.CUBIC):
        v, st = out[m]
        assert (st == m + 1).sum() > 0
        for k, a in enumerate(layers):
            np.testing.assert_array_equal(v[k], a[rc[:, 0], rc[:, 1]])


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def test_affine_and_quadratic_layers(native):
    """The interpolants are exact for these polynomials in exact arithmetic: an affine layer within 4 ulps (linear and
    cubic) and a quadratic within 8 ulps of its largest cell value (cubic), against the polynomial at the point."""
    rows, cols, position, res = 32, 32, (0.5, -0.25), 0.125
    L = (rows * res, cols * res)
    X = np.array([O.axis_position(position[0], L[0], res, i) for i in range(rows)])
    Y = np.array([O.axis_position(position[1], L[1], res, j) for j in range(cols)])
    xx, yy = np.meshgrid(X, Y, indexing="ij")
    # exactly representable cells: small integers
    affine = lambda x, y: 3.0 + 8.0 * (x - position[0]) - 16.0 * (y - position[1])              # noqa: E731
    quad = lambda x, y: 64.0 * (x - position[0]) ** 2 + 32.0 * (x - position[0]) * (y - position[1])  # noqa: E731
    la, lq = affine(xx, yy).astype(np.float32), quad(xx, yy).astype(np.float32)
    assert np.array_equal(la, affine(xx, yy)) and np.array_equal(lq, quad(xx, yy))
    pts = random_points(rows, cols, position, res, 3000, 11, 0.8)
    out = check(native, [la, lq], position, res, pts)
    x, y = pts[:, 0], pts[:, 1]
    for m in (O.LINEAR, O.CUBIC):
        v, st = out[m]
        sel = st == m + 1
        assert sel.sum() > 2000
        assert _ulps(v[0][sel], affine(x[sel], y[sel])).max() <= 4
    v, st = out[O.CUBIC]
    sel = st == O.BY_CUBIC
    err = np.abs(v[1][sel].astype(np.float64) - quad(x[sel], y[sel]))
    assert err.max() <= 8 * np.spacing(np.float32(np.abs(lq).max()))


def test_cubic_weights(native):
    """The weights are Keys' kernel with a = -0.5 and sum to 1."""
    w = np.zeros(4)
    for t in np.linspace(0.0, 1.0, 33):
        native.vah_cubic_weights(float(t), w.ctypes.data)
        assert w.tolist() == O.cubic_weights(float(t))
        keys = lambda s: (1.5 * s ** 3 - 2.5 * s ** 2 + 1 if s <= 1 else  # noqa: E731
                          -0.5 * s ** 3 + 2.5 * s ** 2 - 4 * s + 2 if s < 2 else 0.0)
        np.testing.assert_allclose(w, [keys(abs(t + 1)), keys(abs(t)), keys(abs(t - 1)), keys(abs(t - 2))], atol=1e-15)
        assert abs(w.sum() - 1.0) < 1e-15
