"""CPU: the grid lookups without a GPU.  The header's closed-form walk (csrc/emap_grid_lookup.cuh, compiled natively by
tests/native/lookup_host.cpp) visits the cells of grid_map's stepping LineIterator, for one lane and for 32; projected
line ends are inside the map for every accepted grid, at its bounds, edges and corners; the header's whole queries
(max, values, derivatives) equal the Python-float oracle (tests/grid_lookup_oracle.py) bit for bit on the demo terrains,
NaN-holed layers and lines along the edges; the reference's TestLookup.cpp and TestDerivativeFilter.cpp hold on their
own geometries; the preserved quirks; exact slopes of planes and quadratics; and the grid rejections."""
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
import grid_lookup_oracle as O   # noqa: E402
import plane_scenes as S         # noqa: E402

P = C.c_void_p
D = C.c_double
I64 = C.c_int64
FLT_MAX = O.FLT_MAX


def load_native():
    """The header's host build (compiled on first use)."""
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "liblookup_host.so")
    src = os.path.join(HERE, "native", "lookup_host.cpp")
    csrc = os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc")
    deps = [src, os.path.join(csrc, "emap_grid_lookup.cuh"), os.path.join(csrc, "emap_grid.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                        src], check=True)
    lib = C.CDLL(so)
    lib.glh_walks.argtypes = [I64, P, C.c_int, I64, P, P]
    lib.glh_minor.argtypes = [I64, I64, I64]
    lib.glh_minor.restype = I64
    lib.glh_project.argtypes = [I64, I64, P, D, I64, P, P, P]
    lib.glh_max.argtypes = [P, I64, I64, P, D, I64, P, P, P]
    lib.glh_values.argtypes = [P, I64, I64, P, D, I64, P, P, P, P]
    lib.glh_values.restype = I64
    lib.glh_derivatives.argtypes = [P, I64, I64, P, D, I64, P, C.c_int, P, P]
    lib.glh_check_grid.argtypes = [I64, I64, P, D, I64]
    lib.glh_kernels.argtypes = [D, P, P]
    return lib


@pytest.fixture(scope="module")
def native():
    return load_native()


def _geom(g):
    data = np.ascontiguousarray(g.data, np.float32)
    return data, np.array(g.pos, np.float64)


def host_max(lib, g, lines):
    data, pos = _geom(g)
    q = np.ascontiguousarray(lines, np.float64)
    index, value = np.zeros((len(q), 3), np.int32), np.zeros((len(q), 3))
    lib.glh_max(data.ctypes.data, g.rows, g.cols, pos.ctypes.data, g.res, len(q), q.ctypes.data, index.ctypes.data,
                value.ctypes.data)
    return index, value


def host_values(lib, g, lines):
    data, pos = _geom(g)
    q = np.ascontiguousarray(lines, np.float64)
    counts, first = np.zeros(len(q), np.int32), np.zeros(len(q), np.int64)
    total = lib.glh_values(data.ctypes.data, g.rows, g.cols, pos.ctypes.data, g.res, len(q), q.ctypes.data,
                           counts.ctypes.data, first.ctypes.data, None)
    rows = np.zeros((total, 3))
    total = lib.glh_values(data.ctypes.data, g.rows, g.cols, pos.ctypes.data, g.res, len(q), q.ctypes.data,
                           counts.ctypes.data, first.ctypes.data, rows.ctypes.data)
    return counts, first, rows[:total]


def host_derivatives(lib, g, positions, curvature=False):
    data, pos = _geom(g)
    p = np.ascontiguousarray(positions, np.float64)
    nv = 5 if curvature else 2
    index, value = np.zeros((len(p), 3), np.int32), np.zeros((len(p), nv))
    lib.glh_derivatives(data.ctypes.data, g.rows, g.cols, pos.ctypes.data, g.res, len(p), p.ctypes.data,
                        int(curvature), index.ctypes.data, value.ctypes.data)
    return index, value


def assert_same_bits(a, b):
    """Equal outputs, NaN for NaN, bit for bit."""
    for x, y in zip(a, b):
        x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
        assert x.shape == y.shape, (x.shape, y.shape)
        assert x.tobytes() == y.tobytes(), np.argwhere(x != y)[:5]


def check_all(lib, g, lines, positions):
    """Host build == oracle, bit for bit, for the three lookups."""
    assert_same_bits(host_max(lib, g, lines), O.max_batch(g, lines))
    assert_same_bits(host_values(lib, g, lines), O.values_batch(g, lines))
    for curv in (False, True):
        assert_same_bits(host_derivatives(lib, g, positions, curv), O.derivative_batch(g, positions, curv))


# ---- the walk ----
def _stepping_walks(ends, n_max):
    """grid_map's LineIterator stepping (the numerator loop), vectorised over lines: (lines, n_max, 2) cells, -1 past
    the end."""
    s, e = ends[:, :2].astype(np.int64), ends[:, 2:].astype(np.int64)
    d = np.abs(e - s)
    step = np.where(e >= s, 1, -1)
    row_major = d[:, 0] >= d[:, 1]
    den = np.where(row_major, d[:, 0], d[:, 1])
    num = den // 2
    add = np.where(row_major, d[:, 1], d[:, 0])
    n = den + 1
    idx = s.copy()
    out = np.full((len(ends), n_max, 2), -1, np.int64)
    for i in range(n_max):
        live = i < n
        out[live, i] = idx[live]
        num = num + add
        cross = num >= den
        num = np.where(cross, num - den, num)
        minor = np.where(row_major, 1, 0)
        idx[np.arange(len(ends)), minor] += np.where(cross, step[np.arange(len(ends)), minor], 0)
        idx[np.arange(len(ends)), 1 - minor] += step[np.arange(len(ends)), 1 - minor]
    return out, n


@pytest.mark.parametrize("sign", [(1, 1), (1, -1), (-1, 1), (-1, -1)])
def test_closed_form_walk_equals_stepping_iterator(native, sign):
    m = 200
    dr, dc = np.meshgrid(np.arange(m + 1), np.arange(m + 1), indexing="ij")
    r0, c0 = 250, 260
    ends = np.stack([np.full(dr.size, r0), np.full(dr.size, c0), r0 + sign[0] * dr.ravel(),
                     c0 + sign[1] * dc.ravel()], 1).astype(np.int32)
    want, n = _stepping_walks(ends, m + 1)
    for lanes in (1, 32):
        got = np.full((len(ends), m + 1, 2), -1, np.int32)
        cnt = np.zeros(len(ends), np.int64)
        native.glh_walks(len(ends), ends.ctypes.data, lanes, m + 1, got.ctypes.data, cnt.ctypes.data)
        assert np.array_equal(cnt, n)
        assert np.array_equal(got, want)
    assert np.array_equal(want[np.arange(len(ends)), n - 1], ends[:, 2:])      # every walk ends on its end cell


def test_closed_form_minor_steps_large_lines(native):
    rng = np.random.default_rng(3)
    for _ in range(2000):
        major = int(rng.integers(0, 2 ** 31 - 1))
        minor = int(rng.integers(0, major + 1))
        i = int(rng.integers(0, major + 1))
        want = 0 if major == 0 else (major // 2 + i * minor) // major
        assert native.glh_minor(major, minor, i) == want
        if major:
            assert native.glh_minor(major, minor, major) == minor       # the end cell
    # the stepping numerator over the first cells of large random lines
    ends = np.array([[0, 0, int(a), int(b)] for a, b in rng.integers(0, 2 ** 30, (64, 2))], np.int32)
    want, _ = _stepping_walks(ends, 3000)
    got = np.full((len(ends), 3000, 2), -1, np.int32)
    cnt = np.zeros(len(ends), np.int64)
    native.glh_walks(len(ends), ends.ctypes.data, 32, 3000, got.ctypes.data, cnt.ctypes.data)
    assert np.array_equal(got, want)


def _extreme_grids():
    rng = np.random.default_rng(11)
    out = [(10, 20, (0.1, 0.2), 0.1), (1, 1, (0.0, 0.0), 2.0 ** -20), (2, 1, (-3.0, 7.0), 2.0 ** -20),
           (2047, 2047, (0.0, 0.0), 0.04), (7, 3, (2.0 ** 20 - 7 * 0.5, -(2.0 ** 20 - 3 * 0.5)), 0.5),
           (1 << 20, 1, (0.0, 2.0 ** 20 - 2.0 ** -20), 2.0 ** -20), (1, 1 << 20, (2.0 ** 19, 0.0), 0.5)]
    for _ in range(200):
        rows, cols = (int(v) for v in rng.integers(1, 3000, 2))
        res = float(2.0 ** rng.uniform(-20, 3))
        ext = [rows * res, cols * res]
        if max(ext) > 2.0 ** 20:
            continue
        pos = tuple(float(rng.choice([-1, 1]) * (2.0 ** 20 - e) * rng.choice([1.0, rng.random()])) for e in ext)
        out.append((rows, cols, pos, res))
    return out


def test_projected_ends_are_inside_every_accepted_grid(native):
    """getIndexLimitedToMapRange's stepping loop never runs: every projected point is inside the map."""
    nan, inf = float("nan"), float("inf")
    for rows, cols, pos, res in _extreme_grids():
        p = np.array(pos, np.float64)
        assert native.glh_check_grid(rows, cols, p.ctypes.data, res, 1) == 0, (rows, cols, pos, res)
        hx, hy = 0.5 * rows * res, 0.5 * cols * res
        pts = []
        for sx in (-1, 0, 1):
            for sy in (-1, 0, 1):
                for k in (0.0, 1e-9, 1e-6, 1.0, 1e300):
                    pts.append((pos[0] + sx * (hx + k), pos[1] + sy * (hy + k)))
                    pts.append((pos[0] + sx * (hx - k), pos[1] + sy * (hy - k)))
        pts += [(nan, nan), (nan, pos[1]), (inf, -inf), (-inf, inf), (inf, nan), (np.nextafter(pos[0] + hx, inf), 0.0)]
        xy = np.array(pts, np.float64)
        out, inside = np.zeros_like(xy), np.zeros(len(xy), np.int32)
        native.glh_project(rows, cols, p.ctypes.data, res, len(xy), xy.ctypes.data, out.ctypes.data,
                           inside.ctypes.data)
        assert inside.all(), (rows, cols, pos, res, xy[inside == 0][:3])
        g = O.Grid(np.zeros((1, 1)), pos, res)
        g.rows, g.cols, g.n, g.len = rows, cols, (rows, cols), (rows * res, cols * res)
        want = np.array([O.project(g, tuple(v)) for v in xy.tolist()])
        assert out.tobytes() == want.tobytes()
    # NaN lands on the upper bound, +-inf on its own bound
    g = O.Grid(np.zeros((10, 20)), (0.1, 0.2), 0.1)
    assert O.project(g, (nan, nan)) == ((0.1 + 0.5) - 1e-6, (0.2 + 1.0) - 1e-6)
    assert O.project(g, (-inf, inf)) == ((0.1 - 0.5) + 1e-6, (0.2 + 1.0) - 1e-6)


# ---- host build == oracle ----
def _terrain_grid(name):
    png, scale, _, _ = S.TERRAINS[name]
    img = S.terrain_image(np.load(S.GOLDEN)["grey__" + name], scale, seed=5 if name == "holes" else None)
    return O.Grid(img, (0.37, -1.3), S.RES)


@pytest.mark.parametrize("name", list(S.TERRAINS))
def test_host_build_equals_oracle_on_demo_terrains(native, name):
    g = _terrain_grid(name)
    lines = np.concatenate([O.random_lines(g, 1500, seed=len(name)), O.edge_lines(g)])
    check_all(native, g, lines, O.random_positions(g, 1500, seed=len(name)))


@pytest.mark.parametrize("scene", ["holes", "stairs", "rough"])
def test_host_build_equals_oracle_on_nan_holed_layers(native, scene):
    z = S.synthetic(scene, 97, seed=4)
    z[::7, 3::11] = np.nan
    z[40:45, :] = np.inf
    z[50, 50:60] = -np.inf
    z[60:62, 10:30] = -0.0
    z[63, 10:30] = 0.0
    g = O.Grid(z, (-2.5, 4.0), 0.05)
    lines = np.concatenate([O.random_lines(g, 1500, seed=1, lo=0.2, hi=6.0, outside=0.5), O.edge_lines(g)])
    check_all(native, g, lines, O.random_positions(g, 1500, seed=2))


@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (9, 1), (5, 5), (5, 17), (23, 5)])
def test_host_build_equals_oracle_on_small_grids(native, shape):
    rng = np.random.default_rng(shape[0] * 31 + shape[1])
    z = rng.standard_normal(shape).astype(np.float32)
    g = O.Grid(z, (0.3, -0.2), 0.1)
    lines = np.concatenate([O.random_lines(g, 300, seed=5, lo=0.0, hi=2.0, outside=1.0), O.edge_lines(g)])
    assert_same_bits(host_max(native, g, lines), O.max_batch(g, lines))
    assert_same_bits(host_values(native, g, lines), O.values_batch(g, lines))
    if min(shape) >= 5:
        pos = O.random_positions(g, 300, seed=6)
        for curv in (False, True):
            assert_same_bits(host_derivatives(native, g, pos, curv), O.derivative_batch(g, pos, curv))


# ---- the reference's tests on their own geometries: 1 x 2 m at 0.1 m ----
def test_reference_lookup_constant_map(native):
    g = O.Grid(np.full((10, 20), np.float32(133.7)), (0.1, 0.2), 0.1)
    lines = np.array([[-0.1, -0.2, 0.3, 0.4], [-0.1, -0.2, -0.1, -0.2], [1000.0, 1000.0, 2000.0, 2000.0]])
    index, value = host_max(native, g, lines)
    assert index[:, 0].all()
    assert (value[:, 0] == float(np.float32(133.7))).all()
    assert_same_bits((index, value), O.max_batch(g, lines))


def test_reference_lookup_max_in_middle(native):
    g = O.Grid(np.zeros((10, 20)), (0.1, 0.2), 0.1)
    check = -FLT_MAX
    for col in range(20):
        y = O.position(g, 0, col)[1]
        g.data[:, col] = np.float32(-y * y)
        check = max(check, float(np.float32(-y * y)))
    index, value = host_max(native, g, np.array([[-0.5, -0.5, 0.5, 0.5]]))
    assert index[0, 0] == 1 and value[0, 0] == check


def test_reference_lookup_only_nan(native):
    g = O.Grid(np.full((10, 20), np.nan), (0.1, 0.2), 0.1)
    index, value = host_max(native, g, np.array([[-0.1, -0.2, 0.3, 0.4]]))
    assert index[0].tolist() == [0, 0, 0] and value[0, 0] == -FLT_MAX
    assert tuple(value[0, 1:]) == O.position(g, 0, 0)


def test_reference_derivative_constant_map(native):
    """TestDerivativeFilter.cpp's map (1 x 2 m at 0.1 m, centred at the origin, constant 1): every cell's gradient is
    exactly 0 (the first-derivative kernel is antisymmetric in float) and its curvature within the float rounding of
    the second-derivative kernel's sum.  The reference test never initialises its filter (zero kernels); this one uses
    the kernels of a 0.1 m map."""
    g = O.Grid(np.ones((10, 20)), (0.0, 0.0), 0.1)
    pos = np.array([O.position(g, r, c) for r in range(10) for c in range(20)])
    index, value = host_derivatives(native, g, pos, True)
    assert (index[:, 0] == O.INSIDE).all()
    assert np.array_equal(index[:, 1:], np.array([(r, c) for r in range(10) for c in range(20)]))
    assert (value[:, :2] == 0.0).all() and (value[:, 3] == 0.0).all()
    _, d2 = O.kernels(0.1)
    assert np.abs(value[:, [2, 4]]).max() <= 8 * np.spacing(np.float32(abs(d2[2])))
    assert_same_bits((index, value), O.derivative_batch(g, pos, True))


# ---- the preserved quirks ----
def _row_grid(values):
    """A 1-row grid whose cells hold `values`, at 1 m, so a line along +y from column 0 to the last visits them all."""
    z = np.array([values], np.float32)
    return O.Grid(z, (0.0, 0.0), 1.0)


def _along(g):
    """The line from column cols-1 (-y edge) to column 0 (+y edge): cells in ascending column order? No: from col 0."""
    y0 = O.position(g, 0, 0)[1]
    y1 = O.position(g, 0, g.cols - 1)[1]
    return np.array([[0.0, y0, 0.0, y1]])


def test_quirk_position_is_the_last_finite_cell(native):
    g = _row_grid([1.0, 9.0, 2.0, np.nan, 3.0, np.inf, np.nan])
    index, value = host_max(native, g, _along(g))
    assert index[0].tolist() == [1, 0, 4]            # valid, the last finite cell (column 4), not the maximum's (1)
    assert value[0, 0] == 9.0 and value[0, 2] == O.position(g, 0, 4)[1]
    assert_same_bits((index, value), O.max_batch(g, _along(g)))


@pytest.mark.parametrize("first", [0.0, -0.0])
def test_quirk_signed_zero_ties_keep_the_first(native, first):
    g = _row_grid([-1.0, first, -first, -first, -5.0])
    index, value = host_max(native, g, _along(g))
    assert index[0, 0] == 1 and math.copysign(1.0, value[0, 0]) == math.copysign(1.0, first)
    assert_same_bits((index, value), O.max_batch(g, _along(g)))


def test_quirk_nan_and_inf_queries_clamp_to_the_bounds(native):
    z = np.arange(200, dtype=np.float32).reshape(10, 20)
    g = O.Grid(z, (0.1, 0.2), 0.1)
    nan, inf = float("nan"), float("inf")
    lines = np.array([[nan, nan, nan, nan], [inf, inf, -inf, -inf], [nan, 0.0, -inf, 0.0], [0.0, 0.0, 0.0, inf]])
    index, value = host_max(native, g, lines)
    assert index[:, 0].all()
    assert index[0, 1:].tolist() == [0, 0] and value[0, 0] == 0.0          # NaN -> the upper bounds: cell (0, 0)
    assert index[1, 1:].tolist() == [9, 19] and value[1, 0] == 199.0       # the whole diagonal
    assert_same_bits((index, value), O.max_batch(g, lines))
    assert_same_bits(host_values(native, g, lines), O.values_batch(g, lines))


def test_quirk_lowest_only_line_is_invalid(native):
    g = _row_grid([np.nan, -FLT_MAX, np.nan, -FLT_MAX, np.nan])
    index, value = host_max(native, g, _along(g))
    assert index[0].tolist() == [0, 0, 3] and value[0, 0] == -FLT_MAX     # invalid, yet the last finite cell
    assert_same_bits((index, value), O.max_batch(g, _along(g)))
    g = _row_grid([np.nan, -FLT_MAX, np.nextafter(np.float32(-FLT_MAX), np.float32(0)), np.nan])
    assert host_max(native, g, _along(g))[0][0, 0] == 1


def test_quirk_start_equals_end(native):
    z = np.arange(200, dtype=np.float32).reshape(10, 20)
    g = O.Grid(z, (0.1, 0.2), 0.1)
    p = O.position(g, 4, 7)
    lines = np.array([[p[0], p[1], p[0], p[1]], [p[0] + 0.01, p[1] - 0.02, p[0] - 0.03, p[1] + 0.04]])
    index, value = host_max(native, g, lines)
    assert index[:, 1:].tolist() == [[4, 7], [4, 7]] and (value[:, 0] == 87.0).all()
    counts, first, rows = host_values(native, g, lines)
    assert counts.tolist() == [1, 1] and first.tolist() == [0, 1] and rows.tolist() == [[p[0], p[1], 87.0]] * 2


# ---- analytic derivatives ----
def test_plane_slopes_are_exact_up_to_rounding(native):
    a, b = 0.3, -0.7
    g = O.Grid(np.zeros((23, 31)), (0.4, -0.9), 0.05)
    r, c = np.meshgrid(np.arange(23), np.arange(31), indexing="ij")
    x = (g.pos[0] + (0.5 * g.len[0] - 0.5 * g.res)) - g.res * r
    y = (g.pos[1] + (0.5 * g.len[1] - 0.5 * g.res)) - g.res * c
    g.data[:] = (a * x + b * y + 1.0).astype(np.float32)
    pos = np.stack([x.ravel(), y.ravel()], 1)
    index, value = host_derivatives(native, g, pos, True)
    assert (index[:, 0] == O.INSIDE).all()
    assert np.abs(value[:, 0] - a).max() < 2e-3 and np.abs(value[:, 1] - b).max() < 2e-3     # float heights ~1e-7
    assert np.abs(value[:, 2:]).max() < 0.2
    assert_same_bits((index, value), O.derivative_batch(g, pos, True))


def test_quadratic_is_exact_inside_and_matches_the_shifted_stencil_at_the_edges(native):
    """z = x^2 + 2 y^2 + x y on integer-valued cells (res 1, exact in float): the 5-tap kernels are exact for
    quadratics, so every cell gives the derivatives at its stencil's centre: its own inside, the shifted centre within
    2 cells of an edge."""
    g = O.Grid(np.zeros((12, 9)), (0.0, 0.0), 1.0)
    r, c = np.meshgrid(np.arange(12), np.arange(9), indexing="ij")
    x = (g.pos[0] + (0.5 * g.len[0] - 0.5)) - r
    y = (g.pos[1] + (0.5 * g.len[1] - 0.5)) - c
    g.data[:] = (x * x + 2 * y * y + x * y).astype(np.float32)
    pos = np.stack([x.ravel(), y.ravel()], 1)
    index, value = host_derivatives(native, g, pos, True)
    rr, cc = r.ravel(), c.ravel()
    sr = rr + np.array([O.kernel_center(i, 12) for i in rr])     # the stencil's centre row / column
    sc = cc + np.array([O.kernel_center(j, 9) for j in cc])
    xs = (g.pos[0] + (0.5 * g.len[0] - 0.5)) - sr
    ys = (g.pos[1] + (0.5 * g.len[1] - 0.5)) - sc
    # gx at (centre row, own column), gy at (own row, centre column)
    yo = (g.pos[1] + (0.5 * g.len[1] - 0.5)) - cc
    xo = (g.pos[0] + (0.5 * g.len[0] - 0.5)) - rr
    assert np.allclose(value[:, 0], 2 * xs + yo, atol=1e-4)
    assert np.allclose(value[:, 1], 4 * ys + xo, atol=1e-4)
    assert np.allclose(value[:, 2], 2.0, atol=1e-4) and np.allclose(value[:, 4], 4.0, atol=1e-4)
    assert np.allclose(value[:, 3], 1.0, atol=1e-4)
    inner = (sr == rr) & (sc == cc)
    assert inner.sum() == 8 * 5 and np.allclose(value[inner, 0], 2 * x.ravel()[inner] + y.ravel()[inner], atol=1e-5)
    assert_same_bits((index, value), O.derivative_batch(g, pos, True))


def test_outside_positions_get_zero_derivatives(native):
    g = O.Grid(np.ones((6, 6)), (0.0, 0.0), 0.1)
    pos = np.array([[0.3, 0.0], [0.0, -0.3], [np.nan, 0.0], [np.inf, 0.0], [0.29999, -0.29999], [-0.3, 0.3]])
    index, value = host_derivatives(native, g, pos, True)
    # the upper bound of an axis is inside, its lower bound outside (0 <= -((v - p) - L / 2) < L)
    assert index[:, 0].tolist() == [0, 1, 1, 1, 0, 1]
    out = index[:, 0] == O.OUTSIDE
    assert (index[out, 1:] == -1).all() and (value[out] == 0).all()
    assert index[0, 1] == 0 and index[4, 1:].tolist() == [0, 5]
    assert_same_bits((index, value), O.derivative_batch(g, pos, True))


# ---- rejections ----
@pytest.mark.parametrize("case", [
    ((0, 5, (0.0, 0.0), 0.1, 1), 1), ((5, 0, (0.0, 0.0), 0.1, 1), 1), ((4, 9, (0.0, 0.0), 0.1, 5), 1),
    ((9, 4, (0.0, 0.0), 0.1, 5), 1), ((5, 5, (0.0, 0.0), 0.1, 5), 0), ((1, 1, (0.0, 0.0), 0.1, 1), 0),
    ((1 << 16, 1 << 15, (0.0, 0.0), 2.0 ** -20, 1), 1), ((65536, 32767, (0.0, 0.0), 2.0 ** -20, 1), 0),
    ((10, 10, (0.0, 0.0), float("nan"), 1), 1), ((10, 10, (0.0, 0.0), 0.0, 1), 1),
    ((10, 10, (0.0, 0.0), 2.0 ** -21, 1), 1), ((10, 10, (0.0, 0.0), 2.0 ** -20, 1), 0),
    ((10, 10, (float("inf"), 0.0), 0.1, 1), 1), ((10, 10, (0.0, float("nan")), 0.1, 1), 1),
    ((10, 10, (2.0 ** 20 - 1.0, 0.0), 0.1, 1), 0), ((10, 10, (2.0 ** 20 - 0.5, 0.0), 0.1, 1), 1),
    ((10, 10, (0.0, -(2.0 ** 20)), 0.1, 1), 1), ((1 << 31, 1, (0.0, 0.0), 2.0 ** -20, 1), 1)])
def test_grid_rejections(native, case):
    (rows, cols, pos, res, min_cells), rejected = case
    p = np.array(pos, np.float64)
    assert native.glh_check_grid(rows, cols, p.ctypes.data, res, min_cells) == rejected


def test_kernels_are_float_divisions(native):
    for res in (0.04, 0.1, 0.05, 2.0 ** -20, 3.7):
        d1, d2 = np.zeros(5, np.float32), np.zeros(5, np.float32)
        native.glh_kernels(res, d1.ctypes.data, d2.ctypes.data)
        w1, w2 = O.kernels(res)
        assert d1.tolist() == w1 and d2.tolist() == w2
