"""initialize_map / emap_initialize_map on the device against SciPy (oracle.initialize_map_planes, griddata) and against
tests/initialize_oracle.py (the library's own triangulation and gradients).

Bar: every plane bit-identical, except cells whose fp64 value lies within 1e-12 of an fp32 rounding boundary (relative
to the larger of the value and the largest input height), which may differ by 1 ulp: the device evaluates the same
interpolant in fp64 with other roundings.  Nearest with more than 10 points: a cell with several nearest points holds
one of their heights (SciPy's k-d tree breaks ties by its own order)."""
import numpy as np
import pytest
from scipy.interpolate import CloughTocher2DInterpolator, griddata
from scipy.ndimage import maximum_filter
from scipy.spatial import Delaunay, cKDTree

import initialize_oracle as IO

pytestmark = pytest.mark.gpu

CENTER = np.array([0.013, -0.027, 0.31], np.float32)       # off the cell grid
REL = 1e-12


def _em(W, k):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(W, dilation_size_initialize=k)
    em = ElevationMap(p)
    em.set_state(_cleared(p), center=CENTER.astype(np.float64))
    return em, p


def _cleared(p):
    st = np.zeros((7, p.cell_n, p.cell_n), np.float32)
    st[1] = np.float32(p.initial_variance)
    return st


def _points(name, W, seed=0):
    """(n, 3) fp32 points in the map frame."""
    res = 0.04
    half = (W - 2) * res / 2
    rng = np.random.default_rng(seed)
    c = CENTER.astype(np.float64)
    if name == "tf":             # the TF initializer: the base and the corners of a square around it, one height
        b = c + [0.2, -0.1, 0.1]
        pts = [b] + [b + [sx * 0.5, sy * 0.5, 0] for sx in (-1, 1) for sy in (-1, 1)]
    elif name == "rect":         # four feet on cell centres: an exact rectangle of cells
        pts = [c + [(i + 0.5) * res, (j + 0.5) * res, h] for (i, j), h in
               zip([(-8, -5), (7, -5), (7, 4), (-8, 4)], (0.05, 0.11, -0.02, 0.08))]
    elif name == "dup12":        # 12 points, two of them repeated later with other heights
        q = c + np.c_[rng.uniform(-half * 0.8, half * 0.8, (12, 2)), rng.normal(0, 0.2, 12)]
        q[7, :2] = q[2, :2]
        q[10, :2] = q[5, :2]
        pts = q
    elif name.startswith("n"):   # seeded random points over the map
        n = int(name[1:])
        pts = c + np.c_[rng.uniform(-half, half, (n, 2)), rng.normal(0, 0.3, n)]
    elif name == "outside":      # partly outside the map
        pts = c + np.c_[rng.uniform(-1.6 * half, 1.6 * half, (30, 2)), rng.normal(0, 0.3, 30)]
    return np.asarray(pts, np.float32)


def _near_boundary(v64, zscale):
    """Cells whose fp64 value lies within REL of an fp32 rounding boundary."""
    v = np.nan_to_num(v64)
    tol = REL * np.maximum(np.abs(v), zscale)
    return (v - tol).astype(np.float32) != (v + tol).astype(np.float32)


def _ulps(a, b):
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def _compare(state, ref, interp64, zscale, k, label, tie_ok=None):
    allowed = maximum_filter(_near_boundary(interp64, zscale), size=2 * k + 3) if k else _near_boundary(interp64, zscale)
    for li in (0, 5):
        a, b = state[li], ref[li]
        bad = a.view(np.int32) != b.view(np.int32)
        if tie_ok is not None:
            bad &= ~tie_ok
        assert not (bad & ~allowed).any(), f"{label} plane {li}: {int((bad & ~allowed).sum())} cells differ"
        assert (_ulps(a, b)[bad] <= 1).all(), f"{label} plane {li}: more than 1 ulp"
    for li in (1, 2, 6):
        assert np.array_equal(state[li], ref[li]), f"{label} plane {li}"
    for li in (3, 4):
        assert not state[li].any(), f"{label} plane {li} is not the cleared plane"


def _tie_cells(W, idx, z, state):
    """(cells with several nearest points, whether each such cell holds one of their heights)."""
    tree = cKDTree(idx.astype(np.float64))
    cells = np.stack(np.mgrid[0:W, 0:W], -1).reshape(-1, 2).astype(np.float64)
    d, j = tree.query(cells, k=min(8, len(idx)))
    tied = d == d[:, :1]
    tie = tied.sum(1) > 1
    heights = np.where(tied, z.astype(np.float32)[np.minimum(j, len(idx) - 1)], np.nan)
    holds = (heights == state[0].reshape(-1, 1)).any(1)
    return tie.reshape(W, W), holds.reshape(W, W)


PY_CASES = [(64, "tf", 2), (64, "rect", 3), (202, "dup12", 2), (301, "rect", 0), (301, "outside", 0),
            (1024, "n200", 0), (1024, "tf", 0), (2048, "n20000", 0), (2048, "dup12", 0)]


@pytest.mark.parametrize("method", ["nearest", "linear", "cubic"])
@pytest.mark.parametrize("W,name,k", PY_CASES)
def test_python_path_matches_scipy(oracle_mod, W, name, k, method):
    em, p = _em(W, k)
    pts = _points(name, W)
    em.initialize_map(pts, method)
    state, _ = em.get_state()
    ref = oracle_mod.initialize_map_planes(p, _cleared(p), pts, CENTER, method)
    idx, z = IO.snap(pts, CENTER, p.resolution, W)
    interp = griddata(idx.astype(np.float64), z, tuple(np.mgrid[0:W, 0:W]), method=method)
    tie_ok = None
    if method == "nearest" and len(pts) > 10:
        tie, holds = _tie_cells(W, idx, z, state)
        assert holds[tie].all(), "a tie cell holds none of its nearest points' heights"
        tie_ok = tie
    _compare(state, ref, interp, np.abs(z).max(), k, f"{W} {name} {method}", tie_ok)
    assert state[2].sum() > 0


C_CASES = [(64, "tf"), (64, "rect"), (202, "dup12"), (202, "n200"), (301, "outside"), (1024, "tf"), (2048, "rect")]


def _c_call(em, pts, method, tris=None, grad=None, k=0, n=None):
    n = len(pts) if n is None else n
    pts = np.ascontiguousarray(pts, np.float32)
    t = None if tris is None else np.ascontiguousarray(tris, np.int32)
    return em._L.emap_initialize_map(em._h, pts.ctypes.data, n, method, None if t is None else t.ctypes.data,
                                     0 if t is None else len(t), None if grad is None else grad.ctypes.data,
                                     float(em.param.initialized_variance), k)


@pytest.mark.parametrize("method", ["linear", "cubic", "nearest"])
@pytest.mark.parametrize("W,name", C_CASES)
def test_c_path_matches_oracle(W, name, method):
    """No triangles, no gradients: the library triangulates and estimates.  Against tests/initialize_oracle.py."""
    em, p = _em(W, 0)
    pts = _points(name, W)
    assert _c_call(em, pts, IO.METHODS[method]) == 0
    state, _ = em.get_state()
    idx, z = IO.snap(pts, CENTER, p.resolution, W)
    interp = IO.interpolate(W, method, idx, z)
    e, v, ok = IO.planes(W, interp, p.initialized_variance, p.initial_variance)
    ref = _cleared(p)
    ref[0], ref[1], ref[2] = e, v, ok
    ref[5] = np.where(ok > 0.5, e, 0).astype(np.float32)
    _compare(state, ref, interp, np.abs(z).max(), 0, f"C {W} {name} {method}")


@pytest.mark.parametrize("method", ["linear", "cubic"])
@pytest.mark.parametrize("W,name", [(202, "n200"), (301, "outside"), (1024, "tf"), (2048, "n200")])
def test_c_path_matches_scipy_where_unique(W, name, method):
    """Where the triangulation is unique (no duplicate and no cocircular points: with duplicates Qhull may make a later
    copy the vertex, the library always the first) the C path is SciPy's interpolant: linear to the rounding-boundary
    rule; cubic within the gradient tolerance carried to heights: |dh| <= 4 * 1e-9 * max|grad| * longest edge + 1e-12 * max|z|
    (SciPy stops its gradient sweeps at a 1e-6 relative change, the library runs the same sweeps, and the ordinates are
    sums of a few gradient-times-edge terms)."""
    em, p = _em(W, 0)
    pts = _points(name, W)
    idx, z = IO.snap(pts, CENTER, p.resolution, W)
    d = Delaunay(idx.astype(np.float64))
    assert IO.unique_triangulation(idx, d.simplices)
    assert _c_call(em, pts, IO.METHODS[method]) == 0
    state, _ = em.get_state()
    interp = griddata(idx.astype(np.float64), z, tuple(np.mgrid[0:W, 0:W]), method=method)
    assert np.array_equal(state[2] > 0.5, ~np.isnan(interp))
    if method == "linear":
        ref = np.nan_to_num(interp).astype(np.float32)
        bad = ref.view(np.int32) != state[0].view(np.int32)
        assert not (bad & ~_near_boundary(interp, np.abs(z).max())).any()
    else:
        grad = CloughTocher2DInterpolator(d, z).grad[:, 0, :]
        tris = IO.ccw(idx, d.simplices)
        P = idx.astype(np.float64)
        L = max(np.hypot(*(P[t[a]] - P[t[b]])) for t in tris for a, b in ((0, 1), (1, 2), (2, 0)))
        bound = 4 * 1e-9 * np.abs(grad).max() * L + 1e-12 * np.abs(z).max()
        ok = ~np.isnan(interp)
        assert np.abs(state[0][ok].astype(np.float64) - interp[ok]).max() <= bound + np.spacing(np.abs(interp[ok]).max(), dtype=np.float32)


def test_rejections_leave_the_map_cleared():
    em, p = _em(64, 2)
    good = _points("tf", 64)
    cleared = _cleared(p)

    def dirty():
        em.initialize_map(good, "linear")
        assert em.get_state()[0][2].sum() > 0

    cases = [
        lambda: em.initialize_map(good[:3], "linear"),                       # <= 3 points
        lambda: em.initialize_map(np.array([[0, 0, 0], [0.1, 0.1, 0], [0.2, 0.2, 0], [0.4, 0.4, 1]], np.float32), "cubic"),
        lambda: em.initialize_map(good, "quintic"),
    ]
    errors = (AssertionError, ValueError, RuntimeError)
    for f in cases:
        dirty()
        with pytest.raises(errors):
            f()
        assert np.array_equal(em.get_state()[0], cleared)
    line = np.array([[0, 0, 0], [0.1, 0.1, 0], [0.2, 0.2, 0], [0.4, 0.4, 1]], np.float32)
    too_many = np.zeros((65537, 3), np.float32)
    bad_c = [
        lambda: _c_call(em, good, 1, n=3),
        lambda: _c_call(em, line, 1),
        lambda: _c_call(em, line, 2),
        lambda: _c_call(em, good, 5),
        lambda: _c_call(em, too_many, 0),
        lambda: _c_call(em, good, 1, tris=np.array([[0, 1, 5]])),
        lambda: _c_call(em, good, 1, tris=np.array([[0, -1, 2]])),
        lambda: _c_call(em, good, 1, tris=np.array([[0, 1, 1]])),      # zero area
    ]
    for f in bad_c:
        dirty()
        assert f() == -1
        assert np.array_equal(em.get_state()[0], cleared)
    dirty()
    assert _c_call(em, line, 0) == 0          # nearest needs no triangle


@pytest.mark.parametrize("method", ["nearest", "linear", "cubic"])
def test_repeatable_and_constant_launches(method):
    counts = []
    for W, name in [(64, "tf"), (2048, "n20000")]:
        em, p = _em(W, 2)
        pts = _points(name, W)
        em.initialize_map(pts, method)
        first, _ = em.get_state()
        before = em.launch_count()
        em.initialize_map(pts, method)
        counts.append(em.launch_count() - before)
        again, _ = em.get_state()
        assert np.array_equal(first.view(np.int32), again.view(np.int32))
    assert counts[0] == counts[1], counts


def test_frame_after_initialize_matches_oracle(oracle_mod):
    from elevation_mapping_cupy_b200 import workloads as wl
    from helpers import check_frame
    em, p = _em(202, 2)
    pts = _points("n200", 202)
    em.initialize_map(pts, "cubic")
    om = oracle_mod.OracleElevationMap(p, nthreads=0)
    om.center = CENTER.copy()
    om.elevation_map = oracle_mod.initialize_map_planes(p, _cleared(p), pts, CENTER, "cubic")
    state, _ = em.get_state()
    for li in (1, 2, 5, 6):
        assert np.array_equal(state[li], om.elevation_map[li])
    if not np.array_equal(state[0], om.elevation_map[0]):       # a rounding-boundary cell: start from the same map
        om.elevation_map[0] = state[0]
        om.elevation_map[5] = state[5]
    cloud, R, t = wl.lidar_cloud(0, 0, n_rings=16, n_az=400, max_range=4.0)
    em.input_pointcloud(cloud, ["x", "y", "z"], R, t, 0.02, 0.02)
    om.input_pointcloud(cloud, ["x", "y", "z"], R, t, 0.02, 0.02)
    check_frame(em, om, len(cloud), "frame after initialize_map")
