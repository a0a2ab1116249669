"""The map initialiser's oracle (tests/initialize_oracle.py) pinned against SciPy, with no GPU: the triangulation where it
is unique, the gradient estimate, linear / Clough-Tocher evaluation, the rectangle tie, nearest and duplicate points."""
import itertools

import numpy as np
import pytest
from scipy.interpolate import CloughTocher2DInterpolator, griddata
from scipy.spatial import Delaunay

import initialize_oracle as IO

# SciPy's estimate_gradients_2d_global stops at a relative change below 1e-6; the oracle runs the same sweeps, so the
# two differ by rounding only (largest seen on these cases: 1.6e-15 relative).  The bound leaves room for that.
GRAD_REL = 1e-9


def _point_sets():
    rng = np.random.default_rng(7)
    out = []
    for n, span in [(5, 40), (8, 60), (12, 100), (30, 200), (80, 400), (200, 3000)]:
        for _ in range(4):
            idx = rng.integers(-span // 8, span, (n, 2))
            tri = IO.ccw(idx, Delaunay(idx.astype(np.float64)).simplices)
            if IO.unique_triangulation(idx, tri):
                out.append((idx, rng.standard_normal(n)))
    return out


SETS = _point_sets()


def test_enough_unique_sets():
    assert len(SETS) >= 15


@pytest.mark.parametrize("k", range(15))
def test_triangulation_equals_qhull_where_unique(k):
    idx, _ = SETS[k]
    mine = IO.delaunay(idx)
    ref = IO.canonical(IO.ccw(idx, Delaunay(idx.astype(np.float64)).simplices))
    assert [tuple(t) for t in mine] == ref


@pytest.mark.parametrize("k", range(15))
def test_gradients_match_clough_tocher(k):
    idx, z = SETS[k]
    tri = Delaunay(idx.astype(np.float64))
    ref = CloughTocher2DInterpolator(tri, z).grad[:, 0, :]
    mine = IO.estimate_gradients(idx, z, IO.delaunay(idx))
    rel = np.abs(mine - ref).max() / max(np.abs(ref).max(), 1e-300)
    assert rel < GRAD_REL, rel


@pytest.mark.parametrize("k", [0, 4, 9, 14])
@pytest.mark.parametrize("method", ["linear", "cubic"])
def test_evaluation_matches_griddata(k, method):
    """On the same triangles (unique here) and SciPy's gradients, the oracle's values are SciPy's up to rounding;
    with its own triangulation and gradients the cubic stays within the gradient tolerance."""
    idx, z = SETS[k]
    W = int(idx.max()) + 3 if idx.max() < 400 else 400
    g = tuple(np.mgrid[0:W, 0:W])
    ref = griddata(idx.astype(np.float64), z, g, method=method)
    mine = IO.interpolate(W, method, idx, z)
    assert np.array_equal(np.isnan(ref), np.isnan(mine))
    scale = np.abs(z).max()
    tol = 1e-13 * scale if method == "linear" else 1e-6 * scale
    assert np.nanmax(np.abs(mine - ref)) <= tol


def test_rectangle_tie_is_a_delaunay_triangulation():
    """Four feet of a symmetric stance snap to an exact rectangle: two valid triangulations.  The library keeps the one
    the insertion order gives: (0, 1, 2) is placed first and point 3 lies on its circumcircle, so the diagonal 0-2
    stays.  Both triangles are Delaunay (no point strictly inside a circumcircle) and cover the rectangle."""
    for idx in (np.array([[10, 10], [30, 10], [30, 25], [10, 25]]), np.array([[10, 10], [10, 25], [30, 25], [30, 10]]),
                np.array([[30, 25], [10, 10], [30, 10], [10, 25], [20, 17]])):
        tris = IO.delaunay(idx)
        P = [tuple(map(int, p)) for p in idx]
        area = 0
        for t in tris:
            a, b, c = (P[v] for v in t)
            assert IO.orient(a, b, c) > 0
            area += IO.orient(a, b, c)
            for q in P:
                assert IO.incircle(a, b, c, q) <= 0
        assert area == 2 * 20 * 15
    tris = IO.delaunay(np.array([[10, 10], [30, 10], [30, 25], [10, 25]]))
    assert [tuple(t) for t in tris] == [(0, 1, 2), (0, 2, 3)]


def _ties(W, idx):
    gi, gj = np.mgrid[0:W, 0:W]
    d = np.stack([(gi - x) ** 2 + (gj - y) ** 2 for x, y in idx])
    return (d == d.min(0)).sum(0) > 1


@pytest.mark.parametrize("n", [4, 6, 8, 10, 12, 40, 200])
def test_nearest_matches_griddata(n):
    """<= 10 points (SciPy's k-d tree has them in one leaf): every cell, ties included.  More: every cell without a tie."""
    rng = np.random.default_rng(n)
    W = 48
    idx = rng.integers(-4, W + 4, (n, 2))
    z = rng.standard_normal(n)
    ref = griddata(idx.astype(np.float64), z, tuple(np.mgrid[0:W, 0:W]), method="nearest")
    mine = IO.interpolate(W, "nearest", idx, z)
    ties = _ties(W, idx)
    assert ties.sum() > 0
    if n <= 10:
        assert np.array_equal(mine, ref)
    else:
        assert np.array_equal(mine[~ties], ref[~ties])


@pytest.mark.parametrize("method", ["nearest", "linear", "cubic"])
def test_duplicates_resolve_to_the_first(method):
    """A point repeated later with another height resolves to its first occurrence in the oracle's own triangulation
    and, on this set, in SciPy for all three methods; on SciPy's triangles (what initialize_map passes) the oracle is
    SciPy.  Qhull does not promise the first copy in general: on other sets it makes a later copy the vertex."""
    keep = [i for i in range(9) if i not in (6, 8)]
    for seed in range(100):               # a set whose distinct points triangulate uniquely
        rng = np.random.default_rng(seed)
        idx = rng.integers(0, 30, (9, 2))
        idx[6] = idx[1]
        idx[8] = idx[4]
        z = rng.standard_normal(9)
        if IO.unique_triangulation(idx[keep], IO.ccw(idx[keep], Delaunay(idx[keep].astype(np.float64)).simplices)):
            break
    W = 32
    g = tuple(np.mgrid[0:W, 0:W])
    ref = griddata(idx.astype(np.float64), z, g, method=method)
    d = Delaunay(idx.astype(np.float64))
    grad = CloughTocher2DInterpolator(d, z).grad[:, 0, :] if method == "cubic" else None
    mine = IO.interpolate(W, method, idx, z, None if method == "nearest" else d.simplices, grad)
    assert not {6, 8} & set(IO.delaunay(idx).ravel().tolist())
    ref_first = griddata(idx[keep].astype(np.float64), z[keep], g, method=method)
    assert np.array_equal(np.isnan(ref), np.isnan(mine))
    if method == "nearest":
        assert np.array_equal(mine, ref)
        assert np.array_equal(ref, ref_first)
    else:
        assert np.nanmax(np.abs(mine - ref)) <= 1e-13 * np.abs(z).max()
        assert np.nanmax(np.abs(ref - ref_first)) <= 1e-13


def test_collinear_and_degenerate_inputs():
    with pytest.raises(ValueError):
        IO.delaunay(np.array([[0, 0], [1, 1], [2, 2], [5, 5]]))
    with pytest.raises(ValueError):
        IO.delaunay(np.array([[3, 3]] * 5))
    # collinear points before the first non-collinear one sit on the hull
    tris = IO.delaunay(np.array([[0, 0], [2, 0], [4, 0], [6, 0], [3, 5]]))
    assert len(tris) == 3


def test_snap_matches_the_reference_expression():
    rng = np.random.default_rng(0)
    pts = (rng.standard_normal((50, 3)) * 3).astype(np.float32)
    center = np.array([0.37, -1.21, 0.3], np.float32)
    idx, z = IO.snap(pts, center, 0.04, 301)
    ref = ((pts[:, :2] - center[:2].reshape(1, 2)) / np.float32(0.04) + 301 / 2).astype(np.int32)
    assert np.array_equal(idx, ref)
    assert np.array_equal(z, (pts[:, 2] - center[2]).astype(np.float64))


def test_oracle_is_deterministic_under_permuted_cocircular_input():
    """The tie rule depends on input order only: the same points in two orders may give two triangulations, each valid."""
    sq = np.array([[0, 0], [8, 0], [8, 8], [0, 8], [4, 4], [0, 4], [8, 4]])
    for perm in itertools.islice(itertools.permutations(range(len(sq))), 0, 200, 37):
        idx = sq[list(perm)]
        tris = IO.delaunay(idx)
        P = [tuple(map(int, p)) for p in idx]
        assert sum(IO.orient(*(P[v] for v in t)) for t in tris) == 2 * 64
        for t in tris:
            for q in P:
                assert IO.incircle(*(P[v] for v in t), q) <= 0
        assert np.array_equal(tris, IO.delaunay(idx))
