"""Map windows without a GPU: the library's host window function (emap_submap_windows, the arithmetic every
emap_get_submaps call runs) against the NumPy restatement (tests/submap_oracle.py), and the restatement's index rule
against the cells' extents."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import submap_oracle as SO          # noqa: E402


def _lib():
    from elevation_mapping_cupy_b200 import _lib
    return _lib.load()


def _windows(cell_n, res, center, reqs):
    L = _lib()
    req = np.ascontiguousarray(np.asarray(reqs, np.float64).reshape(-1, 4))
    c = np.ascontiguousarray(np.asarray(center, np.float64)[:2])
    info = np.full((len(req), 5), -7, np.int32)
    cen = np.full((len(req), 2), -7.0)
    rc = L.emap_submap_windows(cell_n, res, c.ctypes.data, len(req), req.ctypes.data, info.ctypes.data, cen.ctypes.data)
    return rc, info, cen


def _requests(cell_n, res, center, rng):
    """Centred, edge-clipped, corner, half-map, whole-map, larger-than-map, zero-length, on-boundary and outside requests,
    and random ones."""
    half = 0.5 * (cell_n - 2) * res
    cx, cy = center[:2]
    out = [(cx, cy, 2.0, 2.0), (cx, cy, 0.0, 0.0), (cx, cy, 2 * half, 2 * half), (cx, cy, 1e9, 1e9),
           (cx, cy, half, 0.0), (cx, cy, 0.0, half), (cx + 0.3, cy - 0.7, 1.0, 0.5)]
    for sx in (-1, 1):
        for sy in (-1, 1):
            out.append((cx + sx * (half - 0.5 * res), cy + sy * (half - 0.5 * res), 2.0, 2.0))     # corners
            out.append((cx + sx * (half - 0.3), cy, 2.0, 0.5))                                      # edges
            out.append((cx, cy + sy * (half - 0.3), 0.5, 2.0))
            out.append((cx + sx * half * 1.01, cy + sy * 0.1, 2.0, 2.0))                            # outside
            out.append((cx + sx * 0.2, cy + sy * half * 1.5, 0.0, 0.0))
    for k in range(-4, 5):                                                    # on cell boundaries
        b = cx + k * res + (0.0 if cell_n % 2 == 0 else 0.5 * res)
        out.append((b, cy, 2 * res, 0.0))
        out.append((b - res, cy + k * res, 4 * res, 3 * res))
    for _ in range(200):
        p = rng.uniform(-1.1 * half, 1.1 * half, 2)
        ln = rng.choice([0.0, 0.5, 2.0, 2 * half], 2) * rng.uniform(0.5, 1.0, 2)
        out.append((cx + p[0], cy + p[1], ln[0], ln[1]))
    out.append((np.nan, cy, 1.0, 1.0))
    out.append((cx, np.inf, 1.0, 1.0))
    return out


@pytest.mark.parametrize("cell_n,res,center", [(202, 0.04, (0.0, 0.0)), (203, 0.04, (0.0, 0.0)),
                                               (1024, 0.04, (12.34, -5.678)), (131, 0.1, (-3.21, 7.0)),
                                               (2048, 0.04, (0.02, -0.06))])
def test_host_window_matches_oracle(cell_n, res, center):
    """Every request of a map of odd and even cell_n, at the origin and moved, against SO.window: info exactly, centre
    bit for bit."""
    c = np.asarray(center, np.float32).astype(np.float64)            # the engine's centre is fp32
    reqs = _requests(cell_n, res, c, np.random.default_rng(cell_n))
    rc, info, cen = _windows(cell_n, res, c, reqs)
    assert rc == 0
    n_ok = n_clip = 0
    for w, r in enumerate(reqs):
        want, wc = SO.window(cell_n, res, c, np.asarray(r, np.float64))
        assert tuple(info[w]) == want, (w, r, info[w], want)
        assert np.array_equal(cen[w], np.asarray(wc), equal_nan=True), (w, r, cen[w], wc)
        ok, r0, c0, rows, cols = want
        if ok:
            n_ok += 1
            assert 0 <= r0 and r0 + rows <= cell_n - 2 and 0 <= c0 and c0 + cols <= cell_n - 2 and rows >= 1 and cols >= 1
            n_clip += r0 == 0 or c0 == 0 or r0 + rows == cell_n - 2 or c0 + cols == cell_n - 2
    assert n_ok > 100 and n_clip > 20


def test_fixed_windows():
    """A few windows worked out by hand on a 10 x 10 exported map (cell_n 12) of 1 m cells centred at the origin:
    state cell i covers [i - 6, i - 5), output index 10 - i."""
    cases = {(0.0, 0.0, 0.0, 0.0): ((1, 4, 4, 1, 1), (0.5, 0.5)),         # x = 0 is the lower edge of state cell 6
             (-0.5, -0.5, 0.0, 0.0): ((1, 5, 5, 1, 1), (-0.5, -0.5)),
             (0.0, 0.0, 2.0, 2.0): ((1, 3, 3, 3, 3), (0.5, 0.5)),         # [-1, 1] meets cells 5, 6 and 7
             (0.5, 0.5, 2.0, 1.0): ((1, 3, 3, 3, 2), (0.5, 1.0)),         # y: [0, 1] meets cells 6 and 7
             (4.5, -4.5, 3.0, 3.0): ((1, 0, 7, 2, 3), (4.0, -3.5)),       # corner: x clipped to 2 cells, y to 3
             (0.0, 0.0, 100.0, 100.0): ((1, 0, 0, 10, 10), (0.0, 0.0)),
             (5.0, 0.0, 1.0, 1.0): ((0, 0, 0, 0, 0), (np.nan, np.nan)),    # x = 5 is the upper edge of the map
             (-5.0, 0.0, 1.0, 1.0): ((1, 9, 4, 1, 2), (-4.5, 0.0))}        # x = -5 is its lower edge
    rc, info, cen = _windows(12, 1.0, (0.0, 0.0), list(cases))
    assert rc == 0
    for w, (want, wc) in enumerate(cases.values()):
        assert tuple(info[w]) == want, (list(cases)[w], info[w])
        assert np.array_equal(cen[w], np.asarray(wc), equal_nan=True), (list(cases)[w], cen[w])


@pytest.mark.parametrize("cell_n", [12, 13, 130, 131])
def test_index_rule_matches_cell_extents(cell_n):
    """The index rule is the half-open extent rule: at a binary resolution and centre, with positions and lengths on
    and between cell boundaries, SO.window and SO.window_cells agree, and so does the library."""
    res, center = 0.25, (1.5, -0.75)
    half = 0.5 * (cell_n - 2) * res
    q = np.arange(-half - 2 * res, half + 2 * res, 0.5 * res)            # every boundary and every cell centre
    rng = np.random.default_rng(cell_n)
    reqs = []
    for _ in range(600):
        x, y = rng.choice(q, 2)
        lx, ly = rng.choice(np.arange(0, 12) * 0.5 * res, 2)
        reqs.append((center[0] + x, center[1] + y, lx, ly))
    rc, info, _ = _windows(cell_n, res, center, reqs)
    assert rc == 0
    n_ok = 0
    for w, r in enumerate(reqs):
        want = SO.window_cells(cell_n, res, center, r)
        assert SO.window(cell_n, res, center, np.asarray(r))[0] == want, r
        assert tuple(info[w]) == want, r
        n_ok += want[0]
    assert n_ok > 200


def test_host_window_rejections():
    L = _lib()
    req = np.array([[0.0, 0.0, 1.0, 1.0]])
    c = np.zeros(2)
    info = np.zeros(5, np.int32)
    cen = np.zeros(2)
    p = lambda a: a.ctypes.data
    assert L.emap_submap_windows(202, 0.04, p(c), 1, p(req), p(info), p(cen)) == 0
    for bad in (-1.0, -1e-300, np.nan, np.inf, -np.inf):
        for a in (2, 3):
            r = req.copy()
            r[0, a] = bad
            assert L.emap_submap_windows(202, 0.04, p(c), 1, p(r), p(info), p(cen)) == -1, (a, bad)
    assert L.emap_submap_windows(202, 0.04, None, 1, p(req), p(info), p(cen)) == -1
    assert L.emap_submap_windows(202, 0.04, p(c), 1, None, p(info), p(cen)) == -1
    assert L.emap_submap_windows(202, 0.04, p(c), 1, p(req), None, p(cen)) == -1
    assert L.emap_submap_windows(202, 0.04, p(c), 1, p(req), p(info), None) == -1
    assert L.emap_submap_windows(2, 0.04, p(c), 1, p(req), p(info), p(cen)) == -1
    for res in (0.0, -0.04, np.nan, np.inf):
        assert L.emap_submap_windows(202, res, p(c), 1, p(req), p(info), p(cen)) == -1
    assert L.emap_submap_windows(202, 0.04, p(c), -1, p(req), p(info), p(cen)) == -1
    assert L.emap_get_submaps(None, 1, p(req), 1, None, None, None, p(cen), 0, 2, p(info), p(cen)) == -1
