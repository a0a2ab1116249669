"""The map point cloud, normal arrows and normal colour without a GPU: the NumPy restatement (tests/map_points_oracle.py)
on small hand-built maps whose answers are written out here, and its geometry against the library's host window
function (emap_submap_windows), which the submap tests already pin."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import map_points_oracle as MO      # noqa: E402

NAN = np.nan
F = np.float32


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


# a 3 x 3 exported map (cell_n 5) at 0.5 m, centred at (1.0, -2.0): rows are x = 1.5, 1.0, 0.5, columns y = -1.5, -2.0, -2.5
ELEV = np.array([[0.1, NAN, 0.3],
                 [NAN, 0.5, 0.6],
                 [0.7, 0.8, NAN]], np.float32)
RES, CENTRE = 0.5, (1.0, -2.0)


def test_positions_of_a_small_map():
    x, y = MO.positions(3, RES, CENTRE)
    assert x.tolist() == [1.5, 1.0, 0.5] and y.tolist() == [-1.5, -2.0, -2.5]
    x, y = MO.positions(4, 0.1, (0.3, 0.0))               # the fp32 centre, widened: 0.30000001192092896
    half = 0.5 * (4 * 0.1) - 0.5 * 0.1                     # 0.15000000000000002 in double
    assert x[0] == (float(np.float32(0.3)) + half) - 0.0
    assert x[3] == (float(np.float32(0.3)) + half) - 0.1 * 3
    assert y.tolist() == [(0.0 + half) - 0.1 * k for k in range(4)]


def test_points_are_column_major_and_skip_nan():
    pts = MO.map_points(ELEV, RES, CENTRE)
    want = np.array([[1.5, -1.5, 0.1], [0.5, -1.5, 0.7],                  # column 0: rows 0, 2
                     [1.0, -2.0, 0.5], [0.5, -2.0, 0.8],                  # column 1: rows 1, 2
                     [1.5, -2.5, 0.3], [1.0, -2.5, 0.6]], np.float32)     # column 2: rows 0, 1
    assert pts.dtype == np.float32 and np.array_equal(_bits(pts), _bits(want))


def test_all_invalid_map_has_no_points_and_no_arrows():
    e = np.full((4, 4), np.nan, np.float32)
    n = np.zeros((4, 4), np.float32)
    assert MO.map_points(e, 0.1, (0, 0)).shape == (0, 3)
    ids, seg = MO.normal_arrows(e, n, n, n + 1, 0.1, (0, 0))
    assert ids.shape == (0,) and seg.shape == (0, 6)


def test_arrows_threshold_order_ids_and_values():
    e = np.array([[1.0, 2.0], [3.0, 4.0]], np.float32)
    t = np.float32(0.1)
    below = np.nextafter(t, np.float32(0))                 # 0.099999994: shorter than 0.1
    nx = np.array([[t, 0.0], [F(0.06), NAN]], np.float32)
    ny = np.array([[0.0, 0.0], [F(0.08), 0.0]], np.float32)
    nz = np.array([[0.0, below], [0.0, 0.0]], np.float32)
    # (0, 0): |n| = 0.10000000149 (kept); (1, 0): sqrt(0.06f^2 + 0.08f^2) = 0.0999999978 (skipped);
    # (0, 1): 0.099999994 (skipped); (1, 1): NaN, which the reference's `norm() < 0.1` skip test keeps
    ids, seg = MO.normal_arrows(e, nx, ny, nz, 1.0, (0.0, 0.0))
    assert ids.tolist() == [0, 3]                          # linear index c * 2 + r: (0, 0) and (1, 1)
    x, y = MO.positions(2, 1.0, (0.0, 0.0))                # x = 0.5, -0.5; y = 0.5, -0.5
    assert seg[0].tolist() == [0.5, 0.5, 1.0, 0.5 + float(t) * 0.1, 0.5 + 0.0, 1.0 + 0.0]
    assert seg[1][:3].tolist() == [-0.5, -0.5, 4.0] and np.isnan(seg[1][3]) and seg[1][4:].tolist() == [-0.5, 4.0]


def test_arrow_start_is_the_point_before_rounding():
    e = np.array([[0.25, 0.5, 0.75]] * 3, np.float32)
    n = np.zeros((3, 3), np.float32)
    ids, seg = MO.normal_arrows(e, n, n, n + 1, 0.1, (0.3, -0.7))
    pts = MO.map_points(e, 0.1, (0.3, -0.7))
    assert ids.tolist() == list(range(9))
    assert np.array_equal(_bits(seg[:, :3].astype(np.float32)), _bits(pts))
    assert np.array_equal(seg[:, 5], seg[:, 2] + 0.1)


@pytest.mark.parametrize("n,want", [
    ((1.0, 1.0, 1.0), 0xFFFFFF),
    ((-1.0, -1.0, 0.0), 0x000000),
    ((0.0, 0.0, 0.5), 0x7F7F7F),                           # 127.5 truncates to 127
    ((0.6, -0.2, 0.8), 0xCC66CC),                          # 204, 102, 204
    # cx = 0.0039215684f, cx * 255 = 0.99999994f truncates to 0; cy * 255 = 128.0f; nz * 255 = 1.0f
    ((np.float32(2 / 255) - np.float32(1), np.float32(1 / 255), np.float32(1 / 255)), 0x008001),
    ((NAN, 0.0, 1.0), 0x007FFF),                           # a NaN channel is 0
    ((0.0, 0.0, -1 / 255), 0xFFFFFFFF),                    # b = -1: its two's complement fills the word
    ((np.inf, 0.0, 0.0), 0xFFFF7F00),                      # saturated to 2^31 - 1, shifted by 16
])
def test_normal_color_channels(n, want):
    got = MO.normal_color(*[np.array([v], np.float32) for v in n])
    assert int(_bits(got)[0]) == want


def test_points_lie_in_their_cells_by_the_submap_rule():
    """Every point's (x, y) lies in exported cell (r, c) by emap_submap_windows' index rule (a zero-length window there
    is that one cell), for odd and even cell_n and off-grid centres."""
    from elevation_mapping_cupy_b200 import _lib
    L = _lib.load()
    rng = np.random.default_rng(0)
    for cell_n, res, centre in ((12, 0.04, (0.0, 0.0)), (13, 0.1, (12.34, -5.678)), (66, 0.04, (0.37, -0.53))):
        n = cell_n - 2
        e = rng.normal(0, 1, (n, n)).astype(np.float32)
        e[rng.random((n, n)) < 0.3] = np.nan
        pts = MO.map_points(e, res, centre)
        rc_ = np.argwhere(np.isfinite(e.T))[:, ::-1]        # (r, c) in column-major order
        req = np.zeros((len(pts), 4), np.float64)
        req[:, :2] = pts[:, :2]
        info = np.zeros((len(pts), 5), np.int32)
        cen = np.zeros((len(pts), 2), np.float64)
        c = np.asarray(centre, np.float32).astype(np.float64)
        assert L.emap_submap_windows(cell_n, res, c.ctypes.data, len(req), req.ctypes.data, info.ctypes.data,
                                     cen.ctypes.data) == 0
        assert (info[:, 0] == 1).all() and (info[:, 3:] == 1).all()
        assert np.array_equal(info[:, 1:3], rc_), cell_n
