"""NumPy restatement of emap_plane_decomposition's resampling (include/emap.h, csrc/emap_resample.cuh), bit for bit, and
the composed oracle of the whole call: plane_segmentation_oracle's fill and median, the resampling, then the
segmentation, planar_regions_oracle.extract and planar_terrain_oracle.postprocess at the resampled resolution and
origin.  geometry() is grid_map_filters_rsl's inpainting::resample arithmetic (inpainting.cpp:244-288) written out on
its own, so that the library's emap_plane_grid_geometry can be held to it."""
import copy

import numpy as np

import planar_terrain_oracle as TO
import plane_segmentation_oracle as PO

F32 = np.float32

# include/emap.h
RESAMPLE_ULPS = 13


def resample_ulps_line(n):
    """EMAP_RESAMPLE_ULPS_LINE(n): the bound for a source of one row or column of n cells."""
    return 2 * n + 6


def geometry(rows, cols, res, new_res):
    """(rows', cols', res'): inpainting::resample's new size and true resolution; unchanged for new_res <= 0 or within
    1e-6 of res (GridMapPreprocessing::changeResolution)."""
    if not new_res > 0.0 or abs(res - new_res) < 1e-6:
        return rows, cols, res
    scaling = res / new_res
    r, c = int(rows * scaling), int(cols * scaling)
    if r == 0 or c == 0:
        return r, c, 0.0
    return r, c, 0.5 * ((rows * res) / r + (cols * res) / c)


def _axis(n, m):
    d = np.arange(m, dtype=np.float64)
    f = (d + 0.5) * (float(n) / float(m)) - 0.5
    s = np.floor(f)
    f = f - s
    edge = (s < 0) | (s >= n - 1)
    s0 = np.clip(s, 0, n - 1).astype(np.int64)
    s1 = np.where(edge, s0, s0 + 1)
    return s0, s1, np.where(edge, 0.0, f).astype(F32), edge


def _pass(a, b, f, edge):
    with np.errstate(invalid="ignore", over="ignore"):
        v = (a + (f * (b - a).astype(F32)).astype(F32)).astype(F32)
    return np.where(edge, a, v).astype(F32)


def resample(img, rows, cols):
    """The library's resampling of img (R, C) float32 to (rows, cols): columns, then rows; see include/emap.h."""
    img = np.asarray(img, F32)
    R, C = img.shape
    s0, s1, f, e = _axis(C, cols)
    h = _pass(img[:, s0], img[:, s1], f[None, :], e[None, :])
    s0, s1, f, e = _axis(R, rows)
    return _pass(h[s0], h[s1], f[:, None], e[:, None])


def ulps(a, b, scale):
    """The largest difference of two float32 arrays in ulps of `scale`; NaN and infinite cells must agree."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    inf = np.isinf(a)
    assert np.array_equal(inf, np.isinf(b)) and np.array_equal(a[inf], b[inf])
    ok = np.isfinite(a)
    d = np.abs(a[ok].astype(np.float64) - b[ok].astype(np.float64)).max(initial=0.0)
    return float(d / np.spacing(F32(abs(scale))))


def decompose(grid, res, centre, p):
    """The composed oracle of emap_plane_decomposition on `grid` (float32, NaN = missing) of resolution res whose cells
    are centred at `centre`, with PlaneSegmentationParams p.  Returns the resampled geometry ("size", "resolution",
    "origin"), the preprocessed "elevation", segment()'s result ("seg") and postprocess()'s layers ("post")."""
    grid = np.asarray(grid, F32)
    img = PO.median(PO.fill_min_values(grid), p.median_kernel, p.median_repeats)
    rows, cols, res2 = geometry(grid.shape[0], grid.shape[1], res, p.resolution)
    if (rows, cols) != img.shape:
        img = resample(img, rows, cols)
    origin = np.asarray(centre, np.float64) + (0.5 * (np.array([rows, cols]) * res2) - 0.5 * res2)
    q = copy.copy(p)
    q.median_repeats = 0                      # the median already ran, before the resampling
    seg = PO.segment(img, res2, origin, q)
    out = {"size": (rows, cols), "resolution": res2, "origin": origin, "elevation": img, "seg": seg}
    if seg["success"]:
        out["post"] = TO.postprocess(seg["elevation"], seg["classification"], res2, p)
    return out
