"""NumPy restatement of the map windows of emap_get_submaps / ElevationMap.get_submaps (the get_raw_submap service).

  * `window`       -- the window of one request, as include/emap.h states the rule: EM.py's cell index in double,
                      floor((p - center) / resolution + cell_n / 2), for the position and for position +- length / 2,
                      the corners clipped to the exported area, output index cell_n - 2 - state index.
  * `window_cells` -- the same window found from the cells' extents instead: every exported row (column) whose half-open
                      interval [lower edge, upper edge) meets the closed interval [position - length / 2,
                      position + length / 2].  Exact where the coordinates are (binary resolutions), which pins the
                      boundary rule independently of the index formula.
  * `crop`         -- the window's cells of a full get_maps_with_names_ref export.
"""
import numpy as np

FAIL = ((0, 0, 0, 0, 0), (np.nan, np.nan))


def _index(p, m, res, cell_n):
    return np.floor((np.float64(p) - np.float64(m)) / np.float64(res) + 0.5 * cell_n)


def window(cell_n, res, center, req):
    """((success, row0, col0, rows, cols), (centre_x, centre_y)) of req = (x, y, length_x, length_y)."""
    m = np.asarray(center, np.float64)[:2]
    for a in range(2):
        i = _index(req[a], m[a], res, cell_n)
        if not (1 <= i <= cell_n - 2):
            return FAIL
    info, centre = [1, 0, 0, 0, 0], [0.0, 0.0]
    for a in range(2):
        half = 0.5 * np.float64(req[2 + a])
        top = int(min(max(_index(req[a] + half, m[a], res, cell_n), 1.0), cell_n - 2.0))
        bot = int(min(max(_index(req[a] - half, m[a], res, cell_n), 1.0), cell_n - 2.0))
        info[1 + a] = cell_n - 2 - top
        info[3 + a] = top - bot + 1
        centre[a] = m[a] + (0.5 * (top + bot + 1) - 0.5 * cell_n) * res
    return tuple(info), tuple(centre)


def window_cells(cell_n, res, center, req):
    """(success, row0, col0, rows, cols) from the cells' extents (output index k <-> state cell cell_n - 2 - k, whose
    extent on its axis is [center + (i - cell_n / 2) * res, center + (i + 1 - cell_n / 2) * res))."""
    out = [1, 0, 0, 0, 0]
    for a in range(2):
        i = np.arange(1, cell_n - 1, dtype=np.float64)
        lo = center[a] + (i - 0.5 * cell_n) * res
        hi = center[a] + (i + 1 - 0.5 * cell_n) * res
        p, half = req[a], 0.5 * req[2 + a]
        if not ((lo <= p) & (p < hi)).any():
            return (0, 0, 0, 0, 0)
        hit = (lo <= p + half) & (hi > p - half)
        k = cell_n - 2 - i[hit].astype(int)
        out[1 + a], out[3 + a] = int(k.min()), int(k.max() - k.min() + 1)
    return tuple(out)


def crop(full, info):
    """(n_layers, rows, cols) cells of a (n_layers, cell_n - 2, cell_n - 2) export for a window's info."""
    ok, r0, c0, rows, cols = (int(v) for v in info)
    return full[:, r0:r0 + rows, c0:c0 + cols]
