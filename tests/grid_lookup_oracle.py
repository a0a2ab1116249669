"""Sequential restatement of the grid lookups (emap_max_values_between, emap_values_between, emap_grid_derivatives) in
Python floats, with every float operation rounded to float32 explicitly.  It follows grid_map_filters_rsl's lookup.cpp
and GridMapDerivative.cpp line by line, over a stepping restatement of grid_map's LineIterator (the numerator loop,
not the closed form the library uses) and grid_map's index arithmetic as include/emap.h states it.

A float32 product or sum computed in double and then rounded to float32 is the correctly rounded float32 result (53 >=
2 * 24 + 2), so f32(a * b) and f32(a + b) are the float operations."""
import math

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)
MARGIN = 1e-6
INSIDE, OUTSIDE = 0, 1


def f32(x):
    return float(np.float32(x))


class Grid:
    """One layer (rows, cols) float32, row-major, grid_map index (r, c); position = the centre of the cells."""

    def __init__(self, data, position, resolution):
        self.data = np.ascontiguousarray(data, np.float32)
        self.rows, self.cols = self.data.shape
        self.n = (self.rows, self.cols)
        self.pos = (float(position[0]), float(position[1]))
        self.res = float(resolution)
        self.len = (self.rows * self.res, self.cols * self.res)

    def at(self, r, c):
        return float(self.data[r, c])


def axis_index(g, v, a):
    """checkIfPositionWithinMap and getIndexFromPosition on axis a: the index, or None outside."""
    o = 0.5 * g.len[a]
    u = -((v - g.pos[a]) - o)
    if not (u >= 0.0 and u < g.len[a]):
        return None
    i = int(-(((v - o) - g.pos[a]) / g.res))          # int() truncates, as the cast to int does
    return min(max(i, 0), g.n[a] - 1)


def index(g, p):
    r, c = axis_index(g, p[0], 0), axis_index(g, p[1], 1)
    return None if r is None or c is None else (r, c)


def position(g, r, c):
    """getPositionFromIndex."""
    return ((g.pos[0] + (0.5 * g.len[0] - 0.5 * g.res)) - g.res * r,
            (g.pos[1] + (0.5 * g.len[1] - 0.5 * g.res)) - g.res * c)


def _fmin(a, b):
    return b if math.isnan(a) else a if math.isnan(b) else (a if a < b else b)


def _fmax(a, b):
    return b if math.isnan(a) else a if math.isnan(b) else (a if a > b else b)


def project(g, p, margin=MARGIN):
    """projectToMapWithMargin."""
    hx, hy = g.len[0] * 0.5, g.len[1] * 0.5
    m = max(margin, 0.0)
    m = min(m, hx)
    m = min(m, hy)
    max_x, min_x = (g.pos[0] + hx) - m, (g.pos[0] - hx) + m
    max_y, min_y = (g.pos[1] + hy) - m, (g.pos[1] - hy) + m
    x, y = _fmin(p[0], max_x), _fmin(p[1], max_y)
    return _fmax(x, min_x), _fmax(y, min_y)


def line_cells(start, end):
    """grid_map's LineIterator from index `start` to index `end`, stepping: initializeIterationParameters and ++."""
    delta = (abs(end[0] - start[0]), abs(end[1] - start[1]))
    inc1 = [1 if end[0] >= start[0] else -1, 1 if end[1] >= start[1] else -1]
    inc2 = list(inc1)
    if delta[0] >= delta[1]:
        inc1[0], inc2[1] = 0, 0
        den, num, add, n = delta[0], delta[0] // 2, delta[1], delta[0] + 1
    else:
        inc2[0], inc1[1] = 0, 0
        den, num, add, n = delta[1], delta[1] // 2, delta[0], delta[1] + 1
    idx = list(start)
    cells = []
    for _ in range(n):
        cells.append((idx[0], idx[1]))
        num += add
        if num >= den:
            num -= den
            idx[0] += inc1[0]
            idx[1] += inc1[1]
        idx[0] += inc2[0]
        idx[1] += inc2[1]
    return cells


def line(g, start, end):
    """The cells of LineIterator(map, projected start, projected end).  getIndexLimitedToMapRange's stepping loop
    only runs for an end outside the map; include/emap.h shows a projected end never is, and this asserts it."""
    s, e = index(g, project(g, start)), index(g, project(g, end))
    assert s is not None and e is not None, "a projected end is outside the map"
    return line_cells(s, e)


def max_value_between(g, start, end):
    """maxValueBetweenLocations: (valid, value, (row, col) of maxIndex, position)."""
    value = -FLT_MAX
    max_index = (0, 0)
    for r, c in line(g, start, end):
        v = g.at(r, c)
        if math.isfinite(v):
            value = v if value < v else value           # std::max(value, v)
            max_index = (r, c)
    return value > -FLT_MAX, value, max_index, position(g, *max_index)


def values_between(g, start, end):
    """valuesBetweenLocations: [(x, y, value)] for the finite cells in iterator order."""
    out = []
    for r, c in line(g, start, end):
        v = g.at(r, c)
        if math.isfinite(v):
            out.append(position(g, r, c) + (v,))
    return out


def kernels(res):
    """GridMapDerivative::initialize(float(res)): float literals divided in float."""
    r = f32(res)
    r2 = f32(r * r)
    d1 = [f32(f32(c) / r) for c in (-1.0 / 12.0, 2.0 / 3.0, 0.0, -2.0 / 3.0, 1.0 / 12.0)]
    d2 = [f32(f32(c) / r2) for c in (-1.0 / 12.0, 4.0 / 3.0, -5.0 / 2.0, 4.0 / 3.0, -1.0 / 12.0)]
    return d1, d2


def dot_contiguous(k, x):
    """Eigen's dot with a contiguous 5-vector on SSE: ((p0 + p2) + (p1 + p3)) + p4."""
    p = [f32(a * b) for a, b in zip(k, x)]
    return f32(f32(f32(p[0] + p[2]) + f32(p[1] + p[3])) + p[4])


def dot_strided(k, x):
    """... with a strided 5-vector (unrolled halving): (p0 + p1) + (p2 + (p3 + p4))."""
    p = [f32(a * b) for a, b in zip(k, x)]
    return f32(f32(p[0] + p[1]) + f32(p[2] + f32(p[3] + p[4])))


def kernel_center(i, n, max_id=2):
    """getKernelCenter on one axis."""
    return -min(i - max_id, 0) - max(i + max_id - (n - 1), 0)


def derivative(g, p, curvature=False):
    """(status, row, col, [gx, gy] or [gx, gy, cxx, cxy, cyy]); outside: zeros."""
    idx = index(g, p)
    nv = 5 if curvature else 2
    if idx is None:
        return OUTSIDE, -1, -1, [0.0] * nv
    r, c = idx
    d1, d2 = kernels(g.res)
    r0, c0 = r - 2 + kernel_center(r, g.rows), c - 2 + kernel_center(c, g.cols)
    col = [g.at(r0 + k, c) for k in range(5)]
    row = [g.at(r, c0 + k) for k in range(5)]
    v = [dot_contiguous(d1, col), dot_strided(d1, row)]
    if curvature:
        gy = [dot_contiguous(d1, [g.at(r0 + k, c0 + j) for k in range(5)]) for j in range(5)]
        v += [dot_contiguous(d2, col), dot_contiguous(d1, gy), dot_strided(d2, row)]
    return INSIDE, r, c, [x if x == x else math.nan for x in v]        # NaN written as 0x7ff8000000000000


# ---- batches, laid out as the calls write them ----
def max_batch(g, lines):
    index = np.zeros((len(lines), 3), np.int32)
    value = np.zeros((len(lines), 3))
    with np.errstate(all="ignore"):
        for q, (x0, y0, x1, y1) in enumerate(np.asarray(lines, np.float64).tolist()):
            ok, v, (r, c), (x, y) = max_value_between(g, (x0, y0), (x1, y1))
            index[q] = (ok, r, c)
            value[q] = (v, x, y)
    return index, value


def values_batch(g, lines):
    counts = np.zeros(len(lines), np.int32)
    first = np.zeros(len(lines), np.int64)
    rows = []
    for q, (x0, y0, x1, y1) in enumerate(np.asarray(lines, np.float64).tolist()):
        first[q] = len(rows)
        got = values_between(g, (x0, y0), (x1, y1))
        counts[q] = len(got)
        rows += got
    return counts, first, np.array(rows, np.float64).reshape(-1, 3)


def derivative_batch(g, positions, curvature=False):
    nv = 5 if curvature else 2
    index = np.zeros((len(positions), 3), np.int32)
    value = np.zeros((len(positions), nv))
    with np.errstate(all="ignore"):
        for q, (x, y) in enumerate(np.asarray(positions, np.float64).tolist()):
            s, r, c, v = derivative(g, (x, y), curvature)
            index[q] = (s, r, c)
            value[q] = v
    return index, value


def random_lines(g, n, seed, lo=0.5, hi=3.0, outside=0.1):
    """n lines of length lo .. hi metres with random starts over the map and `outside` of its length around it."""
    rng = np.random.default_rng(seed)
    s = np.stack([g.pos[a] + (rng.random(n) - 0.5) * g.len[a] * (1.0 + outside) for a in (0, 1)], 1)
    ang = rng.random(n) * 2 * math.pi
    ln = lo + (hi - lo) * rng.random(n)
    return np.concatenate([s, s + np.stack([np.cos(ang), np.sin(ang)], 1) * ln[:, None]], 1)


def edge_lines(g):
    """Lines along and across every edge and between the corners, and ones from far outside, NaN and inf."""
    hx, hy = 0.5 * g.len[0], 0.5 * g.len[1]
    px, py = g.pos
    corners = [(px + sx * hx, py + sy * hy) for sx in (1, -1) for sy in (1, -1)]
    out = []
    for a in corners:
        for b in corners:
            out.append(a + b)
    nan, inf = float("nan"), float("inf")
    out += [(px + hx, py - hy, px + hx, py + hy), (px - hx, py - hy, px - hx, py + hy),
            (px - hx, py + hy, px + hx, py + hy), (px - hx, py - hy, px + hx, py - hy),
            (1e6, 1e6, 2e6, 2e6), (-1e6, 3.0, 1e6, -3.0), (nan, nan, px, py), (px, py, nan, 0.0),
            (inf, -inf, -inf, inf), (px, py, px, py), (px + hx + 5, py, px - hx - 5, py + 0.3)]
    return np.array(out, np.float64)


def random_positions(g, n, seed, outside=0.05):
    rng = np.random.default_rng(seed)
    p = np.stack([g.pos[a] + (rng.random(n) - 0.5) * g.len[a] * (1.0 + outside) for a in (0, 1)], 1)
    # every edge and corner cell's centre, and the exact map bounds
    r = np.arange(g.rows)
    c = np.arange(g.cols)
    xs = (g.pos[0] + (0.5 * g.len[0] - 0.5 * g.res)) - g.res * r
    ys = (g.pos[1] + (0.5 * g.len[1] - 0.5 * g.res)) - g.res * c
    edge = [(x, ys[j]) for x in xs for j in (0, 1, -2, -1)] + [(xs[i], y) for y in ys for i in (0, 1, -2, -1)]
    hx, hy = 0.5 * g.len[0], 0.5 * g.len[1]
    bounds = [(g.pos[0] + sx * hx, g.pos[1] + sy * hy) for sx in (1, -1, 0) for sy in (1, -1, 0)]
    return np.concatenate([p, np.array(edge + bounds + [(float("nan"), 0.0)], np.float64)])
