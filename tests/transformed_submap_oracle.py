"""NumPy restatement of emap_get_transformed_submaps / ElevationMap.get_transformed_submaps (include/emap.h): the node's
get_raw_submap in a requester's frame, grid_map's GridMap::getTransformedMap on the map-frame window.  Restated from
grid_map's published source; not checked against a grid_map build.  Every operation is one IEEE double operation
(Python floats and NumPy element-wise arithmetic round each one; nothing is fused).

  * `geometry`   -- the map-frame window (tests/submap_oracle.py) at T^-1 * position and the new map around it.
  * `sequential` -- the literal scatter loop, cell by cell and sample by sample, on the window's exported layers.
  * `parallel`   -- the same result from the order-free rule the device uses: per target M = max fp32(z), winner the
                    last sample with z >= M, else the first with fp32(z) = M.
"""
import math

import numpy as np

import submap_oracle as SO


def flat(T):
    """The 12 doubles (R row-major, then t) of T given as 12 values or as an (R, t) pair."""
    if isinstance(T, (tuple, list)) and len(T) == 2:
        return [float(v) for v in np.asarray(T[0], np.float64).reshape(-1)] + [float(v) for v in np.asarray(T[1]).reshape(-1)]
    return [float(v) for v in np.asarray(T, np.float64).reshape(-1)]


def apply(R, t, p):
    """R p (+ t): per component ((R_k0 x + R_k1 y) + R_k2 z) (+ t_k); p is a tuple of three floats or arrays."""
    q = []
    for k in range(3):
        v = (R[3 * k] * p[0] + R[3 * k + 1] * p[1]) + R[3 * k + 2] * p[2]
        q.append(v if t is None else v + t[k])
    return q


def geometry(cell_n, res, center, req, T):
    """dict: "map_position" (x, y) of the request, "win" (success, row0, col0, rows, cols) and "centre" of the map-frame
    window, "pos", "len", "size" of the new map (NaN / 0 for a failed window).  req = (px, py, lx, ly) in the request frame, T as `flat` takes it."""
    T = flat(T)
    R, t = T[:9], T[9:]
    Ri = [R[0], R[3], R[6], R[1], R[4], R[7], R[2], R[5], R[8]]
    ti = [-v for v in apply(Ri, None, t)]
    mp = apply(Ri, ti, (float(req[0]), float(req[1]), 0.0))
    win, centre = SO.window(cell_n, res, center, np.array([mp[0], mp[1], req[2], req[3]], np.float64))
    if not win[0]:
        return {"map_position": (mp[0], mp[1]), "win": win, "centre": centre, "pos": (math.nan, math.nan),
                "len": (math.nan, math.nan), "size": (0, 0)}
    hx, hy = win[3] * res * 0.5, win[4] * res * 0.5
    cx, cy = float(centre[0]), float(centre[1])
    corners = [(cx + hx, cy + hy, 0.0), (cx + hx, cy - hy, 0.0), (cx - hx, cy + hy, 0.0), (cx - hx, cy - hy, 0.0)]
    e = [apply(R, t, p) for p in corners]
    c = [0.0, 0.0, 0.0]
    for k in range(4):
        c = [c[a] + e[k][a] for a in range(3)]
    pos, length, size = [], [], []
    for a in range(2):
        ca = c[a] * 0.25
        half = 0.0
        for k in range(4):
            half = max(abs(e[k][a] - ca), half)
        v = 2.0 * half / res
        n = int(math.floor(v))
        n += v - n >= 0.5                                       # std::round: half away from zero (v >= 0)
        pos.append(ca)
        size.append(n)
        length.append(n * res)
    return {"map_position": (mp[0], mp[1]), "win": win, "centre": centre, "pos": tuple(pos), "len": tuple(length),
            "size": tuple(size)}


def target(g, res, qx, qy):
    """(row, col) of the new map for a sample at (qx, qy), or None outside it: inside when
    0 <= -((q - pos) - 0.5 len) < len per axis, index trunc(-(((q - 0.5 len) - pos) / res)) clamped to [0, size - 1]."""
    idx = []
    for a, q in enumerate((qx, qy)):
        o = 0.5 * g["len"][a]
        u = -((q - g["pos"][a]) - o)
        if not (u >= 0.0 and u < g["len"][a]):
            return None
        i = int(-(((q - o) - g["pos"][a]) / res))
        idx.append(min(max(i, 0), g["size"][a] - 1))
    return tuple(idx)


def _samples(g, res, s, row, col, h, n_samples):
    """The samples of window cell (row, col) with elevation h, in order."""
    x0 = float(g["centre"][0]) + (0.5 * (g["win"][3] * res) - 0.5 * res)
    y0 = float(g["centre"][1]) + (0.5 * (g["win"][4] * res) - 0.5 * res)
    x, y = x0 - res * row, y0 - res * col
    out = [(x, y, h)]
    if n_samples == 5:
        out += [(x - s, y + 0.0, h + 0.0), (x + s, y + 0.0, h + 0.0), (x + 0.0, y - s, h + 0.0),
                (x + 0.0, y + s, h + 0.0)]
    return out


def sequential(layers, g, T, res, sample_ratio=0.0):
    """The new map's layers (dict name -> (rows, cols) float32) from the window's exported layers (dict name ->
    (win rows, win cols) float32; "elevation" must be there): grid_map's loop, literally."""
    T = flat(T)
    R, t = T[:9], T[9:]
    nr, nc = g["size"]
    out = {k: np.full((nr, nc), np.nan, np.float32) for k in layers}
    if not g["win"][0]:
        return out
    elev = layers["elevation"]
    rows, cols = g["win"][3], g["win"][4]
    n_samples = 5 if sample_ratio > 0 else 1
    s = res * float(sample_ratio)
    for col in range(cols):
        for row in range(rows):
            h = elev[row, col]
            if np.isnan(h):
                continue
            for p in _samples(g, res, s, row, col, float(h), n_samples):
                q = apply(R, t, p)
                ij = target(g, res, q[0], q[1])
                if ij is None:
                    continue
                cur = out["elevation"][ij]
                if not np.isnan(cur) and float(cur) > q[2]:
                    continue
                for k, v in layers.items():
                    out[k][ij] = np.float32(q[2]) if k == "elevation" else v[row, col]
    return out


def samples(layers, g, T, res, sample_ratio=0.0):
    """Every sample that lands in the new map, vectorised: (visit index j, source row, source col, target cell
    (linear, row-major over the new map), z in double)."""
    T = flat(T)
    R, t = T[:9], T[9:]
    rows, cols = g["win"][3], g["win"][4]
    n_samples = 5 if sample_ratio > 0 else 1
    s = res * float(sample_ratio)
    col, row = np.meshgrid(np.arange(cols), np.arange(rows), indexing="ij")      # visit order: column-major
    row, col = row.reshape(-1), col.reshape(-1)
    i = np.arange(rows * cols, dtype=np.int64)
    h = layers["elevation"][row, col].astype(np.float64)
    keep = ~np.isnan(h)
    row, col, i, h = row[keep], col[keep], i[keep], h[keep]
    x0 = float(g["centre"][0]) + (0.5 * (rows * res) - 0.5 * res)
    y0 = float(g["centre"][1]) + (0.5 * (cols * res) - 0.5 * res)
    x, y = x0 - res * row.astype(np.float64), y0 - res * col.astype(np.float64)
    pts = [(x, y, h)]
    if n_samples == 5:
        pts += [(x - s, y + 0.0, h + 0.0), (x + s, y + 0.0, h + 0.0), (x + 0.0, y - s, h + 0.0), (x + 0.0, y + s, h + 0.0)]
    J, SR, SC, CELL, Z = [], [], [], [], []
    for k, p in enumerate(pts):
        q = apply(R, t, p)
        ok = np.ones(len(i), bool)
        idx = []
        for a in range(2):
            o = 0.5 * g["len"][a]
            with np.errstate(invalid="ignore"):
                u = -((q[a] - g["pos"][a]) - o)
                ok &= (u >= 0.0) & (u < g["len"][a])
                v = -(((q[a] - o) - g["pos"][a]) / res)
            idx.append(np.clip(np.trunc(np.where(ok, v, 0.0)).astype(np.int64), 0, max(g["size"][a] - 1, 0)))
        J.append(n_samples * i[ok] + k)
        SR.append(row[ok])
        SC.append(col[ok])
        CELL.append(idx[0][ok] * g["size"][1] + idx[1][ok])
        Z.append(q[2][ok])
    return tuple(np.concatenate(a) for a in (J, SR, SC, CELL, Z))


def winners(cell, z, j, n_cells):
    """The order-free rule: per target, M = max fp32(z) and the winning sample (an index into the arrays), -1 where no
    sample lands.  Returns (M float32 per cell, winner per cell)."""
    f = z.astype(np.float32)
    M = np.full(n_cells, -np.inf, np.float32)
    np.maximum.at(M, cell, f)
    hit = np.zeros(n_cells, bool)
    hit[cell] = True
    top = np.int64(1) << 40
    cand = f == M[cell]
    key = np.where(z >= M[cell].astype(np.float64), top + j, top - 1 - j)
    best = np.full(n_cells, -1, np.int64)
    np.maximum.at(best, cell[cand], key[cand])
    won = np.nonzero(cand & (key == best[cell]))[0]              # one per hit cell: j is unique
    win = np.full(n_cells, -1, np.int64)
    win[cell[won]] = won
    assert (win[hit] >= 0).all() and (win[~hit] < 0).all()
    return M, win


def parallel(layers, g, T, res, sample_ratio=0.0):
    """`sequential`'s result from the order-free rule (vectorised)."""
    nr, nc = g["size"]
    out = {k: np.full((nr, nc), np.nan, np.float32) for k in layers}
    if not g["win"][0] or nr * nc == 0:
        return out
    j, sr, sc, cell, z = samples(layers, g, T, res, sample_ratio)
    M, win = winners(cell, z, j, nr * nc)
    hit = win >= 0
    for k, v in layers.items():
        flat = out[k].reshape(-1)
        flat[hit] = M[hit] if k == "elevation" else v[sr[win[hit]], sc[win[hit]]]
    return out


def transformed_submap(full, names, cell_n, res, center, req, T, sample_ratio=0.0, loop=False):
    """(geometry, dict name -> new-map layer) of one request on a full export (len(names), cell_n - 2, cell_n - 2)
    of get_maps_with_names_ref; names must include "elevation".  loop: the literal loop instead of the rule."""
    g = geometry(cell_n, res, center, req, T)
    crop = SO.crop(full, g["win"]) if g["win"][0] else full[:, :0, :0]
    layers = {nm: crop[k] for k, nm in enumerate(names)}
    return g, (sequential if loop else parallel)(layers, g, T, res, sample_ratio)


def rot(roll=0.0, pitch=0.0, yaw=0.0):
    """R = Rz(yaw) Ry(pitch) Rx(roll)."""
    cr, sr, cp, sp, cy, sy = (math.cos(roll), math.sin(roll), math.cos(pitch), math.sin(pitch), math.cos(yaw),
                              math.sin(yaw))
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    return Rz @ Ry @ Rx


def iso(R, t):
    """The 12 doubles of a transform: R row-major, then t."""
    return np.concatenate([np.asarray(R, np.float64).reshape(-1), np.asarray(t, np.float64)])


def transforms(res):
    """The tests' transforms: yaw at the right angles (exact matrices) and at arbitrary angles, roll / pitch, and
    translations of whole, half and odd fractions of a cell."""
    exact = {0: np.eye(3), 90: np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]]),
             180: np.diag([-1.0, -1.0, 1.0]), 270: np.array([[0, 1, 0], [-1, 0, 0], [0, 0, 1.0]])}
    out = [iso(R, (0, 0, 0)) for R in exact.values()]
    out += [iso(exact[90], (3 * res, -5 * res, 0.2)), iso(exact[180], (0.5 * res, 1.5 * res, 0)),
            iso(np.eye(3), (0.37 * res, -2.71 * res, -1.0))]
    for yaw in (0.1, 0.7853981633974483, 2.0, -2.9):
        out.append(iso(rot(yaw=yaw), (1.234, -0.567, 0.3)))
    out.append(iso(rot(0.2, -0.15, 0.6), (0.5, 0.25, -0.4)))
    out.append(iso(rot(0.0, 1.39, 0.3), (-0.3, 0.1, 0.0)))      # pitch 80 degrees: many cells per target row
    out.append(iso(rot(0.3, 0.0, 0.0), (0.0, 7 * res, 0.0)))
    return out
