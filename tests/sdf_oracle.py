"""The signed distance field and its queries restated on the host (include/emap.h states the contract).

The volume: occupancy and each column's top slice T in NumPy doubles, the squared distance d2 to the nearest voxel of
the other kind from scipy's exact feature transform (distance_transform_edt's return_indices), squared in integers so
the result does not depend on scipy's float distances, then float32 as specified.  `brute_d2` checks it over every
pair of voxels on small volumes.  The queries are restated in Python floats, one rounded operation at a time."""
import math
import struct

import numpy as np
from scipy import ndimage

MAX_D2 = 1 << 24
QNAN = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000000))[0]


def fill_layer(e):
    """The layer as float64 with non-finite cells set to its lowest finite value (-inf when there is none)."""
    e = np.asarray(e, np.float32).astype(np.float64)
    fin = np.isfinite(e)
    low = e[fin].min() if fin.any() else -np.inf
    return np.where(fin, e, low)


def slices(z_min, n_z, res):
    """z_k = z_min + k * res in double, one multiply then one add."""
    return np.float64(z_min) + np.arange(n_z, dtype=np.float64) * np.float64(res)


def occupancy(e, z_min, n_z, res):
    """(n_z, rows, cols) bool: (double) e(r, c) >= z_k."""
    return fill_layer(e)[None, :, :] >= slices(z_min, n_z, res)[:, None, None]


def top_slice(e, z_min, n_z, res):
    """T(r, c): the highest occupied slice, -1 for none (occupancy is monotone in k)."""
    occ = occupancy(e, z_min, n_z, res)
    assert np.array_equal(occ, np.cumsum(occ[::-1], 0)[::-1] > 0), "occupancy is not monotone"
    return occ.sum(0).astype(np.int64) - 1


def _d2_to(targets):
    """Per voxel the exact squared distance (int64) to the nearest True voxel of `targets`; -1 when there is none."""
    if not targets.any():
        return np.full(targets.shape, -1, np.int64)
    idx = ndimage.distance_transform_edt(~targets, return_distances=False, return_indices=True)
    d2 = np.zeros(targets.shape, np.int64)
    for a in range(targets.ndim):
        shape = [1] * targets.ndim
        shape[a] = -1
        d2 += (idx[a].astype(np.int64) - np.arange(targets.shape[a], dtype=np.int64).reshape(shape)) ** 2
    return d2


def d2_field(occ):
    """Signed int64 d2 per voxel: + the distance to occupancy for free voxels, - the distance to free space for
    occupied ones; 0 stands for none (the value is then +-inf)."""
    to_occ, to_free = _d2_to(occ), _d2_to(~occ)
    return np.where(occ, -np.where(to_free < 0, 0, to_free), np.where(to_occ < 0, 0, to_occ))


def metres(d2, occ, res):
    """+-fl(sqrt(float(d2)) * float(res)) as float32, +-inf where d2 is 0 (no voxel of the other kind)."""
    a = np.abs(d2)
    assert a.max(initial=0) < MAX_D2
    m = np.sqrt(a.astype(np.float32)) * np.float32(res)
    m = np.where(a == 0, np.float32(np.inf), m).astype(np.float32)
    return np.where(occ, -m, m).astype(np.float32)


def field(e, z_min, n_z, res):
    """The (n_z, rows, cols) float32 volume emap_signed_distance_field writes."""
    occ = occupancy(e, z_min, n_z, res)
    return metres(d2_field(occ), occ, res)


def brute_d2(occ):
    """d2_field by brute force over every pair of voxels (small volumes only)."""
    pts = np.argwhere(np.ones(occ.shape, bool))
    kind = occ.reshape(-1)
    out = np.zeros(len(pts), np.int64)
    for i, p in enumerate(pts):
        other = pts[kind != kind[i]]
        if len(other):
            d = int(((other - p) ** 2).sum(1).min())
            out[i] = -d if kind[i] else d
    return out.reshape(occ.shape)


def brute_envelope(f):
    """min over p of (q - p)^2 + f[p] for every q, f[p] = None meaning no site; None where there is no site."""
    sites = [(p, v) for p, v in enumerate(f) if v is not None]
    return [min(((q - p) ** 2 + v for p, v in sites), default=None) for q in range(len(f))]


def default_range(e, res, clearance):
    """signed_distance_field's z_min and n_z without z_range."""
    e = np.asarray(e, np.float32)
    fin = e[np.isfinite(e)]
    lo, hi = float(fin.min()), float(fin.max())
    z_min = lo - float(clearance)
    return z_min, int(math.floor(((hi + float(clearance)) - z_min) / res)) + 1


def _origin(p, n, res):
    return p + (0.5 * (n * res) - 0.5 * res)


def _lerp(a, b, t):
    return a + t * (b - a)


def value(vol, pos, res, z_min, x, y, z):
    """emap_sdf_values for one point: [value, d/dx, d/dy, d/dz] in Python floats."""
    if x != x or y != y or z != z:
        return [QNAN] * 4
    n_z, rows, cols = vol.shape
    n = (rows, cols, n_z)
    fi = ((_origin(pos[0], rows, res) - x) / res, (_origin(pos[1], cols, res) - y) / res, (z - z_min) / res)
    i0, i1, t, off = [], [], [], []
    for a in range(3):
        top = float(n[a] - 1)
        u = 0.0 if fi[a] < 0.0 else top if fi[a] > top else fi[a]
        off.append(fi[a] - u)
        lo = 0 if n[a] == 1 else min(math.floor(u), n[a] - 2)
        i0.append(lo)
        i1.append(lo if n[a] == 1 else lo + 1)
        t.append(u - float(lo))
    V = lambda k, r, c: float(vol[k, r, c])  # noqa: E731
    Y, R, E = [], [], []
    for k in (i0[2], i1[2]):
        X, D = [], []
        for r in (i0[0], i1[0]):
            a0, a1 = V(k, r, i0[1]), V(k, r, i1[1])
            X.append(_lerp(a0, a1, t[1]))
            D.append(a1 - a0)
        Y.append(_lerp(X[0], X[1], t[0]))
        R.append(X[1] - X[0])
        E.append(_lerp(D[0], D[1], t[0]))
    dist = math.sqrt((off[0] * off[0] + off[1] * off[1]) + off[2] * off[2]) * res
    out = [_lerp(Y[0], Y[1], t[2]) + dist,
           0.0 if rows == 1 else -(_lerp(R[0], R[1], t[2]) / res),
           0.0 if cols == 1 else -(_lerp(E[0], E[1], t[2]) / res),
           0.0 if n_z == 1 else (Y[1] - Y[0]) / res]
    return [QNAN if v != v else v for v in out]


def values(vol, pos, res, z_min, points):
    """(n, 4) float64: value() per point."""
    vol = np.asarray(vol, np.float32)
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    return np.array([value(vol, pos, res, z_min, *map(float, p)) for p in pts], np.float64).reshape(-1, 4)


def position_of(pos, n_rows, n_cols, res, r, c):
    """getPositionFromIndex of cell (r, c) (the voxel centres' x, y)."""
    return _origin(pos[0], n_rows, res) - res * r, _origin(pos[1], n_cols, res) - res * c
