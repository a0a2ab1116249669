"""NumPy restatement of the exported map as a point cloud, as normal arrows and as the normal colour (include/emap.h,
DESIGN §4i): grid_map's toPointCloud(map, {"elevation"}, "elevation"), the node's publishNormalAsArrow and the bridge's
addNormalColorLayer, applied to a full export (elevation, normal_x/y/z: (cell_n-2, cell_n-2) arrays in
get_maps_with_names_ref's coordinates) and the map's fp32 centre and resolution.  Restated from grid_map's published
source; not checked against a grid_map build."""
import numpy as np


def positions(n, resolution, center):
    """x of exported rows 0..n-1 and y of exported columns 0..n-1, in double: getPositionFromIndex with buffer start
    (0, 0) and the geometry get_grid_map sets (length n * resolution, position = the fp32 centre widened)."""
    res = float(resolution)
    L = n * res
    idx = np.arange(n, dtype=np.float64)
    out = []
    for a in range(2):
        first = float(np.float64(np.float32(center[a]))) + (0.5 * L - 0.5 * res)
        out.append(first - res * idx)
    return out[0], out[1]


def _column_major(a):
    return np.asarray(a).reshape(a.shape[0], a.shape[1]).ravel(order="F")


def map_points(elevation, resolution, center):
    """(M, 3) float32 rows (x, y, z): the cells with a finite elevation, column-major (linear index c * n + r)."""
    n = elevation.shape[0]
    x, y = positions(n, resolution, center)
    X = np.broadcast_to(x[:, None], (n, n))
    Y = np.broadcast_to(y[None, :], (n, n))
    e = _column_major(elevation)
    keep = np.isfinite(e)
    return np.stack([_column_major(X)[keep].astype(np.float32), _column_major(Y)[keep].astype(np.float32),
                     e[keep].astype(np.float32)], 1)


def normal_arrows(elevation, nx, ny, nz, resolution, center):
    """(ids int32 (M,), segments float64 (M, 6)): cells with a finite elevation whose normal is not shorter than 0.1
    (skipped when sqrt((nx^2 + ny^2) + nz^2) < 0.1 in double), column-major; id = the linear index c * n + r;
    start = (x, y, elevation), end = start + normal * 0.1, in double."""
    n = elevation.shape[0]
    x, y = positions(n, resolution, center)
    X = _column_major(np.broadcast_to(x[:, None], (n, n)))
    Y = _column_major(np.broadcast_to(y[None, :], (n, n)))
    e = _column_major(elevation).astype(np.float64)
    N = [_column_major(a).astype(np.float64) for a in (nx, ny, nz)]
    with np.errstate(invalid="ignore"):
        norm = np.sqrt((N[0] * N[0] + N[1] * N[1]) + N[2] * N[2])
        keep = np.isfinite(e) & ~(norm < 0.1)
    ids = np.nonzero(keep)[0].astype(np.int32)
    start = np.stack([X[keep], Y[keep], e[keep]], 1)
    end = np.stack([start[:, k] + N[k][keep] * 0.1 for k in range(3)], 1)
    return ids, np.concatenate([start, end], 1)


def _channel(v):
    """int(v * 255.0f): a float32 product truncated toward zero; NaN gives 0, beyond the int32 range saturates."""
    p = (np.asarray(v, np.float32) * np.float32(255.0)).astype(np.float32)
    out = np.zeros(p.shape, np.int64)
    ok = ~np.isnan(p)
    out[ok] = np.clip(np.trunc(p[ok].astype(np.float64)), -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)
    return out


def normal_color(nx, ny, nz):
    """float32 array: the float whose bits are (r << 16) | (g << 8) | b, r = int(float((nx + 1.0) / 2.0) * 255.0f),
    g likewise from ny, b = int(nz * 255.0f)."""
    cx = ((np.asarray(nx, np.float32).astype(np.float64) + 1.0) / 2.0).astype(np.float32)
    cy = ((np.asarray(ny, np.float32).astype(np.float64) + 1.0) / 2.0).astype(np.float32)
    bits = ((_channel(cx) << 16) | (_channel(cy) << 8) | _channel(nz)) & 0xFFFFFFFF
    return bits.astype(np.uint32).view(np.float32)
