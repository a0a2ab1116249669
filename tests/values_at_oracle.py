"""Sequential restatement of layer values at points (include/emap.h: emap_grid_values_at / emap_map_values_at), written
from the header's contract in Python floats (IEEE double, each operation rounded on its own) with one rounding to
float32 at the end.  Layers are (rows, cols) float32 arrays of one geometry; positions (N, 2) float64."""
import math

import numpy as np

NEAREST, LINEAR, CUBIC = 0, 1, 2                          # EMAP_VALUES_*
OUTSIDE, BY_NEAREST, BY_LINEAR, BY_CUBIC = 0, 1, 2, 3     # EMAP_VALUE_*
QNAN = np.frombuffer(np.uint32(0x7FC00000).tobytes(), np.float32)[0]
M = ((0.0, 2.0, 0.0, 0.0), (-1.0, 0.0, 1.0, 0.0), (2.0, -5.0, 4.0, -1.0), (-1.0, 3.0, -3.0, 1.0))


def axis_index(v, p, length, res, n):
    """The cell of coordinate v on one axis, None outside: 0 <= -((v - p) - o) < L, trunc(-(((v - o) - p) / res))
    clamped to [0, n - 1]."""
    o = 0.5 * length
    u = -((v - p) - o)
    if not (u >= 0.0 and u < length):
        return None
    i = math.trunc(-(((v - o) - p) / res))
    return min(max(i, 0), n - 1)


def axis_position(p, length, res, i):
    """(p + (0.5 L - 0.5 res)) - res i"""
    return (p + (0.5 * length - 0.5 * res)) - res * float(i)


def cubic_weights(t):
    """w_j = 0.5 (((M0j + M1j t) + M2j t^2) + M3j t^3)"""
    t2 = t * t
    t3 = t2 * t
    return [0.5 * (((M[0][j] + M[1][j] * t) + M[2][j] * t2) + M[3][j] * t3) for j in range(4)]


def _f32(v):
    with np.errstate(over="ignore", invalid="ignore"):
        f = np.float32(v)
    return QNAN if f != f else f


def point(layers, position, res, method, x, y):
    """(status, [value per layer]) of one point."""
    rows, cols = layers[0].shape
    L = (rows * res, cols * res)
    r = axis_index(x, position[0], L[0], res, rows)
    c = axis_index(y, position[1], L[1], res, cols)
    if r is None or c is None:
        return OUTSIDE, [QNAN] * len(layers)

    def F(a, i, j):
        return float(a[i, j])

    nearest = (BY_NEAREST, [_f32(F(a, r, c)) for a in layers])
    if method == NEAREST:
        return nearest
    rn = r - 1 if x >= axis_position(position[0], L[0], res, r) else r + 1
    cn = c - 1 if y >= axis_position(position[1], L[1], res, c) else c + 1
    if not (0 <= rn < rows and 0 <= cn < cols):
        return nearest
    r0, c0 = max(r, rn), max(c, cn)
    tx = (x - axis_position(position[0], L[0], res, r0)) / res
    ty = (y - axis_position(position[1], L[1], res, c0)) / res
    if method == CUBIC and r0 + 1 < rows and r0 - 2 >= 0 and c0 + 1 < cols and c0 - 2 >= 0:
        wx, wy = cubic_weights(tx), cubic_weights(ty)
        out = []
        for a in layers:
            g = []
            for i in range(4):
                rr = r0 + 1 - i
                s = ((wy[0] * F(a, rr, c0 + 1) + wy[1] * F(a, rr, c0)) + wy[2] * F(a, rr, c0 - 1)) + wy[3] * F(a, rr, c0 - 2)
                g.append(s)
            out.append(_f32(((wx[0] * g[0] + wx[1] * g[1]) + wx[2] * g[2]) + wx[3] * g[3]))
        return BY_CUBIC, out
    ux, uy = 1.0 - tx, 1.0 - ty
    out = []
    for a in layers:
        f0, f1, f2, f3 = F(a, r0, c0), F(a, r0 - 1, c0), F(a, r0, c0 - 1), F(a, r0 - 1, c0 - 1)
        out.append(_f32((((f0 * ux) * uy + (f1 * tx) * uy) + (f2 * ux) * ty) + (f3 * tx) * ty))
    return BY_LINEAR, out


def values_at(layers, position, res, method, positions):
    """emap_grid_values_at's outputs: values (n_layers, N) float32 and status (N,) int32."""
    layers = [np.asarray(a, np.float32) for a in layers]
    q = np.asarray(positions, np.float64).reshape(-1, 2)
    values = np.zeros((len(layers), len(q)), np.float32)
    status = np.zeros(len(q), np.int32)
    pos = (float(position[0]), float(position[1]))
    with np.errstate(invalid="ignore", over="ignore"):
        for i, (x, y) in enumerate(q.tolist()):
            status[i], vs = point(layers, pos, float(res), method, x, y)
            values[:, i] = vs
    return values, status
