"""NumPy / Python-integer restatement of what emap_initialize_map adds to the map initialiser (include/emap.h states the
rules): the snap of the points to cells, the exact-predicate Delaunay triangulation with its tie rule, SciPy's global
gradient estimate, barycentric and Clough-Tocher evaluation under the lowest-triangle owner rule, and nearest with
lowest-index ties.  Slow and plain on purpose: every predicate is on Python integers, every value a Python float."""
import numpy as np

METHODS = {"nearest": 0, "linear": 1, "cubic": 2}
INF = -1          # the vertex at infinity of the ghost triangles


def snap(points, center, resolution, W):
    """transform_to_map_index as initialize_map applies it: ((xy - center_xy) / fp32(res) + W / 2) in fp32, truncated,
    and z - center_z in fp32.  Returns (idx (n, 2) int64, z (n,) float64)."""
    pts = np.array(points, np.float32, copy=True).reshape(-1, 3)
    c = np.asarray(center, np.float32).reshape(3)
    idx = ((pts[:, :2] - c[:2].reshape(1, 2)) / np.float32(resolution) + W / 2).astype(np.int32)
    z = pts[:, 2] - c[2]
    return idx.astype(np.int64), z.astype(np.float64)


def orient(a, b, c):
    """Twice the signed area of (a, b, c): > 0 counter-clockwise."""
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def incircle(a, b, c, d):
    """> 0 when d lies strictly inside the circumcircle of the counter-clockwise triangle (a, b, c)."""
    adx, ady, bdx, bdy, cdx, cdy = a[0] - d[0], a[1] - d[1], b[0] - d[0], b[1] - d[1], c[0] - d[0], c[1] - d[1]
    return ((adx * adx + ady * ady) * (bdx * cdy - cdx * bdy) + (bdx * bdx + bdy * bdy) * (cdx * ady - adx * cdy)
            + (cdx * cdx + cdy * cdy) * (adx * bdy - bdx * ady))


def _conflict(P, t, p):
    """Whether point p lies in the circumcircle of triangle t; a ghost (u, v, INF) has the open half-plane left of u -> v
    and the open segment (u, v) as its circle."""
    if t[2] != INF:
        return incircle(P[t[0]], P[t[1]], P[t[2]], p) > 0
    u, v = P[t[0]], P[t[1]]
    o = orient(u, v, p)
    if o != 0:
        return o > 0
    return ((p[0] - u[0]) * (v[0] - u[0]) + (p[1] - u[1]) * (v[1] - u[1]) > 0
            and (p[0] - v[0]) * (u[0] - v[0]) + (p[1] - v[1]) * (u[1] - v[1]) > 0)


def _ghost_last(t):
    x, y, z = t
    return (y, z, x) if x == INF else ((z, x, y) if y == INF else t)


def canonical(tris):
    """Each triangle counter-clockwise, rotated to start at its lowest vertex; triangles in lexicographic order."""
    out = []
    for a, b, c in tris:
        r = min(range(3), key=lambda k: (a, b, c)[k])
        out.append(tuple((a, b, c)[(r + k) % 3] for k in range(3)))
    return sorted(out)


def delaunay(idx):
    """The library's triangulation of integer points: Bowyer-Watson with exact predicates, inserting in input order.
    Seed: point 0, the first point that differs from it, the first point not collinear with those two.  A point equal
    to an earlier one is skipped.  A point on the circumcircle of a triangle does not break it, so among cocircular
    points the triangles of the earlier ones stay.  Returns the canonical (T, 3) int64 triangles; ValueError when all
    points are collinear."""
    P = [(int(x), int(y)) for x, y in np.asarray(idx).reshape(-1, 2)]
    n = len(P)
    i1 = next((i for i in range(n) if P[i] != P[0]), None)
    i2 = None if i1 is None else next((i for i in range(n) if orient(P[0], P[i1], P[i]) != 0), None)
    if i2 is None:
        raise ValueError("collinear points")
    a, b, c = (0, i1, i2) if orient(P[0], P[i1], P[i2]) > 0 else (0, i2, i1)
    tris = {(a, b, c), (b, a, INF), (c, b, INF), (a, c, INF)}
    seen = {P[0], P[i1], P[i2]}
    for i in range(n):
        if i in (0, i1, i2) or P[i] in seen:
            continue
        seen.add(P[i])
        cavity = [t for t in tris if _conflict(P, t, P[i])]
        edges = {(t[k], t[(k + 1) % 3]) for t in cavity for k in range(3)}
        tris.difference_update(cavity)
        for u, v in edges:
            if (v, u) not in edges:
                tris.add(_ghost_last((u, v, i)))
    return np.array(canonical([t for t in tris if INF not in t]), np.int64).reshape(-1, 3)


def unique_triangulation(idx, tris):
    """Whether the Delaunay triangulation `tris` of idx is the only one: no two points coincide and no edge's two
    opposite vertices are cocircular with it (exact integer in-circle tests)."""
    P = [tuple(int(v) for v in p) for p in np.asarray(idx).reshape(-1, 2)]
    if len(set(P)) != len(P):
        return False
    tris = ccw(idx, tris)
    for t, row in zip(tris, neighbours(tris)):
        for o in row:
            if o >= 0:
                w = [v for v in tris[o] if v not in t][0]
                if incircle(P[t[0]], P[t[1]], P[t[2]], P[w]) == 0:
                    return False
    return True


def ccw(idx, tris):
    """The triangles with each one's vertices counter-clockwise (caller triangles may come in either order)."""
    P = np.asarray(idx, np.int64)
    out = np.array(tris, np.int64).reshape(-1, 3).copy()
    for t in out:
        if orient(P[t[0]], P[t[1]], P[t[2]]) < 0:
            t[1], t[2] = t[2], t[1]
    return out


def neighbours(tris):
    """(T, 3): the triangle across the edge opposite vertex k, -1 on the hull."""
    at = {}
    for ti, t in enumerate(tris):
        for k in range(3):
            at[(int(t[(k + 1) % 3]), int(t[(k + 2) % 3]))] = ti
    return np.array([[at.get((int(t[(k + 2) % 3]), int(t[(k + 1) % 3])), -1) for k in range(3)] for t in tris],
                    np.int64).reshape(-1, 3)


def estimate_gradients(idx, z, tris, tol=1e-6, maxiter=400):
    """SciPy's estimate_gradients_2d_global (Nielson's minimum-norm network), vertices in index order, each vertex's
    neighbours in ascending order.  A point on no triangle keeps gradient (0, 0)."""
    n = len(idx)
    P = [(float(x), float(y)) for x, y in np.asarray(idx).reshape(-1, 2)]
    nb = [set() for _ in range(n)]
    for t in tris:
        for k in range(3):
            nb[int(t[k])].update((int(t[(k + 1) % 3]), int(t[(k + 2) % 3])))
    nb = [sorted(s) for s in nb]
    f = [float(v) for v in z]
    y = [0.0] * (2 * n)
    for _ in range(maxiter):
        err = 0.0
        for i in range(n):
            if not nb[i]:
                continue
            q0 = q1 = q3 = s0 = s1 = 0.0
            for j in nb[i]:
                ex, ey = P[j][0] - P[i][0], P[j][1] - P[i][1]
                L = np.sqrt(ex * ex + ey * ey)
                L3 = L * L * L
                df2 = -ex * y[2 * j] - ey * y[2 * j + 1]
                q0 += 4 * ex * ex / L3
                q1 += 4 * ex * ey / L3
                q3 += 4 * ey * ey / L3
                s0 += (6 * (f[i] - f[j]) - 2 * df2) * ex / L3
                s1 += (6 * (f[i] - f[j]) - 2 * df2) * ey / L3
            det = q0 * q3 - q1 * q1
            r0 = (q3 * s0 - q1 * s1) / det
            r1 = (-q1 * s0 + q0 * s1) / det
            change = max(abs(y[2 * i] + r0), abs(y[2 * i + 1] + r1))
            y[2 * i], y[2 * i + 1] = -r0, -r1
            change /= max(1.0, max(abs(r0), abs(r1)))
            err = max(err, change)
        if err < tol:
            break
    return np.array(y, np.float64).reshape(n, 2)


CT_NAMES = ("c3000", "c0300", "c0030", "c2100", "c2010", "c1200", "c0210", "c1020", "c0120", "c2001", "c0201", "c0021",
            "c0111", "c1011", "c1101", "c1002", "c0102", "c0012", "c0003")


def ct_coefficients(idx, z, grad, tris, nbr):
    """Per triangle the 19 Bezier ordinates (CT_NAMES order) of SciPy's Clough-Tocher element, split at the centroid,
    with the affine-invariant cross-boundary directions towards the neighbours' centroids."""
    P = np.asarray(idx, np.float64)
    out = np.zeros((len(tris), 19), np.float64)
    for ti, t in enumerate(tris):
        p0, p1, p2 = P[t[0]], P[t[1]], P[t[2]]
        e12, e23, e31 = p1 - p0, p2 - p1, p0 - p2
        f1, f2, f3 = (float(z[t[k]]) for k in range(3))
        d = [grad[t[k]] for k in range(3)]
        df12 = +(d[0][0] * e12[0] + d[0][1] * e12[1])
        df21 = -(d[1][0] * e12[0] + d[1][1] * e12[1])
        df23 = +(d[1][0] * e23[0] + d[1][1] * e23[1])
        df32 = -(d[2][0] * e23[0] + d[2][1] * e23[1])
        df31 = +(d[2][0] * e31[0] + d[2][1] * e31[1])
        df13 = -(d[0][0] * e31[0] + d[0][1] * e31[1])
        c3000, c0300, c0030 = f1, f2, f3
        c2100 = (df12 + 3 * c3000) / 3
        c2010 = (df13 + 3 * c3000) / 3
        c1200 = (df21 + 3 * c0300) / 3
        c0210 = (df23 + 3 * c0300) / 3
        c1020 = (df31 + 3 * c0030) / 3
        c0120 = (df32 + 3 * c0030) / 3
        c2001 = (c2100 + c2010 + c3000) / 3
        c0201 = (c1200 + c0300 + c0210) / 3
        c0021 = (c1020 + c0120 + c0030) / 3
        g = [-0.5, -0.5, -0.5]
        for k in range(3):
            o = nbr[ti][k]
            if o < 0:
                continue
            s = P[tris[o][0]] + P[tris[o][1]] + P[tris[o][2]]       # 3 x the neighbour's centroid
            c = barycentric3(p0, p1, p2, s)
            if k == 0:
                g[k] = (2 * c[2] + c[1] - 1) / (2 - 3 * c[2] - 3 * c[1])
            elif k == 1:
                g[k] = (2 * c[0] + c[2] - 1) / (2 - 3 * c[0] - 3 * c[2])
            else:
                g[k] = (2 * c[1] + c[0] - 1) / (2 - 3 * c[1] - 3 * c[0])
        c0111 = (g[0] * (-c0300 + 3 * c0210 - 3 * c0120 + c0030) + (-c0300 + 2 * c0210 - c0120 + c0021 + c0201)) / 2
        c1011 = (g[1] * (-c0030 + 3 * c1020 - 3 * c2010 + c3000) + (-c0030 + 2 * c1020 - c2010 + c2001 + c0021)) / 2
        c1101 = (g[2] * (-c3000 + 3 * c2100 - 3 * c1200 + c0300) + (-c3000 + 2 * c2100 - c1200 + c2001 + c0201)) / 2
        c1002 = (c1101 + c1011 + c2001) / 3
        c0102 = (c1101 + c0111 + c0201) / 3
        c0012 = (c1011 + c0111 + c0021) / 3
        c0003 = (c1002 + c0102 + c0012) / 3
        out[ti] = [c3000, c0300, c0030, c2100, c2010, c1200, c0210, c1020, c0120, c2001, c0201, c0021,
                   c0111, c1011, c1101, c1002, c0102, c0012, c0003]
    return out


def barycentric3(p0, p1, p2, s):
    """Barycentric coordinates of s / 3 in the triangle (p0, p1, p2), from the cross products of 3 * p against s."""
    a = (p1[0] - p0[0]) * (p2[1] - p0[1]) - (p1[1] - p0[1]) * (p2[0] - p0[0])
    q = [3 * p for p in (p0, p1, p2)]
    l0 = (q[1][0] - s[0]) * (q[2][1] - s[1]) - (q[1][1] - s[1]) * (q[2][0] - s[0])
    l1 = (q[2][0] - s[0]) * (q[0][1] - s[1]) - (q[2][1] - s[1]) * (q[0][0] - s[0])
    l2 = (q[0][0] - s[0]) * (q[1][1] - s[1]) - (q[0][1] - s[1]) * (q[1][0] - s[0])
    return [l0 / (9 * a), l1 / (9 * a), l2 / (9 * a)]


def _bezier(u, v, w, A, B, C, D, E, F, G, H, I, J):
    """The cubic Bezier patch over one sub-triangle at its barycentric coordinates (u, v, w), w for the centroid."""
    uu, vv, ww = u * u, v * v, w * w
    return (uu * u * A + 3 * uu * v * B + 3 * u * vv * C + vv * v * D + 3 * uu * w * E + 6 * u * v * w * F
            + 3 * vv * w * G + 3 * u * ww * H + 3 * v * ww * I + ww * w * J)


def ct_eval(c, b0, b1, b2):
    """The Clough-Tocher element of ordinates c (CT_NAMES order) at barycentric coordinates (b0, b1, b2) (arrays)."""
    (c3000, c0300, c0030, c2100, c2010, c1200, c0210, c1020, c0120, c2001, c0201, c0021,
     c0111, c1011, c1101, c1002, c0102, c0012, c0003) = c
    m = np.minimum(np.minimum(b0, b1), b2)
    e1, e2, e3, e4 = b0 - m, b1 - m, b2 - m, 3 * m
    return np.where(b0 == m,
                    _bezier(e2, e3, e4, c0300, c0210, c0120, c0030, c0201, c0111, c0021, c0102, c0012, c0003),
                    np.where(b1 == m,
                             _bezier(e3, e1, e4, c0030, c1020, c2010, c3000, c0021, c1011, c2001, c0012, c1002, c0003),
                             _bezier(e1, e2, e4, c3000, c2100, c1200, c0300, c2001, c1101, c0201, c1002, c0102, c0003)))


def interpolate(W, method, idx, z, tris=None, grad=None):
    """The (W, W) float64 interpolant over cells (i, j) = (row, column), NaN where it is undefined.  linear / cubic: a
    cell takes the lowest-index triangle that contains it (closed); tris default to delaunay(idx), grad (cubic) to
    estimate_gradients.  nearest: the point at the least squared distance, the lowest index on a tie."""
    idx = np.asarray(idx, np.int64)
    z = np.asarray(z, np.float64)
    out = np.full((W, W), np.nan)
    if method == "nearest":
        gi, gj = np.mgrid[0:W, 0:W]
        best = np.zeros((W, W), np.int64)
        bd = (gi - idx[0, 0]) ** 2 + (gj - idx[0, 1]) ** 2
        for k in range(1, len(idx)):         # strict <: the lowest index keeps a tie
            d = (gi - idx[k, 0]) ** 2 + (gj - idx[k, 1]) ** 2
            take = d < bd
            bd = np.where(take, d, bd)
            best = np.where(take, k, best)
        return z[best]
    tris = delaunay(idx) if tris is None else ccw(idx, tris)
    if method == "cubic":
        if grad is None:
            grad = estimate_gradients(idx, z, tris)
        coef = ct_coefficients(idx, z, np.asarray(grad, np.float64), tris, neighbours(tris))
    owner = np.full((W, W), -1, np.int64)
    for ti in range(len(tris) - 1, -1, -1):          # descending, so the lowest containing index is written last
        sl, o = _cells(W, idx, tris[ti])
        if sl is not None:
            owner[sl][(o[0] >= 0) & (o[1] >= 0) & (o[2] >= 0)] = ti
    for ti in range(len(tris)):
        sl, o = _cells(W, idx, tris[ti])
        if sl is None:
            continue
        mine = owner[sl] == ti
        a = (o[0] + o[1] + o[2]).astype(np.float64)
        b = [o[k].astype(np.float64) / a for k in range(3)]
        if method == "linear":
            v = b[0] * z[tris[ti][0]] + b[1] * z[tris[ti][1]] + b[2] * z[tris[ti][2]]
        else:
            v = ct_eval(coef[ti], *b)
        out[sl][mine] = v[mine]
    return out


def _cells(W, idx, t):
    """(slice of the triangle's bounding box in the grid, the three edge orientations of its cells) or (None, None)."""
    p = [idx[v] for v in t]
    lo = np.maximum(np.min(p, 0), 0)
    hi = np.minimum(np.max(p, 0), W - 1)
    if lo[0] > hi[0] or lo[1] > hi[1]:
        return None, None
    gi, gj = np.mgrid[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1]
    q = (gi, gj)
    return ((slice(lo[0], hi[0] + 1), slice(lo[1], hi[1] + 1)),
            [orient(p[1], p[2], q), orient(p[2], p[0], q), orient(p[0], p[1], q)])


def planes(W, interp, initialized_variance, initial_variance):
    """elevation, variance, is_valid of map_initializer.py:57-61 from the float64 interpolant."""
    ok = ~np.isnan(interp)
    return (np.nan_to_num(interp).astype(np.float32),
            np.where(ok, np.float32(initialized_variance), np.float32(initial_variance)).astype(np.float32),
            ok.astype(np.float32))
