"""Python-float restatement of convex_plane_decomposition's GeometryUtils, SegmentedPlaneProjection and
ConvexRegionGrowing, the oracle of ElevationMap.project_to_planar_regions.  Predicates are exact: a double filter
(Shewchuk's orient2d bound) with a fractions.Fraction fallback.  Constructions are Python float arithmetic in the order
include/emap.h states (CGAL's Cartesian squared distance, Eigen's fixed-size sums).  Both the reference's search (bounding
boxes, sorted, pruned) and the exhaustive one of testConvexApproximation.cpp are here.  The trigonometric table of
createRegularPolygon is the C library's cos / sin of i * ((2 pi) / n), passed in as the device receives it."""
import math
from fractions import Fraction

import numpy as np

ORIENT_BOUND = 3.3306690738754716e-16       # (3 + 16 eps) eps, eps = 2^-53, rounded up
DBL_MAX = 1.7976931348623157e308
MAX_ITER = 1000
GROWN, ZERO_RADIUS, MAX_ITERATIONS, NO_REGION, INVALID_QUERY, BAD_TABLE = range(6)


def _sign(v):
    return (v > 0) - (v < 0)


def orient(ax, ay, bx, by, cx, cy):
    """Sign of (a - c) x (b - c): 1 counter-clockwise, -1 clockwise, 0 collinear, exactly."""
    dl = (ax - cx) * (by - cy)
    dr = (ay - cy) * (bx - cx)
    det = dl - dr
    if dl > 0:
        if dr <= 0:
            return _sign(det)
        ds = dl + dr
    elif dl < 0:
        if dr >= 0:
            return _sign(det)
        ds = -dl - dr
    else:
        return _sign(det)
    if abs(det) >= ORIENT_BOUND * ds:
        return _sign(det)
    F = Fraction
    return _sign((F(ax) - F(cx)) * (F(by) - F(cy)) - (F(ay) - F(cy)) * (F(bx) - F(cx)))


def _between(v, a, b):
    return min(a, b) <= v <= max(a, b)


def _on_segment(p, a, b):
    return _between(p[0], a[0], b[0]) and _between(p[1], a[1], b[1]) and orient(a[0], a[1], b[0], b[1], p[0], p[1]) == 0


def bounded_side(p, poly):
    """CGAL's bounded_side_2: 1 inside, 0 on an edge, -1 outside (the even-odd rule off the edges)."""
    n = len(poly)
    inside = False
    for k in range(n):
        a, b = poly[k], poly[(k + 1) % n]
        if _on_segment(p, a, b):
            return 0
        if (a[1] > p[1]) != (b[1] > p[1]):
            o = orient(a[0], a[1], b[0], b[1], p[0], p[1])
            if (o > 0) if b[1] > a[1] else (o < 0):
                inside = not inside
    return 1 if inside else -1


def segments_intersect(p1, p2, q1, q2):
    """CGAL::do_intersect of two closed segments."""
    o1, o2 = orient(*p1, *p2, *q1), orient(*p1, *p2, *q2)
    o3, o4 = orient(*q1, *q2, *p1), orient(*q1, *q2, *p2)
    if o1 * o2 < 0 and o3 * o4 < 0:
        return True
    return any(o == 0 and _between(c[0], a[0], b[0]) and _between(c[1], a[1], b[1])
               for o, c, a, b in ((o1, q1, p1, p2), (o2, q2, p1, p2), (o3, p1, q1, q2), (o4, p2, q1, q2)))


def _less_xy(a, b):
    return a[0] < b[0] or (a[0] == b[0] and a[1] < b[1])


def is_convex(pts):
    """CGAL's is_convex_2 (Polygon_2_algorithms_impl.h), restated from its published source."""
    n = len(pts)
    if n < 3:
        return True
    first, previous, current, nxt = 0, 0, 1, 2
    while pts[previous] == pts[current]:
        current = nxt
        nxt += 1
        if nxt == n:
            return True
    cw = ccw = False
    order = _less_xy(pts[previous], pts[current])
    changes = 0
    while True:
        while True:
            o = orient(*pts[previous], *pts[current], *pts[nxt])
            if o < 0:
                cw = True
            elif o > 0:
                ccw = True
            elif pts[current] == pts[nxt]:
                if nxt == first:
                    first = current
                nxt += 1
                if nxt == n:
                    nxt = first
                continue
            break
        new_order = _less_xy(pts[current], pts[nxt])
        if order != new_order:
            changes += 1
        if changes > 2 or (cw and ccw):
            return False
        previous, current = current, nxt
        nxt += 1
        if nxt == n:
            nxt = first
        order = new_order
        if previous == first:
            return True


def sqdist_segment(p, s, t):
    """CGAL::squared_distance(Point_2, Segment_2 s -> t), Cartesian kernel, as include/emap.h states it."""
    dx, dy = p[0] - s[0], p[1] - s[1]
    vx, vy = t[0] - s[0], t[1] - s[1]
    d = dx * vx + dy * vy
    if d <= 0.0:
        return dx * dx + dy * dy
    if d > vx * vx + vy * vy:
        ex, ey = p[0] - t[0], p[1] - t[1]
        return ex * ex + ey * ey
    if s[1] == t[1]:
        a = 0.0
        b, c = (1.0, -s[1]) if t[0] > s[0] else (0.0, 0.0) if t[0] == s[0] else (-1.0, s[1])
    elif t[0] == s[0]:
        b = 0.0
        a, c = (-1.0, s[0]) if t[1] > s[1] else (1.0, -s[0])
    else:
        a = s[1] - t[1]
        b = t[0] - s[0]
        c = -s[0] * a - s[1] * b
    w = a * p[0] + b * p[1] + c
    return (w * w) / (a * a + b * b)


def project_segment(p, s, t):
    """GeometryUtils.h's projectToClosestPoint(point, segment)."""
    vx, vy = t[0] - s[0], t[1] - s[1]
    length = math.sqrt(vx * vx + vy * vy)
    nx, ny = (vx / length, vy / length) if length != 0.0 else (math.nan, math.nan)
    dot = nx * (p[0] - s[0]) + ny * (p[1] - s[1])
    m = dot if 0.0 < dot else 0.0
    coeff = length if length < m else m
    return (coeff * nx + s[0], coeff * ny + s[1])


def project_polygon(p, poly):
    """projectToClosestPoint(point, polygon): the first edge of least squared distance."""
    n = len(poly)
    best, bk = sqdist_segment(p, poly[0], poly[1 % n]), 0
    for k in range(1, n):
        d = sqdist_segment(p, poly[k], poly[(k + 1) % n])
        if d < best:
            best, bk = d, k
    return project_segment(p, poly[bk], poly[(bk + 1) % n])


def project_region(p, region):
    """SegmentedPlaneProjection.cpp's projectToPlanarRegion."""
    for inset in region["insets"]:
        if bounded_side(p, inset["outer"]) >= 0:
            for hole in inset["holes"]:
                if bounded_side(p, hole) >= 0:
                    return project_polygon(p, hole)
            return p
    out, best = (math.nan, math.nan), DBL_MAX
    for inset in region["insets"]:
        c = project_polygon(p, inset["outer"])
        dx, dy = c[0] - p[0], c[1] - p[1]
        d = dx * dx + dy * dy
        if d < best:
            out, best = c, d
    return out


def to_plane(T, p):
    """Eigen's Isometry3d::inverse() * p, for T = [R | t] as 3 rows of 4: (x, y, z) in the plane frame."""
    out = []
    for i in range(3):
        u = -((T[0][i] * T[0][3] + T[1][i] * T[1][3]) + T[2][i] * T[2][3])
        out.append(u + ((T[0][i] * p[0] + T[1][i] * p[1]) + T[2][i] * p[2]))
    return out


def to_world(T, x, y):
    return [(T[i][3] + x * T[i][0]) + y * T[i][1] for i in range(3)]


def _cost(p, w, wz):
    dx, dy, dz = p[0] - w[0], p[1] - w[1], p[2] - w[2]
    return ((dx * dx + dy * dy) + dz * dz) + wz * abs(w[2])


def best_exhaustive(p, regions, wz):
    """getBestPlanarRegionAtPositionInWorldNaive: (row, cost, plane xy, world xyz), the first least cost."""
    best = None
    for r, reg in enumerate(regions):
        q = to_plane(reg["T"], p)
        c = project_region((q[0], q[1]), reg)
        w = to_world(reg["T"], c[0], c[1])
        cost = _cost(p, w, wz)
        if best is None or cost < best[1]:
            best = (r, cost, c, w)
    return best


def _interval_sq(v, lo, hi):
    if v < lo:
        return (lo - v) * (lo - v)
    if v < hi:
        return 0.0
    return (hi - v) * (hi - v)


def best_pruned(p, regions, wz):
    """getBestPlanarRegionAtPositionInWorld: regions sorted by the squared distance to their bounding box plus the
    plane-frame z squared, skipped when that bound exceeds the best cost so far."""
    infos = []
    for r, reg in enumerate(regions):
        q = to_plane(reg["T"], p)
        b = reg["bbox"]
        infos.append((_interval_sq(q[0], b[0], b[2]) + _interval_sq(q[1], b[1], b[3]) + q[2] * q[2], r, q))
    infos.sort(key=lambda x: x[0])
    best = (-1, DBL_MAX, None, None)
    for bound, r, q in infos:
        if bound > best[1]:
            continue
        reg = regions[r]
        c = project_region((q[0], q[1]), reg)
        w = to_world(reg["T"], c[0], c[1])
        cost = _cost(p, w, wz)
        if cost < best[1]:
            best = (r, cost, c, w)
    return best


def trig_table(n):
    angle = (2.0 * math.pi) / n
    return [math.cos(i * angle) for i in range(n)], [math.sin(i * angle) for i in range(n)]


def _edges(shape):
    for poly in [shape[0]] + list(shape[1]):
        n = len(poly)
        for k in range(n):
            yield poly[k], poly[(k + 1) % n]


def sq_distance_to_shape(p, shape):
    m = DBL_MAX
    for a, b in _edges(shape):
        d = sqdist_segment(p, a, b)
        m = d if d < m else m
    return m


def inside_with_holes(p, shape):
    """GeometryUtils.h's isInside(point, polygon with holes): a hole's edge counts as inside."""
    return bounded_side(p, shape[0]) >= 0 and all(bounded_side(p, h) <= 0 for h in shape[1])


def grow(shape, center, n, growth, trig):
    """growConvexPolygonInsideShape(shape = (outer, holes), center, n, growth): (vertices, status, sweeps)."""
    cx, cy = center
    sq = sq_distance_to_shape(center, shape)
    radius = 0.999 * (math.sqrt(sq) if sq > 0.0 else 0.0)
    v = [(radius * trig[0][i] + cx, radius * trig[1][i] + cy) for i in range(n)]
    if radius == 0.0:
        return v, ZERO_RADIUS, 0
    spheres = [(cx, cy, radius * radius)] * n
    blocked = [False] * n
    n_blocked, it = 0, 0

    def in_sphere(p, s):
        dx, dy = p[0] - s[0], p[1] - s[1]
        return dx * dx + dy * dy <= s[2]

    while n_blocked < n and it < MAX_ITER:
        for i in range(n):
            if blocked[i]:
                continue
            cand = (growth * (v[i][0] - cx) + cx, growth * (v[i][1] - cy) + cy)
            cw1 = i + 1 if i < n - 1 else 0
            cw2 = cw1 + 1 if cw1 < n - 1 else 0
            ccw1 = i - 1 if i > 0 else n - 1
            ccw2 = ccw1 - 1 if ccw1 > 0 else n - 1
            moved = is_convex([v[cw2], v[cw1], cand, v[ccw1], v[ccw2]])
            if moved:
                n0, n1 = v[cw1], v[ccw1]
                s = spheres[i]
                if not (in_sphere(n0, s) and in_sphere(cand, s) and in_sphere(n1, s)):
                    m, hit = DBL_MAX, False
                    for a, b in _edges(shape):
                        if segments_intersect(n0, cand, a, b) or segments_intersect(n1, cand, a, b):
                            hit = True
                            break
                        d = sqdist_segment(cand, a, b)
                        m = d if d < m else m
                    moved = not hit
                    if moved:
                        spheres[i] = (cand[0], cand[1], m)
            if moved:
                inv = 1.0 / n
                cx = cx + inv * (cand[0] - v[i][0])
                cy = cy + inv * (cand[1] - v[i][1])
                v[i] = cand
            else:
                blocked[i] = True
                n_blocked += 1
        it += 1
    return v, (MAX_ITERATIONS if it == MAX_ITER else GROWN), it


def project(regions, queries, wz=0.0, n_convex=0, growth=1.05):
    """The call's outputs for queries (n, 3): index (n, 3) int32, point (n, 6), convex (n, n_convex, 5)."""
    n = len(queries)
    index = np.zeros((n, 3), np.int32)
    point = np.full((n, 6), np.nan)
    convex = np.full((n, n_convex, 5), np.nan)
    trig = trig_table(n_convex) if n_convex else None
    for k, p in enumerate(np.asarray(queries, np.float64).tolist()):
        if not all(math.isfinite(c) for c in p):
            index[k] = (-1, INVALID_QUERY, 0)
            point[k, 0] = math.inf
            continue
        if not regions:
            index[k] = (-1, NO_REGION, 0)
            point[k, 0] = math.inf
            continue
        r, cost, c, w = best_exhaustive(p, regions, wz)
        index[k] = (r, GROWN, 0)
        point[k] = (cost, c[0], c[1], *w)
        if n_convex:
            reg = regions[r]
            v, status, it = grow((reg["boundary"]["outer"], reg["boundary"]["holes"]), c, n_convex, growth, trig)
            index[k, 1:] = (status, it)
            for i, (x, y) in enumerate(v):
                convex[k, i] = (x, y, *to_world(reg["T"], x, y))
    return index, point, convex


def regions_from_tables(regions, polygons, vertices):
    """The tables as lists of Python floats: per region "T" (3 rows of 4), "bbox", "boundary" and "insets"."""
    regions, polygons, vertices = (np.asarray(a) for a in (regions, polygons, vertices))
    out = [{"T": regions[r, 1:13].reshape(3, 4).tolist(), "bbox": regions[r, 13:17].tolist(),
            "boundary": {"outer": None, "holes": []}, "insets": []} for r in range(len(regions))]
    for region, role, _, v0, nv in polygons.tolist():
        pts = [tuple(x) for x in vertices[v0:v0 + nv].tolist()]
        reg = out[region]
        if role == 0:
            reg["boundary"]["outer"] = pts
        elif role == 1:
            reg["boundary"]["holes"].append(pts)
        elif role == 2:
            reg["insets"].append({"outer": pts, "holes": []})
        else:
            reg["insets"][-1]["holes"].append(pts)
    return out


def tables_from_regions(regions):
    """planar_regions_oracle.extract's regions as the call's three tables."""
    rows, polys, verts = [], [], []

    def add(region, role, inset, pts):
        polys.append([region, role, inset, len(verts), len(pts)])
        verts.extend(np.asarray(pts, np.float64).tolist())

    for r, reg in enumerate(regions):
        rows.append([reg["label"], *np.asarray(reg["transform"])[:3, :4].reshape(-1).tolist(), *reg["bbox"]])
        add(r, 0, -1, reg["boundary"]["outer"])
        for h in reg["boundary"]["holes"]:
            add(r, 1, -1, h)
        for i, ins in enumerate(reg["insets"]):
            add(r, 2, i, ins["outer"])
            for h in ins["holes"]:
                add(r, 3, i, h)
    return (np.array(rows, np.float64).reshape(-1, 17), np.array(polys, np.int32).reshape(-1, 5),
            np.array(verts, np.float64).reshape(-1, 2))


def queries_for(regions, n_grid, seed, box=None):
    """Seeded queries: a random cloud over the regions' extent (and beyond), points on inset and hole edges and at their
    vertices (lifted to the world, some above and below), far points and non-finite ones."""
    rng = np.random.default_rng(seed)
    pts = []
    edge = []
    for reg in regions:
        polys = [(ins["outer"], 2) for ins in reg["insets"]] + [(h, 3) for ins in reg["insets"] for h in ins["holes"]]
        polys += [(h, 1) for h in reg["boundary"]["holes"]]
        for poly, _ in polys:
            for k in rng.choice(len(poly), size=min(len(poly), 3), replace=False):
                a, b = poly[k], poly[(k + 1) % len(poly)]
                t = float(rng.choice([0.0, 0.5, rng.random()]))
                x, y = a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1])
                w = to_world(reg["T"], x, y)
                edge.append([w[0], w[1], w[2] + float(rng.choice([0.0, 0.0, 0.1, -0.2]))])
    edge = np.array(edge).reshape(-1, 3)
    if box is None:
        allw = edge if len(edge) else np.zeros((1, 3))
        box = (allw.min(0) - 0.3, allw.max(0) + 0.3)
    lo, hi = np.asarray(box[0], float), np.asarray(box[1], float)
    pts.append(lo + (hi - lo) * rng.random((n_grid, 3)))
    if len(edge):
        pts.append(edge[rng.permutation(len(edge))[:max(n_grid // 2, 1)]])
    pts.append(np.array([[1e3, -1e3, 5.0], [-50.0, 20.0, -3.0]]))
    pts.append(np.array([[math.nan, 0.0, 0.0], [0.0, math.inf, 0.0], [0.0, 0.0, -math.inf]]))
    return np.ascontiguousarray(np.concatenate(pts), np.float64)
