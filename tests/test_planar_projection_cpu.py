"""CPU: projection onto the planar regions and convex growth without a GPU.  The library header's exact predicates
(csrc/emap_terrain_query.cuh, compiled natively by tests/native/projection_host.cpp) agree with Fraction arithmetic on
near-degenerate inputs; the header's whole query (projection and growth) equals the Python-float oracle bit for bit on
the regions of the five demo terrains from the CPU pipeline; the reference's own tests hold (pruned search = exhaustive
search on terrain.png's grid, every grown vertex inside the boundary, the two region-growing cases); the chosen region
has the least cost and the projection lies on its inset; and malformed host tables are rejected."""
import ctypes as C
import json
import math
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import planar_projection_oracle as PP   # noqa: E402

P = C.c_void_p
D = C.c_double


def load_native():
    """The header's host build (compiled on first use)."""
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libprojection_host.so")
    src = os.path.join(HERE, "native", "projection_host.cpp")
    deps = [src, os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc", "emap_terrain_query.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                        src], check=True)
    lib = C.CDLL(so)
    lib.pqh_orient.argtypes = [D] * 6
    lib.pqh_segments_intersect.argtypes = [D] * 8
    lib.pqh_bounded_side.argtypes = [D, D, P, C.c_int]
    lib.pqh_is_convex5.argtypes = [P, P]
    lib.pqh_sqdist_segment.argtypes = [D] * 6
    lib.pqh_sqdist_segment.restype = D
    lib.pqh_check_tables.argtypes = [P, C.c_int64, P, C.c_int64, P, C.c_int64]
    lib.pqh_project.argtypes = [P, C.c_int64, P, C.c_int64, P, C.c_int64, C.c_int64, P, D, C.c_int, D, P, P, P]
    return lib


@pytest.fixture(scope="module")
def native():
    return load_native()


def host_project(lib, tables, queries, wz=0.0, n_convex=0, growth=1.05):
    """The header's query, one thread per query on the CPU: (index, point, convex) as the call returns them."""
    reg, poly, vert = (np.ascontiguousarray(a, dt) for a, dt in zip(tables, (np.float64, np.int32, np.float64)))
    q = np.ascontiguousarray(queries, np.float64)
    n = len(q)
    index = np.zeros((n, 3), np.int32)
    point = np.zeros((n, 6))
    convex = np.zeros((n, max(n_convex, 1), 5))
    rc = lib.pqh_project(reg.ctypes.data, len(reg), poly.ctypes.data, len(poly), vert.ctypes.data, len(vert), n,
                         q.ctypes.data, wz, n_convex, growth, index.ctypes.data, point.ctypes.data, convex.ctypes.data)
    assert rc == 0
    return index, point, convex[:, :n_convex]


def assert_same_bits(a, b):
    """Equal outputs, NaN for NaN, bit for bit."""
    for x, y in zip(a, b):
        x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
        assert x.shape == y.shape
        assert x.tobytes() == y.tobytes(), np.argwhere(x != y)[:5]


# ---- exact predicates ----
def _exact_orient(a, b, c):
    F = Fraction
    v = (F(a[0]) - F(c[0])) * (F(b[1]) - F(c[1])) - (F(a[1]) - F(c[1])) * (F(b[0]) - F(c[0]))
    return (v > 0) - (v < 0)


def _near_degenerate(rng, count):
    """Triples with c on the line through a and b (rounded), scaled by 2^k, with nudges of an ulp."""
    for _ in range(count):
        k = int(rng.integers(-30, 30))
        a = rng.normal(0, 1, 2) * 2.0 ** k
        b = a + rng.normal(0, 1, 2) * 2.0 ** k
        t = float(rng.choice([0.0, 1.0, 0.5, rng.random(), 1.0 + rng.random(), -rng.random()]))
        c = a + t * (b - a)
        if rng.random() < 0.3:
            c = np.nextafter(c, c + rng.choice([-1.0, 1.0], 2))
        yield tuple(a.tolist()), tuple(b.tolist()), tuple(c.tolist())


def test_orientation_is_exact(native):
    rng = np.random.default_rng(0)
    zero = 0
    for a, b, c in _near_degenerate(rng, 20000):
        want = _exact_orient(a, b, c)
        assert native.pqh_orient(*a, *b, *c) == want
        assert PP.orient(*a, *b, *c) == want
        zero += want == 0
    assert zero > 100
    # an integer lattice scaled by 2^k: every answer is decided by the exact fallback or the filter alike
    for k in (-40, 0, 40):
        s = 2.0 ** k
        pts = [(i * s, j * s) for i in range(-2, 3) for j in range(-2, 3)]
        for a in pts[::3]:
            for b in pts[1::4]:
                for c in pts:
                    assert native.pqh_orient(*a, *b, *c) == _exact_orient(a, b, c)


def _exact_intersect(p1, p2, q1, q2):
    o = [_exact_orient(p1, p2, q1), _exact_orient(p1, p2, q2), _exact_orient(q1, q2, p1), _exact_orient(q1, q2, p2)]
    if o[0] * o[1] < 0 and o[2] * o[3] < 0:
        return True

    def on(c, a, b):
        return min(a[0], b[0]) <= c[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= c[1] <= max(a[1], b[1])
    return any(oo == 0 and on(c, a, b) for oo, c, a, b in
               zip(o, (q1, q2, p1, p2), (p1, p1, q1, q1), (p2, p2, q2, q2)))


def test_segment_intersection_is_exact(native):
    rng = np.random.default_rng(1)
    hits = 0
    for a, b, c in _near_degenerate(rng, 6000):
        d = tuple((np.array(c) + rng.normal(0, 1, 2) * abs(c[0] - a[0] + 1e-300) * rng.choice([0.0, 1.0])).tolist())
        for seg in ((a, b, c, d), (a, b, c, c), (a, a, c, d), (a, c, b, d), (c, d, a, b)):
            want = _exact_intersect(*seg)
            assert bool(native.pqh_segments_intersect(*seg[0], *seg[1], *seg[2], *seg[3])) == want
            assert PP.segments_intersect(*seg) == want
            hits += want
    assert hits > 1000


def _exact_side(p, poly):
    F = Fraction
    n = len(poly)
    for k in range(n):
        a, b = poly[k], poly[(k + 1) % n]
        if _exact_orient(a, b, p) == 0 and min(a[0], b[0]) <= p[0] <= max(a[0], b[0]) and \
                min(a[1], b[1]) <= p[1] <= max(a[1], b[1]):
            return 0
    inside = False
    for k in range(n):
        (ax, ay), (bx, by) = poly[k], poly[(k + 1) % n]
        if (ay > p[1]) != (by > p[1]):
            x = F(ax) + (F(p[1]) - F(ay)) * (F(bx) - F(ax)) / (F(by) - F(ay))
            if x > F(p[0]):
                inside = not inside
    return 1 if inside else -1


def test_bounded_side_is_exact(native):
    rng = np.random.default_rng(2)
    counts = {-1: 0, 0: 0, 1: 0}
    for trial in range(300):
        n = int(rng.integers(3, 12))
        s = 2.0 ** int(rng.integers(-20, 20))
        ang = np.sort(rng.random(n)) * 2 * math.pi
        rad = rng.uniform(0.3, 1.0, n)
        poly = [(float(r * math.cos(t) * s), float(r * math.sin(t) * s)) for r, t in zip(rad, ang)]
        if trial % 5 == 0:
            poly.insert(2, poly[2])                      # a repeated vertex
        xy = np.ascontiguousarray(poly, np.float64)
        pts = [poly[k] for k in range(len(poly))]
        for k in range(len(poly)):                       # on edges (rounded), and an ulp off them
            a, b = np.array(poly[k]), np.array(poly[(k + 1) % len(poly)])
            m = a + float(rng.random()) * (b - a)
            pts += [tuple(m.tolist()), tuple(np.nextafter(m, m + 1).tolist()), tuple(np.nextafter(m, m - 1).tolist())]
        pts += [tuple((rng.normal(0, 0.7, 2) * s).tolist()) for _ in range(10)]
        pts += [(poly[0][0], float(y)) for y in rng.normal(0, 0.5, 3) * s]   # on a vertex's horizontal line
        for p in pts:
            want = _exact_side(p, poly)
            assert native.pqh_bounded_side(p[0], p[1], xy.ctypes.data, len(poly)) == want
            assert PP.bounded_side(p, poly) == want
            counts[want] += 1
    assert min(counts.values()) > 200


def test_is_convex_matches_between_header_and_oracle(native):
    """is_convex_2 on 5 points: regular pentagons, collinear and repeated points (the sub-polygons of n = 3 and 4
    repeat vertices), reflex points and near-collinear ones."""
    rng = np.random.default_rng(3)
    seen = set()
    for trial in range(4000):
        ang = np.sort(rng.random(5)) * 2 * math.pi * float(rng.choice([1.0, -1.0]))
        pts = [(math.cos(t), math.sin(t)) for t in ang]
        kind = trial % 5
        if kind == 1:
            i, j = rng.choice(5, 2, replace=False)
            pts[j] = pts[i]
        elif kind == 2:                                   # n = 3: vertices 0 and 3, 1 and 4 coincide
            pts[3], pts[4] = pts[0], pts[1]
        elif kind == 3:
            a, b = np.array(pts[1]), np.array(pts[3])
            pts[2] = tuple((a + (b - a) * float(rng.choice([0.5, rng.random(), 1.5]))).tolist())
        elif kind == 4:
            pts[2] = (pts[2][0] * float(rng.uniform(0.0, 1.2)), pts[2][1] * float(rng.uniform(0.0, 1.2)))
        x = np.ascontiguousarray([p[0] for p in pts])
        y = np.ascontiguousarray([p[1] for p in pts])
        want = PP.is_convex(pts)
        assert bool(native.pqh_is_convex5(x.ctypes.data, y.ctypes.data)) == want, pts
        seen.add(want)
    assert seen == {True, False}


def test_squared_distance_formula(native):
    rng = np.random.default_rng(4)
    for _ in range(3000):
        p, s, t = (tuple(v) for v in rng.normal(0, 1, (3, 2)).tolist())
        if rng.random() < 0.2:
            t = (s[0], t[1])
        elif rng.random() < 0.2:
            t = (t[0], s[1])
        got = native.pqh_sqdist_segment(*p, *s, *t)
        assert got == PP.sqdist_segment(p, s, t)
        F = Fraction
        vx, vy = F(t[0]) - F(s[0]), F(t[1]) - F(s[1])
        u = max(F(0), min(F(1), ((F(p[0]) - F(s[0])) * vx + (F(p[1]) - F(s[1])) * vy) / (vx * vx + vy * vy)))
        ex = (F(s[0]) + u * vx - F(p[0])) ** 2 + (F(s[1]) + u * vy - F(p[1])) ** 2
        assert abs(got - float(ex)) <= 1e-12 * (1 + float(ex))


# ---- whole queries on the CPU pipeline's regions ----
_TERRAINS = {}


def terrain_tables(name):
    """The five demo terrains through plane_segmentation_oracle and planar_regions_oracle: (tables, window box)."""
    if name not in _TERRAINS:
        pytest.importorskip("cv2")
        import plane_scenes as S
        import plane_segmentation_oracle as PO
        import planar_regions_oracle as RO
        from elevation_mapping_cupy_b200 import _lib
        L = _lib.load()
        png, scale, pos, ln = S.TERRAINS[name]
        g = np.load(S.GOLDEN)
        img = S.terrain_image(g["grey__" + name], scale, seed=5 if name == "holes" else None)
        req = np.array(list(pos) + list(ln), np.float64)
        info, centre = np.zeros(5, np.int32), np.zeros(2)
        c = np.zeros(2)
        assert L.emap_submap_windows(img.shape[0] + 2, S.RES, c.ctypes.data, 1, req.ctypes.data, info.ctypes.data,
                                     centre.ctypes.data) == 0
        _, r0, c0, rows, cols = info.tolist()
        origin = centre + (0.5 * (np.array([rows, cols]) * S.RES) - 0.5 * S.RES)
        p = S.params()
        o = PO.segment(img[r0:r0 + rows, c0:c0 + cols], S.RES, origin, p)
        regions = RO.extract(o["segmentation"], o["planes"], origin, S.RES, p.margin_size,
                             p.extracted_planes_height_offset)
        _TERRAINS[name] = PP.tables_from_regions(regions)
    return _TERRAINS[name]


TERRAIN_NAMES = ["terrain", "slope", "straight_stairs", "real_stairs", "holes"]


@pytest.mark.parametrize("name", TERRAIN_NAMES)
def test_projection_equals_oracle(native, name):
    tables = terrain_tables(name)
    regions = PP.regions_from_tables(*tables)
    assert len(regions) > 0
    q = PP.queries_for(regions, 120, seed=TERRAIN_NAMES.index(name))
    for wz in (0.0, 0.1):
        got = host_project(native, tables, q, wz)
        want = PP.project(regions, q, wz)
        assert_same_bits(got[:2], want[:2])
    assert (got[0][:, 0] >= 0).sum() > 100 and (got[0][:, 1] == PP.INVALID_QUERY).sum() == 3


@pytest.mark.parametrize("name", TERRAIN_NAMES)
def test_growth_equals_oracle(native, name):
    tables = terrain_tables(name)
    regions = PP.regions_from_tables(*tables)
    q = PP.queries_for(regions, 4, seed=10 + TERRAIN_NAMES.index(name))
    q = np.concatenate([q[:6], q[-1:]])
    statuses = set()
    for n, g in ((3, 1.01), (4, 1.11), (5, 1.21), (6, 1.05), (16, 1.05)):
        got = host_project(native, tables, q, 0.0, n, g)
        want = PP.project(regions, q, 0.0, n, g)
        assert_same_bits(got, want)
        statuses |= set(got[0][:, 1].tolist())
    assert PP.GROWN in statuses


def test_reference_convex_approximation_on_terrain(native):
    """testConvexApproximation.cpp on terrain.png's 3 m window: its query grid, penalty 0.1 |z|: the pruned, sorted
    search equals the exhaustive one, and every vertex grown inside the boundary is inside it (holes included) for
    n = 3 .. 6 and growth 1.01, 1.11, 1.21."""
    tables = terrain_tables("terrain")
    regions = PP.regions_from_tables(*tables)
    q = np.array([[x, y, z] for x in np.arange(-1.5, 1.5, 0.75) for y in np.arange(-1.5, 1.5, 0.75)
                  for z in np.arange(-1.25, 1.25, 0.625)])
    for p in q.tolist():
        a, b = PP.best_pruned(p, regions, 0.1), PP.best_exhaustive(p, regions, 0.1)
        assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2]
    for n in range(3, 7):
        for g in (1.01, 1.11, 1.21):
            index, point, convex = host_project(native, tables, q, 0.1, n, g)
            assert (index[:, 0] >= 0).all()
            for k in range(len(q)):
                reg = regions[index[k, 0]]
                shape = (reg["boundary"]["outer"], reg["boundary"]["holes"])
                for v in convex[k, :, :2].tolist():
                    assert PP.inside_with_holes(tuple(v), shape)


def _single_region(outer, holes, inset=None):
    T = np.eye(4)
    reg = {"label": 1, "transform": T, "bbox": np.array([0.0, 0.0, 0.0, 0.0]),
           "boundary": {"outer": np.array(outer, float), "holes": [np.array(h, float) for h in holes]},
           "insets": [{"outer": np.array(inset if inset is not None else outer, float), "holes": []}]}
    return PP.tables_from_regions([reg])


def test_reference_region_growing_cases(native):
    with open(os.path.join(HERE, "golden", "region_growing_cases.json")) as f:
        cases = json.load(f)["cases"]
    for name, c in cases.items():
        tables = _single_region(c["outer"], c["holes"])
        regions = PP.regions_from_tables(*tables)
        q = np.array([[c["center"][0], c["center"][1], 0.0]])
        got = host_project(native, tables, q, 0.0, c["n_vertices"], c["growth_factor"])
        assert_same_bits(got, PP.project(regions, q, 0.0, c["n_vertices"], c["growth_factor"]))
        assert got[1][0, 1:3].tolist() == c["center"]
        v = [tuple(p) for p in got[2][0, :, :2].tolist()]
        assert PP.is_convex(v)
        shape = (regions[0]["boundary"]["outer"], regions[0]["boundary"]["holes"])
        assert all(PP.inside_with_holes(p, shape) for p in v), name
    assert got[0][0, 1] == PP.GROWN and got[0][0, 2] > 1          # debug_case grows


@pytest.mark.parametrize("name", ["terrain", "holes"])
def test_chosen_region_has_least_cost_and_projection_on_inset(native, name):
    tables = terrain_tables(name)
    regions = PP.regions_from_tables(*tables)
    q = PP.queries_for(regions, 40, seed=20)
    index, point, _ = host_project(native, tables, q, 0.1)
    for k, p in enumerate(q.tolist()):
        r = index[k, 0]
        if r < 0:
            continue
        costs = []
        for reg in regions:
            pl = PP.to_plane(reg["T"], p)
            c = PP.project_region((pl[0], pl[1]), reg)
            w = PP.to_world(reg["T"], *c)
            costs.append(((p[0] - w[0]) ** 2 + (p[1] - w[1]) ** 2 + (p[2] - w[2]) ** 2) + 0.1 * abs(w[2]))
        assert point[k, 0] == min(costs) and costs.index(min(costs)) == r
        # in an inset and not strictly in one of its holes, or (a projection onto an edge is rounded) within 1e-10
        # of an inset's edge
        c = tuple(point[k, 1:3].tolist())
        insets = regions[r]["insets"]
        near = min(PP.sq_distance_to_shape(c, (ins["outer"], ins["holes"])) for ins in insets)
        assert near <= 1e-20 or any(PP.bounded_side(c, ins["outer"]) >= 0 and
                                    all(PP.bounded_side(c, h) <= 0 for h in ins["holes"]) for ins in insets)


def test_query_inside_inset_is_unchanged(native):
    outer = [(0.0, 0.0), (2.0, 0.0), (2.0, 2.0), (0.0, 2.0)]
    hole = [(0.8, 0.8), (1.2, 0.8), (1.2, 1.2), (0.8, 1.2)]
    tables = _single_region(outer, [], inset=None)
    reg, poly, vert = tables
    reg[0, 1:13] = [0.0, -1.0, 0.0, 0.5, 1.0, 0.0, 0.0, -0.25, 0.0, 0.0, 1.0, 0.3]    # a rotation about z and a shift
    # an inset hole: an inset outer followed by its hole
    poly = np.vstack([poly, [[0, 3, 0, len(vert), 4]]]).astype(np.int32)
    vert = np.vstack([vert, hole])
    tables = (reg, poly, vert)
    regions = PP.regions_from_tables(*tables)
    rng = np.random.default_rng(5)
    pl = rng.uniform(0.05, 1.95, (200, 2))
    pl = pl[~((np.abs(pl - 1.0) <= 0.2).all(1))]
    dz = rng.uniform(-1, 1, len(pl))
    q = np.array([PP.to_world(regions[0]["T"], x, y) for x, y in pl.tolist()])
    q[:, 2] += dz
    index, point, _ = host_project(native, tables, q, 0.2)
    assert_same_bits((index, point), PP.project(regions, q, 0.2)[:2])
    # the plane-frame query is kept as it is: the cost is the distance to its world point (dz^2 up to rounding) plus
    # the penalty
    kept = np.array([PP.to_plane(regions[0]["T"], p)[:2] for p in q.tolist()])
    assert np.array_equal(point[:, 1:3], kept) and np.abs(kept - pl).max() < 1e-12
    w = np.array([PP.to_world(regions[0]["T"], x, y) for x, y in kept.tolist()])
    assert np.abs(w[:, 2] - (q[:, 2] - dz)).max() < 1e-12
    d = q - w
    assert np.array_equal(point[:, 0], ((d[:, 0] ** 2 + d[:, 1] ** 2) + d[:, 2] ** 2) + 0.2 * np.abs(w[:, 2]))
    # a query in the hole goes to the hole's edge
    index, point, _ = host_project(native, tables, np.array([PP.to_world(regions[0]["T"], 1.1, 1.0)]), 0.0)
    assert tuple(point[0, 1:3]) == (1.2, 1.0)


def _bad_tables():
    good = _single_region([(0.0, 0.0), (1.0, 0.0), (1.0, 1.0)], [[(0.2, 0.2), (0.3, 0.2), (0.3, 0.3)]])
    reg, poly, vert = good
    assert poly[:, 1].tolist() == [0, 1, 2]
    out = {}

    def mut(name, f):
        r, p, v = reg.copy(), poly.copy(), vert.copy()
        res = f(r, p, v)
        out[name] = res if res is not None else (r, p, v)

    mut("region out of range", lambda r, p, v: p.__setitem__((2, 0), 1))
    mut("negative region", lambda r, p, v: p.__setitem__((0, 0), -1))
    mut("role out of range", lambda r, p, v: p.__setitem__((1, 1), 4))
    mut("inset first", lambda r, p, v: p.__setitem__((0, 1), 2))
    mut("no inset", lambda r, p, v: (r, p[:2].copy(), v))
    mut("boundary inset index", lambda r, p, v: p.__setitem__((1, 2), 0))
    mut("inset index", lambda r, p, v: p.__setitem__((2, 2), 1))
    mut("vertex range", lambda r, p, v: p.__setitem__((2, 4), 7))
    mut("negative first vertex", lambda r, p, v: p.__setitem__((1, 3), -1))
    mut("no vertex", lambda r, p, v: p.__setitem__((1, 4), 0))
    mut("region without polygons", lambda r, p, v: (np.vstack([r, r]), p, v))
    mut("polygons without regions", lambda r, p, v: (r[:0], p, v))
    mut("descending regions", lambda r, p, v: (np.vstack([r, r]), np.vstack([p + [1, 0, 0, 0, 0], p]), v))
    return good, out


def test_host_tables_are_checked(native):
    good, bad = _bad_tables()

    def check(t):
        r, p, v = (np.ascontiguousarray(a, dt) for a, dt in zip(t, (np.float64, np.int32, np.float64)))
        return native.pqh_check_tables(r.ctypes.data, len(r), p.ctypes.data, len(p), v.ctypes.data, len(v))
    assert check(good) == 0
    two = (np.vstack([good[0], good[0]]), np.vstack([good[1], good[1] + [1, 0, 0, 0, 0]]), good[2])
    assert check(two) == 0
    for name, t in bad.items():
        assert check(t) == 1, name
