"""NumPy restatement of the reference's polygon safety check, the yardstick of the engine's
emap_polygon_traversability:
  EM.py:837-889 get_polygon_traversability, CK.py:509-654 polygon_mask_kernel, traversability_polygon.py:10-63
(EM.py = elevation_mapping_cupy/script/elevation_mapping_cupy/elevation_mapping.py, CK.py = kernels/custom_kernels.py).

The mask follows the kernel's integer geometry exactly (and is checked against the reference's own kernel source,
`ref_polygon_mask`); the statistics are fp32 elementwise with fp64 sums; the hull is an exact integer monotone chain
(shapely's hull of the same points, collinear vertices removed), as a ring that starts at its smallest (row, col) vertex
and runs counter-clockwise in (row, col).
"""
import ctypes as C
import os
import subprocess

import numpy as np

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def h16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def shoelace_f32(p):
    """traversability_polygon.py:46-51 on fp32 vertices: terms i = 0..n-1 with p1 = p[i-1], summed in order in fp32."""
    p = np.asarray(p, np.float32)
    area = F(0)
    for i in range(len(p)):
        a, b = p[i - 1], p[i]
        area = F(area + F(F(F(a[0] * b[1]) - F(a[1] * b[0])) / F(2.0)))
    return abs(area)


def clip_polygon(poly, center, W, resolution):
    """EM.py:847-854 in fp32, map_length = (W - 2) * resolution: (clipped vertices, bbox [xmin, ymin, xmax, ymax])."""
    p = np.array(poly, np.float32).reshape(-1, 2)
    half, res = F(0.5 * (W - 2) * resolution), F(resolution)
    c = np.asarray(center, np.float32)[:2]
    lo, hi = F(F(c - half) + res), F(F(c + half) - res)
    p = np.minimum(np.maximum(p, lo), hi).astype(np.float32)
    return p, np.concatenate([p.min(axis=0), p.max(axis=0)]).astype(np.float32)


def vertex_cells(v, c, resolution, W):
    """CK.py:580-603: float16 coordinate and centre, difference in float, / float resolution, + 0.5*W in double,
    truncated, clamped to [0, W-1] through float16 (exact for W - 1 <= 2048)."""
    d = (h16(v) - h16(c)).astype(np.float32)
    q = (d / F(resolution)).astype(np.float32).astype(np.float64) + 0.5 * W
    return np.clip(np.trunc(np.clip(q, -1e9, 1e9)), 0, W - 1).astype(np.int64)


def _orient(px, py, qx, qy, rx, ry):
    v = (qy - py) * (rx - qx) - (qx - px) * (ry - qy)
    return np.where(v == 0, 0, np.where(v > 0, 1, 2))


def _on_seg(px, py, qx, qy, rx, ry):
    return (qx <= np.maximum(px, rx)) & (qx >= np.minimum(px, rx)) & (qy <= np.maximum(py, ry)) & (qy >= np.minimum(py, ry))


def polygon_mask(clipped, bbox, center, resolution, W):
    """CK.py:605-649 for every cell: (W, W) uint8."""
    cx, cy = np.float32(center[0]), np.float32(center[1])
    vx = vertex_cells(clipped[:, 0], cx, resolution, W)
    vy = vertex_cells(clipped[:, 1], cy, resolution, W)
    bx0, bx1 = vertex_cells(bbox[[0, 2]], cx, resolution, W)
    by0, by1 = vertex_cells(bbox[[1, 3]], cy, resolution, W)
    cnt = np.zeros((W, W), np.int64)
    on = np.zeros((W, W), bool)
    n = len(clipped)
    ex = 100000
    for j in range(n):
        ax, ay, bx, by = vx[j], vy[j], vx[(j + 1) % n], vy[(j + 1) % n]
        # only cells of the bbox whose column lies in the edge's column range can be affected
        c_lo, c_hi = max(by0, min(ay, by)), min(by1, max(ay, by))
        if c_lo > c_hi or bx0 > bx1:
            continue
        x, y = np.meshgrid(np.arange(bx0, bx1 + 1), np.arange(c_lo, c_hi + 1), indexing="ij")
        o1, o2 = _orient(ax, ay, bx, by, x, y), _orient(ax, ay, bx, by, ex, y)
        o3, o4 = _orient(x, y, ex, y, ax, ay), _orient(x, y, ex, y, bx, by)
        hit = (((o1 != o2) & (o3 != o4)) | ((o1 == 0) & _on_seg(ax, ay, x, y, bx, by))
               | ((o2 == 0) & _on_seg(ax, ay, ex, y, bx, by)) | ((o3 == 0) & _on_seg(x, y, ax, ay, ex, y))
               | ((o4 == 0) & _on_seg(x, y, bx, by, ex, y)))
        col = _orient(ax, ay, x, y, bx, by) == 0
        on[bx0:bx1 + 1, c_lo:c_hi + 1] |= hit & col & _on_seg(ax, ay, x, y, bx, by)
        cross = hit & ~col & (((ay <= y) & (by > y)) | ((ay > y) & (by <= y)))
        cnt[bx0:bx1 + 1, c_lo:c_hi + 1] += cross
    return (on | (cnt % 2 == 1)).astype(np.uint8)


def _cross(o, a, b):
    return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])


def convex_ring(points):
    """Convex hull of integer (row, col) points without collinear vertices, as a closed ring starting at the smallest
    (row, col) and counter-clockwise in (row, col); None when the hull is empty, a point or a segment."""
    pts = sorted(set(map(tuple, np.asarray(points, np.int64).reshape(-1, 2).tolist())))
    if len(pts) < 3:
        return None
    lower, upper = [], []
    for p in pts:
        while len(lower) >= 2 and _cross(lower[-2], lower[-1], p) <= 0:
            lower.pop()
        lower.append(p)
    for p in reversed(pts):
        while len(upper) >= 2 and _cross(upper[-2], upper[-1], p) <= 0:
            upper.pop()
        upper.append(p)
    hull = lower[:-1] + upper[:-1]           # counter-clockwise in (row, col), starts at the smallest (row, col)
    if len(hull) < 3:
        return None
    return np.array(hull + hull[:1], np.int64)


def polygon_traversability(poly, center, W, resolution, valid, checker, safe_thresh, safe_min_thresh, max_unsafe_n):
    """EM.py:837-889.  valid, checker: (W, W) fp32 planes.  Returns a dict with result [is_safe, t, area], mask (W, W),
    ring (n, 2) metres (empty (0, 2) if none), ring_idx (interior indices), over count, clipped_area, t64."""
    p32 = np.asarray(poly, np.float32).reshape(-1, 2)
    area = shoelace_f32(p32)
    clipped, bbox = clip_polygon(p32, center, W, resolution)
    clipped_area = shoelace_f32(clipped)
    mask = polygon_mask(clipped, bbox, center, resolution, W)
    m = mask[1:-1, 1:-1].astype(np.float32)
    v = np.asarray(valid, np.float32)[1:-1, 1:-1]
    ch = np.asarray(checker, np.float32)[1:-1, 1:-1]
    with np.errstate(invalid="ignore"):
        untrav = np.where(v > F(0.5), (F(1) - ch).astype(np.float32), F(0)).astype(np.float32)
        masked = (untrav * m).astype(np.float32)
        mvalid = (v * m).astype(np.float32)
        s_m, s_v = masked.astype(np.float64).sum(), mvalid.astype(np.float64).sum()
        t64 = s_m / s_v if s_v > 0 else 0.0
        over = masked > F(1.0 - safe_thresh)
        mx = masked.max()
        is_safe = not (over.sum() > max_unsafe_n) and not (mx > F(1.0 - safe_min_thresh))
    if clipped_area < F(0.001):
        is_safe = False
    ring_idx = convex_ring(np.argwhere(over))
    if ring_idx is None:
        ring = np.zeros((0, 2))
    else:
        c = np.asarray(center, np.float32)[:2].astype(np.float64)
        ring = c.reshape(1, 2) + (ring_idx.astype(np.float64) - W / 2.0) * resolution
    return dict(result=np.array([float(is_safe), float(F(t64)), float(area)]), mask=mask, ring=ring, ring_idx=ring_idx,
                over=int(over.sum()), clipped_area=clipped_area, t64=t64)


def same_ring(a, b):
    """Two closed rings are equal up to start vertex and direction."""
    a, b = np.asarray(a)[:-1], np.asarray(b)[:-1]
    if a.shape != b.shape:
        return False
    if len(a) == 0:
        return True
    for r in (b, b[::-1]):
        for s in range(len(r)):
            if np.array_equal(a, np.roll(r, -s, axis=0)):
                return True
    return False


# ---- seeded polygons ---------------------------------------------------------------------------
def star(rng, n, r_lo, r_hi, cx=0.0, cy=0.0):
    ang = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = rng.uniform(r_lo, r_hi, n)
    return np.stack([cx + r * np.cos(ang), cy + r * np.sin(ang)], 1).astype(np.float32)


def mask_cases(W, resolution):
    """(name, polygon (n, 2) fp32, centre (3,) fp32) covering the branches of CK.py:609-649.  L = half the map length."""
    rng = np.random.default_rng(7)
    L = 0.5 * (W - 2) * resolution
    res = resolution
    cases = [
        ("triangle", np.array([[0, 0], [2, 0], [0, 2]], np.float32), (0, 0)),          # test_elevation_mapping.py:101
        ("concave", star(rng, 12, 0.2 * L, 0.8 * L), (0, 0)),
        ("star64", star(rng, 64, 0.1 * L, 0.9 * L), (0, 0)),
        ("star1000", star(rng, 1000, 0.3 * L, 0.7 * L), (0, 0)),
        # a bow tie: two triangles touching at one vertex
        ("self_touching", np.array([[-0.5 * L, -0.5 * L], [0.5 * L, 0.5 * L], [0.5 * L, -0.5 * L],
                                    [-0.5 * L, 0.5 * L]], np.float32), (0, 0)),
        # vertices on cell boundaries: horizontal and vertical edges along the ray and through cell centres
        ("grid_rect", (np.array([[-10, -7], [12, -7], [12, 9], [-10, 9]], np.float64) * res).astype(np.float32), (0, 0)),
        ("grid_stairs", (np.array([[-20, -20], [0, -20], [0, 0], [20, 0], [20, 20], [-20, 20]], np.float64)
                         * res).astype(np.float32), (0, 0)),
        ("partly_outside", np.array([[0.5 * L, -0.3 * L], [1.6 * L, -0.2 * L], [1.4 * L, 0.4 * L],
                                     [0.4 * L, 0.3 * L]], np.float32), (0, 0)),
        ("fully_outside", np.array([[2 * L, 2 * L], [3 * L, 2 * L], [3 * L, 3 * L]], np.float32), (0, 0)),
        ("moved", star(rng, 16, 0.2 * L, 0.6 * L, 123.45, -67.8), (123.45, -67.8)),
        ("moved_far", star(rng, 9, 0.3 * L, 0.7 * L, -1031.3, 517.9), (-1031.3, 517.9)),
    ]
    return [(name, p.astype(np.float32), np.array([c[0], c[1], 0.0], np.float32)) for name, p, c in cases]


# ---- the reference's own kernel source, built for the host (only where the reference checkout exists) -----------------
def ref_mask_available():
    from oracle import build_ref
    return os.path.isdir(build_ref.REF_ROOT)


def build_ref_mask(W, resolution, out_dir):
    """Compiles CK.py's polygon_mask_kernel(W, W, resolution), unmodified, through oracle/ref_shim.h with g++ into
    out_dir; returns the loaded library (function ref_polygon_mask)."""
    from oracle import build_ref
    ck = build_ref._load_with_stub(os.path.join(build_ref.REF_ROOT, "kernels", "custom_kernels.py"), "ref_ck_polygon")
    src = '#include "ref_shim.h"\n' + build_ref._emit(ck.polygon_mask_kernel(W, W, resolution), "polygon_mask", False)
    tag = f"{W}_{resolution!r}".replace(".", "p")
    cc, so = os.path.join(out_dir, f"ref_polygon_{tag}.cc"), os.path.join(out_dir, f"libref_polygon_{tag}.so")
    with open(cc, "w") as f:
        f.write(src)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-w", "-I", os.path.join(ROOT, "oracle"), "-shared",
                    "-fPIC", "-o", so, cc], check=True)
    return C.CDLL(so)


def ref_polygon_mask(lib, clipped, bbox, center, W):
    """The reference kernel over every cell, as EM.py:856-864 launches it."""
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    poly = np.ascontiguousarray(clipped, np.float32)
    cx, cy = np.array([center[0]], np.float32), np.array([center[1]], np.float32)
    n = np.array([len(poly)], np.int16)
    bb = np.ascontiguousarray(bbox, np.float32)
    mask = np.full(W * W, -1, np.float32)
    lib.ref_polygon_mask(C.c_longlong(W * W), p(poly), p(cx), p(cy), p(n), p(bb), p(mask), C.c_int(0))
    return mask.reshape(W, W)
