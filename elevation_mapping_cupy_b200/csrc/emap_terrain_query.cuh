// emap_terrain_query.cuh -- queries on the planar terrain's region tables (emap_project_to_planar_regions), sm_90a.
//
// Reference: convex_plane_decomposition's SegmentedPlaneProjection (getBestPlanarRegionAtPositionInWorld, searched
// exhaustively as testConvexApproximation.cpp's naive version does), PlanarRegion.cpp's frame maps, GeometryUtils.h and
// ConvexRegionGrowing.cpp (growConvexPolygonInsideShape).  include/emap.h states the contract, DESIGN.md §4l the
// restatement.  Predicates are exact (a double filter with Shewchuk's orient2d error bound, then expansion arithmetic),
// constructions are double arithmetic in a fixed order without contraction.
//
// The per-query functions are __host__ __device__: on the device one warp runs them, its lanes striding over the edges
// of the polygon in hand and combining their results with votes and shuffles; on the host (tests/native/
// projection_host.cpp) one thread runs them with the same arithmetic, so the two give the same bits.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#if defined(__CUDACC__)
#define PQ_HD __host__ __device__ __forceinline__
#define PQ_COLD __host__ __device__ __noinline__   // the exact fallback: kept out of the callers' code
#else
#define PQ_HD inline
#define PQ_COLD inline
#endif

#if defined(__CUDA_ARCH__)
#define PQ_MUL(a, b) __dmul_rn((a), (b))
#define PQ_ADD(a, b) __dadd_rn((a), (b))
#define PQ_SUB(a, b) __dsub_rn((a), (b))
#define PQ_DIV(a, b) __ddiv_rn((a), (b))
#define PQ_SQRT(a) __dsqrt_rn((a))
#define PQ_FMA(a, b, c) __fma_rn((a), (b), (c))
#define PQ_LANE ((int)(threadIdx.x & 31))
#define PQ_LANES 32
#else
#define PQ_MUL(a, b) ((double)(a) * (double)(b))
#define PQ_ADD(a, b) ((double)(a) + (double)(b))
#define PQ_SUB(a, b) ((double)(a) - (double)(b))
#define PQ_DIV(a, b) ((double)(a) / (double)(b))
#define PQ_SQRT(a) std::sqrt((double)(a))
#define PQ_FMA(a, b, c) std::fma((a), (b), (c))
#define PQ_LANE 0
#define PQ_LANES 1
#endif

#define PQ_ROW 17                  // emap.h's EMAP_REGION_ROW
#define PQ_POLY 5                  // emap.h's EMAP_REGION_POLYGON
#define PQ_MAX_CONVEX 64           // emap.h's EMAP_CONVEX_MAX_VERTICES
#define PQ_MAX_ITER 1000           // ConvexRegionGrowing.cpp's maxIter
#define PQ_WARPS 8                 // queries (warps) per block

// per-query status (index[3 i + 1]), emap.h's EMAP_PROJECTION_*
enum { PQ_GROWN = 0, PQ_ZERO_RADIUS = 1, PQ_MAX_ITERATIONS = 2, PQ_NO_REGION = 3, PQ_INVALID_QUERY = 4,
       PQ_BAD_TABLE = 5 };
// polygon roles of the region tables
enum { PQ_BOUNDARY = 0, PQ_BOUNDARY_HOLE = 1, PQ_INSET = 2, PQ_INSET_HOLE = 3 };

// ---- warp combination (the identity on the host) ----
PQ_HD bool pq_any(bool v) {
#if defined(__CUDA_ARCH__)
  return __any_sync(0xffffffffu, v);
#else
  return v;
#endif
}

PQ_HD bool pq_odd(bool v) {            // parity of the lanes' flags: XOR of a ballot
#if defined(__CUDA_ARCH__)
  return __popc(__ballot_sync(0xffffffffu, v)) & 1;
#else
  return v;
#endif
}

PQ_HD void pq_sync() {
#if defined(__CUDA_ARCH__)
  __syncwarp();
#endif
}

// least d over the lanes (never a NaN: `o < m`), the same on every lane
PQ_HD double pq_min(double m) {
#if defined(__CUDA_ARCH__)
  for (int s = 16; s; s >>= 1) {
    const double o = __shfl_xor_sync(0xffffffffu, m, s);
    m = o < m ? o : m;
  }
#endif
  return m;
}

// the (d, k) key of the first least d over the lanes (k = INT_MAX: the lane saw no edge), the same on every lane.
// Each lane scans its edges in ascending order with a strict `<`, so for distances that are not NaN this is the
// sequential scan's first minimum.
PQ_HD void pq_min_key(double& d, int& k) {
#if defined(__CUDA_ARCH__)
  for (int s = 16; s; s >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, d, s);
    const int ok = __shfl_xor_sync(0xffffffffu, k, s);
    if (ok != INT_MAX && (k == INT_MAX || od < d || (od == d && ok < k))) {
      d = od;
      k = ok;
    }
  }
#endif
}

// ---- exact predicates ----
PQ_HD void pq_two_sum(double a, double b, double& s, double& e) {
  s = PQ_ADD(a, b);
  const double bv = PQ_SUB(s, a);
  const double av = PQ_SUB(s, bv);
  e = PQ_ADD(PQ_SUB(a, av), PQ_SUB(b, bv));
}

PQ_HD void pq_two_diff(double a, double b, double& s, double& e) {
  s = PQ_SUB(a, b);
  const double bv = PQ_SUB(a, s);
  const double av = PQ_ADD(s, bv);
  e = PQ_ADD(PQ_SUB(a, av), PQ_SUB(bv, b));
}

// Shewchuk's Grow-Expansion with zero elimination: e[0 .. m) + b, in place; returns the new length.
PQ_HD int pq_grow_expansion(double* e, int m, double b) {
  double q = b;
  int k = 0;
  for (int i = 0; i < m; i++) {
    double s, t;
    pq_two_sum(q, e[i], s, t);
    if (t != 0.0) e[k++] = t;
    q = s;
  }
  if (q != 0.0 || k == 0) e[k++] = q;
  return k;
}

// exact sign of (a - c) x (b - c) from 16 exact products summed in an expansion
PQ_COLD int pq_orient_exact(double ax, double ay, double bx, double by, double cx, double cy) {
  double l[4], r[4];               // acx, bcy (left); acy, bcx (right): each a two-term exact difference
  pq_two_diff(ax, cx, l[0], l[1]);
  pq_two_diff(by, cy, l[2], l[3]);
  pq_two_diff(ay, cy, r[0], r[1]);
  pq_two_diff(bx, cx, r[2], r[3]);
  double e[17];
  int m = 0;
  for (int i = 0; i < 2; i++)
    for (int j = 2; j < 4; j++) {
      double p, t;
      p = PQ_MUL(l[i], l[j]);
      t = PQ_FMA(l[i], l[j], -p);
      m = pq_grow_expansion(e, m, p);
      m = pq_grow_expansion(e, m, t);
      p = PQ_MUL(r[i], r[j]);
      t = PQ_FMA(r[i], r[j], -p);
      m = pq_grow_expansion(e, m, -p);
      m = pq_grow_expansion(e, m, -t);
    }
  const double top = e[m - 1];
  return (top > 0.0) - (top < 0.0);
}

// orientation of (a, b, c): 1 counter-clockwise, -1 clockwise, 0 collinear, exact for finite coordinates whose
// products neither overflow nor underflow.  The double filter is Shewchuk's orient2d stage A bound.
PQ_HD int pq_orient(double ax, double ay, double bx, double by, double cx, double cy) {
  const double detleft = PQ_MUL(PQ_SUB(ax, cx), PQ_SUB(by, cy));
  const double detright = PQ_MUL(PQ_SUB(ay, cy), PQ_SUB(bx, cx));
  const double det = PQ_SUB(detleft, detright);
  double detsum;
  if (detleft > 0.0) {
    if (detright <= 0.0) return (det > 0.0) - (det < 0.0);
    detsum = PQ_ADD(detleft, detright);
  } else if (detleft < 0.0) {
    if (detright >= 0.0) return (det > 0.0) - (det < 0.0);
    detsum = PQ_SUB(-detleft, detright);
  } else {
    return (det > 0.0) - (det < 0.0);
  }
  const double bound = PQ_MUL(3.3306690738754716e-16, detsum);     // (3 + 16 eps) eps, eps = 2^-53, rounded up
  if (det >= bound || -det >= bound) return (det > 0.0) - (det < 0.0);
  return pq_orient_exact(ax, ay, bx, by, cx, cy);
}

PQ_HD bool pq_in_box(double px, double py, double ax, double ay, double bx, double by) {
  return (ax < bx ? ax <= px && px <= bx : bx <= px && px <= ax) &&
         (ay < by ? ay <= py && py <= by : by <= py && py <= ay);
}

// CGAL::do_intersect of the closed segments (p1, p2) and (q1, q2): touching and collinear overlap count
PQ_HD bool pq_segments_intersect(double p1x, double p1y, double p2x, double p2y, double q1x, double q1y, double q2x,
                                 double q2y) {
  if (fmax(p1x, p2x) < fmin(q1x, q2x) || fmax(q1x, q2x) < fmin(p1x, p2x) || fmax(p1y, p2y) < fmin(q1y, q2y) ||
      fmax(q1y, q2y) < fmin(p1y, p2y))
    return false;
  const int o1 = pq_orient(p1x, p1y, p2x, p2y, q1x, q1y), o2 = pq_orient(p1x, p1y, p2x, p2y, q2x, q2y);
  const int o3 = pq_orient(q1x, q1y, q2x, q2y, p1x, p1y), o4 = pq_orient(q1x, q1y, q2x, q2y, p2x, p2y);
  if (o1 * o2 < 0 && o3 * o4 < 0) return true;
  return (o1 == 0 && pq_in_box(q1x, q1y, p1x, p1y, p2x, p2y)) || (o2 == 0 && pq_in_box(q2x, q2y, p1x, p1y, p2x, p2y)) ||
         (o3 == 0 && pq_in_box(p1x, p1y, q1x, q1y, q2x, q2y)) || (o4 == 0 && pq_in_box(p2x, p2y, q1x, q1y, q2x, q2y));
}

// One edge's part of CGAL::bounded_side_2 for (px, py): `on` when the point lies on the closed edge, `cross` when the
// edge crosses the ray from the point towards +x (half-open in y, so a vertex on the ray counts once).  A point on no
// edge is inside iff the crossings are odd (the even-odd rule, the same for every ray of a closed polygonal curve).
PQ_HD void pq_edge_side(double px, double py, double ax, double ay, double bx, double by, bool& on, bool& cross) {
  on = false;
  cross = false;
  if (!pq_in_box(px, py, ax, ay, bx, by) && (ay > py) == (by > py)) return;
  const int o = pq_orient(ax, ay, bx, by, px, py);
  on = o == 0 && pq_in_box(px, py, ax, ay, bx, by);
  if ((ay > py) != (by > py)) cross = by > ay ? o > 0 : o < 0;
}

PQ_HD bool pq_less_xy(double ax, double ay, double bx, double by) { return ax < bx || (ax == bx && ay < by); }

// CGAL's is_convex_2 on 5 points (ConvexRegionGrowing.cpp's sub-polygon): orientation, less_xy and equality, equal
// consecutive points skipped.
PQ_HD bool pq_is_convex5(const double* x, const double* y) {
  const int n = 5;
  int first = 0, previous = 0, current = 1, next = 2;
  while (x[previous] == x[current] && y[previous] == y[current]) {
    current = next;
    ++next;
    if (next == n) return true;
  }
  bool cw = false, ccw = false;
  bool order = pq_less_xy(x[previous], y[previous], x[current], y[current]);
  int changes = 0;
  do {
    for (;;) {
      const int o = pq_orient(x[previous], y[previous], x[current], y[current], x[next], y[next]);
      if (o < 0) {
        cw = true;
      } else if (o > 0) {
        ccw = true;
      } else if (x[current] == x[next] && y[current] == y[next]) {
        if (next == first) first = current;
        ++next;
        if (next == n) next = first;
        continue;
      }
      break;
    }
    const bool new_order = pq_less_xy(x[current], y[current], x[next], y[next]);
    if (order != new_order) changes++;
    if (changes > 2) return false;
    if (cw && ccw) return false;
    previous = current;
    current = next;
    ++next;
    if (next == n) next = first;
    order = new_order;
  } while (previous != first);
  return true;
}

// ---- constructions ----
// CGAL::squared_distance(point, segment source -> target), Cartesian (Distance_2/Point_2_Segment_2.h with
// line_from_pointsC2 and Point_2_Line_2.h), restated from CGAL's published source.
PQ_HD double pq_sqdist_segment(double px, double py, double sx, double sy, double tx, double ty) {
  const double dx = PQ_SUB(px, sx), dy = PQ_SUB(py, sy);
  const double vx = PQ_SUB(tx, sx), vy = PQ_SUB(ty, sy);
  const double d = PQ_ADD(PQ_MUL(dx, vx), PQ_MUL(dy, vy));
  if (d <= 0.0) return PQ_ADD(PQ_MUL(dx, dx), PQ_MUL(dy, dy));
  const double e = PQ_ADD(PQ_MUL(vx, vx), PQ_MUL(vy, vy));
  if (d > e) {
    const double ex = PQ_SUB(px, tx), ey = PQ_SUB(py, ty);
    return PQ_ADD(PQ_MUL(ex, ex), PQ_MUL(ey, ey));
  }
  double a, b, c;
  if (sy == ty) {
    a = 0.0;
    if (tx > sx) { b = 1.0; c = -sy; }
    else if (tx == sx) { b = 0.0; c = 0.0; }
    else { b = -1.0; c = sy; }
  } else if (tx == sx) {
    b = 0.0;
    if (ty > sy) { a = -1.0; c = sx; }
    else { a = 1.0; c = -sx; }
  } else {
    a = PQ_SUB(sy, ty);
    b = PQ_SUB(tx, sx);
    c = PQ_SUB(PQ_MUL(-sx, a), PQ_MUL(sy, b));
  }
  const double w = PQ_ADD(PQ_ADD(PQ_MUL(a, px), PQ_MUL(b, py)), c);
  return PQ_DIV(PQ_MUL(w, w), PQ_ADD(PQ_MUL(a, a), PQ_MUL(b, b)));
}

// GeometryUtils.h's projectToClosestPoint(point, segment), as written (Eigen's norm and dot, std::max / std::min)
PQ_HD void pq_project_segment(double px, double py, double sx, double sy, double tx, double ty, double& ox,
                              double& oy) {
  const double vx = PQ_SUB(tx, sx), vy = PQ_SUB(ty, sy);
  const double len = PQ_SQRT(PQ_ADD(PQ_MUL(vx, vx), PQ_MUL(vy, vy)));
  const double nx = PQ_DIV(vx, len), ny = PQ_DIV(vy, len);
  const double dot = PQ_ADD(PQ_MUL(nx, PQ_SUB(px, sx)), PQ_MUL(ny, PQ_SUB(py, sy)));
  const double m = 0.0 < dot ? dot : 0.0;
  const double coeff = len < m ? len : m;
  ox = PQ_ADD(PQ_MUL(coeff, nx), sx);
  oy = PQ_ADD(PQ_MUL(coeff, ny), sy);
}

// ---- the tables ----
struct PqTables {
  const double* regions;           // PQ_ROW doubles per region: label, [R | t] row-major 3 x 4, bbox
  const int32_t* polygons;         // PQ_POLY int32 per polygon: region, role, inset, first vertex, vertex count
  const double* vertices;          // (x, y) per vertex
  int64_t n_regions, n_polygons, n_vertices;
};

// Per region r (from pq_row_ok's tables): polygon rows [first[r], end[r]); the boundary's rows end at inset0[r].
struct PqRanges {
  const int* first;
  const int* inset0;
  const int* end;
};

// Whether polygon row p is consistent with the documented layout, from rows p - 1 .. p + 1 only: region in range and
// regions ascending without a gap (region 0 first, n_regions - 1 last), role 0 .. 3 in the order boundary outer,
// boundary holes, then insets each followed by its holes (so every region has a boundary and an inset), inset = -1
// for the boundary, the running inset index otherwise, and a vertex range of at least one vertex inside n_vertices.
PQ_HD bool pq_row_ok(const int32_t* P, int64_t p, int64_t n_polygons, int64_t n_regions, int64_t n_vertices) {
  const int32_t* w = P + PQ_POLY * p;
  const int64_t region = w[0], role = w[1], inset = w[2], v0 = w[3], nv = w[4];
  if (region < 0 || region >= n_regions || role < 0 || role > 3 || v0 < 0 || nv < 1 || v0 + nv > n_vertices)
    return false;
  const bool first = p == 0 || P[PQ_POLY * (p - 1)] != region;
  const bool last = p == n_polygons - 1 || P[PQ_POLY * (p + 1)] != region;
  if (p == 0 ? region != 0 : (int64_t)P[PQ_POLY * (p - 1)] > region || (int64_t)P[PQ_POLY * (p - 1)] < region - 1)
    return false;
  if (p == n_polygons - 1 && region != n_regions - 1) return false;
  if (last && role < PQ_INSET) return false;
  if (first) return role == PQ_BOUNDARY && inset == -1;
  const int32_t prole = P[PQ_POLY * (p - 1) + 1], pinset = P[PQ_POLY * (p - 1) + 2];
  switch (role) {
    case PQ_BOUNDARY: return false;
    case PQ_BOUNDARY_HOLE: return prole <= PQ_BOUNDARY_HOLE && inset == -1;
    case PQ_INSET: return inset == (prole <= PQ_BOUNDARY_HOLE ? 0 : pinset + 1);
    default: return prole >= PQ_INSET && inset == pinset;
  }
}

// The host's check of host tables before anything launches: nullptr when every row passes pq_row_ok and the counts
// agree, else what is wrong.  With ranges (3 n_regions ints: first, inset0, end), also fills them.
inline const char* pq_check_tables(const PqTables& t, int* ranges) {
  if ((t.n_polygons == 0) != (t.n_regions == 0)) return "regions without polygons or polygons without regions";
  for (int64_t p = 0; p < t.n_polygons; p++) {
    if (!pq_row_ok(t.polygons, p, t.n_polygons, t.n_regions, t.n_vertices))
      return "a polygon row's region, role, inset or vertex range breaks the table layout";
    if (!ranges) continue;
    const int32_t* w = t.polygons + PQ_POLY * p;
    if (p == 0 || w[-PQ_POLY] != w[0]) ranges[w[0]] = (int)p;
    if (w[1] == PQ_INSET && w[-PQ_POLY + 1] <= PQ_BOUNDARY_HOLE) ranges[t.n_regions + w[0]] = (int)p;
    if (p == t.n_polygons - 1 || w[PQ_POLY] != w[0]) ranges[2 * t.n_regions + w[0]] = (int)p + 1;
  }
  return nullptr;
}

PQ_HD int pq_role(const PqTables& t, int p) { return t.polygons[PQ_POLY * (int64_t)p + 1]; }

// bounded side of (px, py) for polygon row p: 1 inside, 0 on the boundary, -1 outside
PQ_HD int pq_bounded_side(const PqTables& t, int p, double px, double py) {
  const int32_t* w = t.polygons + PQ_POLY * (int64_t)p;
  const double* v = t.vertices + 2 * (int64_t)w[3];
  const int n = w[4];
  bool on = false, odd = false;
  for (int k = PQ_LANE; k < n; k += PQ_LANES) {
    const int k1 = k + 1 < n ? k + 1 : 0;
    bool o, c;
    pq_edge_side(px, py, v[2 * k], v[2 * k + 1], v[2 * k1], v[2 * k1 + 1], o, c);
    on |= o;
    odd ^= c;
  }
  if (pq_any(on)) return 0;
  return pq_odd(odd) ? 1 : -1;
}

// GeometryUtils.h's projectToClosestPoint(point, polygon row p): the first edge of least CGAL squared distance
PQ_HD void pq_project_polygon(const PqTables& t, int p, double px, double py, double& ox, double& oy) {
  const int32_t* w = t.polygons + PQ_POLY * (int64_t)p;
  const double* v = t.vertices + 2 * (int64_t)w[3];
  const int n = w[4];
  double best = 0.0;
  int bk = INT_MAX;
  for (int k = PQ_LANE; k < n; k += PQ_LANES) {
    const int k1 = k + 1 < n ? k + 1 : 0;
    const double d = pq_sqdist_segment(px, py, v[2 * k], v[2 * k + 1], v[2 * k1], v[2 * k1 + 1]);
    if (bk == INT_MAX || d < best) {
      best = d;
      bk = k;
    }
  }
  pq_min_key(best, bk);
  const int k1 = bk + 1 < n ? bk + 1 : 0;
  pq_project_segment(px, py, v[2 * bk], v[2 * bk + 1], v[2 * k1], v[2 * k1 + 1], ox, oy);
}

// SegmentedPlaneProjection.cpp's projectToPlanarRegion of the plane-frame point (px, py) onto region r
PQ_HD void pq_project_region(const PqTables& t, const PqRanges& g, int r, double px, double py, double& ox,
                             double& oy) {
  const int e = g.end[r];
  int found = -1;
  for (int p = g.inset0[r]; p < e; p++)
    if (pq_role(t, p) == PQ_INSET && pq_bounded_side(t, p, px, py) >= 0) {
      found = p;
      break;
    }
  if (found >= 0) {
    ox = px;
    oy = py;
    for (int p = found + 1; p < e && pq_role(t, p) == PQ_INSET_HOLE; p++)
      if (pq_bounded_side(t, p, px, py) >= 0) {
        pq_project_polygon(t, p, px, py, ox, oy);
        break;
      }
    return;
  }
  ox = NAN;
  oy = NAN;
  double best = DBL_MAX;
  for (int p = g.inset0[r]; p < e; p++) {
    if (pq_role(t, p) != PQ_INSET) continue;
    double cx, cy;
    pq_project_polygon(t, p, px, py, cx, cy);
    const double dx = PQ_SUB(cx, px), dy = PQ_SUB(cy, py);
    const double d = PQ_ADD(PQ_MUL(dx, dx), PQ_MUL(dy, dy));
    if (d < best) {
      best = d;
      ox = cx;
      oy = cy;
    }
  }
}

// Eigen's Isometry3d::inverse() * p: linear R^T, translation -(R^T t); each product sum ((a0 b0 + a1 b1) + a2 b2)
PQ_HD void pq_to_plane(const double* row, double px, double py, double pz, double& qx, double& qy) {
  const double* T = row + 1;       // T[4 i + j] = R(i, j), T[4 i + 3] = t(i)
  double q[2];
  for (int i = 0; i < 2; i++) {
    const double ti = -PQ_ADD(PQ_ADD(PQ_MUL(T[i], T[3]), PQ_MUL(T[4 + i], T[7])), PQ_MUL(T[8 + i], T[11]));
    q[i] = PQ_ADD(ti, PQ_ADD(PQ_ADD(PQ_MUL(T[i], px), PQ_MUL(T[4 + i], py)), PQ_MUL(T[8 + i], pz)));
  }
  qx = q[0];
  qy = q[1];
}

// PlanarRegion.cpp's positionInWorldFrameFromPosition2dInPlane: (t + x R.col(0)) + y R.col(1)
PQ_HD void pq_to_world(const double* row, double x, double y, double* w) {
  const double* T = row + 1;
  for (int i = 0; i < 3; i++) w[i] = PQ_ADD(PQ_ADD(T[4 * i + 3], PQ_MUL(x, T[4 * i])), PQ_MUL(y, T[4 * i + 1]));
}

// The exhaustive getBestPlanarRegionAtPositionInWorld for world point p: the first region (min_element) of least
// cost ((dx^2 + dy^2) + dz^2) + wz |z|.  point[6] = {cost, plane x, y, world x, y, z}; returns the region row (-1 with
// no region).
PQ_HD int pq_best_region(const PqTables& t, const PqRanges& g, const double* p, double wz, double* point) {
  int best = -1;
  for (int r = 0; r < (int)t.n_regions; r++) {
    const double* row = t.regions + PQ_ROW * (int64_t)r;
    double qx, qy, ox, oy, w[3];
    pq_to_plane(row, p[0], p[1], p[2], qx, qy);
    pq_project_region(t, g, r, qx, qy, ox, oy);
    pq_to_world(row, ox, oy, w);
    const double dx = PQ_SUB(p[0], w[0]), dy = PQ_SUB(p[1], w[1]), dz = PQ_SUB(p[2], w[2]);
    const double cost = PQ_ADD(PQ_ADD(PQ_ADD(PQ_MUL(dx, dx), PQ_MUL(dy, dy)), PQ_MUL(dz, dz)),
                               PQ_MUL(wz, fabs(w[2])));
    if (best < 0 || cost < point[0]) {
      best = r;
      point[0] = cost;
      point[1] = ox;
      point[2] = oy;
      point[3] = w[0];
      point[4] = w[1];
      point[5] = w[2];
    }
  }
  return best;
}

// ---- convex growth (ConvexRegionGrowing.cpp) inside region r's boundary (rows first[r] .. inset0[r]) ----
// the least CGAL squared distance from (px, py) to a boundary edge, from DBL_MAX; with (n0, n1) not null, also
// whether segment (n0, p) or (n1, p) meets an edge (doEdgesIntersectAndSquareDistance; its early return does not
// change the pair)
PQ_HD double pq_boundary_scan(const PqTables& t, const PqRanges& g, int r, double px, double py, const double* n0,
                              const double* n1, bool& hit) {
  double m = DBL_MAX;
  bool any = false;
  for (int p = g.first[r]; p < g.inset0[r]; p++) {
    const int32_t* w = t.polygons + PQ_POLY * (int64_t)p;
    const double* v = t.vertices + 2 * (int64_t)w[3];
    const int n = w[4];
    for (int k = PQ_LANE; k < n; k += PQ_LANES) {
      const int k1 = k + 1 < n ? k + 1 : 0;
      const double ax = v[2 * k], ay = v[2 * k + 1], bx = v[2 * k1], by = v[2 * k1 + 1];
      if (n0 && (pq_segments_intersect(n0[0], n0[1], px, py, ax, ay, bx, by) ||
                 pq_segments_intersect(n1[0], n1[1], px, py, ax, ay, bx, by)))
        any = true;
      const double d = pq_sqdist_segment(px, py, ax, ay, bx, by);
      m = d < m ? d : m;
    }
  }
  hit = pq_any(any);
  return pq_min(m);
}

struct PqTrig {                    // createRegularPolygon's cos / sin of i (2 pi / n), computed by the host's libm
  double c[PQ_MAX_CONVEX], s[PQ_MAX_CONVEX];
};

// The host's table for n vertices (two loops, so that no compiler merges them into one sincos call).
inline void pq_trig_table(int n, PqTrig& trig) {
  const double angle = (2. * M_PI) / n;
  for (int i = 0; i < n; i++) trig.c[i] = std::cos(i * angle);
  for (int i = 0; i < n; i++) trig.s[i] = std::sin(i * angle);
}

// growConvexPolygonInsideShape(boundary of r, (cx, cy), n, growth): vertices in vx / vy, per-vertex free spheres in
// sx / sy / sr (storage the caller gives: shared memory per warp on the device); returns the status, iterations in it.
PQ_HD int pq_grow(const PqTables& t, const PqRanges& g, int r, double cx, double cy, int n, double growth,
                  const PqTrig& trig, double* vx, double* vy, double* sx, double* sy, double* sr, int& it) {
  bool hit;
  const double sq = pq_boundary_scan(t, g, r, cx, cy, nullptr, nullptr, hit);
  const double radius = PQ_MUL(0.999, sq > 0.0 ? PQ_SQRT(sq) : 0.0);
  const double r2 = PQ_MUL(radius, radius);
  if (PQ_LANE == 0)
    for (int i = 0; i < n; i++) {
      vx[i] = PQ_ADD(PQ_MUL(radius, trig.c[i]), cx);
      vy[i] = PQ_ADD(PQ_MUL(radius, trig.s[i]), cy);
      sx[i] = cx;
      sy[i] = cy;
      sr[i] = r2;
    }
  pq_sync();
  it = 0;
  if (radius == 0.0) return PQ_ZERO_RADIUS;
  const double inv_n = PQ_DIV(1.0, (double)n);
  uint64_t blocked = 0;
  int n_blocked = 0;
  while (n_blocked < n && it < PQ_MAX_ITER) {
    for (int i = 0; i < n; i++) {
      if ((blocked >> i) & 1) continue;
      const double px = PQ_ADD(PQ_MUL(growth, PQ_SUB(vx[i], cx)), cx);
      const double py = PQ_ADD(PQ_MUL(growth, PQ_SUB(vy[i], cy)), cy);
      const int cw1 = i < n - 1 ? i + 1 : 0, cw2 = cw1 < n - 1 ? cw1 + 1 : 0;
      const int ccw1 = i > 0 ? i - 1 : n - 1, ccw2 = ccw1 > 0 ? ccw1 - 1 : n - 1;
      const double qx[5] = {vx[cw2], vx[cw1], px, vx[ccw1], vx[ccw2]};
      const double qy[5] = {vy[cw2], vy[cw1], py, vy[ccw1], vy[ccw2]};
      bool moved = pq_is_convex5(qx, qy);
      if (moved) {
        const double n0[2] = {vx[cw1], vy[cw1]}, n1[2] = {vx[ccw1], vy[ccw1]};
        auto in_sphere = [&](double x, double y) {
          const double dx = PQ_SUB(x, sx[i]), dy = PQ_SUB(y, sy[i]);
          return PQ_ADD(PQ_MUL(dx, dx), PQ_MUL(dy, dy)) <= sr[i];
        };
        if (!(in_sphere(n0[0], n0[1]) && in_sphere(px, py) && in_sphere(n1[0], n1[1]))) {
          const double m = pq_boundary_scan(t, g, r, px, py, n0, n1, hit);
          moved = !hit;
          pq_sync();
          if (moved && PQ_LANE == 0) {
            sx[i] = px;
            sy[i] = py;
            sr[i] = m;
          }
        }
      }
      if (moved) {
        const double ox = vx[i], oy = vy[i];
        cx = PQ_ADD(cx, PQ_MUL(inv_n, PQ_SUB(px, ox)));
        cy = PQ_ADD(cy, PQ_MUL(inv_n, PQ_SUB(py, oy)));
        pq_sync();
        if (PQ_LANE == 0) {
          vx[i] = px;
          vy[i] = py;
        }
      } else {
        blocked |= (uint64_t)1 << i;
        n_blocked++;
      }
      pq_sync();
    }
    ++it;
  }
  return it == PQ_MAX_ITER ? PQ_MAX_ITERATIONS : PQ_GROWN;
}

// the query's outputs when nothing is projected: index -1, the status, cost +inf, NaN positions and vertices
PQ_HD void pq_write_none(int32_t* index, double* point, double* convex, int n_convex, int status) {
  index[0] = -1;
  index[1] = status;
  index[2] = 0;
  point[0] = INFINITY;
  for (int k = 1; k < 6; k++) point[k] = NAN;
  for (int k = 0; k < 5 * n_convex; k++) convex[k] = NAN;
}

// the convex polygon's output: plane (x, y) and world (x, y, z) per vertex
PQ_HD void pq_write_convex(const double* row, int n, const double* vx, const double* vy, double* out) {
  for (int i = 0; i < n; i++) {
    out[5 * i] = vx[i];
    out[5 * i + 1] = vy[i];
    pq_to_world(row, vx[i], vy[i], out + 5 * i + 2);
  }
}

#if defined(__CUDACC__)
// ---- kernels ----
// Per polygon row: the row checks; the region's first row, first inset row and end.  `bad` is set for any row that
// fails, and for polygons without regions or regions without polygons.
__global__ void k_pq_ranges(PqTables t, int* first, int* inset0, int* end, int* bad) {
  const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (p == 0 && (t.n_polygons == 0) != (t.n_regions == 0)) atomicOr(bad, 1);
  if (p >= t.n_polygons) return;
  if (!pq_row_ok(t.polygons, p, t.n_polygons, t.n_regions, t.n_vertices)) {
    atomicOr(bad, 1);
    return;
  }
  const int32_t* w = t.polygons + PQ_POLY * p;
  if (p == 0 || w[-PQ_POLY] != w[0]) first[w[0]] = (int)p;
  if (w[1] == PQ_INSET && w[-PQ_POLY + 1] <= PQ_BOUNDARY_HOLE) inset0[w[0]] = (int)p;
  if (p == t.n_polygons - 1 || w[PQ_POLY] != w[0]) end[w[0]] = (int)p + 1;
}

// One warp per query: the exhaustive best region and its projection.  The status is PQ_GROWN and the iterations 0
// until k_pq_grow runs; with n_convex > 0 the vertices of queries without a region are written as NaN here.
__global__ void k_pq_project(PqTables t, PqRanges g, const int* bad,
                                                              const double* queries, int64_t n_queries, double wz,
                                                              int32_t* index, double* point, double* convex,
                                                              int n_convex) {
  const int64_t q = blockIdx.x * (int64_t)PQ_WARPS + (threadIdx.x >> 5);
  if (q >= n_queries) return;
  int32_t* idx = index + 3 * q;
  double* pt = point + 6 * q;
  double* cv = convex ? convex + 5 * (int64_t)n_convex * q : nullptr;
  const double p[3] = {queries[3 * q], queries[3 * q + 1], queries[3 * q + 2]};
  int status = -1;
  if (*bad) status = PQ_BAD_TABLE;
  else if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) status = PQ_INVALID_QUERY;
  else if (t.n_regions == 0) status = PQ_NO_REGION;
  double res[6];
  int best = -1;
  if (status < 0) {
    best = pq_best_region(t, g, p, wz, res);
    if (best < 0) status = PQ_NO_REGION;
  }
  if (PQ_LANE != 0) return;
  if (status >= 0) {
    pq_write_none(idx, pt, cv, cv ? n_convex : 0, status);
    return;
  }
  idx[0] = best;
  idx[1] = PQ_GROWN;
  idx[2] = 0;
  for (int k = 0; k < 6; k++) pt[k] = res[k];
}

// One warp per query with a region: growConvexPolygonInsideShape around its plane point, inside the region's boundary.
__global__ void k_pq_grow(PqTables t, PqRanges g, const PqTrig trig,
                                                           int64_t n_queries, int n_convex, double growth,
                                                           int32_t* index, const double* point, double* convex) {
  __shared__ double s_v[PQ_WARPS][5][PQ_MAX_CONVEX];
  const int warp = threadIdx.x >> 5;
  const int64_t q = blockIdx.x * (int64_t)PQ_WARPS + warp;
  if (q >= n_queries) return;
  const int r = index[3 * q];
  if (r < 0) return;
  double* v = &s_v[warp][0][0];
  int it;
  const int status = pq_grow(t, g, r, point[6 * q + 1], point[6 * q + 2], n_convex, growth, trig, v,
                             v + PQ_MAX_CONVEX, v + 2 * PQ_MAX_CONVEX, v + 3 * PQ_MAX_CONVEX, v + 4 * PQ_MAX_CONVEX,
                             it);
  pq_sync();
  if (PQ_LANE != 0) return;
  index[3 * q + 1] = status;
  index[3 * q + 2] = it;
  pq_write_convex(t.regions + PQ_ROW * (int64_t)r, n_convex, v, v + PQ_MAX_CONVEX,
                  convex + 5 * (int64_t)n_convex * q);
}
#endif
