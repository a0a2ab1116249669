// tests/native/projection_host.cpp -- TEST HELPER: the per-query functions of csrc/emap_terrain_query.cuh (the same
// inline functions the kernels call, one thread in place of a warp) compiled for the CPU, so that the exact predicates,
// the host table checks and whole queries can be compared with tests/planar_projection_oracle.py.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -I<cuda>/include -o tests/native/_build/libprojection_host.so
//          tests/native/projection_host.cpp
#include <vector>

#include "../../elevation_mapping_cupy_b200/csrc/emap_terrain_query.cuh"

extern "C" {

int pqh_orient(double ax, double ay, double bx, double by, double cx, double cy) {
  return pq_orient(ax, ay, bx, by, cx, cy);
}

int pqh_segments_intersect(double p1x, double p1y, double p2x, double p2y, double q1x, double q1y, double q2x,
                           double q2y) {
  return pq_segments_intersect(p1x, p1y, p2x, p2y, q1x, q1y, q2x, q2y);
}

// bounded side of (px, py) for the polygon of n vertices xy
int pqh_bounded_side(double px, double py, const double* xy, int n) {
  const int32_t row[5] = {0, PQ_INSET, 0, 0, n};
  const PqTables t{nullptr, row, xy, 1, 1, n};
  return pq_bounded_side(t, 0, px, py);
}

int pqh_is_convex5(const double* x, const double* y) { return pq_is_convex5(x, y); }

double pqh_sqdist_segment(double px, double py, double sx, double sy, double tx, double ty) {
  return pq_sqdist_segment(px, py, sx, sy, tx, ty);
}

// 0 when the host check accepts the tables, 1 when it rejects them
int pqh_check_tables(const double* regions, int64_t n_regions, const int32_t* polygons, int64_t n_polygons,
                     const double* vertices, int64_t n_vertices) {
  const PqTables t{regions, polygons, vertices, n_regions, n_polygons, n_vertices};
  return pq_check_tables(t, nullptr) ? 1 : 0;
}

// emap_project_to_planar_regions' outputs for host tables, one query after the other; -1 for tables the check rejects
int pqh_project(const double* regions, int64_t n_regions, const int32_t* polygons, int64_t n_polygons,
                const double* vertices, int64_t n_vertices, int64_t n_queries, const double* queries, double wz,
                int n_convex, double growth, int32_t* index, double* point, double* convex) {
  const PqTables t{regions, polygons, vertices, n_regions, n_polygons, n_vertices};
  std::vector<int> ranges(3 * n_regions + 1);
  if (pq_check_tables(t, ranges.data())) return -1;
  const PqRanges g{ranges.data(), ranges.data() + n_regions, ranges.data() + 2 * n_regions};
  PqTrig trig;
  if (n_convex) pq_trig_table(n_convex, trig);
  double v[5][PQ_MAX_CONVEX];
  for (int64_t q = 0; q < n_queries; q++) {
    const double* p = queries + 3 * q;
    int32_t* idx = index + 3 * q;
    double* pt = point + 6 * q;
    double* cv = n_convex ? convex + 5 * n_convex * q : nullptr;
    int status = -1;
    if (!(std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]))) status = PQ_INVALID_QUERY;
    else if (n_regions == 0) status = PQ_NO_REGION;
    int best = -1;
    if (status < 0 && (best = pq_best_region(t, g, p, wz, pt)) < 0) status = PQ_NO_REGION;
    if (status >= 0) {
      pq_write_none(idx, pt, cv, n_convex, status);
      continue;
    }
    idx[0] = best;
    idx[1] = PQ_GROWN;
    idx[2] = 0;
    if (!n_convex) continue;
    int it;
    idx[1] = pq_grow(t, g, best, pt[1], pt[2], n_convex, growth, trig, v[0], v[1], v[2], v[3], v[4], it);
    idx[2] = it;
    pq_write_convex(regions + PQ_ROW * best, n_convex, v[0], v[1], cv);
  }
  return 0;
}
}
