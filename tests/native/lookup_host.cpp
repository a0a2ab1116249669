// tests/native/lookup_host.cpp -- TEST HELPER: the per-query functions of csrc/emap_grid_lookup.cuh (the same inline
// functions the kernels call, one thread in place of a warp) compiled for the CPU, so that walks, whole line lookups
// and derivatives can be compared with tests/grid_lookup_oracle.py.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -I<cuda>/include -o tests/native/_build/liblookup_host.so
//          tests/native/lookup_host.cpp
#include "../../elevation_mapping_cupy_b200/csrc/emap_grid_lookup.cuh"

namespace {
GlGrid make_grid(const float* data, int64_t rows, int64_t cols, const double* position, double res) {
  GlGrid g;
  g.data = data;
  g.rows = (int)rows;
  g.cols = (int)cols;
  g.res = res;
  for (int a = 0; a < 2; a++) {
    g.pos[a] = position[a];
    g.len[a] = (double)(a ? cols : rows) * res;
  }
  return g;
}
}  // namespace

extern "C" {

// The cells of the walk from cell (r0, c0) to (r1, c1) per line (4 ints each), as `lanes` lanes visit them: lane l
// takes cells l, l + lanes, ... through GlCursor; cell i goes to out[2 (max_cells line + i)].  n[line] = its cells.
void glh_walks(int64_t n_lines, const int32_t* ends, int lanes, int64_t max_cells, int32_t* out, int64_t* n) {
  for (int64_t q = 0; q < n_lines; q++) {
    const int32_t* e = ends + 4 * q;
    GlLine L;
    gl_line_from_cells(e[0], e[1], e[2], e[3], L);
    n[q] = L.n;
    for (int lane = 0; lane < lanes; lane++) {
      GlCursor cur(L, lane, lanes);
      for (int64_t i = lane; i < L.n && i < max_cells; i += lanes, cur.next()) {
        int r, c;
        gl_cell(L, i, cur.k, r, c);
        out[2 * (max_cells * q + i)] = r;
        out[2 * (max_cells * q + i) + 1] = c;
      }
    }
  }
}

// k(i) of the closed form for one line and i (64-bit): floor((den / 2 + i add) / den)
int64_t glh_minor(int64_t major, int64_t minor, int64_t i) {
  GlLine L;
  L.add = minor;
  L.half = major / 2;
  L.den = major ? major : 1;
  return GlCursor(L, i, 1).k;
}

// projectToMapWithMargin of each point (2 doubles), and whether the projection is inside (grid_axis_index on both axes)
void glh_project(int64_t rows, int64_t cols, const double* position, double res, int64_t n, const double* xy,
                 double* out, int32_t* inside) {
  const GlGrid g = make_grid(nullptr, rows, cols, position, res);
  for (int64_t k = 0; k < n; k++) {
    gl_project(g, xy[2 * k], xy[2 * k + 1], out + 2 * k);
    int r, c;
    inside[k] = grid_axis_index(out[2 * k], g.pos[0], g.len[0], g.res, g.rows, r) &&
                grid_axis_index(out[2 * k + 1], g.pos[1], g.len[1], g.res, g.cols, c);
  }
}

// emap_max_values_between's outputs for a host grid, one line after the other
void glh_max(const float* data, int64_t rows, int64_t cols, const double* position, double res, int64_t n,
             const double* lines, int32_t* index, double* value) {
  const GlGrid g = make_grid(data, rows, cols, position, res);
  for (int64_t q = 0; q < n; q++) {
    GlLine L;
    gl_line(g, lines + 4 * q, L);
    gl_max_line(g, L, 0, 1, index + 3 * q, value + 3 * q);
  }
}

// emap_values_between's outputs (rows: room for every finite cell, or NULL to count only); returns the total
int64_t glh_values(const float* data, int64_t rows, int64_t cols, const double* position, double res, int64_t n,
                   const double* lines, int32_t* counts, int64_t* first, double* out) {
  const GlGrid g = make_grid(data, rows, cols, position, res);
  int64_t total = 0;
  for (int64_t q = 0; q < n; q++) {
    GlLine L;
    gl_line(g, lines + 4 * q, L);
    first[q] = total;
    counts[q] = (int32_t)gl_finite_cells(g, L, 0, 1, [](int64_t, int, int, float) {});
    if (out) gl_values_line(g, L, 0, 1, out + 3 * total);
    total += counts[q];
  }
  return total;
}

// emap_grid_derivatives' outputs (value: 2 or 5 doubles per position)
void glh_derivatives(const float* data, int64_t rows, int64_t cols, const double* position, double res, int64_t n,
                     const double* xy, int curvature, int32_t* index, double* value) {
  const GlGrid g = make_grid(data, rows, cols, position, res);
  const GlKernels K = gl_kernels(res);
  const int nv = curvature ? 5 : 2;
  for (int64_t q = 0; q < n; q++) gl_derivative(g, K, xy[2 * q], xy[2 * q + 1], curvature, index + 3 * q, value + nv * q);
}

// 0 when the calls accept the grid, 1 when they reject it
int glh_check_grid(int64_t rows, int64_t cols, const double* position, double res, int64_t min_cells) {
  static const float dummy = 0.0f;
  return gl_check_grid(&dummy, rows, cols, position, res, min_cells) ? 1 : 0;
}

// the kernels gl_kernels builds
void glh_kernels(double res, float* d1, float* d2) {
  const GlKernels K = gl_kernels(res);
  for (int k = 0; k < 5; k++) {
    d1[k] = K.d1[k];
    d2[k] = K.d2[k];
  }
}
}
