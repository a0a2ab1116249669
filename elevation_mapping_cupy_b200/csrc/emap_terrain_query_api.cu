// emap_terrain_query_api.cu -- queries on the planar terrain and its layers of the C ABI (include/emap.h):
// emap_project_to_planar_regions over the kernels of emap_terrain_query.cuh, emap_max_values_between,
// emap_values_between and emap_grid_derivatives over those of emap_grid_lookup.cuh, emap_grid_values_at over
// emap_values_at.cuh's, and emap_signed_distance_field and emap_sdf_values over those of emap_sdf.cuh.
#include <algorithm>

#include "emap_grid_lookup.cuh"
#include "emap_handle.cuh"
#include "emap_sdf.cuh"
#include "emap_terrain_query.cuh"
#include "emap_values_at.cuh"

namespace {

// One call's device block: the per-region ranges and the bad-table flag, then (host output) the outputs in the order
// they are copied back in one piece: points, convex vertices, index words.
struct QueryScratch {
  int *first, *inset0, *end, *bad;
  char* back;
};

size_t carve_query(void* base, int64_t n_regions, size_t back_bytes, QueryScratch& s) {
  Carver b{(uintptr_t)base};
  s.first = b.take<int>(n_regions);
  s.inset0 = b.take<int>(n_regions);
  s.end = b.take<int>(n_regions);
  s.bad = b.take<int>(1);
  s.back = b.take<char>(back_bytes);
  return b.bytes;
}

const char* check_arguments(const emap_region_tables* t, int32_t tables_on_device, int64_t n_queries,
                            const double* queries, double penalty_z_weight, int32_t n_convex, double growth_factor,
                            const emap_projection_out* out) {
  if (!t || !out) return "null argument";
  if (t->n_regions < 0 || t->n_polygons < 0 || t->n_vertices < 0 || n_queries < 0)
    return "counts must be >= 0";
  if (t->n_regions > INT32_MAX || t->n_polygons > INT32_MAX || n_queries > INT32_MAX)
    return "n_regions, n_polygons and n_queries must be at most 2^31 - 1";
  if ((t->n_regions && !t->regions) || (t->n_polygons && !t->polygons) || (t->n_vertices && !t->vertices))
    return "null table with a count above 0";
  if (n_queries && (!queries || !out->index || !out->point || (n_convex && !out->convex)))
    return "null queries or output";
  if (n_convex != 0 && (n_convex < 3 || n_convex > EMAP_CONVEX_MAX_VERTICES))
    return "n_convex must be 0 or 3 .. EMAP_CONVEX_MAX_VERTICES";
  if (!(std::isfinite(growth_factor) && growth_factor > 1.0)) return "growth_factor must be finite and > 1";
  if (!(std::isfinite(penalty_z_weight) && penalty_z_weight >= 0.0)) return "penalty_z_weight must be finite and >= 0";
  if (!tables_on_device) {
    const PqTables ht{t->regions, t->polygons, t->vertices, t->n_regions, t->n_polygons, t->n_vertices};
    return pq_check_tables(ht, nullptr);
  }
  return nullptr;
}

// The grid and query checks the three lookups share (min_cells: the fewest rows and columns the call takes).
const char* check_lookup(const emap_grid* g, int64_t min_cells, int64_t n, const double* queries, bool outputs) {
  if (const char* e = gl_check_grid(g->data, g->rows, g->cols, g->position, g->resolution, min_cells)) return e;
  if (n < 0 || n > INT32_MAX) return "n_queries must be 0 .. 2^31 - 1";
  if (n && (!queries || !outputs)) return "null queries or output";
  return nullptr;
}

// The grid and queries as the kernels read them: a host grid and host queries (per_query doubles each) staged and
// uploaded in one copy.
int lookup_inputs(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, int64_t n, const double* queries,
                  int32_t queries_on_device, int per_query, GlGrid& g, const double*& q) {
  g.rows = (int)grid->rows;
  g.cols = (int)grid->cols;
  g.res = grid->resolution;
  for (int a = 0; a < 2; a++) {
    g.pos[a] = grid->position[a];
    g.len[a] = (double)(a ? grid->cols : grid->rows) * grid->resolution;
  }
  g.data = grid->data;
  q = queries;
  return stage_inputs(h, h->lookup.up, g.data, grid_on_device ? 0 : sizeof(float) * grid->rows * grid->cols, q,
                      queries_on_device ? 0 : sizeof(double) * per_query * n);
}

// The volumes the field calls accept, after the lookups' grid checks: nullptr, or why not
const char* check_volume(int64_t rows, int64_t cols, int64_t n_z, double z_min) {
  if (n_z < 1) return "n_z must be >= 1";
  if (!std::isfinite(z_min)) return "z_min must be finite";
  if (rows > SDF_MAX_LINE || cols > SDF_MAX_LINE || n_z > SDF_MAX_LINE ||
      (rows - 1) * (rows - 1) + (cols - 1) * (cols - 1) + (n_z - 1) * (n_z - 1) >= SDF_MAX_D2)
    return "(rows - 1)^2 + (cols - 1)^2 + (n_z - 1)^2 must be below 2^24";
  if (rows * cols * n_z > INT32_MAX) return "rows * cols * n_z must be below 2^31";
  return nullptr;
}

}  // namespace

static_assert(EMAP_GRID_MAX_EXTENT == GL_MAX_EXTENT && EMAP_GRID_MIN_RESOLUTION == GL_MIN_RES, "the grid bounds");
static_assert((int)EMAP_DERIVATIVE_INSIDE == (int)GL_INSIDE && (int)EMAP_DERIVATIVE_OUTSIDE == (int)GL_OUTSIDE,
              "the derivative statuses");

static_assert(EMAP_SDF_MAX_D2 == SDF_MAX_D2, "the field's limit");

static_assert(EMAP_VALUES_MAX_LAYERS == VA_MAX_LAYERS && (int)EMAP_VALUES_NEAREST == (int)VA_NEAREST &&
                  (int)EMAP_VALUES_LINEAR == (int)VA_LINEAR && (int)EMAP_VALUES_CUBIC == (int)VA_CUBIC,
              "the point values' limits and methods");
static_assert((int)EMAP_VALUE_OUTSIDE == (int)VA_OUT && (int)EMAP_VALUE_NEAREST == (int)VA_BY_NEAREST &&
                  (int)EMAP_VALUE_LINEAR == (int)VA_BY_LINEAR && (int)EMAP_VALUE_CUBIC == (int)VA_BY_CUBIC,
              "the point values' statuses");

static_assert(EMAP_REGION_ROW == PQ_ROW && EMAP_REGION_POLYGON == PQ_POLY, "the region table layout");
static_assert(EMAP_CONVEX_MAX_VERTICES == PQ_MAX_CONVEX && EMAP_GROW_MAX_ITER == PQ_MAX_ITER, "the growth limits");
static_assert(EMAP_PROJECTION_BAD_TABLE == PQ_BAD_TABLE && EMAP_PROJECTION_ZERO_RADIUS == PQ_ZERO_RADIUS,
              "the statuses");

extern "C" {

int emap_project_to_planar_regions(emap_handle* h, const emap_region_tables* tables, int32_t tables_on_device,
                                   int64_t n_queries, const double* queries, int32_t queries_on_device,
                                   double penalty_z_weight, int32_t n_convex, double growth_factor,
                                   const emap_projection_out* out, int32_t out_is_device) {
  ENTER(h);
  if (const char* e = check_arguments(tables, tables_on_device, n_queries, queries, penalty_z_weight, n_convex,
                                      growth_factor, out))
    return fail(h, EMAP_ERR_INVALID, (std::string("emap_project_to_planar_regions: ") + e).c_str());
  if (n_queries == 0) return EMAP_OK;
  NvtxRange nv("project_to_planar_regions");
  const int64_t N = n_queries, R = tables->n_regions;
  const size_t pt_bytes = sizeof(double) * 6 * N, cv_bytes = sizeof(double) * 5 * n_convex * N;
  const size_t back_bytes = out_is_device ? 0 : pt_bytes + cv_bytes + sizeof(int32_t) * 3 * N;
  QueryScratch s;
  const size_t need = carve_query(nullptr, R, back_bytes, s);
  if (int rc = grow(h, h->query.block, need, 0, false)) return rc;
  carve_query(h->query.block, R, back_bytes, s);
  PqTables t{tables->regions, tables->polygons, tables->vertices, R, tables->n_polygons, tables->n_vertices};
  const double* q = queries;
  const bool host_tables = !tables_on_device;
  if (int rc = stage_inputs(h, h->query.up, t.regions, host_tables ? sizeof(double) * PQ_ROW * R : 0, t.polygons,
                            host_tables ? sizeof(int32_t) * PQ_POLY * t.n_polygons : 0, t.vertices,
                            host_tables ? sizeof(double) * 2 * t.n_vertices : 0, q,
                            queries_on_device ? 0 : sizeof(double) * 3 * N))
    return rc;
  double* point = out_is_device ? out->point : (double*)s.back;
  double* convex = !n_convex ? nullptr : out_is_device ? out->convex : (double*)(s.back + pt_bytes);
  int32_t* index = out_is_device ? out->index : (int32_t*)(s.back + pt_bytes + cv_bytes);
  CK(cudaMemsetAsync(s.first, 0xff, (char*)s.bad - (char*)s.first, h->stream));    // ranges -1, then the flag 0
  CK(cudaMemsetAsync(s.bad, 0, sizeof(int), h->stream));
  const PqRanges g{s.first, s.inset0, s.end};
  k_pq_ranges<<<std::max(cdiv(tables->n_polygons, 256), 1), 256, 0, h->stream>>>(t, s.first, s.inset0, s.end, s.bad);
  LAUNCH_CHECK();
  const int blocks = cdiv(N, PQ_WARPS);
  k_pq_project<<<blocks, 32 * PQ_WARPS, 0, h->stream>>>(t, g, s.bad, q, N, penalty_z_weight, index, point, convex,
                                                         n_convex);
  LAUNCH_CHECK();
  if (n_convex) {
    PqTrig trig;
    pq_trig_table(n_convex, trig);
    k_pq_grow<<<blocks, 32 * PQ_WARPS, 0, h->stream>>>(t, g, trig, N, n_convex, growth_factor, index, point, convex);
    LAUNCH_CHECK();
  }
  if (!out_is_device) {
    if (int rc = read_back(h, h->query, s.back, back_bytes)) return rc;
    memcpy(out->point, h->query.down, pt_bytes);
    if (n_convex) memcpy(out->convex, h->query.down + pt_bytes, cv_bytes);
    memcpy(out->index, h->query.down + pt_bytes + cv_bytes, sizeof(int32_t) * 3 * N);
  }
  return EMAP_OK;
}

int emap_max_values_between(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, int64_t n_queries,
                            const double* lines, int32_t lines_on_device, const emap_line_max_out* out,
                            int32_t out_is_device) {
  ENTER(h);
  const char* e = !grid || !out ? "null argument"
                                : check_lookup(grid, 1, n_queries, lines, out->index && out->value);
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_max_values_between: ") + e).c_str());
  if (n_queries == 0) return EMAP_OK;
  NvtxRange nv("max_values_between");
  const int64_t N = n_queries;
  const size_t vb = sizeof(double) * 3 * N, ib = sizeof(int32_t) * 3 * N;
  if (!out_is_device)
    if (int rc = grow(h, h->lookup.block, vb + ib, 0, false)) return rc;
  GlGrid g;
  const double* q;
  if (int rc = lookup_inputs(h, grid, grid_on_device, N, lines, lines_on_device, 4, g, q)) return rc;
  double* value = out_is_device ? out->value : (double*)(char*)h->lookup.block;
  int32_t* index = out_is_device ? out->index : (int32_t*)(h->lookup.block + vb);
  k_gl_max<<<cdiv(N, GL_WARPS), 32 * GL_WARPS, 0, h->stream>>>(g, q, N, index, value);
  LAUNCH_CHECK();
  if (!out_is_device) {
    if (int rc = read_back(h, h->lookup, h->lookup.block, vb + ib)) return rc;
    memcpy(out->value, h->lookup.down, vb);
    memcpy(out->index, h->lookup.down + vb, ib);
  }
  return EMAP_OK;
}

int emap_values_between(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, int64_t n_queries,
                        const double* lines, int32_t lines_on_device, const emap_line_values_out* out,
                        int32_t out_is_device) {
  ENTER(h);
  const char* e = !grid || !out ? "null argument"
                                : check_lookup(grid, 1, n_queries, lines, out->counts && out->first);
  if (!e && !out->info) e = "null info";
  if (!e && out->capacity < 0) e = "capacity must be >= 0";
  if (!e && out->capacity > 0 && !out->rows) e = "null rows with a capacity above 0";
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_values_between: ") + e).c_str());
  if (n_queries == 0) {
    if (out_is_device) {
      CK(cudaMemsetAsync(out->info, 0, 2 * sizeof(int64_t), h->stream));
      CK(cudaMemsetAsync((char*)(out->info + 1), 1, 1, h->stream));     // complete = 1 (little-endian)
    } else {
      out->info[0] = 0;
      out->info[1] = 1;
    }
    return EMAP_OK;
  }
  NvtxRange nv("values_between");
  const int64_t N = n_queries, nb = cdiv(N, GL_WARPS);
  // the block: per-block sums (then offsets), then what host output copies back first, in one piece: info, counts
  Carver c0{0};
  c0.take<int64_t>(nb);
  c0.take<int64_t>(2);
  c0.take<int32_t>(N);
  if (int rc = grow(h, h->lookup.block, c0.bytes, 0, false)) return rc;
  Carver c{(uintptr_t)(char*)h->lookup.block};
  int64_t* block_sum = c.take<int64_t>(nb);
  int64_t* info = out_is_device ? out->info : c.take<int64_t>(2);
  int32_t* counts = out_is_device ? out->counts : c.take<int32_t>(N);
  GlGrid g;
  const double* q;
  if (int rc = lookup_inputs(h, grid, grid_on_device, N, lines, lines_on_device, 4, g, q)) return rc;
  k_gl_count<<<nb, 32 * GL_WARPS, 0, h->stream>>>(g, q, N, counts, block_sum);
  LAUNCH_CHECK();
  k_gl_scan<<<1, GL_SCAN_THREADS, 0, h->stream>>>(block_sum, nb, out->capacity, info);
  LAUNCH_CHECK();
  if (out_is_device) {
    k_gl_values<<<nb, 32 * GL_WARPS, 0, h->stream>>>(g, q, N, counts, block_sum, info, out->first, out->rows);
    LAUNCH_CHECK();
    return EMAP_OK;
  }
  // host output: info and the counts come back first, and the total sizes the second buffer; then the line offsets
  // and the rows, which k_gl_values writes into it back to back, come back together
  if (int rc = read_back(h, h->lookup, info, (char*)(counts + N) - (char*)info)) return rc;
  memcpy(out->info, h->lookup.down, 2 * sizeof(int64_t));
  memcpy(out->counts, h->lookup.down + ((char*)counts - (char*)info), sizeof(int32_t) * N);
  const size_t row_doubles = out->info[1] ? 3 * (size_t)out->info[0] : 0;
  if (int rc = grow(h, h->line_rows, N + row_doubles, 0, false)) return rc;
  k_gl_values<<<nb, 32 * GL_WARPS, 0, h->stream>>>(g, q, N, counts, block_sum, info, (int64_t*)(double*)h->line_rows,
                                                   h->line_rows + N);
  LAUNCH_CHECK();
  if (int rc = read_back(h, h->lookup, h->line_rows, sizeof(double) * (N + row_doubles))) return rc;
  memcpy(out->first, h->lookup.down, sizeof(int64_t) * N);
  if (row_doubles) memcpy(out->rows, h->lookup.down + sizeof(int64_t) * N, sizeof(double) * row_doubles);
  return EMAP_OK;
}

int emap_grid_derivatives(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, int64_t n_queries,
                          const double* positions, int32_t positions_on_device, int32_t curvature,
                          const emap_derivative_out* out, int32_t out_is_device) {
  ENTER(h);
  const char* e = !grid || !out ? "null argument"
                                : check_lookup(grid, 5, n_queries, positions, out->index && out->value);
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_grid_derivatives: ") + e).c_str());
  if (n_queries == 0) return EMAP_OK;
  NvtxRange nv("grid_derivatives");
  const int64_t N = n_queries;
  const int nv_per = curvature ? 5 : 2;
  const size_t vb = sizeof(double) * nv_per * N, ib = sizeof(int32_t) * 3 * N;
  if (!out_is_device)
    if (int rc = grow(h, h->lookup.block, vb + ib, 0, false)) return rc;
  GlGrid g;
  const double* q;
  if (int rc = lookup_inputs(h, grid, grid_on_device, N, positions, positions_on_device, 2, g, q)) return rc;
  double* value = out_is_device ? out->value : (double*)(char*)h->lookup.block;
  int32_t* index = out_is_device ? out->index : (int32_t*)(h->lookup.block + vb);
  k_gl_derivatives<<<cdiv(N, GL_THREADS), GL_THREADS, 0, h->stream>>>(g, gl_kernels(grid->resolution), q, N,
                                                                      curvature ? 1 : 0, index, value);
  LAUNCH_CHECK();
  if (!out_is_device) {
    if (int rc = read_back(h, h->lookup, h->lookup.block, vb + ib)) return rc;
    memcpy(out->value, h->lookup.down, vb);
    memcpy(out->index, h->lookup.down + vb, ib);
  }
  return EMAP_OK;
}

int emap_grid_values_at(emap_handle* h, int32_t n_layers, const emap_grid* grids, int32_t grids_on_device,
                        int64_t n_points, const double* positions, int32_t positions_on_device, int32_t method,
                        const emap_values_out* out, int32_t out_is_device) {
  ENTER(h);
  const char* e = !grids ? "null argument" : va_check(n_layers, n_points, positions, method, out);
  for (int k = 0; !e && k < n_layers; k++) {
    const emap_grid &a = grids[k], &b = grids[0];
    e = gl_check_grid(a.data, a.rows, a.cols, a.position, a.resolution, 1);
    if (!e && (a.rows != b.rows || a.cols != b.cols || a.position[0] != b.position[0] ||
               a.position[1] != b.position[1] || a.resolution != b.resolution))
      e = "the layers must share rows, cols, position and resolution";
  }
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_grid_values_at: ") + e).c_str());
  if (n_points == 0) return EMAP_OK;
  NvtxRange nv("grid_values_at");
  if (int rc = va_room(h, n_layers, n_points, out_is_device)) return rc;
  const emap_grid& g0 = grids[0];
  // the layers and the positions, host ones uploaded in one copy
  const void* in[VA_MAX_LAYERS + 1];
  size_t bytes[VA_MAX_LAYERS + 1];
  for (int k = 0; k < n_layers; k++) {
    in[k] = grids[k].data;
    bytes[k] = grids_on_device ? 0 : sizeof(float) * g0.rows * g0.cols;
  }
  in[n_layers] = positions;
  bytes[n_layers] = positions_on_device ? 0 : sizeof(double) * 2 * n_points;
  if (int rc = stage_input_list(h, h->lookup.up, n_layers + 1, in, bytes)) return rc;
  VaGeom g;
  g.rows = (int)g0.rows;
  g.cols = (int)g0.cols;
  g.res = g0.resolution;
  for (int a = 0; a < 2; a++) {
    g.pos[a] = g0.position[a];
    g.len[a] = (double)(a ? g0.cols : g0.rows) * g0.resolution;
  }
  VaGridSrc s;
  s.n = n_layers;
  s.cols = g.cols;
  for (int k = 0; k < VA_MAX_LAYERS; k++) s.data[k] = k < n_layers ? (const float*)in[k] : nullptr;
  return va_launch(h, g, s, method, n_points, (const double*)in[n_layers], out, out_is_device);
}

int emap_signed_distance_field(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, double z_min,
                               int64_t n_z, float* out, int64_t capacity, int32_t out_is_device) {
  ENTER(h);
  const char* e = !grid || !out ? "null argument" : gl_check_grid(grid->data, grid->rows, grid->cols, grid->position,
                                                                 grid->resolution, 1);
  if (!e) e = check_volume(grid->rows, grid->cols, n_z, z_min);
  if (!e && capacity < grid->rows * grid->cols * n_z) e = "capacity below rows * cols * n_z";
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_signed_distance_field: ") + e).c_str());
  NvtxRange nv("signed_distance_field");
  const int rows = (int)grid->rows, cols = (int)grid->cols, nz = (int)n_z;
  const size_t vol_bytes = sizeof(float) * rows * cols * nz;
  // the block: the fill key, then (host output) the volume
  const size_t vol_off = 256;
  if (int rc = grow(h, h->lookup.block, vol_off + (out_is_device ? 0 : vol_bytes), 0, false)) return rc;
  uint32_t* key = (uint32_t*)(char*)h->lookup.block;
  int32_t* vol = out_is_device ? (int32_t*)out : (int32_t*)(h->lookup.block + vol_off);
  const float* data = grid->data;
  if (int rc = stage_inputs(h, h->lookup.up, data, grid_on_device ? 0 : sizeof(float) * rows * cols)) return rc;
  CK(cudaMemsetAsync(key, 0xff, sizeof(uint32_t), h->stream));     // SDF_KEY_NONE
  const int64_t cells = (int64_t)rows * cols;
  k_sdf_min<<<std::min(cdiv(cells, SDF_THREADS * 8), 1024), SDF_THREADS, 0, h->stream>>>(data, cells, key);
  LAUNCH_CHECK();
  k_sdf_cols<<<dim3(rows, nz), SDF_LINE_THREADS, sdf_line_smem(cols), h->stream>>>(
      data, rows, cols, nz, z_min, grid->resolution, key, vol);
  LAUNCH_CHECK();
  k_sdf_rows<<<dim3(cols, nz), SDF_LINE_THREADS, sdf_line_smem(rows), h->stream>>>(rows, cols,
                                                                                  (float)grid->resolution, vol);
  LAUNCH_CHECK();
  if (!out_is_device) {
    if (int rc = read_back(h, h->lookup, vol, vol_bytes)) return rc;
    memcpy(out, h->lookup.down, vol_bytes);
  }
  return EMAP_OK;
}

int emap_sdf_values(emap_handle* h, const emap_sdf* field, int32_t field_on_device, int64_t n, const double* points,
                    int32_t points_on_device, double* out, int32_t out_is_device) {
  ENTER(h);
  const char* e = !field ? "null argument" : gl_check_grid(field->data, field->rows, field->cols, field->position,
                                                          field->resolution, 1);
  if (!e) e = check_volume(field->rows, field->cols, field->n_z, field->z_min);
  if (!e && (n < 0 || n > INT32_MAX)) e = "n must be 0 .. 2^31 - 1";
  if (!e && n && (!points || !out)) e = "null points or output";
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_sdf_values: ") + e).c_str());
  if (n == 0) return EMAP_OK;
  NvtxRange nv("sdf_values");
  const size_t ob = sizeof(double) * 4 * n;
  if (!out_is_device)
    if (int rc = grow(h, h->lookup.block, ob, 0, false)) return rc;
  SdfVol f;
  f.rows = (int)field->rows;
  f.cols = (int)field->cols;
  f.n_z = (int)field->n_z;
  f.pos[0] = field->position[0];
  f.pos[1] = field->position[1];
  f.res = field->resolution;
  f.z_min = field->z_min;
  f.data = field->data;
  const double* q = points;
  if (int rc = stage_inputs(h, h->lookup.up, f.data, field_on_device ? 0 : sizeof(float) * f.rows * f.cols * f.n_z, q,
                            points_on_device ? 0 : sizeof(double) * 3 * n))
    return rc;
  double* o = out_is_device ? out : (double*)(char*)h->lookup.block;
  k_sdf_values<<<cdiv(n, SDF_THREADS), SDF_THREADS, 0, h->stream>>>(f, q, n, o);
  LAUNCH_CHECK();
  if (!out_is_device) {
    if (int rc = read_back(h, h->lookup, h->lookup.block, ob)) return rc;
    memcpy(out, h->lookup.down, ob);
  }
  return EMAP_OK;
}

}  // extern "C"
