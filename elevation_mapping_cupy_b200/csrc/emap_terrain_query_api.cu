// emap_terrain_query_api.cu -- queries on the planar terrain of the C ABI (include/emap.h):
// emap_project_to_planar_regions, over the kernels of emap_terrain_query.cuh.
#include <algorithm>

#include "emap_handle.cuh"
#include "emap_terrain_query.cuh"

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

}  // namespace

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
  // uploads: the host tables and the host queries, back to back in one staged copy
  const size_t tab_bytes[3] = {sizeof(double) * PQ_ROW * R, sizeof(int32_t) * PQ_POLY * tables->n_polygons,
                               sizeof(double) * 2 * tables->n_vertices};
  size_t up_off[4] = {0, 0, 0, 0};     // regions, polygons, vertices, queries
  size_t up = 0;
  for (int k = 0; k < 4; k++) {
    up_off[k] = up;
    if (k < 3 ? !tables_on_device : !queries_on_device)
      up = (up + (k < 3 ? tab_bytes[k] : sizeof(double) * 3 * N) + 255) & ~(size_t)255;
  }
  const size_t pt_bytes = sizeof(double) * 6 * N, cv_bytes = sizeof(double) * 5 * n_convex * N;
  const size_t back_bytes = out_is_device ? 0 : pt_bytes + cv_bytes + sizeof(int32_t) * 3 * N;
  QueryScratch s;
  const size_t need = carve_query(nullptr, R, back_bytes, s);
  if (int rc = grow(h, h->query.block, need, 0, false)) return rc;
  carve_query(h->query.block, R, back_bytes, s);
  if (!out_is_device && h->query.down.size() < back_bytes) CK(h->query.down.alloc(back_bytes));
  PqTables t{tables->regions, tables->polygons, tables->vertices, R, tables->n_polygons, tables->n_vertices};
  const double* q = queries;
  if (up) {
    if (int rc = h->query.up.room(h, up)) return rc;
    char* st = h->query.up.host;
    char* dev = h->query.up.dev;
    if (!tables_on_device) {
      memcpy(st + up_off[0], tables->regions, tab_bytes[0]);
      memcpy(st + up_off[1], tables->polygons, tab_bytes[1]);
      memcpy(st + up_off[2], tables->vertices, tab_bytes[2]);
      t.regions = (const double*)(dev + up_off[0]);
      t.polygons = (const int32_t*)(dev + up_off[1]);
      t.vertices = (const double*)(dev + up_off[2]);
    }
    if (!queries_on_device) {
      memcpy(st + up_off[3], queries, sizeof(double) * 3 * N);
      q = (const double*)(dev + up_off[3]);
    }
    if (int rc = h->query.up.send(h, up)) return rc;
  }
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
    CK(cudaMemcpyAsync(h->query.down, s.back, back_bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    memcpy(out->point, h->query.down, pt_bytes);
    if (n_convex) memcpy(out->convex, h->query.down + pt_bytes, cv_bytes);
    memcpy(out->index, h->query.down + pt_bytes + cv_bytes, sizeof(int32_t) * 3 * N);
  }
  return EMAP_OK;
}

}  // extern "C"
