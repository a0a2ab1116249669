// emap_polygon_api.cu -- the polygon safety check of the C ABI (include/emap.h): emap_polygon_traversability and
// emap_polygon_traversability_batch, one host path over the kernels of emap_polygon.cuh.
#include "emap_handle.cuh"
#include "emap_polygon.cuh"

namespace {

constexpr int kRingHead = 256;     // ring vertices of a single call read back with its result
constexpr size_t kBatchRingHead = 4096;    // ring rows of a batch read back with its results
// (longer rings take a second copy)

struct PolyScratch {
  PolyPartial* part;               // one per k_polygon work item
  int *col_min, *col_max;          // the polygons' column windows, back to back
  char* down;                      // read-back region: one PolyResult per polygon, then the rings (PolyStage)
};

// One call's layout of the upload (h->poly.up) and of the read-back region (at the block's tail and in h->poly.down),
// each moved in one copy.  The two poison counts sit at offset 0 of the upload, the results at offset 0 of the read-back.
struct PolyStage {
  size_t desc, xy, up_bytes;
  size_t ring, down_bytes;
};

PolyStage poly_stage(size_t n_poly, size_t n_vert, size_t ring_rows) {
  PolyStage s;
  s.desc = 16;
  s.xy = s.desc + sizeof(PolyDesc) * n_poly;
  s.up_bytes = s.xy + sizeof(float2) * n_vert;
  s.ring = sizeof(PolyResult) * n_poly;
  s.down_bytes = s.ring + sizeof(double2) * ring_rows;
  return s;
}

dim3 polygon_grid(int W) { return dim3(cdiv(W, PG_COLS), cdiv(W, PG_ROWS)); }

size_t carve_polygon(const PolySizes& z, void* base, PolyScratch& s) {
  Carver b{(uintptr_t)base};
  s.part = b.take<PolyPartial>(z.items);
  s.col_min = b.take<int>(z.cols);
  s.col_max = b.take<int>(z.cols);
  s.down = b.take<char>(z.down);
  return b.bytes;
}

// Carves the device block of a call of sizes z, growing it to the largest call so far.
int alloc_polygon_scratch(emap_handle* h, const PolySizes& z, PolyScratch& s) {
  PolySizes& c = h->poly_cap;
  if (!h->poly.block || z.items > c.items || z.cols > c.cols || z.down > c.down) {
    c.items = std::max(c.items, z.items); c.cols = std::max(c.cols, z.cols); c.down = std::max(c.down, z.down);
    CK(h->poly.block.alloc(carve_polygon(c, nullptr, s)));
    carve_polygon(c, h->poly.block, s);
    CK(cudaMemsetAsync(s.col_min, 0x7f, sizeof(int) * c.cols, h->stream));    // "no cell yet": k_hull restores it
    CK(cudaMemsetAsync(s.col_max, 0xff, sizeof(int) * c.cols, h->stream));
  }
  carve_polygon(c, h->poly.block, s);
  return 0;
}

// The device part of a call whose n_poly polygons (n_items work items) are staged in h->poly.up's host side: one upload
// copy, k_poly_poison (with `poison`), k_polygon, k_hull, one copy of the results and the first `head` ring rows into
// h->poly.down, one synchronisation; one more copy and synchronisation only if a ring ends beyond `head`.
int run_polygons(emap_handle* h, const PolyScratch& s, const PolyStage& st, int n_poly, int n_items, bool poison,
                 const float* checker_plane, double safe_thresh, double safe_min_thresh, int32_t max_unsafe_n,
                 float* mask, bool hulls, size_t head) {
  const int W = h->dc.W;
  const size_t C = (size_t)h->dc.C;
  const dim3 g = polygon_grid(W);
  const float* valid = h->map + L_VALID * C;
  const float* checker = checker_plane ? checker_plane : h->map + L_TRAV * C;
  const char* up = h->poly.up.dev;
  PolyArgs a;
  a.poly = (const PolyDesc*)(up + st.desc); a.n_poly = n_poly; a.xy = (const float2*)(up + st.xy);
  a.cx = h->center[0]; a.cy = h->center[1];
  a.thr_over = (float)(1.0 - safe_thresh); a.thr_max = (float)(1.0 - safe_min_thresh);    // traversability_polygon.py:25-26
  a.max_unsafe_n = max_unsafe_n;
  a.poison = poison ? (const int*)up : nullptr;
  memcpy(&a.one, h->poly.up.host + st.desc, sizeof(PolyDesc));
  if (int rc = h->poly.up.send(h, st.up_bytes)) return rc;
  if (poison) {
    k_poly_poison<<<std::min(cdiv((i64)C, 256), 4 * h->n_sm), 256, 0, h->stream>>>(W, valid, checker, (int*)up);
    LAUNCH_CHECK();
  }
  (poison ? k_polygon<true> : k_polygon<false>)<<<n_items, PG_THREADS, 0, h->stream>>>(
      W, h->dc.res_f, a, valid, checker, mask, s.part, hulls ? s.col_min : nullptr, hulls ? s.col_max : nullptr);
  LAUNCH_CHECK();
  k_hull<<<n_poly, HULL_THREADS, 0, h->stream>>>(W, h->cfg.resolution, a, (int)g.x, (int)g.y, s.part, s.col_min,
                                                 s.col_max, (PolyResult*)s.down,
                                                 hulls ? (double2*)(s.down + st.ring) : nullptr);
  LAUNCH_CHECK();
  head = std::min(head, (st.down_bytes - st.ring) / sizeof(double2));
  if (int rc = read_back(h, h->poly, s.down, st.ring + sizeof(double2) * head, st.down_bytes)) return rc;
  char* back = h->poly.down;
  const PolyResult* r = (const PolyResult*)back;
  const PolyDesc* d = (const PolyDesc*)(h->poly.up.host + st.desc);
  size_t end = 0;
  for (int i = 0; i < n_poly; i++)
    if (r[i].n_ring) end = std::max(end, (size_t)d[i].ring_off + r[i].n_ring);
  if (end > head) {
    const size_t off = st.ring + sizeof(double2) * head;
    CK(cudaMemcpyAsync(back + off, s.down + off, sizeof(double2) * (end - head), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}

// The device part and the answers of a call of n_polygons polygons, both entry points' one host path.  Each polygon's
// descriptor holds its cell bounding box and, as work items, the tiles of that box (every tile of the grid with
// `whole_map`), its column window (the whole one with `whole_map`; none without `hulls`) and its ring slot.  Then the
// upload, run_polygons (with `poison`, `mask` and `head`) and the answers: results[3 i ..] = {safe, traversability,
// area}, hull_offsets[i] (unless null) the first hull row of polygon i, and `total` (and hull_offsets[n_polygons]) the
// hull rows of all.  The hulls stay in the read-back staging for copy_hulls, at the layout st.
int check_polygons(emap_handle* h, int n_polygons, const int32_t* n_vertices, const float* polygon_xy,
                   const float* checker_plane, double safe_thresh, double safe_min_thresh, int32_t max_unsafe_n,
                   bool whole_map, bool poison, float* mask, bool hulls, size_t head, double* results,
                   int64_t* hull_offsets, int64_t& total, PolyStage& st) {
  const dim3 g = polygon_grid(h->dc.W);
  // each polygon's tiles (its work items and partials), column window and ring slot
  std::vector<PolyDesc> desc(n_polygons);
  size_t items = 0, cols = 0, rows = 0, v0 = 0;
  for (int i = 0; i < n_polygons; i++) {
    PolyDesc& d = desc[i];
    clip_polygon(h->dc.W, h->cfg.resolution, h->center, polygon_xy + 2 * v0, n_vertices[i], nullptr, d.bbox);
    polygon_tiles(h->dc.W, h->cfg.resolution, h->center, d);
    if (whole_map) {
      d.tr0 = 0; d.tc0 = 0; d.n_tr = g.y; d.n_tc = g.x;
      d.col0 = 0; d.n_col = h->dc.W - 2;
    }
    if (!hulls) d.n_col = 0;
    d.v0 = (int)v0; d.n = n_vertices[i]; d.item0 = (int)items; d.col_off = (int)cols; d.ring_off = (int)rows;
    items += (size_t)d.n_tr * d.n_tc;
    cols += d.n_col;
    rows += d.n_col ? 2 * (size_t)d.n_col + 1 : 0;
    v0 += n_vertices[i];
  }
  st = poly_stage(n_polygons, v0, rows);
  PolySizes z;
  z.items = items; z.cols = cols; z.down = st.down_bytes;
  PolyScratch s;
  int rc = alloc_polygon_scratch(h, z, s);
  if (rc || (rc = h->poly.up.room(h, st.up_bytes))) return rc;
  char* up = h->poly.up.host;
  memset(up, 0, st.desc);                                           // the poison counts start at zero
  memcpy(up + st.desc, desc.data(), sizeof(PolyDesc) * n_polygons);
  float2* xy = (float2*)(up + st.xy);
  std::vector<float> area(n_polygons), clipped_area(n_polygons);
  for (int i = 0; i < n_polygons; i++) {
    const PolyDesc& d = desc[i];
    area[i] = shoelace_f32(polygon_xy + 2 * (size_t)d.v0, d.n);
    float bbox[4];
    clip_polygon(h->dc.W, h->cfg.resolution, h->center, polygon_xy + 2 * (size_t)d.v0, d.n, xy + d.v0, bbox);
    clipped_area[i] = shoelace_f32((const float*)(xy + d.v0), d.n);
  }
  rc = run_polygons(h, s, st, n_polygons, (int)items, poison, checker_plane, safe_thresh, safe_min_thresh, max_unsafe_n,
                    mask, hulls, head);
  if (rc) return rc;
  const PolyResult* r = (const PolyResult*)(char*)h->poly.down;
  total = 0;
  for (int i = 0; i < n_polygons; i++) {
    // EM.py:884-887: a polygon (almost) entirely outside the map is unsafe
    results[3 * i] = (r[i].is_safe && !(clipped_area[i] < 0.001f)) ? 1.0 : 0.0;
    results[3 * i + 1] = r[i].t;
    results[3 * i + 2] = (double)area[i];
    if (hull_offsets) hull_offsets[i] = total;
    total += r[i].n_ring;
  }
  if (hull_offsets) hull_offsets[n_polygons] = total;
  return EMAP_OK;
}

// The hull of every polygon of the last check_polygons (layout st) to hull_xy + 2 hull_offsets[i], as (x, y) rows.
void copy_hulls(emap_handle* h, const PolyStage& st, int n_polygons, const int64_t* hull_offsets, double* hull_xy) {
  const char* back = h->poly.down;
  const PolyResult* r = (const PolyResult*)back;
  const PolyDesc* d = (const PolyDesc*)(h->poly.up.host + st.desc);
  const double2* ring = (const double2*)(back + st.ring);
  for (int i = 0; i < n_polygons; i++) {
    const double2* src = ring + d[i].ring_off;
    double* dst = hull_xy + 2 * hull_offsets[i];
    for (int k = 0; k < r[i].n_ring; k++) { dst[2 * k] = src[k].x; dst[2 * k + 1] = src[k].y; }
  }
}

}  // namespace

extern "C" {

// EM.py:837-889 get_polygon_traversability (WRAP:254-281): area, clip and bounding box on the host in fp32, then a
// batch of one polygon whose work items are every tile of the grid (the mask is written everywhere, and the statistics
// need no poison pass), one device-to-host copy and one synchronisation.
int emap_polygon_traversability(emap_handle* h, const float* polygon_xy, int32_t n_vertices, const float* checker_plane,
                                double safe_thresh, double safe_min_thresh, int32_t max_unsafe_n, double result[3],
                                double* hull_xy, int32_t* n_hull, float* mask) {
  ENTER(h);
  if (!polygon_xy || !result || !n_hull || *n_hull < 0 || (*n_hull > 0 && !hull_xy))
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability: null argument or negative hull capacity");
  if (n_vertices < 3 || n_vertices > EMAP_POLYGON_MAX_VERTICES)
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability: 3 to EMAP_POLYGON_MAX_VERTICES vertices required");
  int64_t off[2], rows;
  PolyStage st;
  const int rc = check_polygons(h, 1, &n_vertices, polygon_xy, checker_plane, safe_thresh, safe_min_thresh, max_unsafe_n,
                                true, false, mask, true, kRingHead, result, off, rows, st);
  if (rc) return rc;
  if (rows > *n_hull) {
    *n_hull = (int32_t)rows;
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability: hull capacity too small (needed length in *n_hull)");
  }
  copy_hulls(h, st, 1, off, hull_xy);
  *n_hull = (int32_t)rows;
  return EMAP_OK;
}

// The check_safety service (CheckSafety.srv) in one call: every polygon's answer is emap_polygon_traversability's.  The
// work items are only the tiles of each polygon's cell bounding box; k_poly_poison carries the map-wide NaN rule to
// the cells outside them.  One upload, one read-back copy and one synchronisation (plus one for long rings).
int emap_polygon_traversability_batch(emap_handle* h, int32_t n_polygons, const int32_t* n_vertices,
                                      const float* polygon_xy, const float* checker_plane, double safe_thresh,
                                      double safe_min_thresh, int32_t max_unsafe_n, double* results, double* hull_xy,
                                      int64_t* hull_offsets, int64_t* hull_rows) {
  ENTER(h);
  if (n_polygons < 1 || n_polygons > EMAP_POLYGON_MAX_BATCH)
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability_batch: 1 to EMAP_POLYGON_MAX_BATCH polygons required");
  if (!n_vertices || !polygon_xy || !results || (hull_xy && (!hull_offsets || !hull_rows)) ||
      (hull_rows && *hull_rows < 0))
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability_batch: null argument or negative hull capacity");
  for (int i = 0; i < n_polygons; i++)
    if (n_vertices[i] < 3 || n_vertices[i] > EMAP_POLYGON_MAX_VERTICES)
      return fail(h, EMAP_ERR_INVALID,
                  "emap_polygon_traversability_batch: 3 to EMAP_POLYGON_MAX_VERTICES vertices required per polygon");
  const bool hulls = hull_xy != nullptr;
  // traversability_polygon.py:25 compares the whole interior: with fp32(1 - safe_thresh) < 0 the masked 0 of every cell
  // outside a polygon is over too, so its count and hull take the whole map.  Every polygon then brings every tile and
  // the whole column window, as the single call does.
  const bool whole_map = (float)(1.0 - safe_thresh) < 0.0f;
  int64_t total;
  PolyStage st;
  const int rc = check_polygons(h, n_polygons, n_vertices, polygon_xy, checker_plane, safe_thresh, safe_min_thresh,
                                max_unsafe_n, whole_map, true, nullptr, hulls, kBatchRingHead, results, hull_offsets,
                                total, st);
  if (rc) return rc;
  if (!hulls) {
    if (hull_rows) *hull_rows = 0;
    return EMAP_OK;
  }
  if (total > *hull_rows) {
    *hull_rows = total;
    return fail(h, EMAP_ERR_INVALID,
                "emap_polygon_traversability_batch: hull capacity too small (needed rows in *hull_rows)");
  }
  copy_hulls(h, st, n_polygons, hull_offsets, hull_xy);
  *hull_rows = total;
  return EMAP_OK;
}

}  // extern "C"
