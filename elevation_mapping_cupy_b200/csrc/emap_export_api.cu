// emap_export_api.cu -- the export calls of the C ABI (include/emap.h): layers, map windows (emap_get_submaps), windows
// in a requester's frame (emap_get_transformed_submaps), plane segmentation of a window, the map point cloud and normal
// arrows, the layer pointers, and the layers' values at points (emap_map_values_at).
#include "emap_handle.cuh"
#include "emap_export.cuh"
#include "emap_submap.cuh"
#include "emap_planes.cuh"
#include "emap_regions.cuh"
#include "emap_postprocess.cuh"
#include "emap_resample.cuh"
#include "emap_grid.cuh"
#include "emap_mapcloud.cuh"
#include "emap_values_at.cuh"
#include "emap_filters.cuh"

namespace {

int layer_index(const char* name) {
  static const char* names[] = {"elevation", "variance", "is_valid", "traversability", "time", "upper_bound", "is_upper_bound"};
  for (int i = 0; i < 7; i++) if (!strcmp(name, names[i])) return i;
  return -1;
}
// export_value's named kinds: kExportNames[k] is kind k, except the last, normal_color (kind EXPORT_KIND_PLANE is a
// caller plane)
const char* const kExportNames[] = {"elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
                                    "normal_x", "normal_y", "normal_z", "normal_color"};
constexpr int kNumExportNames = sizeof(kExportNames) / sizeof(kExportNames[0]);
static_assert(kNumExportNames == EXPORT_KIND_PLANE + 1, "kinds 0..8 are named in order, then normal_color");
inline int export_kind(int name_index) {
  return name_index == kNumExportNames - 1 ? EXPORT_KIND_NORMAL_COLOR : name_index;
}

// The n (<= EXPORT_MAX_LAYERS) layers of an export call.  names[k]: a name of kExportNames, or planes[k] != NULL: a (W,W)
// device plane exported with flags[k] (bit 0 fill_nan, bit 1 add the centre height).  Returns false, with the message
// in h->err, for an unknown name.
bool export_list(emap_handle* h, int32_t n, const char* const* names, const float* const* planes, const int32_t* flags,
                 ExportList& L) {
  memset(&L, 0, sizeof(L));
  L.n = n;
  for (int k = 0; k < n; k++) {
    if (planes && planes[k]) {
      L.kind[k] = EXPORT_KIND_PLANE; L.plane[k] = planes[k]; L.flags[k] = flags ? flags[k] : 0;
      continue;
    }
    int kind = -1;
    if (names && names[k])
      for (int i = 0; i < kNumExportNames; i++) if (!strcmp(names[k], kExportNames[i])) kind = export_kind(i);
    if (kind < 0) { h->err = std::string("Layer ") + (names && names[k] ? names[k] : "(null)") + " is not in the map"; return false; }
    L.kind[k] = kind;
  }
  return true;
}

// Layers by one k_export_multi launch, one device-to-host copy and one synchronisation (layers as export_list).
int export_layers(emap_handle* h, int32_t n, const char* const* names, const float* const* planes, const int32_t* flags,
                  float* out_host, int64_t n_out_total) {
  if (n < 1 || n > EXPORT_MAX_LAYERS || !out_host) return fail(h, EMAP_ERR_INVALID, "emap_get_layers: 1..24 layers, non-null output");
  const int Wo = h->dc.W - 2;
  const size_t per = (size_t)Wo * Wo;
  if (n_out_total != (int64_t)(per * n)) return fail(h, EMAP_ERR_INVALID, "output must hold n * (cell_n-2)^2 floats");
  ExportList L;
  if (!export_list(h, n, names, planes, flags, L)) return EMAP_ERR_NOLAYER;
  int rc = grow(h, h->d_export, per * n, 0, false);
  if (rc) return rc;
  const auto kern = export_has_colour(L) ? k_export_multi<true> : k_export_multi<false>;
  kern<<<dim3(cdiv((i64)per, 256), n), 256, 0, h->stream>>>(h->dc, h->map, h->normal, h->d_export, L, h->center[2],
                                                             h->cfg.use_only_above_for_upper_bound);
  LAUNCH_CHECK();
  CK(cudaMemcpyAsync(out_host, h->d_export, sizeof(float) * per * n, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

// emap_get_map_points (ARROWS false) / emap_get_normal_arrows (true): the count pass and the scan, one synchronisation
// for the total; then, if the caller's capacity holds it, the write pass, the payload's copies and one more
// synchronisation.  Nothing reaches the caller's rows when the capacity is too small.
template <bool ARROWS>
int map_cloud(emap_handle* h, int64_t* n_rows, float* xyz, int32_t* ids, double* seg) {
  const int Wo = h->dc.W - 2;
  const int n_chunks = cdiv(Wo, MC_TILE), n_tiles = cdiv(Wo, MC_TILE);
  const int n = Wo * n_chunks, span = MC_TILE * n_chunks;      // count entries; entries of one scan CTA
  static_assert(MC_TILE % 4 == 0, "k_mapcloud_scan reads whole spans as int4");
  // cell_n <= 2049 (emap_create): at most 64 chunks, a span of at most 2048 entries, two per scan thread
  if (span > 2 * 1024) return fail(h, EMAP_ERR_INVALID, "map point cloud: cell_n too large for k_mapcloud_scan");
  int rc = grow(h, h->mapcloud.table, 2 * (size_t)n + 1, 0, false);
  if (rc) return rc;
  if (!h->mapcloud.count) CK(h->mapcloud.count.alloc(1));
  int* cnt = h->mapcloud.table;
  int* off = cnt + n;
  const dim3 grid(n_tiles, n_chunks);
  const MapCloudGeom g = {(double)h->center[0], (double)h->center[1], h->cfg.resolution};
  MapCloudOut o = {nullptr, nullptr, nullptr};
  k_mapcloud<ARROWS, false><<<grid, MC_THREADS, 0, h->stream>>>(h->dc, h->map, h->normal, h->center[2], cnt, nullptr, g, o);
  LAUNCH_CHECK();
  k_mapcloud_scan<<<cdiv(n, span), 1024, 0, h->stream>>>(cnt, off, n, span);
  LAUNCH_CHECK();
  CK(cudaMemcpyAsync(h->mapcloud.count, off + n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  const int64_t total = *h->mapcloud.count;
  if (total > *n_rows) {
    *n_rows = total;
    return fail(h, EMAP_ERR_INVALID, "map point cloud: capacity too small (needed rows in the count argument)");
  }
  *n_rows = total;
  if (!total) return EMAP_OK;
  const size_t id_bytes = ARROWS ? (sizeof(int32_t) * (size_t)total + 255) & ~(size_t)255 : 0;
  const size_t row_bytes = ARROWS ? 6 * sizeof(double) : 3 * sizeof(float);
  rc = grow(h, h->mapcloud.out, id_bytes + row_bytes * (size_t)total, 0, false);
  if (rc) return rc;
  char* base = h->mapcloud.out;
  o.xyz = (float*)base; o.ids = (int32_t*)base; o.seg = (double*)(base + id_bytes);
  k_mapcloud<ARROWS, true><<<grid, MC_THREADS, 0, h->stream>>>(h->dc, h->map, h->normal, h->center[2], cnt, off, g, o);
  LAUNCH_CHECK();
  if (ARROWS) {
    CK(cudaMemcpyAsync(ids, o.ids, sizeof(int32_t) * total, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(seg, o.seg, 6 * sizeof(double) * total, cudaMemcpyDeviceToHost, h->stream));
  } else {
    CK(cudaMemcpyAsync(xyz, o.xyz, 3 * sizeof(float) * total, cudaMemcpyDeviceToHost, h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

// emap_map_values_at's cells: cell (r, c) of the full export (the (W-2)^2 planes of emap_get_layers, flipped on both
// axes) is state cell (W - 2 - r, W - 2 - c), read through export_cell like every export.  value() picks the layer's
// kind once, so each cell read is that kind's alone (KIND -1: the kind read at run time, for the normal planes and
// normal_color).
template <bool COLOUR>
struct VaMapSrc {
  int n;
  DevCfg c;
  const float* map;
  const float* normal;
  ExportList L;
  float center_z;
  int only_above;
  template <int KIND>
  struct Cell {
    const VaMapSrc& s;
    __device__ __forceinline__ float at(int l, int r, int cc) const {
      return export_cell<COLOUR>(s.c, s.map, s.normal, s.c.W - 2 - r, s.c.W - 2 - cc, KIND < 0 ? s.L.kind[l] : KIND,
                                 s.center_z, s.only_above, s.L.plane[l], s.L.flags[l]);
    }
  };
  __device__ __forceinline__ float value(const VaPoint& p, int l) const {
    switch (L.kind[l]) {
      case 0: return va_value(p, Cell<0>{*this}, l);
      case 1: return va_value(p, Cell<1>{*this}, l);
      case 2: return va_value(p, Cell<2>{*this}, l);
      case 3: return va_value(p, Cell<3>{*this}, l);
      case 4: return va_value(p, Cell<4>{*this}, l);
      case 5: return va_value(p, Cell<5>{*this}, l);
      case EXPORT_KIND_PLANE: return va_value(p, Cell<EXPORT_KIND_PLANE>{*this}, l);
      default: return va_value(p, Cell<-1>{*this}, l);
    }
  }
};

}  // namespace

extern "C" {

int emap_get_map_with_name(emap_handle* h, const char* name, float* out_host, int64_t n_out) {
  ENTER(h);
  if (!name || !out_host) return fail(h, EMAP_ERR_INVALID, "null argument");
  return export_layers(h, 1, &name, nullptr, nullptr, out_host, n_out);
}

// Several layers in one launch, one device-to-host copy and one synchronisation (WRAP:213-252 get_grid_map exports a list
// of layers per call).
int emap_get_layers(emap_handle* h, int32_t n, const char* const* names, const float* const* planes, const int32_t* flags,
                    float* out_host, int64_t n_out_total) {
  ENTER(h);
  return export_layers(h, n, names, planes, flags, out_host, n_out_total);
}

static_assert(EMAP_SUBMAP_MAX_WINDOWS == SUBMAP_MAX_WINDOWS && EMAP_SUBMAP_MAX_LAYERS == EXPORT_MAX_LAYERS,
              "emap.h states the kernel's limits");

static bool submap_lengths_ok(int64_t n, const double* windows) {
  for (int64_t w = 0; w < n; w++)
    for (int a = 2; a < 4; a++)
      if (!(std::isfinite(windows[4 * w + a]) && windows[4 * w + a] >= 0.0)) return false;
  return true;
}

// submap_window for each of n windows: info[5 w ..] and centres[2 w ..]
static void submap_windows(int32_t cell_n, double res, const double m[2], int32_t n, const double* windows,
                           int32_t* info, double* centres) {
  for (int32_t w = 0; w < n; w++) submap_window(cell_n, res, m, windows + 4 * w, info + 5 * w, centres + 2 * w);
}

// The host part of emap_get_submaps on its own (no handle, no device).
int emap_submap_windows(int32_t cell_n, double resolution, const double center[2], int32_t n_windows,
                        const double* windows, int32_t* info, double* centres) {
  if (!center || !windows || !info || !centres || cell_n < 3 || !(std::isfinite(resolution) && resolution > 0.0) ||
      n_windows < 0 || !submap_lengths_ok(n_windows, windows))
    return EMAP_ERR_INVALID;
  submap_windows(cell_n, resolution, center, n_windows, windows, info, centres);
  return EMAP_OK;
}

// Appends the successful window q = submap_window's info to k_submap's table: its first work item is `tiles` and its
// first output float `total`, both advanced past it.
static void submap_add(SubmapArgs& a, int W, const int32_t q[5], int n_layers, int& tiles, long long& total) {
  SubmapWin& s = a.win[a.n_win++];
  s.r0 = (int16_t)(W - 2 - q[1]); s.c0 = (int16_t)(W - 2 - q[2]);
  s.rows = (int16_t)q[3]; s.cols = (int16_t)q[4];
  s.tile0 = tiles; s.off = total;
  tiles += cdiv(q[3], SUBMAP_ROWS);
  total += (long long)n_layers * q[3] * q[4];
}

// The get_raw_submap service (elevation_mapping_ros.cpp:507-553) for a batch of windows: the windows on the host
// (submap_window), every (window, layer, row) of the batch in one k_submap launch whose table is its parameters.  Host
// output: one device-to-host copy and one synchronisation; device output: stream-ordered, no synchronisation.  Every
// check runs before anything is written or launched.
int emap_get_submaps(emap_handle* h, int32_t n_windows, const double* windows, int32_t n_layers, const char* const* names,
                     const float* const* planes_device, const int32_t* flags, float* out, int32_t out_is_device,
                     int64_t out_floats, int32_t* info, double* centres) {
  ENTER(h);
  NvtxRange nv("emap:get_submaps");
  if (!windows || !names || !out || !info || !centres) return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: null argument");
  if (n_windows < 1 || n_windows > EMAP_SUBMAP_MAX_WINDOWS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: 1 to EMAP_SUBMAP_MAX_WINDOWS windows required");
  if (n_layers < 1 || n_layers > EMAP_SUBMAP_MAX_LAYERS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: 1 to EMAP_SUBMAP_MAX_LAYERS layers required");
  if (!submap_lengths_ok(n_windows, windows))
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: lengths must be finite and >= 0");
  SubmapArgs a;
  if (!export_list(h, n_layers, names, planes_device, flags, a.L)) return EMAP_ERR_INVALID;
  const int W = h->dc.W;
  const double m[2] = {h->center[0], h->center[1]};
  std::vector<int32_t> inf(5 * (size_t)n_windows);
  std::vector<double> cen(2 * (size_t)n_windows);
  a.n_win = 0;
  int tiles = 0;
  long long total = 0;
  submap_windows(W, h->cfg.resolution, m, n_windows, windows, inf.data(), cen.data());
  for (int w = 0; w < n_windows; w++)
    if (inf[5 * w]) submap_add(a, W, &inf[5 * w], n_layers, tiles, total);
  if (total > out_floats)
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: out_floats is below the layers times the windows' cells");
  memcpy(info, inf.data(), sizeof(int32_t) * inf.size());
  memcpy(centres, cen.data(), sizeof(double) * cen.size());
  if (!a.n_win) return EMAP_OK;
  float* dst = out;
  if (!out_is_device) {
    const int rc = grow(h, h->d_export, (size_t)total, 0, false);
    if (rc) return rc;
    dst = h->d_export;
  }
  const auto kern = export_has_colour(a.L) ? k_submap<true> : k_submap<false>;
  kern<<<dim3(tiles, n_layers), dim3(32, SUBMAP_ROWS), 0, h->stream>>>(h->dc, h->map, h->normal, dst, a, h->center[2],
                                                                       h->cfg.use_only_above_for_upper_bound);
  LAUNCH_CHECK();
  if (!out_is_device) {
    CK(cudaMemcpyAsync(out, dst, sizeof(float) * total, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}

// The live map's layers at points: emap_grid_values_at on the full export (rows = cols = cell_n - 2, position = the map
// centre's x and y widened to double, the handle's resolution), its cells read in place.  The centre travels in the
// kernel's parameters.
int emap_map_values_at(emap_handle* h, int32_t n_layers, const char* const* names, const float* const* planes_device,
                       const int32_t* flags, int64_t n_points, const double* positions, int32_t positions_on_device,
                       int32_t method, const emap_values_out* out, int32_t out_is_device) {
  ENTER(h);
  const char* e = !names ? "null argument" : va_check(n_layers, n_points, positions, method, out);
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_map_values_at: ") + e).c_str());
  ExportList L;
  if (!export_list(h, n_layers, names, planes_device, flags, L)) return EMAP_ERR_INVALID;
  if (n_points == 0) return EMAP_OK;
  NvtxRange nv("map_values_at");
  if (int rc = va_room(h, n_layers, n_points, out_is_device)) return rc;
  const double* xy = positions;
  if (int rc = stage_inputs(h, h->lookup.up, xy, positions_on_device ? 0 : sizeof(double) * 2 * n_points)) return rc;
  const int Wo = h->dc.W - 2;
  VaGeom g;
  g.rows = g.cols = Wo;
  g.res = h->cfg.resolution;
  for (int a = 0; a < 2; a++) {
    g.pos[a] = (double)h->center[a];
    g.len[a] = (double)Wo * h->cfg.resolution;
  }
  if (export_has_colour(L)) {
    const VaMapSrc<true> s{n_layers, h->dc, h->map, h->normal, L, h->center[2], h->cfg.use_only_above_for_upper_bound};
    return va_launch(h, g, s, method, n_points, xy, out, out_is_device);
  }
  const VaMapSrc<false> s{n_layers, h->dc, h->map, h->normal, L, h->center[2], h->cfg.use_only_above_for_upper_bound};
  return va_launch(h, g, s, method, n_points, xy, out, out_is_device);
}

static_assert(EMAP_TRANSFORM_TOLERANCE == TSUB_ORTHO_TOL && EMAP_TRANSFORMED_WINDOWS_PER_LAUNCH == TSUB_MAX_WINDOWS,
              "emap.h states the transformed windows' limits");

// Why n windows and their transforms are rejected (nullptr: accepted); else the new maps' geometry (transformed_window)
// in g.
static const char* transformed_windows(int32_t cell_n, double res, const double m[2], int32_t n, const double* windows,
                                       const double* transforms, std::vector<TSubGeom>& g) {
  if (!submap_lengths_ok(n, windows)) return "lengths must be finite and >= 0";
  for (int32_t w = 0; w < n; w++)
    if (!tsub_transform_ok(transforms + 12 * w))
      return "a transform is not finite or its R is not orthonormal within EMAP_TRANSFORM_TOLERANCE";
  g.resize(n);
  for (int32_t w = 0; w < n; w++) transformed_window(cell_n, res, m, windows + 4 * w, transforms + 12 * w, g[w]);
  return nullptr;
}

// info {success, rows, cols} and geometry {centre, length} of every new map
static void write_transformed(const std::vector<TSubGeom>& g, int32_t* info, double* geometry) {
  for (size_t w = 0; w < g.size(); w++) {
    info[3 * w] = g[w].win[0]; info[3 * w + 1] = g[w].size[0]; info[3 * w + 2] = g[w].size[1];
    for (int a = 0; a < 2; a++) { geometry[4 * w + a] = g[w].pos[a]; geometry[4 * w + 2 + a] = g[w].len[a]; }
  }
}

// The host part of emap_get_transformed_submaps on its own (no handle, no device).
int emap_transformed_submap_windows(int32_t cell_n, double resolution, const double center[2], int32_t n_windows,
                                    const double* windows, const double* transforms, int32_t* info, double* geometry) {
  std::vector<TSubGeom> g;
  if (!center || !windows || !transforms || !info || !geometry || cell_n < 3 ||
      !(std::isfinite(resolution) && resolution > 0.0) || n_windows < 0 ||
      transformed_windows(cell_n, resolution, center, n_windows, windows, transforms, g))
    return EMAP_ERR_INVALID;
  write_transformed(g, info, geometry);
  return EMAP_OK;
}

// get_raw_submap with a request frame other than the map frame (elevation_mapping_ros.cpp:507-553 with grid_map's
// getTransformedMap): the geometry on the host (transformed_window), then per launch of up to TSUB_MAX_WINDOWS windows
// the two scatter passes and the gather (csrc/emap_submap.cuh), each launch's table in its parameters.  Output, stream
// and graph rules as emap_get_submaps; every check runs before anything is written or launched.
int emap_get_transformed_submaps(emap_handle* h, int32_t n_windows, const double* windows, const double* transforms,
                                 double sample_ratio, int32_t n_layers, const char* const* names,
                                 const float* const* planes_device, const int32_t* flags, float* out,
                                 int32_t out_is_device, int64_t out_floats, int32_t* info, double* geometry) {
  ENTER(h);
  NvtxRange nv("emap:get_transformed_submaps");
  if (!windows || !transforms || !names || !out || !info || !geometry)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: null argument");
  if (n_windows < 1 || n_windows > EMAP_SUBMAP_MAX_WINDOWS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: 1 to EMAP_SUBMAP_MAX_WINDOWS windows required");
  if (n_layers < 1 || n_layers > EMAP_SUBMAP_MAX_LAYERS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: 1 to EMAP_SUBMAP_MAX_LAYERS layers required");
  const int W = h->dc.W;
  const double res = h->cfg.resolution;
  const double m[2] = {h->center[0], h->center[1]};
  std::vector<TSubGeom> g;
  if (const char* e = transformed_windows(W, res, m, n_windows, windows, transforms, g))
    return fail(h, EMAP_ERR_INVALID, (std::string("emap_get_transformed_submaps: ") + e).c_str());
  if (!(std::isfinite(sample_ratio) && sample_ratio >= 0.0))
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: sample_ratio must be finite and >= 0");
  ExportList L;
  if (!export_list(h, n_layers, names, planes_device, flags, L)) return EMAP_ERR_INVALID;
  long long cells = 0;
  for (int w = 0; w < n_windows; w++) {
    const long long n = (long long)g[w].size[0] * g[w].size[1];
    if (n > INT32_MAX - TSUB_THREADS)
      return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: a new map of 2^31 cells or more");
    cells += n;
  }
  if (n_layers * cells > out_floats)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: out_floats is below the layers times the new maps' cells");
  write_transformed(g, info, geometry);
  if (!cells) return EMAP_OK;
  int rc;
  if ((rc = grow(h, h->tsub.key1, (size_t)cells, 0, true)) || (rc = grow(h, h->tsub.key2, (size_t)cells, 0, true))) return rc;
  float* dst = out;
  if (!out_is_device) {
    if ((rc = grow(h, h->d_export, (size_t)(n_layers * cells), 0, false))) return rc;
    dst = h->d_export;
  }
  const bool colour = export_has_colour(L);
  TSubArgs a;
  a.L = L;
  a.n_samples = sample_ratio > 0.0 ? 5 : 1;
  a.res = res;
  a.s = res * sample_ratio;
  long long cell0 = 0;
  for (int w0 = 0; w0 < n_windows;) {
    a.n_win = 0;
    int blk_src = 0, blk_dst = 0;
    for (; w0 < n_windows && a.n_win < TSUB_MAX_WINDOWS; w0++) {
      const TSubGeom& q = g[w0];
      if (!q.win[0] || !q.size[0] || !q.size[1]) continue;
      TSubWin& s = a.win[a.n_win++];
      for (int k = 0; k < 9; k++) s.R[k] = transforms[12 * w0 + k];
      for (int k = 0; k < 3; k++) s.t[k] = transforms[12 * w0 + 9 + k];
      s.x0 = q.centre[0] + (0.5 * (q.win[3] * res) - 0.5 * res);
      s.y0 = q.centre[1] + (0.5 * (q.win[4] * res) - 0.5 * res);
      for (int k = 0; k < 2; k++) { s.pos[k] = q.pos[k]; s.len[k] = q.len[k]; }
      s.r0 = (int16_t)(W - 2 - q.win[1]); s.c0 = (int16_t)(W - 2 - q.win[2]);
      s.rows = (int16_t)q.win[3]; s.cols = (int16_t)q.win[4];
      s.nrows = q.size[0]; s.ncols = q.size[1];
      s.blk_src = blk_src; s.blk_dst = blk_dst; s.cell0 = cell0;
      blk_src += cdiv((i64)q.win[3] * q.win[4], TSUB_THREADS);
      blk_dst += cdiv((i64)q.size[0] * q.size[1], TSUB_THREADS);
      cell0 += (long long)q.size[0] * q.size[1];
    }
    if (!a.n_win) continue;
    k_tsub_scatter<1><<<blk_src, TSUB_THREADS, 0, h->stream>>>(h->dc, h->map, h->tsub.key1, h->tsub.key2, a, h->center[2]);
    LAUNCH_CHECK();
    k_tsub_scatter<2><<<blk_src, TSUB_THREADS, 0, h->stream>>>(h->dc, h->map, h->tsub.key1, h->tsub.key2, a, h->center[2]);
    LAUNCH_CHECK();
    const auto gather = colour ? k_tsub_gather<true> : k_tsub_gather<false>;
    gather<<<blk_dst, TSUB_THREADS, 0, h->stream>>>(h->dc, h->map, h->normal, h->tsub.key1, h->tsub.key2, dst, a,
                                                    h->center[2], h->cfg.use_only_above_for_upper_bound);
    LAUNCH_CHECK();
  }
  if (!out_is_device) {
    CK(cudaMemcpyAsync(out, dst, sizeof(float) * n_layers * cells, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}

// ---- plane segmentation of one window (emap_segment_planes, csrc/emap_planes.cuh) ----------------------------------

// The scratch of a window of n cells with `slots` label slots, one block: the window, two image planes (fill / median
// ping-pong), union-find parents, flags and ranks, fill keys, the planarity masks, scan block sums, the header words,
// the label statistics and decisions, and the host outputs (carve_plane_out).  With the post-processing
// (emap_planar_terrain) the block also holds its three fp32 planes and the box filter's double row sums, and the host
// outputs all EMAP_TERRAIN_LAYERS layers.
// n is the larger of the input and the resampled grid (emap_plane_decomposition), n_out the resampled one the staged
// layers have; a window is not resampled (n == n_out).
namespace {

struct PlaneScratch {
  float *raw, *img[2];
  int *parent, *flag, *rank, *lab, *bsum, *hdr, *keep;
  unsigned* key;
  unsigned char *bin, *tmp, *bg;
  unsigned long long* st;
  float* pp;
  double* pd;
  int32_t* info;
  double* planes;
  float* layers;
  double* regions;
  int32_t* polys;
  double* verts;
};

// The host outputs, carved alike at the block's tail and in the pinned staging they are read back into: info, the
// plane table, the layers, then the region tables at the capacities of `tables` (none if null).
size_t carve_plane_out(void* base, int64_t n_out, int64_t plane_rows, bool post, const emap_region_out* tables,
                       PlaneScratch& s) {
  Carver c{(uintptr_t)base};
  s.info = c.take<int32_t>(16);
  s.planes = c.take<double>(7 * plane_rows);
  s.layers = c.take<float>((post ? EMAP_TERRAIN_LAYERS : 4) * n_out);
  s.regions = c.take<double>(tables ? RG_ROW * tables->regions_capacity : 0);
  s.polys = c.take<int32_t>(tables ? RG_POLY * tables->polygons_capacity : 0);
  s.verts = c.take<double>(tables ? 2 * tables->vertices_capacity : 0);
  return c.bytes;
}

size_t carve_planes(int64_t n, int64_t n_out, int64_t slots, int64_t plane_rows, bool host_out, bool post,
                    const emap_region_out* tables, void* base, PlaneScratch& s) {
  Carver c{(uintptr_t)base};
  const int64_t m = std::max(n, slots);
  s.raw = c.take<float>(n); s.img[0] = c.take<float>(n); s.img[1] = c.take<float>(n);
  s.parent = c.take<int>(n); s.flag = c.take<int>(m); s.rank = c.take<int>(m); s.lab = c.take<int>(n);
  s.bsum = c.take<int>(m / PL_SCAN + 1); s.hdr = c.take<int>(8); s.keep = c.take<int>(slots);
  s.key = c.take<unsigned>(n);
  s.bin = c.take<unsigned char>(n); s.tmp = c.take<unsigned char>(n); s.bg = c.take<unsigned char>(slots);
  s.st = c.take<unsigned long long>(slots * PL_STAT);
  s.pp = c.take<float>(post ? 3 * n : 0);
  s.pd = c.take<double>(post ? n : 0);
  if (host_out) c.bytes += carve_plane_out((void*)(c.base + c.bytes), n_out, plane_rows, post, tables, s);
  return c.bytes;
}

// Raster-order ranks of the n values in flag into rank (exclusive sums where the value is not 0, else -1), their sum
// into *total (three launches; bsum holds n / PL_SCAN + 1 words).
int scan_ranks(emap_handle* h, const int* flag, int* rank, int* bsum, int64_t n, int* total) {
  const int nb = cdiv(n, PL_SCAN);
  k_pl_scan_blocks<<<nb, PL_SCAN, 0, h->stream>>>(flag, (int)n, bsum);
  LAUNCH_CHECK();
  k_pl_scan_top<<<1, PL_SCAN, 0, h->stream>>>(bsum, nb, total);
  LAUNCH_CHECK();
  k_pl_scan_rank<<<nb, PL_SCAN, 0, h->stream>>>(flag, (int)n, bsum, rank);
  LAUNCH_CHECK();
  return 0;
}

int plane_scan(emap_handle* h, const PlaneScratch& s, int64_t n, int* total) {
  return scan_ranks(h, s.flag, s.rank, s.bsum, n, total);
}

// Union-find merge and flatten of the cells whose parent is >= 0.
int plane_components(emap_handle* h, const PlaneScratch& s, int rows, int cols, int conn8) {
  const int64_t n = (int64_t)rows * cols;
  k_pl_uf_merge<<<cdiv(n, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.parent, rows, cols, conn8);
  LAUNCH_CHECK();
  k_pl_uf_flatten<<<cdiv(n, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.parent, (int)n);
  LAUNCH_CHECK();
  return 0;
}

// One segmentation call's grid and scratch, as plane_check (a window) or grid_plane_check (a caller's grid) and
// segment_window leave them.  The pipeline runs on rows x cols cells of resolution res from the fill's output on: the
// input's in_rows x in_cols resampled, or the input itself.
struct PlaneCall {
  int32_t q[5];                    // submap_window: {success, r0, c0, rows, cols}; a grid: {1, 0, 0, in_rows, in_cols}
  double centre[2];                // the centre of the cells (kept by the resampling)
  const float* grid = nullptr;     // the caller's grid (emap_plane_decomposition), else the window by k_submap
  bool grid_on_device = false;
  int in_rows = 0, in_cols = 0;    // the input
  int rows = 0, cols = 0;          // the pipeline's grid
  double res = 0.0;
  int64_t n = 0, n_in = 0, slots = 0, plane_rows = 0;
  bool post = false;               // emap_planar_terrain: the post-processing's scratch and layers
  const emap_region_out* tables = nullptr;   // host output: the region tables to stage (their capacities)
  double ox = 0.0, oy = 0.0;       // the centre of window cell (0, 0)
  PlaneScratch s;
  double* dst_planes = nullptr;    // where the plane table is written (the caller's or the staging)
  int32_t* dst_info = nullptr;
};

}  // namespace

static_assert(EMAP_PLANE_EIGEN_MIN == PL_EIG_MIN, "emap.h states the fit's threshold");

// Why p is rejected (nullptr: accepted) for a map of resolution `res`; a resampling only when `resample` is false.
static const char* plane_params_error(const emap_plane_params& p, double res, bool resample) {
  if (p.ransac) return "RANSAC refinement is not supported (ransac must be 0)";
  const int mk = std::max(1, std::min(p.median_kernel, 5));
  if (mk != 1 && mk != 3 && mk != 5) return "the median kernel must clamp to 1, 3 or 5";
  if (p.median_repeats < 0 || p.median_repeats > EMAP_PLANE_MAX_REPEATS)
    return "median_repeats must be in [0, EMAP_PLANE_MAX_REPEATS]";
  if (std::isnan(p.resolution)) return "resolution must not be NaN";
  if (!resample && p.resolution > 0.0 && !(std::fabs(res - p.resolution) < 1e-6))
    return "resampling is not supported (resolution must be <= 0 or the map's)";
  if (p.kernel_size < 3 || p.kernel_size % 2 == 0 || p.kernel_size > EMAP_PLANE_MAX_KERNEL)
    return "kernel_size must be odd, >= 3 and <= EMAP_PLANE_MAX_KERNEL";
  if (p.opening < 0 || p.opening > EMAP_PLANE_MAX_OPENING)
    return "opening must be in [0, EMAP_PLANE_MAX_OPENING]";
  if (p.connectivity != 4 && p.connectivity != 8) return "connectivity must be 4 or 8";
  if (!std::isfinite(p.plane_inclination_cos) || !std::isfinite(p.local_inclination_cos) ||
      !std::isfinite(p.patch_error))
    return "the inclination cosines and the patch error must be finite";
  return nullptr;
}

int64_t emap_plane_capacity(int64_t rows, int64_t cols, const emap_plane_params* params) {
  if (!params || rows < 0 || cols < 0) return -1;
  return rows * cols / std::max(params->min_points, 3);
}

// EMAP_ERR_INVALID with "<fn>: <msg>" as the handle's message.
static int fail_in(emap_handle* h, const char* fn, const char* msg) {
  h->err = std::string(fn) + ": " + msg;
  return EMAP_ERR_INVALID;
}

// The checks both segmentation entry points make before anything is written or launched, and the window (c.q,
// c.centre, c.rows, c.cols, c.n, c.plane_rows).  Returns the error's message (without the entry point's name), or nullptr.
static const char* plane_check(emap_handle* h, const double window[4], const emap_plane_params& p, int64_t out_floats,
                               int64_t planes_capacity, PlaneCall& c) {
  if (!submap_lengths_ok(1, window)) return "lengths must be finite and >= 0";
  const double res = h->cfg.resolution;
  if (const char* e = plane_params_error(p, res, false)) return e;
  const double m[2] = {h->center[0], h->center[1]};
  submap_window(h->dc.W, res, m, window, c.q, c.centre);
  c.rows = c.in_rows = c.q[3];
  c.cols = c.in_cols = c.q[4];
  c.res = res;
  c.n = c.n_in = (int64_t)c.rows * c.cols;
  if (c.q[0] && out_floats < 4 * c.n) return "out_floats is below 4 * rows * cols";
  c.plane_rows = emap_plane_capacity(c.rows, c.cols, &p);
  if (c.q[0] && planes_capacity < c.plane_rows)
    return "planes_capacity is below emap_plane_capacity()";
  return nullptr;
}

// The largest grid side emap_plane_decomposition takes, before and after the resampling: the largest window (cell_n <=
// 2049 exports at most 2047 rows), so its scratch never exceeds the window calls'.
constexpr int64_t kPlaneGridMax = 2047;

// emap_plane_decomposition's checks of the grid and its resampling, before anything is written or launched, and the
// call's geometry (c.q, c.centre, c.in_rows / c.in_cols, c.rows / c.cols the resampled size, c.res, c.n, c.n_in,
// c.plane_rows).  Returns the error's message, or nullptr.
static const char* grid_plane_check(const emap_grid& g, int32_t grid_on_device, const emap_plane_params& p,
                                    int64_t out_floats, int64_t planes_capacity, PlaneCall& c) {
  if (const char* e = gl_check_grid(g.data, g.rows, g.cols, g.position, g.resolution, 1)) return e;
  if (g.rows > kPlaneGridMax || g.cols > kPlaneGridMax) return "the grid has more than 2047 rows or columns";
  if (const char* e = plane_params_error(p, g.resolution, true)) return e;
  int64_t size[2];
  rs_geometry(g.rows, g.cols, g.resolution, p.resolution, size, &c.res);
  if (!size[0] || !size[1]) return "the resampled grid has no rows or no columns";
  if (size[0] > kPlaneGridMax || size[1] > kPlaneGridMax) return "the resampled grid has more than 2047 rows or columns";
  c.grid = g.data;
  c.grid_on_device = grid_on_device != 0;
  c.in_rows = (int)g.rows;
  c.in_cols = (int)g.cols;
  c.rows = (int)size[0];
  c.cols = (int)size[1];
  c.q[0] = 1; c.q[1] = c.q[2] = 0; c.q[3] = c.in_rows; c.q[4] = c.in_cols;
  c.centre[0] = g.position[0];
  c.centre[1] = g.position[1];
  c.n_in = g.rows * g.cols;
  c.n = (int64_t)c.rows * c.cols;
  c.plane_rows = emap_plane_capacity(c.rows, c.cols, &p);
  if (out_floats < EMAP_TERRAIN_LAYERS * c.n) return "out_floats is below EMAP_TERRAIN_LAYERS * rows * cols (resampled)";
  if (planes_capacity < c.plane_rows) return "planes_capacity is below emap_plane_capacity() of the resampled grid";
  return nullptr;
}

// The segmentation of a window that plane_check accepted and found inside the map, or of a grid that grid_plane_check
// accepted (ConvexPlaneDecompositionRos.cpp:115-149 up to SlidingWindowPlaneExtractor, without RANSAC): the window by
// k_submap or the caller's grid (staged if on the host), the fill and the median on the input, the resampling when the
// sizes differ (csrc/emap_resample.cuh), then the passes of csrc/emap_planes.cuh on the pipeline's grid, queued on the
// handle's stream.  With host output the layers, plane table and info go to the host outputs at the scratch's tail, which also
// hold the region tables of c.tables.  Layer 0 is the input; a grid's is not written (it is the caller's).
static int segment_window(emap_handle* h, const emap_plane_params& p, bool out_is_device, float* layers_out,
                          double* planes_out, int32_t* info, PlaneCall& c) {
  const int rows = c.rows, cols = c.cols;
  const int64_t n = c.n, n_in = c.n_in, n_scratch = std::max(n, n_in);
  const double res = c.res;
  // labels are at most ceil(n / 2) (a 4-connected checkerboard), plus 0.  The statistics are sized and zeroed for that
  // worst case (128 bytes a slot) because the label count is known only on the device.
  c.slots = n / 2 + 2;
  const int64_t slots = c.slots;
  PlaneScratch& s = c.s;
  int rc = grow(h, h->planes.block,
                carve_planes(n_scratch, n, slots, c.plane_rows, !out_is_device, c.post, c.tables, nullptr, s), 0, false);
  if (rc) return rc;
  carve_planes(n_scratch, n, slots, c.plane_rows, !out_is_device, c.post, c.tables, h->planes.block, s);
  float* dst = out_is_device ? layers_out : s.layers;
  c.dst_planes = out_is_device ? planes_out : s.planes;
  c.dst_info = out_is_device ? info : s.info;
  const float* raw = s.raw;
  if (c.grid) {
    // the caller's grid, read in place on the device and from its staged copy if on the host
    raw = c.grid;
    if ((rc = stage_inputs(h, h->planes.up, raw, c.grid_on_device ? 0 : sizeof(float) * n_in))) return rc;
  } else {
    // the window: k_submap's elevation layer into s.raw
    SubmapArgs a;
    const char* elevation = "elevation";
    if (!export_list(h, 1, &elevation, nullptr, nullptr, a.L)) return EMAP_ERR_CUDA;
    a.n_win = 0;
    int tiles = 0;
    long long total = 0;
    submap_add(a, h->dc.W, c.q, 1, tiles, total);
    k_submap<false><<<dim3(tiles, 1), dim3(32, SUBMAP_ROWS), 0, h->stream>>>(h->dc, h->map, h->normal, s.raw, a,
                                                                             h->center[2],
                                                                             h->cfg.use_only_above_for_upper_bound);
    LAUNCH_CHECK();
  }
  CK(cudaMemsetAsync(s.hdr, 0, 8 * sizeof(int), h->stream));
  CK(cudaMemsetAsync(s.st, 0, sizeof(unsigned long long) * slots * PL_STAT, h->stream));
  // fill: minValues' fixed point per NaN component, on the input
  const int ib = cdiv(n_in, PL_THREADS);
  k_pl_fill_init<<<ib, PL_THREADS, 0, h->stream>>>(raw, s.parent, s.key, s.hdr, (int)n_in);
  LAUNCH_CHECK();
  if ((rc = plane_components(h, s, c.in_rows, c.in_cols, 0))) return rc;
  k_pl_fill_min<<<ib, PL_THREADS, 0, h->stream>>>(raw, s.parent, s.key, c.in_rows, c.in_cols);
  LAUNCH_CHECK();
  k_pl_fill_write<<<ib, PL_THREADS, 0, h->stream>>>(raw, s.parent, s.key, s.img[0], (int)n_in);
  LAUNCH_CHECK();
  // median, numberOfRepeats times
  const int mk = std::max(1, std::min(p.median_kernel, 5));
  int cur = 0;
  if (mk > 1)
    for (int r = 0; r < p.median_repeats; r++, cur ^= 1) {
      (mk == 3 ? k_pl_median<3> : k_pl_median<5>)<<<ib, PL_THREADS, 0, h->stream>>>(s.img[cur], s.img[cur ^ 1],
                                                                                    c.in_rows, c.in_cols);
      LAUNCH_CHECK();
    }
  // changeResolution: inpainting::resample to the pipeline's grid
  if (rows != c.in_rows || cols != c.in_cols) {
    k_rs_resample<<<cdiv(n, RS_THREADS), RS_THREADS, 0, h->stream>>>(s.img[cur], c.in_rows, c.in_cols, s.img[cur ^ 1],
                                                                     rows, cols);
    LAUNCH_CHECK();
    cur ^= 1;
  }
  const int cb = cdiv(n, PL_THREADS);
  const float* img = s.img[cur];
  // sliding-window planarity, opening, labels
  k_pl_fit<<<cb, PL_THREADS, 0, h->stream>>>(img, s.bin, rows, cols, p.kernel_size, res, p.patch_error * p.patch_error,
                                             p.local_inclination_cos);
  LAUNCH_CHECK();
  if (p.opening > 0) {
    k_pl_morph<false><<<cb, PL_THREADS, 0, h->stream>>>(s.bin, s.tmp, rows, cols, p.opening);
    LAUNCH_CHECK();
    k_pl_morph<true><<<cb, PL_THREADS, 0, h->stream>>>(s.tmp, s.bin, rows, cols, p.opening);
    LAUNCH_CHECK();
  }
  k_pl_cc_init<<<cb, PL_THREADS, 0, h->stream>>>(s.bin, s.parent, s.key, s.flag, (int)n);
  LAUNCH_CHECK();
  const bool conn8 = p.connectivity == 8;
  if ((rc = plane_components(h, s, rows, cols, conn8))) return rc;
  (conn8 ? k_pl_first<2> : k_pl_first<1>)<<<cb, PL_THREADS, 0, h->stream>>>(s.parent, s.key, rows, cols);
  LAUNCH_CHECK();
  k_pl_first_flag<<<cb, PL_THREADS, 0, h->stream>>>(s.parent, s.key, s.flag, (int)n);
  LAUNCH_CHECK();
  const int64_t n_blocks = conn8 ? (int64_t)cdiv(rows, 2) * cdiv(cols, 2) : n;
  if ((rc = plane_scan(h, s, n_blocks, s.hdr + 1))) return rc;
  k_pl_label<<<cb, PL_THREADS, 0, h->stream>>>(s.parent, s.key, s.rank, s.lab, (int)n);
  LAUNCH_CHECK();
  // per-label planes
  k_pl_stats<<<cdiv(cdiv(n, PL_RUN), PL_THREADS), PL_THREADS, 0, h->stream>>>(img, s.lab, s.st, rows, cols);
  LAUNCH_CHECK();
  c.ox = c.centre[0] + (0.5 * (rows * res) - 0.5 * res);
  c.oy = c.centre[1] + (0.5 * (cols * res) - 0.5 * res);
  const PlaneLabelArgs la = {c.ox, c.oy, res, p.plane_inclination_cos, p.min_points};
  k_pl_decide<<<cdiv(slots, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.st, s.hdr, s.flag, s.bg, (int)slots, la);
  LAUNCH_CHECK();
  if ((rc = plane_scan(h, s, slots, s.hdr + 2))) return rc;
  k_pl_planes<<<cdiv(slots, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.st, s.rank, s.hdr, c.dst_planes, (int)slots, la);
  LAUNCH_CHECK();
  k_pl_out<<<cb, PL_THREADS, 0, h->stream>>>(c.grid ? nullptr : s.raw, img, s.lab, s.bg, s.hdr, dst, c.dst_info, rows,
                                             cols);
  LAUNCH_CHECK();
  return 0;
}

// Host output: the block's tail (carve_plane_out) in one read-back; the caller's buffers take the layers and planes
// only when the window had a finite cell.  Returns the read-back outputs in t.
static int plane_copy_back(emap_handle* h, const PlaneCall& c, float* layers_out, double* planes_out, int32_t* info,
                           int n_info, PlaneScratch& t) {
  const size_t bytes = carve_plane_out(nullptr, c.n, c.plane_rows, c.post, c.tables, t);
  if (int rc = read_back(h, h->planes, c.s.info, bytes)) return rc;
  carve_plane_out(h->planes.down, c.n, c.plane_rows, c.post, c.tables, t);
  memcpy(info, t.info, n_info * sizeof(int32_t));
  if (info[0]) {
    memcpy(planes_out, t.planes, sizeof(double) * 7 * info[4]);
    const int64_t skip = c.grid ? c.n : 0;      // a grid's layer 0 is the caller's
    memcpy(layers_out + skip, t.layers + skip, sizeof(float) * ((c.post ? EMAP_TERRAIN_LAYERS : 4) * c.n - skip));
  }
  return 0;
}

// The plane decomposition node's segmented planes map for one window: segment_window.  Host output: the copies and
// one synchronisation; device output: stream-ordered, no synchronisation.  Every check runs before anything is written
// or launched.
int emap_segment_planes(emap_handle* h, const double window[4], const emap_plane_params* params, float* layers_out,
                        int32_t out_is_device, int64_t out_floats, double* planes_out, int64_t planes_capacity,
                        int32_t* info) {
  ENTER(h);
  NvtxRange nv("emap:segment_planes");
  if (!window || !params || !layers_out || !planes_out || !info)
    return fail(h, EMAP_ERR_INVALID, "emap_segment_planes: null argument");
  const emap_plane_params p = *params;
  PlaneCall c;
  if (const char* e = plane_check(h, window, p, out_floats, planes_capacity, c))
    return fail_in(h, "emap_segment_planes", e);
  if (!c.q[0]) {
    if (out_is_device) CK(cudaMemsetAsync(info, 0, 5 * sizeof(int32_t), h->stream));
    else memset(info, 0, 5 * sizeof(int32_t));
    return EMAP_OK;
  }
  int rc = segment_window(h, p, out_is_device, layers_out, planes_out, info, c);
  if (rc) return rc;
  PlaneScratch t;
  if (!out_is_device && (rc = plane_copy_back(h, c, layers_out, planes_out, info, 5, t))) return rc;
  return EMAP_OK;
}

// ---- planar regions of one window (emap_extract_planar_regions, csrc/emap_regions.cuh) -----------------------------

namespace {

// The region passes' scratch for U upsampled pixels, `rows` plane rows and n source cells (49 bytes per upsampled
// pixel, EMAP_REGION_SCRATCH_PER_PIXEL): the mask bytes, the two images' union-find parents (U + 1 words: the edge
// node), the point counts, the boundary marks, the kept flags and their ranks, the scan block sums, the polygon
// records (key, point count, start) and the per-row tables.  After the two passes the parents, marks, flags and ranks
// are reused as the output order's arrays (see emap_extract_planar_regions).
struct RegionScratch {
  unsigned char* mask;
  int *pa, *pb, *cnt, *have, *flag, *rank, *bsum, *pr, *hdr, *ok, *lcnt, *lreg, *loff, *roff, *lfill;
  unsigned long long *khi, *klo;
  int *rn, *rcode;
};

size_t carve_regions(int64_t U, int64_t rows, int64_t n, void* base, RegionScratch& s) {
  Carver c{(uintptr_t)base};
  s.mask = c.take<unsigned char>(U);
  s.pa = c.take<int>(U + 1); s.pb = c.take<int>(U + 1); s.cnt = c.take<int>(U); s.have = c.take<int>(U);
  s.flag = c.take<int>(U); s.rank = c.take<int>(U); s.bsum = c.take<int>(U / PL_SCAN + 1);
  s.pr = c.take<int>(n); s.hdr = c.take<int>(8); s.ok = c.take<int>(6 * (rows + 1));
  s.lcnt = s.ok + (rows + 1); s.lreg = s.lcnt + (rows + 1); s.loff = s.lreg + (rows + 1);
  s.roff = s.loff + (rows + 1); s.lfill = s.roff + (rows + 1);
  s.khi = c.take<unsigned long long>(U); s.klo = c.take<unsigned long long>(U);
  s.rn = c.take<int>(U); s.rcode = c.take<int>(U);
  return c.bytes;
}

}  // namespace

static_assert(EMAP_REGION_MAX_MARGIN == RG_MAX_MARGIN, "emap.h states the margin's bound");
static_assert(EMAP_REGION_ROW == RG_ROW && EMAP_REGION_POLYGON == RG_POLY, "emap.h states the table rows");

static_assert(EMAP_POST_MAX_KERNEL == PP_MAX_KERNEL && EMAP_POST_MAX_OFFSET == PP_MAX_OFFSET,
              "emap.h states the post-processing's bounds");

// The post-processing's kernel sizes and the final pass's arithmetic, as postprocess_window launches them.
struct PostCall {
  int dil = 0, box = 0, gauss = 0;  // the smoothing's kernel sizes (kernelSizeInPixels)
  PpFinal fin;
};

// Why q is rejected (nullptr: accepted) for a map of resolution res; else pc.
static const char* post_params_error(const emap_postprocess_params& q, double res, double ext_offset, PostCall& pc) {
  pc.dil = pp_kernel_size(q.smoothing_dilation_size, res);
  pc.box = pp_kernel_size(q.smoothing_box_kernel_size, res);
  pc.gauss = pp_kernel_size(q.smoothing_gauss_kernel_size, res);
  if (pc.dil < 0 || pc.box < 0 || pc.gauss < 0)
    return "the smoothing sizes must be finite, >= 0 and give kernels of at most EMAP_POST_MAX_KERNEL cells";
  if (q.nonplanar_horizontal_offset < 0 || q.nonplanar_horizontal_offset > EMAP_POST_MAX_OFFSET)
    return "nonplanar_horizontal_offset must be in [0, EMAP_POST_MAX_OFFSET]";
  if (!std::isfinite(q.nonplanar_height_offset)) return "nonplanar_height_offset must be finite";
  // Eigen narrows a double scalar to the float matrix's scalar type before the fp32 operation (promote_scalar_arg)
  pc.fin.dil = q.nonplanar_horizontal_offset > 0;
  pc.fin.add_on = ext_offset != 0.0 || q.nonplanar_height_offset != 0.0;
  pc.fin.sub_on = q.nonplanar_height_offset != 0.0;
  pc.fin.add = (float)(ext_offset + q.nonplanar_height_offset);
  pc.fin.sub = (float)q.nonplanar_height_offset;
  return nullptr;
}

static PpEllipse pp_ellipse(int size) {
  PpEllipse e;
  e.r = (size - 1) / 2;
  for (int i = 0; i < size; i++) e.half[i] = rg_ellipse_half(e.r, i);
  return e;
}

// Postprocessing::postprocess on the layers segment_window left in dst (layer 1 is E, layer 3 M): layers 4 .. 9.  The
// scratch is the block's three post planes (a: fill input, then the box output; b: fill output, then the dilated E; t:
// the closing's and the Gaussian's intermediates) and its double row sums.  The launches depend on the parameters only.
static int postprocess_window(emap_handle* h, PlaneCall& c, const emap_postprocess_params& q, const PostCall& pc, float* dst) {
  PlaneScratch& s = c.s;
  const int rows = c.rows, cols = c.cols, n = (int)c.n, cb = cdiv(c.n, PL_THREADS);
  float *a = s.pp, *b = s.pp + c.n, *t = s.pp + 2 * c.n;
  float* L[EMAP_TERRAIN_LAYERS];
  for (int k = 0; k < EMAP_TERRAIN_LAYERS; k++) L[k] = dst + (int64_t)k * c.n;
  int rc;
  // elevationWithNaN, then minValues with the segmentation's fill; its finite-cell word is hdr[3], so the call's
  // success (hdr[0]) stays the segmentation's
  k_pp_mask<<<cb, PL_THREADS, 0, h->stream>>>(dst, a, L[4], s.hdr, n);
  LAUNCH_CHECK();
  k_pl_fill_init<<<cb, PL_THREADS, 0, h->stream>>>(a, s.parent, s.key, s.hdr + 3, n);
  LAUNCH_CHECK();
  if ((rc = plane_components(h, s, rows, cols, 0))) return rc;
  k_pl_fill_min<<<cb, PL_THREADS, 0, h->stream>>>(a, s.parent, s.key, rows, cols);
  LAUNCH_CHECK();
  k_pl_fill_write<<<cb, PL_THREADS, 0, h->stream>>>(a, s.parent, s.key, b, n);
  LAUNCH_CHECK();
  // MORPH_CLOSE (its dilation also stores elevationWithNaN_i), then the sloped dilation
  const PpEllipse ec = pp_ellipse(pc.dil);
  k_pp_morph<true><<<cb, PL_THREADS, 0, h->stream>>>(b, t, L[5], s.hdr, rows, cols, ec);
  LAUNCH_CHECK();
  k_pp_morph<false><<<cb, PL_THREADS, 0, h->stream>>>(t, L[6], nullptr, s.hdr, rows, cols, ec);
  LAUNCH_CHECK();
  k_pp_slope<<<cb, PL_THREADS, 0, h->stream>>>(L[6], L[7], s.hdr, rows, cols, pc.dil, (float)c.res);
  LAUNCH_CHECK();
  // smooth_planar: boxFilter, then GaussianBlur (rows, then columns)
  k_pp_box_rows<<<cb, PL_THREADS, 0, h->stream>>>(L[7], s.pd, s.hdr, rows, cols, pc.box);
  LAUNCH_CHECK();
  k_pp_box_cols<<<cb, PL_THREADS, 0, h->stream>>>(s.pd, a, s.hdr, rows, cols, pc.box / 2,
                                                   1.0 / ((double)pc.box * pc.box));
  LAUNCH_CHECK();
  PpGauss g;
  g.h = pc.gauss / 2;
  pp_gauss_coeffs(pc.gauss, g.c);
  k_pp_gauss<true><<<cb, PL_THREADS, 0, h->stream>>>(a, t, s.hdr, rows, cols, g);
  LAUNCH_CHECK();
  k_pp_gauss<false><<<cb, PL_THREADS, 0, h->stream>>>(t, L[8], s.hdr, rows, cols, g);
  LAUNCH_CHECK();
  // dilationInNonplanarRegions and addHeightOffset
  if (pc.fin.dil) {
    k_pp_morph<true><<<cb, PL_THREADS, 0, h->stream>>>(L[1], b, nullptr, s.hdr, rows, cols,
                                                        pp_ellipse(2 * q.nonplanar_horizontal_offset + 1));
    LAUNCH_CHECK();
  }
  k_pp_final<<<cb, PL_THREADS, 0, h->stream>>>(dst, b, L[9], s.hdr, n, pc.fin);
  LAUNCH_CHECK();
  return 0;
}

// ContourExtraction::extractPlanarRegions and addHeightOffset after segment_window (the window entry points with
// `window`, emap_plane_decomposition with `grid`), then, with post != nullptr, Postprocessing::postprocess's map passes
// (emap_planar_terrain, emap_plane_decomposition): see include/emap.h and DESIGN.md §4l.  Every check runs before
// anything is written or launched; the launches depend on the parameters and the grid sizes only.  fn names the entry
// point in the messages.
static int planar_regions(emap_handle* h, const char* fn, const double* window, const emap_grid* grid,
                          int32_t grid_on_device, const emap_plane_params& p,
                          const emap_region_params& rp, const emap_postprocess_params* post, float* layers_out,
                          int32_t out_is_device, int64_t out_floats, double* planes_out, int64_t planes_capacity,
                          const emap_region_out& o, int32_t* info) {
  if (rp.margin_size < 0 || rp.margin_size > EMAP_REGION_MAX_MARGIN)
    return fail_in(h, fn, "margin_size must be in [0, EMAP_REGION_MAX_MARGIN]");
  if (!std::isfinite(rp.plane_height_offset)) return fail_in(h, fn, "plane_height_offset must be finite");
  if (o.regions_capacity > EMAP_REGION_MAX_ROWS || o.polygons_capacity > EMAP_REGION_MAX_ROWS ||
      o.vertices_capacity > EMAP_REGION_MAX_ROWS)
    return fail_in(h, fn, "a table capacity is above EMAP_REGION_MAX_ROWS");
  if (o.regions_capacity < 0 || o.polygons_capacity < 0 || o.vertices_capacity < 0 ||
      (o.regions_capacity && !o.regions) || (o.polygons_capacity && !o.polygons) ||
      (o.vertices_capacity && !o.vertices))
    return fail_in(h, fn, "a table capacity is negative or a table with a capacity is null");
  PlaneCall c;
  if (const char* e = grid ? grid_plane_check(*grid, grid_on_device, p, out_floats, planes_capacity, c)
                           : plane_check(h, window, p, out_floats, planes_capacity, c))
    return fail_in(h, fn, e);
  PostCall pc;
  if (post) {
    if (const char* e = post_params_error(*post, c.res, rp.plane_height_offset, pc)) return fail_in(h, fn, e);
    if (c.q[0] && out_floats < EMAP_TERRAIN_LAYERS * c.n)
      return fail_in(h, fn, "out_floats is below EMAP_TERRAIN_LAYERS * rows * cols");
    if (c.q[0] && (c.rows < pc.dil || c.cols < pc.dil))
      return fail_in(h, fn, grid ? "the resampled grid has fewer rows or columns than the smoothing's dilation kernel"
                                 : "the window has fewer rows or columns than the smoothing's dilation kernel");
    c.post = true;
  }
  if (!c.q[0]) {
    if (out_is_device) {
      k_rg_none<<<1, 1, 0, h->stream>>>(info, 0);
      LAUNCH_CHECK();
    } else {
      memset(info, 0, 8 * sizeof(int32_t));
      info[8] = 1;
    }
    return EMAP_OK;
  }
  const bool regions = c.rows >= 2 && c.cols >= 2;
  if (regions) c.tables = &o;
  int rc = segment_window(h, p, out_is_device, layers_out, planes_out, info, c);
  if (rc) return rc;
  PlaneScratch& s = c.s;
  RgOut ro;
  ro.regions = out_is_device ? o.regions : s.regions;
  ro.polys = out_is_device ? o.polygons : s.polys;
  ro.verts = out_is_device ? o.vertices : s.verts;
  ro.planes = c.dst_planes;
  ro.ox = c.ox;
  ro.oy = c.oy;
  ro.res3 = c.res / 3.0;
  ro.offset = rp.plane_height_offset;
  if (!regions) {
    k_rg_none<<<1, 1, 0, h->stream>>>(c.dst_info, 5);   // upSample needs 2 x 2 cells: no region
    LAUNCH_CHECK();
  } else {
    const RgGeom g = {c.rows, c.cols, 3 * c.rows - 2, 3 * c.cols - 2};
    const int64_t U = (int64_t)g.UR * g.UC, prow = c.plane_rows;
    RegionScratch r;
    if ((rc = grow(h, h->regions, carve_regions(U, prow, c.n, nullptr, r), 0, false))) return rc;
    carve_regions(U, prow, c.n, h->regions, r);
    const int ub = cdiv(U, PL_THREADS);
    CK(cudaMemsetAsync(r.hdr, 0, 8 * sizeof(int), h->stream));
    CK(cudaMemsetAsync(r.ok, 0, 6 * (prow + 1) * sizeof(int), h->stream));   // ok, lcnt, lreg, loff, roff, lfill
    k_rg_rows<<<cdiv(c.n, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.lab, s.rank, r.pr, (int)c.n);
    LAUNCH_CHECK();
    RgKernel kern[2];
    kern[0].r = 1 + rp.margin_size;
    for (int i = 0; i <= 2 * kern[0].r; i++) kern[0].half[i] = rg_ellipse_half(kern[0].r, i);
    kern[1].r = 1;
    kern[1].half[0] = 0; kern[1].half[1] = 1; kern[1].half[2] = 0;
    // pass 0: the margin erosion; pass 1: the cross erosion of the plane rows pass 0 left without a region
    for (int ph = 0; ph < 2; ph++) {
      k_rg_erode<<<ub, PL_THREADS, 0, h->stream>>>(r.pr, r.ok, r.mask, g, kern[ph], ph);
      LAUNCH_CHECK();
      k_rg_inset<<<ub, PL_THREADS, 0, h->stream>>>(r.mask, g, ph);
      LAUNCH_CHECK();
      const int bo = 1 << (2 * ph);
      int* par[2] = {r.pa, r.pb};
      for (int im = 0; im < 2; im++) {
        k_rg_uf_init<<<cdiv(U + 1, PL_THREADS), PL_THREADS, 0, h->stream>>>(par[im], (int)U);
        LAUNCH_CHECK();
        k_rg_uf_merge<<<ub, PL_THREADS, 0, h->stream>>>(r.mask, bo << im, par[im], g);
        LAUNCH_CHECK();
        k_pl_uf_flatten<<<cdiv(U + 1, PL_THREADS), PL_THREADS, 0, h->stream>>>(par[im], (int)U + 1);
        LAUNCH_CHECK();
      }
      k_rg_count<<<ub, PL_THREADS, 0, h->stream>>>(r.mask, r.pa, r.pb, r.cnt, g, ph);
      LAUNCH_CHECK();
      CK(cudaMemsetAsync(r.have, 0, U * sizeof(int), h->stream));
      k_rg_have<<<ub, PL_THREADS, 0, h->stream>>>(r.mask, r.pa, r.pb, r.cnt, r.have, g, ph);
      LAUNCH_CHECK();
      k_rg_keep<<<ub, PL_THREADS, 0, h->stream>>>(r.mask, r.pa, r.pb, r.cnt, r.have, r.pr, r.flag, r.ok, g, ph);
      LAUNCH_CHECK();
      if ((rc = scan_ranks(h, r.flag, r.rank, r.bsum, U, r.hdr + ph))) return rc;
      k_rg_append<<<ub, PL_THREADS, 0, h->stream>>>(r.mask, r.pa, r.pb, r.cnt, r.pr, r.flag, r.rank, r.hdr, r.khi,
                                                     r.klo, r.rn, r.rcode, r.lcnt, r.lreg, g, ph);
      LAUNCH_CHECK();
    }
    // the output order: per plane row offsets of polygons and regions, buckets, and per record its position, region
    // and inset; the arrays of the passes are reused for it (bucket: rank; sorted counts: flag; record, region,
    // inset: pa, pb, have; first vertices: cnt)
    if ((rc = scan_ranks(h, r.lcnt, r.loff, r.bsum, prow + 1, r.hdr + 2))) return rc;
    if ((rc = scan_ranks(h, r.lreg, r.roff, r.bsum, prow + 1, r.hdr + 3))) return rc;
    k_rg_bucket<<<ub, PL_THREADS, 0, h->stream>>>(r.khi, r.hdr, r.loff, r.lfill, r.rank, (int)U);
    LAUNCH_CHECK();
    CK(cudaMemsetAsync(r.flag, 0, U * sizeof(int), h->stream));
    k_rg_rank<<<ub, PL_THREADS, 0, h->stream>>>(r.khi, r.klo, r.rn, r.hdr, r.lcnt, r.loff, r.roff, r.rank, r.flag,
                                                 r.pa, r.pb, r.have, (int)U);
    LAUNCH_CHECK();
    if ((rc = scan_ranks(h, r.flag, r.cnt, r.bsum, U, r.hdr + 4))) return rc;
    k_rg_info<<<1, 1, 0, h->stream>>>(r.hdr, c.dst_info, o.regions_capacity, o.polygons_capacity, o.vertices_capacity);
    LAUNCH_CHECK();
    k_rg_write<<<ub, PL_THREADS, 0, h->stream>>>(r.mask, r.khi, r.klo, r.rcode, r.hdr, r.flag, r.pa, r.pb, r.have,
                                                  r.cnt, ro, g, (int)U);
    LAUNCH_CHECK();
  }
  if (post && (rc = postprocess_window(h, c, *post, pc, out_is_device ? layers_out : s.layers))) return rc;
  if (!out_is_device) {
    PlaneScratch t;
    if ((rc = plane_copy_back(h, c, layers_out, planes_out, info, 9, t))) return rc;
    if (regions && info[8]) {
      memcpy(o.regions, t.regions, sizeof(double) * RG_ROW * info[5]);
      memcpy(o.polygons, t.polys, sizeof(int32_t) * RG_POLY * info[6]);
      memcpy(o.vertices, t.verts, sizeof(double) * 2 * info[7]);
    }
  }
  return EMAP_OK;
}

int emap_extract_planar_regions(emap_handle* h, const double window[4], const emap_plane_params* plane_params,
                                const emap_region_params* region_params, float* layers_out, int32_t out_is_device,
                                int64_t out_floats, double* planes_out, int64_t planes_capacity,
                                const emap_region_out* regions_out, int32_t* info) {
  ENTER(h);
  NvtxRange nv("emap:extract_planar_regions");
  if (!window || !plane_params || !region_params || !layers_out || !planes_out || !regions_out || !info)
    return fail(h, EMAP_ERR_INVALID, "emap_extract_planar_regions: null argument");
  return planar_regions(h, "emap_extract_planar_regions", window, nullptr, 0, *plane_params, *region_params, nullptr,
                        layers_out, out_is_device, out_floats, planes_out, planes_capacity, *regions_out, info);
}

// Postprocessing::postprocess after extract_planar_regions' passes: see include/emap.h and DESIGN.md §4l.
int emap_planar_terrain(emap_handle* h, const double window[4], const emap_plane_params* plane_params,
                        const emap_region_params* region_params, const emap_postprocess_params* post_params,
                        float* layers_out, int32_t out_is_device, int64_t out_floats, double* planes_out,
                        int64_t planes_capacity, const emap_region_out* regions_out, int32_t* info) {
  ENTER(h);
  NvtxRange nv("emap:planar_terrain");
  if (!window || !plane_params || !region_params || !post_params || !layers_out || !planes_out || !regions_out || !info)
    return fail(h, EMAP_ERR_INVALID, "emap_planar_terrain: null argument");
  const emap_postprocess_params q = *post_params;
  return planar_regions(h, "emap_planar_terrain", window, nullptr, 0, *plane_params, *region_params, &q, layers_out,
                        out_is_device, out_floats, planes_out, planes_capacity, *regions_out, info);
}

// The resampled size and resolution emap_plane_decomposition runs at (rs_geometry): see include/emap.h.
int emap_plane_grid_geometry(int64_t rows, int64_t cols, double resolution, const emap_plane_params* params,
                             int64_t out_size[2], double* out_resolution) {
  if (!params || !out_size || !out_resolution || rows < 1 || cols < 1 ||
      !(std::isfinite(resolution) && resolution > 0.0) || std::isnan(params->resolution))
    return EMAP_ERR_INVALID;
  rs_geometry(rows, cols, resolution, params->resolution, out_size, out_resolution);
  return EMAP_OK;
}

// PlaneDecompositionPipeline::update's grid map part on a caller's grid: GridMapPreprocessing with its resampling, the
// segmentation, the regions and the post-processing (planar_regions), at the resampled size.  See include/emap.h.
int emap_plane_decomposition(emap_handle* h, const emap_grid* grid, int32_t grid_on_device,
                             const emap_plane_params* plane_params, const emap_region_params* region_params,
                             const emap_postprocess_params* post_params, float* layers_out, int32_t out_is_device,
                             int64_t out_floats, double* planes_out, int64_t planes_capacity,
                             const emap_region_out* regions_out, int32_t* info) {
  ENTER(h);
  NvtxRange nv("emap:plane_decomposition");
  if (!grid || !plane_params || !region_params || !post_params || !layers_out || !planes_out || !regions_out || !info)
    return fail(h, EMAP_ERR_INVALID, "emap_plane_decomposition: null argument");
  const emap_grid g = *grid;
  const emap_postprocess_params q = *post_params;
  return planar_regions(h, "emap_plane_decomposition", nullptr, &g, grid_on_device, *plane_params, *region_params, &q,
                        layers_out, out_is_device, out_floats, planes_out, planes_capacity, *regions_out, info);
}

// The node's publishAsPointCloud (elevation_mapping_ros.cpp:501-505): the points of the exported elevation (map_cloud).
int emap_get_map_points(emap_handle* h, float* xyz_host, int64_t* n_points) {
  ENTER(h);
  NvtxRange nv("emap:get_map_points");
  if (!n_points || *n_points < 0 || (*n_points > 0 && !xyz_host))
    return fail(h, EMAP_ERR_INVALID, "emap_get_map_points: null argument or negative capacity");
  return map_cloud<false>(h, n_points, xyz_host, nullptr, nullptr);
}

// The node's publishNormalAsArrow (elevation_mapping_ros.cpp:751-778): the arrows of the exported normals (map_cloud).
int emap_get_normal_arrows(emap_handle* h, int32_t* ids_host, double* segments_host, int64_t* n_arrows) {
  ENTER(h);
  NvtxRange nv("emap:get_normal_arrows");
  if (!n_arrows || *n_arrows < 0 || (*n_arrows > 0 && (!ids_host || !segments_host)))
    return fail(h, EMAP_ERR_INVALID, "emap_get_normal_arrows: null argument or negative capacity");
  return map_cloud<true>(h, n_arrows, nullptr, ids_host, segments_host);
}

int emap_layer_device_ptr(emap_handle* h, const char* name, void** ptr) {
  ENTER(h);
  if (!name || !ptr) return fail(h, EMAP_ERR_INVALID, "null argument");
  const size_t C = (size_t)h->dc.C;
  int li = layer_index(name);
  if (li >= 0) { *ptr = h->map + li * C; return EMAP_OK; }
  if (!strcmp(name, "elevation_map")) { *ptr = h->map; return EMAP_OK; }
  if (!strcmp(name, "normal_map") || !strcmp(name, "normal_x")) { *ptr = h->normal; return EMAP_OK; }
  if (!strcmp(name, "normal_y")) { *ptr = h->normal + C; return EMAP_OK; }
  if (!strcmp(name, "normal_z")) { *ptr = h->normal + 2 * C; return EMAP_OK; }
  if (!strcmp(name, "traversability_input")) { *ptr = h->trav_input; return EMAP_OK; }
  h->err = std::string("Layer ") + name + " is not in the map";
  return EMAP_ERR_NOLAYER;
}

int emap_exists_layer(const emap_handle* h, const char* name) {
  if (!h || !name) return 0;
  return layer_index(name) >= 0 ? 1 : 0;
}

// ---- layer filters on a caller's grid (emap_grid_filter, csrc/emap_filters.cuh) -------------------------------------

static_assert(EMAP_FILTER_MAX_KERNEL == PP_MAX_KERNEL, "the Gaussian's coefficients hold EMAP_FILTER_MAX_KERNEL taps");

// The Gaussian's kernel size: kernel_size, or for 0 cv::GaussianBlur's size from sigma on a float image,
// cvRound(sigma * 4 * 2 + 1) | 1 (cvRound rounds half to even); 0 when that is not in [1, EMAP_FILTER_MAX_KERNEL].
static int gauss_kernel_size(const emap_filter_op& f) {
  if (f.kernel_size != 0) return f.kernel_size;
  if (!(f.sigma > 0.0)) return 0;
  const double q = std::nearbyint(f.sigma * 4 * 2 + 1);
  return q <= EMAP_FILTER_MAX_KERNEL ? ((int)q | 1) : 0;
}

// Why f is rejected for a rows x cols grid (nullptr: accepted).
static const char* filter_error(const emap_filter_op& f, int64_t rows, int64_t cols) {
  const int k = f.kernel_size;
  const bool sized = f.op != EMAP_FILTER_MIN_VALUES && f.op != EMAP_FILTER_OUTLINE;
  if (f.op < EMAP_FILTER_MIN_VALUES || f.op > EMAP_FILTER_OUTLINE) return "unknown op";
  const bool from_sigma = f.op == EMAP_FILTER_GAUSSIAN_BLUR && k == 0;
  if (sized && !from_sigma && (k < 1 || k > EMAP_FILTER_MAX_KERNEL))
    return "kernel_size must be in [1, EMAP_FILTER_MAX_KERNEL]";
  if ((f.op == EMAP_FILTER_MEDIAN || f.op == EMAP_FILTER_BOX_BLUR) && f.number_of_repeats < 1)
    return "number_of_repeats must be >= 1";
  if (f.op == EMAP_FILTER_MEDIAN) {
    const int64_t last = (int64_t)k + (int64_t)f.delta_kernel_size * (f.number_of_repeats - 1);
    const int64_t top = last <= 5 ? 5 : EMAP_FILTER_MAX_KERNEL;
    if (!(k & 1) || (f.delta_kernel_size & 1) || last < 1 || last > top || (last <= 5 && k > 5))
      return "every median kernel must be odd, 1, 3 or 5 on the float path and at most EMAP_FILTER_MAX_KERNEL on the "
             "8-bit path";
  }
  if (f.op == EMAP_FILTER_GAUSSIAN_BLUR) {
    if (!std::isfinite(f.sigma)) return "sigma must be finite";
    if (!(gauss_kernel_size(f) & 1))
      return "the Gaussian's kernel_size must be odd, or 0 with a sigma above 0 that gives at most EMAP_FILTER_MAX_KERNEL";
  }
  if ((f.op == EMAP_FILTER_DILATE || f.op == EMAP_FILTER_ERODE) && (rows < k || cols < k))
    return "the grid has fewer rows or columns than kernel_size";
  if (f.op == EMAP_FILTER_OUTLINE && (rows < 3 || cols < 3)) return "outline needs at least 3 rows and 3 columns";
  return nullptr;
}

namespace {
// emap_grid_filter's scratch for n cells: the fill's parents and keys, header words (the Gaussian's flag, the 8-bit
// path's range), two float planes, the box's double row sums, two 8-bit images, and the host-bound output.
struct FilterScratch {
  int *parent, *hdr;
  unsigned* key;
  float* f[2];
  double* rs;
  uint8_t* u[2];
  float* out;
};

size_t carve_filter(int64_t n, bool host_out, void* base, FilterScratch& s) {
  Carver c{(uintptr_t)base};
  s.parent = c.take<int>(n); s.key = c.take<unsigned>(n); s.hdr = c.take<int>(8);
  s.f[0] = c.take<float>(n); s.f[1] = c.take<float>(n); s.rs = c.take<double>(n);
  s.u[0] = c.take<uint8_t>(n); s.u[1] = c.take<uint8_t>(n);
  s.out = c.take<float>(host_out ? n : 0);
  return c.bytes;
}
}  // namespace

// The passes of one accepted filter from `in` into `o` (include/emap.h lists them per op).
static int filter_passes(emap_handle* h, const emap_filter_op& f, const float* in, const float* mask, float* o,
                         int rows, int cols, FilterScratch& s) {
  const int n = rows * cols, cb = cdiv(n, GF_THREADS), k = f.kernel_size;
  switch (f.op) {
    case EMAP_FILTER_MIN_VALUES: {
      PlaneScratch p{};
      p.parent = s.parent; p.key = s.key;
      k_pl_fill_init<<<cb, PL_THREADS, 0, h->stream>>>(in, s.parent, s.key, s.hdr, n);
      LAUNCH_CHECK();
      if (int rc = plane_components(h, p, rows, cols, 0)) return rc;
      k_pl_fill_min<<<cb, PL_THREADS, 0, h->stream>>>(in, s.parent, s.key, rows, cols);
      LAUNCH_CHECK();
      k_pl_fill_write<<<cb, PL_THREADS, 0, h->stream>>>(in, s.parent, s.key, o, n);
      LAUNCH_CHECK();
      return 0;
    }
    case EMAP_FILTER_MEDIAN: {
      const int R = f.number_of_repeats, d = f.delta_kernel_size;
      if (k + d * (R - 1) <= 5) {
        const float* src = in;
        for (int r = 0; r < R; r++) {
          float* dst = r == R - 1 ? o : s.f[r & 1];
          const int kr = k + d * r;
          if (kr == 1) CK(cudaMemcpyAsync(dst, src, sizeof(float) * n, cudaMemcpyDeviceToDevice, h->stream));
          else {
            (kr == 3 ? k_pl_median<3, true> : k_pl_median<5, true>)<<<cb, PL_THREADS, 0, h->stream>>>(src, dst, rows,
                                                                                                    cols);
            LAUNCH_CHECK();
          }
          src = dst;
        }
        return 0;
      }
      unsigned* w = (unsigned*)s.hdr;
      CK(cudaMemsetAsync(w, 0, 3 * sizeof(unsigned), h->stream));
      k_gf_range<<<cb, GF_THREADS, 0, h->stream>>>(in, w, n);
      LAUNCH_CHECK();
      k_gf_quantise<<<cb, GF_THREADS, 0, h->stream>>>(in, w, s.u[0], n);
      LAUNCH_CHECK();
      int cur = 0;
      for (int r = 0; r < R; r++) {
        const int kr = k + d * r;
        if (kr == 1) continue;
        k_gf_median_u8<<<dim3(cdiv(cols, GF_MED_COLS), cdiv(rows, GF_MED_ROWS)), GF_MED_COLS, 0, h->stream>>>(
            s.u[cur], s.u[cur ^ 1], rows, cols, kr);
        LAUNCH_CHECK();
        cur ^= 1;
      }
      k_gf_dequantise<<<cb, GF_THREADS, 0, h->stream>>>(s.u[cur], w, o, n);
      LAUNCH_CHECK();
      return 0;
    }
    case EMAP_FILTER_BOX_BLUR: {
      const float* src = in;
      if (k <= 5) CK(cudaMemsetAsync(s.hdr, 0xff, sizeof(int), h->stream));     // k_pp_box_rows runs where hdr[0] != 0
      for (int r = 0; r < f.number_of_repeats; r++) {
        float* dst = r == f.number_of_repeats - 1 ? o : s.f[r & 1];
        if (k <= 5) k_pp_box_rows<true><<<cb, PL_THREADS, 0, h->stream>>>(src, s.rs, s.hdr, rows, cols, k);
        else k_gf_box_rows<<<cdiv(rows, 128), 128, 0, h->stream>>>(src, s.rs, rows, cols, k);
        LAUNCH_CHECK();
        k_gf_box_cols<<<cdiv(cols, 128), 128, 0, h->stream>>>(s.rs, dst, rows, cols, k, 1.0 / ((double)k * k));
        LAUNCH_CHECK();
        src = dst;
      }
      return 0;
    }
    case EMAP_FILTER_GAUSSIAN_BLUR: {
      const int kg = gauss_kernel_size(f);
      PpGauss g;
      g.h = kg / 2;
      pp_gauss_coeffs(kg, g.c, f.sigma);
      CK(cudaMemsetAsync(s.hdr, 0xff, sizeof(int), h->stream));     // k_pp_gauss runs where hdr[0] != 0
      k_pp_gauss<true, true><<<cb, PL_THREADS, 0, h->stream>>>(in, s.f[0], s.hdr, rows, cols, g);
      LAUNCH_CHECK();
      k_pp_gauss<false, true><<<cb, PL_THREADS, 0, h->stream>>>(s.f[0], o, s.hdr, rows, cols, g);
      LAUNCH_CHECK();
      return 0;
    }
    case EMAP_FILTER_DILATE:
    case EMAP_FILTER_ERODE: {
      const bool mx = f.op == EMAP_FILTER_DILATE;
      (mx ? k_gf_morph_cols<true> : k_gf_morph_cols<false>)<<<cb, GF_THREADS, 0, h->stream>>>(in, mask, s.f[0], rows,
                                                                                               cols, k);
      LAUNCH_CHECK();
      (mx ? k_gf_morph_rows<true> : k_gf_morph_rows<false>)<<<cb, GF_THREADS, 0, h->stream>>>(
          in, mask, s.f[0], o, rows, cols, k, f.inpaint != 0);
      LAUNCH_CHECK();
      return 0;
    }
    default:
      k_gf_outline<<<cb, GF_THREADS, 0, h->stream>>>(in, o, rows, cols);
      LAUNCH_CHECK();
      return 0;
  }
}

// grid_map_filters_rsl's layer filters on a caller's grid (include/emap.h).  Every check runs before anything is
// written or launched.
int emap_grid_filter(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, const emap_filter_op* f,
                     const float* mask, float* out, int32_t out_is_device) {
  ENTER(h);
  const char* e = !grid || !f || !out ? "null argument"
                                      : gl_check_grid(grid->data, grid->rows, grid->cols, grid->position,
                                                      grid->resolution, 1);
  if (!e) e = filter_error(*f, grid->rows, grid->cols);
  if (e) return fail_in(h, "emap_grid_filter", e);
  NvtxRange nv("emap:grid_filter");
  const emap_filter_op op = *f;
  const int rows = (int)grid->rows, cols = (int)grid->cols;
  const int64_t n = (int64_t)rows * cols;
  const size_t bytes = sizeof(float) * n;
  FilterScratch s;
  if (int rc = grow(h, h->filters.block, carve_filter(n, !out_is_device, nullptr, s), 0, false)) return rc;
  carve_filter(n, !out_is_device, h->filters.block, s);
  const bool morph = op.op == EMAP_FILTER_DILATE || op.op == EMAP_FILTER_ERODE;
  const float* data = grid->data;
  const float* m = morph ? mask : nullptr;
  if (int rc = stage_inputs(h, h->filters.up, data, grid_on_device ? 0 : bytes, m, m && !grid_on_device ? bytes : 0))
    return rc;
  float* o = out_is_device ? out : s.out;
  if (int rc = filter_passes(h, op, data, m, o, rows, cols, s)) return rc;
  if (!out_is_device) {
    if (int rc = read_back(h, h->filters, o, bytes)) return rc;
    memcpy(out, h->filters.down, bytes);
  }
  return EMAP_OK;
}

}  // extern "C"
