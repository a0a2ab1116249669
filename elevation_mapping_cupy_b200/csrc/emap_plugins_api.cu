// emap_plugins_api.cu -- the plugin calls of the C ABI (include/emap.h): min / max filter, erode, robot-centric
// elevation, smooth, inpainting and its statistics, semantic filter and traversability, PCA, camera image fusion and
// map initialisation.
#include "emap_grid.cuh"
#include "emap_handle.cuh"
#include "emap_plugins.cuh"
#include "emap_inpaint.cuh"
#include "emap_semantic_plugins.cuh"
#include "emap_image.cuh"
#include "emap_initialize.cuh"

namespace {

// The inpainting scratch of an H x W image (a W x W map), one block; N = (H + 2) * (W + 2) padded pixels.
struct InpaintScratch {
  InpaintView v;
  int* heap[2];
  int* children;
  InpaintCtl* ctl;
  size_t bytes;
};

InpaintScratch inpaint_scratch(int H, int W, void* base) {
  const size_t N = (size_t)(H + 2) * (W + 2);
  Carver b{(uintptr_t)base};
  InpaintScratch s;
  s.v.rows = H + 2;
  s.v.cols = W + 2;
  s.v.f = b.take<uint8_t>(N); s.v.ck = b.take<uint8_t>(N); s.v.vc[0] = b.take<uint8_t>(N); s.v.vc[1] = b.take<uint8_t>(N);
  s.v.img = b.take<uint8_t>((size_t)H * W);
  s.v.T = b.take<float>(N); s.v.Tc[0] = b.take<float>(N); s.v.Tc[1] = b.take<float>(N);
  s.v.ord = b.take<uint32_t>(N);
  s.heap[0] = b.take<int>(N); s.heap[1] = b.take<int>(N); s.children = b.take<int>(N);
  s.ctl = b.take<InpaintCtl>(1);
  s.v.em = b.take<uint32_t>(N);
  s.bytes = b.bytes;
  return s;
}
InpaintScratch inpaint_scratch(int W, void* base) { return inpaint_scratch(W, W, base); }

// The fast-marching replay of an H x W image whose state k_ip_image_init / k_ip_grid_init and the control block's
// zeroing have queued: band, band flags and the cooperative march with METHOD's estimate, one CTA per SM.
template <int METHOD>
int inpaint_march(emap_handle* h, InpaintScratch& s) {
  int nb = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_ip_march<METHOD>, IP_MARCH_THREADS, 0));
  if (nb < 1) return fail(h, EMAP_ERR_CUDA, "inpainting: the cooperative kernel does not fit on an SM");
  const int nbN = cdiv((i64)s.v.rows * s.v.cols, 256);
  k_ip_band<<<nbN, 256, 0, h->stream>>>(s.v, s.heap[0], s.ctl); LAUNCH_CHECK();
  k_ip_band_flag<<<nbN, 256, 0, h->stream>>>(s.v, (const int*)s.heap[0], s.ctl); LAUNCH_CHECK();
  int cap = 4096;
  void* args[] = {(void*)&s.v, (void*)&s.heap[0], (void*)&s.heap[1], (void*)&s.children, (void*)&s.ctl, (void*)&cap};
  CK(cudaLaunchCooperativeKernel((const void*)k_ip_march<METHOD>, dim3(h->n_sm), dim3(IP_MARCH_THREADS), args, 0, h->stream));
  h->launches++;
  return 0;
}

// cv::inpaint's radius (cvRound, half to even, then at least 1) is 1: the one radius provided
bool inpaint_radius_ok(double r) { return std::isfinite(r) && std::nearbyint(r) <= 1.0; }

// The block of the image calls, carved for H x W with `out_bytes` of host-bound output behind the scratch (at s.bytes),
// zeroed when it grows (see emap_inpaint), its control block zeroed.
int image_scratch(emap_handle* h, int H, int W, size_t out_bytes, InpaintScratch& s) {
  if (int rc = grow(h, h->inpaint_image.block, inpaint_scratch(H, W, nullptr).bytes + out_bytes, 0, true)) return rc;
  s = inpaint_scratch(H, W, h->inpaint_image.block);
  CK(cudaMemsetAsync(s.ctl, 0, sizeof(InpaintCtl), h->stream));
  return 0;
}

int alloc_plugin_scratch(emap_handle* h) {
  for (int i = 0; i < 4; i++) {
    int rc = grow(h, h->plugin.plane[i], h->dc.C, 0, false);
    if (rc) return rc;
  }
  return 0;
}

// emap_min_filter / emap_max_filter: `iteration_n` Jacobi passes ping-ponging between two plane pairs, then the select
template <bool MAX>
int minmax_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                  int32_t* iterations_run) {
  if (!elevation || !is_valid || !out || k < 0 || k > 16 || iteration_n < 1)
    return fail(h, EMAP_ERR_INVALID, "emap_min_filter: bad argument");
  int rc;
  if ((rc = alloc_plugin_scratch(h)) || (rc = grow(h, h->plugin.cnt, (size_t)iteration_n + 1, 0, false))) return rc;
  const size_t B = sizeof(float) * (size_t)h->dc.C;
  float *hA = h->plugin.plane[0], *mA = h->plugin.plane[1], *hB = h->plugin.plane[2], *mB = h->plugin.plane[3];
  CK(cudaMemsetAsync(h->plugin.cnt, 0, sizeof(int) * (iteration_n + 1), h->stream));
  CK(cudaMemcpyAsync(hA, elevation, B, cudaMemcpyDeviceToDevice, h->stream));      // min_filter.py:105-106
  CK(cudaMemcpyAsync(mA, is_valid, B, cudaMemcpyDeviceToDevice, h->stream));
  for (int it = 0; it < iteration_n; it++) {
    const bool even = (it & 1) == 0;
    PER_CELL(k_fill_filter_iter<MAX>, h->dc, k, is_valid, even ? hA : hB, even ? mA : mB, even ? hB : hA, even ? mB : mA,
             h->plugin.cnt, it);
  }
  PER_CELL(k_min_filter_final, h->dc, hA, mA, hB, mB, h->plugin.cnt, iteration_n, out, h->plugin.cnt + iteration_n);
  if (iterations_run) {
    CK(cudaMemcpyAsync(iterations_run, h->plugin.cnt + iteration_n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}
// ---- features_pca ------------------------------------------------------------------------------
struct PcaScratch {
  PcaResult* res;
  double* part;                    // pca_entries(PCA_MAX_F) per k_pca_stats CTA
  double* proj;                    // 3 planes of C projections
};

int pca_stats_grid(emap_handle* h) { return std::min(cdiv(h->dc.C, 32), 2 * h->n_sm); }   // 32 <= tile cells

size_t carve_pca(emap_handle* h, void* base, PcaScratch& s) {
  Carver b{(uintptr_t)base};
  s.res = b.take<PcaResult>(1);
  s.part = b.take<double>((size_t)pca_stats_grid(h) * PCA_MAX_ENTRIES);
  s.proj = b.take<double>(3 * (size_t)h->dc.C);
  return b.bytes;
}

// the planes of a semantic plugin call: a non-null host array of n non-null device pointers
bool planes_ok(int32_t n, const float* const* planes) {
  if (n > 0 && !planes) return false;
  for (int l = 0; l < n; l++) if (!planes[l]) return false;
  return true;
}

// EM.py:913-922 after the interpolation: `iterations` Jacobi passes of the initialiser dilation, then
// upper_bound <- elevation on valid cells
int initialize_finish(emap_handle* h, int32_t dilation_size, int32_t iterations) {
  if (dilation_size < 0 || dilation_size > 64 || iterations < 0 || iterations > 16)
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map_finish: 0 <= dilation_size <= 64, 0 <= iterations <= 16");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  const size_t B = sizeof(float) * (size_t)h->dc.C;
  const int passes = dilation_size > 0 ? iterations : 0;
  for (int it = 0; it < std::max(passes, 1); it++) {
    CK(cudaMemcpyAsync(h->plugin.plane[0], h->map, B, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaMemcpyAsync(h->plugin.plane[1], h->map + 2 * (size_t)h->dc.C, B, cudaMemcpyDeviceToDevice, h->stream));
    PER_CELL(k_init_dilate, h->dc, h->plugin.plane[0], h->plugin.plane[1], h->map, passes ? dilation_size : 0, it == std::max(passes, 1) - 1);
  }
  return EMAP_OK;
}

}  // namespace

extern "C" {

// EM.py:913-922: the device half of initialize_map, after the caller wrote the interpolated planes (emap_set_state):
// `iterations` Jacobi passes of the initialiser dilation, then upper_bound <- elevation on valid cells.
int emap_initialize_map_finish(emap_handle* h, int32_t dilation_size, int32_t iterations) {
  ENTER(h);
  return initialize_finish(h, dilation_size, iterations);
}

// EM.py:899-922 + map_initializer.py:25-62 on the device (include/emap.h, csrc/emap_initialize.cuh): clear, snap, the
// host part (triangulation, gradients, coefficients, tile lists), one upload, one interpolation kernel, then the
// dilation passes and the upper-bound fill of emap_initialize_map_finish.
int emap_initialize_map(emap_handle* h, const float* xyz_host, int32_t n_points, int32_t method,
                        const int32_t* triangles_host, int32_t n_triangles, const double* gradients_host,
                        double initialized_variance, int32_t dilation_size_initialize) {
  ENTER(h);
  NvtxRange nv("emap:initialize_map");
  int rc = clear_map(h);                 // EM.py:906: every failure below leaves the map cleared
  if (rc) return rc;
  if (!xyz_host) return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: null points");
  if (n_points <= 3) return fail(h, EMAP_ERR_INVALID, "Initialization points must be more than 3.");
  if (n_points > EMAP_INIT_MAX_POINTS)
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: more than EMAP_INIT_MAX_POINTS points");
  if (method < 0 || method > 2) return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: method must be 0 (nearest), 1 (linear) or 2 (cubic)");
  if (triangles_host && (n_triangles < 1 || n_triangles > 2 * EMAP_INIT_MAX_POINTS))
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: 1 to 2 * EMAP_INIT_MAX_POINTS triangles required");
  if (dilation_size_initialize < 0 || dilation_size_initialize > 64 || !std::isfinite(initialized_variance))
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: 0 <= dilation_size_initialize <= 64 and a finite variance required");
  // transform_to_map_index as elevation_mapping.py applies it, in fp32: ((xy - center) / res + W / 2), truncated
  const int W = h->dc.W, n = n_points;
  const float res_f = (float)h->cfg.resolution, half_f = (float)(0.5 * W);
  std::vector<long long> xy(2 * (size_t)n);
  std::vector<double> z(n);
  bool narrow = true;
  for (int i = 0; i < n; i++) {
    const float* q = xyz_host + 3 * (size_t)i;
    if (!std::isfinite(q[0]) || !std::isfinite(q[1]) || !std::isfinite(q[2]))
      return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: non-finite point");
    for (int d = 0; d < 2; d++) {
      const float v = (q[d] - h->center[d]) / res_f;
      const float c = v + half_f;
      if (!(c >= -2147483648.f && c < 2147483648.f))
        return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: a point's cell index is outside the int32 range");
      xy[2 * i + d] = (long long)(int32_t)c;
      narrow &= std::llabs(xy[2 * i + d]) <= INIT_NARROW;
    }
    z[i] = (double)(float)(q[2] - h->center[2]);
  }
  InitArgs a;
  memset(&a, 0, sizeof(a));
  a.W = W; a.C = h->dc.C; a.tiles_x = (W + INIT_TILE - 1) / INIT_TILE;
  a.var = (float)initialized_variance;
  // the upload: one block, 256-byte aligned arrays, the same layout in pinned and in device memory
  std::vector<int> tri, nb, off, list;
  std::vector<double> grad, coef;
  Carver up{0};           // base 0: take() returns byte offsets
  size_t o_pxy = 0, o_pz = 0, o_txy = 0, o_coef = 0, o_off = 0, o_list = 0;
  if (method == 0) {
    a.n = n;
    o_pxy = (size_t)up.take<int2>(n);
    o_pz = (size_t)up.take<float>(n);
  } else {
    if (triangles_host) {
      tri.assign(triangles_host, triangles_host + 3 * (size_t)n_triangles);
      for (int t = 0; t < n_triangles; t++) {
        int* v = &tri[3 * (size_t)t];
        if (v[0] < 0 || v[0] >= n || v[1] < 0 || v[1] >= n || v[2] < 0 || v[2] >= n)
          return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: triangle index outside [0, n_points)");
        const int o = init_host::orient_sign(&xy[2 * (size_t)v[0]], &xy[2 * (size_t)v[1]], &xy[2 * (size_t)v[2]]);
        if (o == 0) return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: a triangle of zero area");
        if (o < 0) std::swap(v[1], v[2]);
      }
    } else if (!init_host::delaunay(xy, tri)) {
      return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: the points are collinear (no triangulation)");
    }
    const int T = (int)(tri.size() / 3);
    a.n = T;
    if (method == 2) {
      init_host::neighbours(tri, nb);
      if (!gradients_host) init_host::estimate_gradients(xy, z, tri, grad);
      coef.resize((size_t)INIT_CT * T);
      init_host::ct_coefficients(xy, z, gradients_host ? gradients_host : grad.data(), tri, nb, coef.data());
    } else {
      coef.resize(3 * (size_t)T);
      for (size_t k = 0; k < coef.size(); k++) coef[k] = z[tri[k]];
    }
    init_host::bin_tiles(W, xy, tri, off, list);
    o_txy = (size_t)up.take<int>(6 * (size_t)T);
    o_coef = (size_t)up.take<double>(coef.size());
    o_off = (size_t)up.take<int>(off.size());
    o_list = (size_t)up.take<int>(std::max<size_t>(list.size(), 1));
  }
  if ((rc = h->init_up.room(h, up.bytes))) return rc;
  char* hb = h->init_up.host;
  char* db = h->init_up.dev;
  if (method == 0) {
    int2* pxy = (int2*)(hb + o_pxy);
    float* pz = (float*)(hb + o_pz);
    for (int i = 0; i < n; i++) { pxy[i] = make_int2((int)xy[2 * i], (int)xy[2 * i + 1]); pz[i] = (float)z[i]; }
    a.pxy = (const int2*)(db + o_pxy); a.pz = (const float*)(db + o_pz);
  } else {
    int* txy = (int*)(hb + o_txy);
    for (size_t k = 0; k < tri.size(); k++) { txy[2 * k] = (int)xy[2 * (size_t)tri[k]]; txy[2 * k + 1] = (int)xy[2 * (size_t)tri[k] + 1]; }
    memcpy(hb + o_coef, coef.data(), sizeof(double) * coef.size());
    memcpy(hb + o_off, off.data(), sizeof(int) * off.size());
    if (!list.empty()) memcpy(hb + o_list, list.data(), sizeof(int) * list.size());
    a.txy = (const int*)(db + o_txy); a.coef = (const double*)(db + o_coef);
    a.tile_off = (const int*)(db + o_off); a.tile_tri = (const int*)(db + o_list);
  }
  if ((rc = h->init_up.send(h, up.bytes))) return rc;
  const int grid = a.tiles_x * a.tiles_x;
  if (method == 0) {
    if (narrow) k_init_nearest<long long><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
    else k_init_nearest<__int128><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
  } else if (method == 1) {
    if (narrow) k_init_interp<long long, false><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
    else k_init_interp<__int128, false><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
  } else {
    if (narrow) k_init_interp<long long, true><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
    else k_init_interp<__int128, true><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
  }
  LAUNCH_CHECK();
  return initialize_finish(h, dilation_size_initialize, 2);
}
int emap_min_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                    int32_t* iterations_run) {
  ENTER(h);
  return minmax_filter<false>(h, elevation, is_valid, out, k, iteration_n, iterations_run);
}

int emap_max_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                    int32_t* iterations_run) {
  ENTER(h);
  return minmax_filter<true>(h, elevation, is_valid, out, k, iteration_n, iterations_run);
}

int emap_erode(emap_handle* h, const float* layer, float* out, int32_t kernel_size, int32_t iterations, int32_t reverse) {
  ENTER(h);
  if (!layer || !out || kernel_size < 1 || kernel_size > 31 || iterations < 1 || iterations > 64)
    return fail(h, EMAP_ERR_INVALID, "emap_erode: bad argument");
  int rc;
  if ((rc = alloc_plugin_scratch(h)) || (rc = grow(h, h->plugin.cnt, 2, 30, false))) return rc;
  u32* const mm = (u32*)(int*)h->plugin.cnt;      // min / max of the layer
  const u32 init[2] = {0xffffffffu, 0u};
  CK(cudaMemcpyAsync(mm, init, sizeof(init), cudaMemcpyHostToDevice, h->stream));
  PER_CELL(k_layer_minmax, h->dc, layer, reverse, mm);
  const int ks = kernel_size + (iterations - 1) * (kernel_size - 1), anchor = (kernel_size / 2) * iterations;
  const float* src = layer;
  if (layer == out) {        // in-place call: erode from a copy
    CK(cudaMemcpyAsync(h->plugin.plane[0], layer, sizeof(float) * (size_t)h->dc.C, cudaMemcpyDeviceToDevice, h->stream));
    src = h->plugin.plane[0];
  }
  PER_CELL(k_erode, h->dc, src, out, ks, anchor, reverse, (const u32*)mm);
  return EMAP_OK;
}

int emap_robot_centric_elevation(emap_handle* h, const float* elevation, const float* is_valid, const float R[9], float* out,
                                 double resolution, double threshold, int32_t use_threshold) {
  ENTER(h);
  if (!elevation || !is_valid || !R || !out) return fail(h, EMAP_ERR_INVALID, "null argument");
  PER_CELL(k_robot_centric, h->dc, elevation, is_valid, out, R[6], R[7], R[8], resolution, threshold, use_threshold);
  return EMAP_OK;
}

int emap_smooth_filter(emap_handle* h, const float* in, float* out) {
  ENTER(h);
  if (!in || !out) return fail(h, EMAP_ERR_INVALID, "null argument");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  PER_CELL(k_box3, h->dc, in, h->plugin.plane[0], 0);
  PER_CELL(k_box3, h->dc, h->plugin.plane[0], h->plugin.plane[1], 1);
  PER_CELL(k_box3, h->dc, h->plugin.plane[1], h->plugin.plane[0], 0);
  PER_CELL(k_box3, h->dc, h->plugin.plane[0], out, 1);
  return EMAP_OK;
}

// plugins/inpainting.py:53-63: 8-bit normalisation, cv.inpaint(h, mask, 1, INPAINT_TELEA), de-normalisation -- OpenCV's
// fast-marching fill replayed on the device in parallel (emap_inpaint.cuh), bit-identical to cv2's result.
int emap_inpaint(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t method) {
  ENTER(h);
  NvtxRange nv("emap:inpaint");
  if (!elevation || !is_valid || !out) return fail(h, EMAP_ERR_INVALID, "emap_inpaint: null argument");
  if (method != 0) return fail(h, EMAP_ERR_INVALID, "emap_inpaint: only method 0 (telea) is implemented; 'ns' (Navier-Stokes) is not");
  const int W = h->dc.W;
  const size_t N = (size_t)(W + 2) * (W + 2), C = (size_t)W * W;
  // zero-filled once: the march loads a pixel's child fields (ck, Tc, vc) speculatively, before it knows the pixel is a
  // child of the running round; the values of non-children are never used, but they should not be uninitialised memory
  int rc = grow(h, h->inpaint.block, inpaint_scratch(W, nullptr).bytes, 0, true);
  if (rc) return rc;
  if (!h->inpaint.grid) {
    int nb = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_ip_march<IP_TELEA>, IP_MARCH_THREADS, 0));
    if (nb < 1) return fail(h, EMAP_ERR_CUDA, "emap_inpaint: the cooperative kernel does not fit on an SM");
    h->inpaint.grid = h->n_sm;          // one CTA per SM: the fronts are thin, and a grid barrier costs less with fewer CTAs
  }
  InpaintScratch s = inpaint_scratch(W, h->inpaint.block);
  InpaintView& v = s.v;
  InpaintCtl* ctl = s.ctl;
  InpaintCtl init;
  memset(&init, 0, sizeof(init));
  init.mm[0] = 0xffffffffu; init.mm[1] = 0u;
  CK(cudaMemcpyAsync(ctl, &init, sizeof(init), cudaMemcpyHostToDevice, h->stream));     // pageable: staged before return
  const int nbN = cdiv((i64)N, 256);
  PER_CELL(k_ip_minmax, (int)C, elevation, is_valid, ctl);
  k_ip_init<<<nbN, 256, 0, h->stream>>>(W, elevation, is_valid, v, (const InpaintCtl*)ctl); LAUNCH_CHECK();
  k_ip_band<<<nbN, 256, 0, h->stream>>>(v, s.heap[0], ctl); LAUNCH_CHECK();
  k_ip_band_flag<<<nbN, 256, 0, h->stream>>>(v, (const int*)s.heap[0], ctl); LAUNCH_CHECK();
  {
    int cap = 4096;
    void* args[] = {(void*)&v, (void*)&s.heap[0], (void*)&s.heap[1], (void*)&s.children, (void*)&ctl, (void*)&cap};
    CK(cudaLaunchCooperativeKernel((const void*)k_ip_march<IP_TELEA>, dim3(h->inpaint.grid), dim3(IP_MARCH_THREADS), args, 0, h->stream));
    h->launches++;
  }
  PER_CELL(k_ip_finish, (int)C, (const uint8_t*)v.img, elevation, out, (const InpaintCtl*)ctl);
  return EMAP_OK;
}

// cv2.inpaint for one 8-bit channel: Telea (the replay emap_inpaint runs) or Navier-Stokes, radius 1 (include/emap.h)
int emap_inpaint_image(emap_handle* h, const uint8_t* img, const uint8_t* mask, int64_t rows, int64_t cols,
                       double radius, int32_t method, uint8_t* out, int32_t on_device) {
  ENTER(h);
  const char* e = nullptr;
  if (!img || !mask || !out) e = "null argument";
  else if (method != 0 && method != 1) e = "method must be 0 (telea) or 1 (ns)";
  else if (rows < (method ? 1 : 2) || cols < (method ? 1 : 2) || rows > EMAP_INPAINT_MAX_SIDE || cols > EMAP_INPAINT_MAX_SIDE)
    e = method ? "rows and cols must be 1 .. EMAP_INPAINT_MAX_SIDE" : "rows and cols must be 2 .. EMAP_INPAINT_MAX_SIDE for telea";
  else if (!inpaint_radius_ok(radius)) e = "radius must be finite and round to at most 1 (only radius 1 is provided)";
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_inpaint_image: ") + e).c_str());
  NvtxRange nv("emap:inpaint_image");
  const int H = (int)rows, W = (int)cols;
  const size_t n = (size_t)H * W;
  InpaintScratch s;
  if (int rc = image_scratch(h, H, W, 0, s)) return rc;
  if (int rc = stage_inputs(h, h->inpaint_image.up, img, on_device ? 0 : n, mask, on_device ? 0 : n)) return rc;
  k_ip_image_init<<<cdiv((i64)s.v.rows * s.v.cols, 256), 256, 0, h->stream>>>(img, mask, s.v); LAUNCH_CHECK();
  if (int rc = method ? inpaint_march<IP_NS>(h, s) : inpaint_march<IP_TELEA>(h, s)) return rc;
  if (on_device) {
    CK(cudaMemcpyAsync(out, s.v.img, n, cudaMemcpyDeviceToDevice, h->stream));
  } else {
    if (int rc = read_back(h, h->inpaint_image, s.v.img, n)) return rc;
    memcpy(out, h->inpaint_image.down, n);
  }
  return EMAP_OK;
}

// grid_map_filters_rsl's inpainting::nonlinearInterpolation on a caller's grid (include/emap.h)
int emap_nonlinear_interpolation(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, double inpaint_radius,
                                 float* out, int32_t out_is_device) {
  ENTER(h);
  const char* e = !grid || !out ? "null argument" : gl_check_grid(grid->data, grid->rows, grid->cols, grid->position,
                                                                 grid->resolution, 1);
  if (!e && (grid->rows > EMAP_INPAINT_MAX_SIDE || grid->cols > EMAP_INPAINT_MAX_SIDE))
    e = "rows and cols must be at most EMAP_INPAINT_MAX_SIDE";
  if (!e && !inpaint_radius_ok(inpaint_radius / grid->resolution))
    e = "inpaint_radius / resolution must be finite and round to at most 1 (only radius 1 is provided)";
  if (e) return fail(h, EMAP_ERR_INVALID, (std::string("emap_nonlinear_interpolation: ") + e).c_str());
  NvtxRange nv("emap:nonlinear_interpolation");
  const int H = (int)grid->rows, W = (int)grid->cols;
  const size_t bytes = sizeof(float) * H * W;
  InpaintScratch s;
  if (int rc = image_scratch(h, H, W, out_is_device ? 0 : bytes, s)) return rc;
  const float* data = grid->data;
  if (int rc = stage_inputs(h, h->inpaint_image.up, data, grid_on_device ? 0 : bytes)) return rc;
  k_ip_finite_range<<<cdiv((i64)H * W, 256), 256, 0, h->stream>>>(H * W, data, s.ctl); LAUNCH_CHECK();
  k_ip_grid_init<<<cdiv((i64)s.v.rows * s.v.cols, 256), 256, 0, h->stream>>>(data, s.v, (const InpaintCtl*)s.ctl);
  LAUNCH_CHECK();
  if (int rc = inpaint_march<IP_NS>(h, s)) return rc;
  float* o = out_is_device ? out : (float*)(h->inpaint_image.block + s.bytes);
  k_ip_grid_out<<<cdiv((i64)H * W, 256), 256, 0, h->stream>>>(H * W, (const uint8_t*)s.v.img, data, o,
                                                              (const InpaintCtl*)s.ctl);
  LAUNCH_CHECK();
  if (!out_is_device) {
    if (int rc = read_back(h, h->inpaint_image, o, bytes)) return rc;
    memcpy(out, h->inpaint_image.down, bytes);
  }
  return EMAP_OK;
}

// plugins/semantic_filter.py:89-133: argmax over the planes, palette entry of the class id (bits)
int emap_semantic_filter(emap_handle* h, int32_t n_layers, const float* const* planes, float* out) {
  ENTER(h);
  if (!out || n_layers < 0 || n_layers > EMAP_SEMANTIC_FILTER_MAX_LAYERS || !planes_ok(n_layers, planes))
    return fail(h, EMAP_ERR_INVALID, "emap_semantic_filter: 0 to EMAP_SEMANTIC_FILTER_MAX_LAYERS non-null planes and a non-null output required");
  SemFilterArgs a;
  memset(&a, 0, sizeof(a));
  a.n = n_layers;
  for (int l = 0; l < n_layers; l++) a.plane[l] = planes[l];
  PER_CELL(k_semantic_filter, h->dc.C, a, (u32*)out);
  return EMAP_OK;
}

// plugins/semantic_traversability.py:59-83: per-layer threshold votes (fp64 comparisons), fp32(0.1) or 1
int emap_semantic_traversability(emap_handle* h, int32_t n_layers, const float* const* planes, const double* thresholds,
                                 const int32_t* is_traversability_type, float* out) {
  ENTER(h);
  if (!out || n_layers < 0 || n_layers > EMAP_SEMANTIC_TRAVERSABILITY_MAX_LAYERS || !planes_ok(n_layers, planes) ||
      (n_layers > 0 && (!thresholds || !is_traversability_type)))
    return fail(h, EMAP_ERR_INVALID, "emap_semantic_traversability: 0 to EMAP_SEMANTIC_TRAVERSABILITY_MAX_LAYERS non-null planes, "
                                     "thresholds, types and a non-null output required");
  SemTravArgs a;
  memset(&a, 0, sizeof(a));
  a.n = n_layers;
  for (int l = 0; l < n_layers; l++) {
    a.plane[l] = planes[l];
    a.thr[l] = thresholds[l];
    if (is_traversability_type[l]) a.is_trav[l >> 5] |= 1u << (l & 31);
  }
  PER_CELL(k_semantic_traversability, h->dc.C, a, out);
  return EMAP_OK;
}

// plugins/features_pca.py:44-96: exact 3-component PCA of the clipped features on the device, packed to colour bits.
// Four launches and one synchronisation, at the end, to read the NaN flag.
int emap_features_pca(emap_handle* h, int32_t n_features, const float* const* planes, float* out) {
  ENTER(h);
  NvtxRange nv("emap:features_pca");
  if (!out || n_features < 3 || n_features > EMAP_PCA_MAX_FEATURES || !planes_ok(n_features, planes))
    return fail(h, EMAP_ERR_INVALID, "emap_features_pca: 3 to EMAP_PCA_MAX_FEATURES non-null planes and a non-null output required");
  PcaScratch s;
  int rc = grow(h, h->pca_block, carve_pca(h, nullptr, s), 0, false);
  if (rc) return rc;
  carve_pca(h, h->pca_block, s);
  const int C = h->dc.C, F = n_features;
  PcaArgs a;
  memset(&a, 0, sizeof(a));
  a.F = F;
  for (int f = 0; f < F; f++) a.plane[f] = planes[f];
  const size_t eig_smem = sizeof(double) * 2 * F * (F + 1);
  CK(cudaFuncSetAttribute(k_pca_eigen, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eig_smem));
  CK(cudaMemsetAsync(&s.res->nan, 0, sizeof(int), h->stream));
  const int grid = pca_stats_grid(h);
  k_pca_stats<<<grid, PCA_THREADS, 0, h->stream>>>(C, a, s.part, s.res);
  LAUNCH_CHECK();
  k_pca_eigen<<<1, PCA_THREADS, eig_smem, h->stream>>>(C, F, grid, s.part, s.res);
  LAUNCH_CHECK();
  PER_CELL(k_pca_project, C, a, s.res, s.proj);
  PER_CELL(k_pca_pack, C, (const PcaResult*)s.res, (const double*)s.proj, (u32*)out);
  int nan = 0;
  CK(cudaMemcpyAsync(&nan, &s.res->nan, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (nan) return fail(h, EMAP_ERR_INVALID, "emap_features_pca: NaN in the input features");
  return EMAP_OK;
}

// EM.py:468-562 input_image + semantic_map.py:261-309 update_layers_image: the host part (image_camera) and one
// k_image_fuse launch.  A host image is copied into pinned staging and from there, once, to the device; a device image
// is read in place, with no host synchronisation.
int emap_input_image(emap_handle* h, int32_t n_planes, const float* image, int is_device_ptr, int32_t height, int32_t width,
                     const float K[9], const float* D, int32_t n_D, const char* distortion_model, const float R[9],
                     const float t[3], int32_t n_fused, const int32_t* plane, const int32_t* kind, const int32_t* layer,
                     float* semantic_map_device, int32_t n_layers) {
  ENTER(h);
  NvtxRange nv("emap:input_image");
  if (!image || !K || !R || !t || !distortion_model || (n_D > 0 && !D) || n_D < 0 ||
      (n_fused > 0 && (!plane || !kind || !layer || !semantic_map_device)))
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: null argument");
  if (n_planes < 1 || height < 1 || width < 1 || (int64_t)height * width > (1ll << 24))
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: n_planes >= 1 and 1 <= height * width <= 2^24 required");
  if (n_fused < 0 || n_fused > EMAP_IMAGE_MAX_CHANNELS)
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: 0 to EMAP_IMAGE_MAX_CHANNELS fused channels required");
  ImageArgs a;
  memset(&a, 0, sizeof(a));
  for (int k = 0; k < n_fused; k++) {
    if (kind[k] != EMAP_IMAGE_COLOR && kind[k] != EMAP_IMAGE_EXPONENTIAL)
      return fail(h, EMAP_ERR_INVALID, "emap_input_image: kind must be EMAP_IMAGE_COLOR or EMAP_IMAGE_EXPONENTIAL");
    if (plane[k] < 0 || plane[k] >= n_planes || (kind[k] == EMAP_IMAGE_COLOR && n_planes < 3))
      return fail(h, EMAP_ERR_INVALID, "emap_input_image: plane outside the image, or a colour channel with fewer than 3 planes");
    if (layer[k] < 0 || layer[k] >= n_layers)
      return fail(h, EMAP_ERR_INVALID, "emap_input_image: layer outside [0, n_layers)");
    a.plane[k] = plane[k];
    a.kind[k] = kind[k] == EMAP_IMAGE_COLOR ? IMG_COLOR : IMG_EXPONENTIAL;
    a.layer[k] = layer[k];
  }
  const int cam = image_camera(K, D, n_D, distortion_model, R, t, h->center, h->dc.W, h->cfg.resolution, &a.cam);
  if (cam == IMG_CAM_NONFINITE) return fail(h, EMAP_ERR_INVALID, "emap_input_image: non-finite K, R or t");
  if (cam == IMG_CAM_OUTSIDE)
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: camera cell cell_n / 2 + t / resolution outside [0, 2^24)");
  if (n_fused == 0) return EMAP_OK;       // the correspondence alone changes nothing
  const size_t plane_sz = (size_t)height * width, n_img = plane_sz * n_planes;
  const float* img = image;
  if (int rc = stage_inputs(h, h->img_up, img, is_device_ptr ? 0 : sizeof(float) * n_img)) return rc;
  for (int k = 0; k < 3; k++) a.center[k] = h->center[k];
  a.res = h->cfg.resolution;
  a.W = h->dc.W; a.C = h->dc.C;
  a.img_w = (float)width; a.img_h = (float)height;
  a.n_img = (long long)n_img; a.plane_sz = (long long)plane_sz;
  a.image = img; a.sem = semantic_map_device; a.n = n_fused;
  PER_CELL(k_image_fuse, a, (const float*)h->map);
  return EMAP_OK;
}

// rounds / Jacobi statistics of the last emap_inpaint call (diagnostics)
int emap_inpaint_stats(emap_handle* h, int32_t* rounds, int32_t* max_jacobi, int32_t* not_converged) {
  ENTER(h);
  if (!h->inpaint.block) return fail(h, EMAP_ERR_STATE, "emap_inpaint has not run");
  InpaintCtl c;
  CK(cudaMemcpyAsync(&c, inpaint_scratch(h->dc.W, h->inpaint.block).ctl, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (rounds) *rounds = c.rounds;
  if (max_jacobi) *max_jacobi = c.max_jacobi;
  if (not_converged) *not_converged = c.not_converged;
  return EMAP_OK;
}

}  // extern "C"
