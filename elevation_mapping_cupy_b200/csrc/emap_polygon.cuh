// emap_polygon.cuh -- the polygon safety check (sm_90a): EM.py:837-889 get_polygon_traversability, CK.py:509-654
// polygon_mask_kernel, traversability_polygon.py:10-58.  One call checks a batch of polygons; the single call is a batch
// of one that also writes the mask.
//
// k_polygon: one CTA per work item, a (polygon, tile) pair.  Tiles are PG_COLS columns by PG_ROWS rows of one fixed grid
// over the map; each polygon brings the tiles that meet its cell bounding box (CK.py:609-615), or every tile when the
// mask is written.  A CTA turns its polygon's vertices into cells (CK.py:580-603) once, keeps the edges that can touch
// its tile, and every cell runs the reference's integer inside test against those edges only.  The same pass reads
// is_valid and the checker plane and reduces the statistics of traversability_polygon.py:10-34 over the tile's share of
// the interior [1:-1, 1:-1] into one partial per item, plus the per-column extremes of the over-threshold cells.
// k_poly_poison: counts the interior cells whose NaN / inf reaches every polygon's sums through `untrav * mask` (NaN * 0,
// inf * 0), for the polygons whose tiles do not cover the interior.
// k_hull: one CTA per polygon sums its partials in a fixed order (the result does not depend on scheduling) and builds
// the convex hull of its over-threshold cells (traversability_polygon.py:46-53) from the column extremes.
#pragma once
#include <algorithm>
#include <cmath>

#include "emap_device.cuh"

#define PG_COLS 32               // columns per k_polygon tile (one warp wide: coalesced rows)
#define PG_ROWS 64               // rows per k_polygon tile
#define PG_THREADS 256
#define HULL_THREADS 1024
#define HULL_MAX_PTS 4096        // >= 2 * (W - 2) column extremes for W <= 2049
#define HULL_GROUP 8             // chunks merged per thread and level of k_hull's chain reduction

struct PolyPartial {             // one k_polygon work item's share of the interior
  double sum_masked, sum_valid;
  float max_masked;              // max of the non-NaN masked values (-inf if none)
  int nan_masked;                // a masked value was NaN (CuPy's max propagates it)
  int over;                      // cells with masked > 1 - safe_thresh
  int poison;                    // tile cells counted by k_poly_poison: untraversability (low 16 bits), is_valid (high)
};

struct PolyResult {              // what the host reads back
  double t;                      // Σmasked / Σmasked_valid (0 unless Σmasked_valid > 0), rounded to fp32 like CuPy's
  double sum_masked, sum_valid;
  float max_masked;              // NaN if any masked value was NaN
  int over;                      // count(over)
  int is_safe;                   // traversability_polygon.py:37-43 (the host adds the clipped-area rule, EM.py:884-886)
  int n_ring;                    // ring length including the closing vertex, 0 if the hull is a point, a line or empty
  int pad[2];
};
// the double2 rings are carved directly behind the results (one read-back copy): keep them 16-byte aligned
static_assert(sizeof(PolyResult) % 16 == 0, "PolyResult must keep the rings behind it 16-byte aligned");

struct PolyDesc {                // one polygon of a call, staged by the host
  int v0, n;                     // its clipped fp32 vertices xy[v0 .. v0 + n) (EM.py:847-851)
  float bbox[4];                 // min x, min y, max x, max y of the clipped vertices (EM.py:852-854)
  int item0;                     // its first work item, which is also the index of its first partial
  int tr0, tc0, n_tr, n_tc;      // its tiles: rows tr0 .. tr0 + n_tr - 1, columns tc0 .. tc0 + n_tc - 1 of the grid
  int col0, n_col;               // interior columns col0 .. col0 + n_col - 1 hold its column extremes ...
  int col_off;                   // ... at col_min / col_max + col_off (n_col = 0: no hull)
  int ring_off;                  // its ring (2 n_col + 1 vertices at most) at ring + ring_off
  int pad;
};
static_assert(sizeof(PolyDesc) % 16 == 0, "PolyDesc keeps the vertices behind it 8-byte aligned");

struct PolyArgs {
  const PolyDesc* poly;          // n_poly descriptors, ordered by item0
  PolyDesc one;                  // poly[0] of a call of one polygon (k_polygon<false> reads it from its parameters)
  int n_poly;
  const float2* xy;
  float cx, cy;                  // map centre, fp32 (EM.py:61)
  float thr_over, thr_max;       // fp32(1 - safe_thresh), fp32(1 - safe_min_thresh): CuPy compares in fp32
  int max_unsafe_n;
  const int* poison;             // k_poly_poison's two counts over the interior; NULL when every polygon covers it
};

// CK.py:580-603 get_x_idx / get_idx for one coordinate: the coordinate and the centre are CuPy float16, their difference
// is taken in float, divided by the float `resolution`, 0.5 * width is added in double and the sum truncated to int;
// clamp() goes through float16, which is exact for W - 1 <= 2048.  The host runs the same sequence to find a polygon's
// tiles; its truncation saturates like __double2int_rz (NaN gives 0).
__host__ __device__ __forceinline__ int poly_axis_cell(float v, float c, float res_f, int W) {
#ifdef __CUDA_ARCH__
  const float d = __fsub_rn(h16(v), h16(c));
  const int i = __double2int_rz((double)__fdiv_rn(d, res_f) + 0.5 * (double)W);
  return min(max(i, 0), W - 1);
#else
  const float d = __half2float(__float2half_rn(v)) - __half2float(__float2half_rn(c));
  const double q = (double)(d / res_f) + 0.5 * (double)W;
  const int i = q != q ? 0 : (q >= 2147483647.0 ? 2147483647 : (q <= -2147483648.0 ? (-2147483647 - 1) : (int)q));
  return i < 0 ? 0 : (i > W - 1 ? W - 1 : i);
#endif
}

// EM.py:847-854: each coordinate clipped to [center - map_length/2 + resolution, center + map_length/2 - resolution],
// fp32 throughout; map_length is the map's true length (W - 2) * resolution.  Writes the clipped vertices (unless out
// is NULL) and their bounding box.
inline void clip_polygon(int W, double resolution, const float* center, const float* xy, int n, float2* out,
                         float bbox[4]) {
  const float half = (float)(0.5 * (double)(W - 2) * resolution), res_f = (float)resolution;
  float lo[2], hi[2], bmin[2], bmax[2];
  for (int k = 0; k < 2; k++) {
    lo[k] = (center[k] - half) + res_f;
    hi[k] = (center[k] + half) - res_f;
  }
  for (int i = 0; i < n; i++) {
    float v[2];
    for (int k = 0; k < 2; k++) {
      v[k] = std::min(std::max(xy[2 * i + k], lo[k]), hi[k]);
      bmin[k] = i ? std::min(bmin[k], v[k]) : v[k];
      bmax[k] = i ? std::max(bmax[k], v[k]) : v[k];
    }
    if (out) out[i] = make_float2(v[0], v[1]);
  }
  bbox[0] = bmin[0]; bbox[1] = bmin[1]; bbox[2] = bmax[0]; bbox[3] = bmax[1];
}

// The tiles of k_polygon's grid that meet the polygon's cell bounding box d.bbox (CK.py:609-615, the cells k_polygon
// tests) and the interior columns of that box, the only ones that can hold its over-threshold cells.
inline void polygon_tiles(int W, double resolution, const float* center, PolyDesc& d) {
  const float rf = (float)resolution;
  const int bx0 = poly_axis_cell(d.bbox[0], center[0], rf, W), bx1 = poly_axis_cell(d.bbox[2], center[0], rf, W);
  const int by0 = poly_axis_cell(d.bbox[1], center[1], rf, W), by1 = poly_axis_cell(d.bbox[3], center[1], rf, W);
  d.tr0 = bx0 / PG_ROWS; d.n_tr = bx1 / PG_ROWS - d.tr0 + 1;
  d.tc0 = by0 / PG_COLS; d.n_tc = by1 / PG_COLS - d.tc0 + 1;
  d.col0 = std::max(by0, 1) - 1;
  d.n_col = std::max(0, std::min(by1, W - 2) - std::max(by0, 1) + 1);
}

// traversability_polygon.py:46-51 calculate_area on fp32 vertices: every operation in fp32, terms in order i = 0..n-1
// with p1 = polygon[i - 1], the absolute value at the end
inline float shoelace_f32(const float* xy, int n) {
  float area = 0.0f;
  for (int i = 0; i < n; i++) {
    const int j = i ? i - 1 : n - 1;
    const float a = xy[2 * j] * xy[2 * i + 1];
    const float b = xy[2 * j + 1] * xy[2 * i];
    area = area + (a - b) / 2.0f;
  }
  return std::fabs(area);
}

// CK.py:513-560: orientation of the ordered integer triplet (0 collinear, 1 clockwise, 2 counter-clockwise) and the
// collinear on-segment test
__device__ __forceinline__ int poly_orient(int px, int py, int qx, int qy, int rx, int ry) {
  const int v = (qy - py) * (rx - qx) - (qx - px) * (ry - qy);
  return v == 0 ? 0 : (v > 0 ? 1 : 2);
}
__device__ __forceinline__ bool poly_on_seg(int px, int py, int qx, int qy, int rx, int ry) {
  return qx <= max(px, rx) && qx >= min(px, rx) && qy <= max(py, ry) && qy >= min(py, ry);
}

// CK.py:616-648 for one cell (x, y) against one edge (ax, ay) - (bx, by): 2 = the cell lies on the edge (mask 1),
// 1 = the edge crosses the ray from the cell to (100000, y), 0 = neither.
__device__ __forceinline__ int poly_edge_test(int x, int y, int ax, int ay, int bx, int by) {
  const int ex = 100000;
  const int o1 = poly_orient(ax, ay, bx, by, x, y), o2 = poly_orient(ax, ay, bx, by, ex, y);
  const int o3 = poly_orient(x, y, ex, y, ax, ay), o4 = poly_orient(x, y, ex, y, bx, by);
  const bool hit = (o1 != o2 && o3 != o4) || (o1 == 0 && poly_on_seg(ax, ay, x, y, bx, by)) ||
                   (o2 == 0 && poly_on_seg(ax, ay, ex, y, bx, by)) || (o3 == 0 && poly_on_seg(x, y, ax, ay, ex, y)) ||
                   (o4 == 0 && poly_on_seg(x, y, bx, by, ex, y));
  if (!hit) return 0;
  if (poly_orient(ax, ay, x, y, bx, by) == 0) return poly_on_seg(ax, ay, x, y, bx, by) ? 2 : 0;
  return ((ay <= y && by > y) || (ay > y && by <= y)) ? 1 : 0;
}

// An interior cell whose untraversability (is_valid) is not finite makes Σmasked (Σmasked_valid) of every polygon NaN
// when the cell lies outside the polygon: traversability_polygon.py:16-18 multiplies the whole interior by the mask.
// Returns the cell's count for each sum, packed as k_poly_poison and PolyPartial::poison add them.
__device__ __forceinline__ int poly_poison(float v, float untrav) {
  return (isfinite(untrav) ? 0 : 1) | (isfinite(v) ? 0 : 1 << 16);
}

// the polygon of work item g: the last descriptor whose item0 <= g
__device__ __forceinline__ int poly_of_item(const PolyDesc* poly, int n_poly, int g) {
  int lo = 0, hi = n_poly - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (poly[mid].item0 <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// grid: one CTA per work item, PG_THREADS threads.  kBatch: several polygons, whose partials also count the poisoned
// cells for k_hull; without it the call is one polygon (the single call, whose tiles cover the map, needs no poison
// count and keeps the registers of a 5-CTA-per-SM kernel).  mask: NULL, or the (W, W) mask of a batch of one whose
// tiles cover the map.  col_min / col_max: NULL (no hulls), or per interior column of each polygon's window, the smallest / largest
// interior row of an over-threshold cell; INT_MAX / -1 on entry, k_hull resets them.
template <bool kBatch>
__global__ void __launch_bounds__(PG_THREADS, kBatch ? 4 : 5) k_polygon(int W, float res_f, PolyArgs a, const float* __restrict__ valid,
                                                        const float* __restrict__ checker, float* __restrict__ mask,
                                                        PolyPartial* __restrict__ part, int* __restrict__ col_min,
                                                        int* __restrict__ col_max) {
  __shared__ int4 s_edge[1024];
  __shared__ int s_ne, s_cmin[PG_COLS], s_cmax[PG_COLS];
  __shared__ double s_sm[PG_THREADS / 32], s_sv[PG_THREADS / 32];
  __shared__ float s_mx[PG_THREADS / 32];
  __shared__ int s_nan[PG_THREADS / 32], s_over[PG_THREADS / 32], s_poison[PG_THREADS / 32];
  const int tx = threadIdx.x % PG_COLS, ty = threadIdx.x / PG_COLS;
  const PolyDesc& d = kBatch ? a.poly[poly_of_item(a.poly, a.n_poly, blockIdx.x)] : a.one;
  const int item = blockIdx.x - d.item0;
  const int c0 = (d.tc0 + item % d.n_tc) * PG_COLS, r0 = (d.tr0 + item / d.n_tc) * PG_ROWS;
  const int c1 = min(c0 + PG_COLS, W) - 1;
  const float2* xy = a.xy + d.v0;
  const int n = d.n;
  if (threadIdx.x == 0) s_ne = 0;
  if (threadIdx.x < PG_COLS) { s_cmin[threadIdx.x] = INT_MAX; s_cmax[threadIdx.x] = -1; }
  // CK.py:609-615: the cell bounding box of the clipped polygon
  const int bx0 = poly_axis_cell(d.bbox[0], a.cx, res_f, W), by0 = poly_axis_cell(d.bbox[1], a.cy, res_f, W);
  const int bx1 = poly_axis_cell(d.bbox[2], a.cx, res_f, W), by1 = poly_axis_cell(d.bbox[3], a.cy, res_f, W);
  const bool tile_in_box = !(r0 + PG_ROWS - 1 < bx0 || r0 > bx1 || c1 < by0 || c0 > by1);
  __syncthreads();
  // An edge matters to a cell (x, y) only if its column range contains y (the on-edge and the crossing tests both need
  // that) and it reaches row x or beyond (the ray runs toward +x).  Order does not matter: the count's parity and "on an
  // edge" are all the cell needs.
  if (tile_in_box) {
    for (int j = threadIdx.x; j < n; j += PG_THREADS) {
      const float2 p = xy[j], q = xy[j + 1 == n ? 0 : j + 1];
      const int ax = poly_axis_cell(p.x, a.cx, res_f, W), ay = poly_axis_cell(p.y, a.cy, res_f, W);
      const int bx = poly_axis_cell(q.x, a.cx, res_f, W), by = poly_axis_cell(q.y, a.cy, res_f, W);
      if (max(ay, by) < c0 || min(ay, by) > c1 || max(ax, bx) < r0) continue;
      s_edge[atomicAdd(&s_ne, 1)] = make_int4(ax, ay, bx, by);
    }
  }
  __syncthreads();
  const int ne = s_ne;
  double sm = 0.0, sv = 0.0;
  float mx = -INFINITY;
  int nan = 0, over = 0, poison = 0;
  const int y = c0 + tx;
  for (int x = r0 + ty; x < min(r0 + PG_ROWS, W); x += PG_THREADS / PG_COLS) {
    if (y >= W) break;
    const size_t i = (size_t)x * W + y;
    int in = 0;
    if (x >= bx0 && x <= bx1 && y >= by0 && y <= by1) {
      int cnt = 0;
      for (int e = 0; e < ne; e++) {
        const int4 g = s_edge[e];
        if (y < min(g.y, g.w) || y > max(g.y, g.w)) continue;
        const int r = poly_edge_test(x, y, g.x, g.y, g.z, g.w);
        if (r == 2) { cnt = 1; break; }
        cnt += r;
      }
      in = cnt & 1;
    }
    const float m = in ? 1.0f : 0.0f;
    if (mask) mask[i] = m;
    if (x < 1 || x > W - 2 || y < 1 || y > W - 2) continue;
    // traversability_polygon.py:10-20, 25-30
    const float v = valid[i];
    const float untrav = v > 0.5f ? __fsub_rn(1.0f, checker[i]) : 0.0f;
    const float masked = __fmul_rn(untrav, m);
    sm += (double)masked;
    sv += (double)__fmul_rn(v, m);
    if (kBatch) poison += poly_poison(v, untrav);
    if (masked != masked) nan = 1; else mx = fmaxf(mx, masked);
    if (masked > a.thr_over) {
      over++;
      atomicMin(&s_cmin[tx], x - 1);
      atomicMax(&s_cmax[tx], x - 1);
    }
  }
  // fixed-order block reduction
  for (int o = 16; o; o >>= 1) {
    sm += __shfl_xor_sync(0xffffffffu, sm, o);
    sv += __shfl_xor_sync(0xffffffffu, sv, o);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    nan |= __shfl_xor_sync(0xffffffffu, nan, o);
    over += __shfl_xor_sync(0xffffffffu, over, o);
    if (kBatch) poison += __shfl_xor_sync(0xffffffffu, poison, o);
  }
  const int w = threadIdx.x / 32;
  if (threadIdx.x % 32 == 0) {
    s_sm[w] = sm; s_sv[w] = sv; s_mx[w] = mx; s_nan[w] = nan; s_over[w] = over; s_poison[w] = poison;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    PolyPartial p = {0.0, 0.0, -INFINITY, 0, 0, 0};
    for (int k = 0; k < PG_THREADS / 32; k++) {
      p.sum_masked += s_sm[k]; p.sum_valid += s_sv[k]; p.max_masked = fmaxf(p.max_masked, s_mx[k]);
      p.nan_masked |= s_nan[k]; p.over += s_over[k]; p.poison += s_poison[k];
    }
    part[blockIdx.x] = p;
  }
  // Interior column c0 + threadIdx.x - 1 of the tile lies in the polygon's window whenever it has an over cell: over
  // cells lie in the mask, hence in the box, unless 1 - safe_thresh < 0 makes the cells outside the mask over too, and
  // then the host gives every polygon the whole grid and window.  The bound keeps the atomics in the window regardless.
  if (col_min && threadIdx.x < PG_COLS && s_cmax[threadIdx.x] >= 0) {
    const int j = c0 + threadIdx.x - 1 - d.col0;
    if (j >= 0 && j < d.n_col) {
      atomicMin(&col_min[d.col_off + j], s_cmin[threadIdx.x]);
      atomicMax(&col_max[d.col_off + j], s_cmax[threadIdx.x]);
    }
  }
}

// Counts poly_poison over the interior into count[0] (untraversability) and count[1] (is_valid); zero on entry.
__global__ void __launch_bounds__(256) k_poly_poison(int W, const float* __restrict__ valid,
                                                     const float* __restrict__ checker, int* __restrict__ count) {
  int pu = 0, pv = 0;
  const size_t C = (size_t)W * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < C; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i / W), y = (int)(i % W);
    if (x < 1 || x > W - 2 || y < 1 || y > W - 2) continue;
    const float v = valid[i];
    const int p = poly_poison(v, v > 0.5f ? __fsub_rn(1.0f, checker[i]) : 0.0f);
    pu += p & 0xffff; pv += p >> 16;
  }
  for (int o = 16; o; o >>= 1) {
    pu += __shfl_xor_sync(0xffffffffu, pu, o);
    pv += __shfl_xor_sync(0xffffffffu, pv, o);
  }
  if (threadIdx.x % 32 == 0 && (pu | pv)) {
    atomicAdd(&count[0], pu);
    atomicAdd(&count[1], pv);
  }
}

// lower chain (Andrew's monotone chain, collinear points dropped) over the points of `n_src` sorted runs, written in
// place from dst.  Each point is read before any write reaches its slot, so the runs may overlap dst.
// cnt: the runs' lengths (NULL: one point each).
__device__ __forceinline__ int hull_chain(u32* pts, int dst, int n_src, int src_stride, const int* cnt) {
  int top = 0;
  for (int s = 0; s < n_src; s++) {
    const int base = dst + s * src_stride, m = cnt ? cnt[s] : 1;
    for (int k = 0; k < m; k++) {
      const u32 p = pts[base + k];
      const int pu = p >> 16, pv = p & 0xffff;
      while (top >= 2) {
        const u32 o = pts[dst + top - 2], q = pts[dst + top - 1];
        const int ou = o >> 16, ov = o & 0xffff;
        if ((int)((q >> 16) - ou) * (pv - ov) - (int)((q & 0xffff) - ov) * (pu - ou) > 0) break;
        top--;
      }
      pts[dst + top++] = p;
    }
  }
  return top;
}

// One CTA of HULL_THREADS per polygon.  Reduces the polygon's partials, decides safety, builds the ring of the convex
// hull of its over-threshold cells in metres (traversability_polygon.py:46-58, EM.py:876-879) and resets its column
// extremes.  A call without hulls (ring NULL) gives every polygon an empty column window, so no ring is built.
// Partials are summed as if the polygon had one per tile of the whole gx x gy grid: thread t takes tiles t, t + 1024,
// ...  A tile outside the polygon's tiles would give exact zero sums (its cells are outside the mask), which leave every
// partial sum unchanged, so a polygon that brings only its bounding box gets the bits the whole grid would give.  Such
// a tile's only other trace is a masked 0 in the maximum, and the NaN of a poisoned cell (counted by k_poly_poison).
// (__launch_bounds__(1024) makes ptxas cap the kernel at 32 registers and spill; 48 fit a 1024-thread CTA without spills.)
__global__ void __maxnreg__(48) k_hull(int W, double resolution, PolyArgs a, int gx, int gy,
                                       const PolyPartial* __restrict__ part, int* __restrict__ col_min,
                                       int* __restrict__ col_max, PolyResult* __restrict__ out,
                                       double2* __restrict__ ring) {
  __shared__ u32 s_pts[2][HULL_MAX_PTS];        // column extremes as (col << 16 | row): forward, and reversed
  __shared__ int s_cnt[2][2][HULL_MAX_PTS / HULL_GROUP];   // ping-pong survivor counts, per chain
  __shared__ int s_scan[HULL_THREADS / 32];
  __shared__ double s_sm[HULL_THREADS / 32], s_sv[HULL_THREADS / 32];
  __shared__ float s_mx[HULL_THREADS / 32];
  __shared__ int s_nan[HULL_THREADS / 32], s_over[HULL_THREADS / 32], s_pu[HULL_THREADS / 32], s_pv[HULL_THREADS / 32];
  __shared__ u32 s_start[HULL_THREADS / 32];
  const int t = threadIdx.x, lane = t % 32, w = t / 32;
  const PolyDesc& d = a.poly[blockIdx.x];
  // ---- statistics: each thread a fixed stride of the grid's tiles, then a fixed tree
  {
    double sm = 0.0, sv = 0.0;
    float mx = -INFINITY;
    int nan = 0, over = 0, pu = 0, pv = 0;
    const bool whole = d.n_tr == gy && d.n_tc == gx;      // the polygon's tiles are the grid: partial k is tile k
    for (int k = t; k < gx * gy; k += HULL_THREADS) {
      int q = k;
      if (!whole) {
        const int kr = k / gx - d.tr0, kc = k % gx - d.tc0;
        if (kr < 0 || kr >= d.n_tr || kc < 0 || kc >= d.n_tc) continue;
        q = kr * d.n_tc + kc;
      }
      const PolyPartial p = part[d.item0 + q];
      sm += p.sum_masked; sv += p.sum_valid; mx = fmaxf(mx, p.max_masked); nan |= p.nan_masked; over += p.over;
      pu += p.poison & 0xffff; pv += p.poison >> 16;
    }
    for (int o = 16; o; o >>= 1) {
      sm += __shfl_xor_sync(0xffffffffu, sm, o);
      sv += __shfl_xor_sync(0xffffffffu, sv, o);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      nan |= __shfl_xor_sync(0xffffffffu, nan, o);
      over += __shfl_xor_sync(0xffffffffu, over, o);
      pu += __shfl_xor_sync(0xffffffffu, pu, o);
      pv += __shfl_xor_sync(0xffffffffu, pv, o);
    }
    if (lane == 0) { s_sm[w] = sm; s_sv[w] = sv; s_mx[w] = mx; s_nan[w] = nan; s_over[w] = over; s_pu[w] = pu; s_pv[w] = pv; }
  }
  int m;                                                   // hull vertices
  {
    // ---- column extremes -> sorted points: two consecutive window columns per thread, compacted by a block scan
    const int n_col = d.n_col;
    int* cmin = col_min + d.col_off;
    int* cmax = col_max + d.col_off;
    auto take = [&](int c, int& l, int& u) {
      l = 0; u = -1;
      if (c < n_col && cmax[c] >= 0) {
        l = cmin[c]; u = cmax[c];
        cmin[c] = INT_MAX; cmax[c] = -1;
      }
    };
    int lo0, hi0, lo1, hi1;
    take(2 * t, lo0, hi0);
    take(2 * t + 1, lo1, hi1);
    auto n_of = [](int l, int u) { return u < 0 ? 0 : (u != l ? 2 : 1); };
    const int k_mine = n_of(lo0, hi0) + n_of(lo1, hi1);
    int incl = k_mine;
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) s_scan[w] = incl;
    __syncthreads();
    int before = 0, n = 0;
    for (int k = 0; k < HULL_THREADS / 32; k++) { if (k < w) before += s_scan[k]; n += s_scan[k]; }
    before += incl - k_mine;
    auto emit = [&](int c, int l, int u) {         // the column's row-min cell, then its row-max cell if different
      if (u < 0) return;
      c += d.col0;
      s_pts[0][before] = ((u32)c << 16) | (u32)l; s_pts[1][n - 1 - before] = ((u32)c << 16) | (u32)l; before++;
      if (u == l) return;
      s_pts[0][before] = ((u32)c << 16) | (u32)u; s_pts[1][n - 1 - before] = ((u32)c << 16) | (u32)u; before++;
    };
    emit(2 * t, lo0, hi0);
    emit(2 * t + 1, lo1, hi1);
    __syncthreads();
    // ---- lower chain of the forward order (row-min side) and of the reversed order (row-max side).  Level by level,
    // one thread chains HULL_GROUP consecutive runs of the previous level into one; the first level's runs are single
    // points.  A point dropped from the chain of some of the points is not a vertex of the chain of all of them.
    int n_run = n, stride = 1, cur = 1;
    while (n_run > 1) {
      const int n_next = (n_run + HULL_GROUP - 1) / HULL_GROUP;
      for (int k = t; k < 2 * n_next; k += HULL_THREADS) {
        const int ch = k / n_next, j = k % n_next;
        s_cnt[cur ^ 1][ch][j] = hull_chain(s_pts[ch], j * HULL_GROUP * stride, min(HULL_GROUP, n_run - j * HULL_GROUP),
                                           stride, stride == 1 ? nullptr : &s_cnt[cur][ch][j * HULL_GROUP]);
      }
      __syncthreads();
      cur ^= 1; n_run = n_next; stride *= HULL_GROUP;
    }
    // ---- the ring
    const int n_lo = n > 1 ? s_cnt[cur][0][0] : n, n_hi = n > 1 ? s_cnt[cur][1][0] : n;
    m = n > 1 ? (n_lo - 1) + (n_hi - 1) : 0;      // hull vertices, counter-clockwise in (col, row)
    const bool poly = m >= 3;
    // vertex k of the ring before rotation: the hull reversed, so that it runs counter-clockwise in (row, col)
    auto vert = [&](int k) -> u32 {
      const int h = m - 1 - k;
      return h < n_lo - 1 ? s_pts[0][h] : s_pts[1][h - (n_lo - 1)];
    };
    auto row_col = [](u32 p) -> u32 { return ((p & 0xffffu) << 16) | (p >> 16); };
    // the ring starts at its smallest (row, col) vertex
    u32 key = 0xffffffffu;
    for (int k = t; poly && k < m; k += HULL_THREADS) key = min(key, row_col(vert(k)));
    for (int o = 16; o; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
    if (lane == 0) s_start[w] = key;
    __syncthreads();
    key = 0xffffffffu;
    for (int k = 0; k < HULL_THREADS / 32; k++) key = min(key, s_start[k]);
    for (int k = t; poly && k < m; k += HULL_THREADS)
      if (row_col(vert(k)) == key) s_scan[0] = k;
    __syncthreads();
    const int start = s_scan[0];
    const double half = 0.5 * (double)W;
    double2* rg = ring + d.ring_off;
    for (int k = t; poly && k <= m; k += HULL_THREADS) {
      const u32 p = vert((start + k) % m);
      // traversability_polygon.py:56-58 in float64, multiply and add rounded separately as NumPy / CuPy do
      rg[k] = make_double2(__dadd_rn((double)a.cx, __dmul_rn((double)(p & 0xffff) - half, resolution)),
                           __dadd_rn((double)a.cy, __dmul_rn((double)(p >> 16) - half, resolution)));
    }
  }
  if (t == 0) {
    PolyResult r;
    r.sum_masked = 0.0; r.sum_valid = 0.0; r.max_masked = -INFINITY;
    int any_nan = 0, n_over = 0, pu = 0, pv = 0;
    for (int k = 0; k < HULL_THREADS / 32; k++) {
      r.sum_masked += s_sm[k]; r.sum_valid += s_sv[k]; r.max_masked = fmaxf(r.max_masked, s_mx[k]);
      any_nan |= s_nan[k]; n_over += s_over[k]; pu += s_pu[k]; pv += s_pv[k];
    }
    // the interior cells outside the polygon's tiles: masked 0 (NaN * 0 and inf * 0 for the poisoned ones)
    const bool covers = d.tr0 * PG_ROWS <= 1 && (d.tr0 + d.n_tr) * PG_ROWS >= W - 1 && d.tc0 * PG_COLS <= 1 &&
                        (d.tc0 + d.n_tc) * PG_COLS >= W - 1;
    if (!covers) r.max_masked = fmaxf(r.max_masked, 0.0f);
    if (a.poison && a.poison[0] > pu) { r.sum_masked = __longlong_as_double(0x7ff8000000000000ll); any_nan = 1; }
    if (a.poison && a.poison[1] > pv) r.sum_valid = __longlong_as_double(0x7ff8000000000000ll);
    if (any_nan) r.max_masked = __int_as_float(0x7fffffff);
    r.over = n_over;
    // EM.py:859-862 (a NaN sum fails the > 0 test); traversability_polygon.py:37-43 (a NaN maximum fails the > test)
    r.t = r.sum_valid > 0.0 ? (double)(float)(r.sum_masked / r.sum_valid) : 0.0;
    r.is_safe = !(n_over > a.max_unsafe_n) && !(r.max_masked > a.thr_max);
    r.n_ring = m >= 3 ? m + 1 : 0;
    r.pad[0] = r.pad[1] = 0;
    out[blockIdx.x] = r;
  }
}
