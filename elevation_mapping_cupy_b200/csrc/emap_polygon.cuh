// emap_polygon.cuh -- the polygon safety check (sm_90a): EM.py:837-889 get_polygon_traversability, CK.py:509-654
// polygon_mask_kernel, traversability_polygon.py:10-58.
//
// k_polygon: one pass over the map.  Each CTA owns a strip of PG_COLS columns and PG_ROWS rows; it turns the polygon's
// vertices into cells (CK.py:580-603) once, keeps the edges that can touch its strip, and every cell runs the reference's
// integer inside test against those edges only.  The same pass reads is_valid and the checker plane and reduces the
// statistics of traversability_polygon.py:10-34 over the interior [1:-1, 1:-1] into one partial per CTA, plus the
// per-column extremes of the over-threshold cells.
// k_hull: one CTA sums the partials in a fixed order (the result does not depend on scheduling) and builds the convex hull
// of the over-threshold cells (traversability_polygon.py:46-53) from the column extremes.
#pragma once
#include "emap_device.cuh"

#define PG_COLS 32               // columns per k_polygon CTA (one warp wide: coalesced rows)
#define PG_ROWS 64               // rows per k_polygon CTA
#define PG_THREADS 256
#define HULL_THREADS 1024
#define HULL_MAX_PTS 4096        // >= 2 * (W - 2) column extremes for W <= 2049
#define HULL_GROUP 8             // chunks merged per thread and level of k_hull's chain reduction

struct PolyPartial {             // one k_polygon CTA's share of the interior
  double sum_masked, sum_valid;
  float max_masked;              // max of the non-NaN masked values (-inf if none)
  int nan_masked;                // a masked value was NaN (CuPy's max propagates it)
  int over;                      // cells with masked > 1 - safe_thresh
  int pad;
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
// the double2 ring is carved directly behind the result (one read-back copy): keep it 16-byte aligned
static_assert(sizeof(PolyResult) % 16 == 0, "PolyResult must keep the ring behind it 16-byte aligned");

struct PolyArgs {
  const float2* xy;              // clipped fp32 vertices (EM.py:847-851)
  int n;
  float cx, cy;                  // map centre, fp32 (EM.py:61)
  float bbox[4];                 // min x, min y, max x, max y of the clipped vertices (EM.py:852-854)
  float thr_over, thr_max;       // fp32(1 - safe_thresh), fp32(1 - safe_min_thresh): CuPy compares in fp32
  int max_unsafe_n;
};

// CK.py:580-603 get_x_idx / get_idx for one coordinate: the coordinate and the centre are CuPy float16, their difference
// is taken in float, divided by the float `resolution`, 0.5 * width is added in double and the sum truncated to int;
// clamp() goes through float16, which is exact for W - 1 <= 2048.
__device__ __forceinline__ int poly_axis_cell(float v, float c, float res_f, int W) {
  const float d = __fsub_rn(h16(v), h16(c));
  const int i = __double2int_rz((double)__fdiv_rn(d, res_f) + 0.5 * (double)W);
  return min(max(i, 0), W - 1);
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

// grid (cdiv(W, PG_COLS), cdiv(W, PG_ROWS)), PG_THREADS threads.  col_min / col_max: per interior column, the smallest /
// largest interior row of an over-threshold cell; INT_MAX / -1 on entry, k_hull resets them.
__global__ void __launch_bounds__(PG_THREADS) k_polygon(int W, float res_f, PolyArgs a, const float* __restrict__ valid,
                                                        const float* __restrict__ checker, float* __restrict__ mask,
                                                        PolyPartial* __restrict__ part, int* __restrict__ col_min,
                                                        int* __restrict__ col_max) {
  __shared__ int4 s_edge[1024];
  __shared__ int s_ne, s_cmin[PG_COLS], s_cmax[PG_COLS];
  __shared__ double s_sm[PG_THREADS / 32], s_sv[PG_THREADS / 32];
  __shared__ float s_mx[PG_THREADS / 32];
  __shared__ int s_nan[PG_THREADS / 32], s_over[PG_THREADS / 32];
  const int tx = threadIdx.x % PG_COLS, ty = threadIdx.x / PG_COLS;
  const int c0 = blockIdx.x * PG_COLS, r0 = blockIdx.y * PG_ROWS;
  const int c1 = min(c0 + PG_COLS, W) - 1;
  if (threadIdx.x == 0) s_ne = 0;
  if (threadIdx.x < PG_COLS) { s_cmin[threadIdx.x] = INT_MAX; s_cmax[threadIdx.x] = -1; }
  // CK.py:609-615: the cell bounding box of the clipped polygon
  const int bx0 = poly_axis_cell(a.bbox[0], a.cx, res_f, W), by0 = poly_axis_cell(a.bbox[1], a.cy, res_f, W);
  const int bx1 = poly_axis_cell(a.bbox[2], a.cx, res_f, W), by1 = poly_axis_cell(a.bbox[3], a.cy, res_f, W);
  const bool tile_in_box = !(r0 + PG_ROWS - 1 < bx0 || r0 > bx1 || c1 < by0 || c0 > by1);
  __syncthreads();
  // An edge matters to a cell (x, y) only if its column range contains y (the on-edge and the crossing tests both need
  // that) and it reaches row x or beyond (the ray runs toward +x).  Order does not matter: the count's parity and "on an
  // edge" are all the cell needs.
  if (tile_in_box) {
    for (int j = threadIdx.x; j < a.n; j += PG_THREADS) {
      const float2 p = a.xy[j], q = a.xy[j + 1 == a.n ? 0 : j + 1];
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
  int nan = 0, over = 0;
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
  }
  const int w = threadIdx.x / 32;
  if (threadIdx.x % 32 == 0) { s_sm[w] = sm; s_sv[w] = sv; s_mx[w] = mx; s_nan[w] = nan; s_over[w] = over; }
  __syncthreads();
  if (threadIdx.x == 0) {
    PolyPartial p = {0.0, 0.0, -INFINITY, 0, 0, 0};
    for (int k = 0; k < PG_THREADS / 32; k++) {
      p.sum_masked += s_sm[k]; p.sum_valid += s_sv[k]; p.max_masked = fmaxf(p.max_masked, s_mx[k]);
      p.nan_masked |= s_nan[k]; p.over += s_over[k];
    }
    part[blockIdx.y * gridDim.x + blockIdx.x] = p;
  }
  if (threadIdx.x < PG_COLS && s_cmax[threadIdx.x] >= 0) {
    atomicMin(&col_min[c0 + threadIdx.x - 1], s_cmin[threadIdx.x]);
    atomicMax(&col_max[c0 + threadIdx.x - 1], s_cmax[threadIdx.x]);
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

// One CTA of HULL_THREADS.  Reduces the n_part partials, decides safety, builds the ring of the over-threshold cells'
// convex hull in metres (traversability_polygon.py:46-58, EM.py:876-879) and resets col_min / col_max.
// (__launch_bounds__(1024) makes ptxas cap the kernel at 32 registers and spill; 48 fit a 1024-thread CTA without spills.)
__global__ void __maxnreg__(48) k_hull(int W, double resolution, PolyArgs a,
                                                       const PolyPartial* __restrict__ part, int n_part,
                                                       int* __restrict__ col_min, int* __restrict__ col_max,
                                                       PolyResult* __restrict__ out, double2* __restrict__ ring) {
  __shared__ u32 s_pts[2][HULL_MAX_PTS];        // column extremes as (col << 16 | row): forward, and reversed
  __shared__ int s_cnt[2][2][HULL_MAX_PTS / HULL_GROUP];   // ping-pong survivor counts, per chain
  __shared__ int s_scan[HULL_THREADS / 32];
  __shared__ double s_sm[HULL_THREADS / 32], s_sv[HULL_THREADS / 32];
  __shared__ float s_mx[HULL_THREADS / 32];
  __shared__ int s_nan[HULL_THREADS / 32], s_over[HULL_THREADS / 32];
  __shared__ u32 s_start[HULL_THREADS / 32];
  const int t = threadIdx.x, lane = t % 32, w = t / 32;
  // ---- statistics: each thread a fixed stride of partials, then a fixed tree
  double sm = 0.0, sv = 0.0;
  float mx = -INFINITY;
  int nan = 0, over = 0;
  for (int k = t; k < n_part; k += HULL_THREADS) {
    const PolyPartial p = part[k];
    sm += p.sum_masked; sv += p.sum_valid; mx = fmaxf(mx, p.max_masked); nan |= p.nan_masked; over += p.over;
  }
  for (int o = 16; o; o >>= 1) {
    sm += __shfl_xor_sync(0xffffffffu, sm, o);
    sv += __shfl_xor_sync(0xffffffffu, sv, o);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    nan |= __shfl_xor_sync(0xffffffffu, nan, o);
    over += __shfl_xor_sync(0xffffffffu, over, o);
  }
  if (lane == 0) { s_sm[w] = sm; s_sv[w] = sv; s_mx[w] = mx; s_nan[w] = nan; s_over[w] = over; }
  // ---- column extremes -> sorted points: two consecutive interior columns per thread, compacted by a block scan
  const int n_col = W - 2;
  auto take = [&](int c, int& l, int& u) {
    l = 0; u = -1;
    if (c < n_col && col_max[c] >= 0) {
      l = col_min[c]; u = col_max[c];
      col_min[c] = INT_MAX; col_max[c] = -1;
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
    s_pts[0][before] = ((u32)c << 16) | (u32)l; s_pts[1][n - 1 - before] = ((u32)c << 16) | (u32)l; before++;
    if (u == l) return;
    s_pts[0][before] = ((u32)c << 16) | (u32)u; s_pts[1][n - 1 - before] = ((u32)c << 16) | (u32)u; before++;
  };
  emit(2 * t, lo0, hi0);
  emit(2 * t + 1, lo1, hi1);
  __syncthreads();
  // ---- lower chain of the forward order (row-min side) and of the reversed order (row-max side).  Level by level, one
  // thread chains HULL_GROUP consecutive runs of the previous level into one; the first level's runs are single points.
  // A point dropped from the chain of some of the points is not a vertex of the chain of all of them.
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
  // ---- result
  const int n_lo = n > 1 ? s_cnt[cur][0][0] : n, n_hi = n > 1 ? s_cnt[cur][1][0] : n;
  const int m = n > 1 ? (n_lo - 1) + (n_hi - 1) : 0;      // hull vertices, counter-clockwise in (col, row)
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
  for (int k = t; poly && k <= m; k += HULL_THREADS) {
    const u32 p = vert((start + k) % m);
    // traversability_polygon.py:56-58 in float64, multiply and add rounded separately as NumPy / CuPy do
    ring[k] = make_double2(__dadd_rn((double)a.cx, __dmul_rn((double)(p & 0xffff) - half, resolution)),
                           __dadd_rn((double)a.cy, __dmul_rn((double)(p >> 16) - half, resolution)));
  }
  if (t == 0) {
    PolyResult r;
    r.sum_masked = 0.0; r.sum_valid = 0.0; r.max_masked = -INFINITY;
    int any_nan = 0, cnt = 0;
    for (int k = 0; k < HULL_THREADS / 32; k++) {
      r.sum_masked += s_sm[k]; r.sum_valid += s_sv[k]; r.max_masked = fmaxf(r.max_masked, s_mx[k]);
      any_nan |= s_nan[k]; cnt += s_over[k];
    }
    if (any_nan) r.max_masked = __int_as_float(0x7fffffff);
    r.over = cnt;
    // EM.py:859-862 (a NaN sum fails the > 0 test); traversability_polygon.py:37-43 (a NaN maximum fails the > test)
    r.t = r.sum_valid > 0.0 ? (double)(float)(r.sum_masked / r.sum_valid) : 0.0;
    r.is_safe = !(cnt > a.max_unsafe_n) && !(r.max_masked > a.thr_max);
    r.n_ring = poly ? m + 1 : 0;
    r.pad[0] = r.pad[1] = 0;
    *out = r;
  }
}
