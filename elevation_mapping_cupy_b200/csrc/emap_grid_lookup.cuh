// emap_grid_lookup.cuh -- lookups along lines and derivatives at points on one fp32 grid layer (emap_max_values_between,
// emap_values_between, emap_grid_derivatives), sm_90a.
//
// Reference: grid_map_filters_rsl's lookup.cpp (maxValueBetweenLocations, valuesBetweenLocations,
// projectToMapWithMargin) over grid_map_core's LineIterator, and GridMapDerivative.cpp (estimateGradient,
// estimateGradientAndCurvature).  LineIterator and the index arithmetic (emap_grid.cuh) are restated from grid_map's
// published source, Eigen's sum orders from Eigen's; include/emap.h states the contract, DESIGN.md §4l the restatement.
//
// The per-query functions are __host__ __device__: on the device one warp runs a line, its lanes striding over the
// line's cells and combining their results with shuffles and ballots; on the host (tests/native/lookup_host.cpp) one
// thread runs them with the same arithmetic, so the two give the same bits.  A derivative is one thread's work on both.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "emap_grid.cuh"

#define GL_WARPS 8                 // lines (warps) per block of the line kernels
#define GL_THREADS 256             // queries per block of k_gl_derivatives
#define GL_SCAN_THREADS 1024       // k_gl_scan's single block
#define GL_MARGIN 1e-6             // projectToMapWithMargin's default margin

#if defined(__CUDA_ARCH__)
#define GL_LANE ((int)(threadIdx.x & 31))
#define GL_LANES 32
#define GL_FMUL(a, b) __fmul_rn((a), (b))
#define GL_FADD(a, b) __fadd_rn((a), (b))
#else
#define GL_LANE 0
#define GL_LANES 1
#define GL_FMUL(a, b) ((float)(a) * (float)(b))
#define GL_FADD(a, b) ((float)(a) + (float)(b))
#endif

enum { GL_INSIDE = 0, GL_OUTSIDE = 1 };   // emap.h's EMAP_DERIVATIVE_*

// One layer and its grid_map geometry: rows x cols cells, row-major (index (r, c) at r cols + c), position pos (the
// centre of its cells), length len = (rows, cols) res, buffer start index 0.
struct GlGrid {
  const float* data;
  int rows, cols;
  double pos[2], len[2], res;
};

GRID_HD float gl_at(const GlGrid& g, int r, int c) { return g.data[(int64_t)r * g.cols + c]; }

GRID_HD bool gl_finite(float h) { return fabsf(h) <= FLT_MAX; }   // std::isfinite

// ---- lines ----
// projectToMapWithMargin with the default margin: m = min(max(1e-6, 0), L.x / 2, L.y / 2); each coordinate
// fmax(fmin(v, (pos + L / 2) - m), (pos - L / 2) + m) (a NaN goes to the upper bound, as std::fmin returns the other
// operand).
GRID_HD void gl_project(const GlGrid& g, double x, double y, double p[2]) {
  const double half[2] = {GRID_MUL(g.len[0], 0.5), GRID_MUL(g.len[1], 0.5)};
  double m = GL_MARGIN;
  m = half[0] < m ? half[0] : m;
  m = half[1] < m ? half[1] : m;
  const double v[2] = {x, y};
  for (int a = 0; a < 2; a++) {
    const double hi = GRID_ADD(GRID_ADD(g.pos[a], half[a]), -m), lo = GRID_ADD(GRID_ADD(g.pos[a], -half[a]), m);
    p[a] = fmax(fmin(v[a], hi), lo);
  }
}

// LineIterator's walk between two cells (Bresenham): the major axis is the rows (grid_map's x) when |dr| >= |dc|;
// cell i is start + i steps on the major axis and start + k(i) steps on the minor one, k(i) = floor((half + i add) /
// den) with den = the major delta (1 when it is 0: then the line is its start cell), half = den / 2 and add = the minor
// delta.  That is the iterator's numerator: each ++ adds add <= den, so it crosses den at most once per step.
struct GlLine {
  int r0, c0, sr, sc;              // start cell, step per axis (+1 when the end is not below the start, else -1)
  bool row_major;
  int64_t den, half, add, n;       // n: cells, major delta + 1
};

GRID_HD void gl_line_from_cells(int r0, int c0, int r1, int c1, GlLine& L) {
  const int64_t dr = r1 >= r0 ? (int64_t)r1 - r0 : (int64_t)r0 - r1;
  const int64_t dc = c1 >= c0 ? (int64_t)c1 - c0 : (int64_t)c0 - c1;
  L.r0 = r0;
  L.c0 = c0;
  L.sr = r1 >= r0 ? 1 : -1;
  L.sc = c1 >= c0 ? 1 : -1;
  L.row_major = dr >= dc;
  const int64_t major = L.row_major ? dr : dc;
  L.add = L.row_major ? dc : dr;
  L.half = major / 2;
  L.den = major ? major : 1;
  L.n = major + 1;
}

// The line of one query (x0, y0, x1, y1): both ends through gl_project, then getIndex.  For the grids the entry points
// accept a projected end is always inside the map (include/emap.h shows why), so getIndexLimitedToMapRange's stepping
// loop never runs and grid_axis_index always succeeds.
GRID_HD void gl_line(const GlGrid& g, const double* q, GlLine& L) {
  int idx[4] = {0, 0, 0, 0};
  for (int e = 0; e < 2; e++) {
    double p[2];
    gl_project(g, q[2 * e], q[2 * e + 1], p);
    grid_axis_index(p[0], g.pos[0], g.len[0], g.res, g.rows, idx[2 * e]);
    grid_axis_index(p[1], g.pos[1], g.len[1], g.res, g.cols, idx[2 * e + 1]);
  }
  gl_line_from_cells(idx[0], idx[1], idx[2], idx[3], L);
}

// k(i) for i = i0, i0 + step, ...: one division at the start, then additions (step add < 2^36: no sum overflows).
struct GlCursor {
  int64_t k, rem, dk, drem, den;
  GRID_HD GlCursor(const GlLine& L, int64_t i0, int64_t step) {
    const int64_t num = L.half + i0 * L.add, s = step * L.add;
    den = L.den;
    k = num / den;
    rem = num % den;
    dk = s / den;
    drem = s % den;
  }
  GRID_HD void next() {
    k += dk;
    rem += drem;
    if (rem >= den) {
      rem -= den;
      k++;
    }
  }
};

GRID_HD void gl_cell(const GlLine& L, int64_t i, int64_t k, int& r, int& c) {
  r = (int)(L.r0 + (L.row_major ? i : k) * L.sr);
  c = (int)(L.c0 + (L.row_major ? k : i) * L.sc);
}

// ok's rank among the lanes below with ok set, and their count n (the identity on the host)
GRID_HD int gl_rank(bool ok, int& n) {
#if defined(__CUDA_ARCH__)
  const unsigned b = __ballot_sync(0xffffffffu, ok);
  n = __popc(b);
  return __popc(b & ((1u << GL_LANE) - 1u));
#else
  n = ok;
  return 0;
#endif
}

// f(k, r, c, value) for the k-th finite cell of the line, in iterator order; returns the number of finite cells.  The
// lanes take the cells in chunks of `lanes` consecutive ones.
template <typename F>
GRID_HD int64_t gl_finite_cells(const GlGrid& g, const GlLine& L, int lane, int lanes, F&& f) {
  GlCursor cur(L, lane, lanes);
  int64_t w = 0;
  for (int64_t base = 0; base < L.n; base += lanes, cur.next()) {
    const int64_t i = base + lane;
    int r = 0, c = 0, cnt;
    float h = 0.0f;
    bool ok = false;
    if (i < L.n) {
      gl_cell(L, i, cur.k, r, c);
      h = gl_at(g, r, c);
      ok = gl_finite(h);
    }
    const int k = gl_rank(ok, cnt);
    if (ok) f(w + k, r, c, h);
    w += cnt;
  }
  return w;
}

// (v, first): the largest finite value of the cells seen and the first cell (ordinal) that holds it (first < 0: none);
// last: the last finite cell.  Combined over the warp (the identity on the host); the same on every lane.
GRID_HD void gl_max_combine(float& v, int64_t& first, int64_t& last) {
#if defined(__CUDA_ARCH__)
  for (int s = 16; s; s >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, s);
    const int64_t of = __shfl_xor_sync(0xffffffffu, first, s), ol = __shfl_xor_sync(0xffffffffu, last, s);
    if (of >= 0 && (first < 0 || ov > v || (ov == v && of < first))) {
      v = ov;
      first = of;
    }
    last = ol > last ? ol : last;
  }
#endif
}

// maxValueBetweenLocations: idx = {valid, row, col}, val = {value, x, y}.  value: std::max from -FLT_MAX over the
// finite cells in order, i.e. the first cell holding the largest value (its sign for a largest zero); valid: value >
// -FLT_MAX; (row, col): the LAST finite cell (the reference sets maxIndex at every finite cell), (0, 0) without one;
// (x, y): its position.
GRID_HD void gl_max_line(const GlGrid& g, const GlLine& L, int lane, int lanes, int32_t idx[3], double val[3]) {
  float v = -FLT_MAX;
  int64_t first = -1, last = -1;
  GlCursor cur(L, lane, lanes);
  for (int64_t i = lane; i < L.n; i += lanes, cur.next()) {
    int r, c;
    gl_cell(L, i, cur.k, r, c);
    const float h = gl_at(g, r, c);
    if (gl_finite(h)) {
      if (first < 0 || h > v) {
        v = h;
        first = i;
      }
      last = i;
    }
  }
  gl_max_combine(v, first, last);
  int r = 0, c = 0;
  if (last >= 0) gl_cell(L, last, (L.half + last * L.add) / L.den, r, c);
  idx[0] = v > -FLT_MAX;
  idx[1] = r;
  idx[2] = c;
  val[0] = (double)v;
  val[1] = grid_axis_position(g.pos[0], g.len[0], g.res, r);
  val[2] = grid_axis_position(g.pos[1], g.len[1], g.res, c);
}

// valuesBetweenLocations: (x, y, value) per finite cell, in iterator order, from rows (3 doubles per row)
GRID_HD void gl_values_line(const GlGrid& g, const GlLine& L, int lane, int lanes, double* rows) {
  const double x0 = grid_axis_origin(g.pos[0], g.len[0], g.res), y0 = grid_axis_origin(g.pos[1], g.len[1], g.res);
  const double res = g.res;
  gl_finite_cells(g, L, lane, lanes, [=](int64_t k, int r, int c, float h) {
    double* o = rows + 3 * k;
    o[0] = grid_axis_at(x0, res, r);
    o[1] = grid_axis_at(y0, res, c);
    o[2] = (double)h;
  });
}

// ---- derivatives ----
// GridMapDerivative's kernels: float(literal) / float(res) and float(literal) / (float(res) * float(res)), in float
// (Eigen's /= divides element by element).  Built on the host once per call.
struct GlKernels {
  float d1[5], d2[5];
};

inline GlKernels gl_kernels(double res) {
  const float r = (float)res, r2 = r * r;
  const float c1[5] = {(float)(-1.0 / 12.0), (float)(2.0 / 3.0), 0.0f, (float)(-2.0 / 3.0), (float)(1.0 / 12.0)};
  const float c2[5] = {(float)(-1.0 / 12.0), (float)(4.0 / 3.0), (float)(-5.0 / 2.0), (float)(4.0 / 3.0),
                       (float)(-1.0 / 12.0)};
  GlKernels K;
  for (int k = 0; k < 5; k++) {
    K.d1[k] = c1[k] / r;
    K.d2[k] = c2[k] / r2;
  }
  return K;
}

// Eigen's dot of a Matrix<float, 5, 1> with a contiguous 5-vector (a column block, or another Matrix<float, 5, 1>): one
// 4-float packet reduced as (p0 + p2) + (p1 + p3), then the fifth product: ((p0 + p2) + (p1 + p3)) + p4.
GRID_HD float gl_dot_contiguous(const float k[5], const float x[5]) {
  float p[5];
#pragma unroll
  for (int i = 0; i < 5; i++) p[i] = GL_FMUL(k[i], x[i]);
  return GL_FADD(GL_FADD(GL_FADD(p[0], p[2]), GL_FADD(p[1], p[3])), p[4]);
}

// ... with a strided 5-vector (a row block of the column-major matrix): the unrolled halving sum
// (p0 + p1) + (p2 + (p3 + p4)).
GRID_HD float gl_dot_strided(const float k[5], const float x[5]) {
  float p[5];
#pragma unroll
  for (int i = 0; i < 5; i++) p[i] = GL_FMUL(k[i], x[i]);
  return GL_FADD(GL_FADD(p[0], p[1]), GL_FADD(p[2], GL_FADD(p[3], p[4])));
}

// A derivative widened to double; NaN as the one quiet NaN 0x7ff8000000000000 (the device's float operations and the
// host's give NaNs different payloads).
GRID_HD double gl_widen(float f) {
  if (f == f) return (double)f;
#if defined(__CUDA_ARCH__)
  return __longlong_as_double(0x7ff8000000000000ll);
#else
  const uint64_t u = 0x7ff8000000000000ull;
  double d;
  memcpy(&d, &u, sizeof d);
  return d;
#endif
}

// getKernelCenter's shift of the first tap from i - 2: -min(i - 2, 0) - max(i + 2 - (n - 1), 0) (n >= 5)
GRID_HD int gl_tap0(int i, int n) {
  const int lo = i - 2 < 0 ? i - 2 : 0, hi = i + 2 - (n - 1) > 0 ? i + 2 - (n - 1) : 0;
  return i - 2 - lo - hi;
}

// One query position: idx = {status, row, col}; v = {gx, gy} and, with curvature, {cxx, cxy, cyy}.  Outside the map
// (getIndex fails): status OUTSIDE, row = col = -1, every v 0.  Inside, with the 5 taps at rows r0 .. r0 + 4 and
// columns c0 .. c0 + 4 (gl_tap0): gx = d1 . H(r0.., c) (contiguous), gy = d1 . H(r, c0..) (strided), cxx = d2 .
// H(r0.., c), cyy = d2 . H(r, c0..), cxy = d1 . (d1 . H(r0.., c0 + j))_j (both contiguous); each in float, widened
// (gl_widen).
GRID_HD void gl_derivative(const GlGrid& g, const GlKernels& K, double x, double y, int curvature, int32_t idx[3],
                           double* v) {
  int r = 0, c = 0;
  const int nv = curvature ? 5 : 2;
  if (!grid_axis_index(x, g.pos[0], g.len[0], g.res, g.rows, r) ||
      !grid_axis_index(y, g.pos[1], g.len[1], g.res, g.cols, c)) {
    idx[0] = GL_OUTSIDE;
    idx[1] = idx[2] = -1;
#pragma unroll
    for (int k = 0; k < 5; k++)
      if (k < nv) v[k] = 0.0;
    return;
  }
  const int r0 = gl_tap0(r, g.rows), c0 = gl_tap0(c, g.cols);
  float col[5], row[5];
#pragma unroll
  for (int k = 0; k < 5; k++) {
    col[k] = gl_at(g, r0 + k, c);
    row[k] = gl_at(g, r, c0 + k);
  }
  idx[0] = GL_INSIDE;
  idx[1] = r;
  idx[2] = c;
  v[0] = gl_widen(gl_dot_contiguous(K.d1, col));
  v[1] = gl_widen(gl_dot_strided(K.d1, row));
  if (!curvature) return;
  float gy[5];
#pragma unroll
  for (int j = 0; j < 5; j++) {
    float cj[5];
#pragma unroll
    for (int k = 0; k < 5; k++) cj[k] = gl_at(g, r0 + k, c0 + j);
    gy[j] = gl_dot_contiguous(K.d1, cj);
  }
  v[2] = gl_widen(gl_dot_contiguous(K.d2, col));
  v[3] = gl_widen(gl_dot_contiguous(K.d1, gy));
  v[4] = gl_widen(gl_dot_strided(K.d2, row));
}

#if defined(__CUDACC__)
// ---- kernels: one warp per line (GL_WARPS per block), one thread per derivative query ----

__global__ void __launch_bounds__(32 * GL_WARPS)
k_gl_max(const GlGrid g, const double* __restrict__ lines, int64_t n, int32_t* __restrict__ index,
         double* __restrict__ value) {
  const int64_t q = (int64_t)blockIdx.x * GL_WARPS + (threadIdx.x >> 5);
  if (q >= n) return;
  GlLine L;
  gl_line(g, lines + 4 * q, L);
  int32_t idx[3];
  double val[3];
  gl_max_line(g, L, GL_LANE, GL_LANES, idx, val);
  if (GL_LANE == 0)
    for (int k = 0; k < 3; k++) {
      index[3 * q + k] = idx[k];
      value[3 * q + k] = val[k];
    }
}

// counts[q] = the finite cells of line q; block_sum[b] = the sum over block b's lines
__global__ void __launch_bounds__(32 * GL_WARPS)
k_gl_count(const GlGrid g, const double* __restrict__ lines, int64_t n, int32_t* __restrict__ counts,
           int64_t* __restrict__ block_sum) {
  __shared__ int64_t s[GL_WARPS];
  const int w = threadIdx.x >> 5;
  const int64_t q = (int64_t)blockIdx.x * GL_WARPS + w;
  int64_t cnt = 0;
  if (q < n) {
    GlLine L;
    gl_line(g, lines + 4 * q, L);
    cnt = gl_finite_cells(g, L, GL_LANE, GL_LANES, [](int64_t, int, int, float) {});
    if (GL_LANE == 0) counts[q] = (int32_t)cnt;
  }
  if (GL_LANE == 0) s[w] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t t = 0;
    for (int k = 0; k < GL_WARPS; k++) t += s[k];
    block_sum[blockIdx.x] = t;
  }
}

// One block: block_sum becomes its exclusive prefix sum; info = {total, total <= capacity}.  Thread t scans a
// contiguous range of the blocks.
__global__ void __launch_bounds__(GL_SCAN_THREADS)
k_gl_scan(int64_t* __restrict__ block_sum, int64_t n_blocks, int64_t capacity, int64_t* __restrict__ info) {
  __shared__ int64_t s[GL_SCAN_THREADS / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t per = (n_blocks + GL_SCAN_THREADS - 1) / GL_SCAN_THREADS;
  const int64_t b0 = min((int64_t)t * per, n_blocks), b1 = min(b0 + per, n_blocks);
  int64_t sum = 0;
  for (int64_t b = b0; b < b1; b++) sum += block_sum[b];
  int64_t x = sum;                                   // inclusive scan over the warp, then over the warps' totals
  for (int d = 1; d < 32; d <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) s[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int64_t y = s[lane];
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t z = __shfl_up_sync(0xffffffffu, y, d);
      if (lane >= d) y += z;
    }
    s[lane] = y;
  }
  __syncthreads();
  int64_t off = x - sum + (warp ? s[warp - 1] : 0);
  for (int64_t b = b0; b < b1; b++) {
    const int64_t c = block_sum[b];
    block_sum[b] = off;
    off += c;
  }
  if (t == GL_SCAN_THREADS - 1) {
    info[0] = off;
    info[1] = off <= capacity;
  }
}

// first[q] = block_off[b] + the counts of the block's earlier lines; the rows only when info[1] (complete)
__global__ void __launch_bounds__(32 * GL_WARPS)
k_gl_values(const GlGrid g, const double* __restrict__ lines, int64_t n, const int32_t* __restrict__ counts,
            const int64_t* __restrict__ block_off, const int64_t* __restrict__ info, int64_t* __restrict__ first,
            double* __restrict__ rows) {
  const int w = threadIdx.x >> 5;
  const int64_t q0 = (int64_t)blockIdx.x * GL_WARPS, q = q0 + w;
  if (q >= n) return;
  int64_t before = GL_LANE < w ? counts[q0 + GL_LANE] : 0;
  for (int s = 16; s; s >>= 1) before += __shfl_xor_sync(0xffffffffu, before, s);
  const int64_t f = block_off[blockIdx.x] + before;
  if (GL_LANE == 0) first[q] = f;
  if (!info[1]) return;
  GlLine L;
  gl_line(g, lines + 4 * q, L);
  gl_values_line(g, L, GL_LANE, GL_LANES, rows + 3 * f);
}

__global__ void __launch_bounds__(GL_THREADS)
k_gl_derivatives(const GlGrid g, const GlKernels K, const double* __restrict__ pos, int64_t n, int curvature,
                 int32_t* __restrict__ index, double* __restrict__ value) {
  const int64_t q = (int64_t)blockIdx.x * GL_THREADS + threadIdx.x;
  if (q >= n) return;
  int32_t idx[3];
  double v[5];
  gl_derivative(g, K, pos[2 * q], pos[2 * q + 1], curvature, idx, v);
#pragma unroll
  for (int k = 0; k < 3; k++) index[3 * q + k] = idx[k];
  const int nv = curvature ? 5 : 2;
#pragma unroll
  for (int k = 0; k < 5; k++)
    if (k < nv) value[nv * q + k] = v[k];
}
#endif
