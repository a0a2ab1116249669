// emap_filters.cuh -- grid_map_filters_rsl's layer filters on a caller's grid (emap_grid_filter), sm_90a.
//
// Reference: grid_map_filters_rsl's smoothing.cpp (median, boxBlur, gaussianBlur), processing.cpp (dilate, erode,
// outline) and inpainting.cpp's minValues.  include/emap.h states the contract; DESIGN.md §4l the restatement.  The
// minValues fill and the float median are emap_planes.cuh's, the Gaussian emap_postprocess.cuh's; this header holds
// the passes nothing else has: OpenCV's running-sum box filter, the 8-bit median and the clamped-window max / min.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "emap_grid.cuh"
#include "emap_postprocess.cuh"
#include "emap_submap.cuh"

#define GF_THREADS 256
#define GF_MED_COLS 64             // columns (threads) per k_gf_median_u8 CTA, one 256-bin histogram each
#define GF_MED_ROWS 64             // rows each k_gf_median_u8 thread walks down its column

#if defined(__CUDACC__)
// RowSum<float, double> of cv::blur for k > 5, one thread per row, BORDER_REFLECT_101 with the anchor at k / 2: OpenCV's
// running sum s += x[c + k] - x[c] along the row, which is sequential.  For k <= 5 OpenCV sums each window directly;
// that is k_pp_box_rows<true> (emap_postprocess.cuh), one thread per cell.  Its leading 0.0 + x turns a -0.0 into +0.0,
// which the column pass's running sum (it starts at +0.0) would do anyway.
__global__ void k_gf_box_rows(const float* __restrict__ src, double* __restrict__ rs, int rows, int cols, int k) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const float* row = src + (long long)r * cols;
  double* out = rs + (long long)r * cols;
  const int a = k / 2;
  double s = 0.0;
  for (int j = 0; j < k; j++) s = __dadd_rn(s, (double)__ldg(row + pp_reflect101(j - a, cols - 1)));
  out[0] = s;
  for (int c = 0; c + 1 < cols; c++) {
    const double d = __dsub_rn((double)__ldg(row + pp_reflect101(c + k - a, cols - 1)),
                               (double)__ldg(row + pp_reflect101(c - a, cols - 1)));
    s = __dadd_rn(s, d);
    out[c + 1] = s;
  }
}

// ColumnSum<double, float> of cv::blur, one thread per column: a running sum from the top border row down, out =
// float(s0 * scale) with s0 = sum + the entering row, then sum = s0 - the leaving row.  The order is OpenCV's, so a NaN
// or an infinity stays in the sum below its row as in cv2.
__global__ void k_gf_box_cols(const double* __restrict__ rs, float* __restrict__ dst, int rows, int cols, int k,
                              double scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const int a = k / 2;
  double sum = 0.0;
  for (int j = 0; j < k - 1; j++) sum = __dadd_rn(sum, __ldg(rs + (long long)pp_reflect101(j - a, rows - 1) * cols + c));
  for (int r = 0; r < rows; r++) {
    const double s0 = __dadd_rn(sum, __ldg(rs + (long long)pp_reflect101(r + k - 1 - a, rows - 1) * cols + c));
    dst[(long long)r * cols + c] = (float)__dmul_rn(s0, scale);
    sum = __dsub_rn(s0, __ldg(rs + (long long)pp_reflect101(r - a, rows - 1) * cols + c));
  }
}

// minCoeffOfFinites / maxCoeffOfFinites of the grid and its count of finite cells: w[0] the complement of the lowest
// order-preserving key (0: none), w[1] the highest key, w[2] the count; w zeroed before.
__global__ void k_gf_range(const float* __restrict__ h, unsigned* __restrict__ w, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned lo_c = 0u, hi = 0u, nv = 0u;
  if (i < n && isfinite(h[i])) {
    hi = tsub_fkey(h[i]);
    lo_c = ~hi;
    nv = 1u;
  }
  lo_c = __reduce_max_sync(0xffffffffu, lo_c); hi = __reduce_max_sync(0xffffffffu, hi);
  nv = __reduce_add_sync(0xffffffffu, nv);
  if ((threadIdx.x & 31) == 0 && nv) { atomicMax(&w[0], lo_c); atomicMax(&w[1], hi); atomicAdd(&w[2], nv); }
}

// lo / hi of k_gf_range: the finite minimum and maximum, or +-FLT_MAX when nothing is finite (as in the reference).
__device__ __forceinline__ void gf_range(const unsigned* w, float& lo, float& hi) {
  lo = 3.402823466e38f; hi = -3.402823466e38f;
  if (w[2]) { lo = tsub_funkey(~w[0]); hi = tsub_funkey(w[1]); }
}

// toImage<uchar, 1>(lo, hi): a NaN cell gives 0.
__global__ void k_gf_quantise(const float* __restrict__ h, const unsigned* __restrict__ w, uint8_t* __restrict__ img,
                              int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float lo, hi;
  gf_range(w, lo, hi);
  const float x = h[i];
  img[i] = x != x ? (uint8_t)0 : grid_to_u8(x, lo, hi);
}

// convertTo(CV_32F, (hi - lo) / 255, lo) into every cell.
__global__ void k_gf_dequantise(const uint8_t* __restrict__ img, const unsigned* __restrict__ w, float* __restrict__ out,
                                int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float lo, hi;
  gf_range(w, lo, hi);
  out[i] = grid_from_u8(img[i], lo, hi);
}

// cv::medianBlur on CV_8U for an odd k >= 3: the exact median of the k x k window, border replicated.  Each thread walks
// GF_MED_ROWS rows down one column with the window's 256-bin histogram in shared memory (bin b of thread t at
// b * GF_MED_COLS + t): one row of k values enters and one leaves per step, and the median is the first bin where the
// running count exceeds k^2 / 2.  Counts fit 16 bits for k <= 255.
__global__ void __launch_bounds__(GF_MED_COLS) k_gf_median_u8(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                              int rows, int cols, int k) {
  __shared__ unsigned short hist[256 * GF_MED_COLS];
  const int t = threadIdx.x, c = blockIdx.x * GF_MED_COLS + t, r0 = blockIdx.y * GF_MED_ROWS;
  if (c >= cols) return;        // no barrier below: each thread owns its bins
  unsigned short* hb = hist + t;
  for (int b = 0; b < 256; b++) hb[b * GF_MED_COLS] = 0;
  const int a = k / 2, half = (k * k) / 2;
  for (int dr = -a; dr <= a; dr++) {
    const uint8_t* row = src + (long long)min(max(r0 + dr, 0), rows - 1) * cols;
    for (int dc = -a; dc <= a; dc++) hb[__ldg(row + min(max(c + dc, 0), cols - 1)) * GF_MED_COLS]++;
  }
  const int r1 = min(r0 + GF_MED_ROWS, rows);
  for (int r = r0;; r++) {
    int cum = 0, b = 0;
    for (;; b++) {
      cum += hb[b * GF_MED_COLS];
      if (cum > half) break;
    }
    dst[(long long)r * cols + c] = (uint8_t)b;
    if (r + 1 >= r1) break;
    const uint8_t* out_row = src + (long long)max(r - a, 0) * cols;
    const uint8_t* in_row = src + (long long)min(r + 1 + a, rows - 1) * cols;
    for (int dc = -a; dc <= a; dc++) {
      const int cc = min(max(c + dc, 0), cols - 1);
      hb[__ldg(out_row + cc) * GF_MED_COLS]--;
      hb[__ldg(in_row + cc) * GF_MED_COLS]++;
    }
  }
}

// grid_map's scalar_max_of_finites_op (MAX) / scalar_min_of_finites_op, restated from its published
// FunctorsPlugin.hpp: the finite operand when only one is finite, else std::max / std::min, which keep `a` on a tie or
// an unordered comparison.  maxCoeffOfFinites folds it over a block in Eigen's redux order (column-major).
template <bool MAX>
__device__ __forceinline__ float gf_finites_op(float a, float b) {
  if (isfinite(a) != isfinite(b)) return isfinite(a) ? a : b;
  return MAX ? (a < b ? b : a) : (b < a ? b : a);
}

// The column half of processing.cpp's dilate (MAX) or erode: for each cell, the fold of the finite values of in * mask
// (in alone without a mask) down the k rows of its clamped window, NaN when there is none.  Folding each column top to
// bottom and then the columns left to right visits the window in Eigen's column-major order, so where the window has a
// finite value the result is the reference's, the sign of a zero included.
template <bool MAX>
__global__ void k_gf_morph_cols(const float* __restrict__ in, const float* __restrict__ mask, float* __restrict__ tmp,
                                int rows, int cols, int k) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols, r0 = pp_corner(r, rows, k);
  float best = __int_as_float(0x7fc00000);
  for (int j = 0; j < k; j++) {
    const long long o = (long long)(r0 + j) * cols + c;
    float x = __ldg(in + o);
    if (mask) x = __fmul_rn(x, __ldg(mask + o));
    if (isfinite(x)) best = gf_finites_op<MAX>(best, x);
  }
  tmp[i] = best;
}

// The row half: the fold of the column results over the k columns of the window.  A window with no finite value folds
// its k x k cells literally (the functor on non-finite operands); the result is the cell's own value where that is NaN,
// and NaN for a NaN cell unless `inpaint`.
template <bool MAX>
__global__ void k_gf_morph_rows(const float* __restrict__ in, const float* __restrict__ mask,
                                const float* __restrict__ tmp, float* __restrict__ out, int rows, int cols, int k,
                                int inpaint) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols, c0 = pp_corner(c, cols, k);
  const float v = in[i];
  if (!inpaint && v != v) { out[i] = v; return; }
  float best = __int_as_float(0x7fc00000);
  for (int j = 0; j < k; j++) {
    const float x = __ldg(tmp + (long long)r * cols + c0 + j);
    if (x == x) best = gf_finites_op<MAX>(best, x);
  }
  if (best != best) {
    const int r0 = pp_corner(r, rows, k);
    for (int b = 0; b < k; b++)
      for (int a = 0; a < k; a++) {
        const long long o = (long long)(r0 + a) * cols + c0 + b;
        float x = __ldg(in + o);
        if (mask) x = __fmul_rn(x, __ldg(mask + o));
        best = a == 0 && b == 0 ? x : gf_finites_op<MAX>(best, x);
      }
  }
  out[i] = best != best ? v : best;
}

// processing.cpp's outline: a cell keeps its value when its clamped 3 x 3 window has a NaN, else NaN.
__global__ void k_gf_outline(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r0 = pp_corner(i / cols, rows, 3), c0 = pp_corner(i % cols, cols, 3);
  bool nan = false;
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) nan |= isnan(__ldg(in + (long long)(r0 + a) * cols + c0 + b));
  out[i] = nan ? in[i] : __int_as_float(0x7fc00000);
}
#endif
