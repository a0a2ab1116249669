// emap_postprocess.cuh -- the map post-processing of one segmented window (emap_planar_terrain), sm_90a.
//
// Reference: convex_plane_decomposition's Postprocessing::postprocess: addSmoothLayer (the masked layer, grid_map's
// minValues, an elliptic grey closing, grid_map_filters_rsl's applyKernelFunction with a 45 degree slope, cv::boxFilter
// and cv::GaussianBlur), dilationInNonplanarRegions and the map's addHeightOffset.  include/emap.h states the contract;
// DESIGN.md §4l the restatement.  The minValues fill is emap_planes.cuh's, the ellipse rg_ellipse_half.  The kernel
// sizes, the Gaussian coefficients and the slope offsets are host (or __host__ __device__) code so that a native test
// can check them against cv2.
#pragma once
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#include "emap_planes.cuh"

#define PP_MAX_KERNEL 63           // emap.h's EMAP_POST_MAX_KERNEL
#define PP_MAX_OFFSET 31           // emap.h's EMAP_POST_MAX_OFFSET: the non-planar ellipse is at most PP_MAX_KERNEL

// kernelSizeInPixels (Postprocessing.cpp:75-77): 2 * (int)std::round(size / res) + 1 in double (halves away from
// zero); -1 for a size that is not finite and >= 0 or a kernel above PP_MAX_KERNEL.
inline int pp_kernel_size(double size, double res) {
  if (!(std::isfinite(size) && size >= 0.0)) return -1;
  const double q = std::round(size / res);
  if (!(q <= (PP_MAX_KERNEL - 1) / 2)) return -1;
  return 2 * (int)q + 1;
}

// cv::getGaussianKernel(k, sigma, CV_32F) for odd k <= PP_MAX_KERNEL: with sigma <= 0 OpenCV's fixed tables up to
// k = 9, else exp(-x^2 / (2 sigma^2)) with sigma = 0.3 ((k - 1) / 2 - 1) + 0.8 when sigma <= 0, scaled by 1 / its sum,
// in double, rounded to float.
inline void pp_gauss_coeffs(int k, float* out, double sigma = 0.0) {
  static const float t1[] = {1.f}, t3[] = {0.25f, 0.5f, 0.25f}, t5[] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f},
                     t7[] = {0.03125f, 0.109375f, 0.21875f, 0.28125f, 0.21875f, 0.109375f, 0.03125f},
                     t9[] = {4 / 256.f, 13 / 256.f, 30 / 256.f, 51 / 256.f, 60 / 256.f, 51 / 256.f, 30 / 256.f,
                             13 / 256.f, 4 / 256.f};
  const float* tab[] = {t1, t3, t5, t7, t9};
  if (k <= 9 && !(sigma > 0.0)) {
    for (int i = 0; i < k; i++) out[i] = tab[k / 2][i];
    return;
  }
  if (!(sigma > 0.0)) sigma = ((k - 1) * 0.5 - 1) * 0.3 + 0.8;
  const double scale2x = -0.5 / (sigma * sigma);
  double w[PP_MAX_KERNEL], sum = 0.0;
  for (int i = 0; i < k; i++) {
    const double x = i - (k - 1) * 0.5;
    w[i] = std::exp(scale2x * x * x);
    sum += w[i];
  }
  const double s = 1.0 / sum;
  for (int i = 0; i < k; i++) out[i] = (float)(w[i] * s);
}

// The sloped dilation's offset at window row dy, column dx from the centre: float slope times std::sqrt of the int
// dx^2 + dy^2, in double, rounded to float (Postprocessing.cpp:116-125).
PL_HD float pp_slope_offset(float slope, int dy, int dx) {
  return (float)((double)slope * sqrt((double)(dx * dx + dy * dy)));
}

// A MORPH_ELLIPSE of size 2 r + 1 as rg_ellipse_half's row half widths.
struct PpEllipse {
  int r;
  int half[PP_MAX_KERNEL];
};

// The Gaussian's k = 2 h + 1 coefficients, c[h] the centre.
struct PpGauss {
  int h;
  float c[PP_MAX_KERNEL];
};

#if defined(__CUDACC__)
// Every pass reads the header word hdr[0] (the window has a finite cell) and writes nothing when it is 0, so that a
// window without a finite cell leaves the layers unwritten while the launches stay the same.  Reads are border
// replicated (clamped) like BORDER_REPLICATE.

__device__ __forceinline__ int pp_clamp(int v, int hi) { return min(max(v, 0), hi); }

// grid_map_filters_rsl's window corner on one axis of n cells (processing.cpp:37-48): max(v - (k - 1) / 2, 0), pulled
// back to n - k where the window would overshoot.  n >= k (checked on the host).
__device__ __forceinline__ int pp_corner(int v, int n, int k) {
  const int c = max(v - (k - 1) / 2, 0);
  return c + k > n ? n - k : c;
}

// cv::borderInterpolate(v, hi + 1, BORDER_REFLECT_101): reflected about the edge cells, as often as needed.
__device__ __forceinline__ int pp_reflect101(int v, int hi) {
  if (hi == 0) return 0;
  while (v < 0 || v > hi) v = v < 0 ? -v : 2 * hi - v;
  return v;
}

// The index of row or column v of an axis of hi + 1 cells: border replicated (clamped), or BORDER_REFLECT_101.
template <bool REFLECT>
__device__ __forceinline__ int pp_border(int v, int hi) { return REFLECT ? pp_reflect101(v, hi) : pp_clamp(v, hi); }

// elevationWithNaN = plane_classification == 1 ? elevation : NaN (layers 1 and 3 of lay) into the fill's input a and
// into layer 4.
__global__ void k_pp_mask(const float* __restrict__ lay, float* __restrict__ a, float* __restrict__ out,
                          const int* __restrict__ hdr, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = lay[3 * n + i] == 1.0f ? lay[n + i] : __int_as_float(0x7fc00000);
  a[i] = v;
  if (hdr[0]) out[i] = v;
}

// Grey dilation (MAX) or erosion by the ellipse e, border replicated; copy != nullptr also receives src.
template <bool MAX>
__global__ void k_pp_morph(const float* __restrict__ src, float* __restrict__ dst, float* __restrict__ copy,
                           const int* __restrict__ hdr, int rows, int cols, const __grid_constant__ PpEllipse e) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || !hdr[0]) return;
  const int r = i / cols, c = i - r * cols;
  float v = src[i];
  for (int dr = -e.r; dr <= e.r; dr++) {
    const float* row = src + (long long)pp_clamp(r + dr, rows - 1) * cols;
    const int w = e.half[dr + e.r];
    for (int dc = -w; dc <= w; dc++) {
      const float x = __ldg(row + pp_clamp(c + dc, cols - 1));
      v = MAX ? fmaxf(v, x) : fminf(v, x);
    }
  }
  dst[i] = v;
  if (copy) copy[i] = src[i];
}

// applyKernelFunction(k, (data - offsets).maxCoeffOfFinites()) (processing.cpp:145-177): the k x k window's corner is
// max(cell - h, 0), pulled back to rows - k (cols - k) when the window would overshoot, so cells within h of the edge
// use a window that is not centred on them, with the offsets of its own cells.  The max over the finite differences
// (fp32), NaN when there is none.  rows, cols >= k (checked on the host).
__global__ void k_pp_slope(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ hdr, int rows,
                           int cols, int k, float slope) {
  __shared__ float off[PP_MAX_KERNEL * PP_MAX_KERNEL];
  const int h = (k - 1) / 2;
  for (int t = threadIdx.x; t < k * k; t += blockDim.x) off[t] = pp_slope_offset(slope, t / k - h, t % k - h);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || !hdr[0]) return;
  const int r0 = pp_corner(i / cols, rows, k), c0 = pp_corner(i % cols, cols, k);
  float best = __int_as_float(0x7fc00000);
  bool any = false;
  for (int a = 0; a < k; a++) {
    const float* row = src + (long long)(r0 + a) * cols + c0;
    for (int b = 0; b < k; b++) {
      const float x = __fsub_rn(__ldg(row + b), off[a * k + b]);
      if (isfinite(x)) {
        best = any ? fmaxf(best, x) : x;
        any = true;
      }
    }
  }
  dst[i] = best;
}

// cv::boxFilter's sums in double (exact for fp32 values within 29 binary orders of magnitude of each other, so the
// order does not matter): ROWS sums the k cells c - k / 2 .. c - k / 2 + k - 1 of the row into rs, left to right; the
// column pass sums 2 h + 1 of those and rounds sum * scale (OpenCV's double 1 / k^2) to float.  The border is
// replicated, or BORDER_REFLECT_101 with REFLECT (emap_grid_filter's cv::blur row sums for k <= 5).
template <bool REFLECT = false>
__global__ void k_pp_box_rows(const float* __restrict__ src, double* __restrict__ rs, const int* __restrict__ hdr,
                              int rows, int cols, int k) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || !hdr[0]) return;
  const int r = i / cols, c = i - r * cols;
  const float* row = src + (long long)r * cols;
  double s = 0.0;
  for (int d = -(k / 2); d < k - k / 2; d++) s += (double)__ldg(row + pp_border<REFLECT>(c + d, cols - 1));
  rs[i] = s;
}

__global__ void k_pp_box_cols(const double* __restrict__ rs, float* __restrict__ dst, const int* __restrict__ hdr,
                              int rows, int cols, int h, double scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || !hdr[0]) return;
  const int r = i / cols, c = i - r * cols;
  double s = 0.0;
  for (int d = -h; d <= h; d++) s += __ldg(rs + (long long)pp_clamp(r + d, rows - 1) * cols + c);
  dst[i] = (float)__dmul_rn(s, scale);
}

// One pass of the separable Gaussian, along the row (ROW) or the column: s = c[h] x0, then s += c[h + j] (x+j + x-j)
// for j = 1 .. h, each operation rounded to fp32 on its own (no contraction).  Bit-identical to cv::GaussianBlur for
// k = 3 (rows first); DESIGN.md §4l states the bound for longer kernels.  The border is replicated, or BORDER_REFLECT_101
// (cv::GaussianBlur's default, emap_grid_filter) with REFLECT.
template <bool ROW, bool REFLECT = false>
__global__ void k_pp_gauss(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ hdr, int rows,
                           int cols, const __grid_constant__ PpGauss g) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || !hdr[0]) return;
  const int r = i / cols, c = i - r * cols;
  float s = __fmul_rn(g.c[g.h], src[i]);
  for (int j = 1; j <= g.h; j++) {
    const float a = ROW ? __ldg(src + (long long)r * cols + pp_border<REFLECT>(c + j, cols - 1))
                        : __ldg(src + (long long)pp_border<REFLECT>(r + j, rows - 1) * cols + c);
    const float b = ROW ? __ldg(src + (long long)r * cols + pp_border<REFLECT>(c - j, cols - 1))
                        : __ldg(src + (long long)pp_border<REFLECT>(r - j, rows - 1) * cols + c);
    s = __fadd_rn(s, __fmul_rn(g.c[g.h + j], __fadd_rn(a, b)));
  }
  dst[i] = s;
}

// The post-processed elevation (layer 9) from layers 1 (E) and 3 (M) of lay, in fp32 as Eigen evaluates it:
// dilationInNonplanarRegions (dil: E = M E + (1 - M) D, D the grey dilation), then addHeightOffset (add_on: E += add,
// then sub_on: E -= sub M).
struct PpFinal {
  int dil, add_on, sub_on;
  float add, sub;
};

__global__ void k_pp_final(const float* __restrict__ lay, const float* __restrict__ dilated, float* __restrict__ out,
                           const int* __restrict__ hdr, int n, PpFinal f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !hdr[0]) return;
  const float e = lay[n + i], m = lay[3 * n + i];
  float v = e;
  if (f.dil) v = __fadd_rn(__fmul_rn(m, e), __fmul_rn(__fsub_rn(1.0f, m), dilated[i]));
  if (f.add_on) {
    v = __fadd_rn(v, f.add);
    if (f.sub_on) v = __fsub_rn(v, __fmul_rn(f.sub, m));
  }
  out[i] = v;
}
#endif
