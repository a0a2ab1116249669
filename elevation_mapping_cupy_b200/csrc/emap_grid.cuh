// emap_grid.cuh -- grid_map's index and position arithmetic on one axis, __host__ __device__, and the check of a caller's
// grid (kernel-free, so the windows of emap_submap.cuh, the lookups of emap_grid_lookup.cuh and the plane decomposition
// of a grid in emap_export_api.cu include it).
//
// Restated from grid_map_core's published GridMapMath.cpp (not checked against a grid_map build), for a map whose
// buffer start index is 0.  Per axis: pos the map's position (the centre of its cells), len its length (cells * res),
// n its cells; index 0 is the +x (+y) edge.  Every operation is rounded on its own (no contraction), so the host and
// the device give the same bits.
#pragma once
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#if defined(__CUDACC__)
#define GRID_HD __host__ __device__ __forceinline__
#else
#define GRID_HD inline
#endif

#define GL_MAX_EXTENT 1048576.0    // emap.h's EMAP_GRID_MAX_EXTENT: |position| + length per axis, 2^20 m
#define GL_MIN_RES 9.5367431640625e-07   // emap.h's EMAP_GRID_MIN_RESOLUTION, 2^-20 m

#if defined(__CUDA_ARCH__)
#define GRID_ADD(a, b) __dadd_rn((a), (b))
#define GRID_MUL(a, b) __dmul_rn((a), (b))
#define GRID_DIV(a, b) __ddiv_rn((a), (b))
#define GRID_TRUNC(a) __double2int_rz((a))
#else
#define GRID_ADD(a, b) ((double)(a) + (double)(b))
#define GRID_MUL(a, b) ((double)(a) * (double)(b))
#define GRID_DIV(a, b) ((double)(a) / (double)(b))
#define GRID_TRUNC(a) ((int)(a))
#endif

// checkIfPositionWithinMap and getIndexFromPosition on one axis: with o = 0.5 len, q is inside when
// 0 <= -((q - pos) - o) < len; its index is then trunc(-(((q - o) - pos) / res)), clamped to [0, n - 1].  Returns
// whether q is inside; idx is written only then.
GRID_HD bool grid_axis_index(double q, double pos, double len, double res, int n, int& idx) {
  const double o = GRID_MUL(0.5, len);
  const double u = -GRID_ADD(GRID_ADD(q, -pos), -o);
  if (!(u >= 0.0 && u < len)) return false;
  const int i = GRID_TRUNC(-GRID_DIV(GRID_ADD(GRID_ADD(q, -o), -pos), res));
  idx = i < 0 ? 0 : i > n - 1 ? n - 1 : i;
  return true;
}

// getPositionFromIndex on one axis: (pos + (0.5 len - 0.5 res)) - res i; origin = the position of index 0.
GRID_HD double grid_axis_origin(double pos, double len, double res) {
  return GRID_ADD(pos, GRID_ADD(GRID_MUL(0.5, len), -GRID_MUL(0.5, res)));
}
GRID_HD double grid_axis_at(double origin, double res, int64_t i) { return GRID_ADD(origin, -GRID_MUL(res, (double)i)); }
GRID_HD double grid_axis_position(double pos, double len, double res, int64_t i) {
  return grid_axis_at(grid_axis_origin(pos, len, res), res, i);
}

// grid_map_cv's toImage<uchar, 1>(lo, hi) of one non-NaN cell: clamped to [lo, hi] and (uchar)(((v - lo) / (hi - lo)) *
// 255.0f) in float, truncated, a NaN quotient giving 0 (x86's conversion).  emap_nonlinear_interpolation and
// emap_grid_filter's 8-bit median quantise with it.
#if defined(__CUDACC__)
__device__ __forceinline__ uint8_t grid_to_u8(float x, float lo, float hi) {
  x = x < lo ? lo : (x > hi ? hi : x);
  const float r = __fmul_rn(__fdiv_rn(__fsub_rn(x, lo), __fsub_rn(hi, lo)), 255.0f);
  return (r == r) ? (uint8_t)(int)r : (uint8_t)0;
}

// convertTo(CV_32F, (hi - lo) / 255, lo) of one 8-bit value: a fused multiply-add, as cv::Mat::convertTo's x86 path.
__device__ __forceinline__ float grid_from_u8(uint8_t u, float lo, float hi) {
  return __fmaf_rn((float)u, __fdiv_rn(__fsub_rn(hi, lo), 255.0f), lo);
}
#endif

// The grids the calls accept (min_cells: the fewest rows and columns): nullptr, or why not.  Within these bounds a
// projected line end is always inside the map (include/emap.h).
inline const char* gl_check_grid(const float* data, int64_t rows, int64_t cols, const double pos[2], double res,
                                 int64_t min_cells) {
  if (!data) return "null grid data";
  if (rows < min_cells || cols < min_cells)
    return min_cells > 1 ? "rows and cols must be >= 5" : "rows and cols must be >= 1";
  if (rows > INT32_MAX || cols > INT32_MAX || rows * cols > INT32_MAX) return "rows * cols must be below 2^31";
  if (!(std::isfinite(res) && res >= GL_MIN_RES)) return "resolution must be finite and >= EMAP_GRID_MIN_RESOLUTION";
  for (int a = 0; a < 2; a++) {
    if (!std::isfinite(pos[a])) return "position must be finite";
    if (!(std::fabs(pos[a]) + (double)(a ? cols : rows) * res <= GL_MAX_EXTENT))
      return "|position| + length must be at most EMAP_GRID_MAX_EXTENT";
  }
  return nullptr;
}
