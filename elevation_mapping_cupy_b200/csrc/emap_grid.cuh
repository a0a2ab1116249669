// emap_grid.cuh -- grid_map's index and position arithmetic on one axis, __host__ __device__ (kernel-free, so both the
// windows of emap_submap.cuh and the lookups of emap_grid_lookup.cuh include it).
//
// Restated from grid_map_core's published GridMapMath.cpp (not checked against a grid_map build), for a map whose
// buffer start index is 0.  Per axis: pos the map's position (the centre of its cells), len its length (cells * res),
// n its cells; index 0 is the +x (+y) edge.  Every operation is rounded on its own (no contraction), so the host and
// the device give the same bits.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#if defined(__CUDACC__)
#define GRID_HD __host__ __device__ __forceinline__
#else
#define GRID_HD inline
#endif

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
