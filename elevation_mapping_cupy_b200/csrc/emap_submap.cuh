// emap_submap.cuh -- windows of the exported map (emap_get_submaps), sm_90a.
//
// Reference: the ROS node's get_raw_submap service (elevation_mapping_ros.cpp:507-553), which crops grid_map's copy of
// the exported layers (WRAP:213-252, EM.py:720-775) with GridMap::getSubmap.  Here the window arithmetic runs on the
// host (submap_window) and k_submap writes every (window, layer, row) of a batch in one launch, straight from the
// state planes, with the cell values of k_export_multi (export_cell).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#define SUBMAP_MAX_WINDOWS 1024
#define SUBMAP_ROWS 8              // output rows per work item: one warp per row

// One successful window of a call.  r0, c0: state row / column of the window's output cell (0, 0) (rows and columns
// run the other way in the state: output (rr, cc) is state (r0 - rr, c0 - cc)).  tile0: its first work item; off: its
// first output float (its layers follow one another, each rows x cols, row-major).
struct SubmapWin {
  int16_t r0, c0, rows, cols;
  int32_t tile0;
  long long off;
};
static_assert(sizeof(SubmapWin) == 24, "SubmapWin is packed into the kernel parameters");

// The whole table travels as kernel parameters (__grid_constant__: read in place from the parameter bank, which every
// thread of a CTA reads at the same address): no upload, no staging buffer, and a captured graph keeps its own copy.
struct SubmapArgs {
  int n_win;                   // successful windows, in call order
  ExportList L;
  SubmapWin win[SUBMAP_MAX_WINDOWS];
};
static_assert(sizeof(SubmapArgs) <= 32764, "kernel parameters are limited to 32764 bytes");

// EM.py's transform_to_map_index on one axis, in double: the state index floor((p - m) / res + cell_n / 2).  Cells are
// half-open: a coordinate on a boundary belongs to the cell above it (larger x or y, smaller output index).
inline double submap_axis_index(double p, double m, double res, int cell_n) {
  return std::floor((p - m) / res + 0.5 * cell_n);
}

// The window of one request (position_x, position_y, length_x, length_y) on the exported map: the (cell_n - 2)^2
// interior, flipped on both axes (output row 0 is the +x edge, column 0 the +y edge).  The window is the inclusive cell
// rectangle between the cell holding position + length / 2 and the cell holding position - length / 2, each clipped to
// the exported area.  It fails (info[0] = 0, everything else 0, centre NaN) when the position's own cell is outside it.
// info = {success, row0, col0, rows, cols}; centre = the centre of the window's cells, in the map frame.  The lengths
// must be finite and >= 0 (the caller checks).
inline void submap_window(int cell_n, double res, const double m[2], const double req[4], int32_t info[5],
                          double centre[2]) {
  const double lo = 1.0, hi = cell_n - 2.0;
  for (int a = 0; a < 2; a++) {
    const double i = submap_axis_index(req[a], m[a], res, cell_n);
    if (!(i >= lo && i <= hi)) {                     // outside, or not a number
      for (int k = 0; k < 5; k++) info[k] = 0;
      centre[0] = centre[1] = std::nan("");
      return;
    }
  }
  info[0] = 1;
  for (int a = 0; a < 2; a++) {
    const double half = 0.5 * req[2 + a];
    const int32_t top = (int32_t)std::min(std::max(submap_axis_index(req[a] + half, m[a], res, cell_n), lo), hi);
    const int32_t bot = (int32_t)std::min(std::max(submap_axis_index(req[a] - half, m[a], res, cell_n), lo), hi);
    info[1 + a] = cell_n - 2 - top;
    info[3 + a] = top - bot + 1;
    centre[a] = m[a] + (0.5 * (top + bot + 1) - 0.5 * cell_n) * res;
  }
}

// One CTA per (window row tile, layer): warp y writes output row SUBMAP_ROWS * tile + y of the window, lane by lane
// along the row.  Lane k reads state column c0 - k: the warp's 32 addresses are the same 128-byte span as a forward
// read, and the memory system coalesces by address, not by lane order, so neither reads nor writes need staging.
template <bool COLOUR>
__global__ void __launch_bounds__(32 * SUBMAP_ROWS)
k_submap(const DevCfg c, const float* __restrict__ map, const float* __restrict__ normal, float* __restrict__ out,
         const __grid_constant__ SubmapArgs a, float center_z, int only_above) {
  const int t = blockIdx.x, l = blockIdx.y;
  int lo = 0, hi = a.n_win - 1;                      // the last window whose first item is <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.win[mid].tile0 <= t) lo = mid; else hi = mid - 1;
  }
  const SubmapWin& w = a.win[lo];
  const int rows = w.rows, cols = w.cols;
  const int rr = (t - w.tile0) * SUBMAP_ROWS + (int)threadIdx.y;
  if (rr >= rows) return;
  const int kind = a.L.kind[l], flags = a.L.flags[l];
  const float* plane = a.L.plane[l];
  float* dst = out + w.off + ((long long)l * rows + rr) * cols;
  const int sr = w.r0 - rr;
  for (int cc = (int)threadIdx.x; cc < cols; cc += 32)
    dst[cc] = export_cell<COLOUR>(c, map, normal, sr, w.c0 - cc, kind, center_z, only_above, plane, flags);
}
