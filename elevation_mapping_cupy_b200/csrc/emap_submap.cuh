// emap_submap.cuh -- windows of the exported map (emap_get_submaps) and in a requester's frame
// (emap_get_transformed_submaps), sm_90a.
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

#include "emap_export.cuh"
#include "emap_grid.cuh"

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

// ---- windows in the requester's frame (emap_get_transformed_submaps) -----------------------------------------------
// The node's get_raw_submap with a frame_id other than the map frame: the window of T^-1 * position, then grid_map's
// GridMap::getTransformedMap(T, "elevation", frame_id) on it, restated from grid_map's published source (not checked
// against a grid_map build; include/emap.h states every step).  T = (R row-major, t) maps map-frame points into the
// request frame.  The host part (transformed_window) is handle-free; the device part is three passes over the batch.

#define TSUB_MAX_WINDOWS 128       // windows per launch: the table travels in the kernels' parameters
#define TSUB_THREADS 256
#define TSUB_ORTHO_TOL 1e-6        // |R^T R - I| per entry

// q = R p + t in double, per component ((R_k0 x + R_k1 y) + R_k2 z) + t_k (t NULL: R p alone): Eigen's Matrix3d and
// Isometry3d products on x86-64 SSE2.  The host compiler targets plain x86-64 (no FMA instructions), so nothing is
// contracted here.
inline void tsub_apply(const double R[9], const double* t, const double p[3], double q[3]) {
  for (int k = 0; k < 3; k++) {
    q[k] = (R[3 * k] * p[0] + R[3 * k + 1] * p[1]) + R[3 * k + 2] * p[2];
    if (t) q[k] += t[k];
  }
}

// Whether T = (R row-major, t) is finite and R orthonormal within TSUB_ORTHO_TOL.
inline bool tsub_transform_ok(const double T[12]) {
  for (int k = 0; k < 12; k++)
    if (!std::isfinite(T[k])) return false;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      const double d = T[i] * T[j] + T[3 + i] * T[3 + j] + T[6 + i] * T[6 + j] - (i == j ? 1.0 : 0.0);
      if (!(std::fabs(d) <= TSUB_ORTHO_TOL)) return false;
    }
  return true;
}

// One request's geometry.  win / centre: the map-frame window of submap_window (info {success, row0, col0, rows, cols})
// at the map-frame position; pos / len / size: the new map in the request frame (centre, length, rows and cols).
struct TSubGeom {
  int32_t win[5];
  double centre[2];
  double pos[2], len[2];
  int32_t size[2];
};

// req = (position_x, position_y) in the request frame and (length_x, length_y); T as tsub_transform_ok accepts it.
// 1. The map-frame position is T^-1 (px, py, 0) with Eigen's Isometry3d::inverse(): R' = R^T, t' = -(R' t).
// 2. The window is submap_window's at that position and the given length; failed: size 0, pos and len NaN.
// 3. Its corners (c +- L/2) with L = (rows, cols) * res, in the order (+,+), (+,-), (-,+), (-,-), go through T; the
//    new centre is 0.25 * their sum (in that order), the new length 2 * max |corner - centre| per axis, and
//    setGeometry gives size = round(length / res) (half away from zero), length = size * res.
inline void transformed_window(int cell_n, double res, const double m[2], const double req[4], const double T[12],
                               TSubGeom& g) {
  const double* R = T;
  const double Ri[9] = {R[0], R[3], R[6], R[1], R[4], R[7], R[2], R[5], R[8]};
  const double p[3] = {req[0], req[1], 0.0};
  double ti[3], mp[3];
  tsub_apply(Ri, nullptr, T + 9, ti);
  for (int k = 0; k < 3; k++) ti[k] = -ti[k];
  tsub_apply(Ri, ti, p, mp);
  const double mreq[4] = {mp[0], mp[1], req[2], req[3]};
  submap_window(cell_n, res, m, mreq, g.win, g.centre);
  if (!g.win[0]) {
    g.pos[0] = g.pos[1] = g.len[0] = g.len[1] = std::nan("");
    g.size[0] = g.size[1] = 0;
    return;
  }
  const double hx = g.win[3] * res * 0.5, hy = g.win[4] * res * 0.5;
  const double cx = g.centre[0], cy = g.centre[1];
  const double corner[4][3] = {{cx + hx, cy + hy, 0.0}, {cx + hx, cy - hy, 0.0}, {cx - hx, cy + hy, 0.0},
                               {cx - hx, cy - hy, 0.0}};
  double e[4][3], c[3] = {0.0, 0.0, 0.0};
  for (int k = 0; k < 4; k++) {
    tsub_apply(R, T + 9, corner[k], e[k]);
    for (int a = 0; a < 3; a++) c[a] += e[k][a];
  }
  for (int a = 0; a < 2; a++) {
    c[a] *= 0.25;
    double half = 0.0;
    for (int k = 0; k < 4; k++) half = std::fmax(std::fabs(e[k][a] - c[a]), half);
    g.size[a] = (int32_t)std::round(2.0 * half / res);
    g.pos[a] = c[a];
    g.len[a] = g.size[a] * res;
  }
}

// One window of a launch.  x0, y0: map-frame position of the map-frame window's cell (0, 0) (grid_map's
// getPositionFromIndex: (c + (0.5 L - 0.5 res)) per axis; cell (r, c) is at x0 - res r, y0 - res c); r0, c0: its state
// row / column (output (rr, cc) is state (r0 - rr, c0 - cc)); rows, cols: its size; pos, len, nrows, ncols: the new
// map; blk_src / blk_dst: the first block of the window in the scatter passes / in k_tsub_gather; cell0: its first key
// and output cell (its output starts at float n_layers * cell0, layer after layer, each nrows x ncols row-major).
struct TSubWin {
  double R[9], t[3];
  double x0, y0;
  double pos[2], len[2];
  int16_t r0, c0, rows, cols;
  int32_t nrows, ncols;
  int32_t blk_src, blk_dst;
  long long cell0;
};
static_assert(sizeof(TSubWin) == 176, "TSubWin is packed into the kernel parameters");

struct TSubArgs {
  int n_win;                   // windows of this launch, in call order
  int n_samples;               // 1, or 5 with sample_ratio > 0
  double res, s;               // resolution, res * sample_ratio
  ExportList L;
  TSubWin win[TSUB_MAX_WINDOWS];
};
static_assert(sizeof(TSubArgs) <= 32764, "kernel parameters are limited to 32764 bytes");

// The window of block b: the last whose first block (field F) is <= b.
template <int32_t TSubWin::*F>
__device__ __forceinline__ const TSubWin& tsub_window(const TSubArgs& a, int b) {
  int lo = 0, hi = a.n_win - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.win[mid].*F <= b) lo = mid; else hi = mid - 1;
  }
  return a.win[lo];
}

// Order-preserving 32-bit key of a float (0 is below every float's key: "nothing here").
__device__ __forceinline__ u32 tsub_fkey(float f) {
  const u32 u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float tsub_funkey(u32 k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Sample k of window cell (row, col) with exported elevation h, through T, in double with every operation rounded
// on its own (no contraction): p = (x, y, h), then for k = 1..4 (x - s, y), (x + s, y), (x, y - s), (x, y + s).
// Returns its key / output cell, or -1 when (q.x, q.y) is outside the new map (grid_axis_index: checkIfPositionWithinMap
// and getIndexFromPosition).
__device__ __forceinline__ long long tsub_sample(const TSubWin& w, const TSubArgs& a, int row, int col, double h, int k,
                                                 double& qz) {
  double p[3] = {__dadd_rn(w.x0, -__dmul_rn(a.res, (double)row)), __dadd_rn(w.y0, -__dmul_rn(a.res, (double)col)), h};
  if (k) {
    const double d = (k & 1) ? -a.s : a.s;
    p[0] = __dadd_rn(p[0], k <= 2 ? d : 0.0);
    p[1] = __dadd_rn(p[1], k <= 2 ? 0.0 : d);
    p[2] = __dadd_rn(p[2], 0.0);
  }
  double q[3];
#pragma unroll
  for (int r = 0; r < 3; r++)
    q[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(w.R[3 * r], p[0]), __dmul_rn(w.R[3 * r + 1], p[1])),
                               __dmul_rn(w.R[3 * r + 2], p[2])), w.t[r]);
  qz = q[2];
  int idx[2];
#pragma unroll
  for (int ax = 0; ax < 2; ax++)
    if (!grid_axis_index(q[ax], w.pos[ax], w.len[ax], a.res, ax ? w.ncols : w.nrows, idx[ax])) return -1;
  return w.cell0 + (long long)idx[0] * w.ncols + idx[1];
}

// The scatter passes, one thread per map-frame window cell (lanes along its columns), over its samples.  grid_map
// visits the cells column-major (i = col * rows + row) and, per cell, its samples in order: sample j = n_samples i + k.
// A target's final elevation is M = max F(z) over the samples that reach it (F: rounding to fp32), and its winner is
// the largest j with z >= M (in double) if there is one, else the smallest j with F(z) = M.
//   PASS 1: key1 = atomicMax of tsub_fkey(F(z));
//   PASS 2: for samples with F(z) = M, key2 = atomicMax of z >= M ? 2^40 + j : 2^40 - 1 - j.
// Cells whose exported elevation is NaN have no samples.
template <int PASS>
__global__ void __launch_bounds__(TSUB_THREADS)
k_tsub_scatter(const DevCfg c, const float* __restrict__ map, u32* __restrict__ key1, u64* __restrict__ key2,
               const __grid_constant__ TSubArgs a, float center_z) {
  const TSubWin& w = tsub_window<&TSubWin::blk_src>(a, blockIdx.x);
  const int rows = w.rows, cols = w.cols;
  const int t = (blockIdx.x - w.blk_src) * TSUB_THREADS + threadIdx.x;
  if (t >= rows * cols) return;
  const int row = t / cols, col = t - row * cols;
  const float h = export_cell(c, map, nullptr, w.r0 - row, w.c0 - col, 0, center_z, 0, nullptr, 0);
  if (isnan(h)) return;
  const long long i = (long long)col * rows + row;
  for (int k = 0; k < a.n_samples; k++) {
    double z;
    const long long cell = tsub_sample(w, a, row, col, (double)h, k, z);
    if (cell < 0) continue;
    const float f = __double2float_rn(z);
    if (PASS == 1) {
      atomicMax(&key1[cell], tsub_fkey(f));
    } else if (tsub_fkey(f) == key1[cell]) {
      const u64 j = (u64)(a.n_samples * i + k), top = 1ull << 40;
      atomicMax(&key2[cell], z >= (double)f ? top + j : top - 1 - j);
    }
  }
}

// The gather pass, one thread per new-map cell (lanes along its columns): every layer of the winner's source cell
// through export_cell, the elevation layer F(z) of the winning sample, NaN everywhere where nothing won.  Resets the
// cell's keys, so the scratch is zero again for the next call.
template <bool COLOUR>
__global__ void __launch_bounds__(TSUB_THREADS)
k_tsub_gather(const DevCfg c, const float* __restrict__ map, const float* __restrict__ normal, u32* __restrict__ key1,
              u64* __restrict__ key2, float* __restrict__ out, const __grid_constant__ TSubArgs a, float center_z,
              int only_above) {
  const TSubWin& w = tsub_window<&TSubWin::blk_dst>(a, blockIdx.x);
  const int n = w.nrows * w.ncols;
  const int t = (blockIdx.x - w.blk_dst) * TSUB_THREADS + threadIdx.x;
  if (t >= n) return;
  const long long cell = w.cell0 + t;
  const u32 k1 = key1[cell];
  const u64 k2 = key2[cell];
  key1[cell] = 0;
  key2[cell] = 0;
  float* dst = out + (long long)a.L.n * w.cell0 + t;
  if (!k2) {
    for (int l = 0; l < a.L.n; l++) dst[(long long)l * n] = __int_as_float(0x7fc00000);
    return;
  }
  const u64 top = 1ull << 40;
  const long long i = (long long)(k2 >= top ? k2 - top : top - 1 - k2) / a.n_samples;
  const int col = (int)(i / w.rows), row = (int)(i - (long long)col * w.rows);
  const int sr = w.r0 - row, sc = w.c0 - col;
  const float elevation = tsub_funkey(k1);
  for (int l = 0; l < a.L.n; l++) {
    const int kind = a.L.kind[l];
    dst[(long long)l * n] = kind == 0 ? elevation
                                      : export_cell<COLOUR>(c, map, normal, sr, sc, kind, center_z, only_above,
                                                            a.L.plane[l], a.L.flags[l]);
  }
}
