// emap_values_at.cuh -- layer values at points (emap_grid_values_at, emap_map_values_at), sm_90a: grid_map's
// GridMap::atPosition with nearest, linear and cubic-convolution interpolation, for a batch of points and up to 24 layers
// of one geometry.
//
// Restated from grid_map_core's published GridMap.cpp (atPosition, atPositionLinearInterpolated) and
// CubicInterpolation.cpp (bicubic_conv), not checked against a grid_map build; include/emap.h states the rule and its
// one operation order.  The per-point functions are __host__ __device__: the kernel runs them one thread per point, and
// tests/native/values_at_host.cpp runs them on the CPU with the same arithmetic, so the two give the same bits.  The
// point's plan (status, corner cell, weights) is computed once; va_value then combines the 1, 4 or 16 cells of one layer,
// read through the source's at(layer, row, col): a grid (VaGridSrc) or the live map's exported cells (emap_export_api.cu).
#pragma once
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "emap_grid.cuh"

#define VA_THREADS 256             // points per block of k_values_at
#define VA_MAX_LAYERS 24           // emap.h's EMAP_VALUES_MAX_LAYERS

enum { VA_NEAREST = 0, VA_LINEAR = 1, VA_CUBIC = 2 };                             // methods, emap.h's EMAP_VALUES_*
enum { VA_OUT = 0, VA_BY_NEAREST = 1, VA_BY_LINEAR = 2, VA_BY_CUBIC = 3 };        // statuses, emap.h's EMAP_VALUE_*

#if defined(__CUDA_ARCH__)
#define VA_D2F(a) __double2float_rn((a))
#define VA_LDG(p) __ldg((p))
#else
#define VA_D2F(a) ((float)(a))
#define VA_LDG(p) (*(p))
#endif

// The quiet NaN every NaN value is written as (the device and the host give NaNs different payloads)
GRID_HD float va_nan() {
#if defined(__CUDA_ARCH__)
  return __int_as_float(0x7fc00000);
#else
  const uint32_t u = 0x7fc00000u;
  float f;
  memcpy(&f, &u, sizeof f);
  return f;
#endif
}

// The geometry every layer of a call shares: rows x cols cells, position pos (the centre of its cells), length len =
// (rows, cols) res, buffer start index 0 (emap_grid.cuh's arithmetic).
struct VaGeom {
  int rows, cols;
  double pos[2], len[2], res;
};

// One point's plan: status (the method that produces its value); nearest: its cell (r, c); linear and cubic: the corner
// of lowest x and y (r, c) = (r0, c0), and per axis the weights wx, wy: linear {1 - t, t}, cubic the four convolution
// weights of f(-1) .. f(2).
struct VaPoint {
  int status, r, c;
  double wx[4], wy[4];
};

// The 1-D cubic-convolution weights at t (Keys, a = -0.5; grid_map's bicubic_conv matrix M):
// w_j = 0.5 ((((M0j + M1j t) + M2j t^2) + M3j t^3)), t^2 = t t, t^3 = t^2 t.
GRID_HD void va_cubic_weights(double t, double w[4]) {
  const double M[4][4] = {{0.0, 2.0, 0.0, 0.0}, {-1.0, 0.0, 1.0, 0.0}, {2.0, -5.0, 4.0, -1.0}, {-1.0, 3.0, -3.0, 1.0}};
  const double t2 = GRID_MUL(t, t), t3 = GRID_MUL(t2, t);
#pragma unroll
  for (int j = 0; j < 4; j++)
    w[j] = GRID_MUL(0.5, GRID_ADD(GRID_ADD(GRID_ADD(M[0][j], GRID_MUL(M[1][j], t)), GRID_MUL(M[2][j], t2)),
                                  GRID_MUL(M[3][j], t3)));
}

// The plan of point (x, y) for `method` (include/emap.h): outside (or a NaN coordinate) -> VA_OUT; the point's cell
// (r, c); linear needs the neighbours r' (r - 1 when x >= X(r), else r + 1) and c' inside, cubic rows r0 + 1 .. r0 - 2
// and columns c0 + 1 .. c0 - 2 with r0 = max(r, r'), c0 = max(c, c'); each falls back to the method below it.
GRID_HD void va_plan(const VaGeom& g, int method, double x, double y, VaPoint& p) {
  int r = 0, c = 0;
  if (!grid_axis_index(x, g.pos[0], g.len[0], g.res, g.rows, r) ||
      !grid_axis_index(y, g.pos[1], g.len[1], g.res, g.cols, c)) {
    p.status = VA_OUT;
    p.r = p.c = 0;
    return;
  }
  p.status = VA_BY_NEAREST;
  p.r = r;
  p.c = c;
  if (method == VA_NEAREST) return;
  const double xr = grid_axis_position(g.pos[0], g.len[0], g.res, r);
  const double yc = grid_axis_position(g.pos[1], g.len[1], g.res, c);
  const int rn = x >= xr ? r - 1 : r + 1, cn = y >= yc ? c - 1 : c + 1;
  if (rn < 0 || rn >= g.rows || cn < 0 || cn >= g.cols) return;
  const int r0 = r > rn ? r : rn, c0 = c > cn ? c : cn;
  const double tx = GRID_DIV(GRID_ADD(x, -grid_axis_position(g.pos[0], g.len[0], g.res, r0)), g.res);
  const double ty = GRID_DIV(GRID_ADD(y, -grid_axis_position(g.pos[1], g.len[1], g.res, c0)), g.res);
  p.r = r0;
  p.c = c0;
  if (method == VA_CUBIC && r0 + 1 < g.rows && r0 - 2 >= 0 && c0 + 1 < g.cols && c0 - 2 >= 0) {
    p.status = VA_BY_CUBIC;
    va_cubic_weights(tx, p.wx);
    va_cubic_weights(ty, p.wy);
    return;
  }
  p.status = VA_BY_LINEAR;
  p.wx[0] = GRID_ADD(1.0, -tx);
  p.wx[1] = tx;
  p.wy[0] = GRID_ADD(1.0, -ty);
  p.wy[1] = ty;
}

// Layer l's value at a planned point, read through s.at(l, row, col) (a float); every NaN is written as 0x7fc00000.
//  linear: f0 = (r0, c0), f1 = (r0 - 1, c0), f2 = (r0, c0 - 1), f3 = (r0 - 1, c0 - 1);
//    v = (((f0 ux) uy + (f1 tx) uy) + (f2 ux) ty) + (f3 tx) ty  (u = 1 - t);
//  cubic: per row i = 0..3 (row r0 + 1 - i) g_i = ((wy0 F(c0 + 1) + wy1 F(c0)) + wy2 F(c0 - 1)) + wy3 F(c0 - 2), then
//    v = ((wx0 g0 + wx1 g1) + wx2 g2) + wx3 g3.
// Each product and sum in double, rounded on its own; v is rounded to float once.
#if defined(__CUDACC__)
#pragma nv_exec_check_disable     // the live map's source reads its cells on the device only
#endif
template <class Src>
GRID_HD float va_value(const VaPoint& p, const Src& s, int l) {
  float f;
  if (p.status == VA_OUT) {
    f = va_nan();
  } else if (p.status == VA_BY_NEAREST) {
    f = s.at(l, p.r, p.c);
  } else if (p.status == VA_BY_LINEAR) {
    const double f0 = s.at(l, p.r, p.c), f1 = s.at(l, p.r - 1, p.c), f2 = s.at(l, p.r, p.c - 1),
                 f3 = s.at(l, p.r - 1, p.c - 1);
    const double v = GRID_ADD(GRID_ADD(GRID_ADD(GRID_MUL(GRID_MUL(f0, p.wx[0]), p.wy[0]),
                                                GRID_MUL(GRID_MUL(f1, p.wx[1]), p.wy[0])),
                                       GRID_MUL(GRID_MUL(f2, p.wx[0]), p.wy[1])),
                              GRID_MUL(GRID_MUL(f3, p.wx[1]), p.wy[1]));
    f = VA_D2F(v);
  } else {
    double v = 0.0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int r = p.r + 1 - i;
      double gi = GRID_MUL(p.wy[0], (double)s.at(l, r, p.c + 1));
#pragma unroll
      for (int j = 1; j < 4; j++) gi = GRID_ADD(gi, GRID_MUL(p.wy[j], (double)s.at(l, r, p.c + 1 - j)));
      v = i ? GRID_ADD(v, GRID_MUL(p.wx[i], gi)) : GRID_MUL(p.wx[0], gi);
    }
    f = VA_D2F(v);
  }
  return f != f ? va_nan() : f;
}

// Up to VA_MAX_LAYERS row-major layers of one geometry (cols: their row length).
struct VaGridSrc {
  int n, cols;
  const float* data[VA_MAX_LAYERS];
  GRID_HD float at(int l, int r, int c) const { return VA_LDG(data[l] + ((int64_t)r * cols + c)); }
  GRID_HD float value(const VaPoint& p, int l) const { return va_value(p, *this, l); }
};

#if defined(__CUDACC__)
// One thread per point: its plan once, then every layer of the source (Src: n layers; value(p, l): va_value of layer
// l).  values is layer-major (layer l of point i at l n + i).
template <class Src>
__global__ void __launch_bounds__(VA_THREADS)
k_values_at(const VaGeom g, const __grid_constant__ Src s, int method, const double* __restrict__ xy, int n,
            float* __restrict__ values, int32_t* __restrict__ status) {
  const int i = blockIdx.x * VA_THREADS + threadIdx.x;
  if (i >= n) return;
  VaPoint p;
  va_plan(g, method, xy[2 * i], xy[2 * i + 1], p);
  status[i] = p.status;
  for (int l = 0; l < s.n; l++) values[(int64_t)l * n + i] = s.value(p, l);
}

// ---- the host side both entry points share (emap_terrain_query_api.cu: grids; emap_export_api.cu: the live map) ----
#include "emap_handle.cuh"

// What both calls reject, besides their layers: nullptr, or why.
inline const char* va_check(int64_t n_layers, int64_t n, const double* positions, int32_t method,
                            const emap_values_out* out) {
  if (!out) return "null argument";
  if (n_layers < 1 || n_layers > VA_MAX_LAYERS) return "n_layers must be 1 .. EMAP_VALUES_MAX_LAYERS";
  if (method != VA_NEAREST && method != VA_LINEAR && method != VA_CUBIC)
    return "method must be EMAP_VALUES_NEAREST, EMAP_VALUES_LINEAR or EMAP_VALUES_CUBIC";
  if (n < 0 || n > INT32_MAX) return "n_points must be 0 .. 2^31 - 1";
  if (n && (!positions || !out->values || !out->status)) return "null positions or output";
  return nullptr;
}

// Host output's device block (the lookups' staging): the values, then the statuses, copied back in one piece.
inline size_t va_carve(uintptr_t base, int64_t n_layers, int64_t n, float*& values, int32_t*& status) {
  Carver c{base};
  values = c.take<float>((size_t)n_layers * n);
  status = c.take<int32_t>(n);
  return (size_t)((char*)(status + n) - (char*)base);
}

inline int va_room(emap_handle* h, int64_t n_layers, int64_t n, int32_t out_is_device) {
  if (out_is_device) return 0;
  float* v;
  int32_t* st;
  return grow(h, h->lookup.block, va_carve(0, n_layers, n, v, st), 0, false);
}

// The launch (xy: the positions on the device) and, for host output, one read-back and one synchronisation.
template <class Src>
int va_launch(emap_handle* h, const VaGeom& g, const Src& s, int method, int64_t n, const double* xy,
              const emap_values_out* out, int32_t out_is_device) {
  float* values = out->values;
  int32_t* status = out->status;
  size_t bytes = 0;
  if (!out_is_device) bytes = va_carve((uintptr_t)(char*)h->lookup.block, s.n, n, values, status);
  k_values_at<Src><<<cdiv(n, VA_THREADS), VA_THREADS, 0, h->stream>>>(g, s, method, xy, (int)n, values, status);
  LAUNCH_CHECK();
  if (!out_is_device) {
    if (int rc = read_back(h, h->lookup, values, bytes)) return rc;
    memcpy(out->values, h->lookup.down, sizeof(float) * s.n * n);
    memcpy(out->status, h->lookup.down + ((char*)status - (char*)values), sizeof(int32_t) * n);
  }
  return EMAP_OK;
}
#endif
