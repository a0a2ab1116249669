// emap_sdf.cuh -- a signed distance field of one fp32 grid layer and trilinear queries against it
// (emap_signed_distance_field, emap_sdf_values), sm_90a.  include/emap.h states the contract, DESIGN.md §4l (continued)
// the algorithm.
//
// The volume holds n_z slices of the grid at z_k = z_min + k res.  Voxel (r, c, k) is occupied when the layer's
// value (non-finite cells take the layer's lowest finite value) is >= z_k.  The field is an exact separable distance
// transform on integer squared distances in voxel units:
//  - z: each column is occupied up to its top slice T, so its distance to the other kind is k - T (free) or
//    T + 1 - k (occupied), in closed form;
//  - then two 1-D lower envelopes of parabolas (Felzenszwalb and Huttenlocher), along the columns of every row and
//    then along the rows, for every slice.  The breakpoints of the envelope are compared as int64 cross products, so
//    the passes are exact.
// One int32 per voxel carries both fields: positive, a free voxel and its squared distance to occupancy; negative, an
// occupied voxel and minus its squared distance to free space (SDF_INF: none on the line so far).  A free voxel's
// distance to free space and an occupied voxel's distance to occupancy are 0, so nothing is lost, and the passes run in
// place in the output buffer.  The last pass converts to float.
//
// The per-line and per-point functions are __host__ __device__: tests/native/sdf_host.cpp builds them for the CPU
// with the same arithmetic.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "emap_grid.cuh"

#define SDF_INF INT32_MAX          // no site of the other kind on the line (any d2 of an accepted volume is < 2^24)
#define SDF_MAX_D2 16777216        // 2^24: (rows-1)^2 + (cols-1)^2 + (n_z-1)^2 must be below it (emap.h)
#define SDF_MAX_LINE 4096          // so a line has at most 4096 cells and a site index fits in an int16
#define SDF_LINE_THREADS 64        // threads per line of the envelope passes: warp 0 builds the envelope of the free
                                   // voxels' field, warp 1 the occupied voxels', then all evaluate
#define SDF_THREADS 256            // threads per block of k_sdf_min and k_sdf_values

#if defined(__CUDA_ARCH__)
#define SDF_SQRT(a) __dsqrt_rn((a))
#define SDF_FSQRT(a) __fsqrt_rn((a))
#define SDF_FMUL(a, b) __fmul_rn((a), (b))
#else
#define SDF_SQRT(a) std::sqrt((double)(a))
#define SDF_FSQRT(a) std::sqrt((float)(a))
#define SDF_FMUL(a, b) ((float)(a) * (float)(b))
#endif

// ---- occupancy ----
// z_k: one multiply, then one add, in double
GRID_HD double sdf_z(double z_min, double res, int k) { return GRID_ADD(z_min, GRID_MUL((double)k, res)); }

// The highest slice k with e >= z_k, or -1: floor((e - z_min) / res) as the first guess, corrected with the exact
// comparison (z_k is non-decreasing in k, so occupancy is monotone in k).
GRID_HD int sdf_top(float e, double z_min, double res, int n_z) {
  const double h = (double)e;
  const double g = floor(GRID_DIV(GRID_ADD(h, -z_min), res));   // h finite or -inf, so never NaN
  int t = g < -1.0 ? -1 : g > (double)(n_z - 1) ? n_z - 1 : (int)g;
  while (t + 1 < n_z && h >= sdf_z(z_min, res, t + 1)) t++;
  while (t >= 0 && !(h >= sdf_z(z_min, res, t))) t--;
  return t;
}

// The z pass: voxel k of a column whose top slice is t, as a signed squared distance
GRID_HD int32_t sdf_z_value(int t, int k, int n_z) {
  if (k > t) return t < 0 ? SDF_INF : (k - t) * (k - t);
  return t == n_z - 1 ? -SDF_INF : -((t + 1 - k) * (t + 1 - k));
}

// The ordered unsigned key of a float (unsigned order = float order) and back: k_sdf_min takes the least key of the
// finite cells.  No finite float has the key SDF_KEY_NONE, so a buffer set to 0xff bytes starts the minimum.
GRID_HD uint32_t sdf_key(float v) {
  uint32_t b;
  memcpy(&b, &v, 4);
  return (b & 0x80000000u) ? ~b : b | 0x80000000u;
}
#define SDF_KEY_NONE 0xffffffffu   // no finite cell
// The value of non-finite cells: the lowest finite value, or -inf when there is none (every voxel is then free)
GRID_HD float sdf_fill(uint32_t key) {
  if (key == SDF_KEY_NONE) return -INFINITY;
  const uint32_t b = (key & 0x80000000u) ? key & 0x7fffffffu : ~key;
  float v;
  memcpy(&v, &b, 4);
  return v;
}

// ---- the 1-D lower envelope of one line ----
// The two fields of a line of signed values: the free voxels' (distance to occupancy; an occupied voxel is a site at
// 0) and the occupied voxels' (distance to free space; a free voxel is a site at 0).  SDF_INF: not a site.
struct SdfToOccupied {
  const int32_t* s;
  GRID_HD int32_t operator()(int i) const { return s[i] > 0 ? s[i] : 0; }
};
struct SdfToFree {
  const int32_t* s;
  GRID_HD int32_t operator()(int i) const { return s[i] < 0 ? -s[i] : 0; }
};

// h(p) = f(p) + p^2, the parabola of site p in the form the breakpoints use
template <class F>
GRID_HD int64_t sdf_h(const F& f, int p) { return (int64_t)f(p) + (int64_t)p * p; }

// The lower envelope of the parabolas (q - p)^2 + f(p) over the sites p of a line of n cells (f(p) < SDF_INF): its
// sites in v[0 .. m), left to right; returns m.  The parabolas of a and b (a < b) cross at
// s(a, b) = (h(b) - h(a)) / (2 (b - a)); the last site is dropped while s(v[m-2], v[m-1]) >= s(v[m-1], q), compared as
// the int64 cross product (h(b) - h(a)) (q - b) >= (h(q) - h(b)) (b - a).
template <class F>
GRID_HD int sdf_envelope(const F& f, int n, int16_t* v) {
  int m = 0;
  for (int q = 0; q < n; q++) {
    if (f(q) >= SDF_INF) continue;
    const int64_t hq = sdf_h(f, q);
    while (m >= 2) {
      const int a = v[m - 2], b = v[m - 1];
      const int64_t hb = sdf_h(f, b);
      if ((hb - sdf_h(f, a)) * (q - b) >= (hq - hb) * (b - a))
        m--;
      else
        break;
    }
    v[m++] = (int16_t)q;
  }
  return m;
}

// Whether cell q lies past the breakpoint of envelope sites k and k + 1: s(v[k], v[k+1]) < q
template <class F>
GRID_HD bool sdf_past(const F& f, const int16_t* v, int k, int q) {
  const int a = v[k], b = v[k + 1];
  return sdf_h(f, b) - sdf_h(f, a) < 2 * (int64_t)q * (b - a);
}

// The envelope site that covers cell q: the first k with !(k + 1 < m && s(v[k], v[k+1]) < q) (breakpoints are
// non-decreasing in k), by bisection
template <class F>
GRID_HD int sdf_envelope_find(const F& f, const int16_t* v, int m, int q) {
  int lo = 0, hi = m > 0 ? m - 1 : 0;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sdf_past(f, v, mid, q))
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// The envelope at cell q, advancing site k from where the previous (lower) cell left it; SDF_INF with no site
template <class F>
GRID_HD int32_t sdf_envelope_at(const F& f, const int16_t* v, int m, int q, int& k) {
  if (m == 0) return SDF_INF;
  while (k + 1 < m && sdf_past(f, v, k, q)) k++;
  const int d = q - v[k];
  return d * d + f(v[k]);
}

// Cells q0 .. q1 - 1 of one pass over a line s of n signed values, with the envelopes va (m_a sites) of the free
// voxels' field and vb (m_b sites) of the occupied voxels': each cell takes its own kind's field, signed.
// write(q, value) stores the result.
template <class W>
GRID_HD void sdf_line_part(const int32_t* s, const int16_t* va, int ma, const int16_t* vb, int mb, int q0, int q1,
                           W write) {
  const SdfToOccupied fa{s};
  const SdfToFree fb{s};
  int ka = sdf_envelope_find(fa, va, ma, q0), kb = sdf_envelope_find(fb, vb, mb, q0);
  for (int q = q0; q < q1; q++) {
    if (s[q] > 0)
      write(q, sdf_envelope_at(fa, va, ma, q, ka));
    else
      write(q, -sdf_envelope_at(fb, vb, mb, q, kb));
  }
}

// A signed squared distance in voxels as the field's value in metres: +-fl(sqrt(float(d2)) * float(res)), +-INFINITY
// for SDF_INF
GRID_HD float sdf_metres(int32_t v, float res) {
  const int32_t d2 = v < 0 ? -v : v;
  const float m = d2 >= SDF_INF ? INFINITY : SDF_FMUL(SDF_FSQRT((float)d2), res);
  return v < 0 ? -m : m;
}

// ---- queries ----
// A field as the queries read it: n_z slices of rows x cols floats, the grid's geometry and z_min
struct SdfVol {
  const float* data;
  int rows, cols, n_z;
  double pos[2], res, z_min;
};

GRID_HD float sdf_at(const SdfVol& f, int k, int r, int c) {
  return f.data[((int64_t)k * f.rows + r) * f.cols + c];
}

GRID_HD double sdf_lerp(double a, double b, double t) { return GRID_ADD(a, GRID_MUL(t, GRID_ADD(b, -a))); }

// One point's {value, d/dx, d/dy, d/dz} (emap.h states every operation).  Per axis (rows from x, columns from y,
// slices from z) the fractional index f, its clamp u to [0, n - 1], cell i0 = min(floor(u), n - 2) (0 when n = 1) and
// t = u - i0.  Trilinear in the order columns, rows, slices, each step a + t (b - a); the gradient is the analytic one
// of that interpolant, and the distance from the point to the clamped point is added to the value.  A NaN result is
// written as the quiet NaN 0x7ff8000000000000.
GRID_HD void sdf_value(const SdfVol& f, double x, double y, double z, double out[4]) {
  if (x != x || y != y || z != z) {
    for (int j = 0; j < 4; j++) out[j] = NAN;
    return;
  }
  const int n[3] = {f.rows, f.cols, f.n_z};
  const double fi[3] = {
      GRID_DIV(GRID_ADD(grid_axis_origin(f.pos[0], (double)f.rows * f.res, f.res), -x), f.res),
      GRID_DIV(GRID_ADD(grid_axis_origin(f.pos[1], (double)f.cols * f.res, f.res), -y), f.res),
      GRID_DIV(GRID_ADD(z, -f.z_min), f.res)};
  int i0[3], i1[3];
  double t[3], off[3];
  for (int a = 0; a < 3; a++) {
    const double top = (double)(n[a] - 1);
    const double u = fi[a] < 0.0 ? 0.0 : fi[a] > top ? top : fi[a];
    off[a] = GRID_ADD(fi[a], -u);
    if (n[a] == 1) {
      i0[a] = i1[a] = 0;
    } else {
      const double fl = floor(u);
      i0[a] = fl > (double)(n[a] - 2) ? n[a] - 2 : (int)fl;
      i1[a] = i0[a] + 1;
    }
    t[a] = GRID_ADD(u, -(double)i0[a]);
  }
  double xc[2][2], dc[2][2], yk[2], ec[2], dr[2];
  for (int kk = 0; kk < 2; kk++) {
    const int k = kk ? i1[2] : i0[2];
    for (int rr = 0; rr < 2; rr++) {
      const int r = rr ? i1[0] : i0[0];
      const double a0 = (double)sdf_at(f, k, r, i0[1]), a1 = (double)sdf_at(f, k, r, i1[1]);
      xc[kk][rr] = sdf_lerp(a0, a1, t[1]);
      dc[kk][rr] = GRID_ADD(a1, -a0);
    }
    yk[kk] = sdf_lerp(xc[kk][0], xc[kk][1], t[0]);
    dr[kk] = GRID_ADD(xc[kk][1], -xc[kk][0]);
    ec[kk] = sdf_lerp(dc[kk][0], dc[kk][1], t[0]);
  }
  const double value = sdf_lerp(yk[0], yk[1], t[2]);
  const double gr = sdf_lerp(dr[0], dr[1], t[2]), gc = sdf_lerp(ec[0], ec[1], t[2]), gk = GRID_ADD(yk[1], -yk[0]);
  const double dist =
      GRID_MUL(SDF_SQRT(GRID_ADD(GRID_ADD(GRID_MUL(off[0], off[0]), GRID_MUL(off[1], off[1])), GRID_MUL(off[2], off[2]))),
               f.res);
  out[0] = GRID_ADD(value, dist);
  out[1] = n[0] == 1 ? 0.0 : -GRID_DIV(gr, f.res);
  out[2] = n[1] == 1 ? 0.0 : -GRID_DIV(gc, f.res);
  out[3] = n[2] == 1 ? 0.0 : GRID_DIV(gk, f.res);
  for (int j = 0; j < 4; j++)
    if (out[j] != out[j]) out[j] = NAN;
}

// ---- kernels ----
#if defined(__CUDACC__)
// The least key of the finite cells into *key (set to SDF_KEY_NONE before): a grid-stride loop, a warp minimum and
// one atomic per warp
__global__ void __launch_bounds__(SDF_THREADS) k_sdf_min(const float* __restrict__ data, int64_t n, uint32_t* key) {
  uint32_t best = SDF_KEY_NONE;
  for (int64_t i = (int64_t)blockIdx.x * SDF_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * SDF_THREADS) {
    const float e = data[i];
    if (fabsf(e) <= FLT_MAX) best = min(best, sdf_key(e));
  }
  best = __reduce_min_sync(0xffffffffu, best);
  if ((threadIdx.x & 31) == 0 && best != SDF_KEY_NONE) atomicMin(key, best);
}

// Warp 0 builds the envelope of the free voxels' field, warp 1 that of the occupied voxels' (one lane each); then
// every thread evaluates a contiguous part of the line.
template <class W>
__device__ void sdf_line(const int32_t* s, int16_t* va, int16_t* vb, int n, W write) {
  __shared__ int m[2];
  if (threadIdx.x == 0) m[0] = sdf_envelope(SdfToOccupied{s}, n, va);
  if (threadIdx.x == 32) m[1] = sdf_envelope(SdfToFree{s}, n, vb);
  __syncthreads();
  const int q0 = (int)((int64_t)n * threadIdx.x / SDF_LINE_THREADS);
  const int q1 = (int)((int64_t)n * (threadIdx.x + 1) / SDF_LINE_THREADS);
  sdf_line_part(s, va, m[0], vb, m[1], q0, q1, write);
}

// Shared memory of a line of n cells: the signed values, then the two envelopes' sites
inline size_t sdf_line_smem(int n) { return (size_t)n * (sizeof(int32_t) + 2 * sizeof(int16_t)); }

// The z pass and the envelope along the columns of row blockIdx.x in slice blockIdx.y: vol (as int32) gets the signed
// squared distances within the slice's row
__global__ void __launch_bounds__(SDF_LINE_THREADS)
k_sdf_cols(const float* __restrict__ grid, int rows, int cols, int n_z, double z_min, double res,
           const uint32_t* __restrict__ key, int32_t* __restrict__ vol) {
  extern __shared__ int32_t sdf_sm[];
  int32_t* s = sdf_sm;
  int16_t* va = (int16_t*)(s + cols);
  int16_t* vb = va + cols;
  const int r = blockIdx.x, k = blockIdx.y;
  const float fill = sdf_fill(*key);
  const float* row = grid + (int64_t)r * cols;
  for (int c = threadIdx.x; c < cols; c += SDF_LINE_THREADS) {
    float e = row[c];
    if (!(fabsf(e) <= FLT_MAX)) e = fill;
    s[c] = sdf_z_value(sdf_top(e, z_min, res, n_z), k, n_z);
  }
  __syncthreads();
  int32_t* out = vol + ((int64_t)k * rows + r) * cols;
  sdf_line(s, va, vb, cols, [&](int q, int32_t v) { out[q] = v; });
}

// The envelope along the rows of column blockIdx.x in slice blockIdx.y, in place, converted to metres
__global__ void __launch_bounds__(SDF_LINE_THREADS)
k_sdf_rows(int rows, int cols, float res, int32_t* __restrict__ vol) {
  extern __shared__ int32_t sdf_sm[];
  int32_t* s = sdf_sm;
  int16_t* va = (int16_t*)(s + rows);
  int16_t* vb = va + rows;
  const int c = blockIdx.x, k = blockIdx.y;
  int32_t* col = vol + (int64_t)k * rows * cols + c;
  for (int r = threadIdx.x; r < rows; r += SDF_LINE_THREADS) s[r] = col[(int64_t)r * cols];
  __syncthreads();
  float* out = (float*)col;
  sdf_line(s, va, vb, rows, [&](int q, int32_t v) { out[(int64_t)q * cols] = sdf_metres(v, res); });
}

// One thread per point: 3 doubles in, 4 out
__global__ void __launch_bounds__(SDF_THREADS)
k_sdf_values(const SdfVol f, const double* __restrict__ points, int64_t n, double* __restrict__ out) {
  const int64_t q = (int64_t)blockIdx.x * SDF_THREADS + threadIdx.x;
  if (q >= n) return;
  double v[4];
  sdf_value(f, points[3 * q], points[3 * q + 1], points[3 * q + 2], v);
#pragma unroll
  for (int j = 0; j < 4; j++) out[4 * q + j] = v[j];
}
#endif
