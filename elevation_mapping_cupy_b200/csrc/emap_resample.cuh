// emap_resample.cuh -- the plane decomposition pipeline's resampling (emap_plane_decomposition), sm_90a.
//
// Reference: grid_map_filters_rsl's inpainting::resample (inpainting.cpp:244-288), the last step of the plane
// decomposition node's GridMapPreprocessing: cv::resize(INTER_LINEAR) of the filled and median-filtered elevation to
// int(n * res / new_res) cells per axis, and the true resolution that rounding leaves.  include/emap.h states the
// contract, DESIGN.md §4l the cv2 paths it was measured against.  The geometry and the per-cell value are __host__
// __device__ so that a native test runs them on the CPU; every operation is rounded on its own (no contraction).
#pragma once
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#if defined(__CUDACC__)
#define RS_HD __host__ __device__ __forceinline__
#else
#define RS_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define RS_DADD(a, b) __dadd_rn((a), (b))
#define RS_DMUL(a, b) __dmul_rn((a), (b))
#define RS_FADD(a, b) __fadd_rn((a), (b))
#define RS_FSUB(a, b) __fsub_rn((a), (b))
#define RS_FMUL(a, b) __fmul_rn((a), (b))
#else
#define RS_DADD(a, b) ((double)(a) + (double)(b))
#define RS_DMUL(a, b) ((double)(a) * (double)(b))
#define RS_FADD(a, b) ((float)(a) + (float)(b))
#define RS_FSUB(a, b) ((float)(a) - (float)(b))
#define RS_FMUL(a, b) ((float)(a) * (float)(b))
#endif

#define RS_THREADS 256

// The resampled size and true resolution of a rows x cols grid of resolution res for the requested new_res.  new_res
// <= 0 or within 1e-6 of res: unchanged.  Otherwise scaling = res / new_res, n' = int(n * scaling) per axis
// (truncating), and the true resolution 0.5 ((rows res) / rows' + (cols res) / cols'); 0 when a new size is 0.
inline void rs_geometry(int64_t rows, int64_t cols, double res, double new_res, int64_t size[2], double* out_res) {
  if (!(new_res > 0.0) || std::fabs(res - new_res) < 1e-6) {
    size[0] = rows; size[1] = cols; *out_res = res;
    return;
  }
  const double scaling = res / new_res;
  const double r = (double)rows * scaling, c = (double)cols * scaling;
  // int(n * scaling); a product beyond the int range is no grid the callers take, so it saturates
  size[0] = r < 2147483647.0 ? (int64_t)r : INT32_MAX;
  size[1] = c < 2147483647.0 ? (int64_t)c : INT32_MAX;
  *out_res = size[0] && size[1] ? 0.5 * (((double)rows * res) / (double)size[0] + ((double)cols * res) / (double)size[1])
                                : 0.0;
}

// One axis' taps for output index d of m from n source cells: f = (d + 0.5) (n / m) - 0.5 in double, s = floor(f),
// f -= s; s < 0 or s >= n - 1 is a clamped position: the edge cell alone.  Otherwise the cells s, s + 1 and the
// fraction rounded to float once.
struct RsTap {
  int s0, s1;
  float f;
  bool edge;
};

RS_HD RsTap rs_tap(int d, int n, int m) {
  double f = RS_DADD(RS_DMUL(RS_DADD((double)d, 0.5), (double)n / (double)m), -0.5);
  const double s = floor(f);
  f = RS_DADD(f, -s);
  RsTap t;
  t.edge = s < 0.0 || s >= (double)(n - 1);
  t.s0 = s < 0.0 ? 0 : s >= (double)(n - 1) ? n - 1 : (int)s;
  t.s1 = t.edge ? t.s0 : t.s0 + 1;
  t.f = t.edge ? 0.f : (float)f;
  return t;
}

// One pass on two taps: the edge cell as it is, else a + f (b - a) in fp32.
RS_HD float rs_lerp(float a, float b, const RsTap& t) {
  return t.edge ? a : RS_FADD(a, RS_FMUL(t.f, RS_FSUB(b, a)));
}

// Output cell (r, c) of the rows x cols resampling of the R x C row-major src: the columns' pass on the two source rows
// of the rows' taps, then the rows' pass.
RS_HD float rs_cell(const float* src, int R, int C, int rows, int cols, int r, int c) {
  const RsTap tr = rs_tap(r, R, rows), tc = rs_tap(c, C, cols);
  const float* a = src + (int64_t)tr.s0 * C;
  const float* b = src + (int64_t)tr.s1 * C;
  return rs_lerp(rs_lerp(a[tc.s0], a[tc.s1], tc), rs_lerp(b[tc.s0], b[tc.s1], tc), tr);
}

#if defined(__CUDACC__)
// One thread per output cell.
__global__ void k_rs_resample(const float* __restrict__ src, int R, int C, float* __restrict__ dst, int rows, int cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols;
  dst[i] = rs_cell(src, R, C, rows, cols, r, i - r * cols);
}
#endif
