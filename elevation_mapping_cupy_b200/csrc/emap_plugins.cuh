// emap_plugins.cuh -- the map plugins' kernels (sm_90a): min / max fill filter, smooth, erode, robot-centric elevation,
// and the map initialiser's dilation.
#pragma once
#include "emap_device.cuh"

// plugins/min_filter.py:57-82 with Jacobi order (reads iteration k-1, writes iteration k).
// `unfilled[it]` counts cells whose mask is still <= 0.5 after iteration it; an iteration whose
// predecessor left none is skipped on the device (min_filter.py:115 breaks on the host instead).
// MAX: plugins/max_filter.py:68-88 -- same stencil with max, and the fill test looks at the CURRENT mask
// (max_filter.py:102-108 passes copies of the running arrays), where min_filter keeps testing the ORIGINAL one.
template <bool MAX>
__global__ void __launch_bounds__(256)
k_fill_filter_iter(const DevCfg c, int k, const float* __restrict__ mask0, const float* __restrict__ in_h,
                   const float* __restrict__ in_m, float* __restrict__ out_h, float* __restrict__ out_m,
                   int* __restrict__ unfilled, int it) {
  if (it > 0 && unfilled[it - 1] == 0) { if (blockIdx.x == 0 && threadIdx.x == 0) unfilled[it] = 0; return; }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int miss = 0;
  if (i < c.C) {
    float h = in_h[i], m = in_m[i];
    if ((MAX ? m : mask0[i]) < 0.5f) {
      const float none = MAX ? -1000000.0f : 1000000.0f;
      float mv = none;
      for_window(c.W, c.C, i, k, [&](int idx, int, int) {
        const float val = in_h[idx];
        if (in_m[idx] > 0.5f && (MAX ? val > mv : val < mv)) mv = val;
      });
      if (MAX ? mv > none + 1.f : mv < none - 1.f) { h = mv; m = 0.6f; }
    }
    out_h[i] = h; out_m[i] = m;
    miss = !(m > 0.5f);
  }
  miss = __syncthreads_count(miss);
  if (threadIdx.x == 0 && miss) atomicAdd(unfilled + it, miss);
}
// final select: the result is in buffer parity (first it with unfilled[it]==0, else iteration_n-1)
__global__ void __launch_bounds__(256)
k_min_filter_final(const DevCfg c, const float* __restrict__ hA, const float* __restrict__ mA,
                   const float* __restrict__ hB, const float* __restrict__ mB, const int* __restrict__ unfilled,
                   int iteration_n, float* __restrict__ out, int* __restrict__ iters_run) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int last = iteration_n - 1;
  for (int it = 0; it < iteration_n; it++) if (unfilled[it] == 0) { last = it; break; }
  if (i == 0 && iters_run) *iters_run = last + 1;
  if (i >= c.C) return;
  // iteration `it` wrote buffer (it & 1) ? A : B   (it 0 reads A(copy of input) -> writes B)
  const float* h = (last & 1) ? hA : hB; const float* m = (last & 1) ? mA : mB;
  out[i] = m[i] > 0.5f ? h[i] : __int_as_float(0x7fc00000);
}

// plugins/smooth_filter.py:57-58: one 1-D pass of a size-3 uniform filter, 'reflect' boundary,
// double accumulation of x*(1/3) terms, fp32 store (cupyx.scipy.ndimage correlate1d).
__global__ void __launch_bounds__(256)
k_box3(const DevCfg c, const float* __restrict__ in, float* __restrict__ out, int axis) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const int W = c.W, r = i / W, cc = i - r * W;
  const double w = 1.0 / 3.0;
  int ia, ib;
  if (axis == 0) { ia = (r == 0 ? 0 : r - 1) * W + cc; ib = (r == W - 1 ? W - 1 : r + 1) * W + cc; }
  else { ia = r * W + (cc == 0 ? 0 : cc - 1); ib = r * W + (cc == W - 1 ? W - 1 : cc + 1); }
  const double sacc = __dadd_rn(__dadd_rn(__dmul_rn((double)in[ia], w), __dmul_rn((double)in[i], w)), __dmul_rn((double)in[ib], w));
  out[i] = (float)sacc;
}

// ------------------------------------------------------------------------------------------
// plugins/erosion.py:96-113: min / max of the (optionally reversed) layer, 8-bit normalisation, cv.erode with a
// ones(k,k) kernel (OpenCV folds `iterations` of a full rectangle into ONE erosion with a rectangle of side
// k + (iterations-1)(k-1) anchored at (k/2)*iterations; pixels outside the image do not constrain the minimum),
// de-normalisation.  mm = {min, max} as order-preserving keys.
__global__ void __launch_bounds__(256)
k_layer_minmax(const DevCfg c, const float* __restrict__ in, int reverse, u32* __restrict__ mm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  u32 lo = 0xffffffffu, hi = 0u;
  if (i < c.C) {
    float x = in[i];
    if (reverse) x = __fsub_rn(1.0f, x);
    lo = hi = fkey(x);
  }
  lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi);
  if ((threadIdx.x & 31) == 0) { atomicMin(mm, lo); atomicMax(mm + 1, hi); }
}
__global__ void __launch_bounds__(256)
k_erode(const DevCfg c, const float* __restrict__ in, float* __restrict__ out, int ks, int anchor, int reverse,
        const u32* __restrict__ mm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const int W = c.W, r = i / W, cc = i - r * W;
  const float mn = funkey(mm[0]), mx = funkey(mm[1]);
  const float span = (float)((double)mx - (double)mn);            // python float difference, used as float32
  int best = 255;
  for (int dy = -anchor; dy < ks - anchor; dy++) {
    const int rr = r + dy;
    if (rr < 0 || rr >= W) continue;
    for (int dx = -anchor; dx < ks - anchor; dx++) {
      const int c2 = cc + dx;
      if (c2 < 0 || c2 >= W) continue;
      float x = in[rr * W + c2];
      if (reverse) x = __fsub_rn(1.0f, x);
      const int q = (int)(unsigned char)__float2int_rz(__fdiv_rn(__fmul_rn(__fsub_rn(x, mn), 255.0f), span));
      best = min(best, q);
    }
  }
  float y = __fadd_rn(__fdiv_rn(__fmul_rn((float)best, span), 255.0f), mn);
  if (reverse) y = __fsub_rn(1.0f, y);
  out[i] = y;
}

// plugins/robot_centric_elevation.py:66-83: z of the cell in the base frame, optionally thresholded.
__global__ void __launch_bounds__(256)
k_robot_centric(const DevCfg c, const float* __restrict__ elev, const float* __restrict__ valid, float* __restrict__ out,
                float r6, float r7, float r8, double resolution, double threshold, int use_threshold) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const float rz = elev[i];
  float o = rz;                                                   // self.min_filtered = elevation_map[0].copy()
  if (valid[i] > 0.5f) {
    const float rx = (float)((double)(i / c.W) * resolution), ry = (float)((double)(i % c.W) * resolution);
    const float zb = __fmaf_rn(r8, rz, __fmaf_rn(r6, rx, __fmul_rn(r7, ry)));   // r0*x + r1*y + r2*z, nvcc contraction
    if (use_threshold) o = ((double)zb >= threshold) ? 1.0f : 0.0f;
    else o = zb;
  }
  out[i] = o;
}

// EM.py:913-922 after the map initialiser: dilation_filter_kernel (CK.py:392-449) of the elevation into invalid cells with
// mask = is_valid -- the reference runs it IN PLACE (racy); here every pass reads the previous pass's planes (src) and
// writes the map -- and update_upper_bound_with_valid_elevation (EM.py:428-432) on the last pass.
__global__ void __launch_bounds__(256)
k_init_dilate(const DevCfg c, const float* __restrict__ src_h, const float* __restrict__ src_valid, float* __restrict__ map,
              int k, int last) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const int W = c.W, C = c.C;
  float h = src_h[i], valid = src_valid[i];
  if (valid < 0.5f) {
    float distance = 100.f, near_value = 0.f;
    for_window(W, C, i, k, [&](int idx, int dy, int dx) {
      if ((src_valid[idx] > 0.5f) & ((float)(dx + dy) < distance)) { distance = (float)(dx + dy); near_value = src_h[idx]; }
    });
    if (distance < 100.f) { h = near_value; valid = 1.0f; }
  }
  map[i] = h; map[2 * C + i] = valid;
  if (last && valid > 0.5f) { map[5 * C + i] = h; map[6 * C + i] = 0.f; }     // EM.py:430-432
}
