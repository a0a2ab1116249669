// emap_image.cuh -- camera image fusion into the semantic layers (emap_input_image), sm_90a.
//
// Reference: elevation_mapping.py:468-562 (input_image, host part), kernels/custom_image_kernels.py:9-157
// (image_to_map_correspondence_kernel), semantic_map.py:261-309 (update_layers_image) and the two image fusions,
// fusion/image_color.py and fusion/image_exponential.py.  There, one kernel writes a (2, W, W) uv plane and a (W, W)
// valid mask, then one kernel per channel reads them back and writes a new_map layer, which is copied into the
// semantic map.
// Here: k_image_fuse does it all for one cell in one thread -- validity, projection, distortion, the occlusion march and
// the sampling of every fused channel, written straight into the caller's layer buffer.  No uv / valid scratch.
//
// Bit-identity with the reference's own GPU build: nvcc contracts the reference string's products into FMAs (read from
// the SASS of its sm_90a build); those contractions are written out below with __fmaf_rn / __fma_rn, every other
// operation with its _rn intrinsic, so the result does not depend on how this file is compiled.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#define IMG_MAX_CH 64
enum { IMG_COLOR = 0, IMG_EXPONENTIAL = 1 };

// What the host part of EM.py:510-530 makes of one camera: P = K [R | t], the D rule and the camera cell.
struct ImageCam {
  float P[12];
  float fx, fy, cx, cy;     // K[0], K[4], K[2], K[5]
  float D[5];
  int distort;              // D is not all zero (CIK.py:64-66)
  float x1, y1, z1;         // camera cell (integral values) and height, relative to the map centre
};

enum { IMG_CAM_OK = 0, IMG_CAM_NONFINITE = 1, IMG_CAM_OUTSIDE = 2 };

// EM.py:510-530 in fp32: products rounded, sums left to right.  D is padded / truncated to 5 entries (fewer than 4:
// all zero) and zeroed unless the model is "radtan".  The camera cell is uint32(cell_n / 2 + t_cam_map / resolution),
// t_cam_map = -R^T t - center, with NumPy 2 promotion (the Python float operands taken as fp32).  A cell outside
// [0, 2^24) is rejected: beyond 2^32 uint32() is undefined, and from 2^24 on the fp32 copy the kernel gets is rounded.
inline int image_camera(const float K[9], const float* D, int n_D, const char* model, const float R[9], const float t[3],
                        const float center[3], int cell_n, double resolution, ImageCam* c) {
  for (int k = 0; k < 9; k++) if (!std::isfinite(K[k]) || !std::isfinite(R[k])) return IMG_CAM_NONFINITE;
  for (int k = 0; k < 3; k++) if (!std::isfinite(t[k])) return IMG_CAM_NONFINITE;
  memset(c, 0, sizeof(*c));
  for (int r = 0; r < 3; r++)
    for (int col = 0; col < 4; col++) {
      float s = 0.f;
      for (int k = 0; k < 3; k++) {
        const float rt = col < 3 ? R[3 * k + col] : t[k];
        const volatile float prod = K[3 * r + k] * rt;      // rounded product, never contracted
        s = k == 0 ? (float)prod : s + (float)prod;
      }
      c->P[4 * r + col] = s;
    }
  c->fx = K[0]; c->fy = K[4]; c->cx = K[2]; c->cy = K[5];
  if (n_D >= 4 && model && strcmp(model, "radtan") == 0)
    for (int k = 0; k < 5 && k < n_D; k++) c->D[k] = D[k];
  c->distort = !(c->D[0] == 0.f && c->D[1] == 0.f && c->D[2] == 0.f && c->D[3] == 0.f && c->D[4] == 0.f);
  float tc[3];
  for (int col = 0; col < 3; col++) {
    float s = 0.f;
    for (int k = 0; k < 3; k++) {
      const volatile float prod = -R[3 * k + col] * t[k];
      s = k == 0 ? (float)prod : s + (float)prod;
    }
    tc[col] = s - center[col];
  }
  const float half = (float)(cell_n / 2.0), res = (float)resolution;
  float cell[2];
  for (int k = 0; k < 2; k++) {
    const volatile float q = tc[k] / res;
    cell[k] = half + (float)q;
    if (!(cell[k] >= 0.f) || cell[k] >= 16777216.f) return IMG_CAM_OUTSIDE;
  }
  c->x1 = (float)(uint32_t)cell[0];
  c->y1 = (float)(uint32_t)cell[1];
  c->z1 = tc[2];
  return IMG_CAM_OK;
}

struct ImageArgs {
  ImageCam cam;
  float center[3];          // map centre, fp32 (EM.py:61)
  double res;               // resolution, the double literal of the reference string
  int W, C;                 // cell_n, cell_n^2
  float img_w, img_h;       // image width / height as fp32 (CuPy binds them to the map's dtype)
  long long n_img;          // n_planes * H * W: end of the image
  long long plane_sz;       // H * W
  const float* image;       // (n_planes, H, W) fp32, device
  float* sem;               // (n_layers, W, W) fp32, device
  int n;                    // fused channels
  int plane[IMG_MAX_CH];    // image plane an exponential channel reads (colour reads planes 0, 1, 2)
  int kind[IMG_MAX_CH];     // IMG_COLOR / IMG_EXPONENTIAL
  int layer[IMG_MAX_CH];    // semantic layer written
};

// Euclidean cell distance of get_l2_distance (CIK.py): dy * dy rounded, dx * dx fused into the sum.
__device__ __forceinline__ float img_cell_dist(int xa, int ya, int xb, int yb) {
  const float dx = (float)(xa - xb), dy = (float)(ya - yb);
  return __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

// a.b + c.d + e.f + g as nvcc contracts the reference's projection rows: fma(e, f, fma(a, b, c * d)) + g
__device__ __forceinline__ float img_row(float a, float b, float c, float d, float e, float f, float g) {
  return __fadd_rn(__fmaf_rn(e, f, __fmaf_rn(a, b, __fmul_rn(c, d))), g);
}

// One thread per cell: CIK.py:9-157 (correspondence), then every channel of image_color.py / image_exponential.py for
// a cell whose correspondence is valid.  Cells that are not valid keep their layer values and are not written.
__global__ void __launch_bounds__(256) k_image_fuse(const ImageArgs a, const float* __restrict__ map) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.C) return;
  const float* elev = map;
  const float* is_valid = map + 2 * (size_t)a.C;
  if (is_valid[i] != 1.f) return;
  const int W = a.W;
  const int x0 = i / W, y0 = i % W;
  const ImageCam& c = a.cam;
  // cell position: (int) * double literal + fp32 centre, in double, contracted
  const float p1 = (float)__fma_rn((double)(x0 - W / 2), a.res, (double)a.center[0]);
  const float p2 = (float)__fma_rn((double)(y0 - W / 2), a.res, (double)a.center[1]);
  const float z0 = elev[i];
  const float p3 = __fadd_rn(z0, a.center[2]);
  float u = img_row(p1, c.P[0], p2, c.P[1], p3, c.P[2], c.P[3]);
  float v = img_row(p1, c.P[4], p2, c.P[5], p3, c.P[6], c.P[7]);
  const float d = img_row(p1, c.P[8], p2, c.P[9], p3, c.P[10], c.P[11]);
  if (d <= 0.f) return;                     // NaN goes on, as in the reference
  u = __fdiv_rn(u, d);
  v = __fdiv_rn(v, d);
  if (c.distort) {                          // radtan, CIK.py:67-78
    const float k1 = c.D[0], k2 = c.D[1], q1 = c.D[2], q2 = c.D[3], k3 = c.D[4];
    const float x = __fdiv_rn(__fsub_rn(u, c.cx), c.fx);
    const float y = __fdiv_rn(__fsub_rn(v, c.cy), c.fy);
    const float r2 = __fmaf_rn(x, x, __fmul_rn(y, y));
    const float radial = __fmaf_rn(__fmul_rn(__fmul_rn(k3, r2), r2), r2,
                                   __fmaf_rn(__fmul_rn(k2, r2), r2, __fmaf_rn(k1, r2, 1.f)));
    const float uc = __fmaf_rn(q2, __fmaf_rn(__fadd_rn(x, x), x, r2),
                               __fmaf_rn(__fmul_rn(__fadd_rn(q1, q1), x), y, __fmul_rn(x, radial)));
    const float vc = __fmaf_rn(q1, __fmaf_rn(__fadd_rn(y, y), y, r2),
                               __fmaf_rn(__fmul_rn(__fadd_rn(q2, q2), x), y, __fmul_rn(y, radial)));
    u = __fmaf_rn(c.fx, uc, c.cx);
    v = __fmaf_rn(c.fy, vc, c.cy);
  }
  if ((u < 0.f) || (v < 0.f) || (u >= a.img_w) || (v >= a.img_h)) return;
  // Bresenham march from the cell to the camera cell (CIK.py:93-141).  The camera cell is integral and below 2^24, so
  // the reference's float comparisons with it are the integer ones.  The line moves monotonically toward the camera
  // cell: once it has left the map it never comes back, and no later cell can occlude.
  const int x1 = (int)c.x1, y1 = (int)c.y1;
  const float total = img_cell_dist(x0, y0, x1, y1);
  const float dz = __fsub_rn(c.z1, z0);
  const int dx = abs(x1 - x0), sx = x0 < x1 ? 1 : -1;
  const int dy = -abs(y1 - y0), sy = y0 < y1 ? 1 : -1;
  int err = dx + dy, x = x0, y = y0;
  while (true) {
    if (x == x1 && y == y1) break;
    if ((unsigned)x >= (unsigned)W || (unsigned)y >= (unsigned)W) break;
    const int idx = y + x * W;
    if (is_valid[idx] != 0.f) {
      const float ray = __fmaf_rn(__fdiv_rn(img_cell_dist(x0, y0, x, y), total), dz, z0);
      if (__dadd_rn((double)elev[idx], -0.10) > (double)ray) return;     // occluded: valid = false
    }
    const int e2 = 2 * err;
    if (e2 >= dy) {
      if (x == x1) break;
      err += dy; x += sx;
    }
    if (e2 <= dx) {
      if (y == y1) break;
      err += dx; y += sy;
    }
  }
  // the pixel, in fp32 as the fusions compute it: int(u) + int(v) * width (contracted); NaN u / v give 0
  const int iu = __float2int_rz(u), iv = __float2int_rz(v);
  const int pix = __float2int_rz(__fmaf_rn((float)iv, a.img_w, (float)iu));
  const size_t C = (size_t)a.C;
  for (int k = 0; k < a.n; k++) {
    float* out = a.sem + (size_t)a.layer[k] * C + i;
    if (a.kind[k] == IMG_COLOR) {
      // image_color.py: planes 0, 1, 2 of the stack; green = fma(width, height, red), blue = red + (width * height) * 2.
      // Below H * W = 2^24 both are exact; the clamp only keeps a rounded index of a larger image inside the buffer.
      const long long ig = __float2int_rz(__fmaf_rn(a.img_w, a.img_h, (float)pix));
      const long long ib = __float2int_rz(__fadd_rn((float)pix, __fmul_rn(__fmul_rn(a.img_w, a.img_h), 2.f)));
      const unsigned r = __float2uint_rz(a.image[pix]);
      const unsigned g = __float2uint_rz(a.image[min(ig, a.n_img - 1)]);
      const unsigned b = __float2uint_rz(a.image[min(ib, a.n_img - 1)]);
      *out = __uint_as_float((r << 16) + (g << 8) + b);
    } else {
      // image_exponential.py, alpha 0.7 in double: sem * (1 - 0.7) fused with the rounded 0.7 * img
      const float img = a.image[(size_t)a.plane[k] * a.plane_sz + pix];
      *out = (float)__fma_rn((double)*out, 1.0 - 0.7, __dmul_rn((double)img, 0.7));
    }
  }
}
