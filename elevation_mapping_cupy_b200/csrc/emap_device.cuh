// emap_device.cuh -- device-side arithmetic of the fusion path (sm_90a).
//
// Every helper states which reference expression it reproduces; paths are relative to
// /root/reference/elevation_mapping_cupy/script/elevation_mapping_cupy/ (CK.py =
// kernels/custom_kernels.py).  The reference declares helper parameters as CuPy `float16`
// (an fp16 value with implicit float conversions), so each of those is an explicit
// fp32 -> fp16 -> fp32 round trip here (h16), and every expression containing a substituted
// literal is evaluated in double exactly as NVRTC would (or by a proven-equivalent fp32 test).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

typedef unsigned long long u64;
typedef long long i64;
typedef unsigned int u32;

// Layer order of the (7,W,W) state, elevation_mapping.py:69-77.
enum { L_H = 0, L_V = 1, L_VALID = 2, L_TRAV = 3, L_TIME = 4, L_UPPER = 5, L_ISUP = 6 };

// packed per-point record bits (pidx)
#define PT_IDX_MASK 0x00ffffff
#define PT_VALID (1 << 28)
#define PT_INSIDE (1 << 29)
#define PT_SKIP (1 << 30)

// ray-record flag bits
#define RF_VALID 1u       // is_valid >= 0.5 after the fusion stores
#define RF_T05 2u         // time < 0.5
#define RF_T10 4u         // time < 1.0
#define RF_WALL 8u        // inlier count > wall_num_thresh (newmap[3], CK.py:246-247)
// Border-ring cells (CK.py:34-44,211: rays never act on them) are recorded as RF_VALID|RF_T05, the combination
// a ray skips without any effect, so the march needs no separate is_inside test.

#define UKEY_NONE 0xffffffffu

struct DevCfg {
  int W, C;
  int dilation, edge_sharpen, drift_en, visibility, overlap, cell_min, cell_max;
  int n_steps;                 // entries of the ray-march table s_k (CK.py:203)
  double resolution, half_w;   // 0.5 * W in double (CK.py:27)
  double snf, mahal, outlier_var, inlier_var_half, trav_inlier, wall_thresh;
  double min_drift_cnt, max_ray_length, cleanup_step, cos_thresh;
  double mvd2, max_height, ramp_a, ramp_b, ramp_c, max_variance;
  double pos_thresh, ori_thresh;
  float inv_res_f, half_w_f;   // fp32 estimate of the cell coordinate; exact path decides near integers
  float w_plus_half_f;         // (float)W + 0.5f
  float first_step;            // s_0 of the march table (+inf if the table is empty)
  float c_out;                 // (float)outlier_variance, the atomicAdd operand of CK.py:174,251
  float init_var, max_drift_f, drift_alpha_f, max_len16;
  float res_f;                 // CK.py:479-481 resolution() returns float
  float overlap_z_f, time_var_f, time_int_f;
  u32 lut_lim2;                // half2 {LIM, LIM}: the march clamps fp16 coordinates to [-LIM, LIM] before the cell look-up
  int lut_p2;                  // bytes of one half (positive / negative fp16 patterns) of the shared-memory cell table
  int post_tma;                // k_post stages its tiles with TMA tensor copies (row pitch a multiple of 16 B, map >= one box)
  float2 wp[3][2][9];          // traversability conv weights: layer, channel pair p, tap -> {w[2p][tap], w[2p+1][tap]}
  float wout[12];
};

struct Pose {                  // one sensor: R and t rounded to fp16 where the reference does (CK.py:54-57,62-69,83-85)
  float R16[9], t16[3], t[3];
};

struct __align__(16) Ray {     // one valid point's ray: set up once (CK.py:83-101,199-201,250)
  float x, y, z, len;          // end point (fp32) and fp16 march length
  float rx, ry, rz;            // fp16 unit direction
  u32 counts;                  // low 16 bits: n_act = number of march steps s_k < len (CK.py:203);
                               // high 16 bits: k_far = number of steps s_k < len_far -- samples with k < k_far are
                               // provably > sqrt(0.1) m from the end point (the `d < 0.1` test of CK.py:225 cannot fire)
};

struct FrameScalars {          // device-resident scalars of the running frame
  i64 E;                       // sum of (z - h) over drift inliers, 2^-32 fixed point (CK.py:331-332)
  i64 ecnt;                    // CK.py:333
  i64 nvalid;
  i64 ray_steps, ray_visits;
  float shift;                 // value added to every elevation cell this frame (elevation_mapping.py:357)
  int applied, evaluated;
  float mean_error, additive_mean_error, error_sum;
  float overlap_tz;            // t[2] of sensor 0 relative to the map centre (elevation_mapping.py:400-401)
  i64 ecnt_last, nvalid_last;  // copies for emap_get_frame_stats (the accumulators are re-zeroed inside the frame)
};

__device__ __forceinline__ float h16(float x) { return __half2float(__float2half_rn(x)); }

// 2^-32 fixed point of one fp32 term, |x| saturated at 2^20 (oracle/emap_oracle.c fix32)
__device__ __forceinline__ i64 fix32(float x) {
  if (x != x) return 0;
  x = fminf(fmaxf(x, -1048576.0f), 1048576.0f);
  return __float2ll_rn(x * 4294967296.0f);
}
__device__ __forceinline__ double unfix32(i64 s) { return (double)s * (1.0 / 4294967296.0); }

// order-preserving uint32 key of a float
__device__ __forceinline__ u32 fkey(float f) {
  u32 u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float funkey(u32 k) {
  u32 u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}

// CK.py:26-33 + 22-25: clamp(int((c16 - 0)/resolution + 0.5*W), 0, W-1) for an fp16-valued c16.
// The reference evaluates the quotient in double and truncates toward zero.  The fp32 estimate q is
// within 2.5e-4 of it for every |q| <= W+1 <= 2050 (|c16|/res * 2^-24 + ulp(2048)/2), so floor(q)
// decides the cell unless q is within 1e-3 of an integer; those take the double path.  q is first
// clamped to [-0.5, W+0.5] (NaN -> -0.5): everything below 0 clamps to cell 0 and everything above W-1
// to W-1 anyway, and floor == trunc for the in-range values.
__device__ __forceinline__ int axis_cell(const DevCfg& c, float c16) {
  const float q = fminf(fmaxf(fmaf(c16, c.inv_res_f, c.half_w_f), -0.5f), c.w_plus_half_f);
  const float fl = floorf(q);
  int i = (int)fl;
  if (fabsf((q - fl) - 0.5f) > 0.499f) i = __double2int_rz((double)c16 / c.resolution + c.half_w);
  return min(max(i, 0), c.W - 1);                // fp16 clamp is exact for W-1 <= 2048
}

// Both axes with ONE rare branch for the exact path and no integer clamp on the fast path: q is clamped
// to [0.25, W-0.75] first.  Every true quotient below 1 truncates/clamps to cell 0 and every one >= W-1 to
// cell W-1, which is what floor of the clamped value gives; values within 1e-3 of an integer (also 1 and
// W-1 themselves) still go to the double expression.
__device__ __forceinline__ void axis_cell2(float inv_res, float half_w, float q_hi, const DevCfg& c, float x16, float y16,
                                           int& ix, int& iy) {
  const float qx = fminf(fmaxf(fmaf(x16, inv_res, half_w), 0.25f), q_hi);
  const float qy = fminf(fmaxf(fmaf(y16, inv_res, half_w), 0.25f), q_hi);
  // floor without the conversion unit: q + 2^23 rounded toward -inf is exactly floor(q) + 2^23 for 0 <= q < 2^22,
  // and its low mantissa bits are the integer.
  const float rx = __fadd_rd(qx, 8388608.0f), ry = __fadd_rd(qy, 8388608.0f);
  const float fx = rx - 8388608.0f, fy = ry - 8388608.0f;
  ix = __float_as_int(rx) - 0x4b000000; iy = __float_as_int(ry) - 0x4b000000;
  if (fmaxf(fabsf((qx - fx) - 0.5f), fabsf((qy - fy) - 0.5f)) > 0.499f) {
    ix = min(max(__double2int_rz((double)x16 / c.resolution + c.half_w), 0), c.W - 1);
    iy = min(max(__double2int_rz((double)y16 / c.resolution + c.half_w), 0), c.W - 1);
  }
}

// CK.py:22-33 for EVERY fp16 bit pattern: lut[bits] = clamp(int(double(x16)/resolution + 0.5*W), 0, W-1).
// An fp16 coordinate has only 65536 values, so the exact double expression is tabulated once per handle
// (k_build_lut) and the ray march looks cells up instead of recomputing them (k_raycast).
__device__ __forceinline__ int axis_cell_exact(const DevCfg& c, float c16) {
  return min(max(__double2int_rz((double)c16 / c.resolution + c.half_w), 0), c.W - 1);
}

// CK.py:34-44
__device__ __forceinline__ bool cell_inside(int W, int ix, int iy) {
  return ix != 0 && ix != W - 1 && iy != 0 && iy != W - 1;
}

// CK.py:68-81 is_valid; X,Y,Z are the fp16-rounded transformed point.
__device__ __forceinline__ bool point_valid(const DevCfg& c, const Pose& q, float X, float Y, float Z) {
  float dx = X - q.t16[0], dy = Y - q.t16[1], dz = Z - q.t16[2];
  float d = __fmul_rn(dy, dy);                    // contraction nvcc emits for CK.py:64
  d = __fmaf_rn(dx, dx, d);
  d = __fmaf_rn(dz, dz, d);
  float sq = __fsqrt_rn(__fadd_rn(__fmul_rn(X, X), __fmul_rn(Y, Y)));
  float dxy = (float)fmax((double)sq - c.ramp_b, 0.0);
  if ((double)d < c.mvd2) return false;
  double zr = (double)dz;
  if (zr > fma((double)dxy, c.ramp_a, c.ramp_c) || zr > c.max_height) return false;
  return true;
}

struct Geom { float x, y, z, v; int ix, iy; bool valid, inside; };

// CK.py:160-167: transform, sensor noise, cell, validity of one raw point.
__device__ __forceinline__ void point_geom(const DevCfg& c, const Pose& q, float px, float py, float pz, Geom& g) {
  float rx = h16(px), ry = h16(py), rz = h16(pz);
  // CK.py:54-57: products of two fp16 values are exact in fp32, so fma == mul+add here.
  g.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.R16[0], rx), __fmul_rn(q.R16[1], ry)), __fmul_rn(q.R16[2], rz)), q.t16[0]);
  g.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.R16[3], rx), __fmul_rn(q.R16[4], ry)), __fmul_rn(q.R16[5], rz)), q.t16[1]);
  g.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.R16[6], rx), __fmul_rn(q.R16[7], ry)), __fmul_rn(q.R16[8], rz)), q.t16[2]);
  g.v = (float)((c.snf * (double)rz) * (double)rz);            // CK.py:58-60
  float X = h16(g.x), Y = h16(g.y), Z = h16(g.z);
  g.ix = axis_cell(c, X);
  g.iy = axis_cell(c, Y);
  g.inside = cell_inside(c.W, g.ix, g.iy);
  g.valid = point_valid(c, q, X, Y, Z);
}
