// emap_plan.cuh -- a handle's launch plan (host only): the tables, kernel variants and shared-memory layouts the host
// picks from the config and the sensor poses.  It knows no handle and launches nothing, so tests compile and run the
// very code the library runs (tests/native/plan_host.cu).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/emap.h"
#include "emap_device.cuh"

// Geometry of the cells a ray of this frame can reach, and of the coarse maps over them (ray_box below):
// rows [r0, r1) x columns [c0, c1) (c0, c1 multiples of 4 when W is); fine tiles of 2^ts x 2^ts cells aligned to the
// map (tile of a cell = cell >> ts), at most RT x RT of them from tile (ta, tb) on, covering the whole box.
#define RT 64                     // fine tiles per axis of the coarse ray maps
struct RayGrid { int r0, r1, c0, c1, ts, ta, tb; };   // (ta, tb): tile coordinates (cell >> ts) of the coarse maps' origin, both even

#define RC_STRIDE 31              // new march steps per k_raycast warp iteration
struct RcLayout { int off_t8, off_t16, off_steps, off_bar; };     // byte offsets of k_raycast's shared-memory regions

// k_post tile: PT_Y rows x PT_X columns per CTA
#define PT_X 32
#ifndef PT_Y
#define PT_Y 16
#endif

inline float h16_host(float x) { return __half2float(__float2half_rn(x)); }

struct FramePlan {
  std::vector<float> steps;   // the fp16 march variable s_k < max_len16, identical for every ray (CK.py:203,268)
  int n_tab = 0;              // floats of the march table as k_raycast reads it
  int span_cells = 0;         // cells (per axis) one 31-step warp iteration of the march can span
  RcLayout rc_lay{};
  size_t rc_smem = 0;         // k_raycast's dynamic shared memory
  int cells_per_thread = 1;   // k_record / k_finalize: 4 (one 16-byte access) when rows are whole 16-byte vectors, else 1
  int post_instance = 0;      // k_post<K>: the dilation as a compile-time constant for 1..3, 0 = read at run time
  size_t post_smem = 0;       // k_post's dynamic shared memory
};

// The device config and the launch plan of a handle with config c.
inline void make_plan(const emap_config& c, DevCfg& d, FramePlan& p) {
  memset(&d, 0, sizeof(d));
  d.W = c.cell_n; d.C = c.cell_n * c.cell_n;
  d.dilation = c.dilation_size; d.edge_sharpen = c.enable_edge_sharpen; d.drift_en = c.enable_drift_compensation;
  d.visibility = c.enable_visibility_cleanup; d.overlap = c.enable_overlap_clearance;
  // EM.py:87-91
  int cell_range = (int)(c.overlap_clear_range_xy / c.resolution);
  if (cell_range < 0) cell_range = 0;
  if (cell_range > c.cell_n) cell_range = c.cell_n;
  d.cell_min = c.cell_n / 2 - cell_range / 2; d.cell_max = c.cell_n / 2 + cell_range / 2;
  d.resolution = c.resolution; d.half_w = 0.5 * (double)c.cell_n;
  d.snf = c.sensor_noise_factor; d.mahal = c.mahalanobis_thresh; d.outlier_var = c.outlier_variance;
  d.inlier_var_half = c.drift_compensation_variance_inlier / 2.0; d.trav_inlier = c.traversability_inlier;
  d.wall_thresh = c.wall_num_thresh; d.min_drift_cnt = c.min_height_drift_cnt;
  d.max_ray_length = c.max_ray_length; d.cleanup_step = c.cleanup_step; d.cos_thresh = c.cleanup_cos_thresh;
  d.mvd2 = c.min_valid_distance * c.min_valid_distance; d.max_height = c.max_height_range;
  d.ramp_a = c.ramped_height_range_a; d.ramp_b = c.ramped_height_range_b; d.ramp_c = c.ramped_height_range_c;
  d.max_variance = c.max_variance; d.pos_thresh = c.position_noise_thresh; d.ori_thresh = c.orientation_noise_thresh;
  d.inv_res_f = (float)(1.0 / c.resolution); d.half_w_f = (float)(0.5 * (double)c.cell_n);
  d.c_out = (float)c.outlier_variance; d.init_var = (float)c.initial_variance;
  d.max_drift_f = (float)c.max_drift; d.drift_alpha_f = (float)c.drift_compensation_alpha;
  d.max_len16 = h16_host((float)c.max_ray_length);
  d.w_plus_half_f = (float)c.cell_n + 0.5f;
  d.res_f = (float)c.resolution;
  d.overlap_z_f = (float)c.overlap_clear_range_z; d.time_var_f = (float)c.time_variance;
  d.time_int_f = (float)c.time_interval;
  // ray-march cell table: fp16 coordinates are clamped to [-LIM, LIM], LIM = the first fp16 value >= (W/2 + 1) * resolution;
  // every value at or beyond +-LIM maps to cell W-1 / 0, so only the bit patterns [0, P) and [0x8000, 0x8000 + P) are staged
  {
    const double want = (0.5 * (double)c.cell_n + 1.0) * c.resolution;
    __half hl = __float2half_ru((float)std::min(want, 60000.0));
    unsigned short bits = __half_as_ushort(hl);
    if (bits > 0x7bff) bits = 0x7bff;
    d.lut_lim2 = ((u32)bits << 16) | bits;
    d.lut_p2 = (int)(((size_t)(bits + 1) * 2 + 15) & ~(size_t)15);
  }
  {   // CK.py:203,268: the march table
    const double ray_step = c.resolution / std::sqrt(2.0);
    std::vector<float>& st = p.steps;
    st.clear();
    float s = h16_host((float)ray_step);
    while (s < d.max_len16 && st.size() < 65535) {
      st.push_back(s);
      float nx = h16_host((float)((double)s + ray_step));
      if (!(nx > s)) break;      // fp16 spacing exceeded the step: the reference would spin forever
      s = nx;
    }
    d.n_steps = (int)st.size();
    d.first_step = st.empty() ? INFINITY : st[0];
    // as k_raycast reads it: [0] unused (lane 0 of the first warp iteration), [1 + k] = s_k, +inf padding up to a whole
    // number of 31-step warp iterations + one warp of over-read
    p.n_tab = (int)(((st.size() + RC_STRIDE - 1) / RC_STRIDE) * RC_STRIDE + 64) & ~1;
    // one warp iteration of the march: 30 steps between its first and last new sample, in cells (+1: fp16 coordinates)
    double span = 0;
    for (size_t k = 0; k + 1 < st.size(); k++) {
      const size_t e = std::min(st.size() - 1, k + RC_STRIDE - 1);
      span = std::max(span, ((double)st[e] - (double)st[k]) / c.resolution);
    }
    p.span_cells = (int)std::ceil(span) + 2;
  }
  {   // shared-memory layout of k_raycast: coarse maps + march table in the gap between the two halves of the cell table
      // when they fit there, else behind the second half
    const size_t P2 = (size_t)d.lut_p2;
    const size_t need = sizeof(float) * (RT * RT + (RT / 2) * (RT / 2) + (size_t)p.n_tab) + 16;
    size_t base = (P2 + 15) & ~(size_t)15, end = 65536 + P2;
    if (base + need > 65536) { base = (end + 15) & ~(size_t)15; end = base + need; }
    p.rc_lay.off_t8 = (int)base;
    p.rc_lay.off_t16 = (int)(base + sizeof(float) * RT * RT);
    p.rc_lay.off_steps = (int)(base + sizeof(float) * (RT * RT + (RT / 2) * (RT / 2)));
    p.rc_lay.off_bar = (int)((base + need - 16 + 7) & ~(size_t)7);
    p.rc_smem = end;
  }
  // rows of whole 16-byte vectors: 4 cells per thread in k_record / k_finalize, and a row pitch the TMA unit can describe
  const bool rows16 = d.W % 4 == 0;
  p.cells_per_thread = rows16 ? 4 : 1;
  {   // k_post stages (tile + halo) of three planes: TMA tensor copies where the row pitch allows it and the map holds one
      // staged box, plain loads otherwise
    const int HL = d.dilation + 3, HLX = (HL + 3) & ~3;
    d.post_tma = (rows16 && d.W >= PT_X + 2 * HLX && d.W >= PT_Y + 2 * HL) ? 1 : 0;
    p.post_instance = (d.dilation >= 1 && d.dilation <= 3) ? d.dilation : 0;
    const size_t plane = (size_t)(((PT_Y + 2 * HL) * (PT_X + 2 * HLX) + 31) & ~31);
    p.post_smem = sizeof(float) * (3 * plane + (size_t)(PT_Y + 6) * (PT_X + 6) + 2) +
                  sizeof(unsigned long long) * (size_t)(PT_Y + 2 * HL + 2);
  }
}

// Cells a ray of the frame with sensors poses[0, n) can reach.  A sample is t + ray*s with |ray| <= 1 per axis and
// s < len <= max_len16, so it lies within max_len16 of the sensor on each axis; its fp16 rounding moves it by at most
// 2^-11 of its magnitude.  Rows [r0, r1) x columns [c0, c1), columns aligned to cells_per_thread; union over the
// sensors, two cells of slack.  Tile size 2^ts: at most RT tiles per axis, and a double-size tile at least half the span
// of one warp iteration (so that an iteration starting anywhere in a double tile stays inside the 3 x 3 block
// k_raycast tests).
inline RayGrid ray_box(const DevCfg& d, const FramePlan& p, const Pose* poses, int n) {
  const int W = d.W, align = p.cells_per_thread;
  int r0 = W, r1 = 0, c0 = W, c1 = 0;
  const double L = (double)d.max_len16;
  for (int i = 0; i < n; i++) {
    for (int ax = 0; ax < 2; ax++) {
      const double tc = (double)poses[i].t[ax];
      const double e = (std::fabs(tc) + L) * (1.0 / 2048.0) + 1e-4;
      double lo = std::floor((tc - L - e) / d.resolution + d.half_w) - 2.0;
      double hi = std::floor((tc + L + e) / d.resolution + d.half_w) + 3.0;
      if (!(lo == lo) || !(hi == hi)) { lo = 0; hi = W; }         // NaN pose: whole map
      const int a = (int)std::min(std::max(lo, 0.0), (double)W), b = (int)std::min(std::max(hi, 0.0), (double)W);
      if (ax == 0) { r0 = std::min(r0, a); r1 = std::max(r1, b); } else { c0 = std::min(c0, a); c1 = std::max(c1, b); }
    }
  }
  RayGrid g{0, 0, 0, 0, 3, 0, 0};
  if (r1 <= r0 || c1 <= c0) return g;
  c0 = (c0 / align) * align; c1 = std::min(W, ((c1 + align - 1) / align) * align);
  g.r0 = r0; g.r1 = r1; g.c0 = c0; g.c1 = c1;
  // tiles are aligned to the map (tile = cell >> ts) and the coarse maps start at a double-tile boundary at or before
  // (r0, c0): RT tiles per axis must reach the far edge of the box from there
  for (int ts = 2;; ts++) {
    const int al = 2 << ts;
    const int r0a = (r0 / al) * al, c0a = (c0 / al) * al;
    if ((RT << ts) >= std::max(r1 - r0a, c1 - c0a) && (4 << ts) >= p.span_cells + 1) {
      g.ts = ts; g.ta = r0a >> ts; g.tb = c0a >> ts;
      break;
    }
  }
  return g;
}

// Whether k_raycast runs for a sensor with n_rays rays in a frame with ray box g.  With no map cell within reach of the
// frame's sensors (empty box) every sample clamps to the border ring, on which no ray acts, and k_raycast<false>'s
// fine-tile address would lie outside its coarse map.  The counting variant reads no coarse map and still counts the
// march steps.
inline bool raycast_runs(const RayGrid& g, i64 n_rays, int n_steps, bool count_rays) {
  if (n_rays <= 0 || n_steps == 0) return false;
  return count_rays || (g.r1 > g.r0 && g.c1 > g.c0);
}
