// The library's host-side launch plan (emap_plan.cuh) and the polygon check's tile enumeration (emap_polygon.cuh),
// compiled as the library compiles them and exported to the tests through ctypes (tests/plan_host.py).
#include "emap_plan.cuh"
#include "emap_polygon.cuh"

namespace {

void plan_of(int W, double resolution, double max_ray_length, int dilation, DevCfg& d, FramePlan& p) {
  emap_config c = {};
  c.abi_version = EMAP_ABI_VERSION;
  c.cell_n = W; c.resolution = resolution; c.max_ray_length = max_ray_length; c.dilation_size = dilation;
  make_plan(c, d, p);
}

}  // namespace

extern "C" {

// RT, RC_STRIDE, PT_X, PT_Y, PG_COLS, PG_ROWS
void plan_constants(int out[6]) {
  const int v[6] = {RT, RC_STRIDE, PT_X, PT_Y, PG_COLS, PG_ROWS};
  for (int k = 0; k < 6; k++) out[k] = v[k];
}

// The plan of a W x W map (the config's other fields zero).  out: n_steps, n_tab, span_cells, off_t8, off_t16,
// off_steps, off_bar, rc_smem, lut_p2, cells_per_thread, post_tma, post_instance, post_smem; max_len16 and the first
// min(n_steps, cap) march steps.
void plan_make(int W, double resolution, double max_ray_length, int dilation, long long out[13], float* max_len16,
               float* steps, int cap) {
  DevCfg d;
  FramePlan p;
  plan_of(W, resolution, max_ray_length, dilation, d, p);
  const long long v[13] = {d.n_steps, p.n_tab, p.span_cells, p.rc_lay.off_t8, p.rc_lay.off_t16, p.rc_lay.off_steps,
                           p.rc_lay.off_bar, (long long)p.rc_smem, d.lut_p2, p.cells_per_thread, d.post_tma,
                           p.post_instance, (long long)p.post_smem};
  for (int k = 0; k < 13; k++) out[k] = v[k];
  *max_len16 = d.max_len16;
  for (int k = 0; k < d.n_steps && k < cap; k++) steps[k] = p.steps[k];
}

// ray_box of a frame whose n sensors sit at t_rel[3 k .. 3 k + 2] relative to the map centre: r0, r1, c0, c1, ts, ta, tb
void plan_ray_box(int W, double resolution, double max_ray_length, const float* t_rel, int n, int out[7]) {
  DevCfg d;
  FramePlan p;
  plan_of(W, resolution, max_ray_length, 0, d, p);
  std::vector<Pose> poses(n);
  for (int k = 0; k < n; k++)
    for (int ax = 0; ax < 3; ax++) poses[k].t[ax] = t_rel[3 * k + ax];
  const RayGrid g = ray_box(d, p, poses.data(), n);
  const int v[7] = {g.r0, g.r1, g.c0, g.c1, g.ts, g.ta, g.tb};
  for (int k = 0; k < 7; k++) out[k] = v[k];
}

int plan_raycast_runs(const int box[7], long long n_rays, int n_steps, int count_rays) {
  const RayGrid g = {box[0], box[1], box[2], box[3], box[4], box[5], box[6]};
  return raycast_runs(g, n_rays, n_steps, count_rays != 0);
}

// The k_polygon tiles and column window of one polygon of n vertices xy (clipped first, as the batch call does):
// tr0, n_tr, tc0, n_tc, col0, n_col
void plan_polygon_tiles(const float* xy, int n, const float* center, int W, double resolution, int out[6]) {
  PolyDesc d = {};
  clip_polygon(W, resolution, center, xy, n, nullptr, d.bbox);
  polygon_tiles(W, resolution, center, d);
  const int v[6] = {d.tr0, d.n_tr, d.tc0, d.n_tc, d.col0, d.n_col};
  for (int k = 0; k < 6; k++) out[k] = v[k];
}

}  // extern "C"
