/* Minimal C (not C++) client of libemap.so: what a native binding of the reference's bridge does per frame.
 * Build:  gcc -std=c99 -Iinclude examples/c_api_demo.c -Lelevation_mapping_cupy_b200 -lemap -Wl,-rpath,$PWD/elevation_mapping_cupy_b200 -o c_api_demo
 * (compiled, not run, by __graft_entry__.build(): there is no GPU in the build container). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "emap.h"

int main(void) {
  emap_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.abi_version = EMAP_ABI_VERSION;
  cfg.resolution = 0.04; cfg.cell_n = 202;                         /* round(8.0 / 0.04) + 2, parameter.py:287 */
  cfg.dilation_size = 3; cfg.enable_edge_sharpen = 1; cfg.enable_drift_compensation = 1;
  cfg.enable_visibility_cleanup = 1; cfg.enable_overlap_clearance = 1;
  cfg.sensor_noise_factor = 0.05; cfg.mahalanobis_thresh = 2.0; cfg.outlier_variance = 0.01;
  cfg.drift_compensation_variance_inlier = 0.1; cfg.traversability_inlier = 0.9; cfg.wall_num_thresh = 20;
  cfg.min_height_drift_cnt = 100; cfg.max_ray_length = 10.0; cfg.cleanup_step = 0.1; cfg.cleanup_cos_thresh = 0.1;
  cfg.min_valid_distance = 0.5; cfg.max_height_range = 1.0; cfg.ramped_height_range_a = 0.3;
  cfg.ramped_height_range_b = 1.0; cfg.ramped_height_range_c = 0.2; cfg.max_variance = 100.0;
  cfg.initial_variance = 1000.0; cfg.max_drift = 0.1; cfg.drift_compensation_alpha = 0.1;
  cfg.position_noise_thresh = 0.01; cfg.orientation_noise_thresh = 0.01; cfg.overlap_clear_range_xy = 4.0;
  cfg.overlap_clear_range_z = 2.0; cfg.time_variance = 0.0001; cfg.time_interval = 0.1;

  emap_handle* h = NULL;
  if (emap_create(&cfg, 0, &h) != EMAP_OK) { fprintf(stderr, "emap_create: %s\n", emap_last_error(NULL)); return 1; }

  enum { N = 1000 };
  double* pts = (double*)malloc(sizeof(double) * 3 * N);          /* the bridge hands over float64 rows */
  for (int i = 0; i < N; i++) { pts[3 * i] = (i % 40) * 0.1 - 2.0; pts[3 * i + 1] = (i / 40) * 0.1 - 1.2; pts[3 * i + 2] = -1.0; }
  const float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0, 0, 1.0f};
  const double pos[3] = {0, 0, 0};
  int rc = emap_move_to(h, pos, R);
  /* the node's use_initializer_at_start: the base and the corners of a 1 m square, cubic, the library triangulates */
  const float feet[15] = {0, 0, -1, -0.5f, -0.5f, -1, 0.5f, -0.5f, -1, 0.5f, 0.5f, -1, -0.5f, 0.5f, -1};
  if (!rc) rc = emap_initialize_map(h, feet, 5, 2, NULL, 0, NULL, 10.0, 2);
  if (!rc) rc = emap_input_pointcloud(h, pts, N, 3, EMAP_F64, 0, R, t, 0.02f, 0.02f);
  if (!rc) rc = emap_update_variance(h);
  if (!rc) rc = emap_update_time(h);
  const int wo = emap_cell_n(h) - 2;
  float* layer = (float*)malloc(sizeof(float) * (size_t)wo * wo);
  if (!rc) rc = emap_get_map_with_name(h, "elevation", layer, (int64_t)wo * wo);
  /* the get_raw_submap service: a 2 m x 2 m window around the map centre with two layers, sized on the host first */
  double centre[3] = {0, 0, 0}, win[4] = {0, 0, 2.0, 2.0}, win_centre[2];
  int32_t info[5] = {0, 0, 0, 0, 0};
  const char* names[2] = {"elevation", "traversability"};
  float* sub = NULL;
  if (!rc) rc = emap_get_position(h, centre);
  win[0] = centre[0]; win[1] = centre[1];
  if (!rc) rc = emap_submap_windows(emap_cell_n(h), cfg.resolution, centre, 1, win, info, win_centre);
  const int64_t sub_n = 2 * (int64_t)info[3] * info[4];
  if (!rc && sub_n) sub = (float*)malloc(sizeof(float) * (size_t)sub_n);
  if (!rc && sub) rc = emap_get_submaps(h, 1, win, 2, names, NULL, NULL, sub, 0, sub_n, info, win_centre);
  if (rc) fprintf(stderr, "error %d: %s\n", rc, emap_last_error(h));
  else printf("centre cell elevation: %f, window %d x %d at row %d, column %d, kernels launched: %lld\n",
              layer[(wo / 2) * wo + wo / 2], info[3], info[4], info[1], info[2], (long long)emap_launch_count(h));
  free(sub); free(layer); free(pts);
  emap_destroy(h);
  return rc ? 1 : 0;
}
