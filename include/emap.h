/*
 * emap.h -- C ABI of libemap.so, the H100-native (sm_90a) elevation-map fusion engine.
 *
 * This is the drop-in boundary for ONE path of leggedrobotics/elevation_mapping_cupy: the
 * per-frame point-cloud -> grid fusion + post-process chain.  Every entry point names the
 * reference interface it replaces; paths are relative to the reference repository, with
 *   EM.py  = elevation_mapping_cupy/script/elevation_mapping_cupy/elevation_mapping.py
 *   CK.py  = elevation_mapping_cupy/script/elevation_mapping_cupy/kernels/custom_kernels.py
 *   WRAP   = elevation_mapping_cupy/src/elevation_mapping_wrapper.cpp  (the pybind11 bridge)
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success and a
 * negative emap_status on failure (message via emap_last_error); no C++ exception crosses
 * the boundary.  The library owns all device state of a handle; inputs are borrowed for the
 * duration of the call; host outputs are caller-allocated.  One mutex and one CUDA stream
 * per handle: calls on one handle are serialised, handles are independent.  Device work is
 * asynchronous with respect to the host until emap_sync() or a call that returns host data.
 */
#ifndef EMAP_H_
#define EMAP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EMAP_ABI_VERSION 1

typedef struct emap_handle emap_handle;

typedef enum emap_status {
  EMAP_OK = 0,
  EMAP_ERR_INVALID = -1,   /* bad argument */
  EMAP_ERR_CUDA = -2,      /* CUDA runtime error (text in emap_last_error) */
  EMAP_ERR_NOLAYER = -3,   /* unknown layer name (EM.py:767 prints and returns) */
  EMAP_ERR_STATE = -4      /* call sequence error (sharded-frame phases) */
} emap_status;

typedef enum emap_dtype { EMAP_F32 = 0, EMAP_F64 = 1 } emap_dtype;

/* Parameters the path reads: same names, meaning and defaults as the reference's
 * Parameter dataclass (elevation_mapping_cupy/script/elevation_mapping_cupy/parameter.py:137-226).
 * Kernel constants are runtime data here (the reference bakes them into NVRTC source,
 * CK.py:111-121,264-274, and must re-JIT to change one). */
typedef struct emap_config {
  int32_t abi_version;              /* EMAP_ABI_VERSION */
  int32_t cell_n;                   /* parameter.py:287  round(map_length/resolution)+2, <= 2049 */
  int32_t dilation_size;
  int32_t enable_edge_sharpen;
  int32_t enable_drift_compensation;
  int32_t enable_visibility_cleanup;
  int32_t enable_overlap_clearance;
  int32_t use_only_above_for_upper_bound;
  double resolution;
  double sensor_noise_factor;
  double mahalanobis_thresh;
  double outlier_variance;
  double drift_compensation_variance_inlier;
  double traversability_inlier;
  double wall_num_thresh;
  double min_height_drift_cnt;
  double max_ray_length;
  double cleanup_step;
  double cleanup_cos_thresh;
  double min_valid_distance;
  double max_height_range;
  double ramped_height_range_a;
  double ramped_height_range_b;
  double ramped_height_range_c;
  double max_variance;
  double initial_variance;
  double max_drift;
  double drift_compensation_alpha;
  double position_noise_thresh;
  double orientation_noise_thresh;
  double overlap_clear_range_xy;
  double overlap_clear_range_z;
  double time_variance;
  double time_interval;
} emap_config;

/* Per-frame statistics (device scalars of the last frame, read back on request). */
typedef struct emap_frame_stats {
  float mean_error;            /* EM.py:354 */
  float additive_mean_error;   /* EM.py:355, EM.py:412-418 get_additive_mean_error */
  float shift_applied;         /* EM.py:357 */
  float error_sum;
  int64_t error_cnt;           /* EM.py:329 */
  int32_t drift_applied;
  int32_t drift_evaluated;
  int64_t n_points;            /* points in the frame (NaN rows included; a depth-image frame: its kept pixels) */
  int64_t n_valid_points;      /* points passing is_valid (CK.py:68-81) */
  int64_t ray_steps;           /* ray-march iterations (CK.py:203), 0 unless counting is enabled */
  int64_t ray_visits;          /* cells examined by rays past the skips of CK.py:209-226 */
} emap_frame_stats;

/* ---- lifecycle: replaces ElevationMap.__init__ (EM.py:52-117) / WRAP:31-110 initialize ---- */
int emap_create(const emap_config* cfg, int device, emap_handle** out);
int emap_destroy(emap_handle* h);
/* Text of the last error on this handle (h may be NULL: last emap_create failure). */
const char* emap_last_error(const emap_handle* h);
/* Traversability CNN weights: parameter.py:228-240 load_weights / traversability_filter.py:20-24.
 * w1,w2,w3: (4,1,3,3) = 36 floats each; w_out: (1,12,1,1) = 12 floats. */
int emap_set_traversability_weights(emap_handle* h, const float* w1, const float* w2, const float* w3,
                                    const float* w_out);

/* ---- the hot path: replaces ElevationMap.input_pointcloud (EM.py:434-466) == WRAP:173-178 input ----
 * points: n rows of `row_stride` elements of `dtype`, xyz first (extra channels ignored);
 *         rows with NaN in xyz are dropped (EM.py:458).  Host or device memory.
 * R (3x3 row-major), t (absolute sensor position): fp32 as EM.py:462-463 casts them.
 * Runs error count -> drift -> Kalman fusion -> ray-cast cleanup -> average -> overlap clear ->
 * dilation -> traversability -> normals, i.e. everything in update_map_with_kernel (EM.py:316-391). */
int emap_input_pointcloud(emap_handle* h, const void* points, int64_t n, int64_t row_stride, int dtype,
                          int is_device_ptr, const float R[9], const float t[3], float position_noise,
                          float orientation_noise);
/* Several sensors of one time slice fused against the same map snapshot (SURVEY 8(e)); with
 * n_sensors == 1 identical to emap_input_pointcloud.  points[s] has n[s] rows. */
int emap_input_sensors(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n,
                       int64_t row_stride, int dtype, int is_device_ptr, const float* R /*9*n_sensors*/,
                       const float* t /*3*n_sensors*/, float position_noise, float orientation_noise);
/* The write-back of CK.py:260-262 for the last frame, per input row (NaN rows: idx -1). */
int emap_get_point_record(emap_handle* h, int32_t* idx, uint8_t* valid, uint8_t* inside, int64_t n);
int emap_get_frame_stats(emap_handle* h, emap_frame_stats* out);
int emap_set_ray_counting(emap_handle* h, int enable);

/* ---- semantic point-channel fusion (SURVEY 8(f)2): semantic_map.py:223-259 update_layers_pointcloud, called by
 * EM.py:371 inside the frame.  Configure once (or whenever the channel set changes); every following
 * emap_input_pointcloud / emap_input_sensors then also fuses the configured feature columns of the cloud into the caller's
 * (n_layers, W, W) fp32 device buffer.  kind: 0 = fusion/pointcloud_average.py, 1 = fusion/pointcloud_class_average.py
 * (average_weight = parameter.py:163), 2 = fusion/pointcloud_color.py (feature = packed 0x00RRGGBB bits in a float).
 * n_channels = 0 switches it off.  Sharded frames fuse kinds 0..4 too (emap_shard_begin); they refuse kind 5. */
int emap_semantic_configure(emap_handle* h, int32_t n_channels, const int32_t* column, const int32_t* kind,
                            const int32_t* layer, float* semantic_map_device, int32_t n_layers, double average_weight);
/* The kinds of emap_semantic_configure (0..2) and of emap_semantic_configure_ext (0..5). */
#define EMAP_SEM_AVERAGE 0
#define EMAP_SEM_CLASS_AVERAGE 1
#define EMAP_SEM_COLOR 2
#define EMAP_SEM_CLASS_BAYESIAN 3
#define EMAP_SEM_BAYESIAN_INFERENCE 4
#define EMAP_SEM_CLASS_MAX 5
/* emap_semantic_configure with every point-cloud fusion of the reference, and the state two of them keep.  The arguments
 * of emap_semantic_configure mean the same; kind may also be
 *   3 = fusion/pointcloud_class_bayesian.py: per frame, the sum of the channel's values >= 0 at each cell, divided by the
 *       sum over the class_bayesian channels (1 where that is 0), in every cell;
 *   4 = fusion/pointcloud_bayesian_inference.py: where the frame fused n > 0 points, m' = m/(n*s + 1) + n*s*mean/(n*s + 1)
 *       and s' = s/(n*s + 1) in fp32, with the variance s of the layer read from and written to variance_device
 *       ((n_layers, W, W) fp32, device, caller-owned, indexed by layer like semantic_map_device; start it at 1.0);
 *   5 = fusion/pointcloud_class_max.py: the feature's bits are an fp16 probability (low 16) and a class id (high 16).
 *       For the j-th class_max channel, each cell takes the largest per-class probability sum over the ids of the frame's
 *       rows and of id_max (absent or earlier-won ids count 0, ties to the smallest id, NaN is the largest); the id goes
 *       to plane j of id_max_device ((n_id_max, W, W) int32, device, caller-owned, n_id_max >= the class_max channels),
 *       and every id that won anywhere counts 0 in the later channels.  The layers hold the maxima divided by their
 *       sum over the class_max channels (1 where that is 0), in every cell.
 * variance_device may be NULL without a kind 4 channel, id_max_device without a kind 5 channel.  Sums are exact fixed
 * point (DESIGN.md §4d).  emap_semantic_configure_ext(h, 0, ...) switches the fusion off. */
int emap_semantic_configure_ext(emap_handle* h, int32_t n_channels, const int32_t* column, const int32_t* kind,
                                const int32_t* layer, float* semantic_map_device, int32_t n_layers, double average_weight,
                                float* variance_device, int32_t* id_max_device, int32_t n_id_max);
/* CK.py:260-262 write-back of the last frame, on the DEVICE: one packed int32 per input row (bits 0..23 cell index,
 * bit 28 valid, bit 29 inside, bit 30 row dropped as NaN); valid until the next frame. */
int emap_point_record_device_ptr(emap_handle* h, const int32_t** packed_device, int64_t* n);

/* ---- depth cameras: the semantic sensor node's depth-image -> cloud step (sensor_processing/semantic_sensor/script/
 * semantic_sensor/pointcloud_node.py:205-274 create_pcl_from_image, get_coordinates, process_image) fused into the frame
 * with no intermediate cloud.  Per camera: depth (height, width) fp32 metres (the node's 32FC1 `passthrough`), optional
 * confidence (height, width) fp32, optional rgb (height, width, 3) uint8, optional features (n_features, height, width)
 * fp32; fx, fy, cx, cy = CameraInfo P[0], P[5], P[2], P[6]; R (3x3 row-major), t: the optical frame -> map pose, fp32 as
 * for emap_input_sensors.
 *  1. Mask: pixel (v, u) is kept iff isfinite(d) && d > 0 && d < max_depth && (no confidence || q >= confidence_threshold),
 *     compared in fp32 (the node's max(rint(fin + pos + conf + low - 2.6), 0) is this AND; its max_depth is 8).
 *  2. The kept pixels in row-major order (v, then u: nonzero's order), camera after camera, are the rows of the cloud.
 *  3. x = fp32(((double)u - cx) * (double)d / fx), y = fp32(((double)v - cy) * (double)d / fy), each operation rounded
 *     once in double, no contraction; z = d.
 *  4. Extra channel j (column 3 + j of the row, as emap_semantic_configure* addresses it) reads channel_source[j]: -1 the
 *     packed colour (r << 16) | (g << 8) | b as fp32 bits (at most one channel), k >= 0 feature plane k, bits as they are.
 *  5. The frame is bit for bit emap_input_sensors(h, n_cameras, clouds, ..., R, t, ...) of the clouds of steps 1-4
 *     (state, normals, semantic layers and their fusion state, emap_get_frame_stats; n_points = the kept pixels).
 *  6. Point record: one row per PIXEL, camera after camera; masked pixels are dropped rows (idx -1, bit 30 on the device
 *     record), the kept ones equal the cloud frame's record.
 * Inputs are all host memory or all device memory (is_device_ptr), staged as clouds are: device images are read in place
 * (no host synchronisation, capturable into a CUDA graph under the rules of emap_set_stream, which binds the image
 * pointers, sizes, intrinsics and channel sources too), page-locked host images over PCIe, pageable ones are staged;
 * host images are free to reuse on return.  Kernel launches: those of the cloud frame with the same channel
 * configuration.  emap_shard_begin_depth_images and emap_input_depth_images_sharded spread the cameras of one frame over
 * ranks.
 * EMAP_ERR_INVALID, with nothing launched and the state unchanged, for: n_cameras outside [1, EMAP_DEPTH_MAX_CAMERAS], a
 * NULL depth, height or width <= 0 or height * width > 2^24 (so a frame has fewer than 2^31 pixels), non-finite or zero fx / fy,
 * non-finite cx / cy / R / t, n_channels outside [0, EMAP_DEPTH_MAX_CHANNELS], n_features outside
 * [0, EMAP_DEPTH_MAX_FEATURES], a source outside [-1, n_features), more
 * than one colour channel, a colour channel without rgb or a feature channel without features, and a configured semantic
 * column >= 3 + n_channels.  EMAP_ERR_STATE on a handle attached to sharded scratch. */
#define EMAP_DEPTH_MAX_CAMERAS 16
#define EMAP_DEPTH_MAX_CHANNELS 16
#define EMAP_DEPTH_MAX_FEATURES 255
typedef struct emap_depth_camera {
  int32_t height, width;
  const float* depth;
  const float* confidence;       /* or NULL */
  const uint8_t* rgb;            /* or NULL */
  const float* features;         /* or NULL */
  double fx, fy, cx, cy;
  float R[9];
  float t[3];
} emap_depth_camera;
int emap_input_depth_images(emap_handle* h, int32_t n_cameras, const emap_depth_camera* cameras, int is_device_ptr,
                            int32_t n_channels, const int32_t* channel_source, int32_t n_features,
                            float confidence_threshold, float max_depth, float position_noise, float orientation_noise);
/* emap_input_depth_images with one camera. */
int emap_input_depth_image(emap_handle* h, const emap_depth_camera* camera, int is_device_ptr, int32_t n_channels,
                           const int32_t* channel_source, int32_t n_features, float confidence_threshold, float max_depth,
                           float position_noise, float orientation_noise);

/* ---- sharded frame (one rank per GPU, replicated grid; SURVEY 8(e)).  Between the phases the
 * caller all-reduces the exchange buffers in place (SUM for the int64/uint32 words named
 * "sum", MAX / MIN as named) with NCCL; single-GPU callers never need these. ---- */
typedef struct emap_exchange {
  void* ptr;        /* device pointer */
  int64_t count;    /* number of elements */
  int32_t kind;     /* 0: int64 SUM, 1: int64 MAX (keys < 2^63), 2: int32 MIN (keys offset to signed order), 3: int32 SUM */
} emap_exchange;
/* Semantic channels (emap_semantic_configure*) of kinds 0..4 are fused by sharded frames: each rank sums its own points'
 * channels in phase 1, the sums are reduced with the others (exchange 2, or the multicast block), and every replica
 * writes the layers in phase 3, bit for bit those of the single-GPU frame of all ranks' inputs.  A class_max channel
 * (kind 5) is refused: any sharded begin returns EMAP_ERR_INVALID with nothing queued while one is configured. */
int emap_shard_begin(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n,
                     int64_t row_stride, int dtype, int is_device_ptr, const float* R, const float* t,
                     int64_t global_point_offset, float position_noise, float orientation_noise);
/* emap_shard_begin for depth cameras: arguments, checks and rows as emap_input_depth_images.  The rows are the pixels,
 * camera after camera (masked pixels are dropped rows), so global_point_offset is the number of PIXELS (height * width
 * summed) of the cameras on lower ranks; then the upper-bound keys ("last point in input order") are those of a single-GPU
 * emap_input_depth_images of all ranks' cameras in rank order.  global_point_offset + this rank's pixels < 2^31.  The
 * phases, barriers and exchanges that follow are those of emap_shard_begin. */
int emap_shard_begin_depth_images(emap_handle* h, int32_t n_cameras, const emap_depth_camera* cameras, int is_device_ptr,
                                  int32_t n_channels, const int32_t* channel_source, int32_t n_features,
                                  float confidence_threshold, float max_depth, int64_t global_point_offset,
                                  float position_noise, float orientation_noise);
/* NVLink-multicast mode (replaces the three all-reduces): the caller allocates one symmetric block of
 * emap_shard_scratch_bytes() per rank (e.g. torch.distributed._symmetric_memory), rendezvouses it and hands
 * the library its own base and the MULTICAST alias.  From then on every per-cell accumulation of the frame
 * kernels is a single `multimem.red` that the NVSwitch applies to the replicas of all ranks -- the scatter and
 * the collective are one instruction.  Frame = emap_shard_begin, barrier, phase 0 (index), barrier, phase 1,
 * barrier, phase 2, barrier, phase 3; the barriers are the caller's (stream-ordered, cross-rank).
 * The block holds the exchange scratch and then the semantic sum planes of the current configuration, so its size
 * depends on that configuration: a sharded begin on a handle whose block is smaller than emap_shard_scratch_bytes()
 * returns EMAP_ERR_STATE; attach a new block of that size (every rank, collectively) and begin again. */
int64_t emap_shard_scratch_bytes(const emap_handle* h);
int emap_shard_attach(emap_handle* h, void* local_base, void* multicast_base, int64_t bytes);
/* Height reference of clear_overlap_map (EM.py:400-401) for a sharded frame: the absolute z of the
 * FIRST sensor of the whole frame (rank 0's), so that every replica clears the same cells.  Call
 * between emap_shard_begin and phase 3; without it a rank uses its own first sensor. */
int emap_shard_set_overlap_z(emap_handle* h, float sensor_z_absolute);
/* The arrays to reduce after phase `phase` (1..3): phase 1 the counts and drift statistics; phase 2 the height sums,
 * the fused counts (listed second: the only array phase 2 reads, the others are read in phase 3), the last-writer keys,
 * then the semantic sums where the configuration has them (int64 SUM of the averaged channels, int32 SUM of the colour
 * channels); phase 3 the decrements, ray counts and upper-bound keys.  *n_out: the capacity on entry (>= 3), the count
 * on return; a capacity below the count returns EMAP_ERR_INVALID with *n_out set to the count. */
#define EMAP_SHARD_MAX_EXCHANGES 5
int emap_shard_exchange(emap_handle* h, int32_t phase, emap_exchange* out, int32_t* n_out /*in: capacity*/);
int emap_shard_phase(emap_handle* h, int32_t phase);   /* 0: index (attached handles only), 1: fusion, 2: ray-cast, 3: finalise+post */

/* ---- sharded frames for a caller WITHOUT a host framework (SURVEY 8(b) emap_comm_init): NCCL through the C ABI.
 * libnccl.so.2 is loaded at run time.  One rank obtains an id (emap_comm_unique_id == ncclGetUniqueId), distributes the
 * 128 bytes by its own means, every rank calls emap_comm_init, and then every frame is ONE collective call:
 * emap_input_sensors_sharded fuses this rank's sensors (arguments as emap_shard_begin) with all other ranks' into the
 * replicated grid using integer NCCL all-reduces between the phases.  overlap_sensor_z_absolute: absolute z of the
 * frame's FIRST sensor overall (the same value on every rank, see emap_shard_set_overlap_z). */
typedef struct emap_nccl_id { char internal[128]; } emap_nccl_id;      /* == ncclUniqueId */
int emap_comm_unique_id(emap_nccl_id* out);
int emap_comm_init(emap_handle* h, const emap_nccl_id* id, int32_t rank, int32_t nranks);
int emap_input_sensors_sharded(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n,
                               int64_t row_stride, int dtype, int is_device_ptr, const float* R, const float* t,
                               int64_t global_point_offset, float overlap_sensor_z_absolute, float position_noise,
                               float orientation_noise);
/* emap_input_sensors_sharded for depth cameras: arguments as emap_shard_begin_depth_images, plus the absolute z of the
 * frame's first camera overall (rank 0's first). */
int emap_input_depth_images_sharded(emap_handle* h, int32_t n_cameras, const emap_depth_camera* cameras, int is_device_ptr,
                                    int32_t n_channels, const int32_t* channel_source, int32_t n_features,
                                    float confidence_threshold, float max_depth, int64_t global_point_offset,
                                    float overlap_sensor_z_absolute, float position_noise, float orientation_noise);

/* ---- pose / time: EM.py:139-170 move, move_to (WRAP:180-186); EM.py:119-128 clear (WRAP:188-191);
 * EM.py:420-426 update_variance, update_time (WRAP:193-203) ---- */
int emap_move_to(emap_handle* h, const double position[3], const float R[9]);
int emap_move(emap_handle* h, const double delta_position[3]);
int emap_clear(emap_handle* h);
int emap_update_variance(emap_handle* h);
int emap_update_time(emap_handle* h);
/* EM.py:564-577 update_normal(dilated_map): device pointer to a (W,W) fp32 plane, or NULL for
 * the engine's own traversability_input. */
int emap_update_normal(emap_handle* h, const float* dilated_map_device);
/* EM.py:899-922 initialize_map, device half only: after the caller has written interpolated elevation / variance /
 * is_valid planes (emap_set_state), run `iterations` passes of the initialiser's dilation (CK.py:392-449 with
 * dilation_size_initialize, mask = is_valid) and update_upper_bound_with_valid_elevation (EM.py:428-432).
 * emap_initialize_map below does the whole initialisation, interpolation included, and runs this as its last step. */
int emap_initialize_map_finish(emap_handle* h, int32_t dilation_size_initialize, int32_t iterations);
/* EM.py:899-922 + map_initializer.py:25-62 initialize_map, on the device: clear the map (as emap_clear), then
 * interpolate n_points (x, y, z) fp32 points in the map frame over every cell, then two passes of
 * emap_initialize_map_finish with dilation_size_initialize.
 *  - Snap: cell = (int32)((xy - center_xy) / (float)resolution + cell_n / 2) and z - center_z, all in fp32 (the
 *    reference's transform_to_map_index).  Cell (i, j) is state element [i * cell_n + j].
 *  - method 0 nearest: the point at the least squared cell distance, the lowest input index on a tie (SciPy's k-d tree
 *    agrees whenever there are at most 10 points).  1 linear / 2 cubic: barycentric / Clough-Tocher (SciPy's
 *    LinearNDInterpolator / CloughTocher2DInterpolator) over the triangles, in fp64.  A cell takes the lowest-index
 *    triangle that contains it, edges and vertices included; cells outside every triangle keep the cleared values.
 *  - Cells with a value get elevation = (float)value, variance = initialized_variance, is_valid = 1.
 *  - triangles_host: (n_triangles, 3) indices into the points, either orientation, or NULL.  With NULL the library
 *    triangulates: exact integer predicates, Bowyer-Watson inserting the points in input order from the seed (point
 *    0, the first point that differs from it, the first point not collinear with those two); a point equal to an
 *    earlier one is skipped; a point ON a triangle's circumcircle does not break it, so among four or more cocircular
 *    points the triangles of the earlier points stay.  Triangles are then numbered in order of (lowest vertex, next
 *    vertex counter-clockwise, last).
 *  - gradients_host (cubic only): (n_points, 2) fp64 vertex gradients, or NULL for SciPy's
 *    estimate_gradients_2d_global (tol 1e-6, maxiter 400, vertices in index order).
 * EMAP_ERR_INVALID, with the map cleared: NULL points, n_points <= 3 (the reference's assertion), more than
 * EMAP_INIT_MAX_POINTS, an unknown method, a non-finite point or one whose cell is outside the int32 range, collinear
 * points (linear / cubic without triangles), a triangle index outside [0, n_points), a triangle of zero area,
 * n_triangles outside [1, 2 * EMAP_INIT_MAX_POINTS].  One host-to-device upload of the points or of the triangles, their
 * coefficients and tile lists, and kernels on the handle's stream: no device-to-host copy and no host synchronisation
 * (except when the upload's staging grows, and a wait for the previous call's upload to leave it). */
#define EMAP_INIT_MAX_POINTS 65536
int emap_initialize_map(emap_handle* h, const float* xyz_host, int32_t n_points, int32_t method,
                        const int32_t* triangles_host, int32_t n_triangles, const double* gradients_host,
                        double initialized_variance, int32_t dilation_size_initialize);
int emap_get_position(emap_handle* h, double out[3]);          /* EM.py:130-137 */

/* ---- export: EM.py:720-775 get_map_with_name_ref (WRAP:205-252): NaN-fill, +center_z, crop the
 * border ring, flip both axes; writes (cell_n-2)^2 floats to caller memory.  Names: elevation,
 * variance, traversability, time, upper_bound, is_upper_bound, normal_x, normal_y, normal_z, normal_color.
 * normal_color is the C++ bridge's addNormalColorLayer (WRAP:296-314, enable_normal_color), which the bridge stores as
 * its `color` layer, for every exported cell, from the exported normal_x/y/z: cx = float((nx + 1.0) / 2.0),
 * cy = float((ny + 1.0) / 2.0) (computed in double), cz = nz; each channel is int(c * 255.0f) (a float product truncated
 * toward zero); the value is the float whose bits are (r << 16) | (g << 8) | b (grid_map's colorVectorToValue).  Where
 * the reference leaves it undefined: a channel whose product is NaN is 0, one beyond the int32 range saturates, and a
 * negative channel contributes its 32-bit two's complement to the OR.  This is restated from grid_map's published
 * source and was not checked against a grid_map build. ---- */
int emap_get_map_with_name(emap_handle* h, const char* name, float* out_host, int64_t n_out);
/* Batched export: what WRAP:213-252 (ElevationMappingWrapper::get_grid_map) does layer by layer -- n layers with ONE
 * kernel, one device-to-host copy, one synchronisation.  names[k] is a basic layer of emap_get_map_with_name, or
 * planes[k] a (W,W) fp32 device plane (plugin or semantic layer) exported with flags[k]: EM.py:579-596,762-775
 * process_map_for_publish, bit 0: fill_nan, bit 1: add the centre height.  out_host holds n consecutive (cell_n-2)^2
 * planes. */
int emap_get_layers(emap_handle* h, int32_t n, const char* const* names, const float* const* planes_device,
                    const int32_t* flags, float* out_host, int64_t n_out_total);
/* ---- windows of the exported map: the ROS node's get_raw_submap service (elevation_mapping_ros.cpp:507-553, grid_map's
 * GridMap::getSubmap on the exported layers).  Coordinates are those of emap_get_layers' output: the (cell_n-2)^2
 * interior, flipped on both axes, so row 0 is the +x edge and column 0 the +y edge; rows follow x, columns y.
 * windows[4w .. 4w+3] = (position_x, position_y, length_x, length_y) in the map frame, lengths finite and >= 0.
 * A coordinate p lies in state cell floor((p - center) / resolution + cell_n / 2) (EM.py's index, in double, half-open:
 * a coordinate on a cell boundary belongs to the cell on its +x / +y side), state cell i is output index cell_n - 2 - i.
 * Window w is the inclusive cell rectangle between the cell holding position + length / 2 and the cell holding
 * position - length / 2, each clipped to the exported area; a length of 0 gives one cell.  It fails when the position's
 * own cell is outside the exported area (or the position is not a number).
 * info[5w .. 5w+4] = {success (1/0), row0, col0, rows, cols}, all 0 on failure; centres[2w .. 2w+1] = the centre of the
 * window's cells in the map frame (NaN on failure).
 * emap_submap_windows: that arithmetic alone, on the host, for a map of cell_n cells at `resolution` centred at
 * center; no handle, no device.  EMAP_ERR_INVALID for NULL arguments, cell_n < 3, a resolution that is not finite and
 * > 0, n_windows < 0 and a length that is not finite and >= 0. */
int emap_submap_windows(int32_t cell_n, double resolution, const double center[2], int32_t n_windows,
                        const double* windows, int32_t* info, double* centres);
/* emap_get_submaps: the windows of the handle's map, with n_layers layers each, named as for emap_get_layers (names[k],
 * or planes_device[k] != NULL with flags[k]); every value is bit-identical to the same cell of emap_get_layers.
 * out receives, window after window, each successful window's layers one after another, each rows x cols row-major
 * (failed windows take no space): out_floats must be at least n_layers times the sum of rows * cols.  out is host memory
 * (out_is_device 0: one device-to-host copy and one synchronisation) or device memory (out_is_device != 0: no host
 * synchronisation; the work is queued on the handle's stream, see emap_wait_for_stream / emap_stream_wait_for, and the
 * call can be captured into a CUDA graph: its window table travels in the kernel's parameters).  One kernel per call.
 * EMAP_ERR_INVALID, with nothing written or launched, for a NULL windows / names / out / info / centres, n_windows
 * outside [1, EMAP_SUBMAP_MAX_WINDOWS], n_layers outside [1, EMAP_SUBMAP_MAX_LAYERS], a length that is not finite and
 * >= 0, an unknown layer name and an output too small. */
#define EMAP_SUBMAP_MAX_WINDOWS 1024
#define EMAP_SUBMAP_MAX_LAYERS 24
int emap_get_submaps(emap_handle* h, int32_t n_windows, const double* windows, int32_t n_layers, const char* const* names,
                     const float* const* planes_device, const int32_t* flags, float* out, int32_t out_is_device,
                     int64_t out_floats, int32_t* info, double* centres);
/* ---- windows in the requester's frame: get_raw_submap with a frame_id other than the map frame
 * (elevation_mapping_ros.cpp:507-553): the window around T^-1 * position, then grid_map's
 * GridMap::getTransformedMap(T, "elevation", frame_id, sample_ratio) on it.  Restated from grid_map's published source
 * (GridMap::getTransformedMap, GridMapMath.cpp); not checked against a grid_map build.
 * transforms[12w .. 12w+11] = T of window w: R row-major (9), then t (3), in double; T maps map-frame points into the
 * request frame (lookupTransform(frame_id, map_frame)).  R must be finite and orthonormal: every entry of R^T R - I
 * within EMAP_TRANSFORM_TOLERANCE; t finite.  windows[4w .. 4w+3] = (position_x, position_y) in the request frame and
 * (length_x, length_y), finite and >= 0.  Every product and sum below is one IEEE double operation, nothing is fused,
 * and a matrix-vector product is ((R_k0 x + R_k1 y) + R_k2 z) (+ t_k) per component (Eigen on x86-64 SSE2).
 *  1. Window: the map-frame position is R' (px, py, 0) + t' with R' = R^T, t' = -(R' t) (Isometry3d::inverse()); the
 *     length is not transformed.  The window is the one emap_get_submaps cuts there: same cells, centre c, length
 *     L = (rows, cols) * resolution.  A failed window fails here too (info {0, 0, 0}, geometry NaN, no cells).
 *  2. New map: the corners (c_x + L_x / 2, c_y + L_y / 2, 0), (+, -), (-, +), (-, -), in that order, go through T; the
 *     new centre is 0.25 * ((((0 + e0) + e1) + e2) + e3), the new length 2 * max |e_k - centre| per axis; size =
 *     round(length / resolution) (half away from zero), length = size * resolution.  Every cell starts as NaN.
 *  3. Scatter: the window's cells in grid_map order, column-major (i = col * rows + row); a cell whose exported
 *     elevation h is NaN is skipped.  Its samples are p = (x, y, h) with x = (c_x + (0.5 L_x - 0.5 res)) - res * row,
 *     y likewise with col (emap_get_map_points' formula on the window's geometry), and with sample_ratio > 0 four more,
 *     in order (x - s, y, h), (x + s, y, h), (x, y - s, h), (x, y + s, h), s = resolution * sample_ratio (the
 *     unchanged components + 0.0).  Each goes to q = R p + t.  With o = 0.5 * length per axis of the new map and its
 *     centre m: q is inside when 0 <= -((q - m) - o) < length on both axes (checkIfPositionWithinMap), and then lands
 *     on output index trunc(-(((q - o) - m) / resolution)) per axis (getIndexFromPosition), clamped to [0, size - 1]
 *     (grid_map wraps an index of `size`, which only rounding can produce; parity on exact cell boundaries is not
 *     claimed).  A sample is skipped when the target's stored elevation is not NaN and > q.z (the stored float
 *     widened); otherwise the target's elevation becomes float(q.z) and every other layer takes the source cell's
 *     exported value as it is (normals are copied, not rotated, as grid_map does).
 *  The result is that sequential loop's, computed in parallel: a target's elevation is M = max float(q.z) over the
 *  samples that reach it, and its winner is the last sample (in visit order, j = 5 i + k, or i with one sample) with
 *  q.z >= M, else the first with float(q.z) = M.  The node passes sample_ratio 0, which leaves NaN holes at angles other
 *  than multiples of 90 degrees (grid_map's behaviour); e.g. 0.5 fills them.
 * info[3w .. 3w+2] = {success, rows, cols} of the new map; geometry[4w .. 4w+3] = its centre (x, y) in the request
 * frame and its length (x, y).  Output row r, column c of window w is grid_map index (r, c) of its new map (row 0 is the
 * +x edge, column 0 the +y edge of the request frame).  out, out_is_device, out_floats, layers, limits and the stream
 * and graph rules are those of emap_get_submaps, with rows x cols the new map's size; the elevation layer drives the
 * scatter whether or not it is asked for.  Three kernels per EMAP_TRANSFORMED_WINDOWS_PER_LAUNCH windows (their table
 * travels in the kernels' parameters).  The per-cell scratch is the handle's and grows to the largest call (a call
 * that grows it synchronises and cannot be captured: capture after an eager call of the largest size).
 * EMAP_ERR_INVALID, with nothing written or launched, for what emap_get_submaps rejects, a NULL transforms / geometry,
 * a transform as above, a sample_ratio that is not finite and >= 0, and a new map of 2^31 cells or more.
 * emap_transformed_submap_windows: steps 1 and 2 alone, on the host (info and geometry as above), for a map of cell_n
 * cells at `resolution` centred at center; no handle, no device; EMAP_ERR_INVALID for what emap_submap_windows
 * rejects and a transform as above. */
#define EMAP_TRANSFORM_TOLERANCE 1e-6
#define EMAP_TRANSFORMED_WINDOWS_PER_LAUNCH 128
int emap_transformed_submap_windows(int32_t cell_n, double resolution, const double center[2], int32_t n_windows,
                                    const double* windows, const double* transforms, int32_t* info, double* geometry);
int emap_get_transformed_submaps(emap_handle* h, int32_t n_windows, const double* windows, const double* transforms,
                                 double sample_ratio, int32_t n_layers, const char* const* names,
                                 const float* const* planes_device, const int32_t* flags, float* out,
                                 int32_t out_is_device, int64_t out_floats, int32_t* info, double* geometry);
/* ---- plane segmentation of one window: the plane decomposition node's segmented planes map
 * (convex_plane_decomposition_ros: ConvexPlaneDecompositionRos.cpp:115-149, GridMapPreprocessing, then
 * SlidingWindowPlaneExtractor without RANSAC refinement), for one window of the exported elevation.
 *  Window: the one emap_get_submaps cuts for window = (position_x, position_y, length_x, length_y), with its clipping,
 *    success flag and orientation (row 0 the +x edge, column 0 the +y edge); origin = the centre of window cell (0, 0),
 *    centre + (0.5 * n * resolution - 0.5 * resolution) per axis with n = rows / cols (grid_map's getPosition(Index(0, 0))).
 *  Fill (inpainting::minValues): every NaN cell of a 4-connected NaN component takes the minimum of the non-NaN
 *    4-neighbours of the component.  Only NaN is missing; +-inf are values.  -0.0 counts as below +0.0 (minValues'
 *    `<` treats them as equal and keeps the one its scan meets first), so a filled zero may differ in its sign bit.
 *    A window with no finite cell gives info {0, rows, cols, 0, 0} and leaves the layers and the plane table
 *    unwritten; the kernels are launched all the same (they find that out on the device).
 *  Median (smoothing::median): k = max(1, min(median_kernel, 5)), which must be 1, 3 or 5; median_repeats times the
 *    exact median of the k x k values around each cell, border replicated (cv::medianBlur on CV_32F).
 *  Resolution: `resolution` <= 0, or within 1e-6 of the map's, means no resampling; anything else is rejected.
 *  Per-cell fit: the kernel_size x kernel_size window (odd, >= 3) around each cell, cells outside the window and
 *    non-finite heights skipped, points (-kr * res, -kc * res, h) for window row kr, column kc, summed in double.  With
 *    n < 3 points, or the middle eigenvalue of S / n - mean mean^T <= EMAP_PLANE_EIGEN_MIN, the fit is (UnitZ, 1e30);
 *    else the normal is the smallest eigenvalue's eigenvector flipped to z >= 0 and the error that eigenvalue clamped
 *    at 0.  A cell is planar iff its height is finite, error < patch_error^2 and normal.z > local_inclination_cos.
 *  Opening: with opening = r > 0, MORPH_OPEN once with a (2r + 1) cross, border replicated.
 *  Labels: cv::connectedComponents(planar, connectivity 4 or 8): background 0, components 1 .. N - 1 in raster order of
 *    their first cell with connectivity 4, of their first 2 x 2 cell block (blocks in raster order) with 8, as
 *    OpenCV's SAUF and Spaghetti scans number them; highest_label = N - 1.
 *  Per-label fit: the finite cells of label L as points (origin_x - row * res, origin_y - col * res, h).  With fewer
 *    than max(min_points, 3) points the label stays and gets no plane.  Else support = the mean and normal as in the
 *    per-cell fit; normal.z > plane_inclination_cos appends (L, support, normal), labels ascending; otherwise every
 *    cell of L becomes 0.  The sums are exact integer (fixed-point) sums, so support and normal agree with a double
 *    evaluation of the same formulas to rounding (the tests hold them to 1e-9); every other output is exact.
 * layers_out: 4 planes of rows x cols row-major: elevation_raw (the window), elevation (filled and denoised),
 * segmentation (the labels as float) and plane_classification (1.0 where the label is > 0, else 0.0); out_floats >=
 * 4 * rows * cols.  planes_out: 7 doubles per plane (label, support xyz, normal xyz), planes_capacity >=
 * emap_plane_capacity(rows, cols, params) rows (rows * cols always suffices).  info = {success, rows, cols,
 * highest_label, n_planes}; a failed window gives all 0 and writes nothing else.
 * Host output (out_is_device 0): info, the plane table and the layers come back in one device-to-host copy (through
 * the handle's pinned staging) and one synchronisation; only the n_planes rows of planes_out are written.  Device output: layers_out, planes_out and info are device memory, the work is queued on the handle's
 * stream with no host synchronisation (see emap_wait_for_stream / emap_stream_wait_for).  The kernels launched depend on
 * the parameters only, not on the scene.  The map state is not changed.  The scratch is the handle's and grows to the
 * largest window (a call that grows it synchronises).
 * EMAP_ERR_INVALID, with nothing written or launched, for a NULL argument, a length that is not finite and >= 0,
 * ransac != 0, a median kernel or repeat count, resolution, kernel_size, opening or connectivity as above, non-finite
 * cosines or patch error, and an output too small. */
typedef struct emap_plane_params {
  int32_t median_kernel;           /* preprocessing/kernelSize */
  int32_t median_repeats;          /* preprocessing/numberOfRepeats, 0 .. EMAP_PLANE_MAX_REPEATS */
  double resolution;               /* preprocessing/resolution */
  int32_t kernel_size;             /* sliding_window_plane_extractor/kernel_size, odd, 3 .. EMAP_PLANE_MAX_KERNEL */
  int32_t opening;                 /* planarity_opening_filter, 0 .. EMAP_PLANE_MAX_OPENING */
  int32_t min_points;              /* min_number_points_per_label */
  int32_t connectivity;            /* 4 or 8 */
  double plane_inclination_cos;    /* cos(plane_inclination_threshold_degrees) */
  double local_inclination_cos;    /* cos(local_plane_inclination_threshold_degrees) */
  double patch_error;              /* plane_patch_error_threshold [m] */
  int32_t ransac;                  /* include_ransac_refinement: must be 0 */
} emap_plane_params;
#define EMAP_PLANE_EIGEN_MIN 1e-8
#define EMAP_PLANE_MAX_REPEATS 64
#define EMAP_PLANE_MAX_KERNEL 63
#define EMAP_PLANE_MAX_OPENING 64
/* The least planes_capacity for a rows x cols window: rows * cols / max(min_points, 3) (every plane has that many
 * cells); -1 for a NULL params or a negative size. */
int64_t emap_plane_capacity(int64_t rows, int64_t cols, const emap_plane_params* params);
int emap_segment_planes(emap_handle* h, const double window[4], const emap_plane_params* params, float* layers_out,
                        int32_t out_is_device, int64_t out_floats, double* planes_out, int64_t planes_capacity,
                        int32_t* info);
/* ---- planar regions: the plane decomposition node's PlanarTerrain.planarRegions for one window, on the device:
 * ContourExtraction::extractPlanarRegions (plane_segmentation/convex_plane_decomposition) and
 * Postprocessing::addHeightOffset, after emap_segment_planes.  DESIGN.md §4l gives the parallel restatement.
 * Takes everything emap_segment_planes takes and writes the same layers_out, planes_out and info[0 .. 4], byte for
 * byte; then, for a window of R x C >= 2 x 2 cells:
 *  Upsampling: the label image becomes (3R - 2) x (3C - 2) pixels; the first and last source rows and columns take 2
 *    pixels each, every inner one 3.  Pixel (x = column, y = row) is at world (ox - y res / 3, oy - x res / 3), (ox,
 *    oy) the centre of window cell (0, 0).
 *  Per plane row, labels ascending: binary = (up == label) eroded once, BORDER_REPLICATE, by MORPH_ELLIPSE of size
 *    2 (1 + margin_size) + 1 (cv::getStructuringElement's shape).  Boundaries = its polygons; insets = the polygons of
 *    its erosion by the 3 x 3 cross (BORDER_REPLICATE) with the first and last rows and columns cleared.  A polygon is
 *    a cv::findContours(RETR_CCOMP, CHAIN_APPROX_SIMPLE) top-level contour with more than one point, with its child
 *    contours as holes.  A boundary keeps, in inset order, the insets whose first outer vertex is inside it (on an
 *    edge counts as inside); boundaries without an inset are dropped.  When no boundary of the label is kept, the
 *    same is redone from (up == label) eroded once by the 3 x 3 cross (the fallback).
 *  Order (cv2 4.13's RETR_CCOMP order, which the tests pin down): top-level contours by start pixel (the raster-first
 *    pixel of the 8-connected component) descending in raster order, each followed by its holes by start pixel (the
 *    pixel left of the raster-first pixel of the enclosed 4-connected background) descending.
 *  Geometry, in double: every point is mapped to the world as above and projected along gravity into the plane frame
 *    of getTransformLocalToGlobal(support, normal); the region's transform is that one with plane_height_offset added
 *    to its translation z.  bbox = (xmin, ymin, xmax, ymax) of the boundary's outer points in the plane frame.
 * Outputs (emap_region_out): regions, EMAP_REGION_ROW doubles per region: label, the 3 x 4 row-major plane-to-world
 * transform [R | t], bbox.  polygons, EMAP_REGION_POLYGON int32 per polygon: {region, role, inset, first_vertex,
 * n_vertices}; role 0 boundary outer, 1 boundary hole, 2 inset outer, 3 inset hole; inset = the inset's index in its
 * region, -1 for the boundary; per region the boundary outer, its holes, then each inset's outer and its holes.
 * vertices: (x, y) per point in the plane frame, in OpenCV's order.  info = {success, rows, cols, highest_label,
 * n_planes, n_regions, n_polygons, n_vertices, complete}: the counts are always the required totals; when one exceeds
 * its capacity, complete = 0 and no region, polygon or vertex is written (decided on the device).  A window outside
 * the map gives info = {0, ..., 0, 1}; a window with fewer than 2 rows or columns gives n_regions = 0.
 * Host and device output, stream order, graph capture, rejections and the map state as in emap_segment_planes; host
 * output comes back in the same single copy and synchronisation.  The launches depend on the parameters and the
 * window size only.  Scratch: EMAP_REGION_SCRATCH_PER_PIXEL bytes per upsampled pixel on top of emap_segment_planes'
 * (about 1.9 GB for a 2047 x 2047 window).  EMAP_ERR_INVALID, with nothing written or launched, additionally for
 * margin_size outside 0 .. EMAP_REGION_MAX_MARGIN, a non-finite plane_height_offset, a capacity below 0 or above
 * EMAP_REGION_MAX_ROWS, or a NULL table whose capacity is above 0.  With host output the tables are staged at their
 * capacities, so pass capacities near the counts (info[5 .. 7] of an earlier call); a staging that cannot be allocated
 * returns EMAP_ERR_CUDA before anything is launched. */
typedef struct emap_region_params {
  int32_t margin_size;             /* contour_extraction/marginSize, 0 .. EMAP_REGION_MAX_MARGIN */
  double plane_height_offset;      /* postprocessing/extracted_planes_height_offset [m] */
} emap_region_params;
typedef struct emap_region_out {
  double* regions;                 /* EMAP_REGION_ROW doubles per region */
  int64_t regions_capacity;        /* rows */
  int32_t* polygons;               /* EMAP_REGION_POLYGON int32 per polygon */
  int64_t polygons_capacity;
  double* vertices;                /* 2 doubles per vertex */
  int64_t vertices_capacity;
} emap_region_out;
#define EMAP_REGION_MAX_MARGIN 4
#define EMAP_REGION_ROW 17
#define EMAP_REGION_POLYGON 5
#define EMAP_REGION_SCRATCH_PER_PIXEL 49
#define EMAP_REGION_MAX_ROWS 2147483647  /* a table capacity above this (the counts are int32) is rejected */
int emap_extract_planar_regions(emap_handle* h, const double window[4], const emap_plane_params* plane_params,
                                const emap_region_params* region_params, float* layers_out, int32_t out_is_device,
                                int64_t out_floats, double* planes_out, int64_t planes_capacity,
                                const emap_region_out* regions_out, int32_t* info);
/* ---- planar terrain: the grid map of the plane decomposition node's PlanarTerrain message for one window, on the
 * device: Postprocessing::postprocess (convex_plane_decomposition) after emap_extract_planar_regions.  DESIGN.md §4l
 * gives the restatement.  Takes everything emap_extract_planar_regions takes plus post_params and writes the same
 * planes_out, regions, polygons, vertices and info, byte for byte, and layers 0 .. 3 of layers_out as that call does.
 * With res the map's resolution, E layer 1 (elevation) and M layer 3 (plane_classification, 0 or 1):
 *  Kernel sizes (kernelSizeInPixels): 2 (int) round(size / res) + 1 in double, halves away from zero (0.1 / 0.04 =
 *    2.5 gives 7), for the dilation, box and Gauss sizes; each at most EMAP_POST_MAX_KERNEL.
 *  Layer 4 elevationWithNaN = M == 1 ? E : NaN.  Layer 5 elevationWithNaN_i = grid_map's minValues of layer 4 (the fill
 *    of emap_segment_planes; the sign of a filled zero as stated there).  Layer 6 elevationWithNaNClosed =
 *    cv::morphologyEx(MORPH_CLOSE) of layer 5 by MORPH_ELLIPSE of the dilation size, BORDER_REPLICATE.
 *  Layer 7 elevationWithNaNClosedDilated = grid_map_filters_rsl's applyKernelFunction of layer 6 with a k x k window
 *    (k the dilation size, h = (k - 1) / 2) and (data - offsets).maxCoeffOfFinites(): offsets(i, j) =
 *    float(double(float(res)) * sqrt(double((i - h)^2 + (j - h)^2))), the difference in fp32, the window's corner
 *    max(cell - h, 0) moved back to rows - k (cols - k) where the window would overshoot, so a cell within h of the edge
 *    uses a window that is not centred on it.  maxCoeffOfFinites, restated from grid_map's published source (not
 *    checked against a grid_map build): the max over the finite values, NaN when there are none (only when the window
 *    has no planar cell; then layers 4 .. 8 are all NaN).
 *  Layer 8 smooth_planar = cv::boxFilter (normalised, BORDER_REPLICATE) of the box size on layer 7, then
 *    cv::GaussianBlur(ksize, 0, 0, BORDER_REPLICATE) of the Gauss size: the box sums in double times 1 / k^2 (double),
 *    rounded to fp32 (exact, like OpenCV's, while the summed values lie within 29 binary orders of magnitude); the
 *    Gaussian with cv::getGaussianKernel(k, 0, CV_32F)'s coefficients c, rows then columns, each pass c0 x0 + sum over
 *    j of c_j (x_+j + x_-j) in fp32 without contraction: bit-identical to cv2 4.13 for k <= 3.  For a longer kernel
 *    OpenCV's evaluation order is not reproduced; the result differs from cv2's by at most EMAP_POST_GAUSS_ULPS(k) units
 *    in the last place of layer 7's largest magnitude.  That is the worst-case fp32 rounding bound of a k-term sum,
 *    applied to both passes of both evaluations, so it holds for every input and evaluation order (DESIGN.md §4l gives
 *    the derivation and the deviations measured).
 *  Layer 9 elevation: with nonplanar_horizontal_offset > 0, E = M E + (1 - M) D in fp32, D the grey dilation of E by
 *    MORPH_ELLIPSE of 2 offset + 1 (BORDER_REPLICATE); then, when region_params' plane_height_offset (the node's
 *    extracted_planes_height_offset) or nonplanar_height_offset is not 0, E += float(ext + nonpl) and, when nonpl is not
 *    0, E -= float(nonpl) M, each in fp32.  Eigen narrows a double scalar to the float matrix's scalar type before the
 *    operation (promote_scalar_arg in Eigen's XprHelper.h, from Eigen's published source).
 * layers_out: EMAP_TERRAIN_LAYERS planes of rows x cols row-major, out_floats >= EMAP_TERRAIN_LAYERS * rows * cols.
 * Windows outside the map, without a finite cell (nothing but info written) or below 2 x 2 behave as in
 * emap_extract_planar_regions; host output comes back in the same single copy and synchronisation, device output is
 * stream-ordered and can be captured; the launches depend on the parameters and the window size only; the map state is
 * not changed.  The scratch grows emap_segment_planes' block by 20 bytes per cell; with host output the staging at the
 * block's tail and the handle's pinned host buffer each grow by another 24 bytes per cell (six more layers).
 * EMAP_ERR_INVALID, with nothing
 * written or launched, additionally for a NULL post_params, a smoothing size that is not finite and >= 0 or gives a
 * kernel above EMAP_POST_MAX_KERNEL, a horizontal offset outside 0 .. EMAP_POST_MAX_OFFSET, a non-finite
 * nonplanar_height_offset, an out_floats below EMAP_TERRAIN_LAYERS * rows * cols, and a window inside the map with
 * fewer rows or columns than the dilation size. */
typedef struct emap_postprocess_params {
  double nonplanar_height_offset;      /* postprocessing/nonplanar_height_offset [m] */
  int32_t nonplanar_horizontal_offset; /* postprocessing/nonplanar_horizontal_offset [cells], 0 .. EMAP_POST_MAX_OFFSET */
  double smoothing_dilation_size;      /* [m], >= 0 */
  double smoothing_box_kernel_size;    /* [m], >= 0 */
  double smoothing_gauss_kernel_size;  /* [m], >= 0 */
} emap_postprocess_params;
#define EMAP_TERRAIN_LAYERS 10
#define EMAP_POST_MAX_KERNEL 63
#define EMAP_POST_MAX_OFFSET 31
#define EMAP_POST_GAUSS_ULPS(k) (4 * (k) + 1)   /* the bound for a k-tap Gaussian, k >= 5 */
int emap_planar_terrain(emap_handle* h, const double window[4], const emap_plane_params* plane_params,
                        const emap_region_params* region_params, const emap_postprocess_params* post_params,
                        float* layers_out, int32_t out_is_device, int64_t out_floats, double* planes_out,
                        int64_t planes_capacity, const emap_region_out* regions_out, int32_t* info);
/* ---- projection onto the planar regions and convex footholds: convex_plane_decomposition's SegmentedPlaneProjection
 * (getBestPlanarRegionAtPositionInWorld, searched exhaustively as testConvexApproximation.cpp's naive version) and
 * ConvexRegionGrowing (growConvexPolygonInsideShape), for a batch of query points on the device.  DESIGN.md §4l gives
 * the restatement.  tables: the regions, polygons and vertices tables as emap_extract_planar_regions /
 * emap_planar_terrain wrote them (info[8] = complete = 1), in host (tables_on_device 0) or device memory.
 * queries: n_queries world (x, y, z) doubles, host or device.  The handle's map state is not read or changed; the call
 * uses the handle's stream, staging and scratch only.
 * Per query p and region row r (ascending), with [R | t] the region's plane-to-world transform:
 *  Plane frame: q = T^-1 p as Eigen's Isometry3d::inverse() computes it: linear R^T, translation -(R^T t); q_i =
 *    ((A_i0 p0 + A_i1 p1) + A_i2 p2) + u_i, A = R^T, u_i = -((A_i0 t0 + A_i1 t1) + A_i2 t2).
 *  projectToPlanarRegion of (q.x, q.y): the first inset (table order) whose outer polygon contains the point (bounded
 *    side, the boundary counts as inside) keeps it, unless it lies in one of that inset's holes (its boundary counts
 *    as in the hole): then it goes to the first such hole's closest edge.  Inside no inset, it goes to the closest edge
 *    of each inset outer; the inset whose projection c has the least (c.x - q.x)^2 + (c.y - q.y)^2 wins (strict <, the
 *    first from DBL_MAX).  Closest edge of a polygon: the first least CGAL squared distance over its edges in vertex
 *    order (edge k from vertex k to k + 1, the last closing the polygon).  Onto an edge s -> e: v = e - s, L =
 *    sqrt(v.x^2 + v.y^2), n = v / L, coefficient = std::min(std::max(0.0, n . (p - s)), L), result coefficient n + s.
 *  World: w_i = (t_i + x R_i0) + y R_i1.  Cost: ((dx^2 + dy^2) + dz^2) + penalty_z_weight |w_z|, d = p - w.
 *  Result: the first region of least cost (std::min_element over the rows: ties to the lowest row).  The reference's
 *    bounding-box pruning and sort can differ from it only at exact cost ties or sub-ulp violations of its bound; the
 *    device does not prune.
 * Convex growth (n_convex > 0), inside the chosen region's BOUNDARY (outer and holes), around the projected plane
 * point c, with ConvexRegionGrowing.cpp's steps: radius = 0.999 distance(c, boundary) (sqrt of the least squared
 * edge distance, 0 when it is 0); createRegularPolygon (vertex i = (radius cos_i + c.x, radius sin_i + c.y), cos_i and
 * sin_i the host C library's cos / sin of i * ((2 pi) / n_convex)); then at most EMAP_GROW_MAX_ITER sweeps over the
 * unblocked vertices in order: candidate = growth (v - c) + c; it moves when the 5-point sub-polygon (2nd and 1st
 * clockwise neighbours, candidate, 1st and 2nd counter-clockwise neighbours) is convex (CGAL's is_convex_2) and either
 * both neighbours and the candidate lie in the vertex's free circle (squared distance <= squared radius) or neither
 * neighbour-to-candidate segment meets a boundary edge (closed segments); in the second case the free circle becomes
 * (candidate, least squared edge distance).  A move updates the centre c += (1.0 / n) (candidate - v) before v is
 * replaced; a vertex that cannot move is blocked.
 * Arithmetic: every predicate (orientation, bounded side, closed segment intersection, is_convex_2, comparisons) is
 * exact for finite coordinates whose products neither overflow nor underflow (magnitudes and non-zero differences
 * within 2^-480 .. 2^480): a double filter with Shewchuk's orient2d error bound, then expansion arithmetic with
 * TwoSum / TwoProduct (fma).  Bounded side: on a closed edge is the boundary, else the even-odd rule.  Every
 * construction is double arithmetic in the order written here, without contraction.  CGAL's squared distance from a
 * point p to segment s -> e (Distance_2/Point_2_Segment_2.h, line_from_pointsC2, Point_2_Line_2.h) is restated from
 * CGAL's published source and not checked against a CGAL build: d = (p - s) . (e - s); d <= 0 gives |p - s|^2;
 * otherwise with f = |e - s|^2, d > f gives (p.x - e.x)^2 + (p.y - e.y)^2; otherwise (a p.x + b p.y + c)^2 / (a^2 +
 * b^2) with (a, b, c) = (0, 1, -s.y) for a horizontal edge to +x, (0, -1, s.y) to -x, (-1, 0, s.x) for a vertical edge
 * to +y, (1, 0, -s.x) to -y, else (s.y - e.y, e.x - s.x, -s.x a - s.y b).  Eigen's sum orders above are restated from
 * Eigen's published source, not checked against an Eigen build.  The same inputs give the same bits on every call.
 * Outputs (emap_projection_out): index, 3 int32 per query: {region row (-1: none), status, sweeps}; point, 6 doubles:
 * {cost, plane x, y, world x, y, z}; convex (NULL when n_convex is 0), 5 doubles per query and vertex: {plane x, y,
 * world x, y, z} (the world point as above).  Status EMAP_PROJECTION_*: GROWN (also without growth), ZERO_RADIUS (the
 * point is on the boundary: every vertex is the centre, as the reference returns), MAX_ITER (EMAP_GROW_MAX_ITER
 * sweeps ran), NO_REGION (no region), INVALID_QUERY (a non-finite coordinate), BAD_TABLE (device tables that break
 * the layout: see below).  The last three write region -1, cost +inf, NaN positions and NaN vertices.
 * Host tables are checked before anything launches: every polygon row needs a region in range, regions ascending
 * without a gap, roles in the order boundary outer, its holes, then each inset outer followed by its holes (so every
 * region has an inset), inset -1 for the boundary and the running inset index otherwise, at least one vertex and a
 * vertex range inside n_vertices.  Device tables get the same checks on the device; any failure makes every query
 * BAD_TABLE, and no kernel reads outside the counts passed in.
 * Host output comes back in one device-to-host copy and one synchronisation; device output (index, point and convex
 * device memory) is stream-ordered with no host synchronisation and can be captured into a CUDA graph (with device
 * tables and queries; capture after an eager call of the largest size: growing the scratch synchronises).  Host
 * tables or queries are staged and uploaded in one copy.  Kernels: none for n_queries = 0, else 2, plus 1 with
 * n_convex > 0.  One warp per query; the work is the edges of every region's insets per query, plus the boundary's
 * edges per growth step that leaves a free circle.
 * EMAP_ERR_INVALID, with nothing written or launched: a NULL tables / out, a NULL table with a count above 0, NULL
 * queries or outputs with n_queries > 0 (convex with n_convex > 0), a negative count, n_regions, n_polygons or
 * n_queries above 2^31 - 1, n_convex outside 0, 3 .. EMAP_CONVEX_MAX_VERTICES, a growth_factor that is not finite and
 * > 1, a penalty_z_weight that is not finite and >= 0 (the reference's bound needs a non-negative penalty), and host
 * tables that fail the checks above. */
typedef struct emap_region_tables {
  const double* regions;   int64_t n_regions;      /* EMAP_REGION_ROW doubles per region */
  const int32_t* polygons; int64_t n_polygons;     /* EMAP_REGION_POLYGON int32 per polygon */
  const double* vertices;  int64_t n_vertices;     /* 2 doubles per vertex */
} emap_region_tables;
typedef struct emap_projection_out {
  int32_t* index;          /* 3 per query: region row (-1: none), status, growth sweeps */
  double* point;           /* 6 per query: cost, plane-frame x y, world x y z */
  double* convex;          /* 5 per query and vertex: plane-frame x y, world x y z; NULL when n_convex == 0 */
} emap_projection_out;
#define EMAP_CONVEX_MAX_VERTICES 64
#define EMAP_GROW_MAX_ITER 1000   /* ConvexRegionGrowing.cpp's maxIter */
enum { EMAP_PROJECTION_GROWN = 0, EMAP_PROJECTION_ZERO_RADIUS = 1, EMAP_PROJECTION_MAX_ITER = 2,
       EMAP_PROJECTION_NO_REGION = 3, EMAP_PROJECTION_INVALID_QUERY = 4, EMAP_PROJECTION_BAD_TABLE = 5 };
int emap_project_to_planar_regions(emap_handle* h, const emap_region_tables* tables, int32_t tables_on_device,
                                   int64_t n_queries, const double* queries, int32_t queries_on_device,
                                   double penalty_z_weight, int32_t n_convex, double growth_factor,
                                   const emap_projection_out* out, int32_t out_is_device);
/* ---- lookups along lines and derivatives at points on one grid layer: grid_map_filters_rsl's lookup.cpp
 * (maxValueBetweenLocations, valuesBetweenLocations, projectToMapWithMargin) and GridMapDerivative.cpp
 * (estimateGradient, estimateGradientAndCurvature), for a batch of queries on the device.  DESIGN.md §4l gives the
 * restatement.  The handle's map state is not read or changed; the calls use the handle's stream, staging and scratch.
 * Grid (emap_grid): one fp32 layer of rows x cols cells, row-major, grid_map index (r, c) at r * cols + c (row 0 the +x
 * edge, column 0 the +y edge, as every window of this library), in host (grid_on_device 0) or device memory; grid_map
 * geometry position = `position` (the centre of the cells: emap_submap_windows' centre), length L = (rows, cols) *
 * resolution, buffer start index 0.  Index and position arithmetic, restated from grid_map's published GridMapMath.cpp
 * (not checked against a grid_map build), per axis with p the position and o = 0.5 L: a point v is inside when
 * 0 <= -((v - p) - o) < L (checkIfPositionWithinMap), its index is trunc(-(((v - o) - p) / resolution)) clamped to
 * [0, n - 1] (getIndexFromPosition; the same code as emap_get_transformed_submaps'), and index i is at
 * (p + (0.5 L - 0.5 resolution)) - resolution * i (getPositionFromIndex).
 * Lines: queries are n_queries (x0, y0, x1, y1) doubles in the map frame, host or device.  Per line:
 *  Ends: projectToMapWithMargin with the default margin: m = min(1e-6, L.x / 2, L.y / 2), each coordinate
 *    fmax(fmin(v, (p + 0.5 L) - m), (p - 0.5 L) + m).  A NaN coordinate lands on the upper bound (fmin returns the other
 *    operand), +-inf on its bound.  For an accepted grid (|p| + L <= EMAP_GRID_MAX_EXTENT and resolution >=
 *    EMAP_GRID_MIN_RESOLUTION per axis) a projected end is always inside: every intermediate lies below 2^20 in
 *    magnitude, so each of the four roundings between the bound and the inside test is off by at most 2^-33, while
 *    m >= min(1e-6, 2^-21) keeps the exact value at least 4.7e-7 inside.  So LineIterator's getIndexLimitedToMapRange
 *    never steps and its ends are the getIndex cells of the projected ends (tests/test_grid_lookup_cpu.py checks this
 *    at the bounds, edges and corners of extreme grids).
 *  Walk: grid_map's LineIterator (LineIterator.cpp, restated from grid_map's published source, not checked against a
 *    grid_map build): Bresenham from the start cell to the end cell; d = |end - start| per axis, each axis steps +1 when
 *    end >= start, else -1; the major axis is the rows when d.rows >= d.cols; den = d.major, numerator = den / 2, add =
 *    d.minor, den + 1 cells; each step adds `add` to the numerator and, when it is >= den, subtracts den and steps the
 *    minor axis; it always steps the major axis.  Cell i is computed directly: major start + i, minor start +
 *    floor((den / 2 + i add) / den) steps (64-bit; the start cell alone when den is 0).
 *  emap_max_values_between (maxValueBetweenLocations), quirks preserved: value = std::max(value, v) from -FLT_MAX over
 *    the finite cells in order, so on equal values the first is kept (the sign of a largest zero is that of the first
 *    such zero); valid = value > -FLT_MAX (a line whose only finite values are -FLT_MAX is invalid); the returned cell is
 *    the LAST finite cell of the line, not the maximum's (maxIndex is set at every finite cell), and (0, 0) when there
 *    is none; x, y its position.  Outputs (emap_line_max_out): index, 3 int32 per line {valid, row, col}; value, 3
 *    doubles {value (the float widened), x, y}.
 *  emap_values_between (valuesBetweenLocations): (x, y, value) per finite cell, in iterator order, value the float
 *    widened.  Outputs (emap_line_values_out): counts (int32 per line: its rows), first (int64 per line: the exclusive
 *    prefix sum of the counts, where its rows start) and info = {total rows, complete} are always written; rows
 *    (3 doubles per row) only when total <= capacity (complete = 1), decided on the device; otherwise nothing is
 *    written to rows.  Host output reads the total back first (one synchronisation), so the rows' staging is sized
 *    by the total, not the capacity; the rows and the per-line words then come back together (a second one).
 * Derivatives (emap_grid_derivatives): positions are n_queries (x, y) doubles, host or device.  Per position, its
 *  index (r, c) as above; outside the map: status EMAP_DERIVATIVE_OUTSIDE, row = col = -1, zero gradient and curvature
 *  (as GridMapDerivative.hpp documents).  Inside: the kernels d1 = float(-1/12, 2/3, 0, -2/3, 1/12) / float(resolution)
 *  and d2 = float(-1/12, 4/3, -5/2, 4/3, -1/12) / (float(resolution) * float(resolution)), each literal a double rounded
 *  to float, the divisions in float; getKernelCenter's taps rows r0 .. r0 + 4 with r0 = r - 2 - min(r - 2, 0) -
 *  max(r + 2 - (rows - 1), 0), columns c0 .. c0 + 4 likewise (an edge cell gets an off-centre stencil); H(a, b) the
 *  layer.  gx = d1 . H(r0.., c), gy = d1 . H(r, c0..), cxx = d2 . H(r0.., c), cyy = d2 . H(r, c0..), cxy = d1 . g with
 *  g_j = d1 . H(r0.., c0 + j).  Every product and sum is in float without contraction, widened to double at the end (a NaN as the quiet NaN
 *  0x7ff8000000000000, whatever its payload in float).
 *  Eigen's sum orders (restated from Eigen's published source for an SSE build without FMA, not checked against an
 *  Eigen build): a contiguous 5-vector (a column block of the column-major matrix, and g) sums
 *  ((p0 + p2) + (p1 + p3)) + p4; a strided one (a row block) (p0 + p1) + (p2 + (p3 + p4)).  Outputs
 *  (emap_derivative_out): index, 3 int32 per position {status, row, col}; value, 2 doubles {gx, gy}, or with
 *  curvature != 0 5 doubles {gx, gy, cxx, cxy, cyy}.
 * Host grids and queries are staged and uploaded in one copy.  Host output comes back in one copy and synchronisation
 * (emap_values_between: two); device output (every output pointer device memory) is stream-ordered with no host
 * synchronisation and can be captured into a CUDA graph (with a device grid and queries; capture after an eager call of
 * the largest size: growing the scratch synchronises).  Kernels: none for n_queries = 0 (emap_values_between then
 * writes info = {0, 1}); else emap_max_values_between 1 (one warp per line), emap_values_between 3 (count, scan,
 * write; one warp per line), emap_grid_derivatives 1 (one thread per position).
 * EMAP_ERR_INVALID, with nothing written or launched: a NULL grid, out or grid data; rows or cols below 1 (below 5 for
 * emap_grid_derivatives, where the reference's stencil would read outside the layer); rows * cols >= 2^31; a
 * resolution that is not finite or below EMAP_GRID_MIN_RESOLUTION; a position that is not finite; |position| + length
 * above EMAP_GRID_MAX_EXTENT on an axis; n_queries below 0 or above 2^31 - 1; NULL queries or outputs with
 * n_queries > 0; for emap_values_between a NULL info, a capacity below 0 and NULL rows with a capacity above 0. */
typedef struct emap_grid {
  const float* data;       /* rows x cols, row-major */
  int64_t rows, cols;
  double position[2];      /* the centre of the cells, map frame [m] */
  double resolution;       /* [m] */
} emap_grid;
typedef struct emap_line_max_out {
  int32_t* index;          /* 3 per line: valid, row, col */
  double* value;           /* 3 per line: value, x, y */
} emap_line_max_out;
typedef struct emap_line_values_out {
  double* rows;            /* 3 per row: x, y, value */
  int64_t capacity;        /* rows */
  int32_t* counts;         /* 1 per line */
  int64_t* first;          /* 1 per line */
  int64_t* info;           /* {total rows, complete} */
} emap_line_values_out;
typedef struct emap_derivative_out {
  int32_t* index;          /* 3 per position: status, row, col */
  double* value;           /* 2 per position (gx, gy), or 5 with curvature (gx, gy, cxx, cxy, cyy) */
} emap_derivative_out;
#define EMAP_GRID_MAX_EXTENT 1048576.0              /* 2^20 m */
#define EMAP_GRID_MIN_RESOLUTION 9.5367431640625e-07 /* 2^-20 m */
enum { EMAP_DERIVATIVE_INSIDE = 0, EMAP_DERIVATIVE_OUTSIDE = 1 };
int emap_max_values_between(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, int64_t n_queries,
                            const double* lines, int32_t lines_on_device, const emap_line_max_out* out,
                            int32_t out_is_device);
int emap_values_between(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, int64_t n_queries,
                        const double* lines, int32_t lines_on_device, const emap_line_values_out* out,
                        int32_t out_is_device);
int emap_grid_derivatives(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, int64_t n_queries,
                          const double* positions, int32_t positions_on_device, int32_t curvature,
                          const emap_derivative_out* out, int32_t out_is_device);
/* ---- layer values at points: grid_map's GridMap::atPosition(layer, position, method) with nearest, linear and cubic
 * convolution interpolation (GridMap.cpp's atPositionLinearInterpolated, CubicInterpolation.cpp's bicubic_conv;
 * restated from grid_map's published source), for a batch of points and up to EMAP_VALUES_MAX_LAYERS layers of one
 * geometry, on the device.  The cell choice and the operation order below are this library's definition and are
 * tested exactly; bit parity with a grid_map build is not claimed (none was available).
 * Geometry: an emap_grid's, with the lookups' index and position arithmetic above: per axis, a point v is inside when
 *  0 <= -((v - p) - o) < L, its index is trunc(-(((v - o) - p) / resolution)) clamped to [0, n - 1], and index i is at
 *  (p + (0.5 L - 0.5 resolution)) - resolution * i; X(r) and Y(c) below are these positions of row r and column c.
 * Per point (x, y), in IEEE double, every operation rounded on its own (no contraction), the result rounded once to
 * float; F(r, c) is the layer's cell widened to double:
 *  Outside (on either axis, which includes a NaN or infinite coordinate): status EMAP_VALUE_OUTSIDE and every layer the
 *   quiet NaN 0x7fc00000 (grid_map throws here).
 *  (r, c) = the point's cell.  method EMAP_VALUES_NEAREST: F(r, c), status EMAP_VALUE_NEAREST.
 *  Linear (EMAP_VALUES_LINEAR, and the fallback of cubic): r' = r - 1 when x >= X(r), else r + 1; c' = c - 1 when
 *   y >= Y(c), else c + 1.  If r' or c' lies outside [0, rows - 1] / [0, cols - 1], the point falls back to nearest.
 *   Otherwise the corner of lowest x and y is r0 = max(r, r'), c0 = max(c, c'); tx = (x - X(r0)) / resolution,
 *   ty = (y - Y(c0)) / resolution, ux = 1 - tx, uy = 1 - ty; with f0 = F(r0, c0), f1 = F(r0 - 1, c0),
 *   f2 = F(r0, c0 - 1), f3 = F(r0 - 1, c0 - 1):
 *     value = (((f0 ux) uy + (f1 tx) uy) + (f2 ux) ty) + (f3 tx) ty      (grid_map's order), status EMAP_VALUE_LINEAR.
 *   grid_map bounds-checks the four cells by their linear buffer index, so at its edges it can read a wrapped row where
 *   this rule falls back to nearest; that departure is deliberate and not reproduced.
 *  Cubic convolution (EMAP_VALUES_CUBIC; grid_map's INTER_CUBIC_CONVOLUTION, Keys with a = -0.5): r0, c0, tx and ty as
 *   for linear; it needs rows r0 + 1 .. r0 - 2 and columns c0 + 1 .. c0 - 2 inside the grid, else the point falls back
 *   to linear (and from there possibly to nearest).  Weights per axis, t = tx or ty, with grid_map's matrix
 *   M = [[0, 2, 0, 0], [-1, 0, 1, 0], [2, -5, 4, -1], [-1, 3, -3, 1]], t2 = t t, t3 = t2 t:
 *     w_j = 0.5 (((M[0][j] + M[1][j] t) + M[2][j] t2) + M[3][j] t3)           (j = 0 .. 3: f(-1), f(0), f(1), f(2)).
 *   The 1-D pass runs along y for each of the four rows i = 0 .. 3 (row r0 + 1 - i), then along x:
 *     g_i = ((wy_0 F(r, c0 + 1) + wy_1 F(r, c0)) + wy_2 F(r, c0 - 1)) + wy_3 F(r, c0 - 2),
 *     value = ((wx_0 g_0 + wx_1 g_1) + wx_2 g_2) + wx_3 g_3,                              status EMAP_VALUE_CUBIC.
 *  Non-finite cells are not masked: a NaN or +-inf among the cells used propagates by IEEE arithmetic as it does in
 *   grid_map, including 0 * inf = NaN for a zero weight (a point at a cell centre next to an infinite cell is NaN).
 *   Every NaN value is written as 0x7fc00000 (the host and the device give NaNs different payloads).
 *  So at a cell centre with finite neighbours linear and cubic return the cell's value (up to the sign of a zero).
 * Outputs (emap_values_out): values, n_layers x n_points floats, layer-major (layer k of point i at k n_points + i);
 *  status, one int32 per point: the method that produced its values after the fallbacks.
 * emap_grid_values_at: n_layers emap_grids that share rows, cols, position and resolution, every layer's data in host
 *  (grids_on_device 0) or every one in device memory.  Checks: each grid as the lookups check theirs (rows and cols
 *  >= 1).
 * emap_map_values_at: the live map.  The layers are named as for emap_get_layers (a basic name, or planes_device[k] !=
 *  NULL with flags[k]).  The result equals emap_grid_values_at on the full export, bit for bit: the (cell_n - 2)^2
 *  planes of emap_get_layers with position = the map centre's x and y (float) widened to double and the handle's
 *  resolution.  A get_submaps window that covers the whole exported area (at the map centre, lengths >= (cell_n - 2) *
 *  resolution) is that grid: emap_submap_windows reports its centre as center + (0.5 (top + bottom + 1) - 0.5 cell_n)
 *  * resolution with top + bottom + 1 = cell_n, i.e. exactly the map centre.  The cells are read from the map state
 *  (the export is not materialised).  The centre travels in the kernel's parameters, so a captured call is valid only
 *  at its capture centre, as for frames and windows.
 * Both: positions are n_points (x, y) doubles in the map frame, host (positions_on_device 0) or device memory.  One
 *  kernel (one thread per point: the cell, the fallbacks and the weights once, then 1, 4 or 16 cells per layer), none
 *  for n_points = 0.  Host inputs are uploaded in one copy; host output comes back in one copy and one
 *  synchronisation; device output (values and status device memory) is stream-ordered with no host synchronisation and
 *  can be captured into a CUDA graph (with device positions; capture after an eager call of the largest size: growing
 *  the scratch synchronises).  The handle's map state is not changed; the calls use the lookups' staging and scratch.
 *  EMAP_ERR_INVALID, with nothing written or launched: a NULL grids / names / out; n_layers outside
 *  [1, EMAP_VALUES_MAX_LAYERS]; a method other than EMAP_VALUES_*; n_points below 0 or above 2^31 - 1; NULL positions,
 *  values or status with n_points > 0; what the lookups reject for a grid and layers whose geometries differ
 *  (emap_grid_values_at); an unknown layer name (emap_map_values_at). */
#define EMAP_VALUES_MAX_LAYERS 24
enum { EMAP_VALUES_NEAREST = 0, EMAP_VALUES_LINEAR = 1, EMAP_VALUES_CUBIC = 2 };
enum { EMAP_VALUE_OUTSIDE = 0, EMAP_VALUE_NEAREST = 1, EMAP_VALUE_LINEAR = 2, EMAP_VALUE_CUBIC = 3 };
typedef struct emap_values_out {
  float* values;           /* n_layers x n_points, layer-major */
  int32_t* status;         /* 1 per point: EMAP_VALUE_* */
} emap_values_out;
int emap_grid_values_at(emap_handle* h, int32_t n_layers, const emap_grid* grids, int32_t grids_on_device,
                        int64_t n_points, const double* positions, int32_t positions_on_device, int32_t method,
                        const emap_values_out* out, int32_t out_is_device);
int emap_map_values_at(emap_handle* h, int32_t n_layers, const char* const* names, const float* const* planes_device,
                       const int32_t* flags, int64_t n_points, const double* positions, int32_t positions_on_device,
                       int32_t method, const emap_values_out* out, int32_t out_is_device);
/* ---- a signed distance field of one grid layer and distance queries against it, on the device (a legged robot's
 * swing-leg clearance: how far a point is from the terrain and in which direction that distance grows).  DESIGN.md
 * §4l (continued) gives the algorithm.  The handle's map state is not read or changed; the calls use the handle's
 * stream, staging and scratch of the lookups.
 * Field (emap_signed_distance_field): the grid is an emap_grid exactly as the lookups take it (host or device, the same
 *  checks), res its resolution.  Slice k (0 <= k < n_z) lies at z_k = z_min + k * res in double (one multiply, then
 *  one add); the voxels are res apart on all three axes.
 *  Occupancy: a non-finite cell takes the layer's lowest finite value (one device reduction, no host synchronisation;
 *    a layer with no finite cell has no occupied voxel).  Voxel (r, c, k) is occupied iff (double)e(r, c) >= z_k, else
 *    free.  A column's top slice T (the highest occupied slice, -1 for none) is floor((e - z_min) / res) corrected by
 *    the exact comparison, so it agrees with it for every k.
 *  Value: with d2 the exact integer squared Euclidean distance in voxel units between voxel centres, over the voxels
 *    of the volume only, a free voxel holds +fl(sqrt(float(d2)) * float(res)) (correctly rounded float square root and
 *    product) for its nearest occupied voxel, an occupied voxel minus that for its nearest free voxel; +INFINITY
 *    (-INFINITY) when the volume has no voxel of the other kind.
 *  Output: n_z x rows x cols floats, slice after slice, each slice in the grid's row-major layout (slice k reads like a
 *    layer of the grid), in host (out_is_device 0) or device memory; capacity is out's size in floats.
 *  Kernels: 3 (the lowest finite value; the z pass with the envelopes along the columns of every row, one CTA per
 *    row and slice; the envelopes along the rows, one CTA per column and slice, in place in the output).
 * Queries (emap_sdf_values): n points (x, y, z) as doubles, host or device, against a field (emap_sdf: a volume as
 *  emap_signed_distance_field writes it with its grid's geometry and z_min, in host (field_on_device 0) or device
 *  memory).  out: 4 doubles per point {value, d/dx, d/dy, d/dz}.  Every operation is in double, rounded on its own (no
 *  contraction).  Per point:
 *   fractional indices fr = ((p_x + (0.5 L_x - 0.5 res)) - x) / res (the inverse of getPositionFromIndex),
 *     fc = ((p_y + (0.5 L_y - 0.5 res)) - y) / res, fk = (z - z_min) / res, with L = (rows, cols) * res;
 *   per axis of n cells, u = the index clamped to [0, n - 1] (f < 0: 0; f > n - 1: n - 1), i0 = min(floor(u), n - 2)
 *     and i1 = i0 + 1 (both 0 when n = 1), t = u - i0, and off = f - u;
 *   V(k, r, c) the voxel value widened to double; lerp(a, b, t) = a + t * (b - a);
 *   columns: X(k, r) = lerp(V(k, r, c0), V(k, r, c1), tc) and D(k, r) = V(k, r, c1) - V(k, r, c0);
 *   rows: Y(k) = lerp(X(k, r0), X(k, r1), tr), R(k) = X(k, r1) - X(k, r0), E(k) = lerp(D(k, r0), D(k, r1), tr);
 *   slices: value = lerp(Y(k0), Y(k1), tk) + sqrt((off_r^2 + off_c^2) + off_k^2) * res (the distance in metres from the
 *     point to its clamped point, 0 inside the box);
 *   gradient of the interpolant: d/dx = -(lerp(R(k0), R(k1), tk) / res) (the row index grows toward -x),
 *     d/dy = -(lerp(E(k0), E(k1), tk) / res), d/dz = (Y(k1) - Y(k0)) / res; 0 along an axis of one cell.
 *  A NaN coordinate gives four NaNs.  Infinite voxel values (a volume with no voxel of one kind) propagate by IEEE
 *  arithmetic, so such a volume gives infinite or NaN values and NaN gradients.  Every NaN is written as the quiet NaN
 *  0x7ff8000000000000.  Kernels: 1 (one thread per point), none for n = 0.
 * Host grids, fields and points are staged and uploaded in one copy; host output comes back in one copy and
 * synchronisation.  Device output is stream-ordered with no host synchronisation and can be captured into a CUDA graph
 * (with device inputs; capture after an eager call of the largest size: growing the scratch synchronises).
 * EMAP_ERR_INVALID, with nothing written or launched: everything the lookups reject for their grid (emap_sdf_values:
 * for the field's rows, cols, position, resolution and data), n_z below 1, a non-finite z_min,
 * (rows - 1)^2 + (cols - 1)^2 + (n_z - 1)^2 >= EMAP_SDF_MAX_D2 (so that every d2 converts to float exactly),
 * rows * cols * n_z >= 2^31, a NULL out, a capacity below rows * cols * n_z, n below 0 or above 2^31 - 1, and NULL
 * points or out with n > 0. */
#define EMAP_SDF_MAX_D2 16777216   /* 2^24 */
typedef struct emap_sdf {
  const float* data;       /* n_z x rows x cols */
  int64_t rows, cols, n_z;
  double position[2];      /* the centre of the cells, map frame [m] */
  double resolution;       /* [m], also the slice spacing */
  double z_min;            /* the height of slice 0 [m] */
} emap_sdf;
int emap_signed_distance_field(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, double z_min,
                               int64_t n_z, float* out, int64_t capacity, int32_t out_is_device);
int emap_sdf_values(emap_handle* h, const emap_sdf* field, int32_t field_on_device, int64_t n, const double* points,
                    int32_t points_on_device, double* out, int32_t out_is_device);
/* ---- inpainting of an 8-bit image and of a grid layer on the device.  DESIGN.md §4c gives the algorithm.  The
 * handle's map state is not read or changed; the calls use the handle's stream, the lookups' staging and one inpainting
 * scratch block of their own (grown to the largest image, about 37 bytes per padded pixel).
 * emap_inpaint_image: cv2.inpaint(img, mask, radius, flags) for one 8-bit channel, bit for bit.  img, mask and out are
 *  rows x cols bytes, row-major, all three in host (on_device 0) or all three in device memory; a pixel is filled where
 *  its mask byte is non-zero, every other pixel is copied.  radius is rounded as cv::inpaint does (half to even, then at
 *  least 1); only radius 1 is provided, so a radius that rounds above 1 is rejected.
 *   method 0: Telea (INPAINT_TELEA), the device replay emap_inpaint runs; rows and cols >= 2.
 *   method 1: Navier-Stokes (INPAINT_NS); rows and cols >= 1.  On a one-row or one-column image cv2 reads memory
 *     outside the image next to its border and its result is not repeatable; there the reads are clamped to the image.
 *  An image with no masked pixel, or with every pixel masked (no known pixel to start from), comes back unchanged.
 * emap_nonlinear_interpolation: grid_map_filters_rsl's inpainting::nonlinearInterpolation (inpainting.cpp:205-242) on an
 *  emap_grid exactly as the lookups take it (host or device, the same checks), into out (rows x cols floats, host or
 *  device as out_is_device says).  Per call:
 *   mask = isnan(cell); lo / hi = the lowest / highest finite cell (float);
 *   image = grid_map_cv's toImage<uchar, 1>(lo, hi) (restated from its published source, not checked against a
 *     grid_map build): a NaN cell gives 0; every other cell is clamped to [lo, hi] (±inf becomes lo or hi) and gives
 *     (uchar)(((v - lo) / (hi - lo)) * 255.0f) in float, truncated, a NaN quotient giving 0 (x86's conversion);
 *   filled = emap_inpaint_image(image, mask, inpaint_radius / resolution, method 1);
 *   out = fma(filled, (hi - lo) / 255.0f, lo) in float (cv::Mat::convertTo's fused x86 path) in the NaN cells, and
 *     the input bit for bit in every other cell (±inf cells included: they are not NaN, so they are not masked).
 *  Edge cases: a grid with no finite cell comes back unchanged (the reference's scale is then -inf and every filled
 *  value NaN); lo == hi fills every NaN cell with lo (the image is all 0).
 * Host inputs are staged and uploaded in one copy; host output comes back in one copy and synchronisation.  Device output
 * is stream-ordered with no host synchronisation.  Kernels: emap_inpaint_image 4 (setup, band, band flags, one
 * cooperative march), emap_nonlinear_interpolation 6 (the finite range and the image, then those 4, then the write-back).
 * EMAP_ERR_INVALID, with nothing written or launched: a NULL img, mask or out; rows or cols below 1 (below 2 for method
 * 0) or above EMAP_INPAINT_MAX_SIDE; a method other than 0 and 1; a radius that is not finite or rounds above 1; for
 * emap_nonlinear_interpolation everything the lookups reject for their grid, a NULL out, a grid side above
 * EMAP_INPAINT_MAX_SIDE and an inpaint_radius / resolution that is not finite or rounds above 1. */
#define EMAP_INPAINT_MAX_SIDE 8192
int emap_inpaint_image(emap_handle* h, const uint8_t* img, const uint8_t* mask, int64_t rows, int64_t cols,
                       double radius, int32_t method, uint8_t* out, int32_t on_device);
int emap_nonlinear_interpolation(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, double inpaint_radius,
                                 float* out, int32_t out_is_device);
/* ---- plane decomposition of a caller's grid: PlaneDecompositionPipeline::update's grid map part
 * (ConvexPlaneDecompositionRos.cpp:88-162 without RANSAC refinement) on any grid, such as a window of
 * emap_get_submaps or a new map of emap_get_transformed_submaps, with GridMapPreprocessing's resampling
 * (inpainting::resample, grid_map_filters_rsl inpainting.cpp:244-288).  DESIGN.md §4l gives the restatement.
 *  Grid (emap_grid, as the lookups take it): rows x cols fp32 cells, row-major, host (grid_on_device 0: staged in one
 *    upload) or device memory, position = the centre of its cells, resolution res.
 *  Geometry (emap_plane_grid_geometry): with params->resolution <= 0 or within 1e-6 of res the grid is not resampled;
 *    otherwise scaling = res / new_res (double), rows' = int(rows * scaling) and cols' = int(cols * scaling)
 *    (truncating), and the true resolution res' = 0.5 * ((rows * res) / rows' + (cols * res) / cols').  The position is
 *    kept; origin = the centre of cell (0, 0) = position + (0.5 * (n' * res') - 0.5 * res') per axis.
 *  Steps: the fill and the median of emap_segment_planes on the input; then, when the size changes, the resampling
 *    below; then every later step of emap_planar_terrain on the rows' x cols' grid at res' and that origin (the per-cell
 *    fit's res, the per-label origin, the regions' res' / 3 upsampling, kernelSizeInPixels and the sloped dilation's
 *    offsets).
 *  Resampling (cv::resize INTER_LINEAR, as cv2 4.13's default path computes it on x86; DESIGN.md §4l): per axis, for
 *    output index d of m from n cells, f = (d + 0.5) * (n / m) - 0.5 in double, s = floor(f), f -= s; s < 0 or
 *    s >= n - 1 is an edge position that takes cell clamp(s, 0, n - 1) alone; otherwise v = a + float(f) * (b - a) in
 *    fp32 without contraction, a, b cells s and s + 1.  Columns first, on the two source rows of the row taps, then the
 *    rows.  An exact 2x downscale in both axes is this same formula with f = 0.5 everywhere, which is what cv2's
 *    default path computes there, bit for bit.  Against cv2's default path the result is within EMAP_RESAMPLE_ULPS
 *    units in the last place of the input's largest finite magnitude; cv2 takes its scalar path for a source of one
 *    row or column of n cells, and the bound there is EMAP_RESAMPLE_ULPS_LINE(n).  DESIGN.md §4l derives both.  +-inf
 *    inside the grid propagates as in cv2 (inf - inf and 0 * inf are NaN); at edge positions cv2's default path
 *    mixes single and two-tap evaluation, which this restatement does not reproduce.
 * Outputs: emap_planar_terrain's, at rows' x cols': layers_out holds EMAP_TERRAIN_LAYERS planes of rows' x cols' with
 * layer 0 (elevation_raw) left unwritten (in the node it is the grid before the preprocessing, at its own size: the
 * caller's grid); planes, regions, polygons, vertices and info = {success, rows', cols', ...} as there.  A grid with
 * no finite cell gives info[0] = 0.  Host and device output, stream order, graph capture (with a device grid), the
 * capacity rule and the map state as in emap_planar_terrain; the launches depend on the parameters and the sizes
 * only, one more than emap_planar_terrain's when the grid is resampled, and the grid's copy replaces k_submap.
 * EMAP_ERR_INVALID, with nothing written or launched, for everything emap_planar_terrain rejects except the
 * resampling (a NaN resolution is still rejected), the lookups' emap_grid checks, a grid or resampled grid of more
 * than 2047 rows or columns (the largest window, so the scratch never exceeds the window calls'), a resampled size of
 * 0, and a resampled grid with fewer rows or columns than the dilation size. */
#define EMAP_RESAMPLE_ULPS 13
#define EMAP_RESAMPLE_ULPS_LINE(n) (2 * (n) + 6)
/* The resampled size (out_size = {rows', cols'}) and resolution emap_plane_decomposition runs a rows x cols grid of
 * `resolution` at, for params->resolution; out_resolution is 0 when a size is 0.  EMAP_ERR_INVALID for a NULL
 * argument, rows or cols below 1, a resolution that is not finite and > 0, or a NaN params->resolution. */
int emap_plane_grid_geometry(int64_t rows, int64_t cols, double resolution, const emap_plane_params* params,
                             int64_t out_size[2], double* out_resolution);
int emap_plane_decomposition(emap_handle* h, const emap_grid* grid, int32_t grid_on_device,
                             const emap_plane_params* plane_params, const emap_region_params* region_params,
                             const emap_postprocess_params* post_params, float* layers_out, int32_t out_is_device,
                             int64_t out_floats, double* planes_out, int64_t planes_capacity,
                             const emap_region_out* regions_out, int32_t* info);
/* ---- the exported map as a point cloud and as normal arrows: the ROS node's publishAsPointCloud
 * (elevation_mapping_ros.cpp:501-505, grid_map's toPointCloud(map, {"elevation"}, "elevation")) and publishNormalAsArrow
 * (:751-778), restated from grid_map's published source (not checked against a grid_map build).  Coordinates are those of
 * emap_get_layers' output (exported cell (r, c) is state cell (cell_n-2-r, cell_n-2-c)).  Cells are visited in grid_map's
 * storage order, column-major over the exported map: linear index i = c * (cell_n-2) + r.  A cell's position, in double:
 *   x = (cx + (0.5 * L - 0.5 * res)) - res * r,   y = (cy + (0.5 * L - 0.5 * res)) - res * c,
 * with (cx, cy) the handle's fp32 centre widened to double, res the resolution and L = (cell_n-2) * res
 * (getPositionFromIndex with the geometry get_grid_map sets).
 * emap_get_map_points: one row (float x, float y, float z) per cell whose exported elevation is finite, in that order;
 * x and y are the positions rounded to float, z is the exported elevation bit for bit.
 * emap_get_normal_arrows: one arrow per cell whose exported elevation is finite and whose exported normal n is not
 * shorter than 0.1 (skipped when sqrt((nx^2 + ny^2) + nz^2) < 0.1 in double, the reference's test, so a normal that is
 * not a number keeps its arrow; the frame never writes one), in that order.  ids[k] = the cell's linear index i (the
 * marker id); segments[6k .. 6k+5] = (start, end) in double: start = (x, y, elevation), end = start + n * 0.1 per component.
 * *n_points / *n_arrows: the capacity in rows on entry, the number of rows on return.  A capacity below it returns
 * EMAP_ERR_INVALID with the needed number in *n_points / *n_arrows and writes nothing to the rows.  The outputs may be
 * NULL when the capacity is 0 (a count query).  EMAP_ERR_INVALID for a NULL count, a negative capacity or a NULL output
 * with a capacity above 0.  Host output: two synchronisations per call (one for the count, one for the rows); the work
 * is ordered on the handle's stream like the other exports and leaves the map state unchanged. */
int emap_get_map_points(emap_handle* h, float* xyz_host, int64_t* n_points);
int emap_get_normal_arrows(emap_handle* h, int32_t* ids_host, double* segments_host, int64_t* n_arrows);
/* EM.py:807-835 get_layer / raw state access: device pointer of a (W,W) fp32 plane.  Names: the 7
 * layers of EM.py:69-77, normal_x/y/z, traversability_input.  `elevation_map` returns the (7,W,W)
 * base, `normal_map` the (3,W,W) base.  Pointers stay valid until the next emap_move / emap_move_to / emap_destroy. */
int emap_layer_device_ptr(emap_handle* h, const char* name, void** ptr);
int emap_exists_layer(const emap_handle* h, const char* name);  /* EM.py:702-718; 1 / 0 */
/* Bulk state copy (tests, checkpointing): map (7,W,W), normal (3,W,W) fp32, host memory. */
int emap_get_state(emap_handle* h, float* map_host, float* normal_host);
int emap_set_state(emap_handle* h, const float* map_host, const float* normal_host, const double center[3]);

/* ---- polygon safety check: EM.py:837-897 get_polygon_traversability / get_untraversable_polygon (WRAP:254-281, the
 * ROS node's check_safety service).  polygon_xy: n_vertices (x, y) fp32 pairs in host memory, 3 <= n_vertices <=
 * EMAP_POLYGON_MAX_VERTICES.  checker_plane_device: the (W,W) fp32 plane of param.checker_layer, NULL for the
 * traversability layer.  result = {is_safe (1/0), mean untraversability t, shoelace area of the polygon as given}.
 * hull_xy receives the closed ring (first vertex repeated at the end) of the convex hull of the interior cells whose
 * masked untraversability exceeds 1 - safe_thresh, in metres, as rows of (x, y) doubles; *n_hull is its capacity in rows
 * on entry and the ring length on return (0: no polygon).  A capacity below the ring length returns EMAP_ERR_INVALID
 * with the needed length in *n_hull (result is written).  mask_device: optional (W,W) fp32 output of the polygon mask.
 * One device-to-host copy and one synchronisation per call. */
#define EMAP_POLYGON_MAX_VERTICES 1024
int emap_polygon_traversability(emap_handle* h, const float* polygon_xy, int32_t n_vertices,
                                const float* checker_plane_device, double safe_thresh, double safe_min_thresh,
                                int32_t max_unsafe_n, double result[3], double* hull_xy, int32_t* n_hull,
                                float* mask_device);
/* A batch of polygons in one call (CheckSafety.srv's polygons[], is_safe[], traversability[], untraversable_polygons[]).
 * Polygon i has n_vertices[i] vertices (3 to EMAP_POLYGON_MAX_VERTICES); polygon_xy holds all of them as (x, y) fp32
 * pairs, back to back.  results[3i .. 3i + 2] and ring i are what emap_polygon_traversability returns for polygon i
 * on the same map.  hull_xy NULL: no hulls (every ring is empty, less device work); hull_offsets and hull_rows may then
 * be NULL too.  Otherwise ring i is rows [hull_offsets[i], hull_offsets[i + 1]) of hull_xy ((x, y) doubles) and
 * *hull_rows is the capacity in rows on entry and the total on return; a capacity below the total returns
 * EMAP_ERR_INVALID with the needed total in *hull_rows (results and hull_offsets are written).  No mask is written.
 * One host-to-device copy, one device-to-host copy and one synchronisation per call (one more of each of the last two
 * when the rings are long).  The work is proportional to the polygons' bounding boxes plus one pass over the map,
 * except when fp32(1 - safe_thresh) < 0: every cell outside a polygon is then over-threshold too, and every polygon
 * takes the whole map, as the single call does. */
#define EMAP_POLYGON_MAX_BATCH 4096
int emap_polygon_traversability_batch(emap_handle* h, int32_t n_polygons, const int32_t* n_vertices,
                                      const float* polygon_xy, const float* checker_plane_device, double safe_thresh,
                                      double safe_min_thresh, int32_t max_unsafe_n, double* results, double* hull_xy,
                                      int64_t* hull_offsets, int64_t* hull_rows);

/* ---- plugin stencils on device planes (W,W fp32); replace the CuPy / OpenCV / cupyx bodies of
 * plugins/min_filter.py:57-118, plugins/smooth_filter.py:57-58, plugins/inpainting.py:53-63 ---- */
int emap_min_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t dilation_size,
                    int32_t iteration_n, int32_t* iterations_run);
int emap_smooth_filter(emap_handle* h, const float* in, float* out);
/* plugins/max_filter.py:36-113 (Jacobi max-fill), plugins/erosion.py:96-113 (8-bit normalise, cv.erode with a
 * ones(kernel_size) kernel `iterations` times, de-normalise; optional 1-x reversal), and
 * plugins/robot_centric_elevation.py:66-121 (cell height in the base frame, R row-major 3x3). */
int emap_max_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t dilation_size,
                    int32_t iteration_n, int32_t* iterations_run);
int emap_erode(emap_handle* h, const float* layer, float* out, int32_t kernel_size, int32_t iterations, int32_t reverse);
int emap_robot_centric_elevation(emap_handle* h, const float* elevation, const float* is_valid, const float R[9], float* out,
                                 double resolution, double threshold, int32_t use_threshold);
/* plugins/inpainting.py:14-63 (Inpainting plugin; the reference runs cv2.inpaint on the HOST after a D2H copy): 8-bit
 * normalisation over the valid cells, OpenCV's Telea fill with radius 1 of the cells with is_valid < 0.5,
 * de-normalisation; all planes (W,W) fp32 on the device.  method 0 = telea (bit-identical to cv2.inpaint(..., 1,
 * INPAINT_TELEA)); 'ns' is not implemented (EMAP_ERR_INVALID).  With no valid cell the layer is copied (inpainting.py:62). */
int emap_inpaint(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t method);
/* diagnostics of the last emap_inpaint: fast-marching rounds, longest fixed-point iteration, rounds that hit the cap */
int emap_inpaint_stats(emap_handle* h, int32_t* rounds, int32_t* max_jacobi, int32_t* not_converged);

/* ---- semantic plugins: plugins/semantic_filter.py:13-133, plugins/semantic_traversability.py:12-83 and
 * plugins/features_pca.py:13-96.  planes_device is a HOST array of n device pointers to (W,W) fp32 planes; out is a (W,W)
 * fp32 device plane.  The caller selects the planes (the reference's regex / name look-up over its layer stores). ----
 * emap_semantic_filter: per cell the class id = numpy.argmax over the planes (first maximum wins; a NaN is the maximum,
 * the first NaN wins; 0 with no plane), written as the bits of the reference palette entry color_map(255)[id]
 * (r << 16 | g << 8 | b; many are fp32 denormals: read them as uint32). */
#define EMAP_SEMANTIC_FILTER_MAX_LAYERS 255
int emap_semantic_filter(emap_handle* h, int32_t n_layers, const float* const* planes_device, float* out);
/* emap_semantic_traversability: a layer votes where v <= thresholds[l] (is_traversability_type[l] != 0) or v >= thresholds[l]
 * (otherwise), compared in fp64 (the fp32 value widened); NaN never votes.  out = fp32(0.1) where no layer votes, else 1. */
#define EMAP_SEMANTIC_TRAVERSABILITY_MAX_LAYERS 128
int emap_semantic_traversability(emap_handle* h, int32_t n_layers, const float* const* planes_device,
                                 const double* thresholds, const int32_t* is_traversability_type, float* out);
/* emap_features_pca: exact PCA (3 components) of the n_features planes clipped to [-1, 1], every cell a sample,
 * 3 <= n_features <= EMAP_PCA_MAX_FEATURES.  Statistics, eigen-decomposition (Jacobi) and projection in fp64 and in a
 * fixed order (the result is the same every call); each component's largest-|entry| coordinate is positive (sklearn's
 * svd_flip).  out = bits of uint8(trunc((p - min) / (max - min) * 255)) per component packed r << 16 | g << 8 | b; a
 * component of range 0 gives channel 0.  NaN input returns EMAP_ERR_INVALID.  Four kernels and ONE synchronisation, at
 * the end of the call, to read the NaN flag. */
#define EMAP_PCA_MAX_FEATURES 64
int emap_features_pca(emap_handle* h, int32_t n_features, const float* const* planes_device, float* out);

/* ---- camera image fusion: EM.py:468-562 input_image (WRAP:180-185) with semantic_map.py:261-309 update_layers_image,
 * kernels/custom_image_kernels.py:9-157 and fusion/image_color.py / image_exponential.py.
 * image: (n_planes, height, width) fp32, host (is_device_ptr 0) or device memory; height * width <= 2^24.
 * K (3x3 row-major), R (3x3, map -> camera optical frame, row-major), t (3): fp32.  D: n_D distortion coefficients,
 * padded / truncated to 5 (fewer than 4: none) and used only when distortion_model is "radtan".
 * The library computes P = K [R | t] and the camera cell uint32(cell_n / 2 + (-R^T t - center) / resolution) in fp32
 * (products rounded, sums left to right).  A cell is fused where its is_valid is exactly 1, it projects in front of the
 * camera into the image (radtan applied when D is not all zero), and no valid cell on the Bresenham line to the camera
 * cell rises more than 0.10 above the ray.  Fused channel k then writes layer[k] of the caller's (n_layers, W, W) fp32
 * device buffer at that cell, from pixel int(u) + int(v) * width:
 *   EMAP_IMAGE_COLOR:       bits (r << 16) + (g << 8) + b of planes 0, 1, 2 (each converted float -> uint32);
 *   EMAP_IMAGE_EXPONENTIAL: fp32(layer * (1 - 0.7) + 0.7 * image[plane[k]]), in double.
 * Every other cell keeps its value.  Channels are applied in order.  Bit-identical to the reference's kernels built by
 * nvcc for sm_90a.  EMAP_ERR_INVALID for NULL arguments, height * width > 2^24, a colour channel with fewer than 3
 * planes, a plane >= n_planes, a layer outside [0, n_layers), non-finite K, R or t, and a camera cell outside [0, 2^24).
 * One kernel per call.  A host image is copied into pinned staging (the caller may reuse its buffer on return) and to
 * the device once; a device image is read in place and the call does not synchronise with the host. */
#define EMAP_IMAGE_MAX_CHANNELS 64
enum { EMAP_IMAGE_COLOR = 0, EMAP_IMAGE_EXPONENTIAL = 1 };
int emap_input_image(emap_handle* h, int32_t n_planes, const float* image, int is_device_ptr, int32_t height, int32_t width,
                     const float K[9], const float* D, int32_t n_D, const char* distortion_model, const float R[9],
                     const float t[3], int32_t n_fused, const int32_t* plane, const int32_t* kind, const int32_t* layer,
                     float* semantic_map_device, int32_t n_layers);

/* ---- plumbing ---- */
int emap_sync(emap_handle* h);
int emap_stream(emap_handle* h, void** cuda_stream);
/* Run this handle's work on a caller-owned stream (e.g. the framework's current stream); NULL restores
 * the handle's own stream.
 *
 * A frame (emap_input_pointcloud / emap_input_sensors) from device memory makes no host synchronisation, and one from
 * page-locked host memory waits only for the kernel that reads the cloud (not while the stream is being captured), so
 * either can be captured into a CUDA graph on that stream.  The graph binds, at capture:
 *   - the cloud pointer(s), row counts, row stride and dtype (a replay reads the same memory again: keep it alive and
 *     write the next cloud into it; a page-locked host cloud is read over PCIe at every replay);
 *   - the sensor pose relative to the map centre at capture (and the ray box derived from it);
 *   - the semantic configuration (emap_semantic_configure*) and ray counting (emap_set_ray_counting).
 * The state buffer itself keeps its address for the handle's lifetime (moves shift it in place), so moves, ticks and
 * other calls may run between capture and replay.  A replay is valid only at the capture centre, bit for bit: move back
 * to it (emap_get_position) before replaying.  A replay runs after what is already queued on the stream it is launched
 * on; order it after the caller's other streams, as emap_wait_for_stream does for eager calls.
 * Invalidates a graph: any call that grows the handle's buffers (a frame with more points or sensors than any frame
 * before it, a new semantic configuration, more class_max slots): run an eager frame of the largest size and
 * configuration first, then capture.  Cannot be captured: pageable host clouds (staged with a synchronising copy). */
int emap_set_stream(emap_handle* h, void* cuda_stream);
/* ---- layer filters on a caller's grid: grid_map_filters_rsl's inpainting::minValues (inpainting.cpp:25-94),
 * smoothing::median, boxBlur and gaussianBlur (smoothing.cpp) and processing::dilate, erode and outline (processing.cpp)
 * on an emap_grid exactly as the lookups take it (host or device, the same checks), into out (rows x cols floats, host or
 * device as out_is_device says; it must not overlap the grid or the mask).  The handle's map is neither read nor
 * changed.  Results are compared NaN-aware: every non-NaN cell bit for bit, NaN where the reference has NaN (the
 * device's NaN payload is its own).  f->op and its parameters (k = kernel_size):
 *  EMAP_FILTER_MIN_VALUES: every NaN cell takes the least value (±inf included, -0.0 before +0.0) of the non-NaN cells
 *   4-adjacent to its 4-connected NaN component: the fixed point of the reference's in-place sweep.  A component with
 *   no such neighbour (a grid with no non-NaN cell) stays NaN.  Kernels: 5.
 *  EMAP_FILTER_MEDIAN (k, delta_kernel_size, number_of_repeats): with k + delta (repeats - 1) <= 5, repeats of
 *   cv::medianBlur on CV_32F with the kernel k + delta i of repeat i (each 1, 3 or 5; 1 copies), border replicated: the
 *   exact median of each window's values, bit-identical to cv2 where the window holds no NaN.  On a layer with NaN
 *   holes this path is NOT cv2's: every cell whose window holds a NaN may differ (on a grid a quarter NaN, about half
 *   the cells at k = 3).  cv2's sorting network moves a NaN by its SIMD or scalar code path, so its own result there
 *   depends on the column; here a NaN cell stays NaN and the network passes over the other NaNs.
 *   Otherwise toImage<uchar, 1> between the finite minimum lo and maximum hi (emap_nonlinear_interpolation's
 *   quantisation; nothing finite: lo = FLT_MAX, hi = -FLT_MAX), repeats of the 8-bit cv::medianBlur (each kernel odd,
 *   1 .. EMAP_FILTER_MAX_KERNEL) and out = fma(u8, (hi - lo) / 255.0f, lo) into every cell, NaN cells included, as the
 *   reference converts back.  Kernels: one per repeat with a kernel above 1, plus 3 on the 8-bit path.
 *  EMAP_FILTER_BOX_BLUR (k, number_of_repeats): repeats of cv::blur((k, k)), BORDER_REFLECT_101, in OpenCV's order:
 *   row sums in double (k <= 5: each window left to right; else the running sum s += x[c + k] - x[c]), then one
 *   running double sum per column from the top border row down, float(s * (1.0 / k^2)).  NaN and inf propagate down a
 *   column as in cv2.  k may be even (anchor k / 2).  Kernels: 2 per repeat.
 *  EMAP_FILTER_GAUSSIAN_BLUR (k odd, or 0 with sigma > 0, sigma): cv::GaussianBlur((k, k), sigma), BORDER_REFLECT_101;
 *   k = 0 takes cv2's size for a float image, cvRound(8 sigma + 1) | 1.  The coefficients of
 *   cv::getGaussianKernel(k, sigma, CV_32F) (sigma <= 0: from k), rows then columns, c0 x0 + sum c_j (x_+j + x_-j) in
 *   fp32 without contraction.  Bit-identical to cv2 4.13 for k <= 3 with sigma <= 0, NaN and ±inf included; otherwise
 *   within EMAP_POST_GAUSS_ULPS(k) units in the last place of the grid's largest finite magnitude (finite grids).
 *   Kernels: 2.
 *  EMAP_FILTER_DILATE / EMAP_FILTER_ERODE (k, mask, inpaint): processing.cpp's k x k window, its corner max(cell -
 *   (k - 1) / 2, 0) pulled back to rows - k (cols - k) where it would overshoot, over in * mask (fp32; in alone with a
 *   NULL mask).  m = block.maxCoeffOfFinites() (minCoeffOfFinites) as Eigen's redux computes it: grid_map's functor
 *   op(a, b) (restated from its published FunctorsPlugin.hpp: the finite operand when only one is finite, else
 *   std::max(a, b) = a < b ? b : a, or std::min(a, b) = b < a ? b : a) folded over the window's cells from its first,
 *   down each column, column after column.  So m is the window's largest (least) finite value, the earliest in that
 *   order on a tie (the sign of a zero is the earliest zero's); a window with no finite value gives NaN when its first
 *   cell is NaN, else the window's largest (least) infinity.  out = m, or the cell's own value where m is NaN; with
 *   inpaint = 0 a NaN cell stays NaN.  rows and cols must be >= k.  Kernels: 2 (the columns' folds, then the rows'; a
 *   window with no finite value is folded cell by cell in the second).
 *  EMAP_FILTER_OUTLINE: a cell whose clamped 3 x 3 window holds a NaN keeps its value; every other cell becomes NaN.
 *   rows and cols must be >= 3.  Kernels: 1.
 * mask: NULL or rows x cols floats on the grid's side; only dilate and erode read it.  Host inputs (grid, mask) are
 * uploaded in one copy; host output comes back in one copy and one synchronisation.  Device output is stream-ordered
 * with no host synchronisation.
 * EMAP_ERR_INVALID, with nothing written or launched: everything the lookups reject for their grid; a NULL f or out; an
 * unknown op; a kernel size below 1 (a Gaussian's 0 with sigma > 0 excepted) or above EMAP_FILTER_MAX_KERNEL (for the
 * Gaussian's 0, the size from sigma above it), or even where cv2 needs it odd (median, Gaussian;
 * a median kernel sequence that leaves 1 .. EMAP_FILTER_MAX_KERNEL, or a float median kernel other than 1, 3 and 5); a
 * non-positive number_of_repeats (median, box); a sigma that is not finite; a dilate, erode or outline window larger
 * than the grid.
 * Not provided: inpainting::biLinearInterpolation (its weights come from Eigen's float colPivHouseholderQr and its
 * fallback runs nonlinearInterpolation at 2 pixels, which emap_nonlinear_interpolation rejects),
 * processing::applyKernelFunction (it takes a C++ callable) and any plugin or parameter-file wiring. */
#define EMAP_FILTER_MIN_VALUES 0
#define EMAP_FILTER_MEDIAN 1
#define EMAP_FILTER_BOX_BLUR 2
#define EMAP_FILTER_GAUSSIAN_BLUR 3
#define EMAP_FILTER_DILATE 4
#define EMAP_FILTER_ERODE 5
#define EMAP_FILTER_OUTLINE 6
#define EMAP_FILTER_MAX_KERNEL 63
typedef struct emap_filter_op {
  int32_t op;                  /* EMAP_FILTER_* */
  int32_t kernel_size;         /* median, box, Gaussian, dilate, erode */
  int32_t delta_kernel_size;   /* median: the kernel's growth per repeat */
  int32_t number_of_repeats;   /* median, box */
  double sigma;                /* Gaussian */
  int32_t inpaint;             /* dilate, erode */
} emap_filter_op;
int emap_grid_filter(emap_handle* h, const emap_grid* grid, int32_t grid_on_device, const emap_filter_op* f,
                     const float* mask, float* out, int32_t out_is_device);

/* Stream ordering WITHOUT host synchronisation between the handle's stream and a stream of the caller's framework
 * (torch / CuPy current stream; NULL = the legacy default stream): after emap_wait_for_stream the handle's next work runs
 * after everything queued on `cuda_stream` so far (the caller wrote a buffer the library will read); after
 * emap_stream_wait_for, work queued on `cuda_stream` from now on runs after everything the handle has queued so far
 * (the caller will read a layer the library wrote).  The reference has one implicit stream (CuPy's current stream);
 * these two calls are what keeps that ordering when the library runs on its own stream. */
int emap_wait_for_stream(emap_handle* h, void* cuda_stream);
int emap_stream_wait_for(emap_handle* h, void* cuda_stream);
int emap_cell_n(const emap_handle* h);
/* Number of kernels this library has launched on the handle since creation (bench.py gpu_launches). */
int64_t emap_launch_count(const emap_handle* h);
/* Device milliseconds of the last frame's kernels by stage (CUDA events on the handle's stream):
 * out[0..7] = index+error, drift, fusion, record, raycast, finalise, post(dilate+CNN+normal), total. */
int emap_enable_stage_timing(emap_handle* h, int enable);
int emap_get_stage_ms(emap_handle* h, float out[8]);

#ifdef __cplusplus
}
#endif
#endif /* EMAP_H_ */
