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
  int64_t n_points;            /* points in the frame (NaN rows included) */
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
 * n_channels = 0 switches it off.  Not applied to sharded frames. */
int emap_semantic_configure(emap_handle* h, int32_t n_channels, const int32_t* column, const int32_t* kind,
                            const int32_t* layer, float* semantic_map_device, int32_t n_layers, double average_weight);
/* CK.py:260-262 write-back of the last frame, on the DEVICE: one packed int32 per input row (bits 0..23 cell index,
 * bit 28 valid, bit 29 inside, bit 30 row dropped as NaN); valid until the next frame. */
int emap_point_record_device_ptr(emap_handle* h, const int32_t** packed_device, int64_t* n);

/* ---- sharded frame (one rank per GPU, replicated grid; SURVEY 8(e)).  Between the phases the
 * caller all-reduces the exchange buffers in place (SUM for the int64/uint32 words named
 * "sum", MAX / MIN as named) with NCCL; single-GPU callers never need these. ---- */
typedef struct emap_exchange {
  void* ptr;        /* device pointer */
  int64_t count;    /* number of elements */
  int32_t kind;     /* 0: int64 SUM, 1: int64 MAX (keys < 2^63), 2: int32 MIN (keys offset to signed order), 3: int32 SUM */
} emap_exchange;
int emap_shard_begin(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n,
                     int64_t row_stride, int dtype, int is_device_ptr, const float* R, const float* t,
                     int64_t global_point_offset, float position_noise, float orientation_noise);
/* NVLink-multicast mode (replaces the three all-reduces): the caller allocates one symmetric block of
 * emap_shard_scratch_bytes() per rank (e.g. torch.distributed._symmetric_memory), rendezvouses it and hands
 * the library its own base and the MULTICAST alias.  From then on every per-cell accumulation of the frame
 * kernels is a single `multimem.red` that the NVSwitch applies to the replicas of all ranks -- the scatter and
 * the collective are one instruction.  Frame = emap_shard_begin, barrier, phase 0 (index), barrier, phase 1,
 * barrier, phase 2, barrier, phase 3; the barriers are the caller's (stream-ordered, cross-rank). */
int64_t emap_shard_scratch_bytes(const emap_handle* h);
int emap_shard_attach(emap_handle* h, void* local_base, void* multicast_base, int64_t bytes);
/* Height reference of clear_overlap_map (EM.py:400-401) for a sharded frame: the absolute z of the
 * FIRST sensor of the whole frame (rank 0's), so that every replica clears the same cells.  Call
 * between emap_shard_begin and phase 3; without it a rank uses its own first sensor. */
int emap_shard_set_overlap_z(emap_handle* h, float sensor_z_absolute);
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
/* EM.py:899-922 initialize_map, device half: after the caller has written the interpolated elevation / variance /
 * is_valid planes (emap_set_state; the interpolation itself is SciPy's griddata on the host in the reference too,
 * map_initializer.py:25-62), run `iterations` passes of the initialiser's dilation (CK.py:392-449 with
 * dilation_size_initialize, mask = is_valid) and update_upper_bound_with_valid_elevation (EM.py:428-432). */
int emap_initialize_map_finish(emap_handle* h, int32_t dilation_size_initialize, int32_t iterations);
int emap_get_position(emap_handle* h, double out[3]);          /* EM.py:130-137 */

/* ---- export: EM.py:720-775 get_map_with_name_ref (WRAP:205-252): NaN-fill, +center_z, crop the
 * border ring, flip both axes; writes (cell_n-2)^2 floats to caller memory.  Names: elevation,
 * variance, traversability, time, upper_bound, is_upper_bound, normal_x, normal_y, normal_z. ---- */
int emap_get_map_with_name(emap_handle* h, const char* name, float* out_host, int64_t n_out);
/* EM.py:579-596,762-775 for a plugin layer: process_map_for_publish(fill_nan, add_z) of an arbitrary
 * (W,W) fp32 device plane, then crop + flip + copy to the host. */
int emap_export_plane(emap_handle* h, const float* plane_device, int fill_nan, int add_z, float* out_host,
                      int64_t n_out);
/* Batched export: what WRAP:213-252 (ElevationMappingWrapper::get_grid_map) does layer by layer -- n layers with ONE
 * kernel, one device-to-host copy, one synchronisation.  names[k] is a basic layer of emap_get_map_with_name, or
 * planes[k] a (W,W) device plane (plugin layer) exported with flags[k] (bit 0: fill_nan, bit 1: add the centre height).
 * out_host holds n consecutive (cell_n-2)^2 planes. */
int emap_get_layers(emap_handle* h, int32_t n, const char* const* names, const float* const* planes_device,
                    const int32_t* flags, float* out_host, int64_t n_out_total);
/* EM.py:807-835 get_layer / raw state access: device pointer of a (W,W) fp32 plane.  Names: the 7
 * layers of EM.py:69-77, normal_x/y/z, traversability_input.  `elevation_map` returns the (7,W,W)
 * base, `normal_map` the (3,W,W) base.  Pointers stay valid until the next emap_move / emap_move_to / emap_destroy. */
int emap_layer_device_ptr(emap_handle* h, const char* name, void** ptr);
int emap_exists_layer(const emap_handle* h, const char* name);  /* EM.py:702-718; 1 / 0 */
/* Bulk state copy (tests, checkpointing): map (7,W,W), normal (3,W,W) fp32, host memory. */
int emap_get_state(emap_handle* h, float* map_host, float* normal_host);
int emap_set_state(emap_handle* h, const float* map_host, const float* normal_host, const double center[3]);

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

/* ---- plumbing ---- */
int emap_sync(emap_handle* h);
int emap_stream(emap_handle* h, void** cuda_stream);
/* Run this handle's work on a caller-owned stream (e.g. the framework's current stream); NULL restores
 * the handle's own stream. */
int emap_set_stream(emap_handle* h, void* cuda_stream);
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
