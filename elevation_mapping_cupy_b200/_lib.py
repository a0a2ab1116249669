"""ctypes binding of libemap.so (include/emap.h).  The library must be present: the product path has
no CPU or PyTorch fallback, and importing this module without the built extension raises."""
import ctypes as C
import os

PKG = os.path.dirname(os.path.abspath(__file__))
# EMAP_LIB selects an experimental build variant (tools/ A/B runs); the product is libemap.so
LIB_PATH = os.environ.get("EMAP_LIB") or os.path.join(PKG, "libemap.so")

EMAP_ABI_VERSION = 1
EMAP_F32, EMAP_F64 = 0, 1


class EmapConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "abi_version", "cell_n", "dilation_size", "enable_edge_sharpen", "enable_drift_compensation",
        "enable_visibility_cleanup", "enable_overlap_clearance", "use_only_above_for_upper_bound")] + [
        (n, C.c_double) for n in (
            "resolution", "sensor_noise_factor", "mahalanobis_thresh", "outlier_variance",
            "drift_compensation_variance_inlier", "traversability_inlier", "wall_num_thresh",
            "min_height_drift_cnt", "max_ray_length", "cleanup_step", "cleanup_cos_thresh",
            "min_valid_distance", "max_height_range", "ramped_height_range_a", "ramped_height_range_b",
            "ramped_height_range_c", "max_variance", "initial_variance", "max_drift",
            "drift_compensation_alpha", "position_noise_thresh", "orientation_noise_thresh",
            "overlap_clear_range_xy", "overlap_clear_range_z", "time_variance", "time_interval")]


class EmapFrameStats(C.Structure):
    _fields_ = [("mean_error", C.c_float), ("additive_mean_error", C.c_float), ("shift_applied", C.c_float),
                ("error_sum", C.c_float), ("error_cnt", C.c_int64), ("drift_applied", C.c_int32),
                ("drift_evaluated", C.c_int32), ("n_points", C.c_int64), ("n_valid_points", C.c_int64),
                ("ray_steps", C.c_int64), ("ray_visits", C.c_int64)]


class EmapPlaneParams(C.Structure):
    _fields_ = [("median_kernel", C.c_int32), ("median_repeats", C.c_int32), ("resolution", C.c_double),
                ("kernel_size", C.c_int32), ("opening", C.c_int32), ("min_points", C.c_int32),
                ("connectivity", C.c_int32), ("plane_inclination_cos", C.c_double),
                ("local_inclination_cos", C.c_double), ("patch_error", C.c_double), ("ransac", C.c_int32)]


class EmapRegionParams(C.Structure):
    _fields_ = [("margin_size", C.c_int32), ("plane_height_offset", C.c_double)]


class EmapPostprocessParams(C.Structure):
    _fields_ = [("nonplanar_height_offset", C.c_double), ("nonplanar_horizontal_offset", C.c_int32),
                ("smoothing_dilation_size", C.c_double), ("smoothing_box_kernel_size", C.c_double),
                ("smoothing_gauss_kernel_size", C.c_double)]


EMAP_TERRAIN_LAYERS = 10


class EmapRegionOut(C.Structure):
    _fields_ = [("regions", C.c_void_p), ("regions_capacity", C.c_int64), ("polygons", C.c_void_p),
                ("polygons_capacity", C.c_int64), ("vertices", C.c_void_p), ("vertices_capacity", C.c_int64)]


class EmapRegionTables(C.Structure):
    _fields_ = [("regions", C.c_void_p), ("n_regions", C.c_int64), ("polygons", C.c_void_p),
                ("n_polygons", C.c_int64), ("vertices", C.c_void_p), ("n_vertices", C.c_int64)]


class EmapProjectionOut(C.Structure):
    _fields_ = [("index", C.c_void_p), ("point", C.c_void_p), ("convex", C.c_void_p)]


EMAP_CONVEX_MAX_VERTICES = 64
PROJECTION_STATUS = ("grown", "zero_radius", "max_iter", "no_region", "invalid_query", "bad_table")


class EmapGrid(C.Structure):
    _fields_ = [("data", C.c_void_p), ("rows", C.c_int64), ("cols", C.c_int64), ("position", C.c_double * 2),
                ("resolution", C.c_double)]


class EmapFilterOp(C.Structure):
    _fields_ = [("op", C.c_int32), ("kernel_size", C.c_int32), ("delta_kernel_size", C.c_int32),
                ("number_of_repeats", C.c_int32), ("sigma", C.c_double), ("inpaint", C.c_int32)]


EMAP_FILTER_OPS = {"min_values": 0, "median": 1, "box_blur": 2, "gaussian_blur": 3, "dilate": 4, "erode": 5,
                   "outline": 6}


class EmapLineMaxOut(C.Structure):
    _fields_ = [("index", C.c_void_p), ("value", C.c_void_p)]


class EmapLineValuesOut(C.Structure):
    _fields_ = [("rows", C.c_void_p), ("capacity", C.c_int64), ("counts", C.c_void_p), ("first", C.c_void_p),
                ("info", C.c_void_p)]


class EmapDerivativeOut(C.Structure):
    _fields_ = [("index", C.c_void_p), ("value", C.c_void_p)]


EMAP_DERIVATIVE_INSIDE, EMAP_DERIVATIVE_OUTSIDE = 0, 1


class EmapValuesOut(C.Structure):
    _fields_ = [("values", C.c_void_p), ("status", C.c_void_p)]


EMAP_VALUES_MAX_LAYERS = 24
EMAP_VALUES_METHODS = {"nearest": 0, "linear": 1, "cubic": 2}
VALUE_STATUS = ("outside", "nearest", "linear", "cubic")


class EmapSdf(C.Structure):
    _fields_ = [("data", C.c_void_p), ("rows", C.c_int64), ("cols", C.c_int64), ("n_z", C.c_int64),
                ("position", C.c_double * 2), ("resolution", C.c_double), ("z_min", C.c_double)]


EMAP_SDF_MAX_D2 = 1 << 24


class EmapDepthCamera(C.Structure):
    _fields_ = [("height", C.c_int32), ("width", C.c_int32), ("depth", C.c_void_p), ("confidence", C.c_void_p),
                ("rgb", C.c_void_p), ("features", C.c_void_p), ("fx", C.c_double), ("fy", C.c_double),
                ("cx", C.c_double), ("cy", C.c_double), ("R", C.c_float * 9), ("t", C.c_float * 3)]


EMAP_DEPTH_MAX_CAMERAS = 16


class EmapExchange(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("count", C.c_int64), ("kind", C.c_int32)]


EMAP_SHARD_MAX_EXCHANGES = 5


# every symbol include/emap.h declares, with its argument types
SIGNATURES = {
    "emap_create": (C.c_int, [C.POINTER(EmapConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "emap_destroy": (C.c_int, [C.c_void_p]),
    "emap_last_error": (C.c_char_p, [C.c_void_p]),
    "emap_set_traversability_weights": (C.c_int, [C.c_void_p] + [C.c_void_p] * 4),
    "emap_input_pointcloud": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_float, C.c_float]),
    "emap_input_sensors": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int64,
                                     C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_float]),
    "emap_get_point_record": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    "emap_semantic_configure": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                          C.c_double]),
    "emap_semantic_configure_ext": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_int32]),
    "emap_input_depth_images": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(EmapDepthCamera), C.c_int, C.c_int32, C.c_void_p,
                                          C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float]),
    "emap_input_depth_image": (C.c_int, [C.c_void_p, C.POINTER(EmapDepthCamera), C.c_int, C.c_int32, C.c_void_p, C.c_int32,
                                         C.c_float, C.c_float, C.c_float, C.c_float]),
    "emap_point_record_device_ptr": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "emap_get_frame_stats": (C.c_int, [C.c_void_p, C.POINTER(EmapFrameStats)]),
    "emap_set_ray_counting": (C.c_int, [C.c_void_p, C.c_int]),
    "emap_wait_for_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_stream_wait_for": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_shard_begin": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int64,
                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float]),
    "emap_shard_begin_depth_images": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(EmapDepthCamera), C.c_int, C.c_int32,
                                                C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_int64, C.c_float,
                                                C.c_float]),
    "emap_shard_scratch_bytes": (C.c_int64, [C.c_void_p]),
    "emap_shard_attach": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    "emap_shard_set_overlap_z": (C.c_int, [C.c_void_p, C.c_float]),
    "emap_shard_exchange": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(EmapExchange), C.POINTER(C.c_int32)]),
    "emap_shard_phase": (C.c_int, [C.c_void_p, C.c_int32]),
    "emap_comm_unique_id": (C.c_int, [C.c_void_p]),
    "emap_comm_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "emap_input_sensors_sharded": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int64,
                                             C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_float]),
    "emap_input_depth_images_sharded": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(EmapDepthCamera), C.c_int, C.c_int32,
                                                  C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_int64, C.c_float,
                                                  C.c_float, C.c_float]),
    "emap_move_to": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_move": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_clear": (C.c_int, [C.c_void_p]),
    "emap_update_variance": (C.c_int, [C.c_void_p]),
    "emap_update_time": (C.c_int, [C.c_void_p]),
    "emap_update_normal": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_initialize_map_finish": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "emap_initialize_map": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                      C.c_double, C.c_int32]),
    "emap_get_position": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_get_map_with_name": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "emap_get_layers": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int32),
                                  C.c_void_p, C.c_int64]),
    "emap_submap_windows": (C.c_int, [C.c_int32, C.c_double, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_get_submaps": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_void_p),
                                   C.POINTER(C.c_int32), C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "emap_transformed_submap_windows": (C.c_int, [C.c_int32, C.c_double, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p]),
    "emap_get_transformed_submaps": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_double, C.c_int32,
                                               C.POINTER(C.c_char_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int32),
                                               C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "emap_plane_capacity": (C.c_int64, [C.c_int64, C.c_int64, C.c_void_p]),
    "emap_segment_planes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                      C.c_int64, C.c_void_p]),
    "emap_extract_planar_regions": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                              C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "emap_planar_terrain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "emap_project_to_planar_regions": (C.c_int, [C.c_void_p, C.POINTER(EmapRegionTables), C.c_int32, C.c_int64,
                                                 C.c_void_p, C.c_int32, C.c_double, C.c_int32, C.c_double,
                                                 C.POINTER(EmapProjectionOut), C.c_int32]),
    "emap_max_values_between": (C.c_int, [C.c_void_p, C.POINTER(EmapGrid), C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                          C.POINTER(EmapLineMaxOut), C.c_int32]),
    "emap_values_between": (C.c_int, [C.c_void_p, C.POINTER(EmapGrid), C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                      C.POINTER(EmapLineValuesOut), C.c_int32]),
    "emap_grid_derivatives": (C.c_int, [C.c_void_p, C.POINTER(EmapGrid), C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                        C.c_int32, C.POINTER(EmapDerivativeOut), C.c_int32]),
    "emap_grid_values_at": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(EmapGrid), C.c_int32, C.c_int64, C.c_void_p,
                                      C.c_int32, C.c_int32, C.POINTER(EmapValuesOut), C.c_int32]),
    "emap_map_values_at": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_void_p),
                                     C.POINTER(C.c_int32), C.c_int64, C.c_void_p, C.c_int32, C.c_int32,
                                     C.POINTER(EmapValuesOut), C.c_int32]),
    "emap_signed_distance_field": (C.c_int, [C.c_void_p, C.POINTER(EmapGrid), C.c_int32, C.c_double, C.c_int64,
                                             C.c_void_p, C.c_int64, C.c_int32]),
    "emap_sdf_values": (C.c_int, [C.c_void_p, C.POINTER(EmapSdf), C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                  C.c_void_p, C.c_int32]),
    "emap_inpaint_image": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_double, C.c_int32,
                                     C.c_void_p, C.c_int32]),
    "emap_nonlinear_interpolation": (C.c_int, [C.c_void_p, C.POINTER(EmapGrid), C.c_int32, C.c_double, C.c_void_p,
                                               C.c_int32]),
    "emap_grid_filter": (C.c_int, [C.c_void_p, C.POINTER(EmapGrid), C.c_int32, C.POINTER(EmapFilterOp), C.c_void_p,
                                   C.c_void_p, C.c_int32]),
    "emap_plane_grid_geometry": (C.c_int, [C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_plane_decomposition": (C.c_int, [C.c_void_p, C.POINTER(EmapGrid), C.c_int32, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64,
                                           C.c_void_p, C.c_void_p]),
    "emap_get_map_points": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]),
    "emap_get_normal_arrows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]),
    "emap_layer_device_ptr": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "emap_exists_layer": (C.c_int, [C.c_void_p, C.c_char_p]),
    "emap_get_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_set_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_min_filter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                  C.POINTER(C.c_int32)]),
    "emap_smooth_filter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_max_filter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                  C.POINTER(C.c_int32)]),
    "emap_erode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "emap_robot_centric_elevation": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_double, C.c_double, C.c_int32]),
    "emap_inpaint": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]),
    "emap_inpaint_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "emap_semantic_filter": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "emap_semantic_traversability": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_features_pca": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "emap_input_image": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_int32, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_int32]),
    "emap_polygon_traversability": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_double, C.c_double,
                                              C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p]),
    "emap_polygon_traversability_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_double, C.c_double, C.c_int32, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.POINTER(C.c_int64)]),
    "emap_sync": (C.c_int, [C.c_void_p]),
    "emap_stream": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "emap_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_cell_n": (C.c_int, [C.c_void_p]),
    "emap_launch_count": (C.c_int64, [C.c_void_p]),
    "emap_enable_stage_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "emap_get_stage_ms": (C.c_int, [C.c_void_p, C.c_void_p]),
}

_lib = None


def load():
    """Load libemap.so (built in-tree by elevation_mapping_cupy_b200/build.py).  Raises if missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m elevation_mapping_cupy_b200.build` "
                "(nvcc, sm_90a).  There is no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


class EmapError(RuntimeError):
    pass


def check(lib, handle, rc):
    if rc != 0:
        msg = lib.emap_last_error(handle)
        msg = msg.decode() if msg else ""
        if rc == -3:
            raise KeyError(msg)
        raise EmapError(f"libemap error {rc}: {msg}")
