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


class EmapExchange(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("count", C.c_int64), ("kind", C.c_int32)]


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
    "emap_point_record_device_ptr": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "emap_get_frame_stats": (C.c_int, [C.c_void_p, C.POINTER(EmapFrameStats)]),
    "emap_set_ray_counting": (C.c_int, [C.c_void_p, C.c_int]),
    "emap_wait_for_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_stream_wait_for": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_shard_begin": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int64,
                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float]),
    "emap_shard_scratch_bytes": (C.c_int64, [C.c_void_p]),
    "emap_shard_attach": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    "emap_shard_set_overlap_z": (C.c_int, [C.c_void_p, C.c_float]),
    "emap_shard_exchange": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(EmapExchange), C.POINTER(C.c_int32)]),
    "emap_shard_phase": (C.c_int, [C.c_void_p, C.c_int32]),
    "emap_comm_unique_id": (C.c_int, [C.c_void_p]),
    "emap_comm_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "emap_input_sensors_sharded": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int64,
                                             C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_float]),
    "emap_move_to": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "emap_move": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_clear": (C.c_int, [C.c_void_p]),
    "emap_update_variance": (C.c_int, [C.c_void_p]),
    "emap_update_time": (C.c_int, [C.c_void_p]),
    "emap_update_normal": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_initialize_map_finish": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "emap_get_position": (C.c_int, [C.c_void_p, C.c_void_p]),
    "emap_get_map_with_name": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "emap_export_plane": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64]),
    "emap_get_layers": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int32),
                                  C.c_void_p, C.c_int64]),
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
