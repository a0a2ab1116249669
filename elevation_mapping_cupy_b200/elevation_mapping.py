"""Drop-in `ElevationMap` for the fusion path, implemented over libemap.so (hand-written sm_90a CUDA).

Mirrors the public surface of the reference class
(elevation_mapping_cupy/script/elevation_mapping_cupy/elevation_mapping.py:49-922, "EM.py" below):
same method names, positional signatures and error behaviour, so the C++ bridge
(elevation_mapping_cupy/src/elevation_mapping_wrapper.cpp:173-324) and the reference's tests
(script/elevation_mapping_cupy/tests/test_elevation_mapping.py) can drive it unchanged.  All compute
happens in the library; this module only marshals arguments.  Device arrays are handed out as torch
CUDA tensors that alias the library's memory (they also expose `__cuda_array_interface__`).

Point-cloud semantic layers (average / class_average / color fusion) are fused inside the frame (semantic_map.py).
Out of scope (SURVEY.md section 8): image input, image / bayesian semantic fusion, polygon safety check.
"""
import ctypes as C
import threading
from typing import List

import numpy as np

from . import _lib
from .parameter import Parameter
from .plugins.plugin_manager import PluginManager
from .semantic_map import SemanticMap

LAYER_NAMES = ["elevation", "variance", "is_valid", "traversability", "time", "upper_bound", "is_upper_bound"]
EXPORT_NAMES = ["elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
                "normal_x", "normal_y", "normal_z"]


def config_from_parameter(param: Parameter) -> _lib.EmapConfig:
    cfg = _lib.EmapConfig()
    cfg.abi_version = _lib.EMAP_ABI_VERSION
    cfg.cell_n = int(param.cell_n)
    cfg.dilation_size = int(param.dilation_size)
    for k in ("enable_edge_sharpen", "enable_drift_compensation", "enable_visibility_cleanup",
              "enable_overlap_clearance", "use_only_above_for_upper_bound"):
        setattr(cfg, k, int(bool(getattr(param, k))))
    for name, _ in _lib.EmapConfig._fields_[8:]:
        setattr(cfg, name, float(getattr(param, name)))
    return cfg


class _DevView:
    """Minimal __cuda_array_interface__ carrier for a library-owned device buffer."""

    def __init__(self, ptr, shape, owner):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 3, "strides": None}
        self._owner = owner


def _device_pointer(x):
    """(ptr, n_rows, row_stride, dtype_code, keepalive) for a device array, or None."""
    cai = getattr(x, "__cuda_array_interface__", None)
    if cai is None:
        return None
    if cai["typestr"] not in ("<f4", "<f8") or len(cai["shape"]) != 2:
        raise TypeError("device point cloud must be a 2-D float32/float64 array")
    esz = 4 if cai["typestr"] == "<f4" else 8
    n, k = cai["shape"]
    strides = cai.get("strides")
    if strides is not None and (strides[1] != esz or strides[0] % esz):
        raise TypeError("device point cloud must have unit column stride")
    row = k if strides is None else strides[0] // esz
    return int(cai["data"][0]), int(n), int(row), (_lib.EMAP_F32 if esz == 4 else _lib.EMAP_F64), x


class ElevationMap:
    """Core elevation mapping class (EM.py:49)."""

    def __init__(self, param: Parameter, device: int = 0):
        self.param = param
        if param.cell_n is None:
            param.update()
        self.data_type = np.float32
        self.resolution = param.resolution
        self.map_length = param.map_length
        self.cell_n = param.cell_n
        self.layer_names = list(LAYER_NAMES)
        self.initial_variance = param.initial_variance
        self.map_lock = threading.Lock()
        self.device = device
        self._L = _lib.load()
        self._h = C.c_void_p()
        cfg = config_from_parameter(param)
        rc = self._L.emap_create(C.byref(cfg), device, C.byref(self._h))
        if rc != 0:
            raise _lib.EmapError(f"emap_create failed ({rc}): {self._L.emap_last_error(None).decode()}")
        # EM.py:103-104 traversability weights
        if not (np.any(param.w1) or np.any(param.w_out)):
            param.load_weights(param.weight_file)
        ws = [np.ascontiguousarray(w, dtype=np.float32).reshape(-1) for w in (param.w1, param.w2, param.w3, param.w_out)]
        self._check(self._L.emap_set_traversability_weights(self._h, *[w.ctypes.data for w in ws]))
        # EM.py:112-115 plugins
        self.plugin_manager = PluginManager(cell_n=self.cell_n, engine=self)
        if param.plugin_config_file:
            self.plugin_manager.load_plugin_settings(param.plugin_config_file)
        self.semantic_map = SemanticMap(param, engine=self)              # EM.py:106
        self.base_rotation = np.eye(3, dtype=np.float32)
        self._export_tmp = np.zeros((self.cell_n - 2, self.cell_n - 2), np.float32)

    # ---- plumbing -------------------------------------------------------------------------
    def _check(self, rc):
        _lib.check(self._L, self._h, rc)

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                self._L.emap_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def close(self):
        self.__del__()

    def synchronize(self):
        self._check(self._L.emap_sync(self._h))

    def set_stream(self, cuda_stream_handle):
        """Run this handle's kernels on a caller-owned CUDA stream (int handle, e.g. torch.cuda.Stream().cuda_stream);
        None / 0 restores the handle's own stream.  A frame fed from device memory is a fixed sequence of launches with
        no host synchronisation, so it can be captured into a CUDA graph on that stream."""
        self._check(self._L.emap_set_stream(self._h, C.c_void_p(int(cuda_stream_handle or 0))))

    def _after_framework(self):
        """The handle's next work runs after everything the caller's framework (torch / CuPy current stream) has queued:
        buffers it wrote are complete, kernels of its that still read the aliased layers are done.  No host sync."""
        st = _framework_stream()
        if st is not None:
            self._check(self._L.emap_wait_for_stream(self._h, C.c_void_p(st)))

    def _before_framework(self):
        """Work the caller's framework queues from now on runs after everything this handle has queued.  No host sync."""
        st = _framework_stream()
        if st is not None:
            self._check(self._L.emap_stream_wait_for(self._h, C.c_void_p(st)))

    def _ptr(self, name):
        p = C.c_void_p()
        self._check(self._L.emap_layer_device_ptr(self._h, name.encode(), C.byref(p)))
        return p.value

    def _tensor(self, name, shape):
        import torch
        self._before_framework()      # torch work on the view is ordered after the library's (no host sync)
        return torch.as_tensor(_DevView(self._ptr(name), shape, self), device=f"cuda:{self.device}")

    @property
    def elevation_map(self):
        """(7, W, W) fp32 state, layer order EM.py:69-77; torch CUDA tensor aliasing library memory."""
        return self._tensor("elevation_map", (7, self.cell_n, self.cell_n))

    @property
    def normal_map(self):
        return self._tensor("normal_map", (3, self.cell_n, self.cell_n))

    @property
    def traversability_input(self):
        return self._tensor("traversability_input", (self.cell_n, self.cell_n))

    @property
    def center(self):
        out = np.zeros(3, np.float64)
        self._check(self._L.emap_get_position(self._h, out.ctypes.data))
        return out.astype(np.float32)

    @property
    def mean_error(self):
        return self.get_frame_stats().mean_error

    @property
    def additive_mean_error(self):
        return self.get_frame_stats().additive_mean_error

    # ---- mutators (EM.py:119-226, 420-466, 564-577) ------------------------------------------
    def clear(self):
        with self.map_lock:
            self._after_framework()
            self._check(self._L.emap_clear(self._h))
            self.semantic_map.clear()                              # EM.py:126

    def get_position(self, position):
        out = np.zeros(3, np.float64)
        self._check(self._L.emap_get_position(self._h, out.ctypes.data))
        position[0][:] = out

    def move(self, delta_position):
        d = np.ascontiguousarray(np.asarray(delta_position, dtype=np.float64).reshape(3))
        with self.map_lock:
            self._after_framework()
            self._check(self._L.emap_move(self._h, d.ctypes.data))
            if self.semantic_map.layer_names:                     # EM.py:221 semantic layers move with the map
                px = np.rint(d[:2] / self.resolution).astype(int)
                self._before_framework()
                self.semantic_map.shift_map_xy((int(px[0]), int(px[1])))

    def move_to(self, position, R):
        p = np.ascontiguousarray(np.asarray(position, dtype=np.float64).reshape(3))
        Rm = np.ascontiguousarray(_to_host(R), dtype=np.float32).reshape(9)
        self.base_rotation = Rm.reshape(3, 3).copy()
        with self.map_lock:
            shift = None
            if self.semantic_map.layer_names:                     # same cell shift as emap_move_to computes (EM.py:164-170)
                px = np.rint((p[:2] - self.center[:2].astype(np.float64)) / self.resolution).astype(int)
                shift = (-int(px[0]), -int(px[1]))
            self._after_framework()
            self._check(self._L.emap_move_to(self._h, p.ctypes.data, Rm.ctypes.data))
            if shift is not None:
                self._before_framework()
                self.semantic_map.shift_map_xy(shift)

    def update_variance(self):
        self._after_framework()
        self._check(self._L.emap_update_variance(self._h))

    def update_time(self):
        self._after_framework()
        self._check(self._L.emap_update_time(self._h))

    def update_normal(self, dilated_map):
        """EM.py:564-577.  `dilated_map`: a (W,W) fp32 device array (torch / cupy) or None."""
        ptr = None
        if dilated_map is not None:
            cai = getattr(dilated_map, "__cuda_array_interface__", None)
            if cai is None or cai["typestr"] != "<f4" or tuple(cai["shape"]) != (self.cell_n, self.cell_n):
                raise TypeError("update_normal expects a (cell_n, cell_n) float32 device array")
            ptr = cai["data"][0]
            self._after_framework()
        with self.map_lock:
            self._check(self._L.emap_update_normal(self._h, ptr))

    def input_pointcloud(self, raw_points, channels: List[str], R, t, position_noise: float, orientation_noise: float):
        """EM.py:434-466.  raw_points: (N, 3+k) host (numpy / torch CPU, float32 or float64) or device
        (torch CUDA / cupy) array.  Channels beyond x, y, z are fused into semantic layers inside the frame
        (semantic_map.py:223-259; algorithms average / class_average / color)."""
        if channels is not None and (len(channels) > 3 or self.semantic_map._configured is not None):
            self.semantic_map.configure_for(list(channels))
        Rm = np.ascontiguousarray(_to_host(R), dtype=np.float32).reshape(9)
        tv = np.ascontiguousarray(_to_host(t), dtype=np.float32).reshape(3)
        dev = _device_pointer(raw_points)
        with self.map_lock:
            if dev is not None:
                ptr, n, row, dt, _keep = dev
                self._after_framework()
                rc = self._L.emap_input_pointcloud(self._h, ptr, n, row, dt, 1, Rm.ctypes.data, tv.ctypes.data,
                                                   float(position_noise), float(orientation_noise))
            else:
                pts = _to_host(raw_points)
                if pts.dtype not in (np.float32, np.float64):
                    pts = pts.astype(np.float32)
                if pts.ndim != 2 or pts.shape[1] < 3:
                    raise ValueError("raw_points must be (N, >=3)")
                if not pts.flags.c_contiguous:
                    pts = np.ascontiguousarray(pts)
                dt = _lib.EMAP_F32 if pts.dtype == np.float32 else _lib.EMAP_F64
                self._after_framework()       # framework kernels still reading the aliased layers finish first
                rc = self._L.emap_input_pointcloud(self._h, pts.ctypes.data, pts.shape[0], pts.shape[1], dt, 0,
                                                   Rm.ctypes.data, tv.ctypes.data, float(position_noise),
                                                   float(orientation_noise))
            self._check(rc)

    # the pure-Python ROS node of the reference still calls `.input(...)` (elevation_mapping_ros.py:212)
    input = input_pointcloud

    def input_sensors(self, clouds, Rs, ts, position_noise, orientation_noise, device_ptrs=False):
        """Several sensors of one time slice fused against the same snapshot (SURVEY 8(e))."""
        ns = len(clouds)
        keep, ptrs, counts = [], (C.c_void_p * ns)(), (C.c_int64 * ns)()
        stride = dt = None
        for i, c in enumerate(clouds):
            dev = _device_pointer(c) if device_ptrs else None
            if dev is not None:
                ptr, n, row, d, k = dev
            else:
                a = np.ascontiguousarray(_to_host(c))
                if a.dtype not in (np.float32, np.float64):
                    a = a.astype(np.float32)
                ptr, n, row, d, k = a.ctypes.data, a.shape[0], a.shape[1], (_lib.EMAP_F32 if a.dtype == np.float32 else _lib.EMAP_F64), a
            if stride is None:
                stride, dt = row, d
            elif (stride, dt) != (row, d):
                raise ValueError("all sensor clouds must share row stride and dtype")
            keep.append(k); ptrs[i] = ptr; counts[i] = n
        Rm = np.ascontiguousarray(np.stack([np.asarray(_to_host(r), np.float32).reshape(9) for r in Rs]))
        tm = np.ascontiguousarray(np.stack([np.asarray(_to_host(t), np.float32).reshape(3) for t in ts]))
        if device_ptrs:
            self._after_framework()
        with self.map_lock:
            self._check(self._L.emap_input_sensors(self._h, ns, ptrs, counts, stride, dt, int(bool(device_ptrs)),
                                                   Rm.ctypes.data, tm.ctypes.data, float(position_noise),
                                                   float(orientation_noise)))

    # ---- queries -------------------------------------------------------------------------------
    def get_additive_mean_error(self):
        return self.get_frame_stats().additive_mean_error

    def get_frame_stats(self):
        st = _lib.EmapFrameStats()
        self._check(self._L.emap_get_frame_stats(self._h, C.byref(st)))
        return st

    def get_point_record(self, n):
        idx = np.zeros(n, np.int32); valid = np.zeros(n, np.uint8); inside = np.zeros(n, np.uint8)
        self._check(self._L.emap_get_point_record(self._h, idx.ctypes.data, valid.ctypes.data, inside.ctypes.data, n))
        return idx, valid, inside

    def exists_layer(self, name):
        """EM.py:702-718"""
        return (name in self.layer_names or name in self.semantic_map.layer_names
                or name in self.plugin_manager.layer_names)

    def get_layer(self, name):
        """EM.py:807-835: the (W,W) device layer (torch CUDA tensor)."""
        if name in self.layer_names:
            return self.elevation_map[self.layer_names.index(name)]
        if name in self.semantic_map.layer_names:
            self._before_framework()
            return self.semantic_map.semantic_map[self.semantic_map.layer_names.index(name)]
        if name in self.plugin_manager.layer_names:
            self._update_plugin(name)
            return self.plugin_manager.get_map_with_name(name)
        print("Layer {} is not in the map, returning traversabiltiy!".format(name))
        return None

    def _update_plugin(self, name):
        self.plugin_manager.update_with_name(name, self.elevation_map, self.layer_names, self.semantic_map.semantic_map,
                                             self.semantic_map.layer_names, self.base_rotation, self.semantic_map.elements_to_shift)

    def get_map_with_name_ref(self, name, data):
        """EM.py:720-775: write layer `name` (NaN-filled, z-shifted, cropped, flipped) into `data`,
        a caller-owned (cell_n-2, cell_n-2) float32 array."""
        n_out = (self.cell_n - 2) ** 2
        direct = isinstance(data, np.ndarray) and data.dtype == np.float32 and data.flags.c_contiguous and data.size == n_out
        buf = data if direct else self._export_tmp
        with self.map_lock:
            if name in EXPORT_NAMES:
                self._check(self._L.emap_get_map_with_name(self._h, name.encode(), buf.ctypes.data, n_out))
            elif name in self.semantic_map.layer_names:
                # EM.py:747-748: semantic layers are exported as they are (cropped, flipped), no NaN fill, no z offset
                m = self.semantic_map.semantic_map[self.semantic_map.layer_names.index(name)]
                self._after_framework()
                self._check(self._L.emap_export_plane(self._h, m.data_ptr(), 0, 0, buf.ctypes.data, n_out))
            elif name in self.plugin_manager.layer_names:
                self._update_plugin(name)
                m = self.plugin_manager.get_map_with_name(name)
                p = self.plugin_manager.get_param_with_name(name)
                self._after_framework()
                self._check(self._L.emap_export_plane(self._h, m.data_ptr(), int(p.fill_nan), int(p.is_height_layer),
                                                      buf.ctypes.data, n_out))
            else:
                print("Layer {} is not in the map".format(name))
                return
        if not direct:
            data[...] = buf.reshape(data.shape)

    def get_maps_with_names_ref(self, names, data):
        """Several layers at once (what the C++ bridge's get_grid_map does one by one, elevation_mapping_wrapper.cpp:213-252):
        `data` is a caller-owned (len(names), cell_n-2, cell_n-2) float32 array.  One kernel, one D2H copy, one sync."""
        n = len(names)
        n_out = (self.cell_n - 2) ** 2
        direct = isinstance(data, np.ndarray) and data.dtype == np.float32 and data.flags.c_contiguous and data.size == n * n_out
        buf = data if direct else np.zeros((n, self.cell_n - 2, self.cell_n - 2), np.float32)
        c_names = (C.c_char_p * n)(); planes = (C.c_void_p * n)(); flags = (C.c_int32 * n)()
        keep = []
        with self.map_lock:
            for k, name in enumerate(names):
                if name in EXPORT_NAMES:
                    c_names[k] = name.encode(); planes[k] = None
                elif name in self.plugin_manager.layer_names:
                    self._update_plugin(name)
                    m = self.plugin_manager.get_map_with_name(name)
                    p = self.plugin_manager.get_param_with_name(name)
                    keep.append(m)
                    c_names[k] = name.encode(); planes[k] = m.data_ptr()
                    flags[k] = int(bool(p.fill_nan)) | (int(bool(p.is_height_layer)) << 1)
                else:
                    raise KeyError("Layer {} is not in the map".format(name))
            if keep:
                self._after_framework()
            self._check(self._L.emap_get_layers(self._h, n, c_names, planes, flags, buf.ctypes.data, n * n_out))
        if not direct:
            data[...] = buf.reshape(data.shape)

    def get_state(self):
        """Host copies (map (7,W,W), normal (3,W,W)) -- tests / checkpointing."""
        W = self.cell_n
        m = np.zeros((7, W, W), np.float32); nm = np.zeros((3, W, W), np.float32)
        self._check(self._L.emap_get_state(self._h, m.ctypes.data, nm.ctypes.data))
        return m, nm

    def set_state(self, elevation_map, normal_map=None, center=None):
        m = np.ascontiguousarray(elevation_map, np.float32)
        nm = None if normal_map is None else np.ascontiguousarray(normal_map, np.float32)
        c = None if center is None else np.ascontiguousarray(center, np.float64)
        self._after_framework()
        self._check(self._L.emap_set_state(self._h, m.ctypes.data, None if nm is None else nm.ctypes.data,
                                           None if c is None else c.ctypes.data))

    def launch_count(self):
        return int(self._L.emap_launch_count(self._h))

    def enable_stage_timing(self, on=True):
        self._check(self._L.emap_enable_stage_timing(self._h, int(on)))

    def stage_ms(self):
        out = np.zeros(8, np.float32)
        self._check(self._L.emap_get_stage_ms(self._h, out.ctypes.data))
        return out

    # ---- not on the per-frame path ---------------------------------------------------------------
    def input_image(self, *a, **k):
        raise NotImplementedError("image input is outside the fusion path (SURVEY.md section 8)")

    def get_polygon_traversability(self, *a, **k):
        raise NotImplementedError("polygon safety check is outside the fusion path (SURVEY.md section 8)")

    def initialize_map(self, points, method="cubic"):
        """EM.py:899-922 + map_initializer.py:25-62: clear the map, interpolate the given (x, y, z) points (map frame) over
        the grid with scipy.interpolate.griddata ON THE HOST -- exactly what the reference does (it copies to NumPy for
        griddata) -- then, on the device, dilate twice with dilation_size_initialize and set upper_bound to the elevation
        of the valid cells.  Start-up path, not on the per-frame path."""
        from scipy.interpolate import griddata
        self.clear()
        pts = np.array(_to_host(points), dtype=np.float32, copy=True)
        center = self.center
        W = self.cell_n
        # transform_to_map_index (traversability_polygon.py:61-63): truncation toward zero, like astype(int32)
        idx = ((pts[:, :2] - center[:2].reshape(1, 2)) / np.float32(self.resolution) + W / 2).astype(np.int32)
        pts[:, :2] = idx.astype(np.float32)
        pts[:, 2] -= center[2]
        state, normal = self.get_state()
        vi = np.where(state[2] > 0.5)
        points_idx = np.vstack([np.stack(vi).T.astype(np.float32), pts[:, :2]])
        values = np.hstack([state[0][vi], pts[:, 2]])
        assert points_idx.shape[0] > 3, "Initialization points must be more than 3."
        gx, gy = np.mgrid[0:W, 0:W]
        interp = griddata(points_idx, values, (gx, gy), method=method)
        ok = ~np.isnan(interp)
        state[0] = np.nan_to_num(interp).astype(np.float32)
        state[1] = np.where(ok, np.float32(self.param.initialized_variance), np.float32(self.param.initial_variance))
        state[2] = ok.astype(np.float32)
        with self.map_lock:
            self.set_state(state)
            self._check(self._L.emap_initialize_map_finish(self._h, int(self.param.dilation_size_initialize), 2))


def _to_host(x):
    if isinstance(x, np.ndarray):
        return x
    if hasattr(x, "detach") and hasattr(x, "cpu"):      # torch tensor
        return x.detach().cpu().numpy()
    if hasattr(x, "get"):                                # cupy array
        return x.get()
    return np.asarray(x)


def _framework_stream():
    """CUDA stream handle (int; 0 = legacy default stream) the caller's array framework is queueing work on, or None when
    no framework is active (or a CUDA-graph capture is running: the caller then runs the handle on the capturing stream)."""
    import sys
    torch = sys.modules.get("torch")
    if torch is not None and torch.cuda.is_available() and torch.cuda.is_initialized():
        if torch.cuda.is_current_stream_capturing():
            return None
        return int(torch.cuda.current_stream().cuda_stream)
    cupy = sys.modules.get("cupy")
    if cupy is not None:
        try:
            return int(cupy.cuda.get_current_stream().ptr)
        except Exception:
            return None
    return None