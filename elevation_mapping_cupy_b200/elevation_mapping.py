"""Drop-in `ElevationMap` for the fusion path, implemented over libemap.so (hand-written sm_90a CUDA).

Mirrors the public surface of the reference class
(elevation_mapping_cupy/script/elevation_mapping_cupy/elevation_mapping.py:49-922, "EM.py" below):
same method names, positional signatures and error behaviour, so the C++ bridge
(elevation_mapping_cupy/src/elevation_mapping_wrapper.cpp:173-324) and the reference's tests
(script/elevation_mapping_cupy/tests/test_elevation_mapping.py) can drive it unchanged.  All compute
happens in the library; this module only marshals arguments.  Device arrays are handed out as torch
CUDA tensors that alias the library's memory (they also expose `__cuda_array_interface__`).

Point-cloud semantic layers are fused inside the frame with every point-cloud fusion of the reference (average,
class_average, color, class_bayesian, bayesian_inference, class_max; semantic_map.py).
The polygon safety check (get_polygon_traversability) is one library call: mask, statistics and hull on the device;
get_polygons_traversability checks a batch of polygons in one call.
Camera images (input_image) fuse into the semantic layers with the reference's `color` and `exponential` image fusions:
one kernel projects every map cell into the image, tests occlusion along the line to the camera and writes every fused
channel (csrc/emap_image.cuh), bit-identical to the reference's kernels on the same card.
Windows of the exported map (get_submap / get_submaps, the node's get_raw_submap service) come from one library call
and one kernel per batch (csrc/emap_submap.cuh); get_transformed_submap(s) serve them in a requester's frame, as grid_map's
getTransformedMap does, in three kernels per batch.
The rest of the node's map timer is served too: the normals (get_normal_maps / get_normal_ref), the bridge's normal
colour as the exported layer `normal_color`, and the exported map as a point cloud (get_map_points) and as normal arrows
(get_normal_arrows), compacted in grid_map's cell order on the device (csrc/emap_mapcloud.cuh).
Depth cameras (input_depth_image / input_depth_images) fuse without the semantic sensor node's intermediate cloud: the
frame reads the depth, confidence, rgb and feature planes itself (csrc/emap_sources.cuh).
Out of scope (SURVEY.md section 8): the image feature extractors.
"""
import ctypes as C
import math
import threading
from typing import List

import numpy as np

from . import _lib
from .parameter import Parameter
from .plugins.plugin_manager import PluginManager
from .semantic_map import SemanticMap

LAYER_NAMES = ["elevation", "variance", "is_valid", "traversability", "time", "upper_bound", "is_upper_bound"]
EXPORT_NAMES = ["elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
                "normal_x", "normal_y", "normal_z", "normal_color"]
INIT_METHODS = {"nearest": 0, "linear": 1, "cubic": 2}          # emap_initialize_map's method codes


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


def _cloud(x, device):
    """(ptr, n_rows, row_stride, dtype_code, keepalive) of one point cloud: a device array read in place (device=True),
    or a host array (a device array is copied there), float32 unless float64, C-contiguous."""
    if device:
        dev = _device_pointer(x)
        if dev is None:
            raise ValueError("device_ptrs=True needs every point cloud in device memory")
        return dev
    a = _to_host(x)
    if a.dtype not in (np.float32, np.float64):
        a = a.astype(np.float32)
    if a.ndim != 2 or a.shape[1] < 3:
        raise ValueError("raw_points must be (N, >=3)")
    if not a.flags.c_contiguous:
        a = np.ascontiguousarray(a)
    return a.ctypes.data, a.shape[0], a.shape[1], (_lib.EMAP_F32 if a.dtype == np.float32 else _lib.EMAP_F64), a


def _clouds(clouds, device):
    """(ptrs, counts, row_stride, dtype_code, keepalive) of one frame's clouds (_cloud each), which must share row stride
    and dtype"""
    cs = [_cloud(c, device) for c in clouds]
    if len({c[2:4] for c in cs}) > 1:
        raise ValueError("all sensor clouds must share row stride and dtype")
    stride, dt = cs[0][2:4] if cs else (None, None)
    return (C.c_void_p * len(cs))(*[c[0] for c in cs]), (C.c_int64 * len(cs))(*[c[1] for c in cs]), stride, dt, cs


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
        self._region_caps = (256, 1024, 16384)   # extract_planar_regions: the largest table counts seen (rows)
        self._values_cap = 4096                  # values_between_locations: the largest total seen (rows)
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
        # polygon safety check (EM.py:110, 239): the last ring, the library's ring buffer, the mask (made on first use)
        self.untraversable_polygon = np.zeros((1, 2))
        self._ring = np.zeros((2 * (self.cell_n - 2) + 1, 2), np.float64)
        self._mask = None
        self._batch_hull = np.zeros((4096, 2), np.float64)      # rings of get_polygons_traversability, grown on demand
        # rows of get_map_points / get_normal_arrows, grown on demand
        self._mc_points = [np.zeros((0, 3), np.float32)]
        self._mc_arrows = [np.zeros(0, np.int32), np.zeros((0, 6), np.float64)]

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

    def _ordered_call(self, fn, *args, after=False, before=False):
        """fn(*args), a library call, ordered with the caller's framework: after the work it has queued when `after` (the
        call reads memory the framework writes, or writes memory it reads) and before the work it queues next when
        `before` (the call writes device memory the framework reads).  That second wait is queued before a failure
        raises, so framework work that frees or rewrites the call's device inputs still runs after what the call queued."""
        if after:
            self._after_framework()
        rc = fn(*args)
        if before:
            self._before_framework()
        self._check(rc)

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
        (semantic_map.py:223-259; algorithms average / class_average / color / class_bayesian / bayesian_inference /
        class_max)."""
        self._configure_cloud_channels(channels)
        Rm = np.ascontiguousarray(_to_host(R), dtype=np.float32).reshape(9)
        tv = np.ascontiguousarray(_to_host(t), dtype=np.float32).reshape(3)
        dev = _device_pointer(raw_points)
        ptr, n, row, dt, _keep = dev if dev is not None else _cloud(raw_points, False)
        with self.map_lock:
            self._after_framework()       # framework work writing the cloud or reading the aliased layers comes first
            self._check(self._L.emap_input_pointcloud(self._h, ptr, n, row, dt, int(dev is not None), Rm.ctypes.data,
                                                      tv.ctypes.data, float(position_noise), float(orientation_noise)))

    def _configure_cloud_channels(self, channels):
        """The semantic fusion of a cloud with these channel names (x, y, z first); None keeps the configuration."""
        if channels is not None and (len(channels) > 3 or self.semantic_map._configured is not None):
            self.semantic_map.configure_for(list(channels))

    # the pure-Python ROS node of the reference still calls `.input(...)` (elevation_mapping_ros.py:212)
    input = input_pointcloud

    def input_sensors(self, clouds, Rs, ts, position_noise, orientation_noise, device_ptrs=False):
        """Several sensors of one time slice fused against the same snapshot (SURVEY 8(e)).  device_ptrs=True: every
        cloud is a device array, read in place; otherwise every cloud is read from the host."""
        ptrs, counts, stride, dt, _keep = _clouds(clouds, device_ptrs)
        Rm = np.ascontiguousarray(np.stack([np.asarray(_to_host(r), np.float32).reshape(9) for r in Rs]))
        tm = np.ascontiguousarray(np.stack([np.asarray(_to_host(t), np.float32).reshape(3) for t in ts]))
        with self.map_lock:
            self._after_framework()       # framework work writing the clouds or reading the aliased layers comes first
            self._check(self._L.emap_input_sensors(self._h, len(counts), ptrs, counts, stride, dt,
                                                   int(bool(device_ptrs)), Rm.ctypes.data, tm.ctypes.data,
                                                   float(position_noise), float(orientation_noise)))

    def input_depth_image(self, depth, P, R, t, position_noise: float, orientation_noise: float, channels=(), rgb=None,
                          features=None, confidence=None, confidence_threshold: float = 10.0, max_depth: float = 8.0):
        """A depth camera frame: the semantic sensor node's create_pcl_from_image (pointcloud_node.py:205-274) and
        input_pointcloud of its cloud in one library call, with no intermediate cloud (emap_input_depth_image).
        depth: (H, W) metres; P: CameraInfo P (3x4) or K (3x3); R, t: optical frame -> map; confidence: (H, W), pixels
        below `confidence_threshold` are dropped (pointcloud_parameters.py:42), as are pixels that are not finite, <= 0
        or >= `max_depth` (the node's 8 m).  `channels` are the cloud's extra channel names: one whose fusion is `color`
        reads `rgb` ((H, W, 3) uint8), the others read the planes of `features` ((n, H, W) float32) in order.  Arrays of
        any framework; all host or all device."""
        self.input_depth_images([dict(depth=depth, P=P, R=R, t=t, rgb=rgb, features=features, confidence=confidence)],
                                position_noise, orientation_noise, channels, confidence_threshold, max_depth)

    def input_depth_images(self, cameras, position_noise: float, orientation_noise: float, channels=(),
                           confidence_threshold: float = 10.0, max_depth: float = 8.0):
        """Several depth cameras of one time slice fused against the same snapshot, as input_sensors fuses clouds.
        `cameras`: dicts with the keys depth, P, R, t and optionally rgb, features, confidence (see input_depth_image);
        `channels` is shared by every camera."""
        depth = self._depth_frame(cameras, channels)
        with self.map_lock:
            # the frame runs after the framework work writing the images or reading the aliased layers; framework work
            # queued from here on sees the fused map, and the device images (the caller's, or the converted copies in
            # `keep`, freed on return) are released or rewritten only after the frame has read them (no host sync)
            self._ordered_call(self._L.emap_input_depth_images, self._h, *depth.args, float(confidence_threshold),
                               float(max_depth), float(position_noise), float(orientation_noise), after=True, before=True)

    def _depth_frame(self, cameras, channels):
        """The depth cameras of one frame as the library takes them (_DepthFrame), with `channels` configured as the
        extra channels of every camera (the semantic sensor node's rule: the `color` channel reads rgb, the others the
        feature planes in order)."""
        channels = list(channels)
        if channels or self.semantic_map._configured is not None:
            self.semantic_map.configure_for(["x", "y", "z"] + channels)
        sources, k = [], 0
        for ch in channels:                       # the node's rule: the `color` channel takes rgb, the others the planes
            if self.semantic_map.layer_specs_points.get(ch) == "color":
                sources.append(-1)
            else:
                sources.append(k); k += 1
        n = len(cameras)
        if not 1 <= n <= _lib.EMAP_DEPTH_MAX_CAMERAS:
            raise ValueError(f"1 to {_lib.EMAP_DEPTH_MAX_CAMERAS} cameras per call")
        dev = _on_device(cameras[0]["depth"])
        keep, cams, n_features = [], (_lib.EmapDepthCamera * n)(), 0
        for i, cam in enumerate(cameras):
            depth = _depth_input(cam["depth"], np.float32, dev, self.device, keep)
            if depth.ndim != 2:
                raise ValueError("depth must be an (H, W) array")
            H, W = depth.shape
            c = cams[i]
            c.height, c.width, c.depth = H, W, _address(depth)
            for name, dtype, shape in (("confidence", np.float32, (H, W)), ("rgb", np.uint8, (H, W, 3)),
                                       ("features", np.float32, None)):
                if cam.get(name) is None:
                    continue
                a = _depth_input(cam[name], dtype, dev, self.device, keep)
                if tuple(a.shape) != shape and not (shape is None and a.ndim == 3 and tuple(a.shape[1:]) == (H, W)):
                    raise ValueError(f"{name} has shape {tuple(a.shape)} for a {H}x{W} depth image")
                setattr(c, name, _address(a))
                if name == "features":
                    n_features = a.shape[0] if i == 0 else min(n_features, a.shape[0])
            Pm = np.asarray(_to_host(cam["P"]), np.float64)
            c.fx, c.fy, c.cx, c.cy = Pm[0, 0], Pm[1, 1], Pm[0, 2], Pm[1, 2]
            c.R[:] = np.asarray(_to_host(cam["R"]), np.float32).reshape(9).tolist()
            c.t[:] = np.asarray(_to_host(cam["t"]), np.float32).reshape(3).tolist()
        src = (C.c_int32 * max(len(sources), 1))(*sources)
        return _DepthFrame((n, cams, int(dev), len(sources), src, n_features), keep,
                           sum(int(c.height) * int(c.width) for c in cams), float(cams[0].t[2]))

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

    def _exportable(self, name):
        return name in EXPORT_NAMES or name in self.semantic_map.layer_names or name in self.plugin_manager.layer_names

    def _export_source(self, name):
        """(name, device plane, flags, tensor to keep alive) of an exportable layer (_exportable).  Basic layers are
        exported by name; semantic layers as they are (EM.py:747-748: cropped, flipped, no NaN fill, no z offset); plugin
        layers with their fill_nan / is_height_layer (EM.py:762-775: flags bit 0 / bit 1)."""
        if name in EXPORT_NAMES:
            return name, None, 0, None
        if name in self.semantic_map.layer_names:
            m = self.semantic_map.semantic_map[self.semantic_map.layer_names.index(name)]
            return name, m.data_ptr(), 0, m
        self._update_plugin(name)
        m = self.plugin_manager.get_map_with_name(name)
        p = self.plugin_manager.get_param_with_name(name)
        return name, m.data_ptr(), int(bool(p.fill_nan)) | (int(bool(p.is_height_layer)) << 1), m

    def _layer_sources(self, names):
        """The (names, planes, flags) arrays the library takes for the live-map layers `names` (_export_source each), and
        whether any plane is framework memory.  Every name is checked before any source is evaluated (a plugin layer runs
        its plugin): KeyError for a layer the map does not have.  Runs under map_lock."""
        for name in names:
            if not self._exportable(name):
                raise KeyError("Layer {} is not in the map".format(name))
        sources = [self._export_source(name) for name in names]
        n = len(sources)
        planes = (C.c_void_p * n)(*[s[1] for s in sources])
        planes._keep = [s[3] for s in sources]
        return ((C.c_char_p * n)(*[s[0].encode() for s in sources]), planes, (C.c_int32 * n)(*[s[2] for s in sources]),
                any(s[3] is not None for s in sources))

    def _export(self, names, data):
        """Writes the layers `names` (_layer_sources) into `data`, a caller-owned (len(names), cell_n-2, cell_n-2) float32
        array: one kernel, one D2H copy, one sync.  Runs under map_lock."""
        n = len(names)
        n_out = (self.cell_n - 2) ** 2
        direct = isinstance(data, np.ndarray) and data.dtype == np.float32 and data.flags.c_contiguous and data.size == n * n_out
        buf = data if direct else (self._export_tmp if n == 1 else np.zeros((n, n_out), np.float32))
        c_names, planes, flags, framework = self._layer_sources(names)
        self._ordered_call(self._L.emap_get_layers, self._h, n, c_names, planes, flags, buf.ctypes.data, n * n_out,
                           after=framework)
        if not direct:
            data[...] = buf.reshape(data.shape)

    def get_map_with_name_ref(self, name, data):
        """EM.py:720-775: write layer `name` (NaN-filled, z-shifted, cropped, flipped) into `data`,
        a caller-owned (cell_n-2, cell_n-2) float32 array."""
        with self.map_lock:
            if not self._exportable(name):
                print("Layer {} is not in the map".format(name))
                return
            self._export([name], data)

    def get_maps_with_names_ref(self, names, data):
        """Several layers at once (what the C++ bridge's get_grid_map does one by one, elevation_mapping_wrapper.cpp:213-252):
        `data` is a caller-owned (len(names), cell_n-2, cell_n-2) float32 array.  One kernel, one D2H copy, one sync."""
        with self.map_lock:
            self._export(list(names), data)

    def get_submap(self, position, length, layers, out=None):
        """The get_raw_submap service (elevation_mapping_ros.cpp:507-553) in the map frame: the window of the exported
        map around `position` (x, y) of `length` (x, y) metres, as get_submaps returns it for one request."""
        return self.get_submaps([(position, length)], layers, out)[0]

    def get_submaps(self, requests, layers, out=None):
        """Windows of the exported map (get_maps_with_names_ref's coordinates: the interior, flipped on both axes) for
        `requests`, a list of (position, length) pairs of (x, y) metres in the map frame, in one library call
        (emap_get_submaps; include/emap.h states the window rule).  `layers` are named as for get_maps_with_names_ref
        and evaluated once per call.  `out`: None (a new NumPy array), a float32 C-contiguous NumPy array or a float32
        contiguous torch CUDA tensor of at least len(layers) * the windows' cells; with a CUDA tensor the call does not
        synchronise with the host and the results stay on the device.  Returns one dict per request: "layers" maps each
        name to a (rows, cols) view of `out`, "index" is (row0, col0), "size" (rows, cols), "centre" the centre of the
        window's cells and "success" whether the position lies in the map (a failed window has (0, 0) layers)."""
        req = np.zeros((len(requests), 4), np.float64)
        for w, (pos, ln) in enumerate(requests):
            req[w] = _xy(pos) + _xy(ln)
        n = len(req)
        info = np.zeros((n, 5), np.int32)
        centres = np.zeros((n, 2), np.float64)

        def cells():
            c = self.center.astype(np.float64)
            self._check(self._L.emap_submap_windows(self.cell_n, float(self.resolution), c.ctypes.data, n,
                                                    req.ctypes.data, info.ctypes.data, centres.ctypes.data))
            return int((info[:, 3].astype(np.int64) * info[:, 4]).sum())

        def call(nl, c_names, planes, flags, ptr, device, size):
            return self._L.emap_get_submaps(self._h, n, req.ctypes.data, nl, c_names, planes, flags, ptr, device, size,
                                            info.ctypes.data, centres.ctypes.data)

        views = self._window_views(layers, out, cells, call, info[:, 3:5])
        return [{"layers": views[w], "index": (int(info[w, 1]), int(info[w, 2])),
                 "size": (int(info[w, 3]), int(info[w, 4])), "centre": centres[w].copy(), "success": bool(info[w, 0])}
                for w in range(n)]

    def get_transformed_submap(self, position, length, layers, transform, sample_ratio=0.0, out=None):
        """The get_raw_submap service with a request frame other than the map frame, for one request: see
        get_transformed_submaps."""
        return self.get_transformed_submaps([(position, length, transform)], layers, out, sample_ratio)[0]

    def get_transformed_submaps(self, requests, layers, out=None, sample_ratio=0.0):
        """The get_raw_submap service (elevation_mapping_ros.cpp:507-553) in a requester's frame, in one library call
        (emap_get_transformed_submaps; include/emap.h states the rules).  `requests` is a list of (position, length,
        transform): position (x, y) in the request frame, length (x, y) metres, and transform the map -> request frame
        isometry (lookupTransform(frame_id, map_frame)) as a 4 x 4 array or an (R, t) pair.  Each window is the one
        get_submaps cuts at the map-frame position, carried into the request frame as grid_map's getTransformedMap
        does, with `sample_ratio` (>= 0; the node uses 0).  `layers` and `out` as for get_submaps, with each window's
        cells those of its new map.  Returns one dict per request: "layers" maps each name to a (rows, cols) view of
        `out` (row r, column c is grid_map index (r, c) of the new map), "size" (rows, cols), "frame_centre" the new
        map's centre (x, y) in the request frame, "length" its length (x, y), and "success" whether the map-frame
        position lies in the map (a failed window has (0, 0) layers)."""
        n = len(requests)
        req = np.zeros((n, 4), np.float64)
        tf = np.zeros((n, 12), np.float64)
        for w, (pos, ln, T) in enumerate(requests):
            req[w] = _xy(pos) + _xy(ln)
            tf[w] = _isometry(T)
        info = np.zeros((n, 3), np.int32)
        geometry = np.zeros((n, 4), np.float64)

        def cells():
            c = self.center.astype(np.float64)
            self._check(self._L.emap_transformed_submap_windows(self.cell_n, float(self.resolution), c.ctypes.data, n,
                                                                req.ctypes.data, tf.ctypes.data, info.ctypes.data,
                                                                geometry.ctypes.data))
            return int((info[:, 1].astype(np.int64) * info[:, 2]).sum())

        def call(nl, c_names, planes, flags, ptr, device, size):
            return self._L.emap_get_transformed_submaps(self._h, n, req.ctypes.data, tf.ctypes.data, float(sample_ratio),
                                                        nl, c_names, planes, flags, ptr, device, size, info.ctypes.data,
                                                        geometry.ctypes.data)

        views = self._window_views(layers, out, cells, call, info[:, 1:3])
        return [{"layers": views[w], "size": (int(info[w, 1]), int(info[w, 2])),
                 "frame_centre": geometry[w, :2].copy(), "length": geometry[w, 2:].copy(), "success": bool(info[w, 0])}
                for w in range(n)]

    def segment_planes(self, position, length, params=None, out=None):
        """The plane decomposition node's segmented planes map for the get_submap window around `position` (x, y) of
        `length` (x, y) metres, in one library call (emap_segment_planes; include/emap.h states every step).  `params` is
        a PlaneSegmentationParams (None: the node's parameters.yaml without RANSAC refinement).  `out`: None (new NumPy
        arrays) or a contiguous float32 torch CUDA tensor of at least 4 * rows * cols floats; with a tensor the layers
        and the plane table stay on the device, and only the five info words are read back.  Returns a dict: "layers"
        maps elevation_raw, elevation, segmentation and plane_classification to (rows, cols) views; "planes" is an
        (n, 7) float64 array (label, support xyz, normal xyz); "highest_label", "origin" (the centre of window cell
        (0, 0)), "centre" (the centre of the window's cells, as get_submaps returns it), "resolution", "size" and
        "success" (False when the window is outside the map or has no finite cell;
        its layers are then not written)."""
        from .plane_segmentation import PlaneSegmentationParams
        p = (params or PlaneSegmentationParams()).to_c()
        req = np.array(_xy(position) + _xy(length), np.float64)
        device = out is not None and _is_device(out)
        size = None if out is None else _flat_out(out)
        with self.map_lock:
            rows, cols, res, centre, cap = self._plane_window(p, req)
            if out is None:
                out = np.zeros(len(_PLANE_LAYERS) * rows * cols, np.float32)
                size = out.size
            mk = _array_maker(out.device if device else None)
            planes, info = mk((cap, 7), "float64"), mk(5, "int32")
            self._ordered_call(self._L.emap_segment_planes, self._h, req.ctypes.data, C.byref(p), _address(out),
                               int(device), size, _address(planes), cap, _address(info), after=device, before=device)
        return _plane_result(_PLANE_LAYERS, out, rows, cols, res, centre, planes, info.cpu().numpy() if device else info)

    def extract_planar_regions(self, position, length, params=None, out=None, capacities=None):
        """The plane decomposition node's planar regions for the get_submap window around `position` (x, y) of `length`
        (x, y) metres: segment_planes, then contour extraction and the height offset in one library call
        (emap_extract_planar_regions; include/emap.h states every step).  `params` and `out` as in segment_planes
        (the PlaneSegmentationParams' margin_size and extracted_planes_height_offset apply here).  Returns
        segment_planes' dict plus "tables" (the flat "regions" (n, 17), "polygons" (n, 5) and "vertices" (n, 2)
        tables: NumPy arrays, or torch CUDA tensors with a device `out`, of which only the info words are read back) and,
        with host output, "regions": per region a dict of "label", "transform" (4 x 4 plane-to-world), "bbox" (xmin,
        ymin, xmax, ymax in the plane frame), "boundary" {"outer", "holes"} and "insets" [{"outer", "holes"}], each
        polygon an (n, 2) array of plane-frame points.  `capacities`: (regions, polygons, vertices) rows to start from;
        None starts from the largest counts an earlier call of this map returned (a small default on the first call).
        When a table is too small the call is repeated once with the exact sizes; "retried" says whether it was."""
        return self._planar_regions(position, length, params, out, capacities, False)

    def planar_terrain(self, position, length, params=None, out=None, capacities=None):
        """The grid map and planar regions of the plane decomposition node's PlanarTerrain message for the get_submap
        window around `position` (x, y) of `length` (x, y) metres: extract_planar_regions, then the node's
        post-processing, in one library call (emap_planar_terrain; include/emap.h states every step).  `params`,
        `capacities` and the returned dict as in extract_planar_regions (the PlaneSegmentationParams' postprocessing
        fields apply here); a device `out` holds at least 10 * rows * cols floats.  "layers" maps the node's layer names
        to (rows, cols) views: elevation_raw, elevation_before_postprocess (extract_planar_regions' "elevation"),
        segmentation, plane_classification, elevationWithNaN, elevationWithNaN_i, elevationWithNaNClosed,
        elevationWithNaNClosedDilated, smooth_planar and elevation.  Note that "elevation" here is the post-processed
        layer (non-planar cells dilated and lifted), not the one segment_planes and extract_planar_regions return."""
        return self._planar_regions(position, length, params, out, capacities, True)

    def project_to_planar_regions(self, terrain, queries, penalty_z_weight=0.0, convex_vertices=0, growth_factor=1.05,
                                  out=None):
        """The best planar region for each query point and the point projected onto it, optionally with a convex
        polygon grown around it inside the region's boundary (convex_plane_decomposition's
        getBestPlanarRegionAtPositionInWorld, searched exhaustively, and growConvexPolygonInsideShape), in one library
        call (emap_project_to_planar_regions; include/emap.h states every step).  `terrain`: a dict returned by
        extract_planar_regions or planar_terrain; its "tables" are read in place (NumPy or torch CUDA).  `queries`: (N,
        3) world points, float64 NumPy or a CUDA tensor.  The cost of a region is the squared distance to the projected
        point plus penalty_z_weight * |z| of that point.  `convex_vertices`: 0 (no growth) or 3 ..
        EMAP_CONVEX_MAX_VERTICES.  `out`: None, or a dict of "index" (N, 3) int32, "point" (N, 6) float64 and, with
        growth, "convex" (N, V, 5) float64, all NumPy or all torch CUDA tensors, written in place.  Device queries or a
        device `out` keep everything on the device (stream-ordered after the caller's work, no host synchronisation).
        Returns "region" (row, -1 for none), "label", "cost", "position_plane" (N, 2), "position_world" (N, 3), "status"
        (0 grown, 1 zero radius, 2 max iterations, 3 no region, 4 invalid query, 5 bad table), "iterations" and, with
        growth, "convex_plane" (N, V, 2) and "convex_world" (N, V, 3); all views of `out`."""
        tabs = terrain["tables"]
        reg, poly, vert = (_input_array(tabs[k], dt, k[:-1] + " table", cols)
                           for k, dt, cols in (("regions", "float64", 17), ("polygons", "int32", 5),
                                               ("vertices", "float64", 2)))
        tables_dev = _is_device(reg)
        if _is_device(poly) != tables_dev or _is_device(vert) != tables_dev:
            raise TypeError("the region tables must be all NumPy or all torch CUDA")
        if np.ndim(queries) != 2 or np.shape(queries)[1] != 3:
            raise ValueError("queries must be (N, 3)")
        q = _queries((queries,), 3)
        n, n_conv = int(q.shape[0]), int(convex_vertices)
        dev = _output_device([q, *(out or {}).values()])
        device = dev is not None
        specs = {"index": ((n, 3), "int32"), "point": ((n, 6), "float64")}
        if n_conv:
            specs["convex"] = ((n, n_conv, 5), "float64")
        out = _outputs(out, specs, dev)
        t = _lib.EmapRegionTables(_address(reg), len(reg), _address(poly), len(poly), _address(vert), len(vert))
        o = _lib.EmapProjectionOut(_address(out["index"]), _address(out["point"]), _address(out["convex"]) if n_conv else None)
        self._ordered_call(self._L.emap_project_to_planar_regions, self._h, C.byref(t), int(tables_dev), n, _address(q),
                           int(_is_device(q)), float(penalty_z_weight), n_conv, float(growth_factor), C.byref(o),
                           int(device), after=device or tables_dev, before=device)
        index, point = out["index"], out["point"]
        region = index[:, 0]
        if device:
            import torch
            labels = (reg[:, 0] if tables_dev else torch.as_tensor(reg[:, 0])).to(point.device)
            lab = torch.full((n,), float("nan"), dtype=torch.float64, device=point.device)
            if len(reg):
                lab = torch.where(region >= 0, labels[region.clamp(min=0).long()], lab)
        else:
            labels = reg[:, 0].cpu().numpy() if tables_dev else reg[:, 0]
            lab = np.where(region >= 0, labels[np.clip(region, 0, None)] if len(reg) else np.nan, np.nan)
        res = {"region": region, "label": lab, "cost": point[:, 0], "position_plane": point[:, 1:3],
               "position_world": point[:, 3:6], "status": index[:, 1], "iterations": index[:, 2]}
        if n_conv:
            res["convex_plane"] = out["convex"][:, :, :2]
            res["convex_world"] = out["convex"][:, :, 2:]
        return res

    def max_value_between_locations(self, grid, layer, starts, ends, out=None):
        """The largest finite value of `layer` on each line from starts[i] to ends[i] (grid_map_filters_rsl's
        maxValueBetweenLocations, quirks preserved), in one library call (emap_max_values_between; include/emap.h
        states every step).  `grid`: a dict returned by segment_planes, extract_planar_regions, planar_terrain or
        get_submap(s); `layer` names one of its layers, read in place (NumPy or torch CUDA).  `starts`, `ends`: (N, 2)
        map-frame points, float64 NumPy or CUDA tensors.  `out`: None, or a dict of "index" (N, 3) int32 and "value"
        (N, 3) float64, both NumPy or both torch CUDA, written in place.  Device queries or a device `out` keep
        everything on the device.  Returns "valid", "value", "index" (N, 2: the LAST finite cell of the line, as the
        reference returns) and "position" (N, 2: that cell's position); all views of `out`."""
        g = self._grid(grid, layer)
        lines = _queries((starts, ends), 4)
        n = int(lines.shape[0])
        dev = _output_device([lines, *(out or {}).values()])
        out = _outputs(out, {"index": ((n, 3), "int32"), "value": ((n, 3), "float64")}, dev)
        o = _lib.EmapLineMaxOut(_address(out["index"]), _address(out["value"]))
        self._lookup_call(self._L.emap_max_values_between, g, lines, C.byref(o), dev is not None)
        index, value = out["index"], out["value"]
        return {"valid": index[:, 0] != 0, "value": value[:, 0], "index": index[:, 1:], "position": value[:, 1:]}

    def values_between_locations(self, grid, layer, starts, ends, capacity=None):
        """Every finite value of `layer` on each line from starts[i] to ends[i] with its cell's position
        (grid_map_filters_rsl's valuesBetweenLocations), in one library call (emap_values_between; include/emap.h
        states every step).  `grid`, `layer`, `starts` and `ends` as in max_value_between_locations; with device queries
        or a device layer the results stay on the device.  `capacity`: the rows to start from (None: the largest total
        this map has returned before).  When it is too small the call is repeated once with the exact total.  Returns
        "rows" (total, 3: x, y, value), "counts" (N) and "first" (N: where line i's rows start), "retried"."""
        g = self._grid(grid, layer)
        lines = _queries((starts, ends), 4)
        n = int(lines.shape[0])
        dev = _output_device([lines, g._keep])
        mk = _array_maker(dev)
        cap = int(capacity if capacity is not None else self._values_cap)
        counts, first, info = mk((n,), "int32"), mk((n,), "int64"), mk((2,), "int64")
        for attempt in range(2):
            rows = mk((max(cap, 1), 3), "float64")
            o = _lib.EmapLineValuesOut(_address(rows), cap, _address(counts), _address(first), _address(info))
            self._lookup_call(self._L.emap_values_between, g, lines, C.byref(o), dev is not None)
            info_h = info.cpu().numpy() if dev is not None else info
            if info_h[1]:
                break
            cap = int(info_h[0])
        self._values_cap = max(self._values_cap, int(info_h[0]))
        return {"rows": rows[:int(info_h[0])], "counts": counts, "first": first, "retried": attempt > 0}

    def grid_derivatives(self, grid, layer, positions, curvature=False, out=None):
        """The gradient and, with `curvature`, the curvature of `layer` at each position (grid_map_filters_rsl's
        GridMapDerivative::estimateGradient / estimateGradientAndCurvature at the position's cell), in one library call
        (emap_grid_derivatives; include/emap.h states every step).  `grid` and `layer` as in max_value_between_locations
        (at least 5 x 5 cells); `positions`: (N, 2) map-frame points.  `out`: None, or a dict of "index" (N, 3) int32
        and "value" (N, 2 or 5) float64.  Returns "status" (0 inside, 1 outside: zero derivatives), "index" (N, 2),
        "gradient" (N, 2: x, y) and, with curvature, "curvature" (N, 3: xx, xy, yy); all views of `out`."""
        g = self._grid(grid, layer)
        pos = _queries((positions,), 2)
        n = int(pos.shape[0])
        dev = _output_device([pos, *(out or {}).values()])
        out = _outputs(out, {"index": ((n, 3), "int32"), "value": ((n, 5 if curvature else 2), "float64")}, dev)
        o = _lib.EmapDerivativeOut(_address(out["index"]), _address(out["value"]))
        call = lambda *a: self._L.emap_grid_derivatives(*a[:6], int(bool(curvature)), *a[6:])  # noqa: E731
        self._lookup_call(call, g, pos, C.byref(o), dev is not None)
        index, value = out["index"], out["value"]
        res = {"status": index[:, 0], "index": index[:, 1:], "gradient": value[:, :2]}
        if curvature:
            res["curvature"] = value[:, 2:]
        return res

    def values_at(self, positions, layers=("elevation",), method="linear", grid=None, out=None):
        """The value of each layer at each point, as grid_map's GridMap::atPosition gives it with "nearest", "linear" or
        "cubic" (cubic convolution), in one library call (emap_map_values_at / emap_grid_values_at; include/emap.h
        states the rule, its fallbacks at the edges and its operation order).  `positions`: (N, 2) map-frame points,
        float64 NumPy or a CUDA tensor.  `layers`: up to 24 names.  `grid`: None for the live map (layers named as for
        get_maps_with_names_ref, each evaluated once; the map's exported geometry at its current centre), or a dict of
        get_submap(s), get_transformed_submap(s), planar_terrain, plane_decomposition or the caller's own with
        "layers", "centre" and optionally "resolution", its layers read in place (all NumPy or all torch CUDA).
        `out`: None, or a dict of "values" (len(layers), N) float32 and "status" (N,) int32, both NumPy or both torch
        CUDA, written in place.  Device positions or a device `out` keep everything on the device (stream-ordered, no
        host synchronisation).  Returns "values" (a dict of (N,) views per layer name; NaN outside the grid) and
        "status" (N,): the method that produced each point's values after the fallbacks, 0 outside, 1 nearest,
        2 linear, 3 cubic."""
        if isinstance(layers, str):
            layers = (layers,)
        names = list(layers)
        if method not in _lib.EMAP_VALUES_METHODS:
            raise ValueError("method must be 'nearest', 'linear' or 'cubic'")
        if not 1 <= len(names) <= _lib.EMAP_VALUES_MAX_LAYERS:
            raise ValueError("1 to %d layers" % _lib.EMAP_VALUES_MAX_LAYERS)
        nl, m = len(names), _lib.EMAP_VALUES_METHODS[method]
        if grid is not None:
            grids = [self._grid(grid, name) for name in names]
            g_dev = _is_device(grids[0]._keep)
            if any(_is_device(x._keep) != g_dev for x in grids):
                raise TypeError("the grid's layers must be all NumPy or all torch CUDA")
        q = _queries((positions,), 2)
        n, q_dev = int(q.shape[0]), _is_device(q)
        dev = _output_device([q, *(out or {}).values()])
        device = dev is not None
        out = _outputs(out, {"values": ((nl, n), "float32"), "status": ((n,), "int32")}, dev)
        o = _lib.EmapValuesOut(_address(out["values"]), _address(out["status"]))
        if grid is not None:
            self._ordered_call(self._L.emap_grid_values_at, self._h, nl, (_lib.EmapGrid * nl)(*grids), int(g_dev), n,
                               _address(q), int(q_dev), m, C.byref(o), int(device), after=device or g_dev or q_dev,
                               before=device)
        else:
            with self.map_lock:
                c_names, planes, flags, framework = self._layer_sources(names)
                self._ordered_call(self._L.emap_map_values_at, self._h, nl, c_names, planes, flags, n, _address(q),
                                   int(q_dev), m, C.byref(o), int(device), after=device or q_dev or framework,
                                   before=device)
        values = out["values"]
        return {"values": {name: values[k] for k, name in enumerate(names)}, "status": out["status"]}

    def signed_distance_field(self, grid, layer="elevation", height_clearance=0.1, z_range=None, out=None):
        """A signed distance field of `layer` over the grid's box (metres to the terrain surface: positive above it,
        negative below), in one library call (emap_signed_distance_field; include/emap.h states every step).  `grid`
        and `layer` as in max_value_between_locations (a dict of segment_planes, planar_terrain, plane_decomposition,
        get_submap(s) or the caller's own with "layers", "centre" and optionally "resolution").  The slices are res
        apart from z_min: with `z_range` = (z_low, z_high), z_min = z_low and n_z = floor((z_high - z_low) / res) + 1;
        without it, z_min = lowest finite value - height_clearance and n_z = floor(((highest finite value +
        height_clearance) - z_min) / res) + 1, which reads two scalars back (a host synchronisation for a device
        layer), and a layer with no finite cell raises ValueError.  `out`: None, or an (n_z, rows, cols) contiguous
        float32 NumPy array or CUDA tensor, written in place; a device layer or `out` keeps the volume on the device
        (stream-ordered, no host synchronisation with `z_range`).  Returns "volume" (n_z, rows, cols), "rows", "cols",
        "n_z", "position", "resolution" and "z_min": the dict sdf_values takes."""
        g = self._grid(grid, layer)
        g_dev = _is_device(g._keep)
        dev = _output_device([out, g._keep])
        device = dev is not None
        res = float(g.resolution)
        if z_range is None:
            data = g._keep
            if g_dev:
                import torch
                fin = data[torch.isfinite(data)]
                if fin.numel() == 0:
                    raise ValueError("the layer has no finite cell: pass z_range")
                lo, hi = (float(v) for v in torch.aminmax(fin))
            else:
                fin = data[np.isfinite(data)]
                if fin.size == 0:
                    raise ValueError("the layer has no finite cell: pass z_range")
                lo, hi = float(fin.min()), float(fin.max())
            z_min = lo - float(height_clearance)
            n_z = int(math.floor(((hi + float(height_clearance)) - z_min) / res)) + 1
        else:
            z_min = float(z_range[0])
            n_z = int(math.floor((float(z_range[1]) - z_min) / res)) + 1
        shape = (n_z, int(g.rows), int(g.cols))
        if out is None:
            out = _array_maker(dev)(shape, "float32")
        _check_out({"volume": out}, {"volume": (shape, "float32")}, device)
        self._ordered_call(self._L.emap_signed_distance_field, self._h, C.byref(g), int(g_dev), z_min, n_z,
                           _address(out), out.numel() if device else out.size, int(device), after=device or g_dev,
                           before=device)
        return {"volume": out, "rows": int(g.rows), "cols": int(g.cols), "n_z": n_z,
                "position": np.array(g.position[:], np.float64), "resolution": res, "z_min": z_min}

    def sdf_values(self, field, points, out=None):
        """The field's value and gradient at each point, in one library call (emap_sdf_values; include/emap.h states
        every step): trilinear inside the box, plus the distance to the box outside it.  `field`: a dict returned by
        signed_distance_field (its "volume" read in place, NumPy or torch CUDA).  `points`: (N, 3) map-frame points,
        float64 NumPy or a CUDA tensor.  `out`: None, or an (N, 4) float64 array, NumPy or torch CUDA, written in place.
        Device points or a device `out` keep everything on the device.  Returns (N, 4): value, d/dx, d/dy, d/dz."""
        vol = _input_array(field["volume"], "float32", "volume")
        n_z, rows, cols = (int(field[k]) for k in ("n_z", "rows", "cols"))
        if tuple(vol.shape) != (n_z, rows, cols):
            raise ValueError("the volume must be (n_z, rows, cols)")
        pos = np.asarray(_to_host(field["position"]), np.float64)
        f = _lib.EmapSdf(_address(vol), rows, cols, n_z, (C.c_double * 2)(*pos.tolist()), float(field["resolution"]),
                         float(field["z_min"]))
        f._keep = vol
        q = _queries((points,), 3)
        n = int(q.shape[0])
        dev = _output_device([q, out])
        if out is None:
            out = _array_maker(dev)((n, 4), "float64")
        _check_out({"value": out}, {"value": ((n, 4), "float64")}, dev is not None)
        self._lookup_call(self._L.emap_sdf_values, f, q, _address(out), dev is not None)
        return out

    def inpaint_image(self, image, mask, radius=1, method="ns", out=None):
        """cv2.inpaint(image, mask, radius, INPAINT_NS or INPAINT_TELEA) for one 8-bit channel, bit for bit, in one
        library call (emap_inpaint_image; include/emap.h states every step).  `image`, `mask`: (rows, cols) uint8, NumPy
        or torch CUDA; a pixel is filled where its mask is non-zero.  `radius` is rounded as cv2 rounds it; only radius 1
        is provided.  `method`: "ns" (Navier-Stokes) or "telea" (at least 2 x 2 pixels).  `out`: None, or a contiguous
        (rows, cols) uint8 array, written in place.  A CUDA image, mask or `out` keeps everything on the device
        (stream-ordered, no host synchronisation); host inputs are then uploaded first.  Returns `out`."""
        methods = {"telea": 0, "ns": 1}
        if method not in methods:
            raise ValueError("method must be 'ns' or 'telea'")
        dev = _output_device([image, mask, out])
        device = dev is not None
        if device:
            import torch
            image, mask = (torch.as_tensor(a, device=dev).to(torch.uint8).contiguous() for a in (image, mask))
        else:
            image, mask = (np.ascontiguousarray(_to_host(a), np.uint8) for a in (image, mask))
        if image.ndim != 2 or tuple(mask.shape) != tuple(image.shape):
            raise ValueError("image and mask must be (rows, cols) of the same shape")
        rows, cols = (int(v) for v in image.shape)
        if out is None:
            out = _array_maker(dev)((rows, cols), "uint8")
        _check_out({"image": out}, {"image": ((rows, cols), "uint8")}, device)
        self._ordered_call(self._L.emap_inpaint_image, self._h, _address(image), _address(mask), rows, cols,
                           float(radius), methods[method], _address(out), int(device), after=device, before=device)
        return out

    def nonlinear_interpolation(self, grid, layer="elevation", inpaint_radius=None, out=None):
        """grid_map_filters_rsl's inpainting::nonlinearInterpolation: the NaN cells of `layer` filled by cv2's
        Navier-Stokes inpainting of the layer quantised to 8 bits between its finite minimum and maximum, every other cell
        copied bit for bit, in one library call (emap_nonlinear_interpolation; include/emap.h states every step and the
        edge cases).  `grid` and `layer` as in max_value_between_locations (a dict of get_submap(s),
        get_transformed_submap(s), planar_terrain, plane_decomposition or the caller's own).  `inpaint_radius` [m]
        (None: the grid's resolution) must round to 1 pixel.  `out`: None (on the layer's side), or a contiguous (rows,
        cols) float32 NumPy array or CUDA tensor, written in place; device output is stream-ordered with no host
        synchronisation.  Returns `out`."""
        g = self._grid(grid, layer)
        g_dev = _is_device(g._keep)
        dev = _output_device([g._keep if out is None else out])
        device = dev is not None
        shape = (int(g.rows), int(g.cols))
        if out is None:
            out = _array_maker(dev)(shape, "float32")
        _check_out({"layer": out}, {"layer": (shape, "float32")}, device)
        radius = float(g.resolution if inpaint_radius is None else inpaint_radius)
        self._ordered_call(self._L.emap_nonlinear_interpolation, self._h, C.byref(g), int(g_dev), radius, _address(out),
                           int(device), after=device or g_dev, before=device)
        return out

    def min_values(self, grid, layer="elevation", out=None):
        """grid_map_filters_rsl's inpainting::minValues: every NaN cell of `layer` takes the least non-NaN value next to
        its NaN region.  `grid`, `layer` and `out` as in nonlinear_interpolation; include/emap.h (emap_grid_filter)
        states every filter's rule.  Returns `out`."""
        return self._grid_filter("min_values", grid, layer, out)

    def median(self, grid, layer="elevation", *, kernel_size, delta_kernel_size=2, number_of_repeats=1, out=None):
        """smoothing::median: cv2.medianBlur on the float layer while kernel_size + delta_kernel_size *
        (number_of_repeats - 1) <= 5, else on the layer quantised to 8 bits between its finite minimum and maximum; the
        kernel grows by delta_kernel_size per repeat.  The float path is not cv2's on a layer with NaN holes: only
        windows without a NaN are (include/emap.h)."""
        return self._grid_filter("median", grid, layer, out, kernel_size=kernel_size,
                                 delta_kernel_size=delta_kernel_size, number_of_repeats=number_of_repeats)

    def box_blur(self, grid, layer="elevation", *, kernel_size, number_of_repeats=1, out=None):
        """smoothing::boxBlur: number_of_repeats of cv2.blur((kernel_size, kernel_size)), bit for bit."""
        return self._grid_filter("box_blur", grid, layer, out, kernel_size=kernel_size,
                                 number_of_repeats=number_of_repeats)

    def gaussian_blur(self, grid, layer="elevation", *, kernel_size, sigma, out=None):
        """smoothing::gaussianBlur: cv2.GaussianBlur((kernel_size, kernel_size), sigma); kernel_size 0 takes cv2's size
        from sigma."""
        return self._grid_filter("gaussian_blur", grid, layer, out, kernel_size=kernel_size, sigma=sigma)

    def dilate(self, grid, layer="elevation", *, kernel_size, mask=None, inpaint=True, out=None):
        """processing::dilate: the max of the finite values of layer * mask (a (rows, cols) float32 array on the
        layer's side; None, the reference's empty mask, reads the layer alone) in grid_map's clamped kernel_size
        window."""
        return self._grid_filter("dilate", grid, layer, out, kernel_size=kernel_size, mask=mask, inpaint=inpaint)

    def erode(self, grid, layer="elevation", *, kernel_size, mask=None, inpaint=True, out=None):
        """processing::erode: as dilate, with the min."""
        return self._grid_filter("erode", grid, layer, out, kernel_size=kernel_size, mask=mask, inpaint=inpaint)

    def outline(self, grid, layer="elevation", out=None):
        """processing::outline: the cells next to a NaN keep their value, every other cell becomes NaN."""
        return self._grid_filter("outline", grid, layer, out)

    def _grid_filter(self, op, grid, layer, out, kernel_size=1, delta_kernel_size=0, number_of_repeats=1, sigma=0.0,
                     mask=None, inpaint=True):
        """One emap_grid_filter call: `op` on grid["layers"][layer] into `out` (None: a new array on the layer's side,
        else a contiguous (rows, cols) float32 NumPy array or CUDA tensor, written in place; device output is
        stream-ordered with no host synchronisation).  Returns `out`."""
        g = self._grid(grid, layer)
        g_dev = _is_device(g._keep)
        shape = (int(g.rows), int(g.cols))
        m = None
        if mask is not None:
            m = _input_array(mask, "float32", "mask")
            if tuple(m.shape) != shape or _is_device(m) != g_dev:
                raise ValueError("mask must be a (rows, cols) float32 array on the layer's side")
        dev = _output_device([g._keep if out is None else out])
        device = dev is not None
        if out is None:
            out = _array_maker(dev)(shape, "float32")
        _check_out({"layer": out}, {"layer": (shape, "float32")}, device)
        f = _lib.EmapFilterOp(_lib.EMAP_FILTER_OPS[op], int(kernel_size), int(delta_kernel_size),
                              int(number_of_repeats), float(sigma), int(bool(inpaint)))
        self._ordered_call(self._L.emap_grid_filter, self._h, C.byref(g), int(g_dev), C.byref(f), _address(m),
                           _address(out), int(device), after=device or g_dev, before=device)
        return out

    def _grid(self, grid, layer):
        """The EmapGrid of grid["layers"][layer] (_input_array, kept alive as g._keep), centred at the dict's "centre" or,
        in a get_transformed_submap(s) dict, its "frame_centre", with its "resolution" or the map's."""
        data = _input_array(grid["layers"][layer], "float32", "layer")
        rows, cols = (int(s) for s in data.shape)
        centre = np.asarray(_to_host(grid["centre"] if "centre" in grid else grid["frame_centre"]), np.float64)
        g = _lib.EmapGrid(_address(data), rows, cols, (C.c_double * 2)(*centre.tolist()),
                          float(grid.get("resolution", self.resolution)))
        g._keep = data
        return g

    def _lookup_call(self, fn, g, queries, out, device):
        """fn(handle, grid, grid on device, n, queries, queries on device, out, device output), the lookup on `g` (an
        EmapGrid or EmapSdf whose array is g._keep) of the (n, k) `queries` (_queries), stream-ordered."""
        g_dev, q_dev = _is_device(g._keep), _is_device(queries)
        self._ordered_call(fn, self._h, C.byref(g), int(g_dev), int(queries.shape[0]), _address(queries), int(q_dev),
                           out, int(device), after=device or g_dev or q_dev, before=device)

    def plane_decomposition(self, grid, layer="elevation", params=None, out=None, capacities=None):
        """The plane decomposition node's pipeline (PlaneDecompositionPipeline::update without RANSAC refinement) on a
        grid rather than a window of this map, with the preprocessing's resampling to params.resolution, in one library
        call (emap_plane_decomposition; include/emap.h states every step).  `grid`: a dict returned by get_submap(s),
        get_transformed_submap(s) or planar_terrain; `layer` names one of its layers, read in place (NumPy or torch
        CUDA).  `params`, `out` and `capacities` as in planar_terrain, with a device `out` of at least 10 * rows *
        cols floats of the resampled grid.  Returns planar_terrain's dict for the resampled grid: "size",
        "resolution", "origin" and "centre" are its geometry, and "elevation_raw" is the input layer itself (the node's
        submap before the preprocessing, at its own size).  The result feeds project_to_planar_regions and the
        lookups as planar_terrain's does."""
        g = self._grid(grid, layer)
        result = self._planar_regions(None, None, params, out, capacities, True, g)
        result["layers"]["elevation_raw"] = g._keep
        return result

    def _plane_window(self, p, req=None, grid=None):
        """(rows, cols, resolution, centre, plane-table rows) of a plane call with the emap_plane_params `p`: the
        get_submap window `req` of this map, or the EmapGrid `grid` resampled to p's resolution."""
        if grid is None:
            win, centre = np.zeros(5, np.int32), np.zeros(2, np.float64)
            c = self.center.astype(np.float64)
            self._check(self._L.emap_submap_windows(self.cell_n, float(self.resolution), c.ctypes.data, 1,
                                                    req.ctypes.data, win.ctypes.data, centre.ctypes.data))
            rows, cols, res = int(win[3]), int(win[4]), float(self.resolution)
        else:
            size, r = np.zeros(2, np.int64), C.c_double(0.0)
            self._check(self._L.emap_plane_grid_geometry(grid.rows, grid.cols, grid.resolution, C.byref(p),
                                                         size.ctypes.data, C.addressof(r)))
            rows, cols, res, centre = int(size[0]), int(size[1]), r.value, np.array(grid.position[:], np.float64)
        return rows, cols, res, centre, max(int(self._L.emap_plane_capacity(rows, cols, C.byref(p))), 1)

    def _planar_regions(self, position, length, params, out, capacities, post, grid=None):
        """extract_planar_regions (post False), planar_terrain (post True) and plane_decomposition (post True, `grid` the
        EmapGrid it reads): the call with the capacity retry."""
        from .plane_segmentation import PlaneSegmentationParams
        prm = params or PlaneSegmentationParams()
        p, rp = prm.to_c(), prm.regions_to_c()
        pp = prm.postprocess_to_c() if post else None
        device = out is not None and _is_device(out)
        size = None if out is None else _flat_out(out)
        names = _TERRAIN_LAYERS if post else _PLANE_LAYERS
        if grid is None:
            req = np.array(_xy(position) + _xy(length), np.float64)
            fn = self._L.emap_planar_terrain if post else self._L.emap_extract_planar_regions
            head = (req.ctypes.data, C.byref(p), C.byref(rp)) + ((C.byref(pp),) if post else ())
            reads_framework = device
        else:
            req = None
            fn = self._L.emap_plane_decomposition
            head = (C.byref(grid), int(_is_device(grid._keep)), C.byref(p), C.byref(rp), C.byref(pp))
            reads_framework = device or _is_device(grid._keep)
        caps = tuple(int(v) for v in (capacities or self._region_caps))
        for attempt in range(2):
            with self.map_lock:
                rows, cols, res, centre, cap = self._plane_window(p, req, grid)
                if out is None:
                    out = np.zeros(len(names) * rows * cols, np.float32)
                    size = out.size
                mk = _array_maker(out.device if device else None)
                planes, info = mk((cap, 7), "float64"), mk(9, "int32")
                tables = (mk((max(caps[0], 1), 17), "float64"), mk((max(caps[1], 1), 5), "int32"),
                          mk((max(caps[2], 1), 2), "float64"))
                ro = _lib.EmapRegionOut(_address(tables[0]), caps[0], _address(tables[1]), caps[1], _address(tables[2]),
                                        caps[2])
                self._ordered_call(fn, self._h, *head, _address(out), int(device), size, _address(planes), cap,
                                   C.byref(ro), _address(info), after=reads_framework, before=device)
            info_h = info.cpu().numpy() if device else info
            if info_h[8]:
                break
            caps = (int(info_h[5]), int(info_h[6]), int(info_h[7]))
        self._region_caps = tuple(max(a, int(b)) for a, b in zip(self._region_caps, info_h[5:8]))
        nr, npoly, nv = (int(x) for x in info_h[5:8])
        reg, poly, vert = tables[0][:nr], tables[1][:npoly], tables[2][:nv]
        result = _plane_result(names, out, rows, cols, res, centre, planes, info_h)
        result.update(complete=bool(info_h[8]), tables={"regions": reg, "polygons": poly, "vertices": vert},
                      regions=None, retried=attempt > 0)
        if not device and info_h[8]:
            result["regions"] = regions_from_tables(reg, poly, vert)
        return result

    def _window_views(self, layers, out, cells, call, sizes):
        """What get_submaps and get_transformed_submaps share: checks `out` and the layer names before anything runs,
        sizes a new host `out` with cells() (the host window arithmetic, which fills `sizes`), runs the library call
        `call(n_layers, names, planes, flags, out pointer, is device, out floats)` stream-ordered and returns per window
        a dict of (rows, cols) views of `out` per layer, rows and cols read from `sizes` after the call."""
        names = list(layers)
        nl = len(names)
        device = out is not None and _is_device(out)
        size = None if out is None else _flat_out(out)
        with self.map_lock:
            c_names, planes, flags, framework = self._layer_sources(names)
            if out is None:
                out = np.zeros(nl * cells(), np.float32)
                size = out.size
            # after: the planes and the output buffer are complete / free; before: framework reads of `out` run after
            # the kernel (no host sync)
            self._ordered_call(call, nl, c_names, planes, flags, _address(out), int(device), size,
                               after=device or framework, before=device)
        flat = out.reshape(-1)
        result, off = [], 0
        for rows, cols in sizes:
            rows, cols = int(rows), int(cols)
            views = {}
            for name in names:
                views[name] = flat[off:off + rows * cols].reshape(rows, cols)
                off += rows * cols
            result.append(views)
        return result

    def get_normal_maps(self):
        """EM.py:777-791: a new (3, cell_n-2, cell_n-2) float32 array of the exported normal_x, normal_y, normal_z.  One
        kernel, one D2H copy, one sync."""
        n = self.cell_n - 2
        maps = np.zeros((3, n, n), np.float32)
        with self.map_lock:
            self._export(["normal_x", "normal_y", "normal_z"], maps)
        return maps

    def get_normal_ref(self, normal_x_data, normal_y_data, normal_z_data):
        """EM.py:793-805 (WRAP:239-247 with enable_normal_color): the exported normals into three caller-owned
        (cell_n-2, cell_n-2) arrays."""
        maps = self.get_normal_maps()
        normal_x_data[...] = maps[0]
        normal_y_data[...] = maps[1]
        normal_z_data[...] = maps[2]

    def _map_cloud(self, attr, call):
        """Runs emap_get_map_points / emap_get_normal_arrows into the grow-only buffers in self.<attr> (`call(bufs, n)`
        issues the library call), growing them and retrying once when the map has more rows than they hold.  Returns
        the number of rows."""
        with self.map_lock:
            self._after_framework()
            for attempt in range(2):
                bufs = getattr(self, attr)
                n = C.c_int64(len(bufs[0]))
                rc = call(bufs, n)
                if rc == 0 or attempt or n.value <= len(bufs[0]):
                    self._check(rc)
                    return n.value
                setattr(self, attr, [np.zeros((n.value,) + b.shape[1:], b.dtype) for b in bufs])

    def get_map_points(self):
        """The node's publishAsPointCloud (elevation_mapping_ros.cpp:501-505): an (M, 3) float32 array of (x, y, z), one
        row per cell of the exported map whose elevation is finite, in grid_map's column-major cell order (include/emap.h
        states the rule).  On the device, with the count and the rows read back once each."""
        m = self._map_cloud("_mc_points", lambda b, n: self._L.emap_get_map_points(self._h, b[0].ctypes.data, C.byref(n)))
        return self._mc_points[0][:m].copy()

    def get_normal_arrows(self):
        """The node's publishNormalAsArrow (elevation_mapping_ros.cpp:751-778): (ids, segments), an (M,) int32 array of
        marker ids (the cells' column-major linear index) and an (M, 6) float64 array of (start, end) = ((x, y, z),
        (x, y, z) + 0.1 * normal), one row per valid cell whose normal is not shorter than 0.1 (include/emap.h)."""
        m = self._map_cloud("_mc_arrows", lambda b, n: self._L.emap_get_normal_arrows(self._h, b[0].ctypes.data,
                                                                                       b[1].ctypes.data, C.byref(n)))
        return self._mc_arrows[0][:m].copy(), self._mc_arrows[1][:m].copy()

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

    def input_image(self, image, channels: List[str], R, t, K, D, distortion_model: str, image_height: int,
                    image_width: int):
        """EM.py:468-562 (WRAP:180-185): fuse a camera image into the semantic layers.  `image` is a list of (H, W) arrays
        or a (C, H, W) array of any framework, host or device; channel j of the processed channel list reads plane j.
        R, t: map -> camera optical frame; K: 3x3 intrinsics; D: distortion coefficients, used for "radtan" only.
        One library call, one kernel (semantic_map.py update_layers_image picks the fusions and layers)."""
        dev, img = _image_stack(image, self.device)
        n_planes, H, W = img.shape
        if (H, W) != (int(image_height), int(image_width)):
            raise ValueError(f"image is {H}x{W}, image_height x image_width is {image_height}x{image_width}")
        f32 = lambda x, n: np.ascontiguousarray(_to_host(x), dtype=np.float32).reshape(n)
        Rm, tv, Km = f32(R, 9), f32(t, 3), f32(K, 9)
        Dv = np.ascontiguousarray(_to_host(D), dtype=np.float32).reshape(-1)
        with self.map_lock:
            planes, kinds, layers = self.semantic_map.update_layers_image(list(channels))
            n = len(planes)
            arr = lambda v: (C.c_int32 * max(n, 1))(*v)
            sem = self.semantic_map.semantic_map
            # the kernel runs after the stacked image and any layer the channels added are complete; framework work
            # queued from here on sees the fused layers, and releases or rewrites a device image only after the kernel
            # has read it (no host sync)
            self._ordered_call(
                self._L.emap_input_image, self._h, n_planes, img.data_ptr() if dev else img.ctypes.data, int(dev), H, W,
                Km.ctypes.data, Dv.ctypes.data if Dv.size else None, int(Dv.size), str(distortion_model).encode(),
                Rm.ctypes.data, tv.ctypes.data, n, arr(planes), arr(kinds), arr(layers),
                None if sem is None else sem.data_ptr(), len(self.semantic_map.layer_names), after=True, before=True)

    # ---- not on the per-frame path ---------------------------------------------------------------

    def get_polygon_traversability(self, polygon, result):
        """EM.py:837-889: is the (N, 2) polygon (any array framework, cast to float32 as the C++ bridge passes it) safe to
        stand on?  Writes [is_safe, t, area] into `result`, keeps the convex hull of the polygon's untraversable cells
        for get_untraversable_polygon and returns its ring length (0: no such polygon).  The polygon mask is left in
        `self.mask`.  One kernel pass over the map, one small hull kernel, one device-to-host copy, one sync."""
        poly = np.ascontiguousarray(_to_host(polygon), dtype=np.float32).reshape(-1, 2)
        checker = None
        if self.param.checker_layer != "traversability":
            checker = self.get_layer(self.param.checker_layer)     # None: the layer is absent, traversability is used
        mask = self.mask
        res = np.zeros(3, np.float64)
        n_ring = C.c_int32(len(self._ring))
        with self.map_lock:
            self._after_framework()
            self._check(self._L.emap_polygon_traversability(
                self._h, poly.ctypes.data, poly.shape[0], None if checker is None else checker.data_ptr(),
                float(self.param.safe_thresh), float(self.param.safe_min_thresh), int(self.param.max_unsafe_n),
                res.ctypes.data, self._ring.ctypes.data, C.byref(n_ring), mask.data_ptr()))
        if _clipped_area(poly, self.center, self.cell_n, self.resolution) < np.float32(0.001):
            print("requested polygon is outside of the map")
        result[...] = res
        self.untraversable_polygon = self._ring[:n_ring.value].copy()
        return n_ring.value

    def get_polygons_traversability(self, polygons, results, compute_untraversable_polygon=True):
        """The check_safety service (CheckSafety.srv) in one library call: row i of the (B, 3) float64 `results` gets what
        get_polygon_traversability writes for polygons[i] (an (n_i, 2) array of any framework, cast to float32), and
        the returned list holds polygon i's untraversable ring as a float64 (n, 2) array ((0, 2) if none, and for every
        polygon when compute_untraversable_polygon is False).  self.mask and the single call's ring are left as they were."""
        polys = [np.ascontiguousarray(_to_host(p), dtype=np.float32).reshape(-1, 2) for p in polygons]
        n_vert = np.array([len(p) for p in polys], np.int32)
        xy = np.ascontiguousarray(np.concatenate(polys) if polys else np.zeros((0, 2), np.float32))
        checker = None
        if self.param.checker_layer != "traversability":
            checker = self.get_layer(self.param.checker_layer)     # None: the layer is absent, traversability is used
        B = len(polys)
        res = np.zeros((B, 3), np.float64)
        offsets = np.zeros(B + 1, np.int64)
        rows = C.c_int64(0)
        hull = None
        with self.map_lock:
            self._after_framework()
            while True:
                if compute_untraversable_polygon:
                    hull = self._batch_hull
                    rows.value = len(hull)
                rc = self._L.emap_polygon_traversability_batch(
                    self._h, B, n_vert.ctypes.data, xy.ctypes.data, None if checker is None else checker.data_ptr(),
                    float(self.param.safe_thresh), float(self.param.safe_min_thresh), int(self.param.max_unsafe_n),
                    res.ctypes.data, None if hull is None else hull.ctypes.data, offsets.ctypes.data, C.byref(rows))
                if rc == -1 and hull is not None and rows.value > len(hull):
                    self._batch_hull = np.zeros((rows.value, 2), np.float64)     # same map state, same answer
                    continue
                self._check(rc)
                break
        center = self.center
        for p in polys:
            if _clipped_area(p, center, self.cell_n, self.resolution) < np.float32(0.001):
                print("requested polygon is outside of the map")
        results[...] = res
        if hull is None:
            return [np.zeros((0, 2), np.float64) for _ in polys]
        return [hull[offsets[i]:offsets[i + 1]].copy() for i in range(B)]

    def get_untraversable_polygon(self, untraversable_polygon):
        """EM.py:891-897: copy the ring of the last get_polygon_traversability into the caller's (n, 2) array."""
        untraversable_polygon[...] = self.untraversable_polygon

    @property
    def mask(self):
        """(W, W) float32 polygon mask of the last get_polygon_traversability (EM.py:239 `self.mask`), a torch CUDA tensor."""
        if self._mask is None:
            import torch
            self._mask = torch.zeros((self.cell_n, self.cell_n), dtype=torch.float32, device=f"cuda:{self.device}")
        return self._mask

    def initialize_map(self, points, method="cubic"):
        """EM.py:899-922 + map_initializer.py:25-62: clear the map, interpolate the given (x, y, z) points (map frame) over
        the grid, dilate twice with dilation_size_initialize and set upper_bound to the elevation of the valid cells.
        One library call (emap_initialize_map, include/emap.h) does it on the device.  linear / cubic use the
        reference's own triangulation, scipy.spatial.Delaunay of the snapped points, and cubic SciPy's
        Clough-Tocher gradients on it: O(points) host work."""
        self.clear()                                           # EM.py:906; failures below leave the map cleared
        pts = np.ascontiguousarray(_to_host(points), dtype=np.float32).reshape(-1, 3)
        assert pts.shape[0] > 3, "Initialization points must be more than 3."
        if method not in INIT_METHODS:
            raise ValueError(f"Unknown interpolation method {method!r} for 2-D data")
        tri = grad = None
        if method != "nearest":
            from scipy.spatial import Delaunay
            # transform_to_map_index (traversability_polygon.py:61-63), as the library snaps: truncation toward zero
            c = self.center
            idx = ((pts[:, :2] - c[:2].reshape(1, 2)) / np.float32(self.resolution) + self.cell_n / 2).astype(np.int32)
            d = Delaunay(idx.astype(np.float64))
            tri = np.ascontiguousarray(d.simplices, dtype=np.int32)
            if method == "cubic":
                from scipy.interpolate import CloughTocher2DInterpolator
                z = pts[:, 2] - c[2]
                grad = np.ascontiguousarray(CloughTocher2DInterpolator(d, z.astype(np.float64)).grad[:, 0, :], np.float64)
        with self.map_lock:
            self._after_framework()
            self._check(self._L.emap_initialize_map(
                self._h, pts.ctypes.data, pts.shape[0], INIT_METHODS[method], None if tri is None else tri.ctypes.data,
                0 if tri is None else tri.shape[0], None if grad is None else grad.ctypes.data,
                float(self.param.initialized_variance), int(self.param.dilation_size_initialize)))


class _DepthFrame:
    """The depth cameras of one frame: `args` (n_cameras, cameras, is_device_ptr, n_channels, channel_source, n_features)
    of emap_input_depth_images and its sharded twins, the converted inputs they point at (`keep`), the frame's rows (its
    pixels) and its first camera's t[2]."""

    def __init__(self, args, keep, pixels, first_z):
        self.args, self.keep, self.pixels, self.first_z = args, keep, pixels, first_z


def _to_host(x):
    if isinstance(x, np.ndarray):
        return x
    if hasattr(x, "detach") and hasattr(x, "cpu"):      # torch tensor
        return x.detach().cpu().numpy()
    if hasattr(x, "get"):                                # cupy array
        return x.get()
    return np.asarray(x)


def regions_from_tables(regions, polygons, vertices):
    """extract_planar_regions' per-region dicts from the three flat tables (include/emap.h states their layout)."""
    out = []
    for r in regions:
        T = np.eye(4)
        T[:3, :] = r[1:13].reshape(3, 4)
        out.append({"label": int(r[0]), "transform": T, "bbox": r[13:17].copy(),
                    "boundary": {"outer": None, "holes": []}, "insets": []})
    for region, role, inset, first, count in polygons:
        pts = vertices[first:first + count].copy()
        d = out[region]
        if role == 0:
            d["boundary"]["outer"] = pts
        elif role == 1:
            d["boundary"]["holes"].append(pts)
        elif role == 2:
            d["insets"].append({"outer": pts, "holes": []})
        else:
            d["insets"][inset]["holes"].append(pts)
    return out


_PLANE_LAYERS = ["elevation_raw", "elevation", "segmentation", "plane_classification"]
_TERRAIN_LAYERS = ["elevation_raw", "elevation_before_postprocess", "segmentation", "plane_classification",
                   "elevationWithNaN", "elevationWithNaN_i", "elevationWithNaNClosed", "elevationWithNaNClosedDilated",
                   "smooth_planar", "elevation"]


def _plane_result(names, out, rows, cols, res, centre, planes, info):
    """What segment_planes and the planar-region calls return alike, from the flat layers `out`, the plane table and
    the first five info words: the (rows, cols) views per layer name, the planes, the window's geometry and success."""
    n = rows * cols
    flat = out.reshape(-1)
    return {"layers": {name: flat[k * n:(k + 1) * n].reshape(rows, cols) for k, name in enumerate(names)},
            "planes": planes[:int(info[4])], "highest_label": int(info[3]),
            "origin": centre + (0.5 * (np.array([rows, cols]) * res) - 0.5 * res), "centre": centre.copy(),
            "resolution": res, "size": (rows, cols), "success": bool(info[0])}


def _array_maker(device):
    """make(shape, dtype name) for new NumPy arrays (device None) or torch tensors on `device`."""
    if device is None:
        return lambda shape, dt: np.zeros(shape, dt)
    import torch
    return lambda shape, dt: torch.empty(shape, dtype=getattr(torch, dt), device=device)


def _output_device(arrays):
    """The device of the first CUDA array among `arrays` (None entries skipped): where a call that writes to the side of
    these arrays puts its output; None for host output."""
    return next((a.device for a in arrays if a is not None and _is_device(a)), None)


def _contiguous(a, dtype, device):
    """Is `a` a contiguous `dtype` torch CUDA tensor (device) or a C-contiguous `dtype` NumPy array (host)?"""
    if device:
        return str(getattr(a, "dtype", "")) == "torch." + dtype and a.is_contiguous()
    return isinstance(a, np.ndarray) and a.dtype == dtype and a.flags.c_contiguous


def _outputs(out, specs, dev):
    """The caller's `out` dict, checked against specs (_check_out), or new arrays of specs[k] = (shape, dtype name) on
    the device `dev` (None: NumPy) when it is None."""
    if out is None:
        return {k: _array_maker(dev)(shape, dt) for k, (shape, dt) in specs.items()}
    _check_out(out, specs, dev is not None)
    return out


def _check_out(out, specs, device):
    """Every out[k] is a contiguous array of specs[k] = (shape, dtype name) on the call's side (NumPy for host output,
    CUDA for device)."""
    for k, (shape, dtype) in specs.items():
        a = out[k]
        if tuple(a.shape) != shape or _is_device(a) != device or not _contiguous(a, dtype, device):
            raise TypeError("out[%r] must be a contiguous %s %s array of shape %s" % (
                k, dtype, "CUDA" if device else "NumPy", shape))


def _flat_out(out):
    """The float count of the flat float32 `out` of the window and plane calls, which must be contiguous."""
    if _is_device(out):
        if not _contiguous(out, "float32", True):
            raise TypeError("a device `out` must be a contiguous float32 torch CUDA tensor")
        return out.numel()
    if not _contiguous(out, "float32", False):
        raise TypeError("a host `out` must be a C-contiguous float32 NumPy array")
    return out.size


def _input_array(a, dtype, what, columns=None):
    """A grid layer, distance volume or region table (`what`) as the library reads it: a torch CUDA tensor is read in
    place and must be contiguous `dtype`; a host array becomes a C-contiguous NumPy array of `dtype`.  A table must have
    `columns` columns."""
    if _is_device(a):
        if not _contiguous(a, dtype, True):
            raise TypeError("a device %s must be a contiguous %s torch CUDA tensor" % (what, dtype))
    else:
        a = np.ascontiguousarray(a, dtype)
    if columns is not None and (a.ndim != 2 or a.shape[1] != columns):
        raise TypeError("a %s must have %d columns" % (what, columns))
    return a


def _queries(parts, width):
    """The query arrays `parts` side by side as one contiguous (N, width) float64 array: a torch CUDA tensor when any
    part is one, else NumPy."""
    k = width // len(parts)
    dev = _output_device(parts)
    if dev is not None:
        import torch
        parts = [torch.as_tensor(p, device=dev).to(torch.float64).reshape(-1, k) for p in parts]
        return (torch.cat(parts, 1) if len(parts) > 1 else parts[0]).contiguous()
    parts = [np.asarray(_to_host(p), np.float64).reshape(-1, k) for p in parts]
    return np.ascontiguousarray(np.concatenate(parts, 1) if len(parts) > 1 else parts[0])


def _is_device(x):
    return getattr(x, "__cuda_array_interface__", None) is not None if not hasattr(x, "is_cuda") else bool(x.is_cuda)


def _xy(v):
    """The first two values of a position or length, as a list of two floats."""
    return list(np.asarray(_to_host(v), np.float64).reshape(-1)[:2])


def _isometry(T):
    """The 12 doubles (R row-major, then t) of a 4 x 4 homogeneous transform or an (R, t) pair."""
    if isinstance(T, (tuple, list)) and len(T) == 2:
        R = np.asarray(_to_host(T[0]), np.float64).reshape(3, 3)
        t = np.asarray(_to_host(T[1]), np.float64).reshape(3)
    else:
        M = np.asarray(_to_host(T), np.float64)
        if M.shape != (4, 4):
            raise ValueError("a transform is a 4 x 4 array or an (R, t) pair")
        R, t = M[:3, :3], M[:3, 3]
    return np.concatenate([R.reshape(-1), t])


def _depth_input(x, dtype, dev, device, keep):
    """One input of input_depth_images as a contiguous array of `dtype` (a list of planes is stacked): a torch CUDA tensor
    when the call's inputs are on the device, else a NumPy array (a pinned torch CPU tensor stays in its pinned memory).
    The array is appended to `keep` for the duration of the call."""
    if _on_device(x) != dev:
        raise ValueError("depth-image inputs must be all host or all device arrays")
    if dev:
        import torch
        td = torch.uint8 if dtype == np.uint8 else torch.float32
        as_t = lambda p: torch.as_tensor(p, device=f"cuda:{device}")
        a = (torch.stack([as_t(p) for p in x]) if isinstance(x, (list, tuple)) else as_t(x)).to(td).contiguous()
    else:
        a = np.ascontiguousarray(np.stack([_to_host(p) for p in x]) if isinstance(x, (list, tuple)) else _to_host(x),
                                 dtype=dtype)
    keep.append(a)
    return a


def _on_device(x):
    """Is x (an array, or a list of planes that are all host or all device arrays) in device memory?"""
    if isinstance(x, (list, tuple)):
        kinds = {_is_device(p) for p in x}
        if len(kinds) != 1:
            raise ValueError("a list of planes must be all host or all device arrays")
        return kinds.pop()
    return _is_device(x)


def _address(a):
    """The data pointer of a NumPy array or torch tensor; None for None."""
    if a is None:
        return None
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def _image_stack(image, device):
    """(on_device, contiguous fp32 (C, H, W) array) of an input_image image (EM.py:504-509: np.stack, then a 2-D result
    gets a leading axis).  Device input stays on the device (a torch tensor); host input becomes a NumPy array."""
    parts = list(image) if isinstance(image, (list, tuple)) else None
    if any(_is_device(x) for x in (parts if parts is not None else [image])):
        import torch
        as_t = lambda x: torch.as_tensor(x, device=f"cuda:{device}")
        img = torch.stack([as_t(x) for x in parts]) if parts is not None else as_t(image)
        if img.dim() == 2:
            img = img[None]
        if img.dim() != 3:
            raise ValueError("image must be (C, H, W) or a list of (H, W) planes")
        return True, img.to(torch.float32).contiguous()
    img = np.stack([_to_host(x) for x in parts]) if parts is not None else _to_host(image)
    if img.ndim == 2:
        img = img[None]
    if img.ndim != 3:
        raise ValueError("image must be (C, H, W) or a list of (H, W) planes")
    return False, np.ascontiguousarray(img, dtype=np.float32)


def _clipped_area(poly, center, cell_n, resolution):
    """Shoelace area of the fp32 polygon after the clip of EM.py:847-851 (what emap_polygon_traversability tests against
    0.001 to declare the polygon outside of the map); every operation in fp32."""
    f = np.float32
    half, res = f(0.5 * (cell_n - 2) * resolution), f(resolution)
    c = np.asarray(center, np.float32)[:2]
    p = np.clip(poly, (c - half) + res, (c + half) - res).astype(np.float32)
    q = np.roll(p, 1, axis=0)                                          # q[i] = p[i - 1]
    terms = (q[:, 0] * p[:, 1] - q[:, 1] * p[:, 0]) / f(2)
    return abs(np.cumsum(terms, dtype=np.float32)[-1])                 # in order i = 0..n-1


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