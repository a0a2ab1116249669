"""Point-channel semantic layers of the map (SURVEY.md 8(f)2), fused by libemap.so inside the frame.

Mirrors the point-cloud half of the reference class
(elevation_mapping_cupy/script/elevation_mapping_cupy/semantic_map.py:13-259: layer bookkeeping, `get_fusion`,
`get_matching_fusion`, `get_indices_fusion`, `update_layers_pointcloud`) for the three fusion algorithms that ride on the
frame's point record: `average` (fusion/pointcloud_average.py), `class_average` (fusion/pointcloud_class_average.py, the
reference's default) and `color` (fusion/pointcloud_color.py).  The kernels are csrc/emap_semantic.cuh; this class only
decides which column of the cloud goes to which layer and hands the layer buffer to the engine
(`emap_semantic_configure_ext`).  The plugins that consume these layers (semantic_filter, semantic_traversability,
features_pca) are in plugins/.
The reference's three other point-cloud fusions fuse in the same frame: `class_bayesian`
(fusion/pointcloud_class_bayesian.py), `bayesian_inference` (pointcloud_bayesian_inference.py) and `class_max`
(pointcloud_class_max.py), as DESIGN §4d defines them.  `bayesian_inference` keeps a variance plane per layer
(`variance`, 1.0 at the start, reset to 1.0 by `clear`, moved with the map and padded with 1.0); `class_max` keeps the
class id of each of its rounds in `elements_to_shift["id_max"]` ((n_class_max, W, W) int32, 0 at the start, moved with
the map and padded with 0, kept by `clear`).
Camera images (ElevationMap.input_image) fuse into the same layers: `update_layers_image` picks each channel's fusion
(`image_channel_fusions`: `color`, fusion/image_color.py, or `exponential`, fusion/image_exponential.py) and layer, and
one library call (`emap_input_image`, csrc/emap_image.cuh) projects, tests occlusion and writes every channel.  A layer
an image adds reallocates the buffer; the point-channel registration is moved to the new buffer at once.
The image feature extractors are out of scope.
"""
import ctypes as C
import re
from typing import Dict, List

import numpy as np

KINDS = {"average": 0, "class_average": 1, "color": 2,            # EMAP_SEM_*
         "class_bayesian": 3, "bayesian_inference": 4, "class_max": 5}
IMAGE_KINDS = {"color": 0, "exponential": 1}          # EMAP_IMAGE_COLOR, EMAP_IMAGE_EXPONENTIAL


class SemanticMap:
    def __init__(self, param, engine=None):
        self.param = param
        self.engine = engine
        self.layer_specs_points: Dict[str, str] = {}
        self.layer_specs_image: Dict[str, str] = {}
        self.layer_names: List[str] = []
        self.semantic_map = None           # torch (n_layers, W, W) float32 on the engine's device, grown by add_layer
        self._configured = None
        self._registered = None            # (columns, kinds, layers) the engine fuses point channels with, or None
        self.variance = None               # (n_layers, W, W) float32 variance planes of bayesian_inference, made on first use
        self.elements_to_shift = {}        # "id_max": (n_class_max, W, W) int32, made when a class_max channel is configured

    # ---- layer bookkeeping (semantic_map.py:47-99) ----------------------------------------------------------------
    def _alloc(self, n):
        import torch
        W = self.param.cell_n
        return torch.zeros((n, W, W), dtype=torch.float32, device=f"cuda:{self.engine.device}")

    def clear(self):
        if self.semantic_map is not None:
            self.semantic_map.zero_()
        if self.variance is not None:
            self.variance.fill_(1.0)

    def add_layer(self, name):
        import torch
        if name in self.layer_names:
            return
        self.layer_names.append(name)
        new = self._alloc(1)
        if self.semantic_map is None:
            self.semantic_map = new
        else:
            self.engine._before_framework()        # the engine's queued writes to the old buffer come first
            self.semantic_map = torch.cat([self.semantic_map, new], 0)
            if self.variance is not None:
                self.variance = torch.cat([self.variance, torch.ones_like(new)], 0)
        if self._registered is not None:           # the old buffer is freed: point the engine's fusion at the new one
            self._register(*self._registered)

    def get_matching_fusion(self, channel: str, fusion_algs: Dict[str, str]):
        for pattern, alg in fusion_algs.items():          # semantic_map.py:186-191
            if re.match(f"^{pattern}$", channel):
                return alg
        return None

    def get_fusion(self, channels: List[str], channel_fusions: Dict[str, str], layer_specs: Dict[str, str]):
        """semantic_map.py:150-184: the fusion algorithm of every channel (regex match, then `default`)."""
        fusion_list, process_channels = [], []
        for channel in channels:
            if channel not in layer_specs:
                matched = self.get_matching_fusion(channel, channel_fusions)
                if matched is None:
                    if "default" in channel_fusions:
                        matched = channel_fusions["default"]
                        print(f"[WARNING] Layer {channel} not found in layer_specs. Using {matched} algorithm as default.")
                    else:
                        print(f"[WARNING] Layer {channel} not found in layer_specs ({layer_specs}) and no default fusion is configured. Skipping.")
                        continue
                layer_specs[channel] = matched
            fusion_list.append(layer_specs[channel])
            process_channels.append(channel)
        return process_channels, fusion_list

    # ---- the frame hook (semantic_map.py:223-259) --------------------------------------------------------------------
    def configure_for(self, channels: List[str]):
        """Called by ElevationMap.input_pointcloud with the cloud's channel names (x, y, z first): registers the feature
        columns with the engine so that the frame fuses them.  Idempotent for an unchanged channel list."""
        feats = list(channels[3:])
        key = tuple(channels)
        if self._configured == key:
            return
        if not feats:
            self._register(None)
            self._configured = key
            return
        fusions = getattr(self.param, "pointcloud_channel_fusions", None) or {"rgb": "color", "default": "class_average"}
        process, fusion = self.get_fusion(feats, fusions, self.layer_specs_points)
        cols, kinds, layers = [], [], []
        for ch, alg in zip(process, fusion):
            if alg not in KINDS:
                raise NotImplementedError(f"point-cloud fusion '{alg}' (channel {ch}) is not implemented; available: {sorted(KINDS)}")
            if ch not in self.layer_names:
                print(f"Layer {ch} not found, adding it to the semantic map")
                self.add_layer(ch)
            cols.append(3 + feats.index(ch)); kinds.append(KINDS[alg]); layers.append(self.layer_names.index(ch))
        self._alloc_state(kinds)
        self._register(cols, kinds, layers)        # no channel has a fusion: nothing to fuse
        self._configured = tuple(channels)

    def _alloc_state(self, kinds):
        """The variance planes (first bayesian_inference channel) and id_max (grown to this cloud's class_max channels;
        new planes start at 0)."""
        import torch
        if KINDS["bayesian_inference"] in kinds and self.variance is None:
            self.engine._before_framework()
            self.variance = torch.ones_like(self.semantic_map)
        n_max = kinds.count(KINDS["class_max"])
        old = self.elements_to_shift.get("id_max")
        if n_max and (old is None or old.shape[0] < n_max):
            W = self.param.cell_n
            new = torch.zeros((n_max, W, W), dtype=torch.int32, device=self.semantic_map.device)
            if old is not None:
                self.engine._before_framework()
                new[:old.shape[0]] = old
            self.elements_to_shift["id_max"] = new

    def _register(self, cols, kinds=None, layers=None):
        """Hands the point-channel fusion (or None: no fusion), the current layer buffer and the fusion state (variance
        planes, id_max) to the engine."""
        eng = self.engine
        if not cols:
            eng._check(eng._L.emap_semantic_configure_ext(eng._h, 0, None, None, None, None, 0, 0.0, None, None, 0))
            self._registered = None
            return
        n = len(cols)
        arr = lambda v: (C.c_int32 * n)(*v)
        id_max = self.elements_to_shift.get("id_max")
        eng._check(eng._L.emap_semantic_configure_ext(
            eng._h, n, arr(cols), arr(kinds), arr(layers), C.c_void_p(self.semantic_map.data_ptr()), len(self.layer_names),
            float(getattr(self.param, "average_weight", 0.5)),
            None if self.variance is None else C.c_void_p(self.variance.data_ptr()),
            None if id_max is None else C.c_void_p(id_max.data_ptr()), 0 if id_max is None else id_max.shape[0]))
        self._registered = (cols, kinds, layers)

    # ---- the image hook (semantic_map.py:261-309) ----------------------------------------------------------------------
    def update_layers_image(self, channels: List[str]):
        """The channel selection of update_layers_image: (planes, kinds, layers) of the channels the image fuses.  Channel j
        of the processed list reads image plane j; a missing layer is added; a fusion other than color / exponential
        prints the reference's warning and is skipped (its layer is still added)."""
        fusions = getattr(self.param, "image_channel_fusions", None) or {"rgb": "color", "default": "exponential"}
        process, fusion = self.get_fusion(channels, fusions, self.layer_specs_image)
        planes, kinds, layers = [], [], []
        for j, (alg, ch) in enumerate(zip(fusion, process)):
            if ch not in self.layer_names:
                print(f"Layer {ch} not found, adding it to the semantic map")
                self.add_layer(ch)
            if alg not in IMAGE_KINDS:
                print(f"[WARNING] Plugin image_{alg} is not in the list: {['image_' + k for k in IMAGE_KINDS]}")
                continue
            planes.append(j); kinds.append(IMAGE_KINDS[alg]); layers.append(self.layer_names.index(ch))
        return planes, kinds, layers

    # ---- queries (semantic_map.py:318-385) ----------------------------------------------------------------------------
    def get_map_with_name(self, name):
        return self.semantic_map[self.layer_names.index(name)][1:-1, 1:-1].clone()

    def get_index(self, name):
        return self.layer_names.index(name) if name in self.layer_names else -1

    @staticmethod
    def _shift(buf, sx, sy, pad):
        import torch
        m = torch.roll(buf, (sx, sy), dims=(1, 2))
        if sx > 0: m[:, :sx, :] = pad
        elif sx < 0: m[:, sx:, :] = pad
        if sy > 0: m[:, :, :sy] = pad
        elif sy < 0: m[:, :, sy:] = pad
        buf.copy_(m)

    def shift_map_xy(self, shift_value):
        """semantic_map.py:131-148: roll + zero padding, applied with the elevation map's shift.  The variance planes
        are padded with 1.0 (their initial value), id_max with 0."""
        if self.semantic_map is None or (shift_value[0] == 0 and shift_value[1] == 0):
            return
        sx, sy = int(shift_value[0]), int(shift_value[1])
        self._shift(self.semantic_map, sx, sy, 0.0)
        if self.variance is not None:
            self._shift(self.variance, sx, sy, 1.0)
        if "id_max" in self.elements_to_shift:
            self._shift(self.elements_to_shift["id_max"], sx, sy, 0)
