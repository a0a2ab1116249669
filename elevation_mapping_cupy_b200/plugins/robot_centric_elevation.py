"""robot_centric_elevation plugin: height of every valid cell in the base frame, optionally thresholded
(reference: elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/robot_centric_elevation.py:12-121).
Runs in libemap.so (`emap_robot_centric_elevation`)."""
from typing import List

import numpy as np

from .plugin_manager import PluginBase
from ._engine import require_engine, run_plugin


class RobotCentricElevation(PluginBase):
    def __init__(self, cell_n: int = 100, resolution: float = 0.05, threshold: float = 0.4, use_threshold: bool = 0,
                 engine=None, **kwargs):
        super().__init__()
        self.width = self.height = cell_n
        self.resolution = float(resolution)
        self.threshold = float(threshold)
        self.use_threshold = int(bool(use_threshold))
        self.engine = engine

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str],
                 semantic_map, semantic_layer_names: List[str], rotation, *args):
        eng = require_engine(self.engine, "RobotCentricElevation")
        R = rotation.detach().cpu().numpy() if hasattr(rotation, "detach") else np.asarray(rotation)
        R = np.ascontiguousarray(R, dtype=np.float32).reshape(9)
        return run_plugin(eng, "emap_robot_centric_elevation", (elevation_map[0], elevation_map[2]), self.resolution,
                          self.threshold, self.use_threshold, ptrs=(R.ctypes.data,))
