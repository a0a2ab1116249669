"""Parameter set of the elevation map -- host-side mirror of the reference's
`Parameter` dataclass (elevation_mapping_cupy/script/elevation_mapping_cupy/parameter.py:137-226,
update() at :282-289) restricted to the fields the fusion path reads, with the same
names, defaults and reflection helpers (`get_names/get_types/set_value/get_value`,
parameter.py:242-280) the C++ bridge uses to push rosparams
(elevation_mapping_cupy/src/elevation_mapping_wrapper.cpp:45-77).

`simple_parsing.Serializable` is not needed for the path and is not a dependency.
"""
from dataclasses import dataclass, field, fields
import os
import pickle

import numpy as np

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
DEFAULT_WEIGHT_FILE = os.path.join(_PKG_DIR, "config", "core", "weights.dat")
DEFAULT_PLUGIN_CONFIG = os.path.join(_PKG_DIR, "config", "core", "plugin_config.yaml")


@dataclass
class Parameter:
    resolution: float = 0.04
    subscriber_cfg: dict = field(default_factory=dict)
    additional_layers: list = field(default_factory=list)
    fusion_algorithms: list = field(default_factory=list)
    pointcloud_channel_fusions: dict = field(default_factory=lambda: {"rgb": "color", "default": "class_average"})  # parameter.py:160
    image_channel_fusions: dict = field(default_factory=lambda: {"rgb": "color", "default": "exponential"})  # parameter.py:161
    data_type: str = np.float32
    average_weight: float = 0.5

    map_length: float = 8.0
    sensor_noise_factor: float = 0.05
    mahalanobis_thresh: float = 2.0
    outlier_variance: float = 0.01
    drift_compensation_variance_inlier: float = 0.1
    time_variance: float = 0.01
    time_interval: float = 0.1

    max_variance: float = 1.0
    dilation_size: float = 2
    dilation_size_initialize: float = 10
    drift_compensation_alpha: float = 1.0

    traversability_inlier: float = 0.1
    wall_num_thresh: float = 100
    min_height_drift_cnt: float = 100

    max_ray_length: float = 2.0
    cleanup_step: float = 0.01
    cleanup_cos_thresh: float = 0.5
    min_valid_distance: float = 0.3
    max_height_range: float = 1.0
    ramped_height_range_a: float = 0.3
    ramped_height_range_b: float = 1.0
    ramped_height_range_c: float = 0.2

    safe_thresh: float = 0.5
    safe_min_thresh: float = 0.5
    max_unsafe_n: int = 20
    checker_layer: str = "traversability"

    min_filter_size: int = 5
    min_filter_iteration: int = 3

    max_drift: float = 0.10

    overlap_clear_range_xy: float = 4.0
    overlap_clear_range_z: float = 2.0

    enable_edge_sharpen: bool = True
    enable_drift_compensation: bool = True
    enable_visibility_cleanup: bool = True
    enable_overlap_clearance: bool = True
    use_only_above_for_upper_bound: bool = True
    use_chainer: bool = False          # no chainer path here: the CNN is a CUDA kernel
    position_noise_thresh: float = 0.1
    orientation_noise_thresh: float = 0.1

    plugin_config_file: str = DEFAULT_PLUGIN_CONFIG
    weight_file: str = DEFAULT_WEIGHT_FILE

    initial_variance: float = 10.0
    initialized_variance: float = 10.0
    w1: np.ndarray = field(default_factory=lambda: np.zeros((4, 1, 3, 3)))
    w2: np.ndarray = field(default_factory=lambda: np.zeros((4, 1, 3, 3)))
    w3: np.ndarray = field(default_factory=lambda: np.zeros((4, 1, 3, 3)))
    w_out: np.ndarray = field(default_factory=lambda: np.zeros((1, 12, 1, 1)))

    true_map_length: float = None
    cell_n: int = None
    true_cell_n: int = None

    def __post_init__(self):
        if self.cell_n is None:
            self.update()

    def load_weights(self, filename):
        """parameter.py:228-240 -- pickle of numpy arrays keyed like the torch module."""
        with open(filename, "rb") as file:
            weights = pickle.load(file)
            self.w1 = weights["conv1.weight"]
            self.w2 = weights["conv2.weight"]
            self.w3 = weights["conv3.weight"]
            self.w_out = weights["conv_final.weight"]

    def get_names(self):
        return [f.name for f in fields(self)]

    def get_types(self):
        return [getattr(f.type, "__name__", str(f.type)) for f in fields(self)]

    def set_value(self, name, value):
        setattr(self, name, value)

    def get_value(self, name):
        return getattr(self, name)

    def update(self):
        """parameter.py:282-289: +2 is the never-fused border ring."""
        self.cell_n = int(round(self.map_length / self.resolution)) + 2
        self.true_cell_n = round(self.map_length / self.resolution)
        self.true_map_length = self.true_cell_n * self.resolution


# Values deployed by elevation_mapping_cupy/config/core/core_param.yaml.  The YAML key
# `drift_compensation_variance_inler` (core_param.yaml:7) is misspelt, so the field
# `drift_compensation_variance_inlier` keeps its dataclass default 0.1 (SURVEY section 5).
CORE_PARAM_YAML = dict(
    resolution=0.04, map_length=8.0, sensor_noise_factor=0.05, mahalanobis_thresh=2.0,
    outlier_variance=0.01, max_drift=0.1, drift_compensation_alpha=0.1, time_variance=0.0001,
    max_variance=100.0, initial_variance=1000.0, traversability_inlier=0.9, dilation_size=3,
    wall_num_thresh=20, min_height_drift_cnt=100, position_noise_thresh=0.01,
    orientation_noise_thresh=0.01, min_valid_distance=0.5, max_height_range=1.0,
    ramped_height_range_a=0.3, ramped_height_range_b=1.0, ramped_height_range_c=0.2,
    time_interval=0.1, max_ray_length=10.0, cleanup_step=0.1, cleanup_cos_thresh=0.1,
    safe_thresh=0.7, safe_min_thresh=0.4, max_unsafe_n=10, overlap_clear_range_xy=4.0,
    overlap_clear_range_z=2.0, enable_edge_sharpen=True, enable_visibility_cleanup=True,
    enable_drift_compensation=True, enable_overlap_clearance=True,
    use_only_above_for_upper_bound=False, dilation_size_initialize=2,
)


def core_parameter(cell_n=None, **overrides):
    """Parameter with the deployed core_param.yaml values; `cell_n` picks map_length
    so that round(map_length/resolution)+2 == cell_n (e.g. 1024 -> 40.88 m)."""
    kw = dict(CORE_PARAM_YAML)
    kw.update(overrides)
    if cell_n is not None:
        kw["map_length"] = round((cell_n - 2) * kw["resolution"], 6)
    p = Parameter(**kw)
    p.update()
    if cell_n is not None:
        assert p.cell_n == cell_n, (p.cell_n, cell_n)
    return p
