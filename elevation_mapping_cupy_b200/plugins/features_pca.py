"""features_pca plugin -- the 3 principal components of the feature layers as a colour.

Behavioural mirror of the reference plugin (elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/
features_pca.py:13-96): the layers whose names `re.match` one of `process_layer_names` are taken from the map, the plugin
layers and the semantic layers, in that order; every cell is a sample, every value is clipped to [-1, 1]; the three
principal components are scaled to 0..255 each over the map and packed 0x00RRGGBB into the layer's bits.  The reference
copies the planes to the host and runs sklearn's PCA there; here it is one libemap.so call (emap_features_pca) that stays
on the device: fp64 statistics and eigen-decomposition, deterministic.  Differences: a component of range 0 gives channel
0 (the reference casts NaN); NaN input raises ValueError, as sklearn does; fewer than 3 layers raise ValueError, as
sklearn does; no layer gives zeros, as in the reference.
"""
from typing import List

from .. import _lib
from ._engine import pointer_array, require_engine, run_plugin, select_planes
from .plugin_manager import PluginBase


class FeaturesPca(PluginBase):
    def __init__(self, cell_n: int = 100, process_layer_names: List[str] = [], engine=None, **kwargs):
        super().__init__()
        self.process_layer_names = process_layer_names
        self.engine = engine

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str],
                 semantic_map, semantic_layer_names: List[str], *args):
        import torch
        eng = require_engine(self.engine, "FeaturesPca")
        planes = select_planes(self.process_layer_names, ((elevation_map, layer_names),
                                                          (plugin_layers, plugin_layer_names),
                                                          (semantic_map, semantic_layer_names)))
        if not planes:
            return torch.zeros_like(elevation_map[0])
        if len(planes) < 3:
            raise ValueError(f"features_pca needs at least 3 feature layers for 3 components, got {len(planes)}")
        try:
            return run_plugin(eng, "emap_features_pca", (), ptrs=(len(planes), pointer_array(planes)),
                              like=elevation_map[0])
        except _lib.EmapError as e:
            if "NaN" in str(e):
                raise ValueError(f"features_pca: input contains NaN ({e})") from e
            raise
