"""smooth_filter plugin: the chosen layer passed twice through a 3x3 mean with mirrored borders.

The reference (elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/smooth_filter.py:12-59) calls
cupyx.scipy.ndimage.uniform_filter(size=3) two times; here the four 1-D passes run in libemap.so
(`emap_smooth_filter`) with the same double-precision accumulation per pass.  Falls back to the elevation
layer, with the reference's message, when `input_layer_name` is unknown.
"""
from typing import List

from .plugin_manager import PluginBase
from ._engine import require_engine, run_plugin


class SmoothFilter(PluginBase):
    def __init__(self, cell_n: int = 100, input_layer_name: str = "elevation", engine=None, **kwargs):
        super().__init__()
        self.input_layer_name = input_layer_name
        self.engine = engine

    def _source(self, elevation_map, layer_names, plugin_layers, plugin_layer_names):
        want = self.input_layer_name
        for names, store in ((layer_names, elevation_map), (plugin_layer_names, plugin_layers)):
            if want in names:
                return store[names.index(want)]
        print("layer name {} was not found. Using elevation layer.".format(want))
        return elevation_map[0]

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str], *args):
        eng = require_engine(self.engine, "SmoothFilter")
        return run_plugin(eng, "emap_smooth_filter", (self._source(elevation_map, layer_names, plugin_layers, plugin_layer_names),))
