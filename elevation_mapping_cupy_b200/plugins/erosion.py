"""erosion plugin: 8-bit normalise a layer, erode it with a ones(kernel_size) kernel, de-normalise
(reference: elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/erosion.py:12-113, which moves the layer
to the host and calls cv2.erode).  Here the same arithmetic runs on the device (`emap_erode`)."""
from typing import List

from .plugin_manager import PluginBase
from ._engine import require_engine, run_plugin


class Erosion(PluginBase):
    def __init__(self, input_layer_name="traversability", kernel_size: int = 3, iterations: int = 1,
                 reverse: bool = False, default_layer_name: str = "traversability", engine=None, **kwargs):
        super().__init__()
        self.input_layer_name = input_layer_name
        self.kernel_size = int(kernel_size)
        self.iterations = int(iterations)
        self.reverse = bool(reverse)
        self.default_layer_name = default_layer_name
        self.engine = engine

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str],
                 semantic_map, semantic_layer_names: List[str], *args):
        eng = require_engine(self.engine, "Erosion")
        semantic_layer_names = semantic_layer_names or []
        layer = None
        for name in (self.input_layer_name, self.default_layer_name, "traversability"):    # erosion.py:62-95
            layer = self.get_layer_data(elevation_map, layer_names, plugin_layers, plugin_layer_names, semantic_map,
                                        semantic_layer_names, name)
            if layer is not None:
                break
            print(f"No layers are found, using {self.default_layer_name}!")
        return run_plugin(eng, "emap_erode", (layer,), self.kernel_size, self.iterations, int(self.reverse))
