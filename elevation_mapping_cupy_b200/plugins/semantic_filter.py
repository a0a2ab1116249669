"""semantic_filter plugin -- the colour of the most likely class per cell.

Behavioural mirror of the reference plugin (elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/
semantic_filter.py:13-133): the layers whose names `re.match` one of `classes` are taken from the map, the plugin layers and
the semantic layers, in that order; the class id of a cell is `argmax` over them (the first maximum wins, a NaN is the
maximum) and the layer holds the bits of that id's entry of the reference palette `color_map(255)` (packed 0x00RRGGBB, read
the plane as uint32).  One libemap.so call (emap_semantic_filter); the library holds the palette.
"""
from typing import List

from ._engine import pointer_array, require_engine, run_plugin, select_planes
from .plugin_manager import PluginBase


class SemanticFilter(PluginBase):
    def __init__(self, cell_n: int = 100, classes: list = ["person", "grass"], engine=None, **kwargs):
        super().__init__()
        self.indices = []
        self.classes = classes
        self.engine = engine

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str],
                 semantic_map, semantic_layer_names: List[str], *args):
        eng = require_engine(self.engine, "SemanticFilter")
        planes = select_planes(self.classes, ((elevation_map, layer_names), (plugin_layers, plugin_layer_names),
                                              (semantic_map, semantic_layer_names)))
        return run_plugin(eng, "emap_semantic_filter", (), ptrs=(len(planes), pointer_array(planes)),
                          like=elevation_map[0])
