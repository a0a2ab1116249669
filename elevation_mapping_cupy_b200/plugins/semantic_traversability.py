"""semantic_traversability plugin -- traversability voted by thresholded layers.

Behavioural mirror of the reference plugin (elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/
semantic_traversability.py:12-83): each of `layers` is looked up in the map, then in the plugin layers (the reference does
not search the semantic layers); a cell scores one per layer whose value is <= its threshold (`type` "traversability") or
>= it (any other type); the layer is fp32(0.1) where the score is 0 and 1 elsewhere.  The comparison is made in fp64 (the
fp32 value widened, the threshold as given).  A name found nowhere prints the reference's message and, unlike the
reference (which returns None and fails on the assignment), returns the traversability layer as max_layer_filter does.
One libemap.so call (emap_semantic_traversability).
"""
import ctypes as C
from typing import List

from ._engine import as_plane, pointer_array, require_engine, run_plugin
from .plugin_manager import PluginBase


class SemanticTraversability(PluginBase):
    def __init__(self, cell_n: int = 100, layers: list = ["traversability"], thresholds: list = [0.5],
                 type: list = ["traversability"], engine=None, **kwargs):
        super().__init__()
        self.layers = layers
        self.thresholds = [float(t) for t in thresholds]
        self.type = type
        self.engine = engine

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str],
                 semantic_map, semantic_layer_names: List[str], *args):
        eng = require_engine(self.engine, "SemanticTraversability")
        planes = []
        for name in self.layers:
            if name in layer_names:
                planes.append(as_plane(elevation_map[layer_names.index(name)]))
            elif name in plugin_layer_names:
                planes.append(as_plane(plugin_layers[plugin_layer_names.index(name)]))
            else:
                print("Layer {} is not in the map, returning traversabiltiy!".format(name))
                return elevation_map[layer_names.index("traversability")]
        n = len(planes)
        thr = (C.c_double * n)(*self.thresholds[:n]) if n else None
        trav = (C.c_int32 * n)(*(int(t == "traversability") for t in self.type[:n])) if n else None
        return run_plugin(eng, "emap_semantic_traversability", (), ptrs=(n, pointer_array(planes), thr, trav),
                          like=elevation_map[0])
