"""inpainting plugin: fill the invalid cells of the elevation layer from their valid surroundings.

Reference: elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/inpainting.py:14-63 -- the map is copied to the
host, normalised to 8 bits over the valid cells, passed through `cv2.inpaint(h, mask, 1, INPAINT_TELEA)` on the CPU and
copied back.  Here the whole chain stays on the device: `emap_inpaint` (libemap.so) replays OpenCV's fast-marching fill in
parallel and returns the bit-identical result (csrc/emap_inpaint.cuh), about an order of magnitude faster than the CPU
call on large maps and without the two PCIe copies.  `method="ns"` (Navier-Stokes) is not implemented and raises.
"""
from typing import List

from .plugin_manager import PluginBase
from ._engine import require_engine, run_plugin


class Inpainting(PluginBase):
    def __init__(self, cell_n: int = 100, method: str = "telea", engine=None, **kwargs):
        super().__init__()
        # inpainting.py:25-30: anything that is not "ns" selects Telea
        self.method = 1 if method == "ns" else 0
        self.engine = engine

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str], *args):
        eng = require_engine(self.engine, "Inpainting")
        if self.method != 0:
            raise NotImplementedError("Inpainting(method='ns'): the Navier-Stokes variant is not implemented on the device")
        return run_plugin(eng, "emap_inpaint", (elevation_map[0], elevation_map[2]), self.method)
