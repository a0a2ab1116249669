"""min_filter plugin: fill invalid cells with the minimum of their valid neighbours, iterated
(reference: elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/min_filter.py:12-118).
The stencil iterations run in libemap.so (`emap_min_filter`, Jacobi order, no host sync per iteration)."""
from .plugin_manager import PluginBase
from ._engine import FillFilter


class MinFilter(FillFilter, PluginBase):
    ENTRY = "emap_min_filter"
