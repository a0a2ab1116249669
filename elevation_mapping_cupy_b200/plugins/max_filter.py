"""max_filter plugin: fill invalid cells with the maximum of their valid neighbours, iterated (Jacobi)
(reference: elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/max_filter.py:12-113).
Runs in libemap.so (`emap_max_filter`)."""
from .plugin_manager import PluginBase
from ._engine import FillFilter


class MaxFilter(FillFilter, PluginBase):
    ENTRY = "emap_max_filter"
