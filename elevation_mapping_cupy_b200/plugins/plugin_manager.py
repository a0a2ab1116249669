"""Plugin layer API of the drop-in.

Contract taken from the reference's plugin manager
(elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/plugin_manager.py): the names `PluginParams`,
`PluginBase`, `PluginManager` and their public methods (:15-20, :23-108, :111-235), the YAML schema
(`enable, fill_nan, is_height_layer, layer_name, type?, extra_params`, :134-151), the injection of `cell_n` into the
plugin constructor (:128) and the dispatch on the ARITY of a plugin's `__call__` (:193-225: 5, 7, 8 parameters, else
all of them).  Differences: layers are torch CUDA tensors (they expose `__cuda_array_interface__`), the YAML is read
with PyYAML, and the manager hands its `engine` (the owning ElevationMap) to plugin constructors so that the built-in
plugins can run libemap.so kernels -- user plugins simply swallow it in **kwargs like every reference plugin does.
"""
from abc import ABC
from dataclasses import dataclass
import importlib
import inspect
from typing import Dict, List, Optional

import yaml


@dataclass
class PluginParams:
    name: str                      # module (file) name of the plugin
    layer_name: str                # name of the layer it produces
    fill_nan: bool = False         # export: NaN where the elevation cell is not valid
    is_height_layer: bool = False  # export: add the map centre height


class PluginBase(ABC):
    """Base class: subclass it in a module of the plugin package and implement `__call__`.

    `__call__(elevation_map, layer_names, plugin_layers, plugin_layer_names[, semantic_map, semantic_layer_names
    [, rotation[, elements_to_shift]]])` returns one `(cell_n, cell_n)` device array.  Layer order of
    `elevation_map`: elevation, variance, is_valid, traversability, time, upper_bound, is_upper_bound.
    """

    def __init__(self, *args, **kwargs):
        pass

    def __call__(self, elevation_map, layer_names: List[str], plugin_layers, plugin_layer_names: List[str],
                 semantic_map=None, semantic_layer_names: List[str] = None, *args, **kwargs):
        return None

    def get_layer_data(self, elevation_map, layer_names, plugin_layers, plugin_layer_names, semantic_map,
                       semantic_layer_names, name) -> Optional[object]:
        """A private copy of the layer called `name`, searched in the map, the plugin layers, then the semantic layers."""
        for names, store in ((layer_names, elevation_map), (plugin_layer_names, plugin_layers),
                             (semantic_layer_names or [], semantic_map)):
            if name in names:
                return store[names.index(name)].clone()
        print(f"Could not find layer {name}!")
        return None


class _MissingPlugin(PluginBase):
    """Stands in for a plugin module that is not part of this package."""

    def __init__(self, name):
        super().__init__()
        self.name = name

    def __call__(self, elevation_map, layer_names, plugin_layers, plugin_layer_names, *args):
        raise NotImplementedError(f"plugin {self.name!r} is not provided by this package")


class PluginManager(object):
    def __init__(self, cell_n: int, engine=None, package: str = "elevation_mapping_cupy_b200.plugins"):
        self.cell_n = cell_n
        self.engine = engine
        self.package = package
        self.plugin_params: List[PluginParams] = []
        self.plugins: list = []
        self.layers = None                 # (n_plugins, cell_n, cell_n) fp32, allocated on first use
        self.layer_names: List[str] = []
        self.plugin_names: List[str] = []

    # ---- construction ------------------------------------------------------------------------
    def init(self, plugin_params: List[PluginParams], extra_params: List[Dict]):
        self.plugin_params = list(plugin_params)
        self.plugins = []
        for spec, extra in zip(plugin_params, extra_params):
            try:
                module = importlib.import_module("." + spec.name, package=self.package)
            except ImportError as e:
                # a YAML written for the reference may name a plugin module this package does not provide: keep the
                # layer slot, say so, and fail only if it is evaluated
                print(f"plugin {spec.name!r} is not provided by {self.package} ({e}); its layer will raise when requested")
                self.plugins.append(_MissingPlugin(spec.name))
                continue
            kwargs = dict(extra or {}, cell_n=self.cell_n, engine=self.engine)
            for cls_name, cls in inspect.getmembers(module, inspect.isclass):
                if cls_name != "PluginBase" and issubclass(cls, PluginBase):
                    self.plugins.append(cls(**kwargs))
        self.layers = None
        self.layer_names = self.get_layer_names()
        self.plugin_names = self.get_plugin_names()

    def load_plugin_settings(self, file_path: str):
        print("Start loading plugins...")
        with open(file_path, "r") as stream:
            entries = yaml.safe_load(stream) or {}
        specs, extras = [], []
        for key, entry in entries.items():
            if not entry["enable"]:
                continue
            specs.append(PluginParams(name=entry.get("type", key), layer_name=entry["layer_name"],
                                      fill_nan=entry["fill_nan"], is_height_layer=entry["is_height_layer"]))
            extras.append(entry.get("extra_params", {}))
        self.init(specs, extras)
        print("Loaded plugins are ", *self.plugin_names)

    # ---- look-ups ----------------------------------------------------------------------------
    def get_layer_names(self):
        return [spec.layer_name for spec in self.plugin_params]

    def get_plugin_names(self):
        return [spec.name for spec in self.plugin_params]

    def get_plugin_index_with_name(self, name: str) -> Optional[int]:
        if name in self.plugin_names:
            return self.plugin_names.index(name)
        print("Error with plugin {}: not loaded".format(name))
        return None

    def get_layer_index_with_name(self, name: str) -> Optional[int]:
        if name in self.layer_names:
            return self.layer_names.index(name)
        print("Error with layer {}: not a plugin layer".format(name))
        return None

    def get_map_with_name(self, name: str):
        idx = self.get_layer_index_with_name(name)
        return None if idx is None or self.layers is None else self.layers[idx]

    def get_param_with_name(self, name: str) -> Optional[PluginParams]:
        idx = self.get_layer_index_with_name(name)
        return None if idx is None else self.plugin_params[idx]

    # ---- evaluation --------------------------------------------------------------------------
    def _storage(self, like):
        if self.layers is None:
            import torch
            self.layers = torch.zeros((len(self.plugins), self.cell_n, self.cell_n), dtype=torch.float32,
                                      device=like.device)
        return self.layers

    def update_with_name(self, name: str, elevation_map, layer_names: List[str], semantic_map=None,
                         semantic_params=None, rotation=None, elements_to_shift={}):
        """Recompute the plugin layer `name`.  How many optional arguments the plugin receives depends on how many
        parameters its `__call__` declares (plugin_manager.py:193-225 of the reference)."""
        idx = self.get_layer_index_with_name(name)
        if idx is None or idx >= len(self.plugins):
            return
        layers = self._storage(elevation_map)
        plugin = self.plugins[idx]
        optional = (semantic_map, semantic_params, rotation, elements_to_shift)
        n_optional = {5: 0, 7: 2, 8: 3}.get(len(inspect.signature(plugin).parameters), 4)
        layers[idx] = plugin(elevation_map, layer_names, layers, self.layer_names, *optional[:n_optional])
