"""Helpers shared by the built-in plugins: call a libemap.so stencil on torch CUDA tensors.
Ordering with the caller's torch stream is by stream waits (ElevationMap._ordered_call), never a host sync."""


def require_engine(engine, who):
    if engine is None:
        raise RuntimeError(f"{who} runs libemap.so kernels and needs the ElevationMap engine "
                           "(PluginManager(cell_n, engine=elevation_map)); there is no CPU fallback")
    return engine


def as_plane(t):
    """contiguous float32 CUDA (W,W) tensor"""
    import torch
    if not t.is_cuda:
        raise TypeError("plugin layers must be CUDA tensors")
    return t.to(torch.float32).contiguous()


def run_plugin(eng, entry, planes, *args, ptrs=(), like=None):
    """Runs the library entry point `entry` of the engine `eng` (require_engine) as `entry(handle, *planes, *ptrs, out,
    *args)` and returns `out`, a new (W,W) plane shaped like planes[0] (or `like` when `planes` is empty).  `planes` are
    (W,W) CUDA layers, `ptrs` raw pointers the entry point takes before the output.  The call runs after the torch work
    queued so far and before the torch work queued next."""
    import torch
    planes = [as_plane(p) for p in planes]
    out = torch.empty_like(as_plane(planes[0] if planes else like))
    eng._ordered_call(getattr(eng._L, entry), eng._h, *(p.data_ptr() for p in planes), *ptrs, out.data_ptr(), *args,
                      after=True, before=True)
    return out


def select_planes(patterns, stores):
    """The planes whose layer name `re.match`es one of `patterns`, store by store and in layer order within a store
    (semantic_filter.py:77-89, 116-122 of the reference).  `stores`: (layers, names) pairs; layers may be None when
    `names` is empty (no semantic layer yet)."""
    import re
    return [as_plane(layers[i]) for layers, names in stores for i, name in enumerate(names or [])
            if any(re.match(p, name) for p in patterns)]


def pointer_array(planes):
    """ctypes host array of the planes' device pointers (None for no plane)"""
    import ctypes as C
    return (C.c_void_p * len(planes))(*(p.data_ptr() for p in planes)) if planes else None


class FillFilter:
    """Body of MinFilter and MaxFilter (`ENTRY`: emap_min_filter / emap_max_filter).  Not a PluginBase subclass:
    PluginManager instantiates every PluginBase subclass a plugin module holds, imported ones included."""
    ENTRY = None

    def __init__(self, cell_n: int = 100, dilation_size: int = 5, iteration_n: int = 5, engine=None, **kwargs):
        super().__init__()
        self.iteration_n = int(iteration_n)
        self.dilation_size = int(dilation_size)
        self.width = self.height = cell_n
        self.engine = engine

    def __call__(self, elevation_map, layer_names, plugin_layers, plugin_layer_names, *args):
        eng = require_engine(self.engine, type(self).__name__)
        return run_plugin(eng, self.ENTRY, (elevation_map[0], elevation_map[2]), self.dilation_size, self.iteration_n, None)
