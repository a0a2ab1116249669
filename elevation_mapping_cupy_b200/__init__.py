"""elevation_mapping_cupy_b200 -- H100-native (sm_90a) engine for the point-cloud fusion path of
elevation_mapping_cupy, behind the reference's ElevationMap / plugin API."""
from .parameter import Parameter, core_parameter  # noqa: F401


def __getattr__(name):
    if name == "ElevationMap":
        from .elevation_mapping import ElevationMap
        return ElevationMap
    raise AttributeError(name)
