"""CPU tests of the argument checks the query calls of ElevationMap share (_check_out, _flat_out, _input_array, _grid,
_queries, _layer_sources in elevation_mapping.py): every malformed NumPy `out`, table or layer name is rejected before
the library is touched.  No GPU and no libemap.so: the map's library is a stub that fails on any use."""
import math
import threading
import types

import numpy as np
import pytest

from elevation_mapping_cupy_b200 import _lib
from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap, _queries


@pytest.fixture(autouse=True)
def no_library(monkeypatch):
    def load():
        raise AssertionError("the call loaded libemap.so")
    monkeypatch.setattr(_lib, "load", load)


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"the library was called: {name}")


def _bare_map():
    """an ElevationMap with no handle: any library call fails the test"""
    em = object.__new__(ElevationMap)
    em._L, em._h, em.map_lock = _NoLibrary(), None, threading.Lock()
    em.resolution, em.cell_n = 0.1, 12
    em._region_caps, em._values_cap = (256, 1024, 16384), 4096
    return em


N, ROWS, COLS = 4, 6, 7
GRID = {"layers": {"elevation": np.zeros((ROWS, COLS), np.float32)}, "centre": np.zeros(2), "resolution": 0.1}
FIELD = {"volume": np.zeros((3, ROWS, COLS), np.float32), "n_z": 3, "rows": ROWS, "cols": COLS,
         "position": np.zeros(2), "resolution": 0.1, "z_min": 0.0}
TABLES = {"regions": np.zeros((0, 17)), "polygons": np.zeros((0, 5), np.int32), "vertices": np.zeros((0, 2))}
Z_RANGE = (0.0, 0.4)
N_Z = int(math.floor((Z_RANGE[1] - Z_RANGE[0]) / 0.1)) + 1


def _xy(n=N, k=2):
    return np.arange(n * k, dtype=np.float64).reshape(n, k) * 0.01


# method, the call with a given `out`, and the (shape, dtype) of each array of a valid `out` (a bare array: key None)
_DICT_OUT = {
    "max_value_between_locations": (lambda em, out: em.max_value_between_locations(GRID, "elevation", _xy(), _xy(),
                                                                                   out=out),
                                    {"index": ((N, 3), np.int32), "value": ((N, 3), np.float64)}),
    "grid_derivatives": (lambda em, out: em.grid_derivatives(GRID, "elevation", _xy(), True, out=out),
                         {"index": ((N, 3), np.int32), "value": ((N, 5), np.float64)}),
    "values_at_grid": (lambda em, out: em.values_at(_xy(), ["elevation"], grid=GRID, out=out),
                       {"values": ((1, N), np.float32), "status": ((N,), np.int32)}),
    "values_at_live_map": (lambda em, out: em.values_at(_xy(), ["elevation", "variance"], out=out),
                           {"values": ((2, N), np.float32), "status": ((N,), np.int32)}),
    "project_to_planar_regions": (lambda em, out: em.project_to_planar_regions({"tables": TABLES}, _xy(k=3), 0.0, 4,
                                                                               out=out),
                                  {"index": ((N, 3), np.int32), "point": ((N, 6), np.float64),
                                   "convex": ((N, 4, 5), np.float64)}),
    "signed_distance_field": (lambda em, out: em.signed_distance_field(GRID, "elevation", z_range=Z_RANGE, out=out),
                              {None: ((N_Z, ROWS, COLS), np.float32)}),
    "sdf_values": (lambda em, out: em.sdf_values(FIELD, _xy(k=3), out=out), {None: ((N, 4), np.float64)}),
    "inpaint_image": (lambda em, out: em.inpaint_image(np.zeros((ROWS, COLS), np.uint8), np.zeros((ROWS, COLS), np.uint8),
                                                       out=out),
                      {None: ((ROWS, COLS), np.uint8)}),
    "nonlinear_interpolation": (lambda em, out: em.nonlinear_interpolation(GRID, "elevation", out=out),
                                {None: ((ROWS, COLS), np.float32)}),
}


def _out(spec, bad_key=None, bad=None):
    arrays = {}
    for k, (shape, dtype) in spec.items():
        a = np.zeros(shape, dtype)
        if k == bad_key:
            if bad == "dtype":
                a = np.zeros(shape, np.float32 if dtype != np.float32 else np.float64)
            elif bad == "shape":
                a = np.zeros((shape[0] + 1,) + shape[1:], dtype)
            else:
                a = np.zeros(shape[:-1] + (2 * shape[-1],), dtype)[..., ::2]
                assert not a.flags.c_contiguous
        arrays[k] = a
    return arrays[None] if None in arrays else arrays


@pytest.mark.parametrize("bad", ["dtype", "shape", "non-contiguous"])
@pytest.mark.parametrize("method", sorted(_DICT_OUT))
def test_a_malformed_out_is_rejected_before_the_library(method, bad):
    call, spec = _DICT_OUT[method]
    for key in spec:
        with pytest.raises(TypeError, match="must be a contiguous"):
            call(_bare_map(), _out(spec, key, bad))


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_projection_rejects_a_point_out_of_the_wrong_width(dtype):
    """a float32 out["point"] of the right shape would be written with float64 rows, twice its size"""
    out = _out(_DICT_OUT["project_to_planar_regions"][1])
    out["point"] = np.zeros((N, 6), dtype)
    with pytest.raises(TypeError, match=r"out\['point'\] must be a contiguous float64"):
        _DICT_OUT["project_to_planar_regions"][0](_bare_map(), out)


_FLAT_OUT = {
    "get_submaps": lambda em, out: em.get_submaps([((0.0, 0.0), (0.5, 0.5))], ["elevation"], out),
    "get_transformed_submaps": lambda em, out: em.get_transformed_submaps([((0.0, 0.0), (0.5, 0.5), np.eye(4))],
                                                                          ["elevation"], out),
    "segment_planes": lambda em, out: em.segment_planes((0.0, 0.0), (0.5, 0.5), out=out),
    "extract_planar_regions": lambda em, out: em.extract_planar_regions((0.0, 0.0), (0.5, 0.5), out=out),
    "planar_terrain": lambda em, out: em.planar_terrain((0.0, 0.0), (0.5, 0.5), out=out),
    "plane_decomposition": lambda em, out: em.plane_decomposition(GRID, "elevation", out=out),
}


@pytest.mark.parametrize("bad", ["dtype", "non-contiguous"])
@pytest.mark.parametrize("method", sorted(_FLAT_OUT))
def test_a_malformed_flat_out_is_rejected_before_the_library(method, bad):
    """The window and plane calls take one flat float32 `out` of at least their layers' floats; its size is checked
    by the library, which alone knows the window, so only the dtype and the layout are checked here."""
    out = np.zeros(64, np.float64) if bad == "dtype" else np.zeros(128, np.float32)[::2]
    with pytest.raises(TypeError, match="a host `out` must be a C-contiguous float32 NumPy array"):
        _FLAT_OUT[method](_bare_map(), out)


@pytest.mark.parametrize("table,shape", [("regions", (2, 16)), ("polygons", (2, 6)), ("vertices", (4,))])
def test_projection_rejects_tables_of_the_wrong_width(table, shape):
    tables = dict(TABLES, **{table: np.zeros(shape)})
    with pytest.raises(TypeError, match=table[:-1] + " table must have"):
        _bare_map().project_to_planar_regions({"tables": tables}, _xy(k=3))


def test_a_host_table_is_converted_to_its_dtype():
    em = _bare_map()
    tables = {"regions": np.zeros((1, 17), np.float32), "polygons": np.zeros((1, 5)), "vertices": np.zeros((1, 2))}
    with pytest.raises(AssertionError, match="emap_project_to_planar_regions"):
        em.project_to_planar_regions({"tables": tables}, _xy(k=3))


def test_grid_takes_a_transformed_submap_dict():
    """get_transformed_submap(s) returns "frame_centre" and no "centre" or "resolution"."""
    em = _bare_map()
    layer = np.arange(ROWS * COLS, dtype=np.float64).reshape(COLS, ROWS).T            # F-ordered float64
    sub = {"layers": {"elevation": layer}, "size": (ROWS, COLS), "frame_centre": np.array([1.25, -0.5]),
           "length": np.array([0.6, 0.7]), "success": True}
    g = em._grid(sub, "elevation")
    assert (g.rows, g.cols, list(g.position), g.resolution) == (ROWS, COLS, [1.25, -0.5], em.resolution)
    assert g._keep.dtype == np.float32 and g._keep.flags.c_contiguous and g.data == g._keep.ctypes.data
    assert np.array_equal(g._keep, layer.astype(np.float32))
    g = em._grid(dict(sub, centre=(3.0, 4.0), resolution=0.25), "elevation")
    assert (list(g.position), g.resolution) == ([3.0, 4.0], 0.25)


def test_queries_of_numpy_parts():
    a, b = _xy(5).astype(np.float32), np.asfortranarray(_xy(5) + 1.0)
    q = _queries((a, b), 4)
    assert q.dtype == np.float64 and q.shape == (5, 4) and q.flags.c_contiguous
    assert np.array_equal(q, np.hstack([a.astype(np.float64), b]))
    q = _queries(([[0.0, 1.0, 2.0], [3.0, 4.0, 5.0]],), 3)
    assert q.shape == (2, 3) and q.dtype == np.float64
    assert _queries((np.zeros(6),), 2).shape == (3, 2)


def test_unknown_layers_are_rejected_before_any_plugin_runs():
    em = _bare_map()
    em.semantic_map = types.SimpleNamespace(layer_names=[])
    em.plugin_manager = types.SimpleNamespace(layer_names=["plugin_layer"])
    data = np.zeros((2, em.cell_n - 2, em.cell_n - 2), np.float32)
    with pytest.raises(KeyError, match="no_such_layer is not in the map"):
        em.get_maps_with_names_ref(["plugin_layer", "no_such_layer"], data)
    with pytest.raises(KeyError, match="no_such_layer is not in the map"):
        em.values_at(_xy(), ["plugin_layer", "no_such_layer"])
    with pytest.raises(KeyError, match="no_such_layer is not in the map"):
        em.get_submaps([((0.0, 0.0), (0.5, 0.5))], ["plugin_layer", "no_such_layer"])
    em.get_map_with_name_ref("no_such_layer", data[0])              # prints and returns, as EM.py does
