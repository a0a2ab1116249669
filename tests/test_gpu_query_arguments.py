"""GPU: the argument checks the query calls share, on device arguments, and the grids they read.  A device `out` or
region table of the wrong dtype, layout or width is rejected with TypeError before any launch (the library would read or
write past its end), and the lookups, the distance field and the interpolation take the dict get_transformed_submap
returns ("frame_centre", no "centre") with the same bytes as the same dict with "centre" copied in."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import plane_scenes as S                                          # noqa: E402

pytestmark = pytest.mark.gpu

_MAP = []


def _map():
    """a map whose exported elevation is the holes terrain (NaN holes included) and a yawed transformed window of it"""
    if not _MAP:
        from elevation_mapping_cupy_b200.parameter import core_parameter
        from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
        img = S.terrain_image(np.load(S.GOLDEN)["grey__holes"], S.TERRAINS["holes"][1], seed=5)
        em = ElevationMap(core_parameter(img.shape[0] + 2))
        S.set_image(em, img)
        yaw = 0.3
        T = np.eye(4)
        T[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
        T[:3, 3] = [0.2, -0.1, 0.05]
        sub = em.get_transformed_submap((0.1, -0.05), (1.5, 1.5), ["elevation"], T)
        assert sub["success"] and "centre" not in sub
        _MAP.append((em, sub))
    return _MAP[0]


def _tables(**bad):
    import torch
    t = {"regions": torch.zeros((2, 17), dtype=torch.float64, device="cuda"),
         "polygons": torch.zeros((2, 5), dtype=torch.int32, device="cuda"),
         "vertices": torch.zeros((4, 2), dtype=torch.float64, device="cuda")}
    t.update(bad)
    return {"tables": t}


def _bad_table(case):
    import torch
    z = lambda shape, dtype: torch.zeros(shape, dtype=getattr(torch, dtype), device="cuda")  # noqa: E731
    return {"float32 regions": lambda: _tables(regions=z((2, 17), "float32")),
            "int64 polygons": lambda: _tables(polygons=z((2, 5), "int64")),
            "float32 vertices": lambda: _tables(vertices=z((4, 2), "float32")),
            "non-contiguous regions": lambda: _tables(regions=z((2, 34), "float64")[:, ::2]),
            "non-contiguous vertices": lambda: _tables(vertices=z((2, 4), "float64").T),
            "transposed polygons": lambda: _tables(polygons=z((5, 2), "int32").T),
            "16-column regions": lambda: _tables(regions=z((2, 16), "float64")),
            "host polygons": lambda: _tables(polygons=np.zeros((2, 5), np.int32))}[case]()


@pytest.mark.parametrize("case", ["float32 regions", "int64 polygons", "float32 vertices", "non-contiguous regions",
                                  "non-contiguous vertices", "transposed polygons", "16-column regions",
                                  "host polygons"])
def test_malformed_device_tables_are_rejected_before_any_launch(case):
    import torch
    em, _ = _map()
    terrain = _bad_table(case)
    q = torch.zeros((8, 3), dtype=torch.float64, device="cuda")
    n0 = em.launch_count()
    with pytest.raises(TypeError):
        em.project_to_planar_regions(terrain, q, 0.0, 4)
    assert em.launch_count() == n0


@pytest.mark.parametrize("key,dtype", [("point", "float32"), ("convex", "float32"), ("index", "int64")])
def test_a_device_out_of_the_wrong_dtype_is_rejected_before_any_launch(key, dtype):
    import torch
    em, _ = _map()
    n = 8
    out = {"index": torch.zeros((n, 3), dtype=torch.int32, device="cuda"),
           "point": torch.zeros((n, 6), dtype=torch.float64, device="cuda"),
           "convex": torch.zeros((n, 4, 5), dtype=torch.float64, device="cuda")}
    out[key] = torch.zeros(out[key].shape, dtype=getattr(torch, dtype), device="cuda")
    n0 = em.launch_count()
    with pytest.raises(TypeError, match=r"out\[%r\]" % key):
        em.project_to_planar_regions(_tables(), torch.zeros((n, 3), dtype=torch.float64, device="cuda"), 0.0, 4, out=out)
    assert em.launch_count() == n0
    assert all(not a.any() for a in out.values())


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _bytes(x):
    return _host(x).tobytes()


@pytest.mark.parametrize("side", ["host", "device"])
def test_transformed_submap_grids(side):
    import torch
    em, sub = _map()
    if side == "device":
        sub = dict(sub, layers={k: torch.as_tensor(v, device="cuda") for k, v in sub["layers"].items()})
    by_hand = dict(sub, centre=sub["frame_centre"])
    rng = np.random.default_rng(3)
    pts = sub["frame_centre"] + rng.uniform(-0.9, 0.9, (500, 2))
    starts, ends = pts[:250], pts[250:]
    for method in ("nearest", "linear", "cubic"):
        a, b = (em.values_at(pts, ["elevation"], method, grid=g) for g in (sub, by_hand))
        assert _bytes(a["values"]["elevation"]) == _bytes(b["values"]["elevation"])
        assert _bytes(a["status"]) == _bytes(b["status"]) and (_host(a["status"]) > 0).any()
    a, b = (em.max_value_between_locations(g, "elevation", starts, ends) for g in (sub, by_hand))
    assert all(_bytes(a[k]) == _bytes(b[k]) for k in a) and _host(a["valid"]).any()
    a, b = (em.signed_distance_field(g, "elevation") for g in (sub, by_hand))
    assert _bytes(a["volume"]) == _bytes(b["volume"]) and a["position"].tolist() == b["position"].tolist()
    assert a["position"].tolist() == [float(v) for v in sub["frame_centre"]]
    a, b = (em.nonlinear_interpolation(g, "elevation") for g in (sub, by_hand))
    assert _bytes(a) == _bytes(b)
    assert not np.isnan(np.frombuffer(_bytes(a), np.float32)).any()
