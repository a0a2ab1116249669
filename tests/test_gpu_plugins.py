"""GPU parity of the plugin stencils and of the drop-in API surface (reference test_elevation_mapping.py /
test_plugins.py shapes: 202^2 map, randn layers)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _mk(param):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    return ElevationMap(param)


def _random_state(W, seed, valid_frac=0.5):
    rng = np.random.default_rng(seed)
    m = np.zeros((7, W, W), np.float32)
    m[0] = rng.standard_normal((W, W)).astype(np.float32)
    m[1] = 0.05
    m[2] = (rng.random((W, W)) < valid_frac).astype(np.float32)
    m[3] = 1.0
    m[5] = m[0]
    return m


@pytest.mark.parametrize("k,iters,valid_frac", [(1, 30, 0.5), (2, 3, 0.05), (1, 5, 0.001)])
def test_min_filter_matches_oracle(oracle_mod, k, iters, valid_frac):
    import torch
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.plugins.min_filter import MinFilter
    p = core_parameter(202)
    em = _mk(p)
    st = _random_state(202, 5, valid_frac)
    em.set_state(st)
    plug = MinFilter(cell_n=202, dilation_size=k, iteration_n=iters, engine=em)
    out = plug(em.elevation_map, em.layer_names, None, []).cpu().numpy()
    ref, _ = oracle_mod.min_filter(202, k, iters, st[0], st[2])
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    assert np.array_equal(np.nan_to_num(out), np.nan_to_num(ref))


# (k, iteration_n, valid fraction, exits early): at half the cells valid every cell is filled after 2 of 30 passes; at
# 0.1 % valid, 5 passes never fill the map
@pytest.mark.parametrize("k,iters,valid_frac,early", [(1, 30, 0.5, True), (2, 3, 0.05, False), (1, 5, 0.001, False)])
def test_fill_filters_iterations_run_match_oracle(oracle_mod, k, iters, valid_frac, early):
    """iterations_run of emap_min_filter / emap_max_filter: the passes up to the first one that leaves no cell unfilled"""
    import ctypes as C
    import torch
    from elevation_mapping_cupy_b200.parameter import core_parameter
    em = _mk(core_parameter(202))
    st = _random_state(202, 5, valid_frac)
    h = torch.from_numpy(st[0]).cuda(); m = torch.from_numpy(st[2]).cuda(); o = torch.empty_like(h)
    em._after_framework()
    for entry, oracle_filter in (("emap_min_filter", oracle_mod.min_filter), ("emap_max_filter", oracle_mod.max_filter)):
        n = C.c_int32(-1)
        em._check(getattr(em._L, entry)(em._h, h.data_ptr(), m.data_ptr(), o.data_ptr(), k, iters, C.byref(n)))
        ref_out, ref_n = oracle_filter(202, k, iters, st[0], st[2])
        assert (ref_n < iters) == early, (entry, ref_n)
        assert n.value == ref_n, entry
        assert np.array_equal(np.nan_to_num(o.cpu().numpy(), nan=-7), np.nan_to_num(ref_out, nan=-7)), entry
    em._before_framework()


def test_smooth_filter_matches_oracle_and_scipy(oracle_mod):
    from scipy import ndimage
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.plugins.smooth_filter import SmoothFilter
    p = core_parameter(202)
    em = _mk(p)
    st = _random_state(202, 7)
    em.set_state(st)
    plug = SmoothFilter(cell_n=202, input_layer_name="elevation", engine=em)
    out = plug(em.elevation_map, em.layer_names, None, []).cpu().numpy()
    ref = oracle_mod.smooth(202, st[0])
    assert np.array_equal(out, ref)
    sp = ndimage.uniform_filter(ndimage.uniform_filter(st[0], size=3), size=3)   # smooth_filter.py:57-58 on the host
    assert np.abs(out - sp).max() < 1e-6


def test_update_normal_of_a_plane_matches_oracle(oracle_mod):
    """update_normal(plane) (EM.py:564-577) on an arbitrary device plane: the normals of that plane over the valid cells"""
    import torch
    from elevation_mapping_cupy_b200.parameter import core_parameter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    st = _random_state(W, 9)
    em.set_state(st)
    plane = np.random.default_rng(4).standard_normal((W, W)).astype(np.float32)
    em.update_normal(torch.from_numpy(plane).cuda())
    _, normal = em.get_state()
    assert np.array_equal(normal, oracle_mod.normal(W, p.resolution, plane, st[2]))


def test_reference_api_surface_smoke():
    """The call sequence of the reference's own test (test_elevation_mapping.py:46-118), minus the
    out-of-scope semantic / polygon / initialiser calls."""
    import torch
    from elevation_mapping_cupy_b200.parameter import Parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = Parameter(); p.update()
    em = _mk(p)
    assert len(em.layer_names) == em.elevation_map.shape[0]
    pts, R, t = wl.reference_test_cloud(0, n_ch=5)
    em.input_pointcloud(torch.from_numpy(pts).cuda(), ["x", "y", "z", "a", "b"], R, t, 0, 0)
    em.input(pts.astype(np.float64), ["x", "y", "z", "a", "b"], R, t, 0, 0)
    em.update_normal(em.elevation_map[0].contiguous())
    for i in range(20):
        em.move_to(np.array([i * 0.01, i * 0.02, i * 0.01]), np.random.rand(3, 3))
    data = np.zeros((em.cell_n - 2, em.cell_n - 2), dtype=np.float32)
    for layer in ["elevation", "variance", "traversability", "min_filter", "smooth"]:
        em.get_map_with_name_ref(layer, data)
        assert em.exists_layer(layer)
    pos = np.random.rand(1, 3)
    em.get_position(pos)
    em.clear()
    em.move(np.random.rand(3))
    assert not em.exists_layer("nonexistent")
    with pytest.raises(KeyError):
        em._ptr("nonexistent")


def test_move_and_shift_match_oracle(oracle_mod):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(202)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p)
    st = _random_state(202, 11)
    em.set_state(st); om.elevation_map = st.copy()
    rng = np.random.default_rng(3)
    for i in range(12):
        pos = rng.uniform(-0.6, 0.6, 3) * (i + 1) / 4
        if i % 3 == 2:
            d = rng.uniform(-0.2, 0.2, 3)
            em.move(d); om.move(d)
        else:
            em.move_to(pos, np.eye(3)); om.move_to(pos, np.eye(3))
        state, _ = em.get_state()
        assert np.array_equal(state, om.elevation_map), f"step {i}"
        assert np.array_equal(em.center, om.center)
    em.clear(); om.clear()
    state, _ = em.get_state()
    assert np.array_equal(state, om.elevation_map)


def test_star_plugins_match_oracle(oracle_mod):
    """max_filter, erosion (vs the reference's literal cv2 code), robot_centric_elevation, max_layer_filter"""
    import torch
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.plugins.max_filter import MaxFilter
    from elevation_mapping_cupy_b200.plugins.erosion import Erosion
    from elevation_mapping_cupy_b200.plugins.robot_centric_elevation import RobotCentricElevation
    from elevation_mapping_cupy_b200.plugins.max_layer_filter import MaxLayerFilter
    W = 202
    p = core_parameter(W)
    em = _mk(p)
    st = _random_state(W, 21, 0.3)
    rng = np.random.default_rng(2)
    st[3] = rng.random((W, W)).astype(np.float32)
    em.set_state(st)
    names = em.layer_names
    # max_filter
    out = MaxFilter(cell_n=W, dilation_size=1, iteration_n=6, engine=em)(em.elevation_map, names, None, []).cpu().numpy()
    ref, _ = oracle_mod.max_filter(W, 1, 6, st[0], st[2])
    assert np.array_equal(np.isnan(out), np.isnan(ref)) and np.array_equal(np.nan_to_num(out), np.nan_to_num(ref))
    # erosion: default YAML of the reference (kernel 3, 1 iteration, reverse) and a multi-iteration even kernel
    for ks, it, rev in ((3, 1, True), (3, 3, False), (4, 2, False), (5, 1, True)):
        out = Erosion(input_layer_name="traversability", kernel_size=ks, iterations=it, reverse=rev, engine=em)(
            em.elevation_map, names, None, [], None, []).cpu().numpy()
        ref = oracle_mod.erosion_cv2(st[3], ks, it, rev)
        assert np.array_equal(out, ref.astype(np.float32)), (ks, it, rev, np.abs(out - ref).max())
    # robot_centric_elevation
    R = np.array([[0.9, 0.1, -0.2], [0.0, 1.0, 0.1], [0.15, -0.12, 0.97]], np.float32)
    for thr in (True, False):
        out = RobotCentricElevation(cell_n=W, resolution=0.04, threshold=1.1, use_threshold=thr, engine=em)(
            em.elevation_map, names, None, [], None, [], R).cpu().numpy()
        ref = oracle_mod.robot_centric(W, 0.04, 1.1, thr, st[0], st[2], R)
        assert np.array_equal(out, ref), thr
    # max_layer_filter (element-wise algebra)
    plug = MaxLayerFilter(cell_n=W, layers=["traversability", "variance"], reverse=[True, False], min_or_max="max",
                          thresholds=[False, 0.04], scales=[2.0, 1.0], default_value=0.5)
    out = plug(em.elevation_map, names, None, [], None, []).cpu().numpy()
    a = np.where(st[3] == 0.0, np.float32(0.5), st[3]); a = (np.float32(1.0) - a) * np.float32(2.0)
    b = np.where(st[1] == 0.0, np.float32(0.5), st[1]); b = np.where(b > np.float32(0.04), np.float32(1), np.float32(0))
    assert np.array_equal(out, np.maximum(a, b).astype(np.float32))


def test_default_plugin_yaml_layers_export():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(202)
    em = _mk(p)
    pts, R, t = wl.lidar_cloud(0, 0, n_rings=32, n_az=625, max_range=8.0)
    em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    data = np.zeros((200, 200), np.float32)
    for name in em.plugin_manager.layer_names:
        assert em.exists_layer(name)
        em.get_map_with_name_ref(name, data)
        assert np.isfinite(data).any(), name
    assert "erosion" in em.plugin_manager.layer_names


def _inpaint_stats(em):
    import ctypes as C
    r, mj, nc = C.c_int32(), C.c_int32(), C.c_int32()
    em._check(em._L.emap_inpaint_stats(em._h, C.byref(r), C.byref(mj), C.byref(nc)))
    return r.value, mj.value, nc.value


def test_inpainting_reference_test_shape_bit_identical_to_cv2(oracle_mod):
    """plugins/inpainting.py:53-63 on the 202^2 randn state of the reference's test_plugins.py: the device fill must be
    BIT-identical to cv2.inpaint (the reference's CPU call) -- stricter than one 8-bit quantisation step."""
    pytest.importorskip("cv2")
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.plugins.inpainting import Inpainting
    p = core_parameter(202)
    em = _mk(p)
    for seed, valid_frac in ((11, 0.31), (12, 0.7), (13, 0.02)):
        st = _random_state(202, seed, valid_frac)
        em.set_state(st)
        plug = Inpainting(cell_n=202, method="telea", engine=em)
        out = plug(em.elevation_map, em.layer_names, None, []).cpu().numpy()
        ref = oracle_mod.inpaint_cv2(st[0], st[2]).astype(np.float32)
        rounds, max_j, nc = _inpaint_stats(em)
        assert nc == 0, (rounds, max_j)
        assert np.array_equal(out, ref), (seed, int((out != ref).sum()), float(np.abs(out - ref).max()), rounds, max_j)


def test_inpainting_no_valid_cell_returns_layer_and_ns_raises():
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.plugins.inpainting import Inpainting
    p = core_parameter(130)
    em = _mk(p)
    st = _random_state(130, 3, 0.0)
    em.set_state(st)
    out = Inpainting(cell_n=130, engine=em)(em.elevation_map, em.layer_names, None, []).cpu().numpy()
    assert np.array_equal(out, st[0])                         # inpainting.py:62-63
    with pytest.raises(NotImplementedError):
        Inpainting(cell_n=130, method="ns", engine=em)(em.elevation_map, em.layer_names, None, [])


def test_inpainting_config_d_map_bit_identical_to_cv2(oracle_mod):
    """BASELINE config D: 2048^2 map after a dense depth-camera frame (1.5 % of the cells valid, one hole ~1500 cells deep
    -> ~2000 fast-marching rounds); the exported layer through the plugin manager, against cv2 on the host."""
    pytest.importorskip("cv2")
    import time
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(2048)
    em = _mk(p)
    pts, R, t = wl.depth_camera_cloud(3, 0)
    em.move_to(t, R)
    em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.0, 0.0)
    st, _ = em.get_state()
    assert 0.001 < (st[2] > 0.5).mean() < 0.2
    t0 = time.perf_counter()
    layer = em.get_layer("inpaint").cpu().numpy()
    dt_dev = time.perf_counter() - t0
    t0 = time.perf_counter()
    ref = oracle_mod.inpaint_cv2(st[0], st[2]).astype(np.float32)
    dt_cv = time.perf_counter() - t0
    rounds, max_j, nc = _inpaint_stats(em)
    print(f"config D inpaint: device {dt_dev * 1e3:.1f} ms (first call incl. allocation), cv2 on the host {dt_cv * 1e3:.1f} ms, "
          f"{rounds} rounds, longest fixed point {max_j}")
    import json, os
    out_dir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    # second call: allocation done, map unchanged
    em.plugin_manager.layers = None
    t0 = time.perf_counter(); em.get_layer("inpaint"); em.synchronize(); dt_dev2 = time.perf_counter() - t0
    if os.path.isdir(out_dir):
        json.dump({"workload": "config D map (2048^2, 1M-pt depth frame), inpainting plugin", "device_ms_first": dt_dev * 1e3,
                   "device_ms": dt_dev2 * 1e3, "cv2_host_ms": dt_cv * 1e3, "rounds": rounds, "max_fixed_point_iterations": max_j,
                   "valid_fraction": float((st[2] > 0.5).mean()), "mismatching_cells": int((layer != ref).sum())},
                  open(os.path.join(out_dir, "inpaint_config_d.json"), "w"))
    assert nc == 0
    bad = int((layer != ref).sum())
    assert bad == 0, (bad, float(np.abs(layer - ref).max()), rounds, max_j)
