"""GPU parity: the CUDA engine (through the C ABI / ElevationMap) against the CPU oracle on the same
seeded inputs.  Bar: bit-identical cell indices; height / variance (and every other state plane) bit-identical
to the canonical-serialisation oracle, which is stricter than the 1e-4 of BASELINE.json; traversability 2e-6."""
import numpy as np
import pytest

from helpers import compare_state

pytestmark = pytest.mark.gpu


def _mk(param):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    return ElevationMap(param)


def test_point_index_bit_exact_reference_test_shape(oracle_mod):
    """Reference test workload (test_elevation_mapping.py:51-61): rand(100000,3) cloud, rand(3,3) R, rand(3) t."""
    from elevation_mapping_cupy_b200.parameter import Parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = Parameter(); p.update()
    em = _mk(p)
    for seed in range(3):
        pts, R, t = wl.reference_test_cloud(seed)
        pts = (pts * np.float32(8.0) - np.float32(4.0)).astype(np.float32) if seed else pts
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0, 0)
        idx, valid, inside = em.get_point_record(len(pts))
        t_rel = (t - em.center).astype(np.float32)
        oi, ov, oin, _ = oracle_mod.point_index(p, pts, R, t_rel)
        assert np.array_equal(idx, oi)
        assert np.array_equal(valid, ov)
        assert np.array_equal(inside, oin)


@pytest.mark.parametrize("cell_n,frames", [(256, 6), (202, 4), (131, 3)])
def test_frames_match_oracle(oracle_mod, cell_n, frames):
    """Config A style: several frames with move_to / update_variance / update_time in between."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(cell_n)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    for f in range(frames):
        if f % 2 == 0:
            pts, R, t = wl.uniform_cloud(0, f, n=10000, half_extent=min(4.9, 0.02 * cell_n - 0.3))
        else:
            pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=625, max_range=8.0)
        for m in (em, om):
            m.move_to(t, R)
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"frame {f}")
        st = em.get_frame_stats()
        assert st.error_cnt == om.stats.error_cnt
        assert st.drift_applied == om.stats.drift_applied
        assert np.float32(st.mean_error) == np.float32(om.mean_error) or not om.stats.drift_evaluated
        for m in (em, om):
            m.update_variance(); m.update_time()
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"frame {f} after ticks")


def test_nan_rows_and_f64_input(oracle_mod):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(256)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    pts, R, t = wl.uniform_cloud(0, 3, n=5000)
    pts[::7] = np.nan
    pts64 = np.concatenate([pts.astype(np.float64), np.zeros((len(pts), 2))], 1)   # extra channels, float64 rows
    em.input_pointcloud(pts64, ["x", "y", "z", "a", "b"], R, t, 0.0, 0.0)
    om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.0, 0.0)
    state, normal = em.get_state()
    compare_state(state, normal, om, label="nan/f64")
    idx, valid, inside = em.get_point_record(len(pts))
    assert (idx[::7] == -1).all() and (valid[::7] == 0).all()


def test_export_layers_match_oracle(oracle_mod):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    for only_above in (False, True):
        p = core_parameter(202, use_only_above_for_upper_bound=only_above)
        em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
        for f in range(3):
            pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=625, max_range=8.0)
            for m in (em, om):
                m.move_to(t + np.float32(0.3), R)
                m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        data = np.zeros((p.cell_n - 2, p.cell_n - 2), np.float32)
        for name in ["elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
                     "normal_x", "normal_y", "normal_z"]:
            em.get_map_with_name_ref(name, data)
            ref = om.export_layer(name)
            tol = 2e-6 if name == "traversability" else 0.0
            assert np.array_equal(np.isnan(data), np.isnan(ref)), name
            assert np.nanmax(np.abs(data - ref), initial=0.0) <= tol, name


def test_multi_sensor_frame_matches_oracle(oracle_mod):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(256)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    for f in range(3):
        clouds, Rs, ts = [], [], []
        for s in range(3):
            pts, R, t = wl.lidar_cloud(2, f, n_rings=16, n_az=500, max_range=6.0, sensor=s, n_sensors=3)
            clouds.append(pts); Rs.append(R); ts.append(t)
        em.input_sensors(clouds, Rs, ts, 0.02, 0.02)
        om.input_sensors(clouds, Rs, ts, 0.02, 0.02)
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"multi-sensor frame {f}")


def test_config_b_single_frame(oracle_mod):
    """BASELINE config B at full size: 1024^2, 200k-point LiDAR frame, raycast + overlap clear on."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(1024)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    for f in range(2):
        pts, R, t = wl.lidar_cloud(1, f)
        for m in (em, om):
            m.move_to(t, R)
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
            m.update_time()
    state, normal = em.get_state()
    compare_state(state, normal, om, label="config B")


def test_engine_matches_committed_golden(oracle_mod):
    """tests/golden/frames_core130.npz: outputs of the REFERENCE'S OWN kernel source (order-independent cells)
    and of the oracle, generated in the build container by tests/golden/make_golden.py."""
    import os
    from elevation_mapping_cupy_b200.parameter import core_parameter, Parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    g = np.load(os.path.join(gold, "frames_core130.npz"))
    p = core_parameter(130)
    em = _mk(p)
    for f in range(4):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        state, normal = em.get_state()
        for li in (0, 1, 2, 4, 5, 6):
            assert np.array_equal(state[li], g[f"oracle_state_{f}"][li]), (f, li)
            d = np.abs(state[li] - g[f"ref_state_{f}"][li])
            assert d[~g[f"racy_{f}"]].max() <= 1e-6, (f, li)      # vs the reference source: 1e-6 << 1e-4 (BASELINE)
        assert np.abs(state[3] - g[f"oracle_state_{f}"][3]).max() <= 2e-6
        assert np.array_equal(normal, g[f"oracle_normal_{f}"])
        idx, _, _ = em.get_point_record(len(pts))
        assert np.array_equal(idx, g[f"ref_point_idx_{f}"])       # bit-identical cell indices vs the reference
        em.update_variance(); em.update_time()
    for seed in (0, 1):
        gi = np.load(os.path.join(gold, f"index_default202_seed{seed}.npz"))
        pd = Parameter(); pd.update()
        e2 = _mk(pd)
        pts, R, t = wl.reference_test_cloud(seed, n=20000)
        if seed % 2:
            pts = (pts * np.float32(9.0) - np.float32(4.5)).astype(np.float32)
        e2.input_pointcloud(pts, ["x", "y", "z"], R, t, 0, 0)
        idx, valid, inside = e2.get_point_record(len(pts))
        assert np.array_equal(idx, gi["idx"]) and np.array_equal(valid, gi["valid"]) and np.array_equal(inside, gi["inside"])


@pytest.mark.parametrize("cell_n,dil", [(130, 3), (202, 2), (130, 1), (202, 5)])
def test_post_chain_on_random_state(oracle_mod, cell_n, dil):
    """dilation (incl. the flat-index row wrap of CK.py:403-407) + CNN + normals on a random state, driven by
    an empty cloud; border columns are populated on purpose."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(cell_n, dilation_size=dil, enable_visibility_cleanup=(dil != 2))
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    rng = np.random.default_rng(cell_n + dil)
    W = cell_n
    st = np.zeros((7, W, W), np.float32)
    st[0] = rng.standard_normal((W, W)); st[1] = 0.05
    st[2] = (rng.random((W, W)) < 0.2); st[2][:, :5] = rng.random((W, 5)) < 0.7; st[2][:, -5:] = rng.random((W, 5)) < 0.7
    st[3] = 1.0; st[4] = 1.0
    st[5] = rng.standard_normal((W, W)); st[6] = (rng.random((W, W)) < 0.1) * (st[2] < 0.5)
    st[0] *= st[2]
    em.set_state(st); om.elevation_map = st.copy()
    empty = np.zeros((0, 3), np.float32)
    R = np.eye(3, dtype=np.float32); t = np.array([0, 0, 1.0], np.float32)
    em.input_pointcloud(empty, ["x", "y", "z"], R, t, 0.0, 0.0)
    om.input_pointcloud(empty, ["x", "y", "z"], R, t, 0.0, 0.0)
    state, normal = em.get_state()
    compare_state(state, normal, om, label=f"post {cell_n}/{dil}")
    ti = em.traversability_input.cpu().numpy()
    assert np.array_equal(ti, om.traversability_input)


def test_config_d_depth_camera_2048_with_plugin_chain(oracle_mod):
    """BASELINE config D at full size: 2048^2 grid, 1M-point depth-camera cloud with 5 % NaN pixels, then the
    min_filter -> smooth plugin chain on the result."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(2048)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    pts, R, t = wl.depth_camera_cloud(3, 0)
    assert len(pts) == 1000000 and np.isnan(pts).any()
    for m in (em, om):
        m.move_to(t, R)
        m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    state, normal = em.get_state()
    compare_state(state, normal, om, label="config D")
    idx, valid, inside = em.get_point_record(len(pts))
    oi, ov, oin = om.last_point_record
    nan = np.isnan(pts).any(1)
    assert np.array_equal(idx[~nan], oi[~nan]) and np.array_equal(valid, ov) and np.array_equal(inside, oin)
    data = np.zeros((p.cell_n - 2, p.cell_n - 2), np.float32)
    em.get_map_with_name_ref("min_filter", data)
    mf, _ = oracle_mod.min_filter(p.cell_n, 1, 30, om.elevation_map[0], om.elevation_map[2])
    ref = np.flip(np.flip((mf + om.center[2])[1:-1, 1:-1], 0), 1)
    assert np.array_equal(np.isnan(data), np.isnan(ref))
    assert np.array_equal(np.nan_to_num(data), np.nan_to_num(ref))
    em.get_map_with_name_ref("smooth", data)
    assert np.isfinite(data).any()


def test_config_e_independent_replicas(oracle_mod):
    """BASELINE config E in miniature: independent 512^2 maps, one handle (own stream) each, frames issued
    round-robin without synchronising in between; every replica must equal its own oracle."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(512)
    n_maps = 6
    ems = [_mk(p) for _ in range(n_maps)]
    clouds = [[wl.lidar_cloud(4, f, n_rings=32, n_az=3125, max_range=12.0, sensor=0, n_sensors=1) for f in range(2)]
              for _ in range(n_maps)]
    for m in range(n_maps):       # a different seed offset per map (SURVEY 8(d) E)
        clouds[m] = [wl.lidar_cloud(4, 10 * m + f, n_rings=32, n_az=3125, max_range=12.0) for f in range(2)]
    for f in range(2):
        for m in range(n_maps):
            pts, R, t = clouds[m][f]
            ems[m].move_to(t, R)
            ems[m].input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
            ems[m].update_time()
    for m in (0, n_maps - 1):
        om = oracle_mod.OracleElevationMap(p, nthreads=0)
        for f in range(2):
            pts, R, t = clouds[m][f]
            om.move_to(t, R); om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02); om.update_time()
        state, normal = ems[m].get_state()
        compare_state(state, normal, om, label=f"replica {m}")


def test_edge_case_clouds(oracle_mod):
    """empty / all-NaN / single-point / far-outside / non-finite clouds, and frames without time ticks"""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(130)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    R = np.eye(3, dtype=np.float32); t = np.array([0.1, -0.2, 1.0], np.float32)
    base, _, _ = wl.lidar_cloud(0, 1, n_rings=24, n_az=500, max_range=4.0)
    far = (np.random.default_rng(0).uniform(-400, 400, (3000, 3))).astype(np.float32)           # clamps to the border ring
    weird = base[:2000].copy()
    weird[::5, 0] = np.inf; weird[1::5, 1] = -np.inf; weird[2::5, 2] = 65520.0                   # beyond fp16 range
    cases = [np.zeros((0, 3), np.float32), np.full((100, 3), np.nan, np.float32), base[:1].copy(), base, far, weird,
             base[::3].copy(), base[::3].copy()]                                                  # the last two: no tick in between
    for k, pts in enumerate(cases):
        for m in (em, om):
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"edge case {k}")
        if len(pts):
            idx, valid, inside = em.get_point_record(len(pts))
            oi, ov, oin = om.last_point_record
            ok = ~np.isnan(pts).any(1)
            assert np.array_equal(idx[ok], oi[ok]) and np.array_equal(valid, ov) and np.array_equal(inside, oin), k
        if k < 6:
            for m in (em, om):
                m.update_variance(); m.update_time()


@pytest.mark.parametrize("dil", [0, 4])
def test_unusual_dilation_sizes(oracle_mod, dil):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(130, dilation_size=dil)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    for f in range(2):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        for m in (em, om):
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02); m.update_time()
    state, normal = em.get_state()
    compare_state(state, normal, om, label=f"dilation {dil}")


def test_device_f64_rows_and_torch_input(oracle_mod):
    import torch
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(130)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    pts, R, t = wl.lidar_cloud(0, 2, n_rings=24, n_az=500, max_range=4.0)
    wide = np.concatenate([pts.astype(np.float64), np.ones((len(pts), 4))], 1)
    em.input_pointcloud(torch.from_numpy(wide).cuda(), ["x", "y", "z", "r", "g", "b", "a"], torch.from_numpy(R), t, 0.02, 0.02)
    om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    state, normal = em.get_state()
    compare_state(state, normal, om, label="device f64 rows")


def test_drift_compensation_frames_match_oracle(oracle_mod):
    """the drift path (device-side decision, lazily applied plane shift) with parameters under which it fires"""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    kw = dict(traversability_inlier=0.0, drift_compensation_variance_inlier=10.0, min_height_drift_cnt=10)
    p = core_parameter(130, **kw)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    fired = 0
    for f in range(6):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        pts = pts.copy(); pts[:, 2] += np.float32(0.03 * (f % 2))
        for m in (em, om):
            m.move_to(t, R); m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"drift frame {f}")
        st = em.get_frame_stats()
        assert st.drift_applied == om.stats.drift_applied and st.error_cnt == om.stats.error_cnt
        if st.drift_applied:
            fired += 1
            assert np.float32(st.mean_error) == np.float32(om.stats.mean_error)
            assert np.float32(st.shift_applied) == np.float32(om.stats.shift_applied)
            assert np.float32(st.additive_mean_error) == np.float32(om.additive_mean_error)
        for m in (em, om):
            m.update_variance(); m.update_time()
    assert fired >= 3


@pytest.mark.parametrize("flags", [
    dict(enable_edge_sharpen=False),
    dict(enable_visibility_cleanup=False),
    dict(enable_overlap_clearance=False, enable_drift_compensation=False),
    dict(max_ray_length=2.0, cleanup_step=0.01, cleanup_cos_thresh=0.5, wall_num_thresh=3, dilation_size=2,
         min_valid_distance=0.3, mahalanobis_thresh=1.0),
])
def test_feature_toggles_match_oracle(oracle_mod, flags):
    """the same toggles / thresholds tests/test_oracle_cpu.py pins against the reference's kernel source"""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(130, **flags)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    for f in range(3):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        for m in (em, om):
            m.move_to(t, R); m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
            m.update_variance(); m.update_time()
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"{flags} frame {f}")


def test_batched_export_equals_layer_by_layer(oracle_mod):
    """emap_get_layers (one kernel, one D2H, one sync for N layers -- what the C++ bridge's get_grid_map asks for,
    elevation_mapping_wrapper.cpp:213-252) against the single-layer export and the oracle, plugin layers included."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(202)
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    for f in range(2):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=625, max_range=8.0)
        for m in (em, om):
            m.move_to(t + np.float32(0.2), R)
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    names = ["elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound", "normal_x", "normal_y",
             "normal_z", "min_filter", "smooth"]
    out = np.zeros((len(names), p.cell_n - 2, p.cell_n - 2), np.float32)
    em.get_maps_with_names_ref(names, out)
    one = np.zeros((p.cell_n - 2, p.cell_n - 2), np.float32)
    for k, name in enumerate(names):
        em.get_map_with_name_ref(name, one)
        assert np.array_equal(out[k], one, equal_nan=True), name
        if k < 9:
            ref = om.export_layer(name)
            tol = 2e-6 if name == "traversability" else 0.0
            assert np.array_equal(np.isnan(out[k]), np.isnan(ref)), name
            assert np.nanmax(np.abs(out[k] - ref), initial=0.0) <= tol, name
    with pytest.raises(KeyError):
        em.get_maps_with_names_ref(["no_such_layer"], out[:1])


def test_semantic_point_fusion_matches_oracle(oracle_mod):
    """SURVEY 8(f)2: feature channels of the cloud fused inside the frame (average / class_average / color) against the
    oracle (pinned to the reference's fusion kernel strings on the CPU); exported through the reference's layer API."""
    import torch
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    p = core_parameter(202)
    p.pointcloud_channel_fusions = {"rgb": "color", "feat_avg": "average", "default": "class_average"}
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    W = 202
    rng = np.random.default_rng(9)
    sem_or = np.zeros((3, W, W), np.float32)
    channels = ["x", "y", "z", "feat_avg", "person", "rgb"]
    kinds = ["average", "class_average", "color"]
    for f in range(3):
        pts, R, t = wl.uniform_cloud(0, f, n=20000, half_extent=3.5)
        feats = np.stack([rng.random(len(pts), dtype=np.float32) * 4 - 2, rng.random(len(pts), dtype=np.float32),
                          rng.integers(0, 1 << 24, len(pts)).astype(np.uint32).view(np.float32)], 1)
        cloud = np.ascontiguousarray(np.concatenate([pts, feats], 1))
        # the oracle frame on xyz; fused counts = cells of points that the fusion accepted (new_map[2])
        t_rel = (t - om.center).astype(np.float32)
        idx, valid, inside, _ = oracle_mod.point_index(p, pts, R, t_rel)
        src = torch.from_numpy(cloud).cuda() if f == 1 else cloud          # device rows once, host rows otherwise
        em.input_pointcloud(src, channels, R, t, 0.02, 0.02)
        om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        cnt = om.counts_fused.reshape(-1) if hasattr(om, "counts_fused") else None
        if cnt is None:
            pytest.skip("oracle does not expose the fused counts")
        oracle_mod.semantic_fuse(W, idx, valid, inside, feats, kinds, sem_or, cnt, alpha=0.5)
        got = np.stack([em.get_layer(n).cpu().numpy() for n in ("feat_avg", "person", "rgb")])
        assert np.array_equal(got[2].view(np.uint32), sem_or[2].view(np.uint32)), f
        for k in (0, 1):
            assert np.abs(got[k] - sem_or[k]).max() <= 2e-6 * max(1.0, float(np.abs(sem_or[k]).max())), (f, kinds[k])
    assert em.exists_layer("person") and em.exists_layer("rgb")
    out = np.zeros((W - 2, W - 2), np.float32)
    em.get_map_with_name_ref("person", out)
    assert np.array_equal(out, np.flip(sem_or[1][1:-1, 1:-1], (0, 1)))
    batched = np.zeros((2, W - 2, W - 2), np.float32)
    em.get_maps_with_names_ref(["elevation", "person"], batched)
    assert np.array_equal(batched[1], out)
    # the layers travel with the map (EM.py:221) and clear() empties them (EM.py:126)
    em.move(np.array([0.08, -0.12, 0.0]))
    moved = em.get_layer("person").cpu().numpy()
    ref = np.roll(sem_or[1], (2, -3), (0, 1)); ref[:2, :] = 0; ref[:, -3:] = 0
    assert np.array_equal(moved, ref)
    em.clear()
    assert float(em.get_layer("person").abs().max()) == 0.0


def test_initialize_map_matches_oracle(oracle_mod):
    """EM.py:899-922: griddata on the host (as the reference), dilation x2 + upper-bound fill on the device."""
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(64, dilation_size_initialize=3)
    em = _mk(p)
    em.move_to(np.array([0.4, -0.2, 0.3]), np.eye(3, dtype=np.float32))
    pts = np.array([[0.0, 0.2, 0.31], [0.9, -0.6, 0.42], [-0.3, -0.9, 0.2], [0.1, 0.5, 0.55], [0.8, 0.3, 0.4]], np.float32)
    before, _ = em.get_state()
    em.initialize_map(pts, "linear")
    state, _ = em.get_state()
    cleared = np.zeros_like(before); cleared[1] = np.float32(p.initial_variance)      # clear() first (EM.py:905)
    ref = oracle_mod.initialize_map_planes(p, cleared, pts, em.center, "linear")
    assert (state[2] > 0.5).sum() > 50
    for li in (0, 1, 2, 5, 6):
        assert np.array_equal(state[li], ref[li]), li
