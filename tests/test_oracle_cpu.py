"""CPU tests of the oracle (no GPU): the C restatement against (1) the committed golden vectors produced
by the REFERENCE'S OWN kernel source, (2) an independent NumPy restatement of the index arithmetic,
(3) stored outputs of the reference's kernel source on further seeded inputs (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest

from elevation_mapping_cupy_b200 import workloads as wl
from elevation_mapping_cupy_b200.parameter import Parameter, core_parameter
from helpers import FLAG_CASES, STAR_R, dilation_inputs, drift_frames, semantic_inputs, star_inputs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("seed", [0, 1])
def test_point_index_matches_reference_golden(oracle_mod, seed):
    """bit-identical (idx, valid, inside) vs the reference kernel's write-back (CK.py:260-262)"""
    g = np.load(os.path.join(GOLD, f"index_default202_seed{seed}.npz"))
    p = Parameter(); p.update()
    pts, R, t = wl.reference_test_cloud(seed, n=20000)
    if seed % 2:
        pts = (pts * np.float32(9.0) - np.float32(4.5)).astype(np.float32)
    idx, valid, inside, _ = oracle_mod.point_index(p, pts, R, t)
    assert np.array_equal(idx, g["idx"])
    assert np.array_equal(valid, g["valid"])
    assert np.array_equal(inside, g["inside"])
    # independent NumPy restatement of the same arithmetic
    ni, nv, nin = oracle_mod.point_index_numpy(p, pts, R, t)
    assert np.array_equal(ni, idx) and np.array_equal(nv, valid) and np.array_equal(nin, inside)


def test_index_numpy_vs_c_on_large_map(oracle_mod):
    p = core_parameter(2048)
    rng = np.random.default_rng(5)
    pts = rng.uniform(-45, 45, (50000, 3)).astype(np.float32)
    R = np.eye(3, dtype=np.float32); t = np.array([0.3, -0.2, 1.0], np.float32)
    a = oracle_mod.point_index(p, pts, R, t)
    b = oracle_mod.point_index_numpy(p, pts, R, t)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_frames_match_reference_golden(oracle_mod):
    """4 LiDAR frames on a 130^2 map: the oracle's state equals (a) its own committed output exactly and
    (b) the reference kernel source's output to 1e-6 on every cell whose outcome is order-independent."""
    g = np.load(os.path.join(GOLD, "frames_core130.npz"))
    p = core_parameter(130)
    om = oracle_mod.OracleElevationMap(p)
    for f in range(4):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        om.move_to(t, R)
        om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        for li in (0, 1, 2, 4, 5, 6):
            assert np.array_equal(om.elevation_map[li], g[f"oracle_state_{f}"][li]), (f, li)
        assert np.abs(om.elevation_map[3] - g[f"oracle_state_{f}"][3]).max() < 1e-6
        assert np.array_equal(om.normal_map, g[f"oracle_normal_{f}"])
        racy = g[f"racy_{f}"]
        assert racy.mean() < 0.05
        for li in (0, 1, 2, 4, 5, 6):
            d = np.abs(om.elevation_map[li] - g[f"ref_state_{f}"][li])
            assert d[~racy].max() <= 1e-6, (f, li, d[~racy].max())
        assert np.array_equal(om.last_point_record[0], g[f"ref_point_idx_{f}"])
        om.update_variance(); om.update_time()


def test_oracle_threads_are_deterministic(oracle_mod):
    p = core_parameter(130)
    a = oracle_mod.OracleElevationMap(p, nthreads=1); b = oracle_mod.OracleElevationMap(p, nthreads=4)
    for f in range(2):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        for m in (a, b):
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02); m.update_time()
    assert np.array_equal(a.elevation_map, b.elevation_map)
    assert np.array_equal(a.normal_map, b.normal_map)


def test_multi_sensor_equals_concatenation_when_poses_equal(oracle_mod):
    p = core_parameter(130)
    a = oracle_mod.OracleElevationMap(p); b = oracle_mod.OracleElevationMap(p)
    pts, R, t = wl.lidar_cloud(0, 0, n_rings=24, n_az=500, max_range=4.0)
    a.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.0, 0.0)
    b.input_sensors([pts[:5000], pts[5000:]], [R, R], [t, t], 0.0, 0.0)
    assert np.array_equal(a.elevation_map, b.elevation_map)


def test_traversability_matches_torch_cpu(oracle_mod):
    """traversability_filter.py:15-42 on the host with torch vs the oracle's direct convolution"""
    torch = pytest.importorskip("torch")
    p = core_parameter(130)
    rm_w = oracle_mod.load_weights(p)
    x = np.random.default_rng(0).standard_normal((130, 130)).astype(np.float32)
    ours = oracle_mod.traversability(130, x, rm_w)
    import torch.nn.functional as F
    w1, w2, w3, wo = [torch.from_numpy(w) for w in rm_w]
    e = torch.from_numpy(x).view(1, 1, 130, 130)
    o1 = F.conv2d(e, w1.view(4, 1, 3, 3), dilation=1)[:, :, 2:-2, 2:-2]
    o2 = F.conv2d(e, w2.view(4, 1, 3, 3), dilation=2)[:, :, 1:-1, 1:-1]
    o3 = F.conv2d(e, w3.view(4, 1, 3, 3), dilation=3)
    ref = torch.exp(-F.conv2d(torch.cat((o1, o2, o3), 1).abs(), wo.view(1, 12, 1, 1)))[0, 0].numpy()
    assert np.abs(ours - ref).max() < 2e-6


def test_smooth_matches_scipy(oracle_mod):
    from scipy import ndimage
    x = np.random.default_rng(1).standard_normal((202, 202)).astype(np.float32)
    ours = oracle_mod.smooth(202, x)
    ref = ndimage.uniform_filter(ndimage.uniform_filter(x, size=3), size=3)     # smooth_filter.py:57-58
    assert np.abs(ours - ref).max() < 1e-6


def test_dilation_and_normal_against_reference_source(oracle_mod):
    """the reference's dilation / normal / min_filter kernels, stored in tests/golden/refsrc_core130.npz"""
    g = np.load(os.path.join(GOLD, "refsrc_core130.npz"))
    p = core_parameter(130)
    W = 130
    h, mask = dilation_inputs(W)
    ours, _ = oracle_mod.dilation(W, p.dilation_size, h, mask)
    assert np.array_equal(ours, g["dilation"])
    # the host build of the reference source has no FMA contraction (g++ -ffp-contract=off) while the oracle
    # follows nvcc's contraction of CK.py:497 (fma(nx,nx, ny*ny) + 1): last-ulp differences only
    on = oracle_mod.normal(W, p.resolution, ours, mask)
    assert np.array_equal(on != 0, g["normal"] != 0)
    assert np.abs(on - g["normal"]).max() <= 2.4e-7
    # min_filter: the reference updates in place (Gauss-Seidel); with one iteration on a mask whose invalid
    # cells have no invalid neighbours inside the window the two orders coincide
    m2 = np.ones((W, W), np.float32); m2[5:-5:4, 5:-5:4] = 0
    ours_mf, _ = oracle_mod.min_filter(W, 1, 1, h, m2)
    assert np.array_equal(np.nan_to_num(ours_mf), np.nan_to_num(g["min_filter"]))


def test_star_plugin_oracles_against_reference_source(oracle_mod):
    """max_filter / robot_centric_elevation restatements vs the reference's kernels (stored outputs of the host
    build of their source)."""
    g = np.load(os.path.join(GOLD, "refsrc_core130.npz"))
    p = core_parameter(130)
    W = 130
    h, m = star_inputs(W)
    ours, _ = oracle_mod.max_filter(W, 1, 4, h, m)
    assert np.array_equal(np.nan_to_num(ours, nan=-7), np.nan_to_num(g["max_filter"], nan=-7))
    # robot_centric_elevation.py:118-121
    for thr in (True, False):
        out = g["base_elevation_thr" if thr else "base_elevation_raw"]
        ours = oracle_mod.robot_centric(W, p.resolution, 1.1, thr, h, m, STAR_R)
        if thr:
            assert np.array_equal(ours, out)
        else:       # host build has no FMA contraction: last-ulp differences
            assert np.abs(ours - out).max() <= 5e-7 * max(1.0, np.abs(out).max())


def test_drift_compensation_against_reference_source(oracle_mod):
    """EM.py:346-357 fires (error_cnt > min_height_drift_cnt, |mean| < max_drift): oracle vs the reference's kernels
    (tests/golden/drift_core130.npz; traversability is not compared)"""
    from oracle.configs import DRIFT_OVERRIDES
    g = np.load(os.path.join(GOLD, "drift_core130.npz"))
    p = core_parameter(130, **DRIFT_OVERRIDES)
    om = oracle_mod.OracleElevationMap(p)
    fired = 0
    for f, (pts, R, t) in enumerate(drift_frames()):
        om.move_to(t, R); om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        racy = g[f"racy_{f}"]
        for li in (0, 1, 2, 4, 5, 6):
            assert np.abs(om.elevation_map[li] - g[f"ref_state_{f}"][li])[~racy].max() <= 1e-6
        if om.stats.drift_applied:
            fired += 1
            assert abs(om.stats.mean_error - float(g[f"mean_error_{f}"])) < 1e-6
        om.update_variance(); om.update_time()
    assert fired >= 3


@pytest.mark.parametrize("case", range(len(FLAG_CASES)), ids=[f"flags{i}" for i in range(len(FLAG_CASES))])
def test_flag_combinations_against_reference_source(oracle_mod, case):
    """feature toggles and thresholds are baked into the reference's kernel source: its build per combination,
    run in input order and reversed (tests/golden/flags<case>_core130.npz), against the oracle for three frames on
    the order-independent cells"""
    flags = FLAG_CASES[case]
    g = np.load(os.path.join(GOLD, f"flags{case}_core130.npz"))
    p = core_parameter(130, **flags)
    om = oracle_mod.OracleElevationMap(p)
    for f in range(3):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        om.move_to(t, R); om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        racy = g[f"racy_{f}"]
        n_cmp = int((~racy).sum())
        for li in (0, 1, 2, 4, 5, 6):
            d = np.abs(om.elevation_map[li] - g[f"ref_state_{f}"][li])[~racy]
            assert int((d > 1e-6).sum()) <= 3, (flags, f, li, float(d.max()))      # symmetric order-dependent patterns
        assert np.array_equal(om.last_point_record[0], g[f"ref_point_idx_{f}"])
        assert n_cmp > 0.9 * 130 * 130
        om.update_variance(); om.update_time()


def test_semantic_fusion_oracle_against_reference_source(oracle_mod):
    """SURVEY 8(f)2: the NumPy restatement of the point-channel fusions (average, class_average, color) against the
    reference's own kernel strings (fusion/pointcloud_average.py, pointcloud_class_average.py, pointcloud_color.py),
    compiled for the host by oracle/build_ref.py and run one element at a time in input order (stored outputs)."""
    g = np.load(os.path.join(GOLD, "refsrc_core130.npz"))
    p = core_parameter(130)
    W = 130
    idx, valid, inside, _, feats, cnt = semantic_inputs(p, W)
    kinds = ["average", "class_average", "color"]
    sem_or = np.zeros((3, W, W), np.float32)
    for frame in range(2):                    # second frame exercises class_average's running mix
        sem_ref = g[f"semantic_{frame}"]
        oracle_mod.semantic_fuse(W, idx, valid, inside, feats, kinds, sem_or, cnt, alpha=0.5)
        assert np.array_equal(sem_ref[2].view(np.uint32), sem_or[2].view(np.uint32)), "color"
        for k in (0, 1):
            d = np.abs(sem_ref[k] - sem_or[k])
            assert d.max() <= 2e-6 * max(1.0, float(np.abs(sem_ref[k]).max())), (frame, kinds[k], float(d.max()))
