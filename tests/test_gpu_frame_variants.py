"""GPU: whole frames at the configurations the other frame tests never reach, against OracleElevationMap.  Bar as in
tests/test_gpu_parity.py: every state plane bit-identical except traversability (2e-6), plus the point record and the
frame statistics.  The cases come from tests/frame_variants.py; tests/test_frame_variants_cpu.py checks without a GPU
that each group reaches the host decisions it is meant to reach."""
import types

import numpy as np
import pytest

import frame_variants as fv
from helpers import check_frame as _check_frame, compare_state

pytestmark = pytest.mark.gpu


def _param(cell_n, **kw):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    return core_parameter(cell_n, **kw)


def _mk(p, count_rays=False):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    em = ElevationMap(p)
    if count_rays:
        em._check(em._L.emap_set_ray_counting(em._h, 1))
    return em


def _random_state(W, seed, valid_frac=0.2):
    """the random state of test_post_chain_on_random_state: border columns populated, cells old enough for rays to act"""
    rng = np.random.default_rng(seed)
    st = np.zeros((7, W, W), np.float32)
    st[0] = rng.standard_normal((W, W)); st[1] = 0.05
    st[2] = rng.random((W, W)) < valid_frac
    b = min(5, W)
    st[2][:, :b] = rng.random((W, b)) < 0.7; st[2][:, -b:] = rng.random((W, b)) < 0.7
    st[3] = 1.0; st[4] = 1.0
    st[5] = rng.standard_normal((W, W)); st[6] = (rng.random((W, W)) < 0.1) * (st[2] < 0.5)
    st[0] *= st[2]
    return st


# ---- A: resolution, ray length and map size -------------------------------------------------------------------------
@pytest.mark.parametrize("case", fv.RES_CASES, ids=[c["id"] for c in fv.RES_CASES])
def test_frames_at_other_resolutions_ray_lengths_and_sizes(oracle_mod, case):
    from elevation_mapping_cupy_b200 import workloads as wl
    W, res, L = fv.frame_params(case)
    p = _param(W, **case["kw"])
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    half = 0.5 * (W - 2) * res
    for f in range(3):
        if f % 2 == 0:
            pts, R, t = wl.uniform_cloud(0, f, n=20000, half_extent=min(4.9, 0.9 * half))
        else:
            pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=1000, max_range=min(25.0, L + 6.0))
        for m in (em, om):
            m.move_to(t, R)
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        st, _, _ = _check_frame(em, om, len(pts), f"{case['id']} frame {f}")
        assert st.n_valid_points > 0
        for m in (em, om):
            m.update_variance(); m.update_time()
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"{case['id']} frame {f} after ticks")


# ---- B: every dilation on both k_post paths -------------------------------------------------------------------------
@pytest.mark.parametrize("W", fv.POST_SIZES)
def test_post_every_dilation_on_random_state(oracle_mod, W):
    """dilation K = 0..8 (the flat-index row wrap on populated border columns) + CNN + normals, driven by an empty
    cloud, with TMA staging or plain loads as the host picks them"""
    for K in fv.POST_KS:
        p = _param(W, dilation_size=K, enable_visibility_cleanup=(K % 2 == 0))
        em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
        st = _random_state(W, 1000 * W + K)
        em.set_state(st); om.elevation_map = st.copy()
        empty = np.zeros((0, 3), np.float32)
        R = np.eye(3, dtype=np.float32); t = np.array([0, 0, 1.0], np.float32)
        em.input_pointcloud(empty, ["x", "y", "z"], R, t, 0.0, 0.0)
        om.input_pointcloud(empty, ["x", "y", "z"], R, t, 0.0, 0.0)
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"post {W}/K{K}")
        assert np.array_equal(em.traversability_input.cpu().numpy(), om.traversability_input), (W, K)


# ---- C: sensor poses at and beyond the map edge ---------------------------------------------------------------------
def _pose_cloud(t, rng, n=3000):
    """points around a sensor at t, in the sensor frame (R = I): below it on a rough surface, or, for a sensor below the
    terrain, a little above it (rays going up); every point valid"""
    az = rng.uniform(0, 2 * np.pi, n)
    d = rng.uniform(0.6, 14.0, n)
    up = t[2] < 0
    dz = rng.uniform(0.05, 0.18, n) if up else -rng.uniform(0.3, 2.0, n)
    return np.stack([d * np.cos(az), d * np.sin(az), dz], 1).astype(np.float32)


@pytest.mark.parametrize("W", fv.POSE_SIZES)
def test_sensor_poses_at_and_beyond_the_map_edge(oracle_mod, W):
    """frames without move_to (map centre at the origin) from sensors one cell inside each edge, on the border ring,
    beyond an edge within and beyond max_ray_length (an empty ray box), two sensors far apart and a sensor below the
    terrain; once with the march and once with the step-counting march, whose statistics must equal the oracle's"""
    p = _param(W)
    for k, (cid, ts) in enumerate(fv.pose_cases(W)):
        rng = np.random.default_rng(W + k)
        clouds = [_pose_cloud(t, rng) for t in ts]
        Rs = [np.eye(3, dtype=np.float32)] * len(ts)
        tv = [np.array(t, np.float32) for t in ts]
        em, emc = _mk(p), _mk(p, count_rays=True)
        om = oracle_mod.OracleElevationMap(p, nthreads=0)
        st0 = _random_state(W, W + k, valid_frac=0.5)
        for m in (em, emc):
            m.set_state(st0)
        om.elevation_map = st0.copy()
        n = sum(len(c) for c in clouds)
        for f in range(2):
            for m in (em, emc, om):
                m.input_sensors(clouds, Rs, tv, 0.0, 0.0)
            st, _, _ = _check_frame(em, om, n, f"{W} {cid} frame {f}")
            assert st.n_valid_points > 0, cid
            stc, _, _ = _check_frame(emc, om, n, f"{W} {cid} frame {f} (counting)", counted=True)
            assert stc.ray_steps > 0, cid
            for m in (em, emc, om):
                m.update_time()


# ---- D: input layouts -----------------------------------------------------------------------------------------------
def _layout_source(layout, pts):
    """(the cloud in `layout`, the host buffer the library reads or None)"""
    import torch
    n = len(pts)
    if layout == "f32-host":
        a = pts.copy()
        return a, a
    if layout == "f32x4-device":
        buf = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
        buf[:, :3] = torch.from_numpy(pts).cuda()
        assert buf.data_ptr() % 16 == 0
        return buf, None
    if layout == "f32x4-device-unaligned":
        buf = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
        buf[:, 1:4] = torch.from_numpy(pts).cuda()
        v = buf[:, 1:4]
        assert v.data_ptr() % 16 == 4 and v.stride() == (4, 1)
        return v, None
    if layout in ("f32-pinned", "f64-pinned"):
        a = torch.from_numpy(pts.astype(np.float32 if layout == "f32-pinned" else np.float64)).pin_memory()
        assert a.is_pinned()
        return a, a
    if layout == "f64-device-strided":
        buf = torch.zeros((2 * n, 3), dtype=torch.float64, device="cuda")
        buf[::2] = torch.from_numpy(pts.astype(np.float64)).cuda()
        v = buf[::2]
        assert v.stride() == (6, 1)
        return v, None
    raise KeyError(layout)


def _overwrite(buf):
    """the caller reuses its host buffer as soon as the frame call returns (include/emap.h)"""
    if isinstance(buf, np.ndarray):
        buf[...] = np.nan
    else:
        buf.fill_(float("nan"))


def test_input_layouts_agree_with_the_oracle_and_each_other(oracle_mod):
    """three frames through every input layout, each on its own handle; host buffers are overwritten with NaN as soon
    as each call returns"""
    from elevation_mapping_cupy_b200 import workloads as wl
    p = _param(256)
    frames = [wl.lidar_cloud(0, f, n_rings=32, n_az=625, max_range=8.0) for f in range(3)]
    frames[1][0][::11] = np.nan
    om = oracle_mod.OracleElevationMap(p, nthreads=0)
    ref = []
    for pts, R, t in frames:
        om.move_to(t, R)
        om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        ref.append((types.SimpleNamespace(elevation_map=om.elevation_map.copy(), normal_map=om.normal_map.copy(),
                                          last_point_record=om.last_point_record, stats=om.stats)))
        om.update_variance(); om.update_time()
    first = None
    for layout in fv.LAYOUTS:
        em = _mk(p)
        got = []
        for f, (pts, R, t) in enumerate(frames):
            src, host = _layout_source(layout, pts)
            em.move_to(t, R)
            em.input_pointcloud(src, ["x", "y", "z"], R, t, 0.02, 0.02)
            if host is not None:
                _overwrite(host)
            _, state, normal = _check_frame(em, ref[f], len(pts), f"{layout} frame {f}", nan_rows=np.isnan(pts).any(1))
            got.append((state, normal))
            em.update_variance(); em.update_time()
        if first is None:
            first = got
        for f in range(len(frames)):
            assert np.array_equal(got[f][0], first[f][0]) and np.array_equal(got[f][1], first[f][1]), (layout, f)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_many_sensors_some_empty(oracle_mod, device):
    """a frame of more than 64 sensors (the sensor pointers no longer fit frame_begin's stack array), some with no rows"""
    import torch
    p = _param(256)
    rng = np.random.default_rng(70)
    clouds, Rs, ts = [], [], []
    for s in range(fv.MANY_SENSORS):
        n = 0 if s % 9 == 4 else int(rng.integers(20, 300))
        t = np.array([rng.uniform(-4, 4), rng.uniform(-4, 4), rng.uniform(0.5, 1.5)], np.float32)
        a = rng.uniform(0, 2 * np.pi)
        R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], np.float32)
        off = np.stack([rng.uniform(-6, 6, n), rng.uniform(-6, 6, n), -t[2] + rng.normal(0, 0.05, n)], 1)
        clouds.append(off.astype(np.float32)); Rs.append(R); ts.append(t)
    assert sum(len(c) == 0 for c in clouds) >= 7
    em = _mk(p); om = oracle_mod.OracleElevationMap(p, nthreads=0)
    src = [torch.from_numpy(c).cuda() for c in clouds] if device else clouds
    n = sum(len(c) for c in clouds)
    for f in range(2):
        em.input_sensors(src, Rs, ts, 0.02, 0.02, device_ptrs=device)
        om.input_sensors(clouds, Rs, ts, 0.02, 0.02)
        st, _, _ = _check_frame(em, om, n, f"{fv.MANY_SENSORS} sensors frame {f}")
        assert st.n_valid_points > 0
        for m in (em, om):
            m.update_variance(); m.update_time()
