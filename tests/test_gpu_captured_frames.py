"""GPU: frames captured into CUDA graphs and replayed, and eager frames and ticks ordered against a caller's stream with
no host synchronisation, against OracleElevationMap running the same calls eagerly on the host.  Bar as in
tests/test_gpu_parity.py: every state plane bit-identical except traversability (2e-6), normals bit-identical, plus the
point record and the frame statistics.

A captured frame binds the map buffer, the cloud, and the pose relative to the map centre at capture (include/emap.h),
so a replay is valid only at the capture centre, bit for bit.  The captured maps use a 1/16 m resolution: centres are
then exact binary fractions, and moves that return to a centre return to it exactly.  Every replay first asserts that,
so that a failure points at the frame and not at the centre."""
import numpy as np
import pytest

from helpers import check_frame, compare_state, drift_frames

pytestmark = pytest.mark.gpu

RES = 0.0625
XYZ = ["x", "y", "z"]
DRIFT = dict(traversability_inlier=0.0, drift_compensation_variance_inlier=10.0, min_height_drift_cnt=10)


def _param(W, **kw):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    return core_parameter(W, resolution=RES, **kw)


def _mk(p, count_rays=False, stream=None):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    em = ElevationMap(p)
    if count_rays:
        em._check(em._L.emap_set_ray_counting(em._h, 1))
    if stream is not None:
        em.set_stream(stream.cuda_stream)
    return em


def _on_grid(t):
    """t rounded to the 1/16 m grid: a centre every move_to reaches exactly"""
    return np.round(np.asarray(t, np.float64) / RES) * RES


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _capture(em, s, call, extra=lambda: []):
    """CUDA graph of call() on s, the stream em runs on.  The capture must launch the frame's kernels and run none of
    them: the state (and extra(), e.g. semantic layers) is unchanged after it."""
    import torch
    before = [_bits(a) for a in em.get_state()] + [_bits(a) for a in extra()]
    launches = em.launch_count()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        call()
    assert em.launch_count() >= launches + 5
    s.synchronize()
    after = [_bits(a) for a in em.get_state()] + [_bits(a) for a in extra()]
    assert all(np.array_equal(a, b) for a, b in zip(before, after)), "the capture ran work"
    return g


def _replay(g, em, s, centre, label):
    """replay g on s after the caller's queued work, at the capture centre"""
    import torch
    assert np.array_equal(_bits(em.center), _bits(np.float32(centre))), (label, em.center, centre)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g.replay()


def _ticks(*maps):
    for m in maps:
        m.update_variance(); m.update_time()


# ---- A: replay equals eager, with ticks in between ------------------------------------------------------------------
@pytest.mark.parametrize("W", [256, 130])
def test_replays_equal_eager_frames_with_ticks_between(oracle_mod, W):
    """two captured LiDAR frames (one with a 3 cm bias) replayed alternately with update_variance / update_time between,
    under parameters at which drift compensation fires: the decision is taken on the device at every replay.  At 256 the
    second graph reads a pinned host cloud (zero-copy).  A ray-counting handle replays the same graphs in lockstep."""
    import torch
    p = _param(W, **DRIFT)
    s, sc = torch.cuda.Stream(), torch.cuda.Stream()
    em, emc = _mk(p, stream=s), _mk(p, count_rays=True, stream=sc)
    om = oracle_mod.OracleElevationMap(p, nthreads=0)
    frames = drift_frames(2)
    n = len(frames[0][0])
    assert len(frames[1][0]) == n
    src = [torch.from_numpy(frames[0][0]).cuda(),
           torch.from_numpy(frames[1][0]).pin_memory() if W == 256 else torch.from_numpy(frames[1][0]).cuda()]
    try:
        pts, R, t = frames[0]
        for m, c in ((em, src[0]), (emc, src[0]), (om, pts)):           # warm-up: sizes every buffer of the frame
            m.input_pointcloud(c, XYZ, R, t, 0.02, 0.02)
        check_frame(em, om, n, f"{W} warm-up")
        _ticks(em, emc, om)
        centre = em.center.copy()
        graphs = {}
        for m, st in ((em, s), (emc, sc)):
            graphs[m] = [_capture(m, st, lambda m=m, f=f: m.input_pointcloud(src[f], XYZ, frames[f][1], frames[f][2],
                                                                               0.02, 0.02)) for f in range(2)]
        fired = 0
        for k in range(6):
            f = k % 2
            pts, R, t = frames[f]
            for m, st in ((em, s), (emc, sc)):
                _replay(graphs[m][f], m, st, centre, f"{W} replay {k}")
            om.input_pointcloud(pts, XYZ, R, t, 0.02, 0.02)
            st_, _, _ = check_frame(em, om, n, f"{W} replay {k}")
            check_frame(emc, om, n, f"{W} replay {k} (counting)", counted=True)
            fired += bool(st_.drift_applied)
            _ticks(em, emc, om)
            state, normal = em.get_state()
            compare_state(state, normal, om, label=f"{W} replay {k} after ticks")
        assert fired >= 2, fired
    finally:
        em.set_stream(None); emc.set_stream(None)


# ---- B: replay after moves that return to the capture centre --------------------------------------------------------
@pytest.mark.parametrize("W", [256, 130])
def test_replays_after_moves_back_to_the_capture_centre(oracle_mod, W):
    """three move_to whose cell shifts are all non-zero and add up to zero (an odd number of shifts), a z-only move_to
    and back, then a replay; then move by a non-zero shift and back, and replay the other graph; then a tick and a
    replay with no move at all"""
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    p = _param(W)
    s = torch.cuda.Stream()
    em = _mk(p, stream=s)
    om = oracle_mod.OracleElevationMap(p, nthreads=0)
    frames = [wl.lidar_cloud(1, f, n_rings=24, n_az=500, max_range=4.0) for f in range(2)]
    n = len(frames[0][0])
    src = [torch.from_numpy(pts).cuda() for pts, _, _ in frames]
    R0 = frames[0][1]
    centre = _on_grid(frames[0][2])
    try:
        for m in (em, om):
            m.move_to(centre, R0)
            m.input_pointcloud(frames[0][0], XYZ, R0, frames[0][2], 0.02, 0.02)
        check_frame(em, om, n, f"{W} warm-up")
        _ticks(em, om)
        c32 = em.center.copy()
        assert np.array_equal(c32.astype(np.float64), centre)
        graphs = [_capture(em, s, lambda f=f: em.input_pointcloud(src[f], XYZ, frames[f][1], frames[f][2], 0.02, 0.02))
                  for f in range(2)]

        def frame(f, label):
            _replay(graphs[f], em, s, c32, label)
            pts, R, t = frames[f]
            om.input_pointcloud(pts, XYZ, R, t, 0.02, 0.02)
            check_frame(em, om, n, label)

        shifts = [(3, -2), (-5, 4), (2, -2)]
        assert np.sum(shifts, 0).tolist() == [0, 0]
        pos = centre.copy()
        for d in shifts:
            pos[:2] += np.array(d) * RES
            for m in (em, om):
                m.move_to(pos.copy(), R0)
        for dz in (0.25, 0.0):                                  # z only: the in-place shift
            for m in (em, om):
                m.move_to(centre + [0.0, 0.0, dz], R0)
        frame(0, f"{W} after three moves and a z move")
        for d in ((2 * RES, -3 * RES, 0.0), (-2 * RES, 3 * RES, 0.0)):
            for m in (em, om):
                m.move(np.array(d))
        frame(1, f"{W} after a move and back")
        _ticks(em, om)
        frame(0, f"{W} after ticks")
        for m in (em, om):                                      # the map still moves and takes eager frames
            m.move_to(centre + [5 * RES, RES, 0.0], R0)
            m.input_pointcloud(frames[1][0], XYZ, frames[1][1], frames[1][2], 0.02, 0.02)
        check_frame(em, om, n, f"{W} eager frame after the replays")
    finally:
        em.set_stream(None)


# ---- C: config E in miniature ---------------------------------------------------------------------------------------
def test_config_e_in_miniature(oracle_mod):
    """four 512^2 maps, each on its own torch stream with two pool frames; graph f captured right after move_to(pose f);
    then four steps of move_to(pose f), update_variance, update_time and a round-robin replay of every map's graph,
    with no host synchronisation inside a step"""
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    p = _param(512)
    n_maps, n_steps = 4, 4
    streams = [torch.cuda.Stream() for _ in range(n_maps)]
    ems = [_mk(p, stream=st) for st in streams]
    frames = [[wl.lidar_cloud(4, 10 * m + f, n_rings=32, n_az=1250, max_range=12.0) for f in range(2)]
              for m in range(n_maps)]
    src = [[torch.from_numpy(pts).cuda() for pts, _, _ in fr] for fr in frames]

    def ticks(em, m, f):
        R, t = frames[m][f][1:]
        em.move_to(t, R); em.update_variance(); em.update_time()

    def frame(em, m, f):
        pts, R, t = frames[m][f]
        em.input_pointcloud(src[m][f] if em in ems else pts, XYZ, R, t, 0.02, 0.02)

    try:
        for f in range(2):
            for m, em in enumerate(ems):
                ticks(em, m, f); frame(em, m, f)
        torch.cuda.synchronize()
        graphs, centres = [], []
        for m, em in enumerate(ems):
            gs, cs = [], []
            for f in range(2):
                em.move_to(frames[m][f][2], frames[m][f][1])
                cs.append(em.center.copy())
                gs.append(_capture(em, streams[m], lambda em=em, m=m, f=f: frame(em, m, f)))
            assert not np.array_equal(cs[0], cs[1])
            graphs.append(gs); centres.append(cs)
        for step in range(n_steps):
            f = step % 2
            for m, em in enumerate(ems):
                ticks(em, m, f)
            for m, em in enumerate(ems):
                _replay(graphs[m][f], em, streams[m], centres[m][f], f"map {m} step {step}")
        for m in (0, n_maps - 1):
            om = oracle_mod.OracleElevationMap(p, nthreads=0)
            for f in range(2):
                ticks(om, m, f); frame(om, m, f)
            for f in range(2):
                om.move_to(frames[m][f][2], frames[m][f][1])
            for step in range(n_steps):
                ticks(om, m, step % 2); frame(om, m, step % 2)
            check_frame(ems[m], om, len(frames[m][(n_steps - 1) % 2][0]), f"map {m}")
    finally:
        for em in ems:
            em.set_stream(None)


# ---- D: semantic channels in a captured frame -----------------------------------------------------------------------
def test_semantic_channels_in_a_captured_frame():
    """average, class_average and color channels fused inside captured frames replayed across moves, against an eager
    twin handle given the same calls: every state plane, the normals, the semantic layers and the point record
    bit-identical (eager semantic fusion is pinned to the oracle in tests/test_gpu_parity.py)"""
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    p = _param(202)
    p.pointcloud_channel_fusions = {"rgb": "color", "feat_avg": "average", "default": "class_average"}
    s = torch.cuda.Stream()
    em, twin = _mk(p, stream=s), _mk(p)
    channels = XYZ + ["feat_avg", "person", "rgb"]
    rng = np.random.default_rng(9)
    frames = []
    for f in range(2):
        pts, R, t = wl.uniform_cloud(0, f, n=20000, half_extent=3.5)
        feats = np.stack([rng.random(len(pts), dtype=np.float32) * 4 - 2, rng.random(len(pts), dtype=np.float32),
                          rng.integers(0, 1 << 24, len(pts)).astype(np.uint32).view(np.float32)], 1)
        frames.append((torch.from_numpy(np.ascontiguousarray(np.concatenate([pts, feats], 1))).cuda(), R, t))
    n = frames[0][0].shape[0]
    R0 = frames[0][1]
    centre = _on_grid(frames[0][2] + np.float32(0.3))

    def sem(m):
        return [m.semantic_map.semantic_map.cpu().numpy()]

    def same(label):
        a, b = em.get_state(), twin.get_state()
        for x, y, what in ((a[0], b[0], "state"), (a[1], b[1], "normals"), (sem(em)[0], sem(twin)[0], "semantic")):
            assert np.array_equal(_bits(x), _bits(y)), f"{label}: {what} differ in {int((_bits(x) != _bits(y)).sum())} words"
        assert all(np.array_equal(x, y) for x, y in zip(em.get_point_record(n), twin.get_point_record(n))), label

    try:
        for m in (em, twin):
            m.move_to(centre, R0)
            m.input_pointcloud(frames[0][0], channels, frames[0][1], frames[0][2], 0.02, 0.02)
        same("warm-up")
        assert np.abs(sem(twin)[0]).max() > 0
        c32 = em.center.copy()
        graphs = [_capture(em, s, lambda f=f: em.input_pointcloud(frames[f][0], channels, frames[f][1], frames[f][2],
                                                                   0.02, 0.02), extra=lambda: sem(em)) for f in range(2)]

        def frame(f, label):
            _replay(graphs[f], em, s, c32, label)
            twin.input_pointcloud(frames[f][0], channels, frames[f][1], frames[f][2], 0.02, 0.02)
            same(label)

        pos = centre.copy()
        for d in [(4, 1), (-1, -6), (-3, 5)]:
            pos[:2] += np.array(d) * RES
            for m in (em, twin):
                m.move_to(pos.copy(), R0)
        frame(1, "after three moves")
        for d in ((-RES, 2 * RES, 0.0), (RES, -2 * RES, 0.0)):
            for m in (em, twin):
                m.move(np.array(d))
        frame(0, "after a move and back")
        _ticks(em, twin)
        frame(1, "after ticks")
    finally:
        em.set_stream(None)


# ---- E: eager frames and ticks on a caller stream, without host syncs -----------------------------------------------
def _eager_frames_and_edits_on_a_caller_stream(oracle_mod, frame):
    """the handle on its own stream, torch on a side stream.  Before each frame the side stream sleeps and then edits the
    aliased state (a block of variance, a block of cleared is_valid); then frame(em, host cloud, device cloud, R, t),
    move_to and update_time.  After the last call a layer is cloned on the side stream before any synchronisation.  A
    library call that overtook the edits, or a clone that read the view before the frame finished, gives a state other
    than the oracle's."""
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(256)
    em = _mk(p)
    om, unedited = oracle_mod.OracleElevationMap(p, nthreads=0), oracle_mod.OracleElevationMap(p, nthreads=0)
    frames = [wl.lidar_cloud(0, f, n_rings=32, n_az=625, max_range=8.0) for f in range(3)]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        src = [torch.from_numpy(pts).cuda() for pts, _, _ in frames]
        for f, (pts, R, t) in enumerate(frames):
            r0 = 40 + 30 * f
            torch.cuda._sleep(20_000_000)                   # the edits are still queued when the library's calls are
            view = em.elevation_map
            view[1, r0:r0 + 40, 60:150] = 0.25
            view[2, 120:170, r0:r0 + 50] = 0.0
            om.elevation_map[1, r0:r0 + 40, 60:150] = 0.25
            om.elevation_map[2, 120:170, r0:r0 + 50] = 0.0
            move = np.asarray(t, np.float64) + [0.33, -0.21, 0.05]
            frame(em, pts, src[f], R, t); em.move_to(move, R); em.update_time()
            for m in (om, unedited):
                m.input_pointcloud(pts, XYZ, R, t, 0.02, 0.02); m.move_to(move, R); m.update_time()
        elevation = em.get_layer("elevation").clone()
        variance = em.elevation_map[1].clone()
    torch.cuda.synchronize()
    assert np.array_equal(_bits(elevation.cpu().numpy()), _bits(om.elevation_map[0]))
    assert np.array_equal(_bits(variance.cpu().numpy()), _bits(om.elevation_map[1]))
    changed = [int((om.elevation_map[li] != unedited.elevation_map[li]).sum()) for li in (0, 1, 2)]
    assert changed[0] > 100 and changed[1] > 100 and changed[2] > 0, changed     # the edits matter to the frames
    check_frame(em, om, len(frames[-1][0]), "side stream")


def test_eager_frames_and_edits_on_a_caller_stream(oracle_mod):
    """E with input_pointcloud of device clouds"""
    _eager_frames_and_edits_on_a_caller_stream(
        oracle_mod, lambda em, pts, dev, R, t: em.input_pointcloud(dev, XYZ, R, t, 0.02, 0.02))


def test_eager_host_sensor_frames_and_edits_on_a_caller_stream(oracle_mod):
    """E with input_sensors of host clouds: the staged frame too runs after the caller's queued edits"""
    _eager_frames_and_edits_on_a_caller_stream(
        oracle_mod, lambda em, pts, dev, R, t: em.input_sensors([pts], [R], [t], 0.02, 0.02))
