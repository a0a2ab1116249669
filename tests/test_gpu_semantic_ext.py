"""The class_bayesian, bayesian_inference and class_max point-cloud fusions on the device, against the NumPy definition
(oracle/semantic_ext.py, DESIGN §4d) over multi-frame sequences with move_to and clear between frames: every semantic
layer, every variance plane and id_max bit for bit, all six kinds in one cloud, f32 / f64 rows, host / device clouds and
two-sensor frames.  The per-cell bayesian_inference update is also checked against the reference's own kernel compiled
for sm_90a (oracle/build_ref_semantic.py) given the same sums."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSIONS = {"avg": "average", "ca": "class_average", "rgb": "color", "cb.*": "class_bayesian", "bi.*": "bayesian_inference",
           "cm.*": "class_max"}
CHANNELS = ["x", "y", "z", "avg", "ca", "rgb", "cb1", "cb2", "cb3", "bi1", "bi2", "cm1", "cm2", "cm3"]
IDS = np.array([0, 3, 7, 11, 200, 4095, 65535], np.int64)


def _param(W):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(W)
    p.pointcloud_channel_fusions = dict(FUSIONS)
    return p


def _features(rng, n, f):
    """avg, ca, rgb, cb1..3, bi1..2, cm1..3 columns; some negative / NaN class_bayesian values, fp16 probabilities with
    ties, zeros, negatives and (rarely) NaN / inf for class_max."""
    from oracle import semantic_ext as X
    avg = rng.random(n, dtype=np.float32) * 4 - 2
    ca = rng.random(n, dtype=np.float32)
    rgb = rng.integers(0, 1 << 24, n).astype(np.uint32).view(np.float32)
    cb = rng.random((n, 3), dtype=np.float32)
    cb[rng.random((n, 3)) < 0.1] *= -1
    cb[rng.random((n, 3)) < 0.02] = np.nan
    bi = rng.random((n, 2), dtype=np.float32) * 2 - 0.5
    prob = rng.choice(np.array([0.0, 0.125, 0.25, 0.5, 0.75, 1.0, -0.25], np.float32), (n, 3))
    prob = np.where(rng.random((n, 3)) < 0.5, rng.random((n, 3), dtype=np.float32), prob).astype(np.float32)
    if f == 2:
        prob[rng.random((n, 3)) < 0.002] = np.nan
        prob[rng.random((n, 3)) < 0.002] = np.inf
    ids = rng.choice(IDS[: 4 + f % 4], (n, 3))
    cm = X.encode_max(prob, ids)
    return np.concatenate([avg[:, None], ca[:, None], rgb[:, None], cb, bi, cm], 1).astype(np.float32)


def _cloud(f, n, sensor=0):
    from elevation_mapping_cupy_b200 import workloads as wl
    rng = np.random.default_rng(100 + 7 * f + sensor)
    pts, R, t = wl.uniform_cloud(sensor, f, n=n, half_extent=3.0)
    pts = pts.copy()
    pts[rng.random(n) < 0.01, rng.integers(0, 3)] = np.nan          # dropped rows (EM.py:458)
    t = (t + np.array([0.3 * f, -0.2 * f, 0.0], np.float32)).astype(np.float32)
    pts[:, :2] += t[:2]
    return np.ascontiguousarray(np.concatenate([pts, _features(rng, n, f)], 1)), R, t


class _OracleSemantic:
    """The semantic planes of SemanticMap in NumPy, driven by the same calls."""

    def __init__(self, p, sm):
        W = p.cell_n
        self.W, self.p = W, p
        self.names = list(sm.layer_names)
        L = len(self.names)
        self.sem = np.zeros((L, W, W), np.float32)
        self.sigma = np.ones((L, W, W), np.float32)
        self.id_max = np.zeros((3, W, W), np.int32)
        chans = CHANNELS[3:]
        self.kinds = [FUSIONS[next(k for k in FUSIONS if __import__("re").match(f"^{k}$", c))] for c in chans]
        self.layers = [self.names.index(c) for c in chans]

    def frame(self, rows, idx, valid, inside, dropped, cnt):
        from oracle import semantic_ext as X
        X.fuse(self.W, idx, valid, inside, dropped, rows[:, 3:].astype(np.float32), self.kinds, self.layers, self.sem,
               cnt, alpha=float(self.p.average_weight), sigma=self.sigma, id_max=self.id_max)

    def shift(self, sx, sy):
        for a, pad in ((self.sem, 0), (self.sigma, 1), (self.id_max, 0)):
            m = np.roll(a, (sx, sy), (1, 2))
            if sx > 0: m[:, :sx] = pad
            elif sx < 0: m[:, sx:] = pad
            if sy > 0: m[:, :, :sy] = pad
            elif sy < 0: m[:, :, sy:] = pad
            a[...] = m

    def clear(self):
        self.sem[...] = 0
        self.sigma[...] = 1


def _record(om, dropped):
    """The oracle's point record for the non-dropped rows, spread over all rows (dropped rows: not valid)."""
    idx, valid, inside = om.last_point_record
    n = len(dropped)
    I = np.zeros(n, np.int64); V = np.zeros(n, np.uint8); S = np.zeros(n, np.uint8)
    I[~dropped] = idx; V[~dropped] = valid; S[~dropped] = inside
    return I, V, S


def _same(a, b):
    """Bit for bit, except that a NaN's payload is not compared (the device writes 0x7fffffff, x86 keeps its operand's)."""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb])


def _check(em, osm, tag):
    em.synchronize()
    sm = em.semantic_map
    got = sm.semantic_map.cpu().numpy()
    for li, name in enumerate(osm.names):
        a, b = got[li], osm.sem[li]
        assert _same(a, b), (tag, name, int((np.isnan(a) != np.isnan(b)).sum()),
                             int(((a.view(np.uint32) != b.view(np.uint32)) & ~np.isnan(a) & ~np.isnan(b)).sum()))
    sig = sm.variance.cpu().numpy()
    assert _same(sig, osm.sigma), (tag, "variance")
    idm = sm.elements_to_shift["id_max"].cpu().numpy()
    assert np.array_equal(idm, osm.id_max), (tag, "id_max", int((idm != osm.id_max).sum()))


def _sequence(W, check=True):
    """Frames: f32 host, f64 host, f32 device, f64 device, clear, two-sensor host, two-sensor device; move_to each time."""
    import torch
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from oracle import oracle as O
    p = _param(W)
    em = ElevationMap(p)
    om = O.OracleElevationMap(p, nthreads=0)
    osm = None
    n = 12000
    plan = [("f32", "host", 1), ("f64", "host", 1), ("f32", "device", 1), ("f64", "device", 1), ("clear", None, 0),
            ("f32", "host", 2), ("f64", "device", 2), ("f32", "device", 1)]
    for f, (dt, where, n_sensors) in enumerate(plan):
        if dt == "clear":
            em.clear(); om.clear()
            if osm is not None:
                osm.clear()
                if check:
                    _check(em, osm, f"clear {f}")
            continue
        clouds = [_cloud(f, n, s) for s in range(n_sensors)]
        R0, t0 = clouds[0][1], clouds[0][2]
        shift = None
        if em.semantic_map.layer_names:
            px = np.rint((np.asarray(t0, np.float64)[:2] - em.center[:2].astype(np.float64)) / p.resolution).astype(int)
            shift = (-int(px[0]), -int(px[1]))
        em.move_to(t0, R0); om.move_to(t0, R0)
        if osm is not None and shift is not None and shift != (0, 0):
            osm.shift(*shift)
        rows = [c[0].astype(np.float64) if dt == "f64" else c[0] for c in clouds]
        src = [torch.from_numpy(r).cuda() if where == "device" else r for r in rows]
        if n_sensors == 1:
            em.input_pointcloud(src[0], CHANNELS, R0, t0, 0.02, 0.02)
        else:
            em.input_sensors(src, [c[1] for c in clouds], [c[2] for c in clouds], 0.02, 0.02,
                             device_ptrs=where == "device")
        allrows = np.concatenate([c[0] for c in clouds], 0)
        dropped = np.isnan(allrows[:, :3]).any(1)
        om.input_sensors([c[0][~np.isnan(c[0][:, :3]).any(1), :3] for c in clouds], [c[1] for c in clouds],
                         [c[2] for c in clouds], 0.02, 0.02)
        if osm is None:
            osm = _OracleSemantic(p, em.semantic_map)
        idx, valid, inside = _record(om, dropped)
        eidx, evalid, einside = em.get_point_record(len(allrows))
        assert np.array_equal(evalid.astype(bool), valid.astype(bool)) and np.array_equal(einside.astype(bool), inside.astype(bool))
        osm.frame(allrows, idx, valid, inside, dropped, om.counts_fused.reshape(-1))
        if check:
            _check(em, osm, f"frame {f} {dt} {where} x{n_sensors}")
    em.synchronize()
    sm = em.semantic_map
    return (sm.semantic_map.cpu().numpy(), sm.variance.cpu().numpy(), sm.elements_to_shift["id_max"].cpu().numpy())


@pytest.mark.parametrize("W", [130, 202])
def test_all_kinds_match_definition_bit_for_bit(W):
    _sequence(W)


def test_two_runs_bit_identical():
    a = _sequence(202, check=False)
    b = _sequence(202, check=False)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y)


def test_bayesian_update_matches_reference_gpu_kernel():
    """Given the same sums, the engine's per-cell bayesian_inference update equals the reference's
    bayesian_inference_kernel built by nvcc for sm_90a, bit for bit (layer and variance)."""
    import torch
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from oracle import build_ref_semantic as BS, semantic_ext as X
    from oracle import oracle as O
    from oracle.configs import REF_CONFIGS
    W = 202
    lib = C.CDLL(BS.build(REF_CONFIGS["core202"], tag="core202", gpu=True))
    p = _param(W)
    p.pointcloud_channel_fusions = {"bi.*": "bayesian_inference"}
    chans = ["x", "y", "z", "bi1", "bi2"]
    em = ElevationMap(p)
    om = O.OracleElevationMap(p, nthreads=0)
    for f in range(3):
        rng = np.random.default_rng(40 + f)
        pts, R, t = _cloud(f, 15000)[0][:, :3], np.eye(3, dtype=np.float32), np.array([0, 0, 1.2], np.float32)
        pts = pts[~np.isnan(pts).any(1)]
        feats = (rng.random((len(pts), 2), dtype=np.float32) * 3 - 1).astype(np.float32)
        rows = np.ascontiguousarray(np.concatenate([pts, feats], 1))
        em.synchronize()
        sm = em.semantic_map
        before = None if sm.semantic_map is None else (sm.semantic_map.clone(), sm.variance.clone())
        em.input_pointcloud(rows, chans, R, t, 0.02, 0.02)
        om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        em.synchronize()
        if before is None:
            continue            # first frame: starts from zero layers and unit variance like every later one
        idx, valid, inside = om.last_point_record
        sel = (valid > 0) & (inside > 0)
        L = len(sm.layer_names)
        sums = np.zeros((2, W, W), np.float32)
        for k in range(2):
            sums[k] = X.unfix32(X.cell_sum_fix(idx[sel].astype(np.int64), X.fix32(feats[sel, k]), W * W)).reshape(W, W)
        new_el = np.zeros((7, W, W), np.float32); new_el[2] = om.counts_fused
        sem_r, sig_r = before[0].contiguous(), before[1].contiguous()
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        pcl_chan, map_lay = d(np.array([3, 4], np.int32)), d(np.array([sm.layer_names.index("bi1"), sm.layer_names.index("bi2")], np.int32))
        dims = d(np.array([5, 2], np.int32))
        nel, sum_mean = d(new_el), d(sums)
        ptr = lambda x: C.c_void_p(x.data_ptr())
        torch.cuda.synchronize()
        rc = lib.ref_sem_bayesian_inference(C.c_longlong(W * W * 2), ptr(pcl_chan), ptr(map_lay), ptr(dims), ptr(nel),
                                            ptr(sig_r), ptr(sum_mean), ptr(sem_r), C.c_void_p(0))
        assert rc == 0
        torch.cuda.synchronize()
        assert L >= 2
        for name in ("bi1", "bi2"):
            li = sm.layer_names.index(name)
            assert torch.equal(sm.semantic_map[li].view(torch.int32), sem_r[li].view(torch.int32)), (f, name)
            assert torch.equal(sm.variance[li].view(torch.int32), sig_r[li].view(torch.int32)), (f, name, "variance")


def test_configure_ext_rejections():
    import torch
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    W = 130
    em = ElevationMap(_param(W))
    L = em._L
    sem = torch.zeros((2, W, W), device="cuda")
    one = lambda v: (C.c_int32 * 1)(v)
    ptr = C.c_void_p(sem.data_ptr())
    # the original entry point still takes kinds 0..2 only
    assert L.emap_semantic_configure(em._h, 1, one(3), one(3), one(0), ptr, 2, 0.5) != 0
    # bayesian_inference needs the variance planes, class_max id_max with a plane per channel
    assert L.emap_semantic_configure_ext(em._h, 1, one(3), one(4), one(0), ptr, 2, 0.5, None, None, 0) != 0
    assert L.emap_semantic_configure_ext(em._h, 1, one(3), one(5), one(0), ptr, 2, 0.5, None, None, 0) != 0
    idm = torch.zeros((1, W, W), dtype=torch.int32, device="cuda")
    assert L.emap_semantic_configure_ext(em._h, 1, one(3), one(5), one(0), ptr, 2, 0.5, None, C.c_void_p(idm.data_ptr()), 0) != 0
    assert L.emap_semantic_configure_ext(em._h, 1, one(3), one(6), one(0), ptr, 2, 0.5, None, None, 0) != 0
    assert L.emap_semantic_configure_ext(em._h, 1, one(3), one(5), one(0), ptr, 2, 0.5, None, C.c_void_p(idm.data_ptr()), 1) == 0
    assert L.emap_semantic_configure_ext(em._h, 1, one(3), one(3), one(0), ptr, 2, 0.5, None, None, 0) == 0
    assert L.emap_semantic_configure_ext(em._h, 0, None, None, None, None, 0, 0.0, None, None, 0) == 0
