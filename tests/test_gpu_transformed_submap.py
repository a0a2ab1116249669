"""GPU: windows in the requester's frame (ElevationMap.get_transformed_submaps / emap_get_transformed_submaps).  Every
new map of a batch must be, bit for bit, what tests/transformed_submap_oracle.py computes from a full
get_maps_with_names_ref export of the same state, for the state layers, the normals, normal_color, plugin layers and a
semantic layer, at 202², 1024² and 2048² over the oracle's transforms.  Host and device output, a CUDA-graph replay
after calls with other transforms, the identity transform against get_submaps, every rejection for its own reason, and
get_submaps' launch count."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import transformed_submap_oracle as TO          # noqa: E402

pytestmark = pytest.mark.gpu

PLUGIN_YAML = """
min_filter:
  enable: True
  fill_nan: True
  is_height_layer: True
  layer_name: "min_filter"
  extra_params:
    dilation_size: 1
    iteration_n: 30
smooth_filter:
  enable: True
  fill_nan: False
  is_height_layer: True
  layer_name: "smooth"
  extra_params:
    input_layer_name: "min_filter"
"""
NAMES = ["elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound", "normal_x", "normal_y",
         "normal_z", "normal_color", "min_filter", "smooth", "feat"]
_MAPS = {}


def _make(W, tmp_dir, seed=3):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    cfg = os.path.join(tmp_dir, "plugin_config.yaml")
    with open(cfg, "w") as f:
        f.write(PLUGIN_YAML)
    em = ElevationMap(core_parameter(W, plugin_config_file=cfg, pointcloud_channel_fusions={"default": "average"}))
    rng = np.random.default_rng(seed)
    for fr in range(3):
        pts, R, t = wl.lidar_cloud(seed, fr, n_rings=64 if W > 500 else 32, n_az=1250, max_range=0.45 * W * 0.04)
        feat = rng.normal(0, 1, (len(pts), 1)).astype(np.float32)
        em.move_to(t, R)
        em.input_pointcloud(np.concatenate([pts, feat], 1), ["x", "y", "z", "feat"], R, t, 0.02, 0.02)
    em.move_to(np.asarray(t, np.float64) + [0.37, -0.53, 0.0], R)              # a moved centre, off the cell grid
    return em


def _map(W, tmp_path_factory):
    """(map, full export of NAMES) of a W x W map after seeded LiDAR frames and a move_to, made once per W."""
    if W not in _MAPS:
        em = _make(W, str(tmp_path_factory.mktemp(f"tsubmap{W}")))
        full = np.zeros((len(NAMES), W - 2, W - 2), np.float32)
        em.get_maps_with_names_ref(NAMES, full)
        assert np.isfinite(full[0]).sum() > 1000 and np.isnan(full[0]).sum() > 1000
        _MAPS[W] = (em, full)
    return _MAPS[W]


def _requests(em, tfs, rng, big=False):
    """Per transform: windows of 2 m around the centre and elsewhere, one cell, one clipped at a corner, one outside
    the map, and (big) half the map; positions given in the transform's frame."""
    W, res = em.cell_n, em.resolution
    half = 0.5 * (W - 2) * res
    c = em.center.astype(np.float64)[:2]
    out = []
    for T in tfs:
        R, t = np.asarray(T[:9]).reshape(3, 3), np.asarray(T[9:])
        pts = [(c, (2.0, 2.0)), (c + rng.uniform(-0.8 * half, 0.8 * half, 2), (2.0, 1.3)),
               (c + rng.uniform(-0.5 * half, 0.5 * half, 2), (0.0, 0.0)), (c + (half - 0.2, -half + 0.3), (2.0, 2.0)),
               (c + (half + 0.5, 0.0), (2.0, 2.0))]
        if big:
            pts.append((c, (half, half)))
        for p, ln in pts:
            q = R @ np.array([p[0], p[1], 0.0]) + t
            out.append(((q[0], q[1]), ln, (R, t)))
    return out


def _check(em, full, reqs, res, sample_ratio, names=NAMES):
    """Each request against the oracle: success, size, centre and length exactly, every layer bit for bit."""
    W, rs = em.cell_n, em.resolution
    c = em.center.astype(np.float64)
    n_ok = 0
    for (pos, ln, T), r in zip(reqs, res):
        g, want = TO.transformed_submap(full, NAMES, W, rs, c, (pos[0], pos[1], ln[0], ln[1]), T, sample_ratio)
        assert r["success"] == bool(g["win"][0]) and r["size"] == g["size"], (pos, ln, r["size"], g)
        assert np.array_equal(np.concatenate([r["frame_centre"], r["length"]]), np.array(g["pos"] + g["len"]),
                              equal_nan=True)
        for nm in names:
            got = np.asarray(r["layers"][nm])
            assert got.shape == g["size"], nm
            assert np.array_equal(got.view(np.uint32), want[nm].view(np.uint32)), (nm, pos, ln, T)
        n_ok += r["success"]
    return n_ok


@pytest.mark.parametrize("W", [202, 1024, 2048])
def test_host_output_matches_oracle(W, tmp_path_factory):
    em, full = _map(W, tmp_path_factory)
    tfs = TO.transforms(em.resolution)
    reqs = _requests(em, tfs, np.random.default_rng(W), big=W <= 1024)
    res = em.get_transformed_submaps(reqs, NAMES)
    assert _check(em, full, reqs, res, 0.0) >= 0.7 * len(reqs)
    one = em.get_transformed_submap(*reqs[1][:2], ["feat", "elevation"], reqs[1][2])
    assert np.array_equal(one["layers"]["feat"].view(np.uint32), res[1]["layers"]["feat"].view(np.uint32))


@pytest.mark.parametrize("W", [202, 1024])
@pytest.mark.parametrize("sample_ratio", [0.5, 1.0])
def test_sample_ratio_matches_oracle(W, sample_ratio, tmp_path_factory):
    em, full = _map(W, tmp_path_factory)
    tfs = TO.transforms(em.resolution)
    reqs = _requests(em, tfs, np.random.default_rng(W + 1))
    res = em.get_transformed_submaps(reqs, NAMES, sample_ratio=sample_ratio)
    assert _check(em, full, reqs, res, sample_ratio) >= 0.7 * len(reqs)


def test_transform_forms_and_many_windows(tmp_path_factory):
    """A 4 x 4 matrix and an (R, t) pair give the same result; 400 windows (three launches' worth) match the oracle."""
    em, full = _map(202, tmp_path_factory)
    tfs = TO.transforms(em.resolution)
    reqs = (_requests(em, tfs, np.random.default_rng(11)) * 6)[:400]
    c = em.center.astype(np.float64)
    pos, ln, (R, t) = next(r for r in reqs if np.isfinite(TO.transformed_submap(
        full, NAMES, em.cell_n, em.resolution, c, tuple(r[0]) + tuple(r[1]), r[2])[1]["elevation"]).sum() > 100)
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = R, t
    a = em.get_transformed_submap(pos, ln, ["elevation", "feat"], M)
    b = em.get_transformed_submap(pos, ln, ["elevation", "feat"], (R, t))
    assert a["success"] and np.isfinite(a["layers"]["elevation"]).sum() > 100
    for nm in ("elevation", "feat"):
        assert np.array_equal(a["layers"][nm].view(np.uint32), b["layers"][nm].view(np.uint32))
    launches = em.launch_count()
    res = em.get_transformed_submaps(reqs, ["elevation", "feat"])
    n_win = sum(r["success"] and r["size"][0] * r["size"][1] > 0 for r in res)
    assert n_win > 256 and em.launch_count() - launches == 3 * -(-n_win // 128)      # 3 per 128 windows with cells
    _check(em, full, reqs, res, 0.0, ["elevation", "feat"])


def test_device_output_and_graph_replay(tmp_path_factory):
    import torch
    em, full = _map(202, tmp_path_factory)
    names = ["elevation", "variance", "normal_z", "normal_color", "feat"]
    tfs = TO.transforms(em.resolution)
    reqs = _requests(em, tfs[8:12], np.random.default_rng(5))
    ref = em.get_transformed_submaps(reqs, names)
    total = sum(r["size"][0] * r["size"][1] for r in ref) * len(names)
    s = torch.cuda.Stream()
    em.set_stream(s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            out = torch.full((total + 3,), -7.0, device="cuda")
            torch.cuda._sleep(20_000_000)                  # the fill is still queued when the library's kernels are
            res = em.get_transformed_submaps(reqs, names, out=out)
            host = out.cpu().numpy()
        assert all(isinstance(v, torch.Tensor) and v.is_cuda for v in res[0]["layers"].values())
        assert (host[total:] == -7.0).all()
        flat = np.concatenate([r["layers"][nm].reshape(-1) for r in ref for nm in names])
        assert np.array_equal(host[:total].view(np.uint32), flat.view(np.uint32))
        want = out.clone()
        with torch.cuda.stream(s):
            out.fill_(-7.0)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        launches = em.launch_count()
        with torch.cuda.graph(g, stream=s):
            em.get_transformed_submaps(reqs, names, out=out)
        assert em.launch_count() == launches + 3
        s.synchronize()
        assert (out.cpu().numpy()[:total] == -7.0).all()                       # captured, not run
        other_reqs = _requests(em, tfs[2:4], np.random.default_rng(9))[:4]       # other transforms, fewer cells
        other = torch.zeros(total, device="cuda")
        with torch.cuda.stream(s):
            em.get_transformed_submaps(other_reqs, ["variance"], out=other, sample_ratio=0.5)
        s.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), want.view(torch.int32))
        g.replay()                                              # the keys were reset: a second replay is the same
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), want.view(torch.int32))
    finally:
        em.set_stream(None)
    _check(em, full, reqs, ref, 0.0, names)


@pytest.mark.parametrize("W", [202, 1024])
def test_identity_is_get_submaps(W, tmp_path_factory):
    """The identity transform gives get_submaps' windows: every layer bit for bit where the exported elevation is a
    number, NaN in every layer where it is not (grid_map skips those cells)."""
    em, _ = _map(W, tmp_path_factory)
    T = (np.eye(3), np.zeros(3))
    c = em.center.astype(np.float64)[:2]
    rng = np.random.default_rng(W)
    half = 0.5 * (W - 2) * em.resolution
    pairs = [(c + rng.uniform(-half, half, 2), tuple(rng.choice([0.0, 0.5, 2.0, half], 2))) for _ in range(40)]
    sub = em.get_submaps(pairs, NAMES)
    tsub = em.get_transformed_submaps([(p, ln, T) for p, ln in pairs], NAMES)
    n_ok = 0
    for a, b in zip(sub, tsub):
        assert a["success"] == b["success"] and a["size"] == b["size"]
        assert not a["success"] or np.allclose(b["frame_centre"], a["centre"], rtol=0, atol=1e-9)
        nan = np.isnan(a["layers"]["elevation"])
        for nm in NAMES:
            want = a["layers"][nm].copy()
            want[nan] = np.nan
            assert np.array_equal(b["layers"][nm].view(np.uint32), want.view(np.uint32)), nm
        n_ok += a["success"]
    assert n_ok > 30


def test_get_submaps_launches_one_kernel(tmp_path_factory):
    em, _ = _map(202, tmp_path_factory)
    launches = em.launch_count()
    em.get_submaps([(em.center[:2], (2.0, 2.0))], ["elevation", "variance"])
    assert em.launch_count() == launches + 1


def test_rejections_write_and_launch_nothing(tmp_path_factory):
    em, _ = _map(202, tmp_path_factory)
    L, h = em._L, em._h
    out = np.full(1 << 16, -7.0, np.float32)
    c = em.center.astype(np.float64)
    win = np.array([[c[0], c[1], 0.4, 0.4], [c[0] + 1, c[1], 0.0, 0.2]], np.float64)
    tf = np.stack([TO.iso(np.eye(3), (0, 0, 0)), TO.transforms(em.resolution)[8]])
    win[1, :2] = (tf[1, :9].reshape(3, 3) @ [c[0] + 1, c[1], 0.0] + tf[1, 9:])[:2]        # in the map, seen from T
    names = (C.c_char_p * 2)(b"elevation", b"variance")
    info = np.full((2, 3), -7, np.int32)
    geo = np.full((2, 4), -7.0)
    p = lambda a: None if a is None else a.ctypes.data
    need = 2 * sum(int(TO.geometry(202, em.resolution, c, win[w], tf[w])["size"][0]
                       * TO.geometry(202, em.resolution, c, win[w], tf[w])["size"][1]) for w in range(2))

    def call(w=win, t=tf, sr=0.0, nw=2, nl=2, nm=names, o=out, size=need, i=info, g=geo):
        return L.emap_get_transformed_submaps(h, nw, p(w), p(t), sr, nl, nm, None, None, p(o), 0, size, p(i), p(g))

    def bad_tf(k, v):
        b = tf.copy()
        b[1, k] = v
        return b

    many = (C.c_char_p * 25)(*([b"elevation"] * 25))
    big = np.zeros((1025, 4)); big[:, :2] = c[:2]
    bad_len = win.copy(); bad_len[1, 3] = -0.1
    cases = [(dict(w=None), "null argument"), (dict(t=None), "null argument"), (dict(o=None), "null argument"),
             (dict(i=None), "null argument"), (dict(g=None), "null argument"), (dict(nm=None), "null argument"),
             (dict(nw=0), "windows required"), (dict(w=big, t=np.repeat(tf[:1], 1025, 0), nw=1025), "windows required"),
             (dict(nl=0), "layers required"), (dict(nl=25, nm=many), "layers required"),
             (dict(w=bad_len), "lengths must be finite"),
             (dict(t=bad_tf(0, np.nan)), "orthonormal"), (dict(t=bad_tf(10, np.inf)), "orthonormal"),
             (dict(t=bad_tf(1, 0.01)), "orthonormal"), (dict(sr=-0.5), "sample_ratio"),
             (dict(sr=float("nan")), "sample_ratio"), (dict(sr=float("inf")), "sample_ratio"),
             (dict(nm=(C.c_char_p * 2)(b"elevation", b"no_such_layer")), "no_such_layer is not in the map"),
             (dict(size=need - 1), "out_floats is below")]
    launches = em.launch_count()
    for kw, why in cases:
        assert call(**kw) == -1, kw
        assert why in L.emap_last_error(h).decode(), (kw, L.emap_last_error(h))
        assert (out == -7.0).all() and (info == -7).all() and (geo == -7.0).all(), kw
    assert em.launch_count() == launches
    assert call() == 0
    assert em.launch_count() == launches + 3
    assert (out[need:] == -7.0).all() and info[0, 0] == 1 and info[1, 0] == 1
