"""GPU: map windows (ElevationMap.get_submaps / emap_get_submaps).  Every window of a batch must be, bit for bit, the same
cells of a full get_maps_with_names_ref export of the same state, for the 6 exported state layers, the normals, plugin
layers (inpaint, min_filter with fill_nan, smooth) and a semantic layer (is_valid has no export, as in the reference);
the window itself must be the one tests/submap_oracle.py computes.  Host output, device output on a side stream and a
CUDA-graph capture of the device-output call; a plugin runs once per call; nothing is written or launched on a
rejected call; the call leaves the map state as it was."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import submap_oracle as SO          # noqa: E402

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
inpainting:
  enable: True
  fill_nan: False
  is_height_layer: True
  layer_name: "inpaint"
  extra_params:
    method: "telea"
"""
STATE = ["elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
         "normal_x", "normal_y", "normal_z"]
PLUGINS = ["inpaint", "min_filter", "smooth"]
NAMES = STATE + PLUGINS + ["feat"]
_MAPS = {}


def _frames(em, W, n_frames, seed):
    from elevation_mapping_cupy_b200 import workloads as wl
    rng = np.random.default_rng(seed)
    for f in range(n_frames):
        pts, R, t = wl.lidar_cloud(seed, f, n_rings=64 if W > 500 else 32, n_az=1250, max_range=0.45 * W * 0.04)
        feat = rng.normal(0, 1, (len(pts), 1)).astype(np.float32)
        em.move_to(t, R)
        em.input_pointcloud(np.concatenate([pts, feat], 1), ["x", "y", "z", "feat"], R, t, 0.02, 0.02)
    return R, t


def _make(W, tmp_dir, seed=3):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    cfg = os.path.join(tmp_dir, "plugin_config.yaml")
    with open(cfg, "w") as f:
        f.write(PLUGIN_YAML)
    em = ElevationMap(core_parameter(W, plugin_config_file=cfg, pointcloud_channel_fusions={"default": "average"}))
    R, t = _frames(em, W, 3, seed)
    em.move_to(np.asarray(t, np.float64) + [0.37, -0.53, 0.0], R)              # a moved centre, off the cell grid
    return em


def _map(W, tmp_path_factory):
    """(map, full export of NAMES) of a W x W map after seeded LiDAR frames and a move_to, made once per W."""
    if W not in _MAPS:
        em = _make(W, str(tmp_path_factory.mktemp(f"submap{W}")))
        full = np.zeros((len(NAMES), W - 2, W - 2), np.float32)
        em.get_maps_with_names_ref(NAMES, full)
        assert np.isfinite(full[0]).sum() > 1000 and np.isnan(full[0]).sum() > 1000
        _MAPS[W] = (em, full)
    return _MAPS[W]


def _requests(em, n, rng):
    """n requests: 2 m x 2 m windows anywhere, mixed sizes (0, 0.5 m, 2 m, half the map, more than the map), windows
    clipped at every edge and corner, and a few outside the map."""
    W, res = em.cell_n, em.resolution
    half = 0.5 * (W - 2) * res
    c = em.center.astype(np.float64)[:2]
    fixed = [(c, (2.0, 2.0)), (c, (half, half)), (c, (0.0, 0.0)), (c, (1e4, 3 * half))]
    for sx in (-1, 0, 1):
        for sy in (-1, 0, 1):
            if sx or sy:
                fixed.append((c + (half - 0.3) * np.array([sx, sy]), (2.0, 2.0)))        # clipped at an edge / corner
    fixed.append((c + (half + 0.5, 0.0), (2.0, 2.0)))                                   # outside: fails
    fixed.append((c + (0.0, -half - 2 * res), (4.0, 4.0)))
    out = fixed[:n]
    while len(out) < n:
        size = rng.choice([0.0, 0.5, 2.0, 2.0, 2.0, half])
        out.append((c + rng.uniform(-1.02 * half, 1.02 * half, 2), (size, size * rng.uniform(0.5, 1.5))))
    return out


def _check(em, full, reqs, res, names=NAMES):
    """Each window: the oracle's window, and its layers bit for bit against the crop of the full export."""
    W, rs = em.cell_n, em.resolution
    c = em.center.astype(np.float64)
    cols = [NAMES.index(nm) for nm in names]
    n_ok = 0
    for (pos, ln), r in zip(reqs, res):
        want, centre = SO.window(W, rs, c, np.array([pos[0], pos[1], ln[0], ln[1]], np.float64))
        assert (int(r["success"]),) + r["index"] + r["size"] == want, (pos, ln, r["index"], r["size"], want)
        assert np.array_equal(r["centre"], np.asarray(centre), equal_nan=True)
        crop = SO.crop(full[cols], want)
        for k, nm in enumerate(names):
            got = np.asarray(r["layers"][nm])
            assert got.shape == (want[3], want[4]), nm
            assert np.array_equal(got.view(np.uint32), crop[k].view(np.uint32)), (nm, pos, ln)
        n_ok += r["success"]
    return n_ok


@pytest.mark.parametrize("W", [202, 1024, 2048])
@pytest.mark.parametrize("n", [1, 16, 1024])
def test_host_output_matches_full_export(W, n, tmp_path_factory):
    em, full = _map(W, tmp_path_factory)
    reqs = _requests(em, n, np.random.default_rng(W + n))
    res = em.get_submaps(reqs, NAMES)
    n_ok = _check(em, full, reqs, res)
    assert n_ok >= (1 if n == 1 else 0.7 * n)
    one = em.get_submap(*reqs[0], ["elevation", "feat"])
    assert np.array_equal(one["layers"]["feat"].view(np.uint32), res[0]["layers"]["feat"].view(np.uint32))


@pytest.mark.parametrize("W", [202, 1024])
def test_device_output_on_a_side_stream(W, tmp_path_factory):
    import torch
    em, full = _map(W, tmp_path_factory)
    reqs = _requests(em, 256, np.random.default_rng(7))
    ref = em.get_submaps(reqs, NAMES)
    total = sum(r["size"][0] * r["size"][1] for r in ref) * len(NAMES)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = torch.full((total + 5,), -7.0, device="cuda")
        torch.cuda._sleep(20_000_000)                  # the fill is still queued when the library's kernel is
        res = em.get_submaps(reqs, NAMES, out=out)
        host = out.cpu().numpy()
    assert all(isinstance(v, torch.Tensor) and v.is_cuda for v in res[0]["layers"].values())
    assert (host[total:] == -7.0).all()
    flat = np.concatenate([ref_w["layers"][nm].reshape(-1) for ref_w in ref for nm in NAMES])
    assert np.array_equal(host[:total].view(np.uint32), flat.view(np.uint32))
    _check(em, full, reqs, [dict(r, layers={k: v.cpu().numpy() for k, v in r["layers"].items()}) for r in res])


def test_graph_capture_of_the_device_call(tmp_path_factory):
    import torch
    em, full = _map(202, tmp_path_factory)
    names = STATE + ["feat"]
    reqs = _requests(em, 64, np.random.default_rng(5))
    total = sum(r["size"][0] * r["size"][1] for r in em.get_submaps(reqs, names)) * len(names)
    s = torch.cuda.Stream()
    em.set_stream(s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            out = torch.full((total,), -7.0, device="cuda")
            em.get_submaps(reqs, names, out=out)                                 # warm-up, outside the capture
            want = out.clone()
            out.fill_(-7.0)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        launches = em.launch_count()
        with torch.cuda.graph(g, stream=s):
            res = em.get_submaps(reqs, names, out=out)
        assert em.launch_count() == launches + 1
        s.synchronize()
        assert (out.cpu().numpy() == -7.0).all()                                 # captured, not run
        other = torch.zeros_like(out)                      # an eager call with other windows between capture and replay
        em.get_submaps(_requests(em, 3, np.random.default_rng(9)), ["variance"], out=other)
        s.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), want.view(torch.int32))
        _check(em, full, reqs, [dict(r, layers={k: v.cpu().numpy() for k, v in r["layers"].items()}) for r in res],
               names)
    finally:
        em.set_stream(None)


def test_plugins_run_once_per_call(tmp_path_factory):
    em, full = _map(202, tmp_path_factory)
    calls = []
    pm = em.plugin_manager
    orig = pm.update_with_name
    pm.update_with_name = lambda name, *a, **k: (calls.append(name), orig(name, *a, **k))[1]
    try:
        reqs = _requests(em, 16, np.random.default_rng(2))
        res = em.get_submaps(reqs, NAMES)
        assert sorted(calls) == sorted(PLUGINS)
        calls.clear()
        em.get_submaps(reqs[:1], ["elevation", "feat"])
        assert calls == []
    finally:
        pm.update_with_name = orig
    _check(em, full, reqs, res)


def test_rejected_calls_write_and_launch_nothing(tmp_path_factory):
    em, _ = _map(202, tmp_path_factory)
    L, h = em._L, em._h
    out = np.full(4096, -7.0, np.float32)
    with pytest.raises(KeyError):
        em.get_submaps([(em.center[:2], (1.0, 1.0))], ["elevation", "no_such_layer"], out=out)
    assert (out == -7.0).all()
    c = em.center.astype(np.float64)
    win = np.array([[c[0], c[1], 0.4, 0.4], [c[0] + 1, c[1], 0.0, 0.2]], np.float64)
    want = [SO.window(202, em.resolution, c, w)[0] for w in win]
    need = sum(w[3] * w[4] for w in want)
    names = (C.c_char_p * 2)(b"elevation", b"variance")
    info = np.full((2, 5), -7, np.int32)
    cen = np.full((2, 2), -7.0)
    p = lambda a: a.ctypes.data

    def call(w=win, nw=2, nl=2, nm=names, o=out, size=2 * need, i=info):
        return L.emap_get_submaps(h, nw, None if w is None else p(w), nl, nm, None, None, None if o is None else p(o),
                                  0, size, None if i is None else p(i), p(cen))

    launches = em.launch_count()
    bad_len = win.copy(); bad_len[1, 3] = -0.1
    nan_len = win.copy(); nan_len[0, 2] = np.nan
    inf_len = win.copy(); inf_len[0, 3] = np.inf
    unknown = (C.c_char_p * 2)(b"elevation", b"no_such_layer")
    is_valid = (C.c_char_p * 2)(b"elevation", b"is_valid")
    many = (C.c_char_p * 25)(*([b"elevation"] * 25))
    big = np.zeros((1025, 4)); big[:, :2] = c[:2]
    for kw in (dict(w=None), dict(o=None), dict(i=None), dict(nm=None), dict(nw=0), dict(w=big, nw=1025),
               dict(nl=0), dict(nl=25, nm=many), dict(w=bad_len), dict(w=nan_len), dict(w=inf_len), dict(nm=unknown),
               dict(nm=is_valid), dict(size=2 * need - 1)):
        assert call(**kw) == -1, kw
        assert (out == -7.0).all() and (info == -7).all() and (cen == -7.0).all(), kw
    assert em.launch_count() == launches
    assert call() == 0
    assert em.launch_count() == launches + 1
    assert [tuple(i) for i in info] == want and want[0][3] >= 10 and want[1][3] == 1
    assert (out[2 * need:] == -7.0).all() and not (out[:2 * need] == -7.0).any()


def test_the_call_leaves_the_state_as_it_was(tmp_path):
    """Two maps fed the same frames; one answers submap requests (plugins included) between them.  The next frame gives
    both the same state, and the same plugin layers."""
    a, b = _make(202, str(tmp_path)), _make(202, str(tmp_path))
    reqs = _requests(a, 64, np.random.default_rng(4))
    a.get_submaps(reqs, NAMES)
    _frames(a, 202, 1, 11)
    _frames(b, 202, 1, 11)
    sa, na = a.get_state()
    sb, nb = b.get_state()
    assert np.array_equal(sa.view(np.uint32), sb.view(np.uint32)) and np.array_equal(na.view(np.uint32), nb.view(np.uint32))
    fa = np.zeros((len(NAMES), 200, 200), np.float32)
    fb = np.zeros_like(fa)
    a.get_maps_with_names_ref(NAMES, fa)
    b.get_maps_with_names_ref(NAMES, fb)
    assert np.array_equal(fa.view(np.uint32), fb.view(np.uint32))
