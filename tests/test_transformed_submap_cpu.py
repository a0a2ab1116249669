"""Windows in the requester's frame without a GPU: the library's host geometry (emap_transformed_submap_windows, the
arithmetic every emap_get_transformed_submaps call runs) against tests/transformed_submap_oracle.py; the oracle's index
rule on cell boundaries; and the order-free rule the device uses against grid_map's sequential loop."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import transformed_submap_oracle as TO          # noqa: E402


def _lib():
    from elevation_mapping_cupy_b200 import _lib
    return _lib.load()


def _lib_geometry(cell_n, res, center, reqs, tfs):
    L = _lib()
    req = np.ascontiguousarray(np.asarray(reqs, np.float64).reshape(-1, 4))
    tf = np.ascontiguousarray(np.asarray(tfs, np.float64).reshape(-1, 12))
    c = np.ascontiguousarray(np.asarray(center, np.float64)[:2])
    info = np.full((len(req), 3), -7, np.int32)
    geo = np.full((len(req), 4), -7.0)
    rc = L.emap_transformed_submap_windows(cell_n, res, c.ctypes.data, len(req), req.ctypes.data, tf.ctypes.data,
                                           info.ctypes.data, geo.ctypes.data)
    return rc, info, geo


def _requests(cell_n, res, center, T, rng):
    """Requests in the frame of T: centred, at every border and corner of the map, outside it, on cell boundaries and
    random, of mixed lengths."""
    half = 0.5 * (cell_n - 2) * res
    R, t = np.asarray(T[:9]).reshape(3, 3), np.asarray(T[9:])
    pts = [(0.0, 0.0), (half - 0.3, 0.0), (-half + 0.3, 0.1), (0.2, half - 0.1), (half - res, -half + res),
           (half * 1.02, 0.0), (0.0, -half * 1.3), (0.5 * res, 1.5 * res), (3 * res, -4 * res)]
    pts += [tuple(rng.uniform(-1.05 * half, 1.05 * half, 2)) for _ in range(40)]
    out = []
    for k, (x, y) in enumerate(pts):
        q = R @ np.array([center[0] + x, center[1] + y, 0.0]) + t           # the map-frame point in the request frame
        ln = [(2.0, 2.0), (0.0, 0.0), (0.5, 1.3), (2 * half, 2 * half), (4 * res, 0.0)][k % 5]
        out.append((q[0], q[1], ln[0], ln[1]))
    return out


@pytest.mark.parametrize("cell_n,res,center", [(202, 0.04, (0.0, 0.0)), (203, 0.04, (0.37, -0.53)),
                                               (1024, 0.04, (12.34, -5.678)), (131, 0.1, (-3.21, 7.0))])
def test_host_geometry_matches_oracle(cell_n, res, center):
    """Every request and transform: success and size exactly, the new centre and length bit for bit."""
    c = np.asarray(center, np.float32).astype(np.float64)
    rng = np.random.default_rng(cell_n)
    n_ok = n_fail = n_border = 0
    for T in TO.transforms(res):
        reqs = _requests(cell_n, res, c, T, rng)
        rc, info, geo = _lib_geometry(cell_n, res, c, reqs, [T] * len(reqs))
        assert rc == 0
        for w, r in enumerate(reqs):
            g = TO.geometry(cell_n, res, c, r, T)
            assert tuple(info[w]) == (g["win"][0],) + g["size"], (w, r, info[w], g)
            assert np.array_equal(geo[w], np.array(g["pos"] + g["len"]), equal_nan=True), (w, r, geo[w], g)
            n_ok += g["win"][0]
            n_fail += not g["win"][0]
            ok, r0, c0, rows, cols = g["win"]
            n_border += bool(ok) and (r0 == 0 or c0 == 0 or r0 + rows == cell_n - 2 or c0 + cols == cell_n - 2)
    assert n_ok > 200 and n_fail > 20 and n_border > 20


def test_right_angle_geometry():
    """A 10 x 10 map of 1 m cells at the origin (cell_n 12), a 3 x 3 window at (0.5, 0.5): yaw 90 degrees with an
    integer translation carries it to a 3 x 3 map whose centre is R c + t exactly."""
    T = TO.iso([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]], (2.0, -3.0, 0.0))
    # T^-1 (px, py) = (0.5, 0.5): px = -0.5 + 2, py = 0.5 - 3
    rc, info, geo = _lib_geometry(12, 1.0, (0.0, 0.0), [(1.5, -2.5, 2.0, 2.0)], [T])
    assert rc == 0
    assert tuple(info[0]) == (1, 3, 3)
    assert tuple(geo[0]) == (1.5, -2.5, 3.0, 3.0)


def test_index_rule_on_cell_boundaries():
    """The oracle's (and the device's) index rule at a binary resolution, centre and length, for every cell boundary
    and cell centre: row k holds (pos + L/2 - (k + 1) res, pos + L/2 - k res]; the +x edge is inside (row 0), the -x
    edge outside; likewise for columns."""
    res = 0.25
    g = {"pos": (1.5, -0.75), "len": (10 * res, 7 * res), "size": (10, 7)}
    for a in range(2):
        top = g["pos"][a] + 0.5 * g["len"][a]
        for m in range(-4, 2 * g["size"][a] + 5):
            q = top - m * 0.5 * res
            other = g["pos"][1 - a]
            ij = TO.target(g, res, *((q, other) if a == 0 else (other, q)))
            if m < 0 or m >= 2 * g["size"][a]:
                assert ij is None, (a, m)
            else:
                assert ij is not None and ij[a] == m // 2, (a, m, ij)


def _window_layers(rows, cols, rng, kind):
    """Exported window layers: "elevation" of an adversarial kind and a "tag" layer naming each source cell."""
    if kind == "equal":
        h = np.full((rows, cols), 0.75, np.float32)
    elif kind == "straddle":
        h = (0.3 + rng.integers(-3, 4, (rows, cols)) * 2.0 ** -24).astype(np.float32)
    else:
        h = rng.normal(0.0, 0.05, (rows, cols)).astype(np.float32)
    h[rng.random((rows, cols)) < 0.1] = np.nan
    tag = np.arange(rows * cols, dtype=np.float32).reshape(rows, cols)
    return {"elevation": h, "tag": tag}


@pytest.mark.parametrize("kind", ["random", "equal", "straddle"])
@pytest.mark.parametrize("sample_ratio", [0.0, 0.5, 1.0])
def test_parallel_rule_equals_the_loop(kind, sample_ratio):
    """The order-free rule (TO.parallel) gives exactly grid_map's sequential loop (TO.sequential) for every
    transform, on windows with equal elevations, elevations a few fp32 ulps apart and random ones; the pitched
    transforms put many cells into one target."""
    res, cell_n, c = 0.1, 40, (0.0, 0.0)
    rng = np.random.default_rng(len(kind) * 10 + int(sample_ratio * 2))
    n_multi = most = 0
    for T in TO.transforms(res):
        for length in [(1.3, 0.9), (2.5, 1.7)]:
            g = TO.geometry(cell_n, res, c, (0.0, 0.0) + length, T)
            assert g["win"][0]
            layers = _window_layers(g["win"][3], g["win"][4], rng, kind)
            want = TO.sequential(layers, g, T, res, sample_ratio)
            got = TO.parallel(layers, g, T, res, sample_ratio)
            for k in layers:
                assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), (k, T, length)
            cell = TO.samples(layers, g, T, res, sample_ratio)[3]
            if len(cell):
                n_multi += int((np.bincount(cell) > 2).sum())
                most = max(most, int(np.bincount(cell).max()))
    assert n_multi >= 10 and most >= 6


@pytest.mark.parametrize("cell_n,res,center", [(64, 0.04, (0.0, 0.0)), (65, 0.05, (0.37, -0.53)),
                                               (130, 0.1, (-3.21, 7.0))])
def test_identity_is_the_window(cell_n, res, center):
    """With the identity transform every cell lands on itself: the new map is the map-frame window, layer for layer."""
    c = np.asarray(center, np.float32).astype(np.float64)
    rng = np.random.default_rng(cell_n)
    full = rng.normal(0.0, 1.0, (2, cell_n - 2, cell_n - 2)).astype(np.float32)
    full[0][rng.random((cell_n - 2, cell_n - 2)) < 0.2] = np.nan
    T = TO.iso(np.eye(3), (0.0, 0.0, 0.0))
    half = 0.5 * (cell_n - 2) * res
    n_ok = 0
    for _ in range(100):
        req = (c[0] + rng.uniform(-half, half), c[1] + rng.uniform(-half, half)) + tuple(rng.choice([0.0, 0.3, 1.0, 9.0], 2))
        g, got = TO.transformed_submap(full, ["elevation", "tag"], cell_n, res, c, req, T)
        if not g["win"][0]:
            continue
        n_ok += 1
        crop = full[:, g["win"][1]:g["win"][1] + g["win"][3], g["win"][2]:g["win"][2] + g["win"][4]]
        assert g["size"] == crop.shape[1:]
        for k, nm in enumerate(["elevation", "tag"]):
            want = crop[k].copy()
            if nm == "tag":
                want[np.isnan(crop[0])] = np.nan
            assert np.array_equal(got[nm].view(np.uint32), want.view(np.uint32)), (req, nm)
    assert n_ok > 80


def test_rule_on_random_sample_sets():
    """The rule against the sequential update on 5000 random sample sets that straddle fp32 rounding."""
    rng = np.random.default_rng(0)
    bad = 0
    for _ in range(5000):
        n = int(rng.integers(1, 8))
        base = rng.normal()
        z = base + rng.integers(-3, 4, n) * 2.0 ** -26 + rng.normal(0, 2.0 ** -27, n) * rng.integers(0, 2, n)
        stored, win = None, None
        for j, zj in enumerate(z):
            if stored is not None and float(stored) > zj:
                continue
            stored, win = np.float32(zj), j
        M, w = TO.winners(np.zeros(n, np.int64), z, np.arange(n, dtype=np.int64), 1)
        bad += int(w[0] != win or M[0].view(np.uint32) != stored.view(np.uint32))
    assert bad == 0


def test_host_geometry_rejections():
    L = _lib()
    req = np.array([[0.0, 0.0, 1.0, 1.0]])
    T = TO.iso(np.eye(3), (0, 0, 0))[None, :].copy()
    c = np.zeros(2)
    info = np.zeros(3, np.int32)
    geo = np.zeros(4)
    p = lambda a: a.ctypes.data
    f = L.emap_transformed_submap_windows
    assert f(202, 0.04, p(c), 1, p(req), p(T), p(info), p(geo)) == 0
    bad = []
    for k, v in [(0, np.nan), (4, np.inf), (9, np.nan), (11, -np.inf), (0, 1.0 + 2e-6), (1, 1e-5), (8, 0.5)]:
        b = T.copy()
        b[0, k] = v
        bad.append(b)
    bad.append(TO.iso(2 * np.eye(3), (0, 0, 0))[None, :].copy())
    for b in bad:
        assert f(202, 0.04, p(c), 1, p(req), p(b), p(info), p(geo)) == -1, b
    ok = T.copy()
    ok[0, 0] = 1.0 + 4e-7                        # within EMAP_TRANSFORM_TOLERANCE
    assert f(202, 0.04, p(c), 1, p(req), p(ok), p(info), p(geo)) == 0
    r = req.copy()
    r[0, 2] = -0.1
    assert f(202, 0.04, p(c), 1, p(r), p(T), p(info), p(geo)) == -1
    assert f(202, 0.04, p(c), 1, p(req), None, p(info), p(geo)) == -1
    assert f(202, 0.04, p(c), 1, p(req), p(T), p(info), None) == -1
    assert f(2, 0.04, p(c), 1, p(req), p(T), p(info), p(geo)) == -1
    assert f(202, 0.0, p(c), 1, p(req), p(T), p(info), p(geo)) == -1
