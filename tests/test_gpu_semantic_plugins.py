"""The semantic plugins on the device (emap_semantic_filter, emap_semantic_traversability, emap_features_pca) against the
NumPy yardstick tests/semantic_plugins_oracle.py, through the plugin classes, the C ABI and an ElevationMap driven by a
plugin YAML and real frames."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import semantic_plugins_oracle as SO          # noqa: E402

pytestmark = pytest.mark.gpu


def _mk(W):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    return ElevationMap(core_parameter(W, plugin_config_file=""))


def _bits(t):
    import torch
    return t.contiguous().view(torch.int32).cpu().numpy().view(np.uint32)


def _stores(em, W, n_basic_sel, n_plugin, n_sem, seed, levels=4, nan_frac=0.02):
    """Random integer-valued layers (many exact ties across stores) with NaN cells in all three stores.  Returns the
    store tuples and the stack of the layers the patterns below select, in selection order."""
    import torch
    rng = np.random.default_rng(seed)
    def rnd(n):
        a = rng.integers(0, levels, (n, W, W)).astype(np.float32)
        a[rng.random(a.shape) < nan_frac] = np.nan
        return a
    st = np.zeros((7, W, W), np.float32)
    basic = rnd(2)
    st[0], st[3] = basic                     # elevation, traversability
    em.set_state(st)
    pl = rnd(n_plugin + 1)                   # one plugin layer that no pattern selects
    sem = rnd(n_sem)
    pl_names = [f"cls_pl_{k}" for k in range(n_plugin)] + ["other"]
    sem_names = [f"cls_sem_{k:03d}" for k in range(n_sem)]
    stores = (torch.from_numpy(pl).cuda(), pl_names, torch.from_numpy(sem).cuda() if n_sem else None, sem_names)
    sel = [basic[0], basic[1]][:n_basic_sel] + list(pl[:n_plugin]) + list(sem)
    patterns = ["^elevation$", "^traversability$"][:n_basic_sel] + ["^cls_"]
    return stores, np.array(sel, np.float32).reshape(-1, W, W), patterns


@pytest.mark.parametrize("W", [202, 1024])
@pytest.mark.parametrize("L", [0, 1, 255])
def test_semantic_filter_bits_match_oracle(W, L):
    from elevation_mapping_cupy_b200.plugins.semantic_filter import SemanticFilter
    em = _mk(W)
    if L == 0:
        stores, stack, pats = _stores(em, W, 0, 0, 0, 1)
        pats = ["^nothing$"]
    elif L == 1:
        stores, stack, pats = _stores(em, W, 0, 0, 1, 2)
    else:
        stores, stack, pats = _stores(em, W, 2, 3, 250, 3)
    assert len(stack) == L
    plug = SemanticFilter(cell_n=W, classes=pats, engine=em)
    out = plug(em.elevation_map, em.layer_names, *stores)
    ref = SO.semantic_filter(stack, shape=(W, W))
    assert np.array_equal(_bits(out), ref)
    if L == 255:                             # the cases the stack was built for did occur
        assert np.isnan(stack).any(axis=0).sum() > 0 and (ref >> 23 == 0).any() and (ref >> 23 != 0).any()


def test_semantic_filter_nan_after_maximum_and_ties_between_stores():
    import torch
    from elevation_mapping_cupy_b200.plugins.semantic_filter import SemanticFilter
    W = 202
    em = _mk(W)
    st = np.zeros((7, W, W), np.float32)
    st[0] = 2.0                                                     # elevation: ties with the plugin layer everywhere
    em.set_state(st)
    pl = np.full((1, W, W), 2.0, np.float32)
    sem = np.zeros((2, W, W), np.float32)
    sem[0, 5, :] = 7.0                                              # a larger maximum in a later store
    sem[1, 5, :10] = np.nan                                         # NaN after the maximum: the NaN wins
    sem[0, 6, :] = np.nan; sem[1, 6, :] = np.nan                    # two NaNs: the first wins
    plug = SemanticFilter(cell_n=W, classes=["^elevation$", "^pl$", "^s"], engine=em)
    out = _bits(plug(em.elevation_map, em.layer_names, torch.from_numpy(pl).cuda(), ["pl"],
                     torch.from_numpy(sem).cuda(), ["s0", "s1"]))
    pal = SO.palette()
    assert (out[0] == pal[0]).all()
    assert (out[5, :10] == pal[3]).all() and (out[5, 10:] == pal[2]).all() and (out[6] == pal[2]).all()
    assert np.array_equal(out, SO.semantic_filter(np.stack([st[0], pl[0], sem[0], sem[1]])))


def test_semantic_filter_rejects_256_layers():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    from elevation_mapping_cupy_b200.plugins.semantic_filter import SemanticFilter
    W = 130
    em = _mk(W)
    sem = torch.zeros((256, W, W), device="cuda")
    out = torch.empty((W, W), device="cuda")
    ptrs = (C.c_void_p * 256)(*[sem[k].data_ptr() for k in range(256)])
    assert em._L.emap_semantic_filter(em._h, 256, ptrs, out.data_ptr()) == -1
    assert em._L.emap_semantic_filter(em._h, 255, ptrs, out.data_ptr()) == 0
    plug = SemanticFilter(cell_n=W, classes=["^s"], engine=em)
    with pytest.raises(_lib.EmapError):
        plug(em.elevation_map, em.layer_names, None, [], sem, [f"s{k}" for k in range(256)])


@pytest.mark.parametrize("W", [202, 1024])
def test_semantic_traversability_matches_oracle(W):
    import torch
    from elevation_mapping_cupy_b200.plugins.semantic_traversability import SemanticTraversability
    em = _mk(W)
    rng = np.random.default_rng(W)
    st = np.zeros((7, W, W), np.float32)
    st[3] = rng.random((W, W)).astype(np.float32)
    st[0] = (rng.random((W, W)) * 2 - 1).astype(np.float32)
    thr = [0.3, 0.1, 0.5]
    st[3, :, :7] = np.float32(thr[0])                               # exactly fp32(thr): not <= thr in fp64
    st[0, :7, :] = np.float32(thr[1])                               # exactly fp32(thr): >= thr in fp64
    st[3, 10, :] = np.nan; st[0, 11, :] = np.nan
    em.set_state(st)
    pl = rng.random((2, W, W)).astype(np.float32)
    pl[1, 12, :] = np.nan
    pl[1, :, 7:12] = 0.5                                            # exactly the (fp32-exact) threshold: votes with <=
    pl_t = torch.from_numpy(pl).cuda()
    layers, types = ["traversability", "elevation", "risk"], ["traversability", "elevation", "traversability"]
    plug = SemanticTraversability(cell_n=W, layers=layers, thresholds=thr, type=types, engine=em)
    out = plug(em.elevation_map, em.layer_names, pl_t, ["x", "risk"], None, []).cpu().numpy()
    ref = SO.semantic_traversability(np.stack([st[3], st[0], pl[1]]), thr, types)
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    assert (ref == np.float32(0.1)).any() and (ref == 1.0).any()
    only_risk = (st[3, :, 7:12] > 0.3) & (st[0, :, 7:12] < 0.1)
    assert only_risk.any() and (ref[:, 7:12][only_risk] == 1.0).all()
    # a single layer, each type, and the exact-threshold cells decided by the fp64 rule
    for typ in ("traversability", "elevation"):
        p1 = SemanticTraversability(cell_n=W, layers=["traversability"], thresholds=[0.3], type=[typ], engine=em)
        o1 = p1(em.elevation_map, em.layer_names, pl_t, ["x", "risk"], None, []).cpu().numpy()
        assert np.array_equal(o1, SO.semantic_traversability(st[3:4], [0.3], [typ]))
        assert (o1[:, :7] == (np.float32(0.1) if typ == "traversability" else 1.0))[20:].all()
    # a missing layer: the reference's message, and the traversability layer
    miss = SemanticTraversability(cell_n=W, layers=["traversability", "nope"], thresholds=[0.3, 0.3],
                                  type=types[:2], engine=em)
    o2 = miss(em.elevation_map, em.layer_names, pl_t, ["x", "risk"], None, []).cpu().numpy()
    assert np.array_equal(o2.view(np.uint32), st[3].view(np.uint32))


def _pca_plugin(em, W, names):
    from elevation_mapping_cupy_b200.plugins.features_pca import FeaturesPca
    return FeaturesPca(cell_n=W, process_layer_names=names, engine=em)


def _check_pca(bits, x):
    ref, sc = SO.features_pca(x)
    ours = np.stack([(bits >> 16) & 255, (bits >> 8) & 255, bits & 255]).astype(np.int64)
    theirs = np.stack([(ref >> 16) & 255, (ref >> 8) & 255, ref & 255]).astype(np.int64)
    boundary = np.abs(sc - np.round(sc)) < 1e-6
    d = np.abs(ours - theirs)
    assert d.max() <= 1 and not (d[~boundary] > 0).any(), (int((d > 0).sum()), int(boundary.sum()))


@pytest.mark.parametrize("W", [202, 1024, 2048, 2049])
@pytest.mark.parametrize("F", [3, 8, 16, 64])
def test_features_pca_matches_oracle(W, F):
    import torch
    em = _mk(W)
    x = SO.gapped_features(F, W, 7 * F + W)
    sem = torch.from_numpy(x).cuda()
    names = [f"feat_{k}" for k in range(F)]
    plug = _pca_plugin(em, W, ["^feat_.*$"])
    a = _bits(plug(em.elevation_map, em.layer_names, None, [], sem, names))
    b = _bits(plug(em.elevation_map, em.layer_names, None, [], sem, names))
    assert np.array_equal(a, b)                                     # deterministic
    _check_pca(a, x)


def test_features_pca_edge_cases():
    import torch
    from elevation_mapping_cupy_b200 import _lib
    W = 202
    em = _mk(W)
    rng = np.random.default_rng(5)
    x = np.empty((3, W, W), np.float32)
    x[0] = rng.integers(-8, 9, (W, W)) / 8.0                         # exact sums: the other two components stay exactly 0
    x[1] = 0.25
    x[2] = -0.5
    sem = torch.from_numpy(x).cuda()
    plug = _pca_plugin(em, W, ["^f"])
    bits = _bits(plug(em.elevation_map, em.layer_names, None, [], sem, ["f0", "f1", "f2"]))
    assert ((bits & 0xffff) == 0).all() and (bits >> 16).max() == 255
    assert np.array_equal(bits, SO.features_pca(x)[0])
    # no selected plane: zeros
    none = _pca_plugin(em, W, ["^nothing$"])(em.elevation_map, em.layer_names, None, [], sem, ["f0", "f1", "f2"])
    assert (none == 0).all()
    # NaN: ValueError
    x[1, 3, 4] = np.nan
    with pytest.raises(ValueError):
        plug(em.elevation_map, em.layer_names, None, [], torch.from_numpy(x).cuda(), ["f0", "f1", "f2"])
    with pytest.raises(ValueError):                                  # two layers: sklearn's PCA(3) raises too
        plug(em.elevation_map, em.layer_names, None, [], sem[:2], ["f0", "f1"])
    # F < 3 and F > 64 through the C ABI
    planes = torch.zeros((65, W, W), device="cuda")
    out = torch.empty((W, W), device="cuda")
    ptrs = (C.c_void_p * 65)(*[planes[k].data_ptr() for k in range(65)])
    for F in (0, 1, 2, 65):
        assert em._L.emap_features_pca(em._h, F, ptrs, out.data_ptr()) == -1, F
        assert b"EMAP_PCA_MAX_FEATURES" in em._L.emap_last_error(em._h)
    assert em._L.emap_features_pca(em._h, 64, ptrs, out.data_ptr()) == 0
    assert em._L.emap_features_pca(em._h, 3, None, out.data_ptr()) == -1
    assert em._L.emap_semantic_traversability(em._h, 1, ptrs, None, None, out.data_ptr()) == -1


def test_plugins_on_a_side_stream():
    """Inputs written on a non-default torch stream just before each call: the library's kernels run after them."""
    import torch
    from elevation_mapping_cupy_b200.plugins.semantic_filter import SemanticFilter
    from elevation_mapping_cupy_b200.plugins.semantic_traversability import SemanticTraversability
    W = 1024
    em = _mk(W)
    x = SO.gapped_features(16, W, 3)
    cls = np.random.default_rng(4).random((16, W, W)).astype(np.float32)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        feat = torch.zeros((16, W, W), device="cuda")
        sem = torch.zeros((16, W, W), device="cuda")
        pl = torch.zeros((1, W, W), device="cuda")
        torch.cuda._sleep(20_000_000)                                # the writes below land late on this stream
        feat.copy_(torch.from_numpy(x).to("cuda", non_blocking=True))
        names = [f"feat_{k}" for k in range(16)]
        pca = _pca_plugin(em, W, ["^feat_"])(em.elevation_map, em.layer_names, None, [], feat, names)
        torch.cuda._sleep(20_000_000)
        sem.copy_(torch.from_numpy(cls).to("cuda", non_blocking=True))
        filt = SemanticFilter(cell_n=W, classes=["^c"], engine=em)(em.elevation_map, em.layer_names, None, [], sem,
                                                                   [f"c{k}" for k in range(16)])
        torch.cuda._sleep(20_000_000)
        pl.fill_(0.75)
        trav = SemanticTraversability(cell_n=W, layers=["risk"], thresholds=[0.5], type=["risk"], engine=em)(
            em.elevation_map, em.layer_names, pl, ["risk"], None, [])
        pca_b, filt_b, trav_b = _bits(pca), _bits(filt), trav.cpu().numpy()
    s.synchronize()
    _check_pca(pca_b, x)
    assert np.array_equal(filt_b, SO.semantic_filter(cls))
    assert (trav_b == 1.0).all()


PLUGIN_YAML = """
semantic_filter:
  type: "semantic_filter"
  enable: True
  fill_nan: False
  is_height_layer: False
  layer_name: "max_categories"
  extra_params:
    classes: ["^sem_.*$"]
features_pca:
  type: "features_pca"
  enable: True
  fill_nan: False
  is_height_layer: False
  layer_name: "pca"
  extra_params:
    process_layer_names: ["^feat_.*$"]
semantic_traversability:
  type: "semantic_traversability"
  enable: True
  fill_nan: False
  is_height_layer: False
  layer_name: "semantic_traversability"
  extra_params:
    layers: ["traversability", "elevation"]
    thresholds: [0.3, 0.1]
    type: ["traversability", "elevation"]
"""


def test_turtle_bot_style_yaml_end_to_end(tmp_path):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    cfg = tmp_path / "plugin_config.yaml"
    cfg.write_text(PLUGIN_YAML)
    W = 202
    p = core_parameter(W, plugin_config_file=str(cfg),
                       pointcloud_channel_fusions={"rgb": "color", "feat_.*": "average", "default": "class_average"})
    em = ElevationMap(p)
    sem_names, feat_names = ["sem_a", "sem_b", "sem_c"], [f"feat_{k}" for k in range(8)]
    channels = ["x", "y", "z"] + sem_names + feat_names + ["rgb"]
    rng = np.random.default_rng(11)
    for f in range(3):
        pts, R, t = wl.uniform_cloud(0, f, n=20000, half_extent=3.5)
        n = len(pts)
        sem = rng.random((n, 3)).astype(np.float32)
        feat = (rng.standard_normal((n, 8)) * np.array([0.5, 0.35, 0.25, 0.1, 0.05, 0.04, 0.03, 0.02])).astype(np.float32)
        rgb = rng.integers(0, 1 << 24, n).astype(np.uint32).view(np.float32)
        em.input_pointcloud(np.concatenate([pts, sem, feat, rgb[:, None]], 1), channels, R, t, 0.0, 0.0)
    assert set(sem_names + feat_names) <= set(em.semantic_map.layer_names)
    names = ["max_categories", "pca", "semantic_traversability"] + sem_names + feat_names
    Wo = W - 2
    one = {}
    for nm in names:
        d = np.zeros((Wo, Wo), np.float32)
        em.get_map_with_name_ref(nm, d)
        one[nm] = d
    many = np.zeros((len(names), Wo, Wo), np.float32)
    em.get_maps_with_names_ref(names, many)
    for k, nm in enumerate(names):
        assert np.array_equal(one[nm].view(np.uint32), many[k].view(np.uint32)), nm
    # the filter is per cell: the oracle on the exported semantic layers
    sem_exp = np.stack([one[n] for n in sem_names])
    assert np.array_equal(one["max_categories"].view(np.uint32), SO.semantic_filter(sem_exp))
    # the PCA takes every cell as a sample, the border ring included: the oracle on the full planes, exported the same way
    sm = em.semantic_map.semantic_map.cpu().numpy()
    full = np.stack([sm[em.semantic_map.layer_names.index(n)] for n in feat_names])
    export = lambda m: m[1:-1, 1:-1][::-1, ::-1]
    assert np.array_equal(export(full[0]), one["feat_0"])
    ref_bits, sc = SO.features_pca(full)
    got = one["pca"].view(np.uint32)
    ours = np.stack([(got >> 16) & 255, (got >> 8) & 255, got & 255]).astype(np.int64)
    theirs = np.stack([export(c) for c in ((ref_bits >> 16) & 255, (ref_bits >> 8) & 255, ref_bits & 255)]).astype(np.int64)
    boundary = np.stack([export(c) for c in np.abs(sc - np.round(sc)) < 1e-6])
    d = np.abs(ours - theirs)
    assert d.max() <= 1 and not (d[~boundary] > 0).any()
    # traversability vote on the exported basic layers (traversability is NaN outside the valid cells there: use the state)
    state, _ = em.get_state()
    trav = SO.semantic_traversability(np.stack([state[3], state[0]]), [0.3, 0.1], ["traversability", "elevation"])
    assert np.array_equal(one["semantic_traversability"].view(np.uint32), export(trav).view(np.uint32))
