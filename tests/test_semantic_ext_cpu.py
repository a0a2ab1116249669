"""CPU tests of the class_bayesian, bayesian_inference and class_max fusions (no GPU): the NumPy definition
(oracle/semantic_ext.py) against the reference's own kernel strings (stored outputs, tests/golden/
make_semantic_ext_golden.py), the class_max round rule on hand-built cells, and SemanticMap's bookkeeping of the new kinds
(with a stand-in engine that records what it is handed)."""
import os
import types

import numpy as np
import pytest

import semantic_ext_inputs as SI
from oracle import semantic_ext as X

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_definition_against_reference_source(oracle_mod):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    g = np.load(os.path.join(GOLD, "semantic_ext_core130.npz"))
    W = SI.W
    p = core_parameter(W)
    sem = np.zeros((7, W, W), np.float32)
    sigma = np.ones((7, W, W), np.float32)
    id_max = np.zeros((2, W, W), np.int32)
    tol = lambda ref: 2e-6 * max(1.0, float(np.abs(ref).max()))
    for frame in range(2):
        idx, valid, inside, rows, feats, cnt = SI.frame_inputs(p, frame)
        X.fuse(W, idx, valid, inside, np.zeros(len(idx), bool), feats, SI.KINDS, list(range(7)), sem, cnt, sigma=sigma,
               id_max=id_max)
        for k in range(3):
            assert np.abs(sem[k] - g[f"cb_{frame}"][k]).max() <= tol(g[f"cb_{frame}"][k]), (frame, "class_bayesian", k)
        for k in range(2):
            assert np.abs(sem[3 + k] - g[f"bi_{frame}"][k]).max() <= tol(g[f"bi_{frame}"][k]), (frame, "bayesian", k)
            assert np.abs(sigma[3 + k] - g[f"bi_sigma_{frame}"][k]).max() <= tol(g[f"bi_sigma_{frame}"][k]), (frame, "sigma", k)
            assert np.abs(sem[5 + k] - g[f"cm_{frame}"][k]).max() <= tol(g[f"cm_{frame}"][k]), (frame, "class_max", k)
        assert np.array_equal(id_max, g[f"cm_id_{frame}"]), frame
        assert (sigma[3:5] < 1).any() and (sigma[:3] == 1).all()          # only bayesian_inference layers move


def test_fixed_point_sums_are_order_free():
    rng = np.random.default_rng(0)
    x = rng.random(5000, dtype=np.float32) * 3 - 1
    cells = rng.integers(0, 50, 5000)
    a = X.cell_sum_fix(cells, X.fix32(x), 50)
    perm = rng.permutation(5000)
    assert np.array_equal(a, X.cell_sum_fix(cells[perm], X.fix32(x[perm]), 50))
    ref = np.bincount(cells, weights=x.astype(np.float64), minlength=50)
    assert np.abs(X.unfix32(a) - ref).max() < 1e-5
    assert X.fix32(np.float32(np.nan)) == 0 and X.fix32(np.float32(3e6)) == X.fix32(np.float32(1048576.0))


def test_decode_encode_max_roundtrip():
    prob = np.array([0.0, 0.5, 1.0, -0.25, np.inf, 65504.0], np.float32)
    ids = np.array([0, 1, 65535, 300, 7, 42])
    p, i = X.decode_max(X.encode_max(prob, ids))
    assert np.array_equal(p, prob) and np.array_equal(i, ids)


def _rounds(C, U, cells, n):
    return X.class_max_rounds(C, U, {c: (np.array(i, np.int64), np.array(v, np.float32)) for c, (i, v) in cells.items()}, n)


def test_class_max_all_empty_cell_takes_smallest_id():
    vals, ids = _rounds(3, [5, 2, 9], {0: ([5], [0.7])}, 2)
    assert ids[0, 1] == 2 and ids[0, 2] == 2 and vals[0, 1] == 0          # every id counts 0: the smallest wins
    assert ids[0, 0] == 5 and vals[0, 0] == np.float32(0.7)
    # round 1: 5 and 2 won in round 0 and count 0; 9 is absent: cell 0 ties at 0 -> smallest zero-valued id (2)
    assert ids[1, 0] == 2 and vals[1, 0] == 0


def test_class_max_rounds_rule():
    # equal sums: the smallest id wins
    vals, ids = _rounds(1, [3, 8, 12], {0: ([3, 8, 12], [0.5, 0.75, 0.75])}, 3)
    assert list(ids[:, 0]) == [8, 12, 3] and list(vals[:, 0]) == [0.75, 0.75, 0.5]
    # NaN is the maximum; the smallest NaN id first
    vals, ids = _rounds(1, [1, 2, 3], {0: ([1, 2, 3], [0.9, np.nan, np.nan])}, 3)
    assert list(ids[:, 0]) == [2, 3, 1] and np.isnan(vals[0, 0]) and np.isnan(vals[1, 0]) and vals[2, 0] == np.float32(0.9)
    # an id that wins elsewhere is zeroed here for the later rounds
    vals, ids = _rounds(2, [4, 6], {0: ([4, 6], [0.9, 0.8]), 1: ([4, 6], [0.1, 0.95])}, 2)
    assert ids[0, 0] == 4 and ids[0, 1] == 6
    assert ids[1, 0] == 4 and vals[1, 0] == 0 and ids[1, 1] == 4 and vals[1, 1] == 0   # both won in round 0: all 0
    # negative sums lose to an absent id (0)
    vals, ids = _rounds(1, [1, 5], {0: ([5], [-0.5])}, 1)
    assert ids[0, 0] == 1 and vals[0, 0] == 0


def test_class_max_definition_normalises_and_keeps_id_max():
    W = 4
    C = W * W
    idx = np.array([0, 0, 1, 1, 5])
    one = np.ones(5, np.uint8)
    feats = np.stack([X.encode_max([0.5, 0.25, 0.75, 0.75, 0.0], [7, 7, 2, 9, 3]),
                      X.encode_max([0.25, 0.25, 0.25, 0.5, 0.0], [2, 9, 2, 9, 3])], 1)
    sem = np.zeros((2, W, W), np.float32)
    id_max = np.full((2, W, W), 11, np.int32)
    X.fuse(W, idx, one, one, np.zeros(5, bool), feats, ["class_max"] * 2, [0, 1], sem, np.zeros(C), id_max=id_max)
    # U = {2, 3, 7, 9, 11}; empty cells: 2 wins both rounds with 0
    assert id_max[0].reshape(-1)[0] == 7 and id_max[0].reshape(-1)[1] == 9 and id_max[0].reshape(-1)[2] == 2
    # cell 0 sums 7: 0.75, 2: 0.25, 9: 0.25; cell 1 sums 2: 1.0, 9: 1.25.  Round 0 is won by 7, 9 and 2 (the empty
    # cells), so in round 1 every id of cells 0 and 1 counts 0 and 2 wins there with 0.
    v = sem.reshape(2, C)
    assert id_max[1].reshape(-1)[0] == 2 and id_max[1].reshape(-1)[1] == 2
    assert v[0, 0] == 1 and v[1, 0] == 0 and v[0, 1] == 1 and v[1, 1] == 0
    assert v[0, 2] == 0 and v[1, 2] == 0 and id_max[1].reshape(-1)[5] == 2


class _Engine:
    """Records what SemanticMap hands the engine (no library, no GPU)."""

    def __init__(self):
        self.calls = []
        self.device = "cpu"
        self._h = None
        self._L = types.SimpleNamespace(emap_semantic_configure_ext=lambda *a: self.calls.append(a) or 0)

    def _check(self, rc):
        assert rc == 0

    def _before_framework(self):
        pass


def _semantic_map(W=6, fusions=None):
    torch = pytest.importorskip("torch")
    from elevation_mapping_cupy_b200 import semantic_map as S
    p = types.SimpleNamespace(cell_n=W, pointcloud_channel_fusions=fusions or {
        "cb.*": "class_bayesian", "bi": "bayesian_inference", "cm.*": "class_max", "default": "class_average"},
        average_weight=0.5)
    sm = S.SemanticMap(p, engine=_Engine())
    sm._alloc = lambda n: torch.zeros((n, W, W), dtype=torch.float32)
    return sm, torch


def test_semantic_map_accepts_new_kinds_and_allocates_state():
    sm, torch = _semantic_map()
    sm.configure_for(["x", "y", "z", "cb1", "bi", "cm1", "cm2", "other"])
    assert sm.layer_names == ["cb1", "bi", "cm1", "cm2", "other"]
    assert sm.variance.shape == (5, 6, 6) and bool((sm.variance == 1).all())
    idm = sm.elements_to_shift["id_max"]
    assert idm.shape == (2, 6, 6) and idm.dtype == torch.int32 and int(idm.abs().sum()) == 0
    a = sm.engine.calls[-1]
    assert list(a[2]) == [3, 4, 5, 6, 7] and list(a[3]) == [3, 4, 5, 5, 1] and a[10] == 2
    # a layer added later grows the variance planes with 1.0 and re-registers
    n = len(sm.engine.calls)
    sm.add_layer("late")
    assert sm.variance.shape == (6, 6, 6) and bool((sm.variance[5] == 1).all()) and len(sm.engine.calls) == n + 1


def test_semantic_map_unknown_fusion_still_raises():
    sm, _ = _semantic_map(fusions={"default": "no_such_fusion"})
    with pytest.raises(NotImplementedError):
        sm.configure_for(["x", "y", "z", "a"])


def test_semantic_map_clear_and_shift_rules():
    sm, torch = _semantic_map()
    sm.configure_for(["x", "y", "z", "bi", "cm1"])
    sm.semantic_map.fill_(2.0)
    sm.variance.fill_(0.25)
    sm.elements_to_shift["id_max"].fill_(7)
    sm.shift_map_xy((1, -2))
    assert bool((sm.semantic_map[:, 0, :] == 0).all()) and bool((sm.semantic_map[:, :, -2:] == 0).all())
    assert bool((sm.variance[:, 0, :] == 1).all()) and bool((sm.variance[:, :, -2:] == 1).all())
    assert bool((sm.variance[:, 1:, :-2] == 0.25).all())
    idm = sm.elements_to_shift["id_max"]
    assert bool((idm[:, 0, :] == 0).all()) and bool((idm[:, :, -2:] == 0).all()) and bool((idm[:, 1:, :-2] == 7).all())
    sm.clear()
    assert float(sm.semantic_map.abs().max()) == 0 and bool((sm.variance == 1).all())
    assert bool((idm[:, 1:, :-2] == 7).all())                                      # id_max survives clear()
