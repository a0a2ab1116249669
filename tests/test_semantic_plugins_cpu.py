"""The semantic plugins' yardstick (tests/semantic_plugins_oracle.py) against the reference's formulas and, where sklearn is
installed, against sklearn's PCA.  No GPU."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import semantic_plugins_oracle as SO          # noqa: E402


def _ref_color_map(N=256):
    """semantic_filter.py:30-58 as written there (bitget, float-free uint8 rows)"""
    def bitget(byteval, idx):
        return (byteval & (1 << idx)) != 0

    cmap = np.zeros((N + 1, 3), dtype="uint8")
    for i in range(N + 1):
        r = g = b = 0
        c = i
        for j in range(8):
            r = r | (bitget(c, 0) << 7 - j)
            g = g | (bitget(c, 1) << 7 - j)
            b = b | (bitget(c, 2) << 7 - j)
            c = c >> 3
        cmap[i] = np.array([r, g, b])
    cmap[1] = np.array([81, 113, 162])
    cmap[2] = np.array([81, 113, 162])
    cmap[3] = np.array([188, 63, 59])
    return cmap[1:]


def _ref_transform_color():
    color_classes = _ref_color_map(255)
    r = np.asarray(color_classes[:, 0], dtype=np.uint32)
    g = np.asarray(color_classes[:, 1], dtype=np.uint32)
    b = np.asarray(color_classes[:, 2], dtype=np.uint32)
    return np.array((r << 16) | (g << 8) | (b << 0), dtype=np.uint32)


def test_palette_equals_reference_formula():
    pal = SO.palette()
    assert pal.shape == (255,) and pal.dtype == np.uint32
    assert np.array_equal(pal, _ref_transform_color())
    assert pal[0] == pal[1] == (81 << 16 | 113 << 8 | 162) and pal[2] == (188 << 16 | 63 << 8 | 59)
    # about half of the words are fp32 denormals (red < 128: exponent bits zero)
    assert 100 < int(((pal >> 23) == 0).sum()) < 160


def test_class_ids_equal_numpy_argmax_with_ties_and_nans():
    rng = np.random.default_rng(0)
    for L in (1, 2, 5, 40, 255):
        st = rng.integers(0, 4, (L, 64, 64)).astype(np.float32)        # many exact ties
        st[rng.random(st.shape) < 0.02] = np.nan                        # NaN in later layers than the maximum too
        st[:, 0, :L] = 3.0                                              # all-equal columns: id 0
        assert np.array_equal(SO.class_ids(st), np.argmax(st, axis=0)), L
        assert np.array_equal(SO.semantic_filter(st), _ref_transform_color()[np.argmax(st, axis=0)])
    assert np.array_equal(SO.semantic_filter(np.zeros((0, 8, 8)), shape=(8, 8)), np.full((8, 8), SO.palette()[0]))


def test_class_ids_first_maximum_and_first_nan():
    # three layers over five cells: a tie, a tie, a NaN before a larger value, two NaNs, all equal
    st = np.array([[1, 2, 2, np.nan, 0], [2, 2, np.nan, np.nan, 0], [2, 1, 9, 1, 0]], np.float32)[:, :, None]
    assert SO.class_ids(st)[:, 0].tolist() == [1, 0, 1, 0, 0]
    assert SO.class_ids(st)[:, 0].tolist() == np.argmax(st, axis=0)[:, 0].tolist()


def test_traversability_vote_rule():
    thr = 0.3
    v = np.array([np.float32(thr), np.nextafter(np.float32(thr), np.float32(0)), 0.5, np.nan], np.float32)[None, :, None]
    # fp64 comparison: fp32(0.3) = 0.30000001192... > 0.3, so it does not pass "<= 0.3"
    out = SO.semantic_traversability(v, [thr], ["traversability"])
    assert out[:, 0].tolist() == [np.float32(0.1), 1.0, np.float32(0.1), np.float32(0.1)]
    out = SO.semantic_traversability(v, [thr], ["elevation"])
    assert out[:, 0].tolist() == [1.0, np.float32(0.1), 1.0, np.float32(0.1)]
    assert SO.semantic_traversability(np.zeros((0, 2, 2)), [], [], shape=(2, 2)).tolist() == [[np.float32(0.1)] * 2] * 2


def test_pca_rejects_feature_counts_and_nan():
    x = SO.gapped_features(3, 16, 0)
    with pytest.raises(ValueError):
        SO.pca_fit(x[:2])
    with pytest.raises(ValueError):
        SO.pca_fit(np.zeros((65, 4, 4), np.float32))
    x[1, 3, 3] = np.nan
    with pytest.raises(ValueError):
        SO.features_pca(x)


def test_pca_constant_component_gives_channel_zero():
    x = np.full((4, 32, 32), 0.25, np.float32)           # constant features: every component's range is 0
    bits, sc = SO.features_pca(x)
    assert np.array_equal(bits, np.zeros_like(bits))


@pytest.mark.parametrize("W", [202, 1024])
@pytest.mark.parametrize("F", [3, 8, 16, 64])
def test_pca_oracle_matches_sklearn(W, F):
    skd = pytest.importorskip("sklearn.decomposition")
    x = SO.gapped_features(F, W, 10 * F + W)
    mean, comps, w = SO.pca_fit(x)
    k = min(4, F)
    assert np.all(w[:k - 1] > 1.1 * w[1:k])               # the spectrum really has the gaps
    data = np.clip(x.reshape(F, -1).T, -1, 1)             # features_pca.py:73-75: fp32 samples
    pca = skd.PCA(n_components=3).fit(data)
    assert np.abs(pca.components_ - comps).max() < 1e-4
    assert np.array_equal(np.sign(pca.components_), np.sign(comps))
    # features_pca.py:81-87 in sklearn's precision against the fp64 channels
    desc = pca.transform(data).reshape(W, W, 3)
    lo, hi = desc.min(axis=(0, 1)), desc.max(axis=(0, 1))
    ref_ch = (np.divide(desc - lo, hi - lo) * 255).astype(np.uint8)
    bits, sc = SO.features_pca(x)
    ours = np.stack([(bits >> 16) & 255, (bits >> 8) & 255, bits & 255], -1).astype(np.int64)
    assert np.abs(ours - ref_ch.astype(np.int64)).max() <= 1
