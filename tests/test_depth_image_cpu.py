"""The NumPy restatement of the depth-image -> cloud step (tests/depth_image_oracle.py) against the semantic sensor
node's own output on the golden images (tests/golden/depth_image_core.npz, tests/golden/make_depth_golden.py), the mask
against a literal transliteration of the node's get_coordinates, and the colour packing bit by bit."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import depth_image_oracle as DO          # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "depth_image_core.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def test_geometry_equals_node_cloud(golden):
    cloud, kept = DO.depth_cloud(golden["depth"], golden["P"])
    assert kept.sum() == len(golden["geom_cloud"])
    assert np.array_equal(cloud.view(np.uint32), golden["geom_cloud"])


def test_channels_and_confidence_equal_node_cloud(golden):
    cloud, kept = DO.depth_cloud(golden["depth"], golden["P"], sources=(-1, 0, 1), rgb=golden["rgb"],
                                 features=golden["features"], confidence=golden["confidence"],
                                 confidence_threshold=float(golden["theta"]))
    assert np.array_equal(cloud.view(np.uint32), golden["sem_cloud"])
    # the golden holds every case of the mask
    d, q = golden["depth"], golden["confidence"]
    assert np.isnan(d).any() and np.isposinf(d).any() and np.isneginf(d).any() and (d == 8.0).any()
    assert (np.signbit(d) & (d == 0)).any() and (d < 0).any() and (d == np.nextafter(np.float32(8), 0)).any()
    theta = np.float32(golden["theta"])
    assert (q == theta).any() and (q < theta).any() and (q > theta).any()


def _node_mask(depth, confidence, threshold):
    """pointcloud_node.py get_coordinates, line for line in NumPy."""
    pos = np.where(depth > 0, 1, 0)
    low = np.where(depth < 8, 1, 0)
    if confidence is not None:
        conf = np.where(confidence >= threshold, 1, 0)
    else:
        conf = np.ones(pos.shape)
    fin = np.isfinite(depth)
    temp = np.maximum(np.rint(fin + pos + conf + low - 2.6), 0)
    return np.nonzero(temp)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("with_conf", [False, True])
def test_mask_equals_get_coordinates(seed, with_conf):
    rng = np.random.default_rng(seed)
    H, W = int(rng.integers(1, 40)), int(rng.integers(1, 40))
    d = DO.special_depth(rng, H, W)
    threshold = [10.0, 0.1, 0.5, 0.0, 1e-3, 0.7][seed]
    q = None
    if with_conf:
        q = rng.uniform(-0.5, 1.5, (H, W)).astype(np.float32)
        q[rng.random((H, W)) < 0.2] = np.float32(threshold)
        q[rng.random((H, W)) < 0.05] = np.nan
    with np.errstate(invalid="ignore"):
        v, u = _node_mask(d, q, threshold)
    m = DO.keep_mask(d, q, threshold)
    assert np.array_equal(np.stack(np.nonzero(m)), np.stack([v, u]))


def test_colour_packing_bits():
    rgb = np.array([[[0, 0, 0], [255, 255, 255], [1, 2, 3], [0x80, 0, 0x7f], [0, 0xff, 0]]], np.uint8)
    got = DO.pack_rgb(rgb).view(np.uint32)[0]
    assert got.tolist() == [0, 0xffffff, 0x010203, 0x80007f, 0x00ff00]
    # every byte in every position
    rng = np.random.default_rng(1)
    c = rng.integers(0, 256, (1000, 3), dtype=np.uint8)
    bits = DO.pack_rgb(c).view(np.uint32)
    assert np.array_equal((bits >> 16) & 0xff, c[:, 0]) and np.array_equal((bits >> 8) & 0xff, c[:, 1])
    assert np.array_equal(bits & 0xff, c[:, 2]) and not (bits >> 24).any()
