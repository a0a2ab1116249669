"""Regenerates tests/golden/depth_image_core.npz: the semantic sensor node's own depth-image -> cloud step
(pointcloud_node.py create_pcl_from_image, run unmodified by oracle/build_ref_depth.py) on seeded images.

Cases: `geom` (depth only, the node's max depth of 8 m) and `sem` (depth, a confidence plane with values below, at and
above the threshold, rgb8 colour and two segmentation-style feature planes: a float score and class_max codes).  The
depth holds NaN, +-inf, 0, -0, negative values, exactly 8 and the float just below.  Stored: the inputs, P and the node's
cloud as uint32 bits (rows in the node's order).  Needs the reference tree.  Usage: python tests/golden/make_depth_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref_depth as B          # noqa: E402
import depth_image_oracle as DO                  # noqa: E402

H, W = 48, 64
THETA = 0.1                                      # not an fp32 value: the node compares against fp32(0.1)
P = np.array([[61.25, 0.0, 31.7, 0.0], [0.0, 60.9, 23.3, 0.0], [0.0, 0.0, 1.0, 0.0]], np.float64)


def inputs(seed=7):
    rng = np.random.default_rng(seed)
    depth = DO.special_depth(rng, H, W)
    conf = rng.choice(np.array([0.05, np.float32(THETA), np.nextafter(np.float32(THETA), 0), 0.5, np.nan], np.float32),
                      (H, W))
    rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    score = rng.random((H, W), dtype=np.float32)
    codes = ((rng.integers(0, 300, (H, W)).astype(np.uint32) << 16) |
             rng.integers(0, 1 << 15, (H, W)).astype(np.uint32)).view(np.float32)
    return depth, conf, rgb, np.stack([score, codes])


def main():
    depth, conf, rgb, feats = inputs()
    out = dict(depth=depth, confidence=conf, rgb=rgb, features=feats, P=P, theta=np.float64(THETA))
    geom = B.node_cloud(depth, P)
    out["geom_cloud"] = np.stack([geom[n] for n in geom.dtype.names], 1).view(np.uint32)
    sem = B.node_cloud(depth, P, ["rgb", "score", "cls"], ["color", "class_average", "class_max"], rgb=rgb,
                       features=feats, confidence=conf, confidence_threshold=THETA)
    out["sem_cloud"] = np.stack([sem[n] for n in sem.dtype.names], 1).view(np.uint32)
    path = os.path.join(HERE, "depth_image_core.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
