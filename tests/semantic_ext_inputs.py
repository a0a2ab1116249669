"""Seeded inputs of the class_bayesian / bayesian_inference / class_max comparison against the reference's kernel strings
(tests/test_semantic_ext_cpu.py and tests/golden/make_semantic_ext_golden.py build them from the same seeds)."""
import numpy as np

W = 130
CB_COLS, BI_COLS, CM_COLS = (3, 4, 5), (6, 7), (8, 9)
KINDS = ["class_bayesian"] * 3 + ["bayesian_inference"] * 2 + ["class_max"] * 2
CM_IDS = np.array([1, 4, 9, 300, 65535], np.int64)


def frame_inputs(p, frame):
    """(idx, valid, inside, rows, feats, cnt): rows = [idx, valid, inside, 7 features] as fp32 (the reference's
    points_all layout with the record in front), feats = the 7 feature columns."""
    from elevation_mapping_cupy_b200 import workloads as wl
    from oracle import oracle as O
    from oracle import semantic_ext as X
    rng = np.random.default_rng(11 + frame)
    pts, R, t = wl.uniform_cloud(0, frame, n=6000, half_extent=2.3)
    idx, valid, inside, _ = O.point_index(p, pts, R, t)
    n = len(pts)
    cb = rng.random((n, 3), dtype=np.float32)
    cb[rng.random((n, 3)) < 0.15] *= -1
    bi = (rng.random((n, 2), dtype=np.float32) * 2 - 0.5).astype(np.float32)
    prob = (rng.integers(0, 1025, (n, 2)) / 1024).astype(np.float32)    # fp16-exact, sums exact in fp32: ties are exact
    ids = rng.choice(CM_IDS[: 3 + frame], (n, 2))
    feats = np.concatenate([cb, bi, X.encode_max(prob, ids)], 1).astype(np.float32)
    rows = np.ascontiguousarray(np.concatenate([np.stack([idx, valid, inside], 1).astype(np.float32), feats], 1))
    cnt = np.bincount(idx[(valid > 0) & (inside > 0)], minlength=W * W).astype(np.float32)
    cnt[rng.random(W * W) < 0.3] = 0          # as if some cells' points had been rejected by the fusion (CK.py:174-179)
    return idx, valid, inside, rows, feats, cnt
