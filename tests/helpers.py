"""Shared helpers of the parity tests."""
import numpy as np

LAYERS = ["elevation", "variance", "is_valid", "traversability", "time", "upper_bound", "is_upper_bound"]


def compare_state(eng_map, eng_normal, om, trav_tol=2e-6, exact_layers=(0, 1, 2, 4, 5, 6), label=""):
    """CUDA engine state vs oracle state.  By construction (fixed-point accumulation, pinned
    contractions) every layer except traversability is expected BIT-identical; traversability goes
    through expf (CUDA vs glibc) and is compared to `trav_tol`."""
    for li in exact_layers:
        a, b = eng_map[li], om.elevation_map[li]
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            r, c = bad[0]
            raise AssertionError(f"{label} layer {LAYERS[li]}: {len(bad)} cells differ, first at ({r},{c}): "
                                 f"engine {a[r, c]!r} oracle {b[r, c]!r}; max abs diff {np.nanmax(np.abs(a - b))}")
    d = np.abs(eng_map[3] - om.elevation_map[3])
    assert d.max() <= trav_tol, f"{label} traversability max diff {d.max()}"
    assert np.array_equal(eng_normal, om.normal_map), f"{label} normals differ: max {np.abs(eng_normal - om.normal_map).max()}"


def check_frame(em, om, n, label, counted=False, nan_rows=None):
    """state, point record and frame statistics of the last frame of `em` against the oracle's"""
    state, normal = em.get_state()
    compare_state(state, normal, om, label=label)
    idx, valid, inside = em.get_point_record(n)
    oi, ov, oin = om.last_point_record
    ok = np.ones(n, bool) if nan_rows is None else ~nan_rows
    assert np.array_equal(idx[ok], oi[ok]), label
    assert np.array_equal(valid, ov) and np.array_equal(inside, oin), label
    st = em.get_frame_stats()
    assert st.n_points == n, label
    assert st.n_valid_points == int(ov.sum()), label
    assert st.error_cnt == om.stats.error_cnt and st.drift_applied == om.stats.drift_applied, label
    if om.stats.drift_evaluated:
        assert np.float32(st.mean_error) == np.float32(om.stats.mean_error), label
    if counted:
        assert (st.ray_steps, st.ray_visits) == (om.stats.ray_steps, om.stats.ray_visits), label
    return st, state, normal


# Seeded inputs of the comparisons with the reference's kernel source (tests/test_oracle_cpu.py); the reference's
# outputs on them are stored under tests/golden/ by tests/golden/make_golden.py.
STAR_R = np.array([[0.9, 0.1, -0.2], [0.0, 1.0, 0.1], [0.15, -0.12, 0.97]], np.float32)

FLAG_CASES = [
    dict(enable_edge_sharpen=False),
    dict(enable_visibility_cleanup=False),
    dict(enable_overlap_clearance=False, enable_drift_compensation=False),
    dict(max_ray_length=2.0, cleanup_step=0.01, cleanup_cos_thresh=0.5, wall_num_thresh=3, dilation_size=2,
         min_valid_distance=0.3, mahalanobis_thresh=1.0),
]


def dilation_inputs(W):
    rng = np.random.default_rng(3)
    h = rng.standard_normal((W, W)).astype(np.float32)
    mask = (rng.random((W, W)) < 0.15).astype(np.float32)
    mask[:, :4] = (rng.random((W, 4)) < 0.6); mask[:, -4:] = (rng.random((W, 4)) < 0.6)   # exercise the row wrap-around
    return h, mask


def star_inputs(W):
    rng = np.random.default_rng(8)
    h = rng.standard_normal((W, W)).astype(np.float32)
    m = (rng.random((W, W)) < 0.3).astype(np.float32)
    return h, m


def semantic_inputs(p, W):
    """Point records + channels of the semantic-fusion comparison: (idx, valid, inside, rows, feats, cnt)."""
    from elevation_mapping_cupy_b200 import workloads as wl
    from oracle import oracle as O
    rng = np.random.default_rng(3)
    pts, R, t = wl.uniform_cloud(0, 1, n=6000, half_extent=2.3)
    idx, valid, inside, _ = O.point_index(p, pts, R, t)
    feats = np.stack([rng.random(len(pts), dtype=np.float32) * 3, rng.random(len(pts), dtype=np.float32),
                      rng.integers(0, 1 << 24, len(pts)).astype(np.uint32).view(np.float32)], 1)
    rows = np.ascontiguousarray(np.concatenate([np.stack([idx, valid, inside], 1).astype(np.float32), feats], 1))
    cnt = np.bincount(idx[(valid > 0) & (inside > 0)], minlength=W * W).astype(np.float32)
    cnt[rng.random(W * W) < 0.3] = 0          # as if some cells' points had been rejected by the fusion (CK.py:174-179)
    return idx, valid, inside, rows, feats, cnt


def drift_frames(n=5):
    from elevation_mapping_cupy_b200 import workloads as wl
    out = []
    for f in range(n):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        pts = pts.copy(); pts[:, 2] += np.float32(0.03 * (f % 2))     # alternating 3 cm bias -> non-zero mean error
        out.append((pts, R, t))
    return out
