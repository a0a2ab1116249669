"""The frame-variant cases against the host decisions they are meant to reach, and the ray box against independently
computed march samples (no GPU needed).  The decisions are the library's own (make_plan, ray_box, raycast_runs, through
tests/plan_host.py).  The cases themselves run on the GPU in tests/test_gpu_frame_variants.py."""
import numpy as np
import pytest

import frame_variants as fv
import plan_host as ph


def _sides(cases, side_of):
    """{side: id of the first case on it}"""
    out = {}
    for cid, case in cases:
        out.setdefault(side_of(case), cid)
    return out


def _assert_sides(decision, cases, side_of, want):
    got = _sides(cases, side_of)
    missing = [s for s in want if s not in got]
    assert not missing, f"{decision}: no case on side(s) {missing}; the cases cover {got}"
    return got


def test_every_host_decision_has_a_case_on_each_side():
    a = [(c["id"], fv.frame_params(c)) for c in fv.RES_CASES]
    # resolution: the core value and others (the cell table, LIM, the march table, span_cells, the normals)
    got = _assert_sides("resolution", a, lambda p: "core" if p[1] == fv.CORE_RES else "other", ["core", "other"])
    assert got == {"core": "ray0.5-1024", "other": "res0.02-256"}, got
    # k_raycast shared-memory layout: coarse maps and march table in the gap of the cell table, or behind it
    got = _assert_sides("k_raycast layout", a, lambda p: ph.plan(*p)["where"], ["gap", "behind"])
    assert got == {"gap": "res0.02-256", "behind": "res0.1-2048"}, got
    behind = [cid for cid, p in a if ph.plan(*p)["where"] == "behind"]
    assert behind == ["res0.1-2048", "ray40-1024"], behind
    assert ph.plan(1024, 0.04, 40.0)["n_steps"] == 1313 and ph.plan(2048, 0.1, 10.0)["lut_p2"] == 44256
    # k_record / k_finalize cells per thread
    _assert_sides("k_record/k_finalize V", a, lambda p: ph.plan(*p)["cells_per_thread"], [4, 1])
    assert ph.plan(2049, fv.CORE_RES, fv.CORE_RAY)["cells_per_thread"] == 1
    # what test_frames_at_other_resolutions_ray_lengths_and_sizes runs each case for
    for cid, (W, res, L) in a:
        assert ph.plan(W, res, L)["where"] == ("behind" if cid in ("res0.1-2048", "ray40-1024") else "gap"), cid
        assert (res == fv.CORE_RES) == (cid in ("ray0.5-1024", "ray40-1024", "odd-2049")), cid
        assert ph.plan(W, res, L)["cells_per_thread"] == (1 if W % 4 else 4), cid

    def post(W, K):
        """(TMA staging, k_post instantiation) of a W x W map with dilation K, as the GPU group B handles pick them"""
        p = ph.plan(W, fv.CORE_RES, fv.CORE_RAY, K)
        return p["post_tma"], p["post_instance"]

    b = [(f"{W}/K{K}", (W, K)) for W, K in fv.POST_CASES]
    # k_post: TMA staging or plain loads, times the instantiation
    got = _assert_sides("k_post loads x instantiation", b, lambda c: post(*c),
                        [(t, k) for t in (True, False) for k in (0, 1, 2, 3)])
    for W in (8, 9, 130):
        assert not any(post(W, K)[0] for K in fv.POST_KS), W
    for W in (64, 256, 260):
        assert all(post(W, K)[0] for K in fv.POST_KS), W
    assert [post(48, K)[0] for K in fv.POST_KS] == [True] * 6 + [False] * 3       # TMA up to K = 5
    # what test_post_every_dilation_on_random_state runs each W for
    for W in fv.POST_SIZES:
        paths = set()
        for K in fv.POST_KS:
            tma, inst = post(W, K)
            paths.add((tma, inst))
            if W == 48:
                assert tma == (K <= 5)
        assert len({k for _, k in paths}) == 4 and len({t for t, _ in paths}) == (2 if W == 48 else 1), paths
    assert max(K for _, K in fv.POST_CASES) == 8 and min(fv.POST_SIZES) == 8
    k = ph.constants()
    assert 260 % k["PT_X"] and 260 % k["PT_Y"]                                         # partial edge tiles

    # ray box: empty (no cell within reach of any sensor), clipped by the map edge, several sensors
    for W in fv.POSE_SIZES:
        c = [(cid, ts) for cid, ts in fv.pose_cases(W)]

        def box_side(ts, W=W):
            box = ph.ray_box(W, fv.CORE_RES, fv.CORE_RAY, ts)
            if fv.box_empty(box):
                return "empty"
            return "clipped" if box[0] == 0 or box[2] == 0 or box[1] == W or box[3] == W else "interior"
        got = _assert_sides(f"ray box at {W}", c, box_side, ["empty", "clipped"])
        empty = [cid for cid, ts in c if box_side(ts) == "empty"]
        assert empty == ["beyond-far-rows", "beyond-far-cols", "beyond-far-both"], (W, empty)
        assert box_side(dict(c)["two-sensors"]) != "empty"
        assert box_side(dict(c)["beyond-near"]) == "clipped"
        # what test_sensor_poses_at_and_beyond_the_map_edge runs each pose for
        sides = set()
        for cid, ts in c:
            box = ph.ray_box(W, fv.CORE_RES, fv.CORE_RAY, ts)
            sides.add(fv.box_empty(box))
            assert fv.box_empty(box) == cid.startswith("beyond-far"), (cid, box)
        assert sides == {True, False}

    # input layouts: where the index pass reads the rows and which load it takes; more than 64 sensors
    paths = {fv.layout_path(lay) for lay in fv.LAYOUTS}
    assert {"staged", "zero-copy", "device"} == {w for w, _ in paths}
    assert ("device", True) in paths and ("device", False) in paths
    assert fv.MANY_SENSORS > 64


def test_march_table_restatement():
    """the library's march table against the oracle's loop (emap_oracle.c:527) at the cases' parameters"""
    for W, res, L in {fv.frame_params(c) for c in fv.RES_CASES}:
        st = ph.plan(W, res, L)["steps"]
        step = res / np.sqrt(2.0)
        s, ref = fv.h16(step), []
        while s < fv.h16(L):
            ref.append(s)
            s = fv.h16(s + step)
        assert np.array_equal(st, np.array(ref, np.float32)), (res, L)
        # the oracle loops for ever once the fp16 march variable stops advancing: every case stays below that point
        assert fv.h16(float(st[-1]) + step) > st[-1], (res, L)


def _random_frames(W, res, L, rng, n):
    """seeded sensor sets: one inside, one at an edge, one outside, 2..8 spread across (and beyond) the map"""
    half = 0.5 * W * res
    for i in range(n):
        kind = i % 4
        if kind == 0:
            ts = [rng.uniform(-half, half, 2)]
        elif kind == 1:
            t = rng.uniform(-half, half, 2)
            ax = rng.integers(2)
            t[ax] = rng.choice([-1, 1]) * (half + rng.uniform(-3, 3) * res)
            ts = [t]
        elif kind == 2:
            t = rng.uniform(-half, half, 2)
            for ax in np.flatnonzero(rng.random(2) < 0.6) if rng.random() < 0.8 else [rng.integers(2)]:
                t[ax] = rng.choice([-1, 1]) * (half + rng.uniform(0, 2 * L))
            ts = [t]
        else:
            ts = [rng.uniform(-half - 0.5 * L, half + 0.5 * L, 2) for _ in range(rng.integers(2, 9))]
        yield [np.array([t[0], t[1], rng.uniform(-1, 2)], np.float32) for t in ts]


CONTAIN_CONFIGS = sorted({fv.frame_params(c) for c in fv.RES_CASES} |
                         {(W, fv.CORE_RES, fv.CORE_RAY) for W in fv.POSE_SIZES + [130, 1024]})


@pytest.mark.parametrize("W,res,L", CONTAIN_CONFIGS)
def test_ray_samples_stay_in_the_tiled_box(W, res, L):
    """Every sample at which k_raycast<false> forms a fine-tile address (a new cell) lies in the frame's ray box, and the
    address lies in the t8 region of the shared-memory layout: for seeded sensors inside, at an edge of and outside the
    map, and sets of up to 8 sensors."""
    rng = np.random.default_rng(W * 7 + int(res * 1000) + int(L * 10))
    plan = ph.plan(W, res, L)
    steps = plan["steps"]
    lo, hi = plan["off_t8"], plan["off_t8"] + 4 * ph.constants()["RT"] ** 2
    launched = checked = 0
    for frame in _random_frames(W, res, L, rng, 24):
        box = ph.ray_box(W, res, L, frame)
        r0, r1, c0, c1 = box[:4]
        for t in frame:
            d = rng.standard_normal((24, 3))
            d /= np.linalg.norm(d, axis=1, keepdims=True)
            pts = (t + d * rng.uniform(0.2, 1.5 * L, (24, 1))).astype(np.float32)
            rx, ry, _, length = fv.rays_of(t, pts, L)
            n_rays = int((length > steps[0]).sum()) if len(steps) else 0
            if not ph.raycast_runs(box, n_rays, len(steps)):
                continue
            launched += 1
            ix, iy, live = fv.march_cells(W, res, steps, t, rx, ry, length)
            m = fv.address_samples(W, ix, iy, live)
            ix, iy = ix[m], iy[m]
            checked += len(ix)
            out = ~((ix >= r0) & (ix < r1) & (iy >= c0) & (iy < c1))
            assert not out.any(), (f"sensor {t}: {int(out.sum())} samples outside box {box}, "
                                   f"first at cell ({ix[out][0]}, {iy[out][0]})")
            addr = fv.t8_address(plan, box, ix, iy)
            assert ((addr >= lo) & (addr < hi)).all(), (t, box, int(addr.min()), int(addr.max()), lo, hi)
    assert launched > 10 and checked > 0, (launched, checked)


def test_empty_box_frames_have_rays():
    """the sensors beyond the map have rays (validity does not depend on the map) whose samples all clamp to the border
    ring, and their box is empty: k_raycast<false> is not launched for them"""
    for W in fv.POSE_SIZES:
        for cid, ts in fv.pose_cases(W):
            box = ph.ray_box(W, fv.CORE_RES, fv.CORE_RAY, ts)
            if not fv.box_empty(box):
                continue
            steps = ph.plan(W, fv.CORE_RES, fv.CORE_RAY)["steps"]
            t = np.array(ts[0], np.float32)
            pts = t + np.array([[3.0, 1.0, -1.0], [-2.0, -4.0, -1.2], [0.5, 6.0, -0.8]], np.float32)
            rx, ry, _, length = fv.rays_of(t, pts, fv.CORE_RAY)
            ix, iy, live = fv.march_cells(W, fv.CORE_RES, steps, t, rx, ry, length)
            assert live.any()
            on_ring = (ix == 0) | (ix == W - 1) | (iy == 0) | (iy == W - 1)
            assert on_ring[live].all(), cid
            assert not ph.raycast_runs(box, 3, len(steps))
            assert ph.raycast_runs(box, 3, len(steps), count_rays=True)
