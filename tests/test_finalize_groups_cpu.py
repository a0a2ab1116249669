"""The frame sequences of tests/test_gpu_finalize_groups.py reach what they are for, on the oracle: each makes its
group of k_finalize's full-path cells occur (points only, rays only, overlap window only), and the no-ray frames have
neither marker anywhere.  Also the probe that recovers the rays set against the load accounting's invariants."""
import numpy as np
import pytest

import finalize_groups as fg

SIZES = [256, 203]


def _run(oracle_mod, name, W):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    kw, init, frames = fg.scenario(name, W)
    om = oracle_mod.OracleElevationMap(core_parameter(W, **kw), nthreads=0)
    if init is not None:
        om.elevation_map = init[0].copy(); om.normal_map = init[1].copy()
    out = []
    for pts, R, t in frames:
        om.move_to(t, R)
        masks = fg.frame_groups(om, pts, R, t, 0.02, 0.02)
        om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        out.append((masks, fg.group_counts(*masks), om.counts[1].copy()))
        om.update_variance(); om.update_time()
    return out


@pytest.mark.parametrize("W", SIZES)
@pytest.mark.parametrize("name", fg.SCENARIOS)
def test_scenario_reaches_its_group(oracle_mod, name, W):
    res = _run(oracle_mod, name, W)
    group = fg.SCENARIO_GROUP[name]
    assert max(c[group] for _, c, _ in res) > 0, [c for _, c, _ in res]
    for (pts_m, rays_m, win), c, cnt_all in res:
        assert np.array_equal(pts_m, cnt_all > 0)
        assert c["full_path"] == int((pts_m | rays_m | win).sum())
    if name == "rays_then_none":
        for k in (2, 3):
            pts_m, rays_m, _ = res[k][0]
            assert not pts_m.any() and not rays_m.any(), k
        assert res[1][1]["rays_only"] > 0 and res[4][1]["rays_only"] > 0


def test_load_accounting():
    W = 16
    pts_m = np.zeros((W, W), bool); rays_m = np.zeros((W, W), bool); win = np.zeros((W, W), bool)
    pts_m[0, 0] = True; rays_m[5, 5] = True; pts_m[9, 9] = rays_m[9, 9] = True; win[12, 12] = True
    t = fg.load_traffic(pts_m, rays_m, win)
    assert t["parent"]["loads"] == 4 * 14
    assert t["now"]["loads"] == 4 * 6 + 2 * 4 + 2 * 3
    assert t["parent"]["bytes"] == 4 * (24 + 40 + 16)
    assert t["now"]["bytes"] == 4 * 24 + 2 * 32 + 2 * 16
    assert t["now"]["sectors"] == 4 * 6 + 2 * 4 + 2 * 3      # isolated cells: one sector per load
