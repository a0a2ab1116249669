"""GPU: multi-frame sequences in which k_finalize's scratch groups occur on their own, bit for bit against the oracle
(bar as in tests/test_gpu_parity.py).  k_finalize reads a cell's points group (cnt_fo, SH, SV, last) only where
k_index_error set its points marker and its rays group (n_ray, ukv, DV) only where k_raycast set its rays marker, and
clears both markers: a marker missing where a group was written, or one left set from an earlier frame, shows here.
tests/test_finalize_groups_cpu.py checks on the oracle that each sequence reaches its group.  Both k_finalize
variants run: 4 cells per thread at 256², 1 at 203²."""
import numpy as np
import pytest

import finalize_groups as fg
from helpers import check_frame, compare_state

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("W", [256, 203])
@pytest.mark.parametrize("name", fg.SCENARIOS)
def test_finalize_groups_against_oracle(oracle_mod, name, W):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    kw, init, frames = fg.scenario(name, W)
    p = core_parameter(W, **kw)
    em = ElevationMap(p)
    om = oracle_mod.OracleElevationMap(p, nthreads=0)
    if init is not None:
        em.set_state(init[0], init[1])
        om.elevation_map = init[0].copy(); om.normal_map = init[1].copy()
    for f, (pts, R, t) in enumerate(frames):
        for m in (em, om):
            m.move_to(t, R)
            m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        check_frame(em, om, len(pts), f"{name} {W}² frame {f}")
        for m in (em, om):
            m.update_variance(); m.update_time()
        state, normal = em.get_state()
        compare_state(state, normal, om, label=f"{name} {W}² frame {f} after ticks")
