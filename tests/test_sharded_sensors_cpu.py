"""CPU tests of the host logic of sharded depth and semantic frames: the exchange-2 split into the arrays that gate the
ray-cast and the ones read in phase 3, and the pixel offsets and overlap height of sharded depth frames (gloo,
world size 2)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exchange2_defers_everything_but_the_fused_counts():
    from elevation_mapping_cupy_b200 import sharded
    # the list of exchange 2 with an averaged and a colour channel: SH, counts, last-writer keys, fsum, csum
    todo = [("SH", "SUM"), ("cnt_fo", "SUM"), ("last", "MAX"), ("fsum", "SUM"), ("csum", "SUM")]
    critical, deferred = sharded.split_exchange2(todo)
    assert critical == [("cnt_fo", "SUM")]
    assert deferred == [("SH", "SUM"), ("last", "MAX"), ("fsum", "SUM"), ("csum", "SUM")]
    assert sharded.split_exchange2(todo[:3]) == ([("cnt_fo", "SUM")], [("SH", "SUM"), ("last", "MAX")])


def test_depth_frame_offsets_without_a_collective():
    from elevation_mapping_cupy_b200 import sharded
    assert sharded.depth_frame_offsets(640 * 480, 1.25, static_offsets=(1234, 9999), overlap_z=0.5) == (1234, 0.5)


_GLOO_WORKER = r"""
import os, sys
sys.path.insert(0, %(root)r)
import numpy as np, torch.distributed as dist
from elevation_mapping_cupy_b200 import sharded
dist.init_process_group("gloo")
rk, ws = dist.get_rank(), dist.get_world_size()
# rank r has r + 1 cameras of 640x480 and 1 of 160x120; its first camera is at z = 1 + r / 8 (fp32)
pixels = [(r + 1) * 640 * 480 + 160 * 120 for r in range(ws)]
z = [float(np.float32(1.0 + r / 8 + 1e-7)) for r in range(ws)]
off, oz = sharded.depth_frame_offsets(pixels[rk], z[rk])
assert off == sum(pixels[:rk]) and oz == z[0], (off, oz)
off, oz = sharded.depth_frame_offsets(pixels[rk], z[rk], overlap_z=2.5)
assert off == sum(pixels[:rk]) and oz == 2.5
off, oz = sharded.depth_frame_offsets(pixels[rk], z[rk], static_offsets=(77 * rk, 0))
assert off == 77 * rk and oz == z[0]
dist.barrier()
if rk == 0:
    print("GLOO_DEPTH_OK")
dist.destroy_process_group()
"""


def test_depth_frame_offsets_gloo_world2(tmp_path):
    pytest.importorskip("torch")
    script = tmp_path / "w.py"
    script.write_text(_GLOO_WORKER % {"root": ROOT})
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29537", str(script)],
                       capture_output=True, text=True, timeout=240)
    assert "GLOO_DEPTH_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
