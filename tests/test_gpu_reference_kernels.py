"""The engine's per-point cell records against the REFERENCE'S OWN kernels run on an H100: the CUDA-C strings of
kernels/custom_kernels.py built by nvcc for sm_90a and driven as CuPy launches them (tests/ref_gpu.py).  Their
write-back is deterministic, so its SHA-256 digests are stored in tests/golden/ref_gpu_index.json
(tests/golden/make_golden.py --gpu regenerates them) and compared bit for bit."""
import hashlib
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def index_cases():
    """(tag, parameters, cloud, R, t) of the comparison, rebuilt from seeds."""
    from elevation_mapping_cupy_b200.parameter import Parameter, core_parameter
    from elevation_mapping_cupy_b200 import workloads as wl
    out = []
    for tag, p, cloud in (("default202", Parameter(), "rand"), ("core1024", core_parameter(1024), "lidar")):
        p.update()
        if cloud == "rand":
            pts, R, t = wl.reference_test_cloud(3)
            pts = (pts * np.float32(9.0) - np.float32(4.5)).astype(np.float32)
        else:
            pts, R, t = wl.lidar_cloud(1, 2)
        out.append((tag, p, pts, R, t))
    return out


def record_digest(idx, valid, inside):
    """What ref_gpu_index.json stores for one cloud: counts (for the failure message) and SHA-256 of the arrays
    as int32 / uint8 / uint8."""
    arrays = {"idx": np.asarray(idx, np.int32), "valid": np.asarray(valid, np.uint8), "inside": np.asarray(inside, np.uint8)}
    d = {"n_points": int(len(arrays["idx"])), "n_valid": int(arrays["valid"].sum()), "n_inside": int(arrays["inside"].sum())}
    d.update({f"sha256_{k}": hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest() for k, v in arrays.items()})
    return d


def test_indices_bit_identical_to_reference_gpu_kernels():
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    gold = json.load(open(os.path.join(GOLD, "ref_gpu_index.json")))
    for tag, p, pts, R, t in index_cases():
        em = ElevationMap(p)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0, 0)
        idx, valid, inside = em.get_point_record(len(pts))
        assert record_digest(idx, valid, inside) == gold[tag], tag
