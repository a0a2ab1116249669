"""Times ElevationMap.signed_distance_field (emap_signed_distance_field) and sdf_values (emap_sdf_values) with device
input and output: the field of the node's 3 m x 3 m window of terrain.png at 0.04 m (75^2 cells, the default height
clearance) and of a 2047^2 window with 32 slices, and 10^6 queries against the 2047^2 field.  Each against a copy of the
layer (or volume and points) to the host plus the restatement tests/sdf_oracle.py on the host (NumPy + scipy's exact
feature transform for the field, Python floats for the queries, timed on 10^4 points and scaled; a stand-in for building
the field on the host, not a tuned CPU implementation).  CUDA events over --reps calls after warm-up.  Prints one JSON
line with the card's name and power limit, read in the same run.
  python tools/sdf_timing.py [--reps 20] [--host-reps 1]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from plane_segmentation_timing import card   # noqa: E402
from planar_regions_timing import _device_ms   # noqa: E402


def main():
    import numpy as np
    import torch
    import plane_scenes as S
    import sdf_oracle as O
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    em = ElevationMap(core_parameter(202))
    img = S.terrain_image(np.load(S.GOLDEN)["grey__terrain"], 1.25)
    c = img.shape[0] // 2
    node = img[c - 37:c + 38, c - 37:c + 38]                   # the node's 3 m window: 75^2 cells at 0.04 m
    rows = []
    field = None
    for label, layer, z_range in (("node 3 m window", node, None), ("2047^2 window, 32 slices", S.big_image(),
                                                                     (0.3, 0.3 + 31.5 * S.RES))):
        grid = {"layers": {"elevation": torch.as_tensor(np.ascontiguousarray(layer), device="cuda")},
                "centre": np.zeros(2), "resolution": S.RES}
        f = em.signed_distance_field(grid, z_range=z_range)
        if z_range is None:
            z_range = (f["z_min"], f["z_min"] + (f["n_z"] - 0.5) * S.RES)   # the same slices without the read-back
        out = f["volume"]
        ms = _device_ms(lambda: em.signed_distance_field(grid, z_range=z_range, out=out), a.reps)
        row = {"case": label, "grid": list(layer.shape), "n_z": f["n_z"], "device_ms": round(ms, 4)}
        t = time.perf_counter()
        for _ in range(a.host_reps):
            h = grid["layers"]["elevation"].cpu().numpy()
            O.field(h, f["z_min"], f["n_z"], S.RES)
        row["copy_and_host_restatement_ms"] = round((time.perf_counter() - t) * 1e3 / a.host_reps, 2)
        rows.append(row)
        field = f
    n = 1_000_000
    vol = field["volume"]
    pts = torch.as_tensor(np.random.default_rng(0).uniform(-45.0, 45.0, (n, 3)), device="cuda")
    pts[:, 2] = pts[:, 2] / 30.0 + 0.8
    qout = torch.empty((n, 4), dtype=torch.float64, device="cuda")
    ms = _device_ms(lambda: em.sdf_values(field, pts, out=qout), a.reps)
    row = {"case": "10^6 queries, 2047^2 x 32 field", "device_ms": round(ms, 4)}
    m = 10_000
    t = time.perf_counter()
    hv, hp = vol.cpu().numpy(), pts.cpu().numpy()
    t1 = time.perf_counter()
    O.values(hv, field["position"], S.RES, field["z_min"], hp[:m])
    t2 = time.perf_counter()
    row["copy_and_host_restatement_ms"] = round(((t1 - t) + (t2 - t1) * (n / m)) * 1e3, 1)
    rows.append(row)
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power, "reps": a.reps, "rows": rows}))


if __name__ == "__main__":
    main()
