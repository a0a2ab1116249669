"""Times ElevationMap.plane_decomposition (emap_plane_decomposition) with device output: the node's 3 m x 3 m window of a
0.05 m map resampled to the node's 0.04 m (60^2 -> 75^2), and a 2047^2 window of a 0.02 m map resampled to 0.05 m
(2047^2 -> 818^2), each against planar_terrain on a window of the output size (the same pipeline without the
resampling, run on the resampled elevation, so the difference is mostly the resampling, the fill and median at the
input size and the grid's copy) and against the host restatement
tests/resample_oracle.py (NumPy + cv2: the fill, median, resampling, segmentation, regions and post-processing; a
stand-in for the node's C++, not the node itself).  "resample_kernel_ms" is k_rs_resample's device time per call from
a torch.profiler run of its own.  CUDA events over --reps calls after warm-up.  Prints one JSON line with the card's
name and power limit, read in the same run.
  python tools/plane_decomposition_timing.py [--reps 20] [--host-reps 1]"""
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
from planar_regions_timing import _device_ms, _kernels_ms   # noqa: E402


def main():
    import numpy as np
    import torch
    import plane_scenes as S
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    try:
        import cv2  # noqa: F401
        import resample_oracle as RS
    except ImportError:
        RS = None
    rows = []
    for label, W, res_map, res_new, ln in (("node 3 m window, 0.05 m -> 0.04 m", 202, 0.05, 0.04, 3.0),
                                           ("2047^2 window, 0.02 m -> 0.05 m", 2049, 0.02, 0.05, 100.0)):
        em = ElevationMap(core_parameter(W, resolution=res_map))
        S.set_image(em, S.big_image() if W == 2049 else S.synthetic("stairs", W - 2, 1))
        p = S.params(resolution=res_new)
        g_dev = torch.empty(W * W, dtype=torch.float32, device="cuda")
        grid = em.get_submap((0.0, 0.0), (ln, ln), ["elevation"], out=g_dev)
        if W == 202:                   # the node's 60^2 cells (the window at the origin has 61)
            layer = grid["layers"]["elevation"][:60, :60].contiguous()
            grid = dict(grid, layers={"elevation": layer}, size=(60, 60))
        r0 = em.plane_decomposition(grid, "elevation", p)
        caps = tuple(len(r0["tables"][k]) for k in ("regions", "polygons", "vertices"))
        n_rows, n_cols = r0["size"]
        out = torch.empty(10 * n_rows * n_cols, dtype=torch.float32, device="cuda")
        dec_ms = _device_ms(lambda: em.plane_decomposition(grid, "elevation", p, out=out, capacities=caps), a.reps)
        kernels = _kernels_ms(lambda: em.plane_decomposition(grid, "elevation", p, out=out, capacities=caps), top=None)
        # planar_terrain on a window of the output size of a map at the new resolution holding the resampled elevation
        em2 = ElevationMap(core_parameter(n_rows + 2, resolution=res_new))
        S.set_image(em2, np.ascontiguousarray(r0["layers"]["elevation_before_postprocess"]))
        side = n_rows * res_new
        p2 = S.params(resolution=res_new)
        t0 = em2.planar_terrain((0.0, 0.0), (side, side), p2)
        caps2 = tuple(len(t0["tables"][k]) for k in ("regions", "polygons", "vertices"))
        out2 = torch.empty(10 * t0["size"][0] * t0["size"][1], dtype=torch.float32, device="cuda")
        ter_ms = _device_ms(lambda: em2.planar_terrain((0.0, 0.0), (side, side), p2, out=out2, capacities=caps2), a.reps)
        row = {"case": label, "grid": list(grid["size"]), "resampled": [n_rows, n_cols],
               "plane_decomposition_device_ms": round(dec_ms, 4),
               "planar_terrain_same_size_window_device_ms": round(ter_ms, 4), "planar_terrain_window": list(t0["size"]),
               "resample_kernel_ms": round(sum(v for k, v in kernels.items() if "k_rs_resample" in k), 4)}
        if RS is not None:
            host = np.ascontiguousarray(grid["layers"]["elevation"].cpu().numpy())
            t = time.perf_counter()
            for _ in range(a.host_reps):
                RS.decompose(host, res_map, grid["centre"], p)
            row["host_restatement_ms"] = round((time.perf_counter() - t) * 1e3 / a.host_reps, 2)
        else:
            row["host_restatement_ms"] = "not measured: cv2 is not importable"
        rows.append(row)
        del em, em2
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power, "reps": a.reps, "rows": rows}))


if __name__ == "__main__":
    main()
