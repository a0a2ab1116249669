"""Times ElevationMap.planar_terrain on the device against extract_planar_regions alone, so that the post-processing's
cost shows, and against what a user without it runs: a device-to-host copy of extract_planar_regions' layers followed
by the host restatement tests/planar_terrain_oracle.py (NumPy + cv2; a stand-in for the node's C++, not the node
itself).  Windows: the node's 76^2 (3 m at 0.04 m) and the whole 200^2 default map after LiDAR frames, and the whole
2047^2 window of a 2049^2 map.  Every timed call passes the exact table capacities of a first call.  Device and host
output are the mean of --reps calls; the host restatement the mean of --host-reps.  "kernels_ms" is a
torch.profiler run of its own: the device time per call of each post-processing kernel.  Prints one JSON line with the
card's name and power limit.
  python tools/planar_terrain_timing.py [--reps 20] [--host-reps 1]"""
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
        import planar_terrain_oracle as TO
    except ImportError:
        TO = None
    p = S.params()
    rows = []
    for label, W, ln in (("node 76^2 window, 202^2 map", 202, (3.0, 3.0)),
                         ("whole 200^2 default map", 202, (8.0, 8.0)),
                         ("whole 2047^2 window, 2049^2 map", 2049, (100.0, 100.0))):
        em = ElevationMap(core_parameter(W))
        if W == 2049:
            S.set_image(em, S.big_image())
            pos = (0.0, 0.0)
        else:
            S.lidar_frames(em)
            pos = S.lidar_window(em.center) if ln[0] < 8.0 else tuple(float(v) for v in em.center[:2])
        r0 = em.planar_terrain(pos, ln, p)
        caps = tuple(len(r0["tables"][k]) for k in ("regions", "polygons", "vertices"))
        n_rows, n_cols = r0["size"]
        out = torch.empty(10 * n_rows * n_cols, dtype=torch.float32, device="cuda")
        reg_ms = _device_ms(lambda: em.extract_planar_regions(pos, ln, p, out=out, capacities=caps), a.reps)
        ter_ms = _device_ms(lambda: em.planar_terrain(pos, ln, p, out=out, capacities=caps), a.reps)
        t = time.perf_counter()
        for _ in range(a.reps):
            em.planar_terrain(pos, ln, p, capacities=caps)
        host_out_ms = (time.perf_counter() - t) * 1e3 / a.reps
        kernels = _kernels_ms(lambda: em.planar_terrain(pos, ln, p, out=out, capacities=caps))
        row = {"case": label, "window": [n_rows, n_cols],
               "extract_planar_regions_device_ms": round(reg_ms, 4), "planar_terrain_device_ms": round(ter_ms, 4),
               "postprocess_device_ms": round(ter_ms - reg_ms, 4),
               "planar_terrain_host_out_ms": round(host_out_ms, 4),
               "kernels_ms": {k: v for k, v in kernels.items() if "k_pp_" in k or "fill" in k}}
        if TO is not None:
            res = float(em.resolution)
            t = time.perf_counter()
            for _ in range(a.host_reps):
                r = em.extract_planar_regions(pos, ln, p, capacities=caps)
                TO.postprocess(r["layers"]["elevation"], r["layers"]["plane_classification"], res, p)
            row["copy_plus_host_oracle_ms"] = round((time.perf_counter() - t) * 1e3 / a.host_reps, 2)
        else:
            row["copy_plus_host_oracle_ms"] = "not measured: cv2 is not importable"
        rows.append(row)
        del em
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power,
                      "device_ms": "CUDA events, device output, mean of reps",
                      "host_out_ms": "host clock, host output (ends in a synchronisation), mean of reps",
                      "copy_plus_host_oracle_ms": "host clock, mean of host-reps",
                      "host_path": "extract_planar_regions with host output + NumPy/cv2 post-processing, "
                                   "not the reference's C++",
                      "results": rows}))


if __name__ == "__main__":
    main()
