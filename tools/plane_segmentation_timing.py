"""Times ElevationMap.segment_planes on the device against what a user without it runs: a device-to-host copy of the
window (get_submap) followed by tests/plane_segmentation_oracle.py on the host (NumPy + cv2).  That host path is a
restatement, not the reference's C++ (grid_map, Eigen and CGAL are not part of this project), so its time is only a
stand-in for the node's.  Windows: the node's 75^2 (3 m at 0.04 m) and the whole 200^2 default map, both of a 202^2
map, and the whole 2047^2 window of a 2049^2 map.  Prints one JSON line with the card's name and power limit.
  python tools/plane_segmentation_timing.py [--reps 50] [--host-reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:                     # noqa: BLE001
        return "unknown", str(e)


def main():
    import torch
    import plane_scenes as S
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    try:
        import plane_segmentation_oracle as PO
        import cv2  # noqa: F401
    except ImportError:
        PO = None
    p = S.params()
    rows = []
    for label, W, pos, ln, img in (
            ("node 75^2 window, 202^2 map", 202, (0.0, 0.0), (3.0, 3.0), None),
            ("whole 200^2 default map", 202, (0.0, 0.0), (8.0, 8.0), None),
            ("whole 2047^2 window, 2049^2 map", 2049, (0.0, 0.0), (100.0, 100.0), None)):
        em = ElevationMap(core_parameter(W))
        if W == 2049:
            S.set_image(em, S.big_image())
        else:
            S.lidar_frames(em)
            pos = S.lidar_window(em.center) if ln[0] < 8.0 else tuple(float(v) for v in em.center[:2])
        r0 = em.segment_planes(pos, ln, p)
        n_rows, n_cols = r0["size"]
        out = torch.empty(4 * n_rows * n_cols, dtype=torch.float32, device="cuda")
        for _ in range(5):
            em.segment_planes(pos, ln, p, out=out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            em.segment_planes(pos, ln, p, out=out)
        e1.record()
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / a.reps
        t = time.perf_counter()
        for _ in range(a.reps):
            em.segment_planes(pos, ln, p)
        host_out_ms = (time.perf_counter() - t) * 1e3 / a.reps
        row = {"case": label, "window": [n_rows, n_cols], "device_out_ms": round(dev_ms, 4),
               "host_out_ms": round(host_out_ms, 4), "labels": r0["highest_label"], "planes": len(r0["planes"])}
        if PO is not None:
            t = time.perf_counter()
            for _ in range(a.host_reps):
                w = em.get_submap(pos, ln, ["elevation"])
                PO.segment(w["layers"]["elevation"], S.RES, r0["origin"], p)
            row["copy_plus_host_oracle_ms"] = round((time.perf_counter() - t) * 1e3 / a.host_reps, 2)
        else:
            row["copy_plus_host_oracle_ms"] = "not measured: cv2 is not importable"
        rows.append(row)
        del em
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power, "device_out_ms": "CUDA events, device output, mean of reps",
                      "host_out_ms": "host clock, host output (ends in a synchronisation)",
                      "host_path": "get_submap D2H + NumPy/cv2 restatement, not the reference's C++",
                      "results": rows}))


if __name__ == "__main__":
    main()
