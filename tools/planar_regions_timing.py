"""Times ElevationMap.extract_planar_regions on the device against segment_planes alone and against what a user
without it runs: a device-to-host copy of the window (get_submap) followed by the host restatements
tests/plane_segmentation_oracle.py and tests/planar_regions_oracle.py (NumPy + cv2; a stand-in for the node's C++, not
the node itself).  Windows: the node's 75^2 (3 m at 0.04 m) and the whole 200^2 default map after LiDAR frames, and the
whole 2047^2 window of a 2049^2 map, and a 2047^2 floor with a lattice of single-cell obstacles (one plane with
about 10^5 holes: the largest plane-row bucket k_rg_rank meets).  Every timed call passes the exact table capacities
of a first call, so it runs the pipeline once; "retry_device_ms" times a call that starts from capacities of 1 row and
runs it twice.  "kernels_ms" is a torch.profiler run of its own: the device time per call of each region kernel.
Prints one JSON line with the card's name and power limit.
  python tools/planar_regions_timing.py [--reps 20] [--host-reps 1]"""
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


def _device_ms(call, reps):
    import torch
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _kernels_ms(call, reps=3, top=12):
    """Device time per call of each kernel (torch.profiler, CUDA activities), the `top` largest first (None: all)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = getattr(e, "self_cuda_time_total", 0.0)
        if t > 0:
            name = e.key.split("(")[0].replace("void ", "")
            tot[name] = tot.get(name, 0.0) + t / 1e3 / reps
    return {k: round(v, 4) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:top]}


def _lattice(n):
    import numpy as np
    z = np.zeros((n, n), np.float32)
    for dr in range(3):                # 3 x 3 blocks every 8 cells: a 3 x 3 median keeps them
        for dc in range(3):
            z[4 + dr::8, 4 + dc::8] = 0.3
    return z


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
        import plane_segmentation_oracle as PO
        import planar_regions_oracle as RO
    except ImportError:
        PO = RO = None
    p = S.params()
    rows = []
    for label, W, ln in (("node 76^2 window, 202^2 map", 202, (3.0, 3.0)),
                         ("whole 200^2 default map", 202, (8.0, 8.0)),
                         ("whole 2047^2 window, 2049^2 map", 2049, (100.0, 100.0)),
                         ("2047^2 floor with a lattice of obstacles", -2049, (100.0, 100.0))):
        lattice = W < 0
        W = abs(W)
        em = ElevationMap(core_parameter(W))
        if W == 2049:
            S.set_image(em, _lattice(W - 2) if lattice else S.big_image())
            pos = (0.0, 0.0)
        else:
            S.lidar_frames(em)
            pos = S.lidar_window(em.center) if ln[0] < 8.0 else tuple(float(v) for v in em.center[:2])
        r0 = em.extract_planar_regions(pos, ln, p)
        caps = tuple(len(r0["tables"][k]) for k in ("regions", "polygons", "vertices"))
        n_rows, n_cols = r0["size"]
        out = torch.empty(4 * n_rows * n_cols, dtype=torch.float32, device="cuda")
        seg_ms = _device_ms(lambda: em.segment_planes(pos, ln, p, out=out), a.reps)
        reg_ms = _device_ms(lambda: em.extract_planar_regions(pos, ln, p, out=out, capacities=caps), a.reps)
        retry_ms = _device_ms(lambda: em.extract_planar_regions(pos, ln, p, out=out, capacities=(1, 1, 1)), 3)
        assert em.extract_planar_regions(pos, ln, p, out=out, capacities=caps)["retried"] is False
        t = time.perf_counter()
        for _ in range(a.reps):
            em.extract_planar_regions(pos, ln, p, capacities=caps)
        host_out_ms = (time.perf_counter() - t) * 1e3 / a.reps
        kernels = _kernels_ms(lambda: em.extract_planar_regions(pos, ln, p, out=out, capacities=caps))
        row = {"case": label, "window": [n_rows, n_cols], "segment_planes_device_ms": round(seg_ms, 4),
               "extract_planar_regions_device_ms": round(reg_ms, 4),
               "extract_planar_regions_host_out_ms": round(host_out_ms, 4), "retry_device_ms": round(retry_ms, 4),
               "kernels_ms": kernels, "planes": len(r0["planes"]),
               "regions": len(r0["tables"]["regions"]), "polygons": len(r0["tables"]["polygons"]),
               "vertices": len(r0["tables"]["vertices"])}
        if PO is not None and not lattice:
            t = time.perf_counter()
            for _ in range(a.host_reps):
                w = em.get_submap(pos, ln, ["elevation"])
                o = PO.segment(w["layers"]["elevation"], S.RES, r0["origin"], p)
                RO.extract(o["segmentation"], o["planes"], r0["origin"], S.RES, p.margin_size,
                           p.extracted_planes_height_offset)
            row["copy_plus_host_oracle_ms"] = round((time.perf_counter() - t) * 1e3 / a.host_reps, 2)
        else:
            row["copy_plus_host_oracle_ms"] = "not measured" + ("" if lattice else ": cv2 is not importable")
        rows.append(row)
        del em
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power,
                      "device_ms": "CUDA events, device output, mean of reps",
                      "host_out_ms": "host clock, host output (ends in a synchronisation)",
                      "host_path": "get_submap D2H + NumPy/cv2 restatements, not the reference's C++",
                      "results": rows}))


if __name__ == "__main__":
    main()
