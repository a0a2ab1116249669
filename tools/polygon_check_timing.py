"""Timing of the polygon safety check (emap_polygon_traversability) at 1024^2 and 2048^2.

    python tools/polygon_check_timing.py [--calls 200] [--out result.json]

For each map size and polygon it reports
  * call_us:    host clock around the whole C call (argument checks, H2D of the vertices, both kernels, the D2H copy and
                the synchronisation), median over --calls calls;
  * python_us:  the same through ElevationMap.get_polygon_traversability;
  * k_polygon_us / k_hull_us: kernel durations from torch.profiler (CUDA activity), median over the profiled calls.
The device name and power limit are read in the same run.  Polygons: an 8-vertex footprint of 0.5 m across at the map
centre, and a regular 64-gon covering half of the map.  The map is a seeded random state (90 % valid, 2 % of the cells
untraversable).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def regular(n, r):
    a = 2 * np.pi * np.arange(n) / n
    return np.stack([r * np.cos(a), r * np.sin(a)], 1).astype(np.float32)


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return {"device": name, "power_limit": power}
    except Exception as e:                        # the numbers still stand, but say where they came from
        import torch
        return {"device": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    assert torch.cuda.is_available(), "needs a CUDA device"
    rows = []
    for W in (1024, 2048):
        p = core_parameter(W)
        em = ElevationMap(p)
        rng = np.random.default_rng(W)
        st = np.zeros((7, W, W), np.float32)
        st[2] = (rng.random((W, W)) < 0.9).astype(np.float32)
        st[3] = np.where(rng.random((W, W)) < 0.02, rng.random((W, W)) * 0.5, 1.0).astype(np.float32)
        em.set_state(st)
        side = (W - 2) * p.resolution
        for name, poly in (("footprint8_0.5m", regular(8, 0.25)), ("half_map_64", regular(64, side / np.sqrt(2 * np.pi)))):
            res = np.zeros(3)
            ring = np.zeros((2 * (W - 2) + 1, 2))
            cap = C.c_int32(len(ring))
            mask = em.mask
            call = lambda: em._L.emap_polygon_traversability(em._h, poly.ctypes.data, len(poly), None, p.safe_thresh,
                                                             p.safe_min_thresh, p.max_unsafe_n, res.ctypes.data,
                                                             ring.ctypes.data, C.byref(cap), mask.data_ptr())
            for _ in range(20):                 # warm-up: module load, scratch allocation
                cap.value = len(ring)
                assert call() == 0
            ts = []
            for _ in range(args.calls):
                cap.value = len(ring)
                t0 = time.perf_counter()
                rc = call()
                ts.append(time.perf_counter() - t0)
                assert rc == 0
            out = np.zeros(3)
            tp = []
            for _ in range(args.calls):
                t0 = time.perf_counter()
                n_ring = em.get_polygon_traversability(poly, out)
                tp.append(time.perf_counter() - t0)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(50):
                    cap.value = len(ring)
                    call()
            durs = {}
            for ev in prof.events():
                if ev.device_type.name == "CUDA" and ("k_polygon" in ev.name or "k_hull" in ev.name):
                    durs.setdefault("k_polygon" if "k_polygon" in ev.name else "k_hull", []).append(ev.device_time)
            row = dict(cell_n=W, polygon=name, vertices=len(poly), call_us=1e6 * float(np.median(ts)),
                       python_us=1e6 * float(np.median(tp)), ring_len=int(n_ring), is_safe=float(out[0]),
                       t=float(out[1]), mask_cells=int(mask.sum().item()),
                       k_polygon_us=float(np.median(durs.get("k_polygon", [np.nan]))),
                       k_hull_us=float(np.median(durs.get("k_hull", [np.nan]))))
            rows.append(row)
            print(json.dumps(row))
        em.close()
    info = device_info()
    print(json.dumps(info))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
