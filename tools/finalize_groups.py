"""Cells of k_finalize's full path on bench.py's config-B frames, by scratch group, and the loads and bytes they cost.

Runs the oracle on bench.py's frames (make_frames seeds, the same move / variance / time ticks between frames, no GPU)
and counts per frame the cells touched by points only, rays only, both, and the overlap-clear window alone; then the
full path's loads, requested bytes and distinct 32-byte sectors with the parent's 14 loads per cell and with the group
flags (tests/finalize_groups.py).  Prints one JSON line per frame and a summary line.

    python tools/finalize_groups.py [--frames 12] [--warmup 8]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import finalize_groups as fg   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from oracle import oracle as O
    n_pool = 8                                                    # bench.py N_FRAME_POOL
    frames = [wl.lidar_cloud(1, f, sensor=0, n_sensors=1) for f in range(n_pool)]
    om = O.OracleElevationMap(core_parameter(1024), nthreads=0)
    tot = {}
    for it in range(args.warmup + args.frames):
        f = it % n_pool
        pts, R, t = frames[f]
        om.move_to(t, R)                                          # bench.py between(): pose, then the ticks
        om.update_variance(); om.update_time()
        if it >= args.warmup:
            masks = fg.frame_groups(om, pts, R, t, 0.02, 0.02)
            c = fg.group_counts(*masks)
            tr = fg.load_traffic(*masks)
            row = dict(frame=it, pool_index=f, **c, traffic=tr)
            print(json.dumps(row), flush=True)
            for k, v in c.items():
                tot[k] = tot.get(k, 0) + v
            for arm in ("parent", "now"):
                for k, v in tr[arm].items():
                    tot[arm + "." + k] = tot.get(arm + "." + k, 0) + v
        om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    n = args.frames
    full = tot["full_path"]
    summ = {k: v / n for k, v in tot.items()}
    summ["share_single_group"] = (tot["points_only"] + tot["rays_only"]) / full
    for arm in ("parent", "now"):
        summ[arm + ".bytes_per_full_cell"] = tot[arm + ".bytes"] / full
        summ[arm + ".sector_bytes_per_full_cell"] = tot[arm + ".sector_bytes"] / full
        summ[arm + ".loads_per_full_cell"] = tot[arm + ".loads"] / full
    print(json.dumps({"summary_per_frame": summ, "frames": n, "cells": 1024 * 1024}), flush=True)


if __name__ == "__main__":
    main()
