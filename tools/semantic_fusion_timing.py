"""Semantic point-channel fusion timing (DESIGN.md §4d): the config-B frame (200k-point LiDAR frames, ray-cast and overlap
clearance on) with 0 channels and with 4 channels of one fusion kind, at 1024^2 and 2048^2.

Each frame is a device cloud through ElevationMap.input_pointcloud; per-frame CUDA events on the handle's stream, with
move_to / update_variance / update_time untimed between frames, as bench.py times config B (no L2 flush here).  Prints
the median and the 10th / 90th percentiles per case, and the card name and power limit read in the same run.
Usage: python tools/semantic_fusion_timing.py [--frames N]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KINDS = ["average", "class_average", "color", "class_bayesian", "bayesian_inference", "class_max"]


def _features(rng, n, kind):
    if kind == "color":
        return rng.integers(0, 1 << 24, (n, 4)).astype(np.uint32).view(np.float32)
    if kind == "class_max":
        from oracle import semantic_ext as X
        return X.encode_max(rng.random((n, 4), dtype=np.float32), rng.integers(0, 20, (n, 4)))
    return rng.random((n, 4), dtype=np.float32)


def main():
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    args = ap.parse_args()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:        # noqa: BLE001
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    print(f"card: {q}")
    frames = [wl.lidar_cloud(1, f) for f in range(8)]
    rng = np.random.default_rng(0)
    for W in (1024, 2048):
        for kind in ["none"] + KINDS:
            p = core_parameter(W)
            chans = ["x", "y", "z"]
            if kind != "none":
                p.pointcloud_channel_fusions = {"default": kind}
                chans += [f"c{k}" for k in range(4)]
            em = ElevationMap(p)
            stream = torch.cuda.Stream()           # a real stream: handle 0 would give the library back its own
            torch.cuda.set_stream(stream)
            em.set_stream(stream.cuda_stream)
            dev = []
            for pts, R, t in frames:
                rows = pts if kind == "none" else np.concatenate([pts, _features(rng, len(pts), kind)], 1)
                dev.append(torch.from_numpy(np.ascontiguousarray(rows)).cuda())
            ts = []
            for it in range(args.frames + 10):
                f = it % len(frames)
                _, R, t = frames[f]
                em.move_to(t, R); em.update_variance(); em.update_time()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                em.input_pointcloud(dev[f], chans, R, t, 0.02, 0.02)
                e1.record(stream)
                e1.synchronize()
                if it >= 10:
                    ts.append(e0.elapsed_time(e1))
            ts = np.array(ts)
            print(f"W={W} {kind:18s} frame ms: median {np.median(ts):.4f}  p10 {np.percentile(ts, 10):.4f}  "
                  f"p90 {np.percentile(ts, 90):.4f}", flush=True)
            em.close()
            del dev
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
