"""Depth-camera frames three ways, per frame on one GPU (DESIGN.md §4k):
  (a) `input_depth_image` of device images: the frame reads the depth, confidence, rgb and feature planes itself;
  (b) the semantic sensor node's unprojection restated in torch on the device (mask, nonzero, fp64 x / y, gathered
      channels), then `input_pointcloud` of that device cloud;
  (c) the same cloud copied to the host, as the node hands it over, then `input_pointcloud` of the host cloud.
Sizes 640x480, 1280x720 and 1000x1000; channels none, rgb, and rgb + 4 class_average; maps 1024^2 and 2048^2.  Each
figure is the mean of `--iters` frames between CUDA events after `--warmup` frames, with a device synchronisation at
the end.  Every line carries the card's name and power limit.  Usage: python tools/depth_image_timing.py [--iters N]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elevation_mapping_cupy_b200 import workloads as wl                  # noqa: E402
from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap   # noqa: E402
from elevation_mapping_cupy_b200.parameter import core_parameter         # noqa: E402

CHANNELS = {"none": [], "rgb": ["rgb"], "rgb+4ca": ["rgb", "ca0", "ca1", "ca2", "ca3"]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown card"


def node_cloud_torch(depth, P, rgb, feats, conf, theta, channels):
    """pointcloud_node.py create_pcl_from_image in torch on the device (the fp64 promotion NumPy 2 applies)."""
    import torch
    keep = torch.isfinite(depth) & (depth > 0) & (depth < 8.0) & (conf >= theta)
    v, u = torch.nonzero(keep, as_tuple=True)                   # host synchronisation
    d = depth[v, u]
    cols = [((u.double() - P[0, 2]) * d.double() / P[0, 0]).float(), ((v.double() - P[1, 2]) * d.double() / P[1, 1]).float(), d]
    k = 0
    for ch in channels:
        if ch == "rgb":
            c = rgb[v, u].int()
            cols.append(((c[:, 0] << 16) | (c[:, 1] << 8) | c[:, 2]).view(torch.float32))
        else:
            cols.append(feats[k, v, u]); k += 1
    return torch.stack(cols, 1).contiguous()


def time_frames(fn, warmup, iters):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    name = card()
    theta = 10.0
    for (w, h) in [(640, 480), (1280, 720), (1000, 1000)]:
        depth, P, R, t = wl.depth_image(0, w, h)
        rng = np.random.default_rng(0)
        conf = rng.uniform(0.0, 20.0, depth.shape).astype(np.float32)
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        feats = rng.random((4, h, w), dtype=np.float32)
        d_depth, d_conf, d_rgb, d_feats = (torch.from_numpy(x).cuda() for x in (depth, conf, rgb, feats))
        Pt = torch.from_numpy(P)
        for W in (1024, 2048):
            for cname, channels in CHANNELS.items():
                p = core_parameter(W)
                p.pointcloud_channel_fusions = {"rgb": "color", "default": "class_average"}
                nf = sum(c != "rgb" for c in channels)
                kw = dict(channels=channels, rgb=d_rgb if "rgb" in channels else None,
                          features=d_feats[:nf] if nf else None, confidence=d_conf)
                em = ElevationMap(p)
                em.move_to(t, R)
                ta = time_frames(lambda: em.input_depth_image(d_depth, P, R, t, 0.02, 0.02, **kw), args.warmup, args.iters)
                names = ["x", "y", "z"] + channels
                mk = lambda: node_cloud_torch(d_depth, Pt, d_rgb, d_feats, d_conf, theta, channels)
                tb = time_frames(lambda: em.input_pointcloud(mk(), names, R, t, 0.02, 0.02), args.warmup, args.iters)
                tc = time_frames(lambda: em.input_pointcloud(mk().cpu().numpy(), names, R, t, 0.02, 0.02), args.warmup,
                                 args.iters)
                n_kept = int(em.get_frame_stats().n_points)
                print(f"{w}x{h} map {W}^2 channels {cname:8s} kept {n_kept:7d}: (a) depth frame {ta:.3f} ms  "
                      f"(b) torch cloud + device frame {tb:.3f} ms  (c) host cloud frame {tc:.3f} ms  [{name}]", flush=True)
                em.close()


if __name__ == "__main__":
    main()
