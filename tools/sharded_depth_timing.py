"""Per-frame time of K = 4 depth cameras of 640x480 (workloads.depth_image) on a 1024^2 map, sharded over N GPUs
(ShardedElevationMap.input_depth_images, the cameras split into contiguous runs over the ranks), for N = 1 .. the
visible GPUs (at most 4) in both modes (nccl, multicast), against a single-GPU `input_depth_images` of all four.  With
no channels, and with rgb plus 4 class_average channels.  Each figure is the mean of `--iters` frames of device images
between CUDA events on rank 0 after `--warmup` frames, with a device synchronisation at the end.  Every line carries the
card's name and power limit.  Usage: python tools/sharded_depth_timing.py [--iters N] [--warmup W]
"""
import argparse
import json
import os
import signal
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elevation_mapping_cupy_b200 import workloads as wl                  # noqa: E402
from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap   # noqa: E402
from elevation_mapping_cupy_b200.parameter import core_parameter         # noqa: E402

K, MAP = 4, 1024
CHANNELS = {"none": [], "rgb+4ca": ["rgb", "ca0", "ca1", "ca2", "ca3"]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "unknown card"


def cameras(device):
    import torch
    out = []
    for s in range(K):
        depth, P, R, t = wl.depth_image(0, 640, 480, sensor=s)
        rng = np.random.default_rng(s)
        cam = dict(depth=depth, P=P, R=R, t=t, rgb=rng.integers(0, 256, (480, 640, 3), dtype=np.uint8),
                   features=rng.random((4, 480, 640), dtype=np.float32))
        out.append({k: torch.from_numpy(v).to(device) if k in ("depth", "rgb", "features") else v for k, v in cam.items()})
    return out


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


def worker(args):
    import torch
    import torch.distributed as dist
    from elevation_mapping_cupy_b200.sharded import ShardedElevationMap
    rk, ws = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rk)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{rk}"))
    cams = cameras(f"cuda:{rk}")
    mine = cams[rk * K // ws:(rk + 1) * K // ws]
    for name, ch in CHANNELS.items():
        em = ElevationMap(core_parameter(MAP), device=rk)
        sh = ShardedElevationMap(em, mode=args.mode)
        if sh.mode != args.mode:
            raise RuntimeError(f"mode {args.mode} unavailable")
        ms = time_frames(lambda: sh.input_depth_images(mine, 0.02, 0.02, channels=ch), args.warmup, args.iters)
        if rk == 0:
            print(json.dumps({"gpus": ws, "mode": sh.mode, "channels": name, "ms_per_frame": round(ms, 4)}), flush=True)
        dist.barrier()
        em.close()
    dist.destroy_process_group()


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--mode", default="nccl")
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    name = card()
    cams = cameras("cuda:0")
    for cname, ch in CHANNELS.items():
        em = ElevationMap(core_parameter(MAP), device=0)
        ms = time_frames(lambda: em.input_depth_images(cams, 0.02, 0.02, channels=ch), args.warmup, args.iters)
        print(json.dumps({"gpus": 1, "mode": "single", "channels": cname, "ms_per_frame": round(ms, 4), "card": name}),
              flush=True)
        em.close()
    for n in range(1, min(torch.cuda.device_count(), K) + 1):
        for mode in ("nccl", "multicast"):
            p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
                                  "--master-addr", "127.0.0.1", "--master-port", str(29650 + n), __file__, "--worker",
                                  "--mode", mode, "--iters", str(args.iters), "--warmup", str(args.warmup)],
                                 stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
            try:
                out = p.communicate(timeout=600)[0]
            except subprocess.TimeoutExpired:
                os.killpg(p.pid, signal.SIGKILL)
                out = p.communicate()[0] + "\n[timed out]"
            rows = [ln for ln in out.splitlines() if ln.startswith("{")]
            for ln in rows:
                print(json.dumps(dict(json.loads(ln), card=name)), flush=True)
            if not rows:
                print(json.dumps({"gpus": n, "mode": mode, "card": name, "error": out.strip().splitlines()[-1:]}),
                      flush=True)


if __name__ == "__main__":
    main()
