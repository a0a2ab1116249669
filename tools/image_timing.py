"""Camera image fusion timing (DESIGN.md §4g): ElevationMap.input_image against the reference's sequence on the same card.

At 1024^2 and 2048^2 maps built from LiDAR frames, a 1280 x 720 camera with 3 rgb planes and 2 feature planes
(channels rgb, p1, p2, feat_a, feat_b: one colour and four exponential channels), host and device images:
  * ours: one input_image call (host wall time per call, synchronised);
  * reference: EM.py:468-562 with its own kernels (oracle/_ref/libref_image_gpu_<tag>.so): image upload, uv *= 0,
    valid = False, the host sync of t_cam_map.get(), the correspondence kernel, and per channel one fusion launch and the
    layer copy semantic_map[idx] = new_map[idx].
Prints the card name and power limit with the numbers.  Usage: python tools/image_timing.py [--reps N]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import test_gpu_image as T
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    print(f"card: {name}, power limit: {pl}")
    H, Wi = 720, 1280
    K = T.intrinsics(H, Wi)
    D = np.zeros(5, np.float32)
    chans = ["rgb", "p1", "p2", "feat_a", "feat_b"]
    img = T._image(5, H, Wi, 0)
    img_d = torch.from_numpy(img).cuda()
    R, t = T.cam_pose(1)
    for W in (1024, 2048):
        em = T._map(W)
        ref = T.RefImage(W)
        em.input_image(img, chans, R, t, K, D, "none", H, Wi)           # adds the layers
        sm = em.semantic_map
        planes, kinds, layers = sm.update_layers_image(chans)
        chan = [(p, ["color", "exponential"][k], l) for p, k, l in zip(planes, kinds, layers)]

        def ours(x):
            em.input_image(x, chans, R, t, K, D, "none", H, Wi)
            torch.cuda.synchronize()

        state = em.elevation_map.clone()
        sem = sm.semantic_map.clone()
        center = em.center

        def reference(x):
            xd = torch.from_numpy(x).cuda() if isinstance(x, np.ndarray) else x
            torch.zeros(1, device="cuda").cpu()                             # t_cam_map.get()
            ref.fuse(state, center, sem, xd, K, D, "none", R, t, chan)
            torch.cuda.synchronize()

        for label, fn in (("ours", ours), ("reference", reference)):
            for src, x in (("host", img), ("device", img_d)):
                for _ in range(5):
                    fn(x)
                ts = []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    fn(x)
                    ts.append(time.perf_counter() - t0)
                ts = np.array(ts) * 1e3
                print(f"W={W} {src:6s} {label:9s} median {np.median(ts):.3f} ms  p10 {np.percentile(ts, 10):.3f}  "
                      f"p90 {np.percentile(ts, 90):.3f}")
        # device time of the kernel alone (CUDA events around reps calls of a device image)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.reps):
            em.input_image(img_d, chans, R, t, K, D, "none", H, Wi)
        ev1.record()
        torch.cuda.synchronize()
        print(f"W={W} device image, stream time per call: {ev0.elapsed_time(ev1) / args.reps:.3f} ms")


if __name__ == "__main__":
    main()
