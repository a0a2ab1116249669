"""Map window timing (DESIGN.md §4h): ElevationMap.get_submaps against a full-map get_maps_with_names_ref and a NumPy
crop of every window, which is what a caller without window export does.

At 1024^2 and 2048^2 maps built from LiDAR frames, batches of 1, 16 and 256 windows of 2 m x 2 m around the map centre
and one half-map window, with 3 layers (elevation, traversability, the `smooth` plugin layer) and 8 layers (the 6
exported state layers, normal_z, smooth):
  * full export + crop: get_maps_with_names_ref into a host array, then one NumPy copy per window and layer;
  * submaps, host output: one get_submaps call into a new NumPy array;
  * submaps, device output: one get_submaps call into a preallocated torch CUDA tensor, then torch.cuda.synchronize().
Times are host wall clock per call (median, p10, p90 over --reps calls after warm-up).  The device time of k_submap is
read from torch.profiler in a separate pass.  Prints the card, its power limit and SM clocks with the numbers; with
--out DIR it also writes DIR/submap_timing.md.  Usage: python tools/submap_timing.py [--reps N] [--out DIR]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PLUGIN_YAML = """
smooth_filter:
  enable: True
  fill_nan: False
  is_height_layer: True
  layer_name: "smooth"
  extra_params:
    input_layer_name: "elevation"
"""
LAYERS = {3: ["elevation", "traversability", "smooth"],
          8: ["elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound", "normal_z", "smooth"]}


def _card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "unknown"
    return f"{torch.cuda.get_device_name(0)}; power limit, max SM clock, current SM clock: {q}"


def _map(W, cfg_dir):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    cfg = os.path.join(cfg_dir, "plugin_config.yaml")
    with open(cfg, "w") as f:
        f.write(PLUGIN_YAML)
    em = ElevationMap(core_parameter(W, plugin_config_file=cfg))
    for f in range(3):
        pts, R, t = wl.lidar_cloud(1, f)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    return em


def _windows(em, n):
    """n windows of 2 m x 2 m within 8 m of the centre (n == 0: one half-map window)."""
    c = em.center.astype(np.float64)[:2]
    if n == 0:
        half = 0.5 * (em.cell_n - 2) * em.resolution
        return [(c, (half, half))]
    rng = np.random.default_rng(n)
    return [(c + rng.uniform(-8.0, 8.0, 2), (2.0, 2.0)) for _ in range(n)]


def _time(fn, reps):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    ts = np.array(ts) * 1e3
    return np.median(ts), np.percentile(ts, 10), np.percentile(ts, 90)


def _kernel_ms(em, reqs, names, out, reps):
    """Mean device time of k_submap over reps device-output calls, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            em.get_submaps(reqs, names, out=out)
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if "k_submap" in e.name]
    return (np.mean(ts) / 1e3, len(ts)) if ts else (float("nan"), 0)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("submap_timing needs a CUDA device")
    card = _card()
    lines = [f"card: {card}", "",
             "| map | windows | layers | cells / layer | full export + crop (ms) | submaps, host out (ms) | "
             "submaps, device out (ms) | k_submap (ms) |", "|---|---|---|---|---|---|---|---|"]
    print(lines[0])
    with tempfile.TemporaryDirectory() as tmp:
        for W in (1024, 2048):
            em = _map(W, tmp)
            Wo = W - 2
            for n in (1, 16, 256, 0):
                reqs = _windows(em, n)
                for nl, names in LAYERS.items():
                    res = em.get_submaps(reqs, names)
                    cells = sum(r["size"][0] * r["size"][1] for r in res)
                    full = np.zeros((nl, Wo, Wo), np.float32)
                    boxes = [(r["index"], r["size"]) for r in res]

                    def crop():
                        em.get_maps_with_names_ref(names, full)
                        return [full[:, r0:r0 + rows, c0:c0 + cols].copy() for (r0, c0), (rows, cols) in boxes]

                    dev = torch.empty(nl * cells, dtype=torch.float32, device="cuda")

                    def device():
                        em.get_submaps(reqs, names, out=dev)
                        torch.cuda.synchronize()

                    got = crop()
                    for k, r in enumerate(res):             # same values both ways
                        assert all(np.array_equal(got[k][j].view(np.uint32), r["layers"][nm].view(np.uint32))
                                   for j, nm in enumerate(names))
                    t_crop = _time(crop, args.reps)
                    t_host = _time(lambda: em.get_submaps(reqs, names), args.reps)
                    t_dev = _time(device, args.reps)
                    k_ms, k_n = _kernel_ms(em, reqs, names, dev, args.reps)
                    label = "half map" if n == 0 else f"{n} x 2 m"
                    f = lambda t: f"{t[0]:.3f} ({t[1]:.3f}-{t[2]:.3f})"
                    row = (f"| {W}² | {label} | {nl} | {cells} | {f(t_crop)} | {f(t_host)} | {f(t_dev)} | "
                           f"{k_ms:.4f} ({k_n} launches) |")
                    lines.append(row)
                    print(row, flush=True)
            em.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "submap_timing.md"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
