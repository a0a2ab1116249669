"""Timing of windows in the requester's frame (DESIGN.md §4h'): ElevationMap.get_transformed_submaps against what a
Python caller does without it, get_submaps followed by getTransformedMap on the host.

At 1024^2 and 2048^2 maps built from LiDAR frames, batches of 1, 16 and 256 windows of 2 m x 2 m within 8 m of the
centre, requested in a frame yawed by 30 degrees and shifted (a robot's base frame), with 3 layers (elevation,
traversability, the `smooth` plugin layer) and 8 layers (the 6 exported state layers, normal_z, smooth):
  * get_submaps + host: one get_submaps call into a new NumPy array, then per window the scatter of
    tests/transformed_submap_oracle.py on the host, vectorised (`parallel`; the literal per-cell loop is timed once,
    for one window, on the last line);
  * transformed, host output: one get_transformed_submaps call into a new NumPy array;
  * transformed, device output: one call into a preallocated torch CUDA tensor, then torch.cuda.synchronize().
Times are host wall clock per call (median, p10, p90 over --reps calls after warm-up; the host baseline over
--host-reps).  The device time of the three kernels (k_tsub_scatter twice, k_tsub_gather) per call is read from
torch.profiler in a separate pass.  Prints the card, its power limit and SM clocks with the numbers; with --out DIR it
also writes DIR/transformed_submap_timing.md.
Usage: python tools/transformed_submap_timing.py [--reps N] [--host-reps N] [--out DIR]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

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


def _requests(em, n):
    """n windows of 2 m x 2 m within 8 m of the centre, in a frame yawed by 30 degrees and shifted."""
    import transformed_submap_oracle as TO
    T = TO.iso(TO.rot(yaw=np.pi / 6), (1.3, -0.7, -0.4))
    R, t = T[:9].reshape(3, 3), T[9:]
    c = em.center.astype(np.float64)[:2]
    rng = np.random.default_rng(n)
    out = []
    for _ in range(n):
        p = c + rng.uniform(-8.0, 8.0, 2)
        q = R @ np.array([p[0], p[1], 0.0]) + t
        out.append(((q[0], q[1]), (2.0, 2.0), (R, t)))
    return out


def _host_path(em, reqs, names):
    """get_submaps at the map-frame positions, then the scatter per window on the host."""
    import transformed_submap_oracle as TO
    c = em.center.astype(np.float64)
    gs = [TO.geometry(em.cell_n, em.resolution, c, (p[0], p[1], ln[0], ln[1]), T) for p, ln, T in reqs]
    res = em.get_submaps([(g["map_position"], ln) for g, (p, ln, T) in zip(gs, reqs)], names)
    return [TO.parallel(r["layers"], g, T, em.resolution) for g, r, (p, ln, T) in zip(gs, res, reqs)]


def _time(fn, reps):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    ts = np.array(ts) * 1e3
    return np.median(ts), np.percentile(ts, 10), np.percentile(ts, 90)


def _kernel_ms(em, reqs, names, out, reps):
    """Mean device time per call of the three kernels over reps device-output calls, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            em.get_transformed_submaps(reqs, names, out=out)
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if "k_tsub_" in e.name]
    return (np.sum(ts) / reps / 1e3, len(ts)) if ts else (float("nan"), 0)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transformed_submap_timing needs a CUDA device")
    import transformed_submap_oracle as TO
    card = _card()
    lines = [f"card: {card}", "",
             "| map | windows | layers | cells / layer | get_submaps + host (ms) | transformed, host out (ms) | "
             "transformed, device out (ms) | kernels (ms / call) |", "|---|---|---|---|---|---|---|---|"]
    print(lines[0])
    with tempfile.TemporaryDirectory() as tmp:
        for W in (1024, 2048):
            em = _map(W, tmp)
            for n in (1, 16, 256):
                reqs = _requests(em, n)
                for nl, names in LAYERS.items():
                    res = em.get_transformed_submaps(reqs, names)
                    cells = sum(r["size"][0] * r["size"][1] for r in res)
                    for r, want in zip(res, _host_path(em, reqs, names)):        # same values both ways
                        assert all(np.array_equal(r["layers"][nm].view(np.uint32), want[nm].view(np.uint32))
                                   for nm in names)
                    dev = torch.empty(max(nl * cells, 1), dtype=torch.float32, device="cuda")

                    def device():
                        em.get_transformed_submaps(reqs, names, out=dev)
                        torch.cuda.synchronize()

                    t_base = _time(lambda: _host_path(em, reqs, names), args.host_reps)
                    t_host = _time(lambda: em.get_transformed_submaps(reqs, names), args.reps)
                    t_dev = _time(device, args.reps)
                    k_ms, k_n = _kernel_ms(em, reqs, names, dev, args.reps)
                    f = lambda t: f"{t[0]:.3f} ({t[1]:.3f}-{t[2]:.3f})"
                    row = (f"| {W}² | {n} x 2 m | {nl} | {cells} | {f(t_base)} | {f(t_host)} | {f(t_dev)} | "
                           f"{k_ms:.4f} ({k_n} launches) |")
                    lines.append(row)
                    print(row, flush=True)
            if W == 2048:
                p, ln, T = _requests(em, 1)[0]
                g = TO.geometry(em.cell_n, em.resolution, em.center.astype(np.float64), (p[0], p[1]) + ln, T)
                r = em.get_submaps([(g["map_position"], ln)], ["elevation"])[0]
                t_loop = _time(lambda: TO.sequential({"elevation": r["layers"]["elevation"]}, g, T, em.resolution), 3)
                row = f"literal per-cell loop on the host, 1 x 2 m window, elevation only: {t_loop[0]:.1f} ms"
                lines.append("")
                lines.append(row)
                print(row, flush=True)
            em.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "transformed_submap_timing.md"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
