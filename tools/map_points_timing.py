"""Map point cloud, normal arrows and normal colour timing (DESIGN.md §4i): the device calls (get_map_points,
get_normal_arrows, the `normal_color` export) against the host route a caller without them takes: one batched export of
elevation and normal_x/y/z into a host array, then NumPy compaction, arrows and colour (tests/map_points_oracle.py).

At 1024^2 and 2048^2, on maps built from LiDAR frames and on the same maps with every cell made valid (the most rows
a call can return: (W-2)^2 points; normals shorter than 0.1 are set to +z so every cell has an arrow too).  Call times
are host wall clock around calls that end in a device synchronisation (median, p10, p90 over --reps calls after
warm-up).  Kernel times (k_mapcloud count / write passes,
k_mapcloud_scan, k_export_multi) come from torch.profiler in a separate pass.  The device and host routes are checked
to give the same bytes before they are timed.  Prints the card, its power limit and SM clocks with the numbers; with
--out DIR it also writes DIR/map_points_timing.md.  Usage: python tools/map_points_timing.py [--reps N] [--out DIR]
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
import map_points_oracle as MO      # noqa: E402

NAMES = ["elevation", "normal_x", "normal_y", "normal_z"]


def _card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "unknown"
    return f"{torch.cuda.get_device_name(0)}; power limit, max SM clock, current SM clock: {q}"


def _map(W):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    em = ElevationMap(core_parameter(W))
    for f in range(3):
        pts, R, t = wl.lidar_cloud(1, f)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    return em


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


def _kernel_ms(fns, reps):
    """{kernel name: mean device ms per launch} over reps rounds of fns, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            for fn in fns:
                fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        for key, tag in (("k_mapcloud_scan", "scan"), ("k_mapcloud<false, false>", "count, points"),
                         ("k_mapcloud<true, false>", "count, arrows"), ("k_mapcloud<false, true>", "write, points"),
                         ("k_mapcloud<true, true>", "write, arrows"), ("k_export_multi", "k_export_multi")):
            if key in e.name:
                out.setdefault(tag, []).append(e.device_time / 1e3)
    return {k: (np.mean(v), len(v)) for k, v in out.items()}


def _run(em, W, scene, reps, lines, kernels):
    Wo = W - 2
    full = np.zeros((len(NAMES), Wo, Wo), np.float32)
    colour = np.zeros((Wo, Wo), np.float32)
    res, c = em.resolution, em.center

    def export():
        em.get_maps_with_names_ref(NAMES, full)

    def host_points():
        export()
        return MO.map_points(full[0], res, c)

    def host_arrows():
        export()
        return MO.normal_arrows(full[0], full[1], full[2], full[3], res, c)

    def host_colour():
        export()
        return MO.normal_color(full[1], full[2], full[3])

    def dev_colour():
        em.get_map_with_name_ref("normal_color", colour)

    pts, (ids, seg) = em.get_map_points(), em.get_normal_arrows()
    dev_colour()
    hp, (hi, hs), hc = host_points(), host_arrows(), host_colour()
    assert pts.tobytes() == hp.tobytes() and ids.tobytes() == hi.tobytes() and seg.tobytes() == hs.tobytes()
    assert colour.tobytes() == hc.tobytes()
    t_exp = _time(export, reps)
    f = lambda t: f"{t[0]:.3f} ({t[1]:.3f}-{t[2]:.3f})"
    for label, n, dev, host in (("points", len(pts), em.get_map_points, host_points),
                                ("arrows", len(ids), em.get_normal_arrows, host_arrows),
                                ("normal_color", Wo * Wo, dev_colour, host_colour)):
        row = f"| {W}², {scene} | {label} | {n} | {f(_time(dev, reps))} | {f(_time(host, reps))} | {f(t_exp)} |"
        lines.append(row)
        print(row, flush=True)
    for tag, (ms, n) in sorted(_kernel_ms([em.get_map_points, em.get_normal_arrows, dev_colour], reps).items()):
        kernels.append(f"| {W}², {scene} | {tag} | {ms * 1e3:.1f} ({n} launches) |")


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("map_points_timing needs a CUDA device")
    card = _card()
    lines = [f"card: {card}", "",
             "| map | output | rows | device call (ms) | host route (ms): export + NumPy | of which export (ms) |",
             "|---|---|---|---|---|---|"]
    kernels = []
    print(lines[0])
    for W in (1024, 2048):
        em = _map(W)
        for scene in ("LiDAR", "every cell valid"):
            if scene != "LiDAR":
                m, nm = em.get_state()
                m[2] = 1.0                                      # is_valid
                m[0] = np.nan_to_num(m[0], nan=0.0)
                short = np.sqrt((nm ** 2).sum(0)) < 0.1
                nm[0][short], nm[1][short], nm[2][short] = 0.0, 0.0, 1.0
                em.set_state(m, nm)
            _run(em, W, scene, args.reps, lines, kernels)
        em.close()
    lines += ["", "| map | kernel | µs per launch |", "|---|---|---|"] + kernels
    print("\n".join(lines[-len(kernels) - 3:]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "map_points_timing.md"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
