"""Map initialiser timing (DESIGN.md §4j): initialize_map as the parent commit ran it (clear, get_state, SciPy griddata
over every cell on the host, set_state, emap_initialize_map_finish; restated inline below) against the device path
(initialize_map -> emap_initialize_map), and the interpolation kernel alone (k_init_interp / k_init_nearest, device
time from torch.profiler).  W = 1024 and 2048, nearest / linear / cubic, 5, 200 and 20 000 points.  Call times are host
clocks around a call that ends in a device synchronisation, median of --reps.  Prints the card and its power limit.
Usage: python tools/initialize_map_timing.py [--reps N]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "unknown"
    return f"{torch.cuda.get_device_name(0)}; power limit, max SM clock: {q}"


def old_initialize_map(em, points, method):
    """The parent commit's ElevationMap.initialize_map body."""
    from scipy.interpolate import griddata
    from elevation_mapping_cupy_b200.elevation_mapping import _to_host
    em.clear()
    pts = np.array(_to_host(points), dtype=np.float32, copy=True)
    center = em.center
    W = em.cell_n
    idx = ((pts[:, :2] - center[:2].reshape(1, 2)) / np.float32(em.resolution) + W / 2).astype(np.int32)
    pts[:, :2] = idx.astype(np.float32)
    pts[:, 2] -= center[2]
    state, normal = em.get_state()
    vi = np.where(state[2] > 0.5)
    points_idx = np.vstack([np.stack(vi).T.astype(np.float32), pts[:, :2]])
    values = np.hstack([state[0][vi], pts[:, 2]])
    gx, gy = np.mgrid[0:W, 0:W]
    interp = griddata(points_idx, values, (gx, gy), method=method)
    ok = ~np.isnan(interp)
    state[0] = np.nan_to_num(interp).astype(np.float32)
    state[1] = np.where(ok, np.float32(em.param.initialized_variance), np.float32(em.param.initial_variance))
    state[2] = ok.astype(np.float32)
    with em.map_lock:
        em.set_state(state)
        em._check(em._L.emap_initialize_map_finish(em._h, int(em.param.dilation_size_initialize), 2))


def points(W, n, seed=0):
    rng = np.random.default_rng(seed)
    half = (W - 2) * 0.04 / 2
    if n == 5:       # the TF initializer: the base and a 1 m square around it
        return np.array([[0, 0, 0.1]] + [[sx * 0.5, sy * 0.5, 0.1] for sx in (-1, 1) for sy in (-1, 1)], np.float32)
    return np.c_[rng.uniform(-half, half, (n, 2)), rng.normal(0, 0.3, n)].astype(np.float32)


def median_ms(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def kernel_ms(em, pts, method, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    em.initialize_map(pts, method)
    em.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            em.initialize_map(pts, method)
        em.synchronize()
        torch.cuda.synchronize()
    us = [e.device_time_total for e in prof.key_averages() if e.key.startswith("void k_init_interp")
          or e.key.startswith("void k_init_nearest") or e.key.startswith("k_init_interp") or e.key.startswith("k_init_nearest")]
    return sum(us) / reps / 1e3 if us else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    torch.cuda.init()
    print(_card())
    print("| W | points | method | parent path (ms) | initialize_map (ms) | kernel (ms) | planes 0-2 equal |")
    print("|---|---|---|---|---|---|---|")
    for W in (1024, 2048):
        em = ElevationMap(core_parameter(W))
        for n in (5, 200, 20000):
            pts = points(W, n)
            for method in ("nearest", "linear", "cubic"):
                reps = max(1, args.reps if not (method == "nearest" and n == 20000) else 2)
                t_old = median_ms(lambda: (old_initialize_map(em, pts, method), em.synchronize()), reps)
                a, _ = em.get_state()
                t_new = median_ms(lambda: (em.initialize_map(pts, method), em.synchronize()), reps)
                b, _ = em.get_state()
                eq = "yes" if np.array_equal(a[:3], b[:3]) else f"{int((a[:3] != b[:3]).sum())} cells differ"
                k = kernel_ms(em, pts, method, reps)
                print(f"| {W} | {n} | {method} | {t_old:.1f} | {t_new:.2f} | {k:.3f} | {eq} |", flush=True)


if __name__ == "__main__":
    main()
