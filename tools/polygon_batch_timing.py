"""Timing of the batch polygon check (emap_polygon_traversability_batch) against one single call per polygon.

    python tools/polygon_batch_timing.py [--calls 20] [--out result.json]

Maps of 1024^2 and 2048^2 in the seeded state of tools/polygon_check_timing.py (90 % valid, 2 % of the cells
untraversable).  Batches: B in {1, 16, 128, 1024, 4096} seeded 8-vertex footprints of 0.5 to 1 m along a path across
the map, and a mixed batch of 127 such footprints and a 64-gon covering half of the map.  Each row reports
  * batch_us:   host clock around the whole batch C call (hulls requested) including its synchronisation, median;
  * nohull_us:  the same without hulls;
  * loop_c_us / loop_py_us: the same polygons as a loop of single C calls / of get_polygon_traversability calls, median;
  * k_<name>_us: kernel durations by name from torch.profiler (CUDA activity), in a separate run of 10 batch calls,
                 as the mean per call.
The device name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
from polygon_check_timing import device_info, regular    # noqa: E402


def footprints(rng, B, L):
    """B 8-vertex footprints of 0.5 to 1 m across, centred along a curve across the map."""
    s = np.linspace(-0.9, 0.9, B)
    out = []
    for x, y in zip(s * L, 0.5 * L * np.sin(2.5 * s)):
        a = np.sort(rng.uniform(0, 2 * np.pi, 8))
        r = rng.uniform(0.25, 0.5, 8)
        out.append(np.stack([x + r * np.cos(a), y + r * np.sin(a)], 1).astype(np.float32))
    return out


def median_us(f, n):
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return 1e6 * float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
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
        L = 0.5 * (W - 2) * p.resolution
        batches = [(f"footprints_{B}", footprints(rng, B, L)) for B in (1, 16, 128, 1024, 4096)]
        batches.append(("mixed_127+half_map_64", footprints(rng, 127, L) + [regular(64, 2 * L / np.sqrt(2 * np.pi))]))
        for name, polys in batches:
            B = len(polys)
            nv = np.array([len(q) for q in polys], np.int32)
            xy = np.ascontiguousarray(np.concatenate(polys))
            res = np.zeros((B, 3))
            off = np.zeros(B + 1, np.int64)
            hull = np.zeros((1 << 20, 2))
            rows_c = C.c_int64(0)

            def batch(hulls=True):
                rows_c.value = len(hull)
                rc = em._L.emap_polygon_traversability_batch(
                    em._h, B, nv.ctypes.data, xy.ctypes.data, None, p.safe_thresh, p.safe_min_thresh, p.max_unsafe_n,
                    res.ctypes.data, hull.ctypes.data if hulls else None, off.ctypes.data, C.byref(rows_c))
                assert rc == 0, rc

            ring = np.zeros((2 * (W - 2) + 1, 2))
            cap = C.c_int32(0)
            one = np.zeros(3)

            def loop_c():
                for q in polys:
                    cap.value = len(ring)
                    assert em._L.emap_polygon_traversability(em._h, q.ctypes.data, len(q), None, p.safe_thresh,
                                                             p.safe_min_thresh, p.max_unsafe_n, one.ctypes.data,
                                                             ring.ctypes.data, C.byref(cap), None) == 0

            def loop_py():
                for q in polys:
                    em.get_polygon_traversability(q, one)

            for _ in range(3):                  # warm-up: module load, scratch growth
                batch(); batch(False)
            loop_c()
            n_loop = max(3, min(args.calls, 2048 // B))
            row = dict(cell_n=W, batch=name, polygons=B, batch_us=median_us(batch, args.calls),
                       nohull_us=median_us(lambda: batch(False), args.calls),
                       loop_c_us=median_us(loop_c, n_loop), loop_py_us=median_us(loop_py, n_loop))
            row["speedup_vs_loop_c"] = row["loop_c_us"] / row["batch_us"]
            n_prof = 10
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(n_prof):
                    batch()
                torch.cuda.synchronize()
            row.update(unsafe=int((res[:, 0] == 0).sum()), ring_rows=int(off[-1]))     # of the last (hull) call
            durs = {}
            for ev in prof.events():
                m = re.search(r"\b(k_\w+)", ev.name)
                if ev.device_type.name == "CUDA" and m:
                    durs.setdefault(m.group(1), []).append(ev.device_time)
            for k, v in sorted(durs.items()):
                row[f"{k}_us"] = float(np.sum(v)) / n_prof
            rows.append(row)
            print(json.dumps(row), flush=True)
        em.close()
    info = device_info()
    print(json.dumps(info))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
