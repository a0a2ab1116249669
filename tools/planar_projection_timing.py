"""Times ElevationMap.project_to_planar_regions on the device, and the same queries through the library header built
for the CPU (tests/native/projection_host.cpp, one core, a stand-in for the node's C++, not the node itself).  Scenes:
the terrain.png window (3 m at 0.04 m), the node's 76^2 window of the default map after LiDAR frames, and the whole
2047^2 window of tests/plane_scenes.big_image.  Queries: 10^3, 10^4 and 10^5 seeded points over the regions and on
their edges; projection only and with 16-vertex growth (growth factor 1.05).  Tables, queries and output stay on the
device; "device_ms" is CUDA events over calls (mean), "host_ms_per_query" the host build's clock over the first
`--host-queries` queries.  "kernels_ms" is a torch.profiler run of its own at 10^4 queries: device time per call of
each kernel.  Prints one JSON line with the card's name and power limit.
  python tools/planar_projection_timing.py [--host-queries 200]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from plane_segmentation_timing import card   # noqa: E402
from planar_regions_timing import _kernels_ms   # noqa: E402


def _device_ms(call, budget_ms=2000.0):
    """Mean device time of a call over as many calls as fit in about budget_ms (at least 1, at most 20)."""
    import torch
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call()
    e1.record()
    torch.cuda.synchronize()
    reps = max(1, min(20, int(budget_ms / max(e0.elapsed_time(e1), 1e-3))))
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    import numpy as np
    import torch
    import plane_scenes as S
    import planar_projection_oracle as PP
    from test_planar_projection_cpu import host_project, load_native
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--host-queries", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    lib = load_native()
    p = S.params()
    rows = []
    for label in ("terrain.png 3 m window", "LiDAR map, node window", "whole 2047^2 window"):
        if label.startswith("terrain"):
            png, scale, pos, ln = S.TERRAINS["terrain"]
            img = S.terrain_image(np.load(S.GOLDEN)["grey__terrain"], scale)
            em = ElevationMap(core_parameter(img.shape[0] + 2))
            S.set_image(em, img)
        elif label.startswith("LiDAR"):
            em = ElevationMap(core_parameter(S.LIDAR_W))
            S.lidar_frames(em)
            pos, ln = S.lidar_window(em.center), (3.0, 3.0)
        else:
            em = ElevationMap(core_parameter(S.BIG_W))
            S.set_image(em, S.big_image())
            pos, ln = (0.0, 0.0), (100.0, 100.0)
        res = em.planar_terrain(pos, ln, p)
        tables = tuple(res["tables"][k] for k in ("regions", "polygons", "vertices"))
        regions = PP.regions_from_tables(*tables)
        dev = {"tables": {k: torch.as_tensor(v, device="cuda") for k, v in res["tables"].items()}}
        roles = np.bincount(tables[1][:, 1], minlength=4).tolist()
        inset_edges = int(tables[1][tables[1][:, 1] == 2, 4].sum())
        boundary_edges = int(tables[1][tables[1][:, 1] <= 1, 4].sum())
        q_all = PP.queries_for(regions, 100000, seed=0)
        q_all = q_all[np.isfinite(q_all).all(1)]
        q_all = q_all[np.random.default_rng(1).permutation(len(q_all))[:100000]]
        row = {"case": label, "window": list(res["size"]), "regions": len(tables[0]),
               "polygons_by_role": roles, "inset_outer_edges": inset_edges, "boundary_edges": boundary_edges,
               "results": []}
        for n in (1000, 10000, 100000):
            qd = torch.as_tensor(q_all[:n], device="cuda")
            for n_conv in (0, 16):
                out = {"index": torch.empty((n, 3), dtype=torch.int32, device="cuda"),
                       "point": torch.empty((n, 6), dtype=torch.float64, device="cuda")}
                if n_conv:
                    out["convex"] = torch.empty((n, n_conv, 5), dtype=torch.float64, device="cuda")
                ms = _device_ms(lambda: em.project_to_planar_regions(dev, qd, 0.0, n_conv, 1.05, out=out))
                r = {"queries": n, "convex_vertices": n_conv, "device_ms": round(ms, 4)}
                if n_conv:
                    r["mean_sweeps"] = round(float(out["index"][:, 2].double().mean()), 2)
                if n == 1000:
                    hq = q_all[:a.host_queries]
                    t = time.perf_counter()
                    host_project(lib, tables, hq, 0.0, n_conv, 1.05)
                    r["host_ms_per_query"] = round((time.perf_counter() - t) * 1e3 / len(hq), 4)
                    r["device_ms_per_query"] = round(ms / n, 6)
                if n == 10000:
                    r["kernels_ms"] = _kernels_ms(
                        lambda: em.project_to_planar_regions(dev, qd, 0.0, n_conv, 1.05, out=out))
                row["results"].append(r)
        rows.append(row)
        del em
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power,
                      "device_ms": "CUDA events, device tables, queries and output, mean of calls",
                      "host_ms_per_query": "host clock, the header built for the CPU, one core",
                      "results": rows}))


if __name__ == "__main__":
    main()
