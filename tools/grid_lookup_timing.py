"""Times ElevationMap.max_value_between_locations, values_between_locations and grid_derivatives on the device, and the
same queries through the library header built for the CPU (tests/native/lookup_host.cpp, one core, a stand-in for the
reference's C++, not the reference itself).  Grids: a 4 x 4 m get_submaps window of the default map after LiDAR
frames, and the whole 2047^2 window of tests/plane_scenes.big_image (0.04 m).  Queries: 10^3 .. 10^6 seeded lines of
0.5 to 3 m over the window, and as many derivative positions (gradient and curvature).  Layer, queries and output stay
on the device; "device_ms" is CUDA events over calls (mean), "host_ms_per_query" the host build's clock over the first
`--host-queries` queries.  "kernels_ms" is a torch.profiler run of its own at 10^5 queries: device time per call of
each kernel.  Prints one JSON line with the card's name and power limit.
  python tools/grid_lookup_timing.py [--host-queries 2000]"""
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
from planar_projection_timing import _device_ms   # noqa: E402


def main():
    import numpy as np
    import torch
    import grid_lookup_oracle as O
    import plane_scenes as S
    from test_grid_lookup_cpu import host_derivatives, host_max, host_values, load_native
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--host-queries", type=int, default=2000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    lib = load_native()
    rows = []
    for label in ("LiDAR map, 4 m window", "whole 2047^2 window"):
        if label.startswith("LiDAR"):
            em = ElevationMap(core_parameter(S.LIDAR_W))
            S.lidar_frames(em)
            pos, ln = S.lidar_window(em.center), (4.0, 4.0)
        else:
            em = ElevationMap(core_parameter(S.BIG_W))
            S.set_image(em, S.big_image())
            pos, ln = (0.0, 0.0), (100.0, 100.0)
        out = torch.zeros((em.cell_n - 2) ** 2, dtype=torch.float32, device="cuda")
        grid = em.get_submap(pos, ln, ["elevation"], out=out)
        g = O.Grid(grid["layers"]["elevation"].cpu().numpy(), grid["centre"], em.resolution)
        lines = O.random_lines(g, 10 ** 6, seed=0, outside=0.0)
        posq = lines[:, :2].copy()
        row = {"case": label, "window": list(grid["size"]), "finite_cells": int(np.isfinite(g.data).sum()),
               "results": []}
        for n in (10 ** 3, 10 ** 4, 10 ** 5, 10 ** 6):
            ld = torch.as_tensor(lines[:n], device="cuda")
            pd = torch.as_tensor(posq[:n], device="cuda")
            mx = {"index": torch.empty((n, 3), dtype=torch.int32, device="cuda"),
                  "value": torch.empty((n, 3), dtype=torch.float64, device="cuda")}
            dv = {"index": torch.empty((n, 3), dtype=torch.int32, device="cuda"),
                  "value": torch.empty((n, 5), dtype=torch.float64, device="cuda")}
            total = int(em.values_between_locations(grid, "elevation", ld[:, :2], ld[:, 2:])["rows"].shape[0])
            calls = {
                "max_value_between_locations": lambda: em.max_value_between_locations(
                    grid, "elevation", ld[:, :2], ld[:, 2:], out=mx),
                "values_between_locations": lambda: em.values_between_locations(
                    grid, "elevation", ld[:, :2], ld[:, 2:], capacity=total),
                "grid_derivatives": lambda: em.grid_derivatives(grid, "elevation", pd, True, out=dv)}
            r = {"queries": n, "value_rows": total}
            for name, call in calls.items():
                ms = _device_ms(call)
                r[name] = {"device_ms": round(ms, 4), "device_us_per_query": round(ms * 1e3 / n, 5)}
                if n == 10 ** 5:
                    r[name]["kernels_ms"] = _kernels_ms(call)
            if n == 10 ** 3:
                hq = lines[:a.host_queries]
                for name, fn in (("max_value_between_locations", lambda: host_max(lib, g, hq)),
                                 ("values_between_locations", lambda: host_values(lib, g, hq)),
                                 ("grid_derivatives", lambda: host_derivatives(lib, g, hq[:, :2], True))):
                    t = time.perf_counter()
                    fn()
                    r[name]["host_us_per_query"] = round((time.perf_counter() - t) * 1e6 / len(hq), 4)
            row["results"].append(r)
        rows.append(row)
        del em
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power,
                      "device_ms": "CUDA events, device layer, queries and output, mean of calls "
                                   "(values_between_locations: reads back its two info words per call)",
                      "host_us_per_query": "host clock, the header built for the CPU, one core, a stand-in for "
                                           "the reference's C++",
                      "results": rows}))


if __name__ == "__main__":
    main()
