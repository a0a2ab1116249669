"""Times ElevationMap.values_at on the live map (emap_map_values_at) against what a caller does without it: the whole
export to the host (get_maps_with_names_ref) plus a NumPy bilinear lookup, and a whole-map get_submaps window into a
CUDA tensor plus a torch bilinear gather.  Maps: 1024^2 and 2048^2 after seeded LiDAR frames.  Points: 10^3 .. 10^6
device points over the map; 1 and 4 layers; nearest, linear and cubic.  Every case is CUDA events over calls, mean after
a warm-up call (the host baseline's calls synchronise, so its events span the host work too).  Prints one JSON line
with the card's name and power limit.
  python tools/values_at_timing.py [--budget-ms 300]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from plane_segmentation_timing import card   # noqa: E402
from planar_projection_timing import _device_ms   # noqa: E402

LAYERS = {1: ["elevation"], 4: ["elevation", "variance", "traversability", "upper_bound"]}


def _axis(q, centre, res, n):
    """Fractional row index of q on one axis of the export (row 0 at the +x edge), and its integer corner."""
    import numpy as np
    top = centre + 0.5 * n * res - 0.5 * res
    f = (top - q) / res
    i0 = np.clip(np.floor(f), 0, n - 2).astype(np.int64)
    return f - i0, i0


def numpy_bilinear(planes, centre, res, q):
    import numpy as np
    n = planes.shape[1]
    tx, r0 = _axis(q[:, 0], centre[0], res, n)
    ty, c0 = _axis(q[:, 1], centre[1], res, n)
    out = []
    for p in planes:
        a, b, c, d = p[r0, c0], p[r0 + 1, c0], p[r0, c0 + 1], p[r0 + 1, c0 + 1]
        out.append(((a * (1 - tx) + b * tx) * (1 - ty) + (c * (1 - tx) + d * tx) * ty).astype(np.float32))
    return out


def torch_bilinear(planes, centre, res, q):
    import torch
    n = planes.shape[1]
    top = torch.as_tensor(centre, device=q.device) + 0.5 * n * res - 0.5 * res
    f = (top - q) / res
    i0 = torch.clamp(torch.floor(f), 0, n - 2)
    t = f - i0
    i0 = i0.long()
    r0, c0 = i0[:, 0], i0[:, 1]
    tx, ty = t[:, 0], t[:, 1]
    flat = planes.reshape(planes.shape[0], -1).double()
    a, b = flat[:, r0 * n + c0], flat[:, (r0 + 1) * n + c0]
    c, d = flat[:, r0 * n + c0 + 1], flat[:, (r0 + 1) * n + c0 + 1]
    return (((a * (1 - tx) + b * tx) * (1 - ty) + (c * (1 - tx) + d * tx) * ty)).float()


def main():
    import numpy as np
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget-ms", type=float, default=300.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    rows = []
    for W in (1024, 2048):
        em = ElevationMap(core_parameter(W))
        for f in range(4):
            pts, R, t = wl.lidar_cloud(0, f, n_rings=64, n_az=1250, max_range=0.45 * W * em.resolution)
            em.move_to(t, R)
            em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        n_out = W - 2
        centre = em.center[:2].astype(np.float64)
        half = 0.5 * n_out * em.resolution
        rng = np.random.default_rng(0)
        q_all = rng.uniform(centre - 0.98 * half, centre + 0.98 * half, (10 ** 6, 2))
        row = {"map": [n_out, n_out], "results": []}
        for n in (10 ** 3, 10 ** 4, 10 ** 5, 10 ** 6):
            qh = q_all[:n].copy()
            qd = torch.as_tensor(qh, device="cuda")
            for k, names in LAYERS.items():
                r = {"points": n, "layers": k}
                out = {"values": torch.empty((k, n), device="cuda"),
                       "status": torch.empty(n, dtype=torch.int32, device="cuda")}
                for method in ("nearest", "linear", "cubic"):
                    ms = _device_ms(lambda: em.values_at(qd, names, method, out=out), a.budget_ms)
                    r[method + "_ms"] = round(ms, 4)
                host = np.zeros((k, n_out, n_out), np.float32)

                def export_numpy():
                    em.get_maps_with_names_ref(names, host)
                    return numpy_bilinear(host, centre, em.resolution, qh)

                dev = torch.empty(k * n_out * n_out, dtype=torch.float32, device="cuda")

                def submap_torch():
                    em.get_submaps([(centre, (2 * half + 1.0, 2 * half + 1.0))], names, out=dev)
                    return torch_bilinear(dev.view(k, n_out, n_out), centre, em.resolution, qd)

                r["export_numpy_bilinear_ms"] = round(_device_ms(export_numpy, a.budget_ms), 4)
                r["submap_torch_bilinear_ms"] = round(_device_ms(submap_torch, a.budget_ms), 4)
                row["results"].append(r)
        rows.append(row)
        del em
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power,
                      "timing": "CUDA events over calls, mean after one warm-up call; values_at with device points and "
                                "output; export_numpy_bilinear: get_maps_with_names_ref + NumPy bilinear (host clock "
                                "inside the events); submap_torch_bilinear: whole-map get_submaps into a CUDA tensor + "
                                "torch bilinear gather",
                      "results": rows}))


if __name__ == "__main__":
    main()
