"""Times Navier-Stokes inpainting on the device (ElevationMap.inpaint_image / emap_inpaint_image, and
nonlinear_interpolation / emap_nonlinear_interpolation) with device input and output, against a copy to the host plus
cv2.inpaint(INPAINT_NS) there (for the grid call: plus the NumPy quantisation and write-back of
tests/ns_inpaint_oracle.py): config D's 2048^2 map after a dense depth-camera frame (98 % holes, about 2000 rounds) and
the node's 3 m window (75^2 cells at 0.04 m) of the LiDAR map.  CUDA events over --reps calls after warm-up.  Prints one
JSON line with the card's name and power limit, read in the same run.
  python tools/inpaint_ns_timing.py [--reps 5] [--host-reps 1]"""
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
from planar_regions_timing import _device_ms   # noqa: E402


def _host_ms(fn, reps):
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) * 1e3 / reps


def main():
    import cv2
    import numpy as np
    import torch
    import ns_inpaint_oracle as O
    import plane_scenes as S
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    ns = lambda img, m, r=1: cv2.inpaint(img, m, r, cv2.INPAINT_NS)  # noqa: E731
    rows = []
    # config D's map: the plugin's 8-bit planes
    em = ElevationMap(core_parameter(2048))
    pts, R, t = wl.depth_camera_cloud(3, 0)
    em.move_to(t, R)
    em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.0, 0.0)
    st, _ = em.get_state()
    mask = (st[2] < 0.5).astype(np.uint8)
    hv = st[0][mask < 1]
    q = (st[0] - hv.min()) * np.float32(255) / np.float32(float(hv.max()) - float(hv.min()))
    img = np.clip(np.nan_to_num(np.trunc(q), nan=0.0), 0, 255).astype(np.uint8)
    di, dm = torch.as_tensor(img, device="cuda"), torch.as_tensor(mask, device="cuda")
    out = em.inpaint_image(di, dm)
    row = {"case": "config D map, inpaint_image ns", "image": list(img.shape), "holes": round(float(mask.mean()), 4),
           "device_ms": round(_device_ms(lambda: em.inpaint_image(di, dm, out=out), a.reps), 3)}
    row["copy_and_cv2_ms"] = round(_host_ms(lambda: ns(di.cpu().numpy(), dm.cpu().numpy()), a.host_reps), 1)
    rows.append(row)
    g = {"layers": {"elevation": torch.as_tensor(np.where(mask > 0, np.float32(np.nan), st[0]), device="cuda")},
         "centre": np.zeros(2), "resolution": em.resolution}
    gout = em.nonlinear_interpolation(g, "elevation")
    row = {"case": "config D map, nonlinear_interpolation",
           "device_ms": round(_device_ms(lambda: em.nonlinear_interpolation(g, "elevation", out=gout), a.reps), 3)}
    row["copy_and_host_ms"] = round(_host_ms(lambda: O.nonlinear_interpolation(
        g["layers"]["elevation"].cpu().numpy(), em.resolution, em.resolution, ns), a.host_reps), 1)
    rows.append(row)
    del em
    # the node's 3 m window of the LiDAR map
    em = ElevationMap(core_parameter(S.LIDAR_W))
    S.lidar_frames(em)
    sub = em.get_submap(S.lidar_window(em.center), (3.0, 3.0), ["elevation"])
    h = np.ascontiguousarray(sub["layers"]["elevation"], np.float32)
    g = {"layers": {"elevation": torch.as_tensor(h, device="cuda")}, "centre": sub["centre"], "resolution": em.resolution}
    gout = em.nonlinear_interpolation(g, "elevation")
    row = {"case": "node 3 m window, nonlinear_interpolation", "grid": list(h.shape),
           "holes": round(float(np.isnan(h).mean()), 4),
           "device_ms": round(_device_ms(lambda: em.nonlinear_interpolation(g, "elevation", out=gout), 20 * a.reps), 4)}
    row["copy_and_host_ms"] = round(_host_ms(lambda: O.nonlinear_interpolation(
        g["layers"]["elevation"].cpu().numpy(), em.resolution, em.resolution, ns), 20 * a.host_reps), 3)
    rows.append(row)
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power, "reps": a.reps, "rows": rows}))


if __name__ == "__main__":
    main()
