"""Times the layer filters of emap_grid_filter (ElevationMap.min_values, median, box_blur, gaussian_blur, dilate,
erode, outline) with device input and output at 76^2, 1022^2 and 2047^2, against a copy of the layer to the host plus
what a caller runs there: cv2 for the median (its 8-bit path with the quantisation in NumPy), the box filter and the Gaussian, and the NumPy restatements of
tests/filters_oracle.py for minValues, dilate, erode and outline (grid_map's own loops are slower still).  The layer is
a terrain with a quarter of its cells NaN (finite for the Gaussian).  Device times are CUDA events over repeated calls
after a warm-up call; host times a wall clock around the copy and the host work.  Prints one JSON line with the card's
name and power limit, read in the same run.
  python tools/grid_filters_timing.py [--budget-ms 1000] [--host-reps 1]"""
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
from planar_projection_timing import _device_ms   # noqa: E402

# (label, method, keyword arguments, host call on a NumPy layer)
OPS = [
    ("min_values", "min_values", {}, lambda F, cv2, a: F.min_values(a)),
    ("median k3", "median", dict(kernel_size=3), lambda F, cv2, a: cv2.medianBlur(a, 3)),
    ("median k7 (8-bit)", "median", dict(kernel_size=7), lambda F, cv2, a: _median8(cv2, a, 7)),
    ("box_blur k5", "box_blur", dict(kernel_size=5), lambda F, cv2, a: cv2.blur(a, (5, 5))),
    ("box_blur k9", "box_blur", dict(kernel_size=9), lambda F, cv2, a: cv2.blur(a, (9, 9))),
    ("gaussian_blur k5 s1", "gaussian_blur", dict(kernel_size=5, sigma=1.0),
     lambda F, cv2, a: cv2.GaussianBlur(a, (5, 5), 1.0)),
    ("dilate k5", "dilate", dict(kernel_size=5), lambda F, cv2, a: F.morph(a, 5, None, True, True)),
    ("erode k5", "erode", dict(kernel_size=5), lambda F, cv2, a: F.morph(a, 5, None, True, False)),
    ("outline", "outline", {}, lambda F, cv2, a: F.outline(a)),
]


def _median8(cv2, a, k):
    """smoothing::median's 8-bit path on the host: toImage, cv2.medianBlur, convertTo."""
    import numpy as np
    import ns_inpaint_oracle as NS
    fin = a[np.isfinite(a)]
    lo, hi = fin.min(), fin.max()
    u = cv2.medianBlur(NS.to_image_u8(a, lo, hi), k)
    return u.astype(np.float32) * np.float32((hi - lo) / np.float32(255)) + lo


def _host_ms(fn, reps):
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) * 1e3 / reps


def main():
    import cv2
    import numpy as np
    import torch
    import filters_oracle as F
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget-ms", type=float, default=1000.0)
    ap.add_argument("--host-reps", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to time")
    em = ElevationMap(core_parameter(64))
    rng = np.random.default_rng(0)
    rows = []
    for n in (76, 1022, 2047):
        x, y = np.meshgrid(np.linspace(0, 3, n), np.linspace(0, 2, n))
        terrain = (np.sin(x) * np.cos(2 * y) + 0.3 * np.floor(2 * x)).astype(np.float32)
        holed = terrain.copy()
        holed[rng.random(holed.shape) < 0.25] = np.nan
        for label, method, kw, host in OPS:
            h = terrain if method == "gaussian_blur" else holed
            d = torch.as_tensor(h, device="cuda")
            g = {"layers": {"elevation": d}, "centre": np.zeros(2), "resolution": 0.04}
            out = torch.empty_like(d)
            fn = getattr(em, method)
            row = {"op": label, "cells": [n, n],
                   "device_ms": round(_device_ms(lambda: fn(g, out=out, **kw), a.budget_ms), 4)}
            row["copy_and_host_ms"] = round(_host_ms(lambda: host(F, cv2, d.cpu().numpy()), a.host_reps), 3)
            rows.append(row)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "input_output": "device", "rows": rows}))


if __name__ == "__main__":
    main()
