"""Timing of the semantic plugins (emap_semantic_filter, emap_semantic_traversability, emap_features_pca) at 1024^2 and
2048^2, with L = 16 class layers and F = 16 feature layers.

    python tools/semantic_plugins_timing.py [--calls 100] [--out result.json]

For each map size it reports
  * <plugin>_us:      CUDA-event median per C call on the handle's stream (features_pca includes its one synchronisation);
  * kernel times:     per-kernel durations from torch.profiler (CUDA activity), median over the profiled calls;
  * pca_bytes_bound_us: the F planes read twice (statistics and projection) at the data sheet's 3.35 TB/s, and the
                      measured call's share of it;
  * ref_pca_ms:       where sklearn is installed, the reference's path on the same card: torch D2H of the F planes, clip,
                      sklearn PCA(3) fit + transform, the min-max scaling and the uint8 pack (features_pca.py:66-96).
The device name and power limit are read in the same run.  Inputs are seeded random planes.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return {"device": name, "power_limit": power}
    except Exception as e:                        # the numbers still stand, but say where they came from
        import torch
        return {"device": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def event_median_us(fn, calls, stream):
    import torch
    ts = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts))


def ref_pca(planes):
    """features_pca.py:66-96 on the host, fed by a torch device-to-host copy"""
    from sklearn.decomposition import PCA
    F, W = planes.shape[0], planes.shape[1]
    data = np.clip(planes.reshape(F, -1).T.cpu().numpy(), -1, 1)
    comp = PCA(n_components=3).fit(data).transform(data).reshape(W, W, 3)
    lo, hi = comp.min(axis=(0, 1)), comp.max(axis=(0, 1))
    img = (np.divide(comp - lo, hi - lo) * 255).astype(np.uint8)
    r, g, b = (np.asarray(img[:, :, k], dtype=np.uint32) for k in range(3))
    return ((r << 16) | (g << 8) | b).view(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    assert torch.cuda.is_available(), "needs a CUDA device"
    rows = []
    L = F = 16
    for W in (1024, 2048):
        em = ElevationMap(core_parameter(W, plugin_config_file=""))
        torch.manual_seed(W)
        cls = torch.rand((L, W, W), device="cuda")
        feat = (torch.randn((F, W, W), device="cuda") * torch.linspace(0.4, 0.02, F, device="cuda")[:, None, None])
        out = torch.empty((W, W), device="cuda")
        cp = (C.c_void_p * L)(*[cls[k].data_ptr() for k in range(L)])
        fp = (C.c_void_p * F)(*[feat[k].data_ptr() for k in range(F)])
        thr = (C.c_double * L)(*([0.5] * L))
        typ = (C.c_int32 * L)(*([1, 0] * (L // 2)))
        torch.cuda.synchronize()
        st = torch.cuda.Stream()                                   # events and kernels on one (non-default) stream
        em.set_stream(st.cuda_stream)
        calls = {
            "semantic_filter": lambda: em._L.emap_semantic_filter(em._h, L, cp, out.data_ptr()),
            "semantic_traversability": lambda: em._L.emap_semantic_traversability(em._h, L, cp, thr, typ, out.data_ptr()),
            "features_pca": lambda: em._L.emap_features_pca(em._h, F, fp, out.data_ptr()),
        }
        row = dict(cell_n=W, layers=L, features=F)
        for name, fn in calls.items():
            for _ in range(10):                                  # warm-up: module load, scratch allocation
                assert fn() == 0
            row[name + "_us"] = event_median_us(lambda: fn(), args.calls, st)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                for fn in calls.values():
                    fn()
            torch.cuda.synchronize()
        durs = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA" and ("k_pca" in ev.name or "k_semantic" in ev.name):
                key = ev.name.split("(")[0].split(" ")[-1]
                durs.setdefault(key, []).append(ev.device_time)
        row["kernels_us"] = {k: float(np.median(v)) for k, v in sorted(durs.items())}
        bound_us = 2 * F * 4 * W * W / HBM_BYTES_PER_S * 1e6
        row["pca_bytes_bound_us"] = bound_us
        row["pca_share_of_bound"] = bound_us / row["features_pca_us"]
        try:
            import sklearn  # noqa: F401
            ts = []
            for _ in range(3):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ref_pca(feat)
                ts.append(time.perf_counter() - t0)
            row["ref_pca_ms"] = 1e3 * float(np.median(ts))
        except ImportError:
            row["ref_pca_ms"] = None
        em.set_stream(0)
        rows.append(row)
        print(json.dumps(row))
        em.close()
    info = device_info()
    print(json.dumps(info))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
