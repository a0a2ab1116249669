"""bench.py --config D / --config E: the other two BASELINE.json configurations, same JSON-line contract.

D  configs[3]: 2048 x 2048 grid, 1 M-point dense depth-camera cloud per frame (5 % NaN pixels), full post-process chain:
   the frame itself (dilation + traversability + normals are inside it) followed by the default plugin chain
   min_filter -> smooth -> inpainting -> erosion evaluated on the device and one exported layer.  A step = all of that.
E  configs[4]: batched replay, 64 independent 512 x 512 maps x 100 k points each, 64 / N maps per GPU, one CUDA stream
   per map, every frame replayed as ONE captured CUDA graph (replicas only: no exchange between maps; SURVEY 8(e)).
"""
import time

import numpy as np


def _peaks():
    return 3350.0, "H100 SXM data sheet HBM3 bandwidth (not measured)"


def run_config_d(args, torch, dist, rank, local_rank, world, sampler):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200 import workloads as wl
    import contextlib, sys
    W = 2048
    param = core_parameter(W)
    with contextlib.redirect_stdout(sys.stderr):
        em = ElevationMap(param, device=local_rank)
    stream = torch.cuda.current_stream()
    em.set_stream(stream.cuda_stream)
    n_pool = 3
    frames = [wl.depth_camera_cloud(3, f + 10 * rank) for f in range(n_pool)]
    dev = [torch.from_numpy(p).cuda() for p, _, _ in frames]
    pin = [torch.from_numpy(p).pin_memory() for p, _, _ in frames]
    N = frames[0][0].shape[0]
    flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    export = np.zeros((W - 2, W - 2), np.float32)
    chain = ["min_filter", "smooth", "inpaint", "erosion"]

    def between(f):
        em.move_to(frames[f][2], frames[f][1]); em.update_variance(); em.update_time()
        flush.zero_()

    export4 = np.zeros((len(chain), W - 2, W - 2), np.float32)

    def step(f, pts, ev=None):
        _, R, t = frames[f]
        marks = []

        def mark():
            if ev is not None:
                e = torch.cuda.Event(enable_timing=True); e.record(stream); marks.append(e)
        mark()
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        mark()
        # the consumer's call (WRAP:213-252 get_grid_map): every plugin layer evaluated once on the device, the four layers
        # exported by one kernel + one D2H copy + one synchronisation
        em.get_maps_with_names_ref(chain, export4)
        mark()
        if ev is not None:
            ev.append(marks)

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    n_warm, n_steps = max(3, min(args.warmup, 4)), args.steps
    for it in range(n_warm):
        f = it % n_pool
        between(f); step(f, dev[f])
    barrier()
    t_busy0 = time.time()
    evs, wall = [], 0.0
    for it in range(n_steps):
        f = (n_warm + it) % n_pool
        between(f); torch.cuda.synchronize()
        t0 = time.perf_counter()
        step(f, dev[f], evs)
        torch.cuda.synchronize()
        wall += time.perf_counter() - t0
    ms = 1e3 * wall / n_steps
    # e2e: pinned host cloud
    wall = 0.0
    for it in range(n_steps):
        f = it % n_pool
        between(f); torch.cuda.synchronize()
        t0 = time.perf_counter()
        step(f, pin[f]); em.get_frame_stats()
        wall += time.perf_counter() - t0
    ms_e2e = 1e3 * wall / n_steps
    t_busy1 = time.time()
    barrier()
    tt = torch.tensor([ms, ms_e2e], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    ms, ms_e2e = float(tt[0]), float(tt[1])
    names = ["frame(fusion+raycast+dilation+traversability+normals)", "plugin chain + export of its 4 layers (D2H)"]
    stage = np.zeros(len(names))
    for marks in evs:
        for k in range(len(names)):
            stage[k] += marks[k].elapsed_time(marks[k + 1])
    stage /= len(evs)
    # per-plugin device times (diagnostic pass, untimed above): each layer evaluated on its own
    plugin_ms = {}
    for name in chain:
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(stream); em.get_layer(name); e1.record(stream); torch.cuda.synchronize()
        plugin_ms[name] = float(e0.elapsed_time(e1))
    if rank != 0:
        return None
    import ctypes as C
    r_, mj, nc = C.c_int32(), C.c_int32(), C.c_int32()
    em._check(em._L.emap_inpaint_stats(em._h, C.byref(r_), C.byref(mj), C.byref(nc)))
    hbm, src = _peaks()
    Cc = W * W
    frame_bytes = 24 * N + 80 * Cc                        # SURVEY 8(d): 359.5 MB
    chain_bytes = 4 * 8 * Cc                              # + 8 C per plugin layer produced
    ach = frame_bytes / (stage[0] * 1e-3) / 1e9
    clocks = sampler.stop(t_busy0, t_busy1) if sampler is not None else None
    n_total = N * world
    return {"metric": "Mpoints/s fused + map-update frames/s (2048^2 grid, 1M-pt depth frames, full post-process chain incl. inpainting)",
            "value": n_total / (ms * 1e-3) / 1e6, "unit": "Mpoints/s", "frames_per_s": world * 1e3 / ms, "n_gpus": world,
            "steps": n_steps, "warmup": n_warm, "requested_steps": args.steps, "ms_per_step": ms, "higher_is_better": True,
            "device": torch.cuda.get_device_name(local_rank),
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": "BASELINE configs[3]: 2048x2048 grid, 0.04 m, 1M-pt depth-camera cloud/frame (5% NaN), raycast+overlap-clear+"
                                   "drift on, then min_filter -> smooth -> inpainting(telea) -> erosion on the device, the four layers exported to the host",
                       "parallelism": "1 GPU" if world == 1 else f"{world} independent replicas (replicas only, no exchange)",
                       "l2": "flushed between timed steps (512 MB memset, untimed)", "points_per_step": n_total,
                       "inpaint_rounds": int(r_.value), "inpaint_longest_fixed_point": int(mj.value)},
            "e2e": {"value": n_total / (ms_e2e * 1e-3) / 1e6, "unit": "Mpoints/s", "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": int(N * 12), "d2h_bytes_per_step": int(export4.nbytes + 72),
                    "note": "pinned host cloud in, four plugin layers + frame stats out"},
            "gpu_launches": None, "clocks": clocks,
            "roofline": {"bound": "hbm", "kernel": "frame (6 kernels)", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm,
                         "traffic": None, "peak_source": src, "frame_algorithmic_bytes": frame_bytes,
                         "chain_algorithmic_bytes": chain_bytes,
                         "step_frac": (frame_bytes + chain_bytes) / (ms * 1e-3) / 1e9 / hbm,
                         "stage_ms": {n: float(v) for n, v in zip(names, stage)}, "plugin_ms": plugin_ms},
            "cpu_baseline": None}


def run_config_e(args, torch, dist, rank, local_rank, world, sampler):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200 import workloads as wl
    import contextlib, sys
    N_MAPS, W, NPTS = 64, 512, 100000
    if N_MAPS % world:
        raise SystemExit("--config E needs a GPU count that divides 64")
    n_local = N_MAPS // world
    param = core_parameter(W)
    main = torch.cuda.current_stream()
    maps, streams, clouds, poses, graphs = [], [], [], [], []
    n_pool = 2
    cloud_cache = {}

    def cloud(f):
        if f not in cloud_cache:
            cloud_cache[f] = wl.lidar_cloud(4, f, n_rings=32, n_az=3125, max_range=9.5, sensor=0, n_sensors=1)
        return cloud_cache[f]
    for m in range(n_local):
        gid = rank * n_local + m
        with contextlib.redirect_stdout(sys.stderr):
            em = ElevationMap(param, device=local_rank)
        st = torch.cuda.Stream()
        em.set_stream(st.cuda_stream)
        fr = [cloud(f) for f in (gid % 7, gid % 7 + 1)]
        assert fr[0][0].shape[0] == NPTS
        maps.append(em); streams.append(st)
        clouds.append([torch.from_numpy(p).cuda() for p, _, _ in fr]); poses.append([(R, t) for _, R, t in fr])
    torch.cuda.synchronize()

    def ticks(f):
        for m, em in enumerate(maps):
            R, t = poses[m][f]
            em.move_to(t, R); em.update_variance(); em.update_time()

    def frame_eager(m, f):
        R, t = poses[m][f]
        maps[m].input_pointcloud(clouds[m][f], ["x", "y", "z"], R, t, 0.02, 0.02)

    # warm every map (allocations, first-frame paths), then capture one graph per (map, pool frame)
    for f in range(n_pool):
        ticks(f)
        for m in range(n_local):
            frame_eager(m, f)
    torch.cuda.synchronize()
    use_graph = not getattr(args, "no_graph", False)
    if use_graph:
        for m in range(n_local):
            gs = []
            for f in range(n_pool):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=streams[m]):
                    frame_eager(m, f)
                gs.append(g)
            graphs.append(gs)
        torch.cuda.synchronize()

    def step(f):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(main)
        for m in range(n_local):
            streams[m].wait_stream(main)
            with torch.cuda.stream(streams[m]):
                if use_graph:
                    graphs[m][f].replay()
                else:
                    frame_eager(m, f)
        for m in range(n_local):
            main.wait_stream(streams[m])
        e1.record(main)
        return e0, e1

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    n_warm, n_steps = max(3, args.warmup), args.steps
    for it in range(n_warm):
        ticks(it % n_pool); step(it % n_pool)
    barrier()
    t_busy0 = time.time()
    evs = []
    for it in range(n_steps):
        f = (n_warm + it) % n_pool
        ticks(f); torch.cuda.synchronize()
        evs.append(step(f))
    barrier()
    ms = sum(a.elapsed_time(b) for a, b in evs) / n_steps
    # e2e: wall clock around the launches of one step + a stats read-back of every map
    wall = 0.0
    for it in range(n_steps):
        f = it % n_pool
        ticks(f); torch.cuda.synchronize()
        t0 = time.perf_counter()
        step(f)
        for em in maps:
            em.get_frame_stats()
        wall += time.perf_counter() - t0
    ms_e2e = 1e3 * wall / n_steps
    t_busy1 = time.time()
    tt = torch.tensor([ms, ms_e2e], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    ms, ms_e2e = float(tt[0]), float(tt[1])
    if rank != 0:
        return None
    hbm, src = _peaks()
    Cc = W * W
    frame_bytes = (24 * NPTS + 80 * Cc) * N_MAPS
    clocks = sampler.stop(t_busy0, t_busy1) if sampler is not None else None
    launches_per_frame = None
    try:
        l0 = maps[0].launch_count(); ticks(0); l1 = maps[0].launch_count(); frame_eager(0, 0); launches_per_frame = maps[0].launch_count() - l1
    except Exception:
        pass
    return {"metric": "map-frames/s, batched replay: 64 independent 512^2 maps x 100k-pt frames (one map per stream, one CUDA graph per frame)",
            "value": N_MAPS * 1e3 / ms, "unit": "map-frames/s", "mpoints_per_s": N_MAPS * NPTS / (ms * 1e-3) / 1e6, "n_gpus": world,
            "steps": n_steps, "warmup": n_warm, "ms_per_step": ms, "higher_is_better": True, "scaling": "strong",
            "device": torch.cuda.get_device_name(local_rank),
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": "BASELINE configs[4]: 64 independent 512x512 maps x 100k-pt LiDAR-like frame each per step, raycast+overlap-clear+drift on",
                       "parallelism": f"{n_local} maps per GPU x {world} GPU(s), one stream per map, replicas only (no exchange)",
                       "cuda_graph": bool(use_graph), "maps_per_gpu": n_local,
                       "l2": "not flushed: the %d maps of a GPU (~30 MB of state + scratch each) exceed the 50 MB L2" % n_local
                             if n_local * 30 > 50 else "not flushed (working set may fit L2)",
                       "untimed_between_steps": "move_to, update_variance, update_time on every map"},
            "e2e": {"value": N_MAPS * 1e3 / ms_e2e, "unit": "map-frames/s", "ms_per_step": ms_e2e, "h2d_bytes_per_step": 0,
                    "d2h_bytes_per_step": 72 * n_local, "note": "device-resident replay clouds (a replay batch lives in HBM); wall clock around graph launches + stats read-back"},
            "gpu_launches": None if launches_per_frame is None else int(launches_per_frame * N_MAPS * n_steps // world),
            "gpu_launches_per_frame": launches_per_frame, "clocks": clocks,
            "roofline": {"bound": "hbm", "kernel": "whole step (64 frames)", "achieved": frame_bytes / world / (ms * 1e-3) / 1e9, "peak": hbm,
                         "unit": "GB/s", "frac": frame_bytes / world / (ms * 1e-3) / 1e9 / hbm, "traffic": None, "peak_source": src,
                         "frame_algorithmic_bytes": frame_bytes},
            "cpu_baseline": None}
