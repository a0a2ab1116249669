"""GPU: depth-image frames (ElevationMap.input_depth_image(s), emap_input_depth_images) against the cloud frame of the
same images restated on the host (tests/depth_image_oracle.py, pinned to the semantic sensor node by
tests/test_depth_image_cpu.py).  Two handles start from the same state; one fuses the images, the other input_pointcloud
/ input_sensors of the restated clouds.  Every state plane, the normals, the semantic layers and their fusion state, the
frame statistics and the kept pixels' point record must be bit-identical (the same engine runs both), and masked pixels
must be dropped rows of the record."""
import ctypes as C
import functools

import numpy as np
import pytest

import depth_image_oracle as DO

pytestmark = pytest.mark.gpu

XYZ = ["x", "y", "z"]
FUSIONS = {"rgb": "color", "avg": "average", "ca": "class_average", "bi": "bayesian_inference", "cm": "class_max"}
STATS = ["mean_error", "additive_mean_error", "shift_applied", "error_sum", "error_cnt", "drift_applied",
         "drift_evaluated", "n_points", "n_valid_points", "ray_steps", "ray_visits"]


@functools.lru_cache(maxsize=None)
def _image(frame, width, height, sensor=0):
    from elevation_mapping_cupy_b200 import workloads as wl
    depth, P, R, t = wl.depth_image(frame, width, height, sensor=sensor)
    rng = np.random.default_rng(1000 + 10 * frame + sensor)
    conf = rng.uniform(0.0, 20.0, depth.shape).astype(np.float32)
    conf[rng.random(depth.shape) < 0.05] = np.float32(10.0)            # exactly at the default threshold: kept
    rgb = rng.integers(0, 256, (height, width, 3), dtype=np.uint8)
    avg = rng.random(depth.shape, dtype=np.float32) * 2 - 0.5
    ca = rng.random(depth.shape, dtype=np.float32)
    bi = rng.random(depth.shape, dtype=np.float32)
    prob = rng.random(depth.shape, dtype=np.float32).astype(np.float16).view(np.uint16).astype(np.uint32)
    cm = ((rng.choice(np.array([0, 2, 5, 9], np.uint32), depth.shape) << 16) | prob).view(np.float32)
    return depth, P, R, t, conf, rgb, np.stack([avg, ca, bi, cm])


def _param(W):
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(W)
    p.pointcloud_channel_fusions = dict(FUSIONS)
    return p


def _pair(W):
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    return ElevationMap(_param(W)), ElevationMap(_param(W))


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype in (np.float32, np.int32) else a


def _same_frame(ed, ec, n_pixels, kept, label, twin_is_depth=False):
    """state, normals, semantic state and statistics of ed (depth frame) == ec (cloud frame, or with twin_is_depth the
    same depth frame); kept pixels' record"""
    sd, nd = ed.get_state()
    sc, nc = ec.get_state()
    for li in range(7):
        assert np.array_equal(_bits(sd[li]), _bits(sc[li])), (label, "layer", li, int((_bits(sd[li]) != _bits(sc[li])).sum()))
    assert np.array_equal(_bits(nd), _bits(nc)), (label, "normals")
    a, b = ed.get_frame_stats(), ec.get_frame_stats()
    for f in STATS:
        assert getattr(a, f) == getattr(b, f), (label, f, getattr(a, f), getattr(b, f))
    assert a.n_points == int(kept.sum()), label
    idx, valid, inside = ed.get_point_record(n_pixels)
    ci, cv, cs = ec.get_point_record(n_pixels if twin_is_depth else int(kept.sum()))
    if twin_is_depth:
        ci, cv, cs = ci[kept], cv[kept], cs[kept]
    assert np.array_equal(idx[kept], ci) and np.array_equal(valid[kept], cv) and np.array_equal(inside[kept], cs), label
    assert (idx[~kept] == -1).all() and not valid[~kept].any() and not inside[~kept].any(), label
    smd, smc = ed.semantic_map, ec.semantic_map
    if smd.semantic_map is not None:
        assert smd.layer_names == smc.layer_names
        assert np.array_equal(_bits(smd.semantic_map.cpu().numpy()), _bits(smc.semantic_map.cpu().numpy())), (label, "semantic")
        if smc.variance is not None:
            assert np.array_equal(_bits(smd.variance.cpu().numpy()), _bits(smc.variance.cpu().numpy())), (label, "variance")
        if "id_max" in smc.elements_to_shift:
            assert np.array_equal(smd.elements_to_shift["id_max"].cpu().numpy(),
                                  smc.elements_to_shift["id_max"].cpu().numpy()), (label, "id_max")


def _sources(channels):
    src, k = [], 0
    for ch in channels:
        if FUSIONS[ch] == "color":
            src.append(-1)
        else:
            src.append(k); k += 1
    return src


def _feature_planes(feats, channels):
    return feats[[["avg", "ca", "bi", "cm"].index(c) for c in channels if c != "rgb"]]


# ---- 1. geometry -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [202, 1024])
@pytest.mark.parametrize("size", [(640, 480), (1000, 1000)])
def test_geometry_frames_equal_cloud_frames(W, size):
    ed, ec = _pair(W)
    for f in range(3):
        depth, P, R, t, conf, _, _ = _image(f, *size)
        use_conf = f == 1
        cloud, kept = DO.depth_cloud(depth, P, confidence=conf if use_conf else None)
        for m in (ed, ec):
            m.move_to(t, R)
        ed.input_depth_image(depth, P, R, t, 0.02, 0.02, confidence=conf if use_conf else None)
        ec.input_pointcloud(cloud, XYZ, R, t, 0.02, 0.02)
        _same_frame(ed, ec, depth.size, kept, f"{W} {size} frame {f}")


# ---- 2. channels -------------------------------------------------------------------------------------------------------
def test_channel_frames_equal_cloud_frames():
    channels = ["rgb", "avg", "ca", "bi", "cm"]
    ed, ec = _pair(202)
    for f in range(3):
        depth, P, R, t, conf, rgb, feats = _image(f, 640, 480)
        planes = _feature_planes(feats, channels)
        cloud, kept = DO.depth_cloud(depth, P, _sources(channels), rgb=rgb, features=planes, confidence=conf)
        for m in (ed, ec):
            m.move_to(t, R)
        ed.input_depth_image(depth, P, R, t, 0.02, 0.02, channels=channels, rgb=rgb, features=planes, confidence=conf)
        ec.input_pointcloud(cloud, XYZ + channels, R, t, 0.02, 0.02)
        _same_frame(ed, ec, depth.size, kept, f"channels frame {f}")


# ---- 3. several cameras ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_cam", [2, 3, 4])
def test_several_cameras_equal_input_sensors(n_cam):
    channels = ["ca", "rgb"]
    ed, ec = _pair(202)
    cams, clouds, kept = [], [], []
    for s in range(n_cam):
        depth, P, R, t, conf, rgb, feats = _image(0, 640, 480, sensor=s)
        planes = _feature_planes(feats, channels)
        cams.append(dict(depth=depth, P=P, R=R, t=t, rgb=rgb, features=planes, confidence=conf if s % 2 else None))
        c, k = DO.depth_cloud(depth, P, _sources(channels), rgb=rgb, features=planes, confidence=conf if s % 2 else None)
        clouds.append(c); kept.append(k)
    ec.semantic_map.configure_for(XYZ + channels)
    ed.input_depth_images(cams, 0.02, 0.02, channels=channels)
    ec.input_sensors(clouds, [c["R"] for c in cams], [c["t"] for c in cams], 0.02, 0.02)
    _same_frame(ed, ec, sum(c["depth"].size for c in cams), np.concatenate(kept), f"{n_cam} cameras")


# ---- 4. input kinds ----------------------------------------------------------------------------------------------------
def test_host_pinned_and_device_images_agree_and_launch_like_clouds():
    import torch
    channels = ["rgb", "cm"]
    depth, P, R, t, conf, rgb, feats = _image(0, 640, 480)
    planes = _feature_planes(feats, channels)
    cloud, _ = DO.depth_cloud(depth, P, _sources(channels), rgb=rgb, features=planes, confidence=conf)
    pin = lambda a: torch.from_numpy(a).pin_memory()
    dev = lambda a: torch.from_numpy(a).cuda()
    kinds = {"pageable": lambda a: a, "pinned": pin, "device": dev}
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    results = {}
    for name, to in kinds.items():
        em = ElevationMap(_param(202))
        em.move_to(t, R)
        em.input_depth_image(to(depth), P, R, t, 0.02, 0.02, channels=channels, rgb=to(rgb), features=to(planes),
                             confidence=to(conf))
        n0 = em.launch_count()
        em.input_depth_image(to(depth), P, R, t, 0.02, 0.02, channels=channels, rgb=to(rgb), features=to(planes),
                             confidence=to(conf))
        launches = em.launch_count() - n0
        state, normal = em.get_state()
        results[name] = (state, normal, em.semantic_map.semantic_map.cpu().numpy(), launches)
        # the cloud frame of the same kind of memory
        ec = ElevationMap(_param(202))
        ec.move_to(t, R)
        ec.input_pointcloud(cloud, XYZ + channels, R, t, 0.02, 0.02)
        m0 = ec.launch_count()
        ec.input_pointcloud(dev(cloud) if name == "device" else cloud, XYZ + channels, R, t, 0.02, 0.02)
        assert launches == ec.launch_count() - m0, (name, launches, ec.launch_count() - m0)
    ref = results["pageable"]
    for name, r in results.items():
        for a, b in zip(r[:3], ref[:3]):
            assert np.array_equal(_bits(a), _bits(b)), name


# ---- 5. CUDA graph -----------------------------------------------------------------------------------------------------
def test_captured_device_frame_equals_eager():
    import torch
    channels = ["ca"]
    depth, P, R, t, conf, _, feats = _image(1, 640, 480)
    planes = _feature_planes(feats, channels)
    ed, ee = _pair(256)
    d_depth, d_conf, d_feat = (torch.from_numpy(a).cuda() for a in (depth, conf, planes))
    s = torch.cuda.Stream()
    ed.set_stream(s.cuda_stream)
    for m in (ed, ee):
        m.move_to(t, R)
    call = lambda m: m.input_depth_image(d_depth, P, R, t, 0.02, 0.02, channels=channels, features=d_feat, confidence=d_conf)
    with torch.cuda.stream(s):
        call(ed)                               # eager first: every buffer of the frame at its size
    s.synchronize()
    call(ee)
    torch.cuda.synchronize()
    before = _bits(ed.get_state()[0]).copy()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        call(ed)
    assert np.array_equal(_bits(ed.get_state()[0]), before), "capture ran the frame"
    call(ee)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g.replay()
    s.synchronize()
    torch.cuda.synchronize()
    _same_frame(ed, ee, depth.size, DO.keep_mask(depth, conf).reshape(-1), "graph replay", twin_is_depth=True)


# ---- 6. edge cases -----------------------------------------------------------------------------------------------------
def test_all_masked_equals_empty_cloud():
    depth, P, R, t, _, _, _ = _image(0, 640, 480)
    ed, ec = _pair(202)
    for m in (ed, ec):
        m.move_to(t, R)
    ed.input_depth_image(depth, P, R, t, 0.02, 0.02)
    ec.input_pointcloud(DO.depth_cloud(depth, P)[0], XYZ, R, t, 0.02, 0.02)
    bad = np.full_like(depth, np.nan)
    bad[::3] = 9.0
    bad[1::3] = 0.0
    ed.input_depth_image(bad, P, R, t, 0.02, 0.02)
    ec.input_pointcloud(np.zeros((0, 3), np.float32), XYZ, R, t, 0.02, 0.02)
    _same_frame(ed, ec, depth.size, np.zeros(depth.size, bool), "all masked")


def test_invalid_arguments_launch_nothing():
    """every rejection of include/emap.h returns EMAP_ERR_INVALID for its own reason (the message names it), launches
    nothing and leaves the state as it was"""
    from elevation_mapping_cupy_b200 import _lib
    depth, P, R, t, conf, rgb, feats = _image(0, 640, 480)
    em, _ = _pair(202)
    em.move_to(t, R)
    em.input_depth_image(depth, P, R, t, 0.02, 0.02)
    state0 = [_bits(a).copy() for a in em.get_state()]
    n0 = em.launch_count()

    def cam(**kw):
        c = _lib.EmapDepthCamera()
        c.height, c.width = kw.get("H", 480), kw.get("W", 640)
        c.depth = kw.get("depth", depth.ctypes.data)
        c.rgb = kw.get("rgb", rgb.ctypes.data)
        c.features = kw.get("features", feats.ctypes.data)
        c.fx, c.fy, c.cx, c.cy = kw.get("fx", P[0, 0]), kw.get("fy", P[1, 1]), kw.get("cx", P[0, 2]), P[1, 2]
        c.R[:] = kw.get("R", R.reshape(9).tolist())
        c.t[:] = kw.get("t", t.tolist())
        return c

    def call(c, src=(), n_features=4, n_cam=1, n_channels=None):
        arr = (_lib.EmapDepthCamera * max(1, n_cam))(*([c] * max(1, n_cam)))
        s = (C.c_int32 * max(1, len(src)))(*src)
        rc = em._L.emap_input_depth_images(em._h, n_cam, arr, 0, len(src) if n_channels is None else n_channels, s,
                                           n_features, 10.0, 8.0, 0.02, 0.02)
        return rc, em._L.emap_last_error(em._h).decode()

    SIZE, INTR, SRC, NEEDS = "0 < height * width <= 2^24", "non-finite or zero fx", "channel source outside", "needs rgb"
    COUNT = "0..16 channels"
    cases = {
        "null depth": (call(cam(depth=None)), SIZE),
        "zero height": (call(cam(H=0)), SIZE),
        "negative width": (call(cam(W=-4)), SIZE),
        "over 2^24 pixels": (call(cam(H=4097, W=4097)), SIZE),
        "zero fx": (call(cam(fx=0.0)), INTR),
        "nan fy": (call(cam(fy=float("nan"))), INTR),
        "inf cx": (call(cam(cx=float("inf"))), INTR),
        "nan R": (call(cam(R=[float("nan")] + [0.0] * 8)), INTR),
        "inf t": (call(cam(t=[0.0, float("inf"), 0.0])), INTR),
        "source too large": (call(cam(), src=(4,)), SRC),
        "source below -1": (call(cam(), src=(-2,)), SRC),
        "colour without rgb": (call(cam(rgb=None), src=(-1,)), NEEDS),
        "feature without features": (call(cam(features=None), src=(0,)), NEEDS),
        "two colour channels": (call(cam(), src=(-1, -1)), "more than one colour channel"),
        "17 channels": (call(cam(), src=tuple(range(4)) * 4 + (0,)), COUNT),
        "negative n_channels": (call(cam(), n_channels=-1), COUNT),
        "256 feature planes": (call(cam(), n_features=256), COUNT),
        "negative n_features": (call(cam(), n_features=-1), COUNT),
        "no cameras": (call(cam(), n_cam=0), "n_cameras"),
        "17 cameras": (call(cam(), n_cam=17), "n_cameras"),
    }
    # a semantic configuration whose columns address channel 3 + 1: a call with one channel cannot feed it
    em.semantic_map.configure_for(XYZ + ["ca", "avg"])
    cases["configured column beyond the channels"] = (call(cam(), src=(0,)), "configured semantic column")
    for name, ((rc, msg), want) in cases.items():
        assert rc == -1 and want in msg, (name, rc, msg)
    assert em.launch_count() == n0
    for a, b in zip(state0, em.get_state()):
        assert np.array_equal(a, _bits(b))


# ---- mask boundaries in the kernel ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_depth,threshold", [(8.0, 10.0), (6.5, 0.3)])
def test_special_depths_and_thresholds_equal_cloud_frames(max_depth, threshold):
    """NaN, +-inf, 0, -0, negative depths, max_depth and the float just below it, confidence below, at and above the
    threshold (not an fp32 value in the second case): the kernel's mask is the restatement's"""
    H, W = 240, 320
    rng = np.random.default_rng(5)
    depth = DO.special_depth(rng, H, W, max_depth)
    assert (depth == np.float32(max_depth)).any() and (depth == np.nextafter(np.float32(max_depth), 0)).any()
    assert np.isposinf(depth).any() and (np.signbit(depth) & (depth == 0)).any()
    th = np.float32(threshold)
    conf = rng.choice(np.array([th, np.nextafter(th, 0), np.nextafter(th, np.inf), 0.0, 2 * threshold, np.nan],
                               np.float32), (H, W))
    P = np.array([[160.25, 0, 159.7, 0], [0, 160.5, 119.2, 0], [0, 0, 1, 0]], np.float64)
    from elevation_mapping_cupy_b200 import workloads as wl
    _, _, R, t = wl.depth_image(0, 8, 6)
    ed, ec = _pair(202)
    for use_conf in (False, True):
        cloud, kept = DO.depth_cloud(depth, P, confidence=conf if use_conf else None, confidence_threshold=threshold,
                                     max_depth=max_depth)
        ed.input_depth_image(depth, P, R, t, 0.02, 0.02, confidence=conf if use_conf else None,
                             confidence_threshold=threshold, max_depth=max_depth)
        ec.input_pointcloud(cloud, XYZ, R, t, 0.02, 0.02)
        _same_frame(ed, ec, depth.size, kept, f"special depths max {max_depth} threshold {threshold} conf {use_conf}")


# ---- converted device inputs ---------------------------------------------------------------------------------------------
def test_converted_device_inputs_outlive_the_call():
    """a float64 device depth, a non-contiguous device rgb (an HWC view of a CHW tensor) and a list of device feature
    planes are converted into temporaries the call frees on return; tensors allocated and filled on the current stream
    right after each call must not reach the frame.  The handle runs on a side stream that sleeps before each frame, so
    the frame reads its inputs well after the call has returned."""
    import torch
    channels = ["rgb", "ca", "avg"]
    ed, ec = _pair(1024)
    side = torch.cuda.Stream()
    ed.set_stream(side.cuda_stream)
    for f in range(3):
        depth, P, R, t, conf, rgb, feats = _image(f, 1000, 1000)
        planes = _feature_planes(feats, channels)
        cloud, kept = DO.depth_cloud(depth, P, _sources(channels), rgb=rgb, features=planes, confidence=conf)
        d64 = torch.from_numpy(depth.astype(np.float64)).cuda()
        rgb_hwc = torch.from_numpy(np.ascontiguousarray(rgb.transpose(2, 0, 1))).cuda().permute(1, 2, 0)
        assert not rgb_hwc.is_contiguous()
        plane_list = [torch.from_numpy(p).cuda() for p in planes]
        d_conf = torch.from_numpy(conf).cuda()
        for m in (ed, ec):
            m.move_to(t, R)
        with torch.cuda.stream(side):
            torch.cuda._sleep(50_000_000)
        ed.input_depth_image(d64, P, R, t, 0.02, 0.02, channels=channels, rgb=rgb_hwc, features=plane_list,
                             confidence=d_conf)
        junk = [torch.full((1000, 1000), float("nan"), device="cuda"), torch.full((1000, 1000, 3), 255, dtype=torch.uint8,
                                                                                   device="cuda"),
                torch.full((2, 1000, 1000), -7.0, device="cuda")]
        ec.input_pointcloud(cloud, XYZ + channels, R, t, 0.02, 0.02)
        torch.cuda.synchronize()
        del junk
        _same_frame(ed, ec, depth.size, kept, f"converted inputs frame {f}")
