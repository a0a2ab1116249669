"""Camera image fusion on the device (ElevationMap.input_image / emap_input_image) against the reference's own kernels
built by nvcc for sm_90a (oracle/build_ref_image.py: image_to_map_correspondence_kernel, then one colour or exponential
launch per channel), run on the same card, the same state, P and camera cell.  Layers are compared bit for bit."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import image_oracle as IO          # noqa: E402

pytestmark = pytest.mark.gpu

TAGS = {202: "core202", 1024: "core1024", 2048: "core2048"}
OPT = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], np.float64)     # sensor (x forward, y left, z up) -> optical


def intrinsics(H, Wi):
    f = 0.5 * Wi / np.tan(np.deg2rad(87.0 / 2))
    return np.array([[f, 0, (Wi - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1]], np.float32)


def cam_pose(frame, offset=(0.0, 0.0, 0.0)):
    """Map -> optical R, t of the depth camera of workloads.depth_camera_cloud, moved by offset (metres)."""
    from elevation_mapping_cupy_b200 import workloads as wl
    _, Rs, ts = wl.depth_camera_cloud(0, frame, width=8, height=8)
    R = (OPT @ Rs.astype(np.float64).T).astype(np.float32)
    pos = ts.astype(np.float64) + np.asarray(offset)
    return R, (-R.astype(np.float64) @ pos).astype(np.float32)


class RefImage:
    def __init__(self, W):
        so = os.path.join(ROOT, "oracle", "_ref", f"libref_image_gpu_{TAGS[W]}.so")
        if not os.path.exists(so):
            raise FileNotFoundError(so)
        L = self.lib = C.CDLL(so)
        fp = C.c_void_p
        L.ref_image_corr.argtypes = [C.c_longlong, fp, C.c_float, C.c_float, C.c_float, fp, fp, fp, C.c_float, C.c_float,
                                     fp, fp, fp, fp]
        for fn in (L.ref_image_color, L.ref_image_exponential):
            fn.argtypes = [C.c_longlong, fp, C.c_float, fp, fp, fp, C.c_float, C.c_float, fp, fp]
        assert L.ref_image_cell_n() == W
        self.W = W

    def fuse(self, state, center, sem, img, K, D, model, R, t, chans):
        """EM.py:510-562 with the reference's kernels on torch tensors; sem is updated in place.  Returns (uv, valid)."""
        import torch
        W, L = self.W, self.lib
        cam = IO.camera(K, D, model, R, t, center, W, 0.04)
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda()
        P, Kd, Dd, cd = d(cam["P"]), d(K), d(cam["D"]), d(center)
        uv = torch.zeros((2, W, W), dtype=torch.float32, device="cuda")
        valid = torch.zeros((W, W), dtype=torch.bool, device="cuda")
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = lambda x: C.c_void_p(x.data_ptr())
        _, H, Wi = img.shape
        assert L.ref_image_corr(W * W, p(state), cam["x1"], cam["y1"], cam["z1"], p(P), p(Kd), p(Dd), float(H), float(Wi),
                                p(cd), p(uv), p(valid), st) == 0
        for plane, kind, layer in chans:
            new = torch.zeros_like(sem)
            if kind == "color":
                L.ref_image_color(W * W, p(sem), float(layer), p(img), p(uv), p(valid), float(H), float(Wi), p(new), st)
            else:
                L.ref_image_exponential(W * W, p(sem), float(layer), p(img[plane]), p(uv), p(valid), float(H), float(Wi),
                                        p(new), st)
            sem[layer] = new[layer]
        return uv, valid


def _map(W, frames=3, **kw):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    em = ElevationMap(core_parameter(W, plugin_config_file="", **kw))
    for f in range(frames):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=1000, max_range=0.45 * W * 0.04)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    return em


def _image(n_planes, H, Wi, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (n_planes, H, Wi)).astype(np.float32)
    if n_planes > 3:
        img[3:] = rng.normal(0, 2, (n_planes - 3, H, Wi))
    return img


def _bits(t):
    import torch
    return t.contiguous().view(torch.int32).cpu().numpy()


def _check_call(em, ref, img, channels, R, t, K, D, model, host=True):
    """One input_image call against the reference sequence on a snapshot of the same state and layers."""
    import torch
    sm = em.semantic_map
    for ch in channels:                         # layers exist before the snapshot (adding them is not under test here)
        if ch not in sm.layer_names:
            sm.add_layer(ch)
    planes, kinds, layers = sm.update_layers_image(list(channels))
    chans = [(p, ["color", "exponential"][k], l) for p, k, l in zip(planes, kinds, layers)]
    state = em.elevation_map.clone()
    sem_ref = sm.semantic_map.clone()
    center = em.center
    img_d = torch.from_numpy(img).cuda()
    ref.fuse(state, center, sem_ref, img_d, K, D, model, R, t, chans)
    H, Wi = img.shape[1:]
    em.input_image(img if host else img_d, channels, R, t, K, D, model, H, Wi)
    got = sm.semantic_map
    assert np.array_equal(_bits(got), _bits(sem_ref)), f"{int((_bits(got) != _bits(sem_ref)).sum())} cells differ"
    return sem_ref


@pytest.mark.parametrize("W", [202, 1024, 2048])
def test_bit_identical_to_reference_kernels(W):
    """3 rgb + 2 feature planes at 1280 x 720, colour and exponential channels, host and device images, repeated calls
    with random prefilled layers and the radtan model."""
    import torch
    em = _map(W)
    ref = RefImage(W)
    K = intrinsics(720, 1280)
    D = np.array([-0.05, 0.01, 1e-3, -1e-3, 0.002], np.float32)
    chans = ["rgb", "p1", "p2", "feat_a", "feat_b"]
    n_valid = 0
    for call in range(4):
        R, t = cam_pose(call)
        if call == 1:
            for k in range(len(em.semantic_map.layer_names)):
                em.semantic_map.semantic_map[k] = torch.randn((W, W), device="cuda")
        sem = _check_call(em, ref, _image(5, 720, 1280, call), chans, R, t, K, D, ["radtan", "plumb_bob"][call % 2],
                          host=call % 2 == 0)
        n_valid += int((_bits(sem[3]) != 0).sum())
    assert n_valid > 1000


@pytest.mark.parametrize("size", [(480, 640), (720, 1280)])
def test_color_layer_holds_the_reference_pixel(size):
    """r, g, b planes encoding each pixel's own index and a marker-filled layer: the colour layer's bits are the pixel
    index the reference's correspondence gives, and the marker where the reference's valid is false."""
    import torch
    H, Wi = size
    W = 202
    em = _map(W)
    ref = RefImage(W)
    K = intrinsics(H, Wi)
    idx = np.arange(H * Wi, dtype=np.int64).reshape(H, Wi)
    img = np.stack([idx >> 16, (idx >> 8) & 255, idx & 255]).astype(np.float32)
    em.semantic_map.add_layer("rgb")
    marker = np.float32(-1234.5)
    em.semantic_map.semantic_map[0] = float(marker)
    R, t = cam_pose(2)
    state = em.elevation_map.clone()
    uv, valid = ref.fuse(state, em.center, em.semantic_map.semantic_map.clone(), torch.from_numpy(img).cuda(), K,
                         np.zeros(5, np.float32), "none", R, t, [])
    em.input_image([img[0], img[1], img[2]], ["rgb"], R, t, K, np.zeros(5), "none", H, Wi)
    got = _bits(em.semantic_map.semantic_map[0])
    uv, valid = uv.cpu().numpy(), valid.cpu().numpy()
    pix = IO.pixel(uv[0], uv[1], Wi)
    assert valid.sum() > 500
    assert np.array_equal(got[valid], pix[valid])
    assert (got[~valid] == marker.view(np.int32)).all()


@pytest.mark.parametrize("n_planes", [1, 3, 5])
@pytest.mark.parametrize("model", ["radtan", "equidistant"])
def test_planes_models_and_far_camera(n_planes, model):
    W = 202
    em = _map(W)
    ref = RefImage(W)
    K = intrinsics(480, 640)
    D = np.array([-0.2, 0.05, 2e-3, -1e-3], np.float32)
    chans = (["rgb", "c1", "c2", "c3", "c4"] if n_planes >= 3 else ["mono"])[:n_planes]
    for off in [(0, 0, 0), (20.0, -3.0, 4.0), (-0.5, 0.5, 0.3)]:        # the second camera is far outside the map
        R, t = cam_pose(1, off)
        _check_call(em, ref, _image(n_planes, 480, 640, n_planes), chans, R, t, K, D, model)


def test_side_stream_and_interleaved_point_frames():
    """Images on a torch side stream, alternating with semantic and xyz-only point frames, move, move_to and clear; and
    an image that adds a layer after point channels were configured (the point fusion must follow the new buffer)."""
    import torch
    from elevation_mapping_cupy_b200 import workloads as wl
    W = 202
    em = _map(W, frames=1)
    ref = RefImage(W)
    K = intrinsics(480, 640)
    rng = np.random.default_rng(0)
    s = torch.cuda.Stream()
    for f in range(6):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=16, n_az=500, max_range=3.5)
        if f % 2 == 0:
            rgb = rng.integers(0, 1 << 24, len(pts)).astype(np.uint32).view(np.float32)
            cloud = np.concatenate([pts, rgb[:, None], rng.random((len(pts), 1), dtype=np.float32)], 1)
            em.input_pointcloud(cloud, ["x", "y", "z", "rgb", "feat"], R, t, 0.02, 0.02)
        else:
            em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        if f == 2:
            em.move(np.array([0.2, -0.12, 0.0]))
        if f == 3:
            em.move_to(t, R)
        if f == 4:
            em.clear()
        Rc, tc = cam_pose(f)
        with torch.cuda.stream(s):
            _check_call(em, ref, _image(4, 480, 640, f), ["rgb", "g", "b", f"cam_feat_{f % 3}"], Rc, tc, K,
                        np.zeros(5, np.float32), "none", host=f % 2 == 1)
        torch.cuda.synchronize()
    # a new layer from an image after the point channels were registered, then a feature frame and an xyz frame
    n_before = len(em.semantic_map.layer_names)
    Rc, tc = cam_pose(0)
    em.input_image(_image(2, 480, 640, 9), ["x_new_a", "x_new_b"], Rc, tc, K, np.zeros(5), "none", 480, 640)
    assert len(em.semantic_map.layer_names) == n_before + 2
    pts, R, t = wl.lidar_cloud(0, 7, n_rings=16, n_az=500, max_range=3.5)
    rgb = np.full(len(pts), np.uint32(0x00102030)).view(np.float32)
    cloud = np.concatenate([pts, rgb[:, None], np.full((len(pts), 1), 0.25, np.float32)], 1)
    em.input_pointcloud(cloud, ["x", "y", "z", "rgb", "feat"], R, t, 0.02, 0.02)
    em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    torch.cuda.synchronize()
    col = _bits(em.semantic_map.semantic_map[em.semantic_map.layer_names.index("rgb")])
    assert (col == 0x00102030).sum() > 100           # the point frame wrote the live buffer
    Rc, tc = cam_pose(1)
    _check_call(em, ref, _image(2, 480, 640, 10), ["x_new_a", "x_new_b"], Rc, tc, K, np.zeros(5, np.float32), "none")


def test_rejections():
    import torch
    W = 202
    em = _map(W, frames=1)
    L, h = em._L, em._h
    sem = torch.zeros((2, W, W), dtype=torch.float32, device="cuda")
    img = np.zeros((3, 48, 64), np.float32)
    K = intrinsics(48, 64).reshape(-1).copy()
    R, t = cam_pose(0)
    R, t = R.reshape(-1).copy(), t.copy()
    D = np.zeros(5, np.float32)
    a32 = lambda *v: (C.c_int32 * len(v))(*v)

    def call(n_planes=3, image=img.ctypes.data, H=48, Wi=64, K_=K, R_=R, t_=t, model=b"none", plane=(0,), kind=(0,),
             layer=(1,), sem_p=sem.data_ptr(), n_layers=2, Dp=D.ctypes.data, n_D=5):
        n = len(plane)
        return L.emap_input_image(h, n_planes, image, 0, H, Wi, K_.ctypes.data if K_ is not None else None, Dp, n_D,
                                  model, R_.ctypes.data if R_ is not None else None,
                                  t_.ctypes.data if t_ is not None else None, n, a32(*plane), a32(*kind), a32(*layer),
                                  sem_p, n_layers)

    assert call() == 0
    bad = np.array(K); bad[0] = np.nan
    far = np.array(t); far[0] = -1e7
    far2 = np.array(t); far2[1] = 1e7
    inf = np.array(R); inf[4] = np.inf
    cases = [dict(image=None), dict(K_=None), dict(R_=None), dict(t_=None), dict(model=None), dict(sem_p=None),
             dict(Dp=None), dict(H=4096, Wi=4097), dict(n_planes=2), dict(plane=(3,)), dict(plane=(0, 5), kind=(1, 1), layer=(0, 1)),
             dict(layer=(2,)), dict(layer=(-1,)), dict(kind=(2,)), dict(K_=bad), dict(R_=inf), dict(t_=far),
             dict(t_=far2)]
    for c in cases:
        assert call(**c) == -1, c
    assert call(n_planes=1, plane=(0,), kind=(1,)) == 0
