"""Host-side resources of a handle: the pinned staging of host images (emap_input_image) and of initialize_map uploads
(emap_initialize_map), and everything a handle allocates on demand being released when it is closed."""
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W = 202
OPT = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], np.float64)     # sensor (x forward, y left, z up) -> optical
CHANNELS = ["rgb", "p1", "p2", "feat_a", "feat_b"]                  # one colour and four exponential channels


def _map(frames=2):
    from elevation_mapping_cupy_b200 import workloads as wl
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    em = ElevationMap(core_parameter(W, plugin_config_file=""))
    for f in range(frames):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=32, n_az=1000, max_range=0.45 * W * 0.04)
        em.move_to(t, R)
        em.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
    return em


def _camera(frame, H, Wi):
    """Map -> optical R, t of the depth camera of workloads.depth_camera_cloud, and 87-degree intrinsics."""
    from elevation_mapping_cupy_b200 import workloads as wl
    _, Rs, ts = wl.depth_camera_cloud(0, frame, width=8, height=8)
    R = (OPT @ Rs.astype(np.float64).T).astype(np.float32)
    t = (-R.astype(np.float64) @ ts.astype(np.float64)).astype(np.float32)
    f = 0.5 * Wi / np.tan(np.deg2rad(87.0 / 2))
    K = np.array([[f, 0, (Wi - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1]], np.float32)
    return R, t, K


def _image(H, Wi, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (len(CHANNELS), H, Wi)).astype(np.float32)
    img[3:] = rng.normal(0, 2, (len(CHANNELS) - 3, H, Wi))
    return img


def _init_points(n, seed):
    rng = np.random.default_rng(seed)
    half = (W - 2) * 0.04 / 2
    return np.c_[rng.uniform(-half, half, (n, 2)), rng.normal(0, 0.3, n)].astype(np.float32)


def _same_bits(a, b):
    import torch
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# growing sizes: every call regrows the staging while the previous call's upload may still be queued
IMAGE_SIZES = [(60, 80), (120, 160), (240, 320), (480, 640), (720, 1280)]
INIT_CALLS = [(16, "nearest"), (200, "linear"), (2000, "cubic"), (4000, "cubic")]


def _image_run(poison):
    """Semantic layers after each host-image call, snapshotted on the device (no host synchronisation in between)."""
    em = _map()
    snaps = []
    for i, (H, Wi) in enumerate(IMAGE_SIZES):
        img = _image(H, Wi, i)
        R, t, K = _camera(i, H, Wi)
        em.input_image(img, CHANNELS, R, t, K, np.zeros(5, np.float32), "none", H, Wi)
        if poison:
            img[...] = np.nan                     # the library's copy must already be taken
        snaps.append(em.semantic_map.semantic_map.clone())
    return snaps


def _init_run(poison):
    """The map after each initialize_map call, snapshotted on the device."""
    em = _map(frames=0)
    snaps = []
    for i, (n, method) in enumerate(INIT_CALLS):
        pts = _init_points(n, i)
        em.initialize_map(pts, method)           # a contiguous float32 array: the library reads this very buffer
        if poison:
            pts[...] = np.nan
        snaps.append(em.elevation_map.clone())
    return snaps


@pytest.mark.parametrize("run", [_image_run, _init_run], ids=["image", "initialize"])
def test_host_input_reusable_when_the_call_returns(run):
    """Host inputs overwritten with NaN as soon as the call returns give the layers of an untouched run, bit for bit."""
    ref, got = run(False), run(True)
    for k, (a, b) in enumerate(zip(ref, got)):
        assert _same_bits(a, b), f"call {k} differs"
    assert int((ref[-1] != 0).sum()) > 100


def _every_lazy_path():
    """One handle through every path that allocates on first use, then closed."""
    import torch
    from elevation_mapping_cupy_b200.plugins.inpainting import Inpainting
    em = _map()
    H, Wi = 480, 640
    R, t, K = _camera(0, H, Wi)
    em.input_image(_image(H, Wi, 0), CHANNELS, R, t, K, np.zeros(5, np.float32), "none", H, Wi)
    c = em.center[:2]
    poly = (c + np.array([[-1.0, -1.0], [1.0, -1.0], [1.0, 1.0], [-1.0, 1.0]], np.float32)).astype(np.float32)
    em.get_polygon_traversability(poly, np.zeros(3))
    em.get_polygons_traversability([poly, (c + 0.5 * (poly - c)).astype(np.float32)], np.zeros((2, 3)))
    assert len(em.get_map_points()) > 0
    em.get_normal_arrows()
    Inpainting(cell_n=W, method="telea", engine=em)(em.elevation_map, em.layer_names, None, [])
    em.initialize_map(_init_points(500, 0), "cubic")
    torch.cuda.synchronize()
    em.close()


def test_closed_handles_leave_no_device_memory():
    """Create, run every on-demand path, close: after a warm-up round, device free memory stays put over three rounds."""
    import torch
    free = []
    for _ in range(4):
        _every_lazy_path()
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free.append(torch.cuda.mem_get_info()[0])
    drift = max(free[1:]) - min(free[1:])
    assert drift <= 2 << 20, f"device free memory drifted by {drift} bytes over the rounds: {free}"
