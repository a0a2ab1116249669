"""Scenes of the plane segmentation tests, without cv2: each is an exported elevation image ((W-2)^2, row 0 the +x edge,
NaN = no data) for a map of W cells at 0.04 m centred at the origin, and the windows cut from it.  The reference's demo
terrains are stored as grey images in tests/golden/planes_golden.npz (tests/golden/make_plane_golden.py reads the PNGs);
heights are grid_map's addLayerFromImage<unsigned char, 1>(image, 0, scale): 0 + scale * (grey / 255) in float."""
import hashlib
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "planes_golden.npz")
RES = 0.04

# name -> (PNG, height scale, window position, window length).  terrain.png: testPipeline.cpp:17-29 (3 m x 3 m at
# the centre, scale 1.25); the others: the scale their names give (holes.png: 1 m), the whole map.
TERRAINS = {
    "terrain": ("terrain.png", 1.25, (0.0, 0.0), (3.0, 3.0)),
    "slope": ("slope_1m_1m_20cm.png", 0.2, (0.0, 0.0), (8.0, 8.0)),
    "straight_stairs": ("straight_stairs_1m_1m_60cm.png", 0.6, (0.0, 0.0), (8.0, 8.0)),
    "real_stairs": ("real_stairs_125cm.png", 1.25, (0.0, 0.0), (8.0, 8.0)),
    "holes": ("holes.png", 1.0, (0.0, 0.0), (8.0, 8.0)),
}
BIG_W = 2049            # the largest map a handle takes: a 2047^2 window, 4.2 M cells
LIDAR_W = 202           # the default 8 m map


def params(**kw):
    from elevation_mapping_cupy_b200.plane_segmentation import PlaneSegmentationParams
    # 0.02 m, the node's value, squared is 4e-4 = 0.04^2 / 4: a window of two constant rows has exactly that error, a tie
    # on the threshold that grey-level terrains meet.  0.0205 keeps every scene's decisions clear of it.
    p = PlaneSegmentationParams(plane_patch_error_threshold=0.0205)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def terrain_image(grey, scale, seed=None):
    """The exported image of a map just large enough for the grey image, which sits at its centre (NaN around it).  A
    seed adds NaN holes, some on the image's edge."""
    h = np.float32(0.0) + np.float32(scale) * (grey.astype(np.float32) / np.float32(255.0))
    n = max(h.shape)
    img = np.full((n, n), np.nan, np.float32)
    r0, c0 = (n - h.shape[0]) // 2, (n - h.shape[1]) // 2
    img[r0:r0 + h.shape[0], c0:c0 + h.shape[1]] = h
    if seed is not None:
        _holes(img, np.random.default_rng(seed), 12)
    return img


def _holes(z, rng, count):
    n = z.shape[0]
    for _ in range(count):
        a, b, s = rng.integers(0, n), rng.integers(0, n), rng.integers(1, 6)
        z[max(a - s, 0):a + s, max(b - s, 0):b + s] = np.nan
    z[:, :2] = np.nan
    z[0:4, n // 2:n // 2 + 8] = np.nan


def synthetic(name, n=100, seed=0):
    """Synthetic (n, n) scenes."""
    rng = np.random.default_rng(seed)
    r, c = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    x = -r * RES
    z = np.zeros((n, n))
    if name == "ramps":          # a floor, a 20 degree ramp (a plane) and a 32 degree ramp (locally planar under the
        # 35 degree test, set to background by the 30 degree per-label test), each 0.5 m above what surrounds it
        z = np.where((c >= 35) & (c < 65), 0.5 + math.tan(math.radians(20)) * (x - x[-1, 0]), z)
        z = np.where(c >= 70, 1.0 + math.tan(math.radians(32)) * (x - x[-1, 0]), z)
    elif name == "stairs":       # 0.15 m steps of 12 cells
        z = 0.15 * (r // 12)
    elif name == "holes":        # seeded NaN holes, some on the window edge, on a gently sloped floor with noise
        z = 0.05 * x + 0.002 * rng.standard_normal((n, n))
        _holes(z, rng, 25)
    elif name == "diagonal":     # planar squares that touch only at a corner, separated by rough ground
        z = 0.3 * rng.standard_normal((n, n))
        z[20:40, 20:40] = 0.2
        z[40:60, 40:60] = 0.4
        z[70:72, 10:12] = 0.1
    elif name == "rough":        # rough terrain with flat patches of several sizes
        z = 0.05 * rng.standard_normal((n, n))
        for k in range(8):
            a, b, s = rng.integers(5, n - 10), rng.integers(5, n - 10), rng.integers(2, 9)
            z[a:a + s, b:b + s] = 0.01 * k
    elif name == "empty":
        z = np.full((n, n), np.nan)
    return z.astype(np.float32)


def big_image(seed=7):
    """A (BIG_W - 2)^2 scene: 256-cell tiles of stairs, ramps, flat floor and rough ground, with seeded holes."""
    n = BIG_W - 2
    rng = np.random.default_rng(seed)
    r, c = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    kind = ((r // 256) * 7 + (c // 256) * 3) % 4
    z = np.where(kind == 0, 0.15 * ((r % 256) // 12), 0.0)
    z = np.where(kind == 1, math.tan(math.radians(15)) * (r % 256) * RES, z)
    z = np.where(kind == 2, 0.1 * ((r // 256) % 3), z)
    z = np.where(kind == 3, 0.05 * rng.standard_normal((n, n)), z)
    z = z + 0.5 * ((r // 256 + c // 256) % 2)
    z = z.astype(np.float32)
    for _ in range(400):
        a, b, s = rng.integers(0, n), rng.integers(0, n), rng.integers(1, 12)
        z[max(a - s, 0):a + s, max(b - s, 0):b + s] = np.nan
    z[:, :3] = np.nan
    return z


def lidar_frames(m, n_frames=4):
    """Feeds the default workload's LiDAR frames into m (an ElevationMap or the oracle map: the same calls)."""
    from elevation_mapping_cupy_b200 import workloads as wl
    for f in range(n_frames):
        pts, R, t = wl.lidar_cloud(3, f, n_rings=32, n_az=1250, max_range=4.0)
        m.move_to(t, R)
        m.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)


def lidar_window(center):
    """The node's window on the LiDAR map: 0.3 m ahead and 0.2 m to the right of the map centre (the robot)."""
    return (float(center[0]) + 0.3, float(center[1]) - 0.2)


def oracle_export(om):
    """The exported elevation of the oracle map: is_valid ? elevation + centre z (float) : NaN, interior flipped."""
    m = om.elevation_map
    e = np.where(m[2] > 0.5, (m[0] + np.float32(om.center[2])).astype(np.float32), np.float32(np.nan))
    return np.ascontiguousarray(e[1:-1, 1:-1][::-1, ::-1], np.float32)


def set_image(em, img):
    """Makes img the exported elevation of em (centre at the origin)."""
    m, nm = em.get_state()
    m[:] = 0
    m[0, 1:-1, 1:-1] = np.nan_to_num(img[::-1, ::-1])
    m[2, 1:-1, 1:-1] = ~np.isnan(img[::-1, ::-1])
    em.set_state(m, nm, np.zeros(3))


def digest(a, dtype=np.float32):
    return hashlib.sha256(np.ascontiguousarray(a, dtype).tobytes()).hexdigest()
