"""Deterministic synthetic workloads for the tests and bench.py (SURVEY.md section 8(d)).

Terrain g(x,y) with steps (edges / walls), a 64-ring LiDAR-like scanner, a pitched
depth camera, and the reference test's uniform random cloud
(elevation_mapping_cupy/script/elevation_mapping_cupy/tests/test_elevation_mapping.py:51-61).
All clouds are (N,3) float32 in the SENSOR frame; `R`, `t` map them to the map frame
(p_map = R p + t), as ElevationMap.input_pointcloud expects (elevation_mapping.py:434-466).
"""
import numpy as np

SEED0 = 20260922


def rng_for(config, frame, extra=0):
    return np.random.default_rng(SEED0 + 1000 * config + frame + 7919 * extra)


def terrain(x, y):
    g = 0.3 * np.sin(0.5 * x) * np.cos(0.4 * y) + 0.1 * np.sin(2.1 * x + 0.7)
    g = g + 0.15 * (((np.floor(x) + np.floor(y)) % 4) == 0)
    return g


def _rot_z(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def _ray_terrain(origin, dirs, max_range, coarse=0.1, refine=10):
    """First intersection range of rays origin + r*dirs with z = terrain(x,y); max_range if none."""
    n = dirs.shape[0]
    hit = np.full(n, max_range, np.float64)
    alive = np.ones(n, bool)
    r_prev = np.zeros(n)
    steps = int(np.ceil(max_range / coarse))
    for k in range(1, steps + 1):
        r = min(k * coarse, max_range)
        ia = np.nonzero(alive)[0]
        if ia.size == 0:
            break
        p = origin[None, :] + r * dirs[ia]
        below = p[:, 2] <= terrain(p[:, 0], p[:, 1])
        ib = ia[below]
        if ib.size:
            lo = np.full(ib.size, r - coarse); hi = np.full(ib.size, r)
            lo = np.maximum(lo, 0.0)
            for _ in range(refine):
                mid = 0.5 * (lo + hi)
                pm = origin[None, :] + mid[:, None] * dirs[ib]
                b = pm[:, 2] <= terrain(pm[:, 0], pm[:, 1])
                hi = np.where(b, mid, hi); lo = np.where(b, lo, mid)
            hit[ib] = hi
            alive[ib] = False
        r_prev[:] = r
    return hit


def lidar_pose(frame, sensor=0, n_sensors=1):
    """Sensor pose in the map frame for frame f (SURVEY 8(d) B / C)."""
    f = float(frame)
    if n_sensors == 1:
        t = np.array([0.05 * f, 0.02 * f, 1.5])
        R = _rot_z(0.01 * f) @ _rot_y(0.02)
    else:
        offs = [(0.4, 0.3), (-0.4, 0.3), (-0.4, -0.3), (0.4, -0.3), (0.8, 0.0), (-0.8, 0.0), (0.0, 0.6), (0.0, -0.6)]
        ox, oy = offs[sensor % len(offs)]
        t = np.array([0.05 * f + ox, 0.02 * f + oy, 1.5])
        R = _rot_z(0.01 * f + 0.5 * np.pi * sensor) @ _rot_y(0.02)
    return R.astype(np.float32), t.astype(np.float32)


def lidar_cloud(config, frame, n_rings=64, n_az=3125, max_range=25.0, range_noise=0.02,
                sensor=0, n_sensors=1):
    """64 rings (elevation -25..+15 deg) x n_az azimuths, range = ray-terrain hit capped at
    max_range, range noise N(0, range_noise).  Returns (points_sensor_frame (N,3) f32, R, t)."""
    R, t = lidar_pose(frame, sensor, n_sensors)
    rng = rng_for(config, frame, sensor)
    el = np.deg2rad(np.linspace(-25.0, 15.0, n_rings))
    az = np.linspace(0.0, 2 * np.pi, n_az, endpoint=False)
    E, A = np.meshgrid(el, az, indexing="ij")
    d_s = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)
    d_m = d_s @ R.astype(np.float64).T
    rr = _ray_terrain(t.astype(np.float64), d_m, max_range)
    rr = rr + rng.normal(0.0, range_noise, rr.shape)
    pts = (d_s * rr[:, None]).astype(np.float32)
    return pts, R, t


def depth_camera_cloud(config, frame, width=1000, height=1000, max_range=12.0, nan_frac=0.05):
    """1000x1000 pixel frustum (87 x 58 deg FoV) at 1.0 m height pitched 30 deg down
    (SURVEY 8(d) D); 5 % NaN pixels."""
    f = float(frame)
    rng = rng_for(config, frame)
    t = np.array([0.03 * f, 0.01 * f, 1.0])
    R = (_rot_z(0.005 * f) @ _rot_y(np.deg2rad(30.0))).astype(np.float32)
    u = np.tan(np.deg2rad(87.0 / 2)) * np.linspace(-1, 1, width)
    v = np.tan(np.deg2rad(58.0 / 2)) * np.linspace(-1, 1, height)
    U, V = np.meshgrid(u, v, indexing="xy")
    # camera looks along +x of the sensor frame, y left, z up
    d_s = np.stack([np.ones_like(U), -U, -V], -1).reshape(-1, 3)
    d_s /= np.linalg.norm(d_s, axis=1, keepdims=True)
    d_m = d_s @ R.astype(np.float64).T
    rr = _ray_terrain(t.astype(np.float64), d_m, max_range, coarse=0.05)
    rr = rr + rng.normal(0.0, 0.005, rr.shape)
    pts = (d_s * rr[:, None]).astype(np.float32)
    bad = rng.random(pts.shape[0]) < nan_frac
    pts[bad] = np.nan
    return pts, R, t.astype(np.float32)


def uniform_cloud(config, frame, n=10000, half_extent=4.9, sensor_height=1.2, noise=0.01):
    """Config A: (x,y) ~ U(-half_extent, half_extent)^2, z = g - sensor_height + N(0, noise),
    sensor at (0,0,sensor_height), R = I."""
    rng = rng_for(config, frame)
    xy = rng.uniform(-half_extent, half_extent, (n, 2))
    z = terrain(xy[:, 0], xy[:, 1]) - sensor_height + rng.normal(0, noise, n)
    pts = np.concatenate([xy, z[:, None]], 1).astype(np.float32)
    return pts, np.eye(3, dtype=np.float32), np.array([0, 0, sensor_height], np.float32)


def reference_test_cloud(seed, n=100000, n_ch=3):
    """test_elevation_mapping.py:51-61: rand(n, n_ch) points, rand(3,3) 'R', rand(3) t."""
    rng = np.random.default_rng(seed)
    return (rng.random((n, n_ch), dtype=np.float32), rng.random((3, 3), dtype=np.float32),
            rng.random(3, dtype=np.float32))


def depth_image(frame, width=640, height=480, max_range=10.0, hole_frac=0.03, sensor=0):
    """Depth image (32FC1 metres) of the terrain from an optical camera (x right, y down, z forward) 1.0 m above the
    ground, pitched 30 deg down, with a 90 deg horizontal field of view; rays that hit nothing within max_range read
    max_range, and a fraction of pixels are holes (NaN, 0 or -inf).  Returns (depth (H, W) f32, P (3x4) f64, R, t), R, t
    the optical -> map pose in fp32.  `sensor` turns the camera by 90 deg about z per step."""
    f = float(frame)
    rng = rng_for(9, frame, sensor)
    fx = fy = 0.5 * width
    cx, cy = 0.5 * (width - 1) + 0.25, 0.5 * (height - 1) - 0.25
    P = np.array([[fx, 0, cx, 0], [0, fy, cy, 0], [0, 0, 1, 0]], np.float64)
    R_opt = np.array([[0, 0, 1], [-1, 0, 0], [0, -1, 0]], np.float64)       # optical axes in the body frame
    R = (_rot_z(0.01 * f + 0.5 * np.pi * sensor) @ _rot_y(np.deg2rad(30.0)) @ R_opt).astype(np.float32)
    t = np.array([0.04 * f + 0.2 * sensor, 0.02 * f, 1.0 + terrain(0.04 * f, 0.02 * f)], np.float32)
    u, v = np.meshgrid(np.arange(width), np.arange(height), indexing="xy")
    d_o = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u, np.float64)], -1).reshape(-1, 3)
    norm = np.linalg.norm(d_o, axis=1)
    rr = _ray_terrain(t.astype(np.float64), (d_o / norm[:, None]) @ R.astype(np.float64).T, max_range, coarse=0.1)
    depth = (rr / norm).astype(np.float32).reshape(height, width)
    depth += rng.normal(0.0, 0.003, depth.shape).astype(np.float32)
    holes = rng.random(depth.shape) < hole_frac
    depth[holes] = rng.choice(np.array([np.nan, 0.0, -np.inf], np.float32), int(holes.sum()))
    return depth, P, R, t
