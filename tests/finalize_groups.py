"""Which scratch groups k_finalize reads per cell, counted on the oracle, and the frame sequences that make each group
occur on its own (tests/test_gpu_finalize_groups.py, tests/test_finalize_groups_cpu.py, tools/finalize_groups.py).

A single-GPU frame marks a cell's points byte where a valid, inside point lands (the cells k_fuse may accumulate into)
and its rays byte where the ray-cast carves or decrements.  k_finalize takes its full path on either marker and on the
overlap-clear window, and reads the map planes plus only the flagged groups:
- points group: cnt_fo, SH, SV, last (cnt_ai is only re-zeroed: it is non-zero exactly where the marker is set);
- rays group: n_ray, ukv, DV.
The parent layout read all 14 per full-path cell.

The oracle does not expose its scratch, so the rays set is recovered from two probe frames on copies of the pre-frame
state: ray-cast on and off, both without the overlap clear.  The points side of a frame does not depend on the ray-cast,
and every ray effect changes the state of its cell (a carve lowers the upper-bound key, a decrement changes is_valid and
the variance), so the cells where the probes differ in elevation, variance, is_valid, upper_bound or is_upper_bound
are exactly the cells the ray-cast marks."""
import copy

import numpy as np

# (plane, element bytes) of a full-path cell's loads
MAP_LOADS = [("map.h", 4), ("map.v", 4), ("map.valid", 4), ("map.time", 4), ("map.upper", 4), ("map.is_upper", 4)]
PTS_LOADS = [("cnt_fo", 8), ("cnt_ai", 8), ("SH", 8), ("SV", 8), ("last", 8)]
RAY_LOADS = [("n_ray", 4), ("ukv", 4), ("DV", 8)]
PTS_LOADS_NOW = [x for x in PTS_LOADS if x[0] != "cnt_ai"]
SECTOR = 32


def _probe(om, param, **flags):
    p = copy.copy(param)
    for k, v in flags.items():
        setattr(p, k, v)
    pr = type(om)(p, nthreads=om.nthreads)
    pr.elevation_map = om.elevation_map.copy()
    pr.normal_map = om.normal_map.copy()
    pr.traversability_input = om.traversability_input.copy()
    pr.center = om.center.copy()
    pr.base_rotation = om.base_rotation.copy()
    pr.mean_error, pr.additive_mean_error = om.mean_error, om.additive_mean_error
    return pr


def frame_groups(om, pts, R, t, position_noise, orientation_noise):
    """Masks (W, W) of the frame `om` is about to fuse: points marker, rays marker, overlap-clear window.  `om` is left
    untouched."""
    p = om.param
    on = _probe(om, p, enable_overlap_clearance=False)
    off = _probe(om, p, enable_overlap_clearance=False, enable_visibility_cleanup=False)
    for m in (on, off):
        m.input_pointcloud(pts, ["x", "y", "z"], R, t, position_noise, orientation_noise)
    pts_m = on.counts[1] > 0                                      # cnt_all: valid, inside points
    rays_m = np.zeros_like(pts_m)
    if p.enable_visibility_cleanup:
        for li in (0, 1, 2, 5, 6):
            a, b = on.elevation_map[li], off.elevation_map[li]
            rays_m |= ~((a == b) | (np.isnan(a) & np.isnan(b)))
    win = np.zeros_like(pts_m)
    if p.enable_overlap_clearance:
        lo, hi = om.cell_min, om.cell_max
        win[lo:hi, lo:hi] = True
    return pts_m, rays_m, win


def group_counts(pts_m, rays_m, win):
    both = pts_m & rays_m
    return {"points_only": int((pts_m & ~rays_m).sum()), "rays_only": int((rays_m & ~pts_m).sum()),
            "both": int(both.sum()), "overlap_only": int((win & ~pts_m & ~rays_m).sum()),
            "full_path": int((pts_m | rays_m | win).sum())}


def _sectors(mask, elem):
    idx = np.flatnonzero(mask.ravel())
    return int(np.unique(idx * elem // SECTOR).size)


def load_traffic(pts_m, rays_m, win, rays_ran=True):
    """Loads, requested bytes and distinct 32-byte sectors of k_finalize's full path, parent layout and now"""
    full = pts_m | rays_m | win
    before = MAP_LOADS + PTS_LOADS + (RAY_LOADS if rays_ran else [])
    out = {}
    for name, groups in (("parent", [(full, before)]),
                         ("now", [(full, MAP_LOADS), (pts_m, PTS_LOADS_NOW), (rays_m if rays_ran else rays_m & False, RAY_LOADS)])):
        loads = sum(int(m.sum()) * len(L) for m, L in groups)
        req = sum(int(m.sum()) * sum(e for _, e in L) for m, L in groups)
        sec = sum(_sectors(m, e) for m, L in groups for _, e in L)
        out[name] = {"loads": loads, "bytes": req, "sectors": sec, "sector_bytes": sec * SECTOR}
    return out


# ---- frame sequences in which each group occurs on its own --------------------------------------------------------
def _flat_state(W, seed, valid_frac=0.3, height_sd=1.0):
    """valid cells of random height (old enough for rays to act: time 1), the rest invalid; normals straight up so
    that steep rays pass the incidence test"""
    rng = np.random.default_rng(seed)
    st = np.zeros((7, W, W), np.float32)
    st[2] = rng.random((W, W)) < valid_frac
    st[0] = (rng.standard_normal((W, W)) * height_sd).astype(np.float32) * st[2]
    st[1] = 0.05; st[3] = 1.0; st[4] = 1.0
    normal = np.zeros((3, W, W), np.float32)
    normal[2] = 1.0
    return st, normal


def _ground(rng, n, half, z_sensor, keep=None):
    xy = rng.uniform(-half, half, (4 * n, 2))
    if keep is not None:
        xy = xy[keep(xy)]
    xy = xy[:n]
    z = rng.normal(0.0, 0.02, len(xy)) - z_sensor
    return np.concatenate([xy, z[:, None]], 1).astype(np.float32)


def scenario(name, W):
    """(parameter overrides, (state, normal) or None, frames [(points in the sensor frame, R, t)]) of one sequence"""
    from elevation_mapping_cupy_b200 import workloads as wl
    res = 0.04
    half = 0.45 * (W - 2) * res
    R = np.eye(3, dtype=np.float32)
    rng = np.random.default_rng(1000 + W)
    if name == "short_rays":
        # rays end 1.5 m out: the far LiDAR returns are cells with points and no ray effects
        frames = [wl.lidar_cloud(0, f, n_rings=32, n_az=800, max_range=min(20.0, half)) for f in range(3)]
        return dict(max_ray_length=1.5), None, frames
    if name == "high_sensor":
        # sensor 6 m above a flat floor, 400 points: the rays cross cells no point lands in, carving the invalid ones
        # and decrementing the valid ones that stand above them
        frames = []
        for f in range(3):
            t = np.array([0.04 * f, -0.04 * f, 6.0], np.float32)
            frames.append((_ground(rng, 400, half, 6.0), R, t))
        return dict(max_ray_length=20.0), _flat_state(W, W), frames
    if name == "overlap_window_apart":
        # no point inside the overlap-clear window (4 m square around the centre): its cells are finalised for the
        # clear alone, or for the rays that cross it
        keep = lambda xy: np.maximum(np.abs(xy[:, 0]), np.abs(xy[:, 1])) > 2.3        # noqa: E731
        frames = []
        for f in range(3):
            t = np.array([0.0, 0.0, 1.5], np.float32)
            frames.append((_ground(rng, 3000, half, 1.5, keep), R, t))
        return dict(overlap_clear_range_xy=4.0), _flat_state(W, W + 1, valid_frac=0.2, height_sd=0.3), frames
    if name == "rays_then_none":
        # frames with rays, then a frame with no valid point (no ray at all, nothing fused), then rays again
        frames = []
        for f in range(5):
            t = np.array([0.0, 0.0, 3.0], np.float32)
            if f == 2:
                pts = np.zeros((0, 3), np.float32)
            elif f == 3:
                pts = (rng.standard_normal((500, 3)) * 0.05).astype(np.float32)     # inside min_valid_distance
            else:
                pts = _ground(rng, 1500, half, 3.0)
            frames.append((pts, R, t))
        return dict(), _flat_state(W, W + 2), frames
    raise KeyError(name)


SCENARIOS = ["short_rays", "high_sensor", "overlap_window_apart", "rays_then_none"]
# the group each sequence exists for: it must occur in at least one frame
SCENARIO_GROUP = {"short_rays": "points_only", "high_sensor": "rays_only", "overlap_window_apart": "overlap_only",
                  "rays_then_none": "rays_only"}
