"""The cases of the frame-variant tests and the oracles that check the ray box against march samples.

The host picks kernel variants and shared-memory layouts from cell_n, resolution, max_ray_length, dilation_size, the
sensor poses and the input buffer (make_plan, ray_box and raycast_runs in elevation_mapping_cupy_b200/csrc/emap_plan.cuh,
called through tests/plan_host.py).  tests/test_frame_variants_cpu.py checks that every side of each choice has a case
below, and that the ray box holds the march samples computed here independently of the engine.
"""
import numpy as np

import plan_host

CORE_RES, CORE_RAY = 0.04, 10.0       # resolution and max_ray_length of core_parameter()


def h16(x):
    """fp32 -> fp16 (round to nearest even) -> value, as a Python float."""
    return float(np.float16(np.float32(x)))


# ---- the ray box ----------------------------------------------------------------------------------------------------
def box_empty(box):
    return box[1] <= box[0] or box[3] <= box[2]


def t8_address(plan, box, ix, iy):
    """k_raycast: the shared-memory byte address of the fine-tile maximum k_raycast<false> reads for cell (ix, iy)"""
    _, _, _, _, ts, ta, tb = box
    RT = plan_host.constants()["RT"]
    return plan["off_t8"] + 4 * (((np.asarray(ix) >> ts) - ta) * RT + ((np.asarray(iy) >> ts) - tb))


# ---- rays and march samples -----------------------------------------------------------------------------------------
def rays_of(t_rel, points, max_ray_length):
    """emap_oracle.c:518-524 (ray_vector, CK.py:83-101,199-201) for end points given in the map frame relative to the map
    centre: (rx, ry, rz, len) per point, fp16 values held in fp32."""
    f16 = lambda a: np.asarray(a, np.float32).astype(np.float16).astype(np.float32)
    t16 = f16(np.asarray(t_rel, np.float32))
    P = np.asarray(points, np.float32)
    v = f16(f16(P) - t16)
    norm = f16(np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(norm[:, None] > 0, f16(v / norm[:, None]), np.float32(0))
    length = np.minimum(norm, np.float32(h16(max_ray_length)))
    return r[:, 0], r[:, 1], r[:, 2], length


def march_cells(W, res, steps, t_rel, rx, ry, length):
    """emap_oracle.c:527-530: the cell (ix, iy) of every march sample s_k < len of each ray, as (n_rays, n_steps) arrays,
    and the mask of the samples that exist.  Sample coordinates are fp32 t + r*s (the product of two fp16 values is exact),
    rounded to fp16 and mapped to cells by the exact double expression of CK.py:22-33."""
    s = np.asarray(steps, np.float32)[None, :]
    t = np.asarray(t_rel, np.float32)
    live = s < np.asarray(length, np.float32)[:, None]

    def axis(tc, r):
        c = (np.float32(tc) + np.asarray(r, np.float32)[:, None] * s).astype(np.float32)
        c16 = c.astype(np.float16).astype(np.float64)
        return np.clip(np.trunc(c16 / res + 0.5 * W), 0, W - 1).astype(np.int64)
    return axis(t[0], rx), axis(t[1], ry), live


def address_samples(W, ix, iy, live):
    """The samples at which k_raycast forms a fine-tile address: a cell different from the previous sample's
    (k_raycast; before the first sample lane 0 supplies cell (0, 0), the NaN entry [0] of the march table)."""
    nidx = ix * W + iy
    prev = np.concatenate([np.zeros((nidx.shape[0], 1), np.int64), nidx[:, :-1]], 1)
    return live & (nidx != prev)


# ---- the cases ------------------------------------------------------------------------------------------------------
# A: resolution, ray length and map size.  Each runs LiDAR or uniform frames with move_to / update_variance / update_time.
RES_CASES = [
    dict(id="res0.02-256", cell_n=256, kw=dict(resolution=0.02)),
    dict(id="res0.05-202", cell_n=202, kw=dict(resolution=0.05)),
    dict(id="res0.1-2048", cell_n=2048, kw=dict(resolution=0.1)),
    dict(id="res0.2-130", cell_n=130, kw=dict(resolution=0.2)),
    dict(id="ray0.5-1024", cell_n=1024, kw=dict(max_ray_length=0.5)),
    dict(id="ray40-1024", cell_n=1024, kw=dict(max_ray_length=40.0)),
    dict(id="odd-2049", cell_n=2049, kw=dict()),
]

# B: every dilation on both k_post paths, random state with populated border columns
POST_SIZES = [8, 9, 48, 64, 130, 256, 260]
POST_KS = list(range(9))
POST_CASES = [(W, K) for W in POST_SIZES for K in POST_KS]

# C: sensor poses without move_to (map centre at the origin), core parameters.  Positions are given in cells from the
# map centre, in metres.


def pose_cases(W):
    """(id, [sensor positions t (x, y, z)]) of the sensor-pose group for a W x W map at the core resolution"""
    res, L = CORE_RES, CORE_RAY
    half = 0.5 * W * res                      # the map's edge, relative to its centre
    cell = res
    inside = half - 1.5 * cell                # centre of the cell one inside the border ring
    ring = half - 0.5 * cell                  # centre of the border-ring cell
    near, far = half + 0.5 * L, half + 1.5 * L
    return [
        ("in-x+", [(inside, 0.3, 1.0)]),
        ("in-x-", [(-inside, -0.2, 1.0)]),
        ("in-y+", [(0.1, inside, 1.0)]),
        ("in-y-", [(-0.4, -inside, 1.0)]),
        ("ring", [(ring, 0.5 * half, 1.0)]),
        ("beyond-near", [(near, -0.25 * half, 1.0)]),
        ("beyond-far-rows", [(far, 0.2, 1.0)]),
        ("beyond-far-cols", [(0.2, -far, 1.0)]),
        ("beyond-far-both", [(-far, far, 1.0)]),
        ("two-sensors", [(0.3 * half, -0.2 * half, 1.0), (-far, -far, 1.0)]),
        ("below-terrain", [(0.1 * half, 0.2 * half, -1.0)]),
    ]


POSE_SIZES = [256, 2048]

# D: input layouts of the same three frames, each on its own handle
LAYOUTS = ["f32-host", "f32x4-device", "f32x4-device-unaligned", "f32-pinned", "f64-pinned", "f64-device-strided"]


def layout_path(layout):
    """(where the index pass reads the rows, whether it takes the 16-byte vector load) of a layout:
    FrameInput::stage (staged copy, zero-copy, device; emap_api.cu) and load_point<float> (emap_sources.cuh)"""
    where = {"f32-host": "staged", "f32-pinned": "zero-copy", "f64-pinned": "zero-copy"}.get(layout, "device")
    return where, layout == "f32x4-device"


MANY_SENSORS = 70     # more than 64 sensors in one frame


def frame_params(case):
    """(cell_n, resolution, max_ray_length) of a group A case"""
    kw = case["kw"]
    return case["cell_n"], kw.get("resolution", CORE_RES), kw.get("max_ray_length", CORE_RAY)
