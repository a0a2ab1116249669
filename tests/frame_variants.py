"""The host-side decisions of a frame, restated in NumPy, and the cases of the frame-variant tests.

The host picks kernel variants and shared-memory layouts from cell_n, resolution, max_ray_length, dilation_size, the
sensor poses and the input buffer (elevation_mapping_cupy_b200/csrc/emap_api.cu).  Each function below restates one of
those choices and cites the lines it restates, so that the tests can say which side of every choice a case is on
(tests/test_frame_variants_cpu.py checks that each side has a case) and can check the ray box against march samples
computed independently of the engine.
"""
import math

import numpy as np

RT = 64               # fine tiles per axis of the coarse ray maps (emap_kernels.cuh RT)
RC_STRIDE = 31        # new march steps per warp iteration (emap_kernels.cuh RC_STRIDE)
PT_X, PT_Y = 32, 16   # k_post tile (emap_kernels.cuh PT_X, PT_Y)
CORE_RES, CORE_RAY = 0.04, 10.0       # resolution and max_ray_length of core_parameter()


def h16(x):
    """fp32 -> fp16 (round to nearest even) -> value, as a Python float."""
    return float(np.float16(np.float32(x)))


def _h16_up(x):
    """__float2half_ru of an fp32 value."""
    x = np.float32(x)
    h = np.float16(x)
    if np.float32(h) < x:
        h = np.nextafter(h, np.float16(np.inf))
    return h


# ---- k_post ---------------------------------------------------------------------------------------------------------
def post_tma(W, K):
    """emap_api.cu:616-618 make_post_tm: k_post stages its tiles with TMA tensor copies when the row pitch is a multiple of
    16 bytes and the map holds one staged box; plain loads otherwise."""
    HL = K + 3
    HLX = (HL + 3) & ~3
    return W % 4 == 0 and W >= PT_X + 2 * HLX and W >= PT_Y + 2 * HL


def post_instance(K):
    """emap_api.cu:635-640 launch_post: the k_post<K> instantiation (0 = dilation read at run time)."""
    return K if K in (1, 2, 3) else 0


def record_v(W):
    """emap_api.cu:559 and 647-648: cells per thread of k_record and k_finalize (and the ray box's column alignment)."""
    return 4 if W % 4 == 0 else 1


# ---- ray-march tables and the k_raycast shared-memory layout ----------------------------------------------------------
def max_len16(max_ray_length):
    """emap_api.cu:227 fill_devcfg max_len16"""
    return h16(max_ray_length)


def lut_p2(W, res):
    """emap_api.cu:232-241 fill_devcfg: bytes of one half of the staged cell table (fp16 patterns [0, LIM])."""
    want = (0.5 * W + 1.0) * res
    bits = int(np.array(_h16_up(min(want, 60000.0))).view(np.uint16))
    bits = min(bits, 0x7BFF)
    return ((bits + 1) * 2 + 15) & ~15


def march_steps(res, max_ray_length):
    """emap_api.cu:244-255 build_steps: the fp16 march variable s_k < max_len16 (CK.py:203,268)."""
    step = res / math.sqrt(2.0)
    L = max_len16(max_ray_length)
    out = []
    s = h16(step)
    while s < L and len(out) < 65535:
        out.append(s)
        nx = h16(s + step)
        if not nx > s:
            break
        s = nx
    return np.array(out, np.float32)


def n_steps(res, max_ray_length):
    return len(march_steps(res, max_ray_length))


def n_tab(n):
    """emap_api.cu:889: floats of the march table as k_raycast stages it"""
    return (((n + RC_STRIDE - 1) // RC_STRIDE) * RC_STRIDE + 64) & ~1


def span_cells(res, max_ray_length):
    """emap_api.cu:918-926: cells per axis one 31-step warp iteration of the march can span"""
    st = march_steps(res, max_ray_length).astype(np.float64)
    span = 0.0
    for k in range(len(st) - 1):
        e = min(len(st) - 1, k + RC_STRIDE - 1)
        span = max(span, (st[e] - st[k]) / res)
    return int(math.ceil(span)) + 2


def rc_layout(W, res, max_ray_length):
    """emap_api.cu:927-938 emap_create: byte offsets of k_raycast's shared-memory regions.  The coarse maps and the march
    table sit in the gap between the two halves of the cell table when they fit there ("gap"), else behind the second
    half ("behind")."""
    P2 = lut_p2(W, res)
    need = 4 * (RT * RT + (RT // 2) * (RT // 2) + n_tab(n_steps(res, max_ray_length))) + 16
    base, end = (P2 + 15) & ~15, 65536 + P2
    where = "gap"
    if base + need > 65536:
        base = (end + 15) & ~15
        end = base + need
        where = "behind"
    return dict(where=where, p2=P2, off_t8=base, off_t16=base + 4 * RT * RT,
                off_steps=base + 4 * (RT * RT + (RT // 2) * (RT // 2)), rc_smem=end)


# ---- the ray box ----------------------------------------------------------------------------------------------------
def ray_grid(W, res, max_ray_length, t_rel):
    """emap_api.cu:509-544 ray_grid: (r0, r1, c0, c1, ts, ta, tb), the box of cells the rays of a frame can reach and its
    tiling.  t_rel: the sensors' positions relative to the map centre (fp32, as emap_api.cu:393 computes them)."""
    align = record_v(W)
    L = float(np.float32(max_len16(max_ray_length)))
    half_w = 0.5 * W
    r0, r1, c0, c1 = W, 0, W, 0
    for t in t_rel:
        for ax in range(2):
            tc = float(np.float32(t[ax]))
            e = (abs(tc) + L) * (1.0 / 2048.0) + 1e-4
            lo = math.floor((tc - L - e) / res + half_w) - 2.0
            hi = math.floor((tc + L + e) / res + half_w) + 3.0
            a, b = int(min(max(lo, 0.0), W)), int(min(max(hi, 0.0), W))
            if ax == 0:
                r0, r1 = min(r0, a), max(r1, b)
            else:
                c0, c1 = min(c0, a), max(c1, b)
    if r1 <= r0 or c1 <= c0:
        return (0, 0, 0, 0, 3, 0, 0)
    c0 = (c0 // align) * align
    c1 = min(W, ((c1 + align - 1) // align) * align)
    sp = span_cells(res, max_ray_length)
    ts = 2
    while True:
        al = 2 << ts
        r0a, c0a = (r0 // al) * al, (c0 // al) * al
        if (RT << ts) >= max(r1 - r0a, c1 - c0a) and (4 << ts) >= sp + 1:
            return (r0, r1, c0, c1, ts, r0a >> ts, c0a >> ts)
        ts += 1


def box_empty(box):
    return box[1] <= box[0] or box[3] <= box[2]


def raycast_launched(box, n_rays, n_steps_, count_rays=False):
    """emap_api.cu:568-574 frame_rays: whether k_raycast runs for a sensor.  The counting variant (emap_set_ray_counting) reads no
    coarse map and runs for every sensor with rays; the march itself only where the box holds a cell."""
    if n_rays <= 0 or n_steps_ == 0:
        return False
    return count_rays or not box_empty(box)


def t8_address(layout, box, ix, iy):
    """emap_kernels.cuh:596,670: the shared-memory byte address of the fine-tile maximum k_raycast<false> reads for cell
    (ix, iy)"""
    _, _, _, _, ts, ta, tb = box
    return layout["off_t8"] + 4 * (((np.asarray(ix) >> ts) - ta) * RT + ((np.asarray(iy) >> ts) - tb))


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
    length = np.minimum(norm, np.float32(max_len16(max_ray_length)))
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
    (emap_kernels.cuh:662-665; before the first sample lane 0 supplies cell (0, 0), emap_api.cu:902)."""
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
    emap_api.cu:404-437 frame_begin (staged copy, zero-copy, device) and emap_kernels.cuh:146-154 load_point<float>"""
    where = {"f32-host": "staged", "f32-pinned": "zero-copy", "f64-pinned": "zero-copy"}.get(layout, "device")
    return where, layout == "f32x4-device"


MANY_SENSORS = 70     # more than the 64 sensor pointers frame_begin keeps on the stack (emap_api.cu:400-403)


def frame_params(case):
    """(cell_n, resolution, max_ray_length) of a group A case"""
    kw = case["kw"]
    return case["cell_n"], kw.get("resolution", CORE_RES), kw.get("max_ray_length", CORE_RAY)
