"""Sharded frames of semantic clouds and depth cameras: every replica must equal a single-GPU twin that fuses all ranks'
inputs, bit for bit (state, normals, semantic layers, variance planes), through ShardedElevationMap (NCCL and multicast)
and through the C ABI's own NCCL path; and the refusals of sharded begins.  World size 1 runs on one GPU and goes
through the whole sharded path; world size 2 needs two GPUs."""
import os
import signal
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_COMMON = r"""
import os, sys, time, ctypes as C
sys.path.insert(0, %(root)r)
import numpy as np, torch
rk = int(os.environ["RANK"]); ws = int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rk)
from elevation_mapping_cupy_b200.parameter import core_parameter
from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
from elevation_mapping_cupy_b200 import workloads as wl, _lib
FUSIONS = {"rgb": "color", "avg": "average", "cls": "class_average", "cb.*": "class_bayesian",
           "bi": "bayesian_inference", "cm": "class_max", "default": "class_average"}
CLOUD_CH = ["x", "y", "z", "avg", "cls", "rgb", "cb0", "cb1", "bi"]
DEPTH_CH = ["rgb", "f0", "f1"]

def make_map():
    p = core_parameter(256)
    p.pointcloud_channel_fusions = dict(FUSIONS)
    return ElevationMap(p, device=rk)

def semantic_cloud(f, s):
    pts, R, t = wl.lidar_cloud(2, f, n_rings=16, n_az=500 + 37 * s, max_range=6.0, sensor=s, n_sensors=2)
    rng = np.random.default_rng(1000 * f + s)
    n = len(pts)
    rgb = (rng.integers(0, 256, (n, 3)).astype(np.uint32) * np.array([1 << 16, 1 << 8, 1], np.uint32)).sum(1)
    cols = [rng.normal(0.0, 1.0, n), rng.random(n), rgb.astype(np.uint32).view(np.float32),
            rng.normal(0.2, 0.5, n), rng.normal(0.2, 0.5, n), rng.normal(1.0, 0.3, n)]
    extra = np.stack([c.astype(np.float32) if c.dtype != np.float32 else c for c in cols], 1)
    return np.ascontiguousarray(np.concatenate([pts, extra], 1), np.float32), R, t

def camera(f, s, on_device):
    depth, P, R, t = wl.depth_image(f, width=160, height=120, sensor=s)
    rng = np.random.default_rng(77 + 10 * f + s)
    cam = dict(depth=depth, P=P, R=R, t=t, rgb=rng.integers(0, 256, (120, 160, 3)).astype(np.uint8),
               features=rng.normal(0.0, 1.0, (2, 120, 160)).astype(np.float32))
    if s == 1:
        cam["confidence"] = rng.uniform(0.0, 20.0, (120, 160)).astype(np.float32)
    if on_device:
        cam = {k: (torch.from_numpy(np.ascontiguousarray(v)).cuda() if k in ("depth", "rgb", "features", "confidence") else v)
               for k, v in cam.items()}
    return cam

def bits(x):
    x = x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)
    return np.ascontiguousarray(x).view(np.uint32)

def assert_same(em, twin, what):
    torch.cuda.synchronize()
    s1, n1 = em.get_state(); s2, n2 = twin.get_state()
    for li in range(7):
        assert np.array_equal(bits(s1[li]), bits(s2[li])), (what, "layer", li)
    assert np.array_equal(bits(n1), bits(n2)), (what, "normals")
    a, b = em.semantic_map, twin.semantic_map
    assert a.layer_names == b.layer_names, (what, a.layer_names, b.layer_names)
    assert np.array_equal(bits(a.semantic_map), bits(b.semantic_map)), (what, "semantic layers")
    assert (a.variance is None) == (b.variance is None), what
    if a.variance is not None:
        assert np.array_equal(bits(a.variance), bits(b.variance)), (what, "variance planes")

def my_share(n):
    # items of a frame split over the ranks: 2 + 1 at world size 2, all of them at world size 1
    return list(range(n)) if ws == 1 else ([0, 1] if rk == 0 else [2]) if n == 3 else [s for s in range(n) if s %% ws == rk]
"""

_WORKER = _COMMON + r"""
import torch.distributed as dist
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{rk}"))
from elevation_mapping_cupy_b200.sharded import ShardedElevationMap
em = make_map(); twin = make_map()
sh = ShardedElevationMap(em, mode=os.environ["EMAP_SHARD_MODE"])
print("mode", sh.mode, flush=True)
# clouds: every kind 0..4, two sensors
for f in range(3):
    items = [semantic_cloud(f, s) for s in range(2)]
    R0, t0 = items[0][1], items[0][2]
    em.move_to(t0, R0); twin.move_to(t0, R0)
    mine = my_share(2)
    sh.input_sensors([items[s][0] for s in mine], [items[s][1] for s in mine], [items[s][2] for s in mine], 0.02, 0.02,
                     overlap_z=float(t0[2]), channels=CLOUD_CH)
    twin._configure_cloud_channels(CLOUD_CH)
    twin.input_sensors([c for c, _, _ in items], [R for _, R, _ in items], [t for _, _, t in items], 0.02, 0.02)
    assert_same(em, twin, ("cloud", f))
    em.update_time(); twin.update_time()
# depth: three cameras, rgb + two feature channels, one with confidence; host images, then device images
for f in range(3):
    cams = [camera(f, s, on_device=(f == 1)) for s in range(3)]
    em.move_to(cams[0]["t"], cams[0]["R"]); twin.move_to(cams[0]["t"], cams[0]["R"])
    mine = my_share(3)
    sh.input_depth_images([cams[s] for s in mine], 0.02, 0.02, channels=DEPTH_CH)
    twin.input_depth_images(cams, 0.02, 0.02, channels=DEPTH_CH)
    assert_same(em, twin, ("depth", f))
    px = [c["depth"].shape[0] * c["depth"].shape[1] for c in cams]
    off = sum(px[s] for s in range(3) if s < mine[0])
    n = sum(px[s] for s in mine)
    rec = em.get_point_record(n); full = twin.get_point_record(sum(px))
    for a, b in zip(rec, full):
        assert np.array_equal(a, b[off:off + n]), ("point record", f)
    em.update_time(); twin.update_time()
dist.barrier()
print("SHARDED_SENSORS_OK", rk, flush=True)
dist.destroy_process_group()
"""

_WORKER_C = _COMMON + r"""
# no torch.distributed: the communicator comes from the C ABI (emap_comm_unique_id / emap_comm_init)
L = _lib.load()
idfile = %(idfile)r
buf = (C.c_char * 128)()
if rk == 0:
    assert L.emap_comm_unique_id(buf) == 0
    open(idfile + ".tmp", "wb").write(bytes(buf)); os.rename(idfile + ".tmp", idfile)
else:
    for _ in range(600):
        if os.path.exists(idfile): break
        time.sleep(0.1)
    buf = (C.c_char * 128).from_buffer_copy(open(idfile, "rb").read())
em = make_map(); twin = make_map()
em._check(L.emap_comm_init(em._h, buf, rk, ws))
for f in range(3):
    items = [semantic_cloud(f, s) for s in range(2)]
    R0, t0 = items[0][1], items[0][2]
    em.move_to(t0, R0); twin.move_to(t0, R0)
    mine = my_share(2)
    clouds = [items[s][0] for s in mine]
    ptrs = (C.c_void_p * len(clouds))(*[c.ctypes.data for c in clouds])
    cnt = (C.c_int64 * len(clouds))(*[len(c) for c in clouds])
    Rm = np.ascontiguousarray(np.stack([items[s][1] for s in mine]), np.float32)
    tm = np.ascontiguousarray(np.stack([items[s][2] for s in mine]), np.float32)
    off = sum(len(items[s][0]) for s in range(mine[0]))
    em._configure_cloud_channels(CLOUD_CH)
    em._check(L.emap_input_sensors_sharded(em._h, len(clouds), ptrs, cnt, clouds[0].shape[1], 0, 0, Rm.ctypes.data,
                                           tm.ctypes.data, off, float(t0[2]), 0.02, 0.02))
    twin._configure_cloud_channels(CLOUD_CH)
    twin.input_sensors([c for c, _, _ in items], [R for _, R, _ in items], [t for _, _, t in items], 0.02, 0.02)
    assert_same(em, twin, ("C cloud", f))
for f in range(2):
    cams = [camera(f, s, on_device=(f == 1)) for s in range(3)]
    em.move_to(cams[0]["t"], cams[0]["R"]); twin.move_to(cams[0]["t"], cams[0]["R"])
    mine = my_share(3)
    depth = em._depth_frame([cams[s] for s in mine], DEPTH_CH)
    px = [c["depth"].shape[0] * c["depth"].shape[1] for c in cams]
    off = sum(px[s] for s in range(mine[0]))
    torch.cuda.synchronize()
    em._check(L.emap_input_depth_images_sharded(em._h, *depth.args, 10.0, 8.0, off, float(cams[0]["t"][2]), 0.02, 0.02))
    twin.input_depth_images(cams, 0.02, 0.02, channels=DEPTH_CH)
    assert_same(em, twin, ("C depth", f))
print("C_SHARDED_SENSORS_OK", rk, flush=True)
em.close(); twin.close()
"""

_WORKER_REFUSE = _COMMON + r"""
import torch.distributed as dist
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{rk}"))
from elevation_mapping_cupy_b200.sharded import ShardedElevationMap
L = _lib.load()
INVALID, STATE = -1, -4
em = make_map()
sh = ShardedElevationMap(em, mode=os.environ["EMAP_SHARD_MODE"])
h = em._h
cloud, R, t = semantic_cloud(0, 0)
ptrs = (C.c_void_p * 1)(cloud.ctypes.data); cnt = (C.c_int64 * 1)(len(cloud))
Rm = np.ascontiguousarray(R, np.float32).reshape(9); tm = np.ascontiguousarray(t, np.float32)
def begin():
    return L.emap_shard_begin(h, 1, ptrs, cnt, cloud.shape[1], 0, 0, Rm.ctypes.data, tm.ctypes.data, 0, 0.02, 0.02)
def frozen(call, code, text):
    torch.cuda.synchronize()
    before, launches = em.get_state()[0].copy(), L.emap_launch_count(h)
    assert call() == code, (text, L.emap_last_error(h))
    assert text in L.emap_last_error(h).decode(), L.emap_last_error(h)
    assert L.emap_launch_count(h) == launches, text
    assert np.array_equal(bits(em.get_state()[0]), bits(before)), text

sh.input_sensors([cloud], [R], [t], 0.02, 0.02, channels=CLOUD_CH)          # a map to keep unchanged
# a class_max channel: refused by every sharded begin, nothing queued
em._configure_cloud_channels(CLOUD_CH + ["cm"])
frozen(begin, INVALID, "class_max")
cam = camera(0, 0, False)
depth = em._depth_frame([cam], DEPTH_CH + ["cm"])
frozen(lambda: L.emap_shard_begin_depth_images(h, *depth.args, 10.0, 8.0, 0, 0.02, 0.02), INVALID, "class_max")
try:
    sh.input_sensors([cloud], [R], [t], 0.02, 0.02, channels=CLOUD_CH + ["cm"])
    raise AssertionError("class_max accepted")
except _lib.EmapError as e:
    assert "class_max" in str(e)
# the depth argument checks, through the sharded depth begin
depth = em._depth_frame([cam], DEPTH_CH)
args = list(depth.args)
frozen(lambda: L.emap_shard_begin_depth_images(h, 0, *args[1:], 10.0, 8.0, 0, 0.02, 0.02), INVALID,
       "emap_shard_begin_depth_images: 1 <= n_cameras")
bad_src = (C.c_int32 * 3)(-1, -1, 0)
frozen(lambda: L.emap_shard_begin_depth_images(h, args[0], args[1], args[2], 3, bad_src, args[5], 10.0, 8.0, 0, 0.02, 0.02),
       INVALID, "more than one colour channel")
frozen(lambda: L.emap_shard_begin_depth_images(h, *args, 10.0, 8.0, (1 << 31) - 100, 0.02, 0.02), INVALID, "2^31")
zero = (_lib.EmapDepthCamera * 1)(); C.memmove(zero, args[1], C.sizeof(_lib.EmapDepthCamera)); zero[0].fx = 0.0
frozen(lambda: L.emap_shard_begin_depth_images(h, args[0], zero, *args[2:], 10.0, 8.0, 0, 0.02, 0.02), INVALID,
       "zero fx")
if sh.mode == "nccl":
    # exchange 2 lists the semantic sums: a capacity below their count is refused with the count needed
    em._configure_cloud_channels(CLOUD_CH)
    assert begin() == 0, L.emap_last_error(h)
    arr = (_lib.EmapExchange * 5)(); n = C.c_int32(5)
    assert L.emap_shard_exchange(h, 1, arr, C.byref(n)) == 0 and n.value == 2
    assert L.emap_shard_phase(h, 1) == 0
    n = C.c_int32(3)
    assert L.emap_shard_exchange(h, 2, arr, C.byref(n)) == INVALID and n.value == 5, n.value
    assert "capacity" in L.emap_last_error(h).decode()
    n = C.c_int32(5)
    assert L.emap_shard_exchange(h, 2, arr, C.byref(n)) == 0 and n.value == 5
    assert [arr[k].kind for k in range(5)] == [0, 3, 1, 0, 3]
    cells = em.cell_n * em.cell_n
    assert arr[3].count == 5 * cells and arr[4].count == 4 * cells     # avg, cls, cb0, cb1, bi; one colour channel
    assert L.emap_shard_phase(h, 2) == 0         # one rank: the all-reduces would leave the arrays as they are
    n = C.c_int32(5)
    assert L.emap_shard_exchange(h, 3, arr, C.byref(n)) == 0
    assert L.emap_shard_phase(h, 3) == 0
    # without channels the lists are exactly the plain ones
    em._configure_cloud_channels(["x", "y", "z"])
    sh.input_sensors([cloud[:, :3].copy()], [R], [t], 0.02, 0.02)
else:
    # a configuration that outgrows the attached block: the begin refuses it, the map re-attaches a larger block
    small = int(L.emap_shard_scratch_bytes(h))
    em._configure_cloud_channels(CLOUD_CH + ["avg2"])
    assert int(L.emap_shard_scratch_bytes(h)) > small
    frozen(begin, STATE, "emap_shard_scratch_bytes()")
    wider = np.ascontiguousarray(np.concatenate([cloud, cloud[:, 3:4]], 1))
    sh.input_sensors([wider], [R], [t], 0.02, 0.02, channels=CLOUD_CH + ["avg2"])    # re-attaches a larger block
    assert sh._symm[2] == int(L.emap_shard_scratch_bytes(h)) > small
torch.cuda.synchronize()
dist.barrier()
print("REFUSALS_OK", rk, flush=True)
dist.destroy_process_group()
"""


def _run(script, nproc, port, timeout, env=None):
    """Runs `script` under torch.distributed.run with nproc workers in a session of its own; kills the whole session on
    a timeout or when the run fails.  Returns the combined output."""
    p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True,
                         env=dict(os.environ, **(env or {})))
    try:
        out = p.communicate(timeout=timeout)[0]
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        out = p.communicate()[0] + "\n[timed out]"
    if p.returncode:
        try:
            os.killpg(p.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
    return out


def _need(ws):
    import torch
    if torch.cuda.device_count() < ws:
        pytest.skip(f"needs {ws} GPUs")


def _skip_without_multicast(mode, out):
    if mode == "multicast" and "multicast is not available" in out:
        pytest.skip("fabric has no NVLink multicast")


@pytest.mark.parametrize("ws", [1, 2])
@pytest.mark.parametrize("mode", ["nccl", "multicast"])
def test_sharded_semantic_clouds_and_depth_cameras_match_the_single_gpu_frame(tmp_path, mode, ws):
    _need(ws)
    script = tmp_path / "w.py"
    script.write_text(_WORKER % {"root": ROOT})
    out = _run(script, ws, 29611 + 2 * ws + (mode == "multicast"), 900, {"EMAP_SHARD_MODE": mode})
    _skip_without_multicast(mode, out)
    assert all(f"SHARDED_SENSORS_OK {r}" in out for r in range(ws)), out[-6000:]


@pytest.mark.parametrize("ws", [1, 2])
def test_sharded_semantic_frames_through_the_c_abi(tmp_path, ws):
    _need(ws)
    script = tmp_path / "wc.py"
    script.write_text(_WORKER_C % {"root": ROOT, "idfile": str(tmp_path / "nccl_id.bin")})
    out = _run(script, ws, 29631 + ws, 900)
    assert all(f"C_SHARDED_SENSORS_OK {r}" in out for r in range(ws)), out[-6000:]


@pytest.mark.parametrize("mode", ["nccl", "multicast"])
def test_sharded_begins_refuse_what_they_cannot_fuse(tmp_path, mode):
    _need(1)
    script = tmp_path / "wr.py"
    script.write_text(_WORKER_REFUSE % {"root": ROOT})
    out = _run(script, 1, 29641 + (mode == "multicast"), 600, {"EMAP_SHARD_MODE": mode})
    _skip_without_multicast(mode, out)
    assert "REFUSALS_OK 0" in out, out[-6000:]
