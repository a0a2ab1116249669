"""Generates tests/golden/*.npz.  Run HERE (needs /root/reference): the "ref_*" arrays come from the
REFERENCE'S OWN kernel source (custom_kernels.py strings compiled for the host by oracle/build_ref.py and
driven in the order of elevation_mapping.py:316-391); the "oracle_*" arrays from oracle/emap_oracle.c.

    python tests/golden/make_golden.py          # host build of the reference source
    python tests/golden/make_golden.py --gpu    # ref_gpu_index.json: the reference's kernels on the GPU

Inputs are regenerated from seeds by elevation_mapping_cupy_b200/workloads.py, so only outputs are stored.
The reference kernel is racy (SURVEY 3.5); `racy` marks the cells whose outcome differs between executing the
points in input order, in reverse order and in a fixed random order -- parity is asserted outside that mask.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from elevation_mapping_cupy_b200 import workloads as wl          # noqa: E402
from elevation_mapping_cupy_b200.parameter import Parameter, core_parameter   # noqa: E402
from oracle import oracle as O                                   # noqa: E402
sys.path.insert(0, os.path.dirname(HERE))
from helpers import (FLAG_CASES, STAR_R, dilation_inputs, drift_frames, semantic_inputs,  # noqa: E402
                     star_inputs)


def index_case(seed):
    """reference test shape (test_elevation_mapping.py:51-61), default parameters, 202^2 map"""
    p = Parameter(); p.update()
    pts, R, t = wl.reference_test_cloud(seed, n=20000)
    if seed % 2:
        pts = (pts * np.float32(9.0) - np.float32(4.5)).astype(np.float32)
    rm = O.RefKernelMap(p, "default202")
    rm.input_pointcloud(pts.copy(), ["x", "y", "z"], R, t, 0, 0)
    idx, valid, inside = rm.last_point_record
    return dict(idx=idx, valid=valid, inside=inside)


def frames_case(cell_n=130, n_frames=4, tag="core130"):
    p = core_parameter(cell_n)
    om = O.OracleElevationMap(p)
    out = {}
    perm_rng = np.random.default_rng(99)
    for f in range(n_frames):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        refs = []
        for order in ("fwd", "rev", "perm"):
            rm = O.RefKernelMap(p, tag)
            rm.elevation_map = om.elevation_map.copy(); rm.normal_map = om.normal_map.copy()
            rm.center = om.center.copy(); rm.additive_mean_error = om.additive_mean_error
            pp = pts if order == "fwd" else (pts[::-1].copy() if order == "rev" else pts[perm_rng.permutation(len(pts))])
            rm.move_to(t, R)
            rm.input_pointcloud(pp, ["x", "y", "z"], R, t, 0.02, 0.02)
            refs.append(rm)
        om.move_to(t, R)
        om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        racy = np.zeros((cell_n, cell_n), bool)
        for li in (0, 1, 2, 4, 5, 6):
            for other in refs[1:]:
                racy |= np.abs(refs[0].elevation_map[li] - other.elevation_map[li]) > 1e-6
        out[f"ref_state_{f}"] = refs[0].elevation_map.copy()
        out[f"ref_normal_{f}"] = refs[0].normal_map.copy()
        out[f"racy_{f}"] = racy
        out[f"oracle_state_{f}"] = om.elevation_map.copy()
        out[f"oracle_normal_{f}"] = om.normal_map.copy()
        out[f"ref_point_idx_{f}"] = refs[0].last_point_record[0]
        om.update_variance(); om.update_time()
    return out


def refsrc_case():
    """The reference's dilation / normal / min_filter / max_filter / robot-centric / semantic-fusion kernels on the
    seeded inputs of tests/test_oracle_cpu.py (each input is rebuilt there from the same seed)."""
    import ctypes as C
    from oracle import build_ref
    from oracle.configs import REF_CONFIGS
    p = core_parameter(130)
    W = 130
    rm = O.RefKernelMap(p, "core130")
    _p = O._p
    out = {}
    h, mask = dilation_inputs(W)
    ref = np.zeros((W, W), np.float32); dummy = np.zeros((W, W), np.float32)
    rm.lib.ref_dilation_filter(C.c_longlong(W * W), _p(h), _p(mask), _p(ref), _p(dummy), C.c_int(0))
    out["dilation"] = ref
    rm.elevation_map[2] = mask
    rm.update_normal(ref)
    out["normal"] = rm.normal_map.copy()
    m2 = np.ones((W, W), np.float32); m2[5:-5:4, 5:-5:4] = 0
    rm.elevation_map[0] = h; rm.elevation_map[2] = m2
    out["min_filter"] = rm.min_filter(1)
    h, m = star_inputs(W)
    cur_h, cur_m = h.copy(), m.copy()
    for _ in range(4):                                   # max_filter.py:100-113: every launch reads copies
        ih, im = cur_h.copy(), cur_m.copy()
        rm.lib.ref_max_filter(C.c_longlong(W * W), _p(ih), _p(im), _p(cur_h), _p(cur_m), C.c_int(0))
        if (cur_m > 0.5).all():
            break
    out["max_filter"] = np.where(cur_m > 0.5, cur_h, np.nan).astype(np.float32)
    R = STAR_R
    for thr, fn in ((True, rm.lib.ref_base_elevation_thr), (False, rm.lib.ref_base_elevation_raw)):
        o = h.copy()
        fn(C.c_longlong(W * W), _p(h), _p(m), _p(np.ascontiguousarray(R.reshape(9))), _p(o), C.c_int(0))
        out["base_elevation_thr" if thr else "base_elevation_raw"] = o
    L = C.CDLL(build_ref.build(REF_CONFIGS["core130"], tag="core130", gpu=False))
    idx, valid, inside, pall, feats, cnt = semantic_inputs(p, W)
    new_el = np.zeros((7, W, W), np.float32); new_el[2] = cnt.reshape(W, W)
    fp = lambda a: a.ctypes.data_as(C.c_void_p)
    dummy = np.zeros(16, np.float32)
    sem_ref = np.zeros((3, W, W), np.float32)
    for frame in range(2):
        newmap = np.zeros((3, W, W), np.float32)
        for k, kind in enumerate(("average", "class_average")):
            chan = np.array([3 + k], np.int32); lay = np.array([k], np.int32); dims = np.array([pall.shape[1], 1], np.int32)
            L.ref_sem_sum(C.c_longlong(len(pall)), fp(pall), fp(dummy), fp(dummy), fp(chan), fp(lay), fp(dims), fp(sem_ref), fp(newmap), 0)
            fn = L.ref_sem_average if kind == "average" else L.ref_sem_class_average
            fn(C.c_longlong(W * W), fp(newmap), fp(chan), fp(lay), fp(dims), fp(new_el), fp(sem_ref), 0)
        color_map = np.zeros((4, W, W), np.uint32)
        chan = np.array([5], np.int32); lay = np.array([2], np.int32); dims = np.array([pall.shape[1], 1], np.int32)
        L.ref_sem_add_color(C.c_longlong(len(pall)), fp(pall), fp(dummy), fp(dummy), fp(chan), fp(lay), fp(dims), fp(color_map), 0)
        L.ref_sem_color_average(C.c_longlong(W * W), fp(color_map), fp(chan), fp(lay), fp(dims), fp(sem_ref), 0)
        out[f"semantic_{frame}"] = sem_ref.copy()
    return out


def compared_layers(state):
    """The state with the traversability plane zeroed: the drift and flag comparisons skip it, and it is the
    least compressible plane of the file."""
    s = state.copy()
    s[3] = 0
    return s


def drift_case():
    """Drift compensation fires: the reference kernels run forward and reversed from the oracle's pre-frame state."""
    from oracle.configs import DRIFT_OVERRIDES
    p = core_parameter(130, **DRIFT_OVERRIDES)
    om = O.OracleElevationMap(p)
    out = {}
    for f, (pts, R, t) in enumerate(drift_frames()):
        rf = O.RefKernelMap(p, "drift130"); rr = O.RefKernelMap(p, "drift130")
        for m in (rf, rr):
            m.elevation_map = om.elevation_map.copy(); m.normal_map = om.normal_map.copy(); m.center = om.center.copy()
            m.additive_mean_error = om.additive_mean_error
        for m, pp in ((om, pts), (rf, pts), (rr, pts[::-1].copy())):
            m.move_to(t, R); m.input_pointcloud(pp, ["x", "y", "z"], R, t, 0.02, 0.02)
        racy = np.zeros((130, 130), bool)
        for li in (0, 1, 2, 4, 5, 6):
            racy |= np.abs(rf.elevation_map[li] - rr.elevation_map[li]) > 1e-6
        out[f"ref_state_{f}"] = compared_layers(rf.elevation_map)
        out[f"racy_{f}"] = racy
        out[f"mean_error_{f}"] = np.float32(np.ravel(rf.mean_error)[0])
        om.update_variance(); om.update_time()
    return out


def flags_case(i):
    """FLAG_CASES[i]: the reference source built with those toggles, input order and reversed, three frames."""
    p = core_parameter(130, **FLAG_CASES[i])
    om = O.OracleElevationMap(p)
    out = {}
    for f in range(3):
        pts, R, t = wl.lidar_cloud(0, f, n_rings=24, n_az=500, max_range=4.0)
        refs = []
        for order in (1, -1):
            rm = O.RefKernelMap(p, None)
            rm.elevation_map = om.elevation_map.copy(); rm.normal_map = om.normal_map.copy(); rm.center = om.center.copy()
            rm.additive_mean_error = om.additive_mean_error
            rm.move_to(t, R); rm.input_pointcloud(pts[::order].copy(), ["x", "y", "z"], R, t, 0.02, 0.02)
            refs.append(rm)
        om.move_to(t, R); om.input_pointcloud(pts, ["x", "y", "z"], R, t, 0.02, 0.02)
        racy = np.zeros((130, 130), bool)
        for li in (0, 1, 2, 4, 5, 6):
            racy |= np.abs(refs[0].elevation_map[li] - refs[1].elevation_map[li]) > 1e-6
        out[f"ref_state_{f}"] = compared_layers(refs[0].elevation_map)
        out[f"racy_{f}"] = racy
        out[f"ref_point_idx_{f}"] = refs[0].last_point_record[0]
        om.update_variance(); om.update_time()
    return out


def ref_gpu_index_json():
    """Digests of the reference GPU kernels' per-point write-back (needs a GPU and oracle/_ref/libref_gpu_*.so)."""
    import json
    from ref_gpu import RefGpuMap
    from test_gpu_reference_kernels import index_cases, record_digest
    out = {}
    for tag, p, pts, R, t in index_cases():
        wb = RefGpuMap(p, tag).input_pointcloud(pts, R, t, 0, 0).cpu().numpy()
        out[tag] = record_digest(wb[:, 0].astype(np.int32), wb[:, 1].astype(np.uint8), wb[:, 2].astype(np.uint8))
    with open(os.path.join(HERE, "ref_gpu_index.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    if "--gpu" in sys.argv:
        ref_gpu_index_json()
        sys.exit(0)
    for seed in (0, 1):
        np.savez_compressed(os.path.join(HERE, f"index_default202_seed{seed}.npz"), **index_case(seed))
    np.savez_compressed(os.path.join(HERE, "frames_core130.npz"), **frames_case())
    np.savez_compressed(os.path.join(HERE, "refsrc_core130.npz"), **refsrc_case())
    np.savez_compressed(os.path.join(HERE, "drift_core130.npz"), **drift_case())
    for i in range(len(FLAG_CASES)):
        np.savez_compressed(os.path.join(HERE, f"flags{i}_core130.npz"), **flags_case(i))
    for f in sorted(os.listdir(HERE)):
        print(f, os.path.getsize(os.path.join(HERE, f)))
