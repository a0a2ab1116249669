"""The library's host-side launch plan (csrc/emap_plan.cuh) and the polygon check's tiles (csrc/emap_polygon.cuh),
called through tests/native/plan_host.cu, which is compiled with nvcc as the library is on first use
(tests/native/_build/).  The tests check the code the library runs, not a restatement of it."""
import ctypes as C
import functools
import os
import shutil
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "elevation_mapping_cupy_b200", "csrc")
SRC = os.path.join(HERE, "native", "plan_host.cu")
DEPS = [SRC, os.path.join(ROOT, "include", "emap.h")] + [
    os.path.join(CSRC, f) for f in ("emap_plan.cuh", "emap_polygon.cuh", "emap_device.cuh")]


@functools.lru_cache(None)
def _lib():
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libplan_host.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in DEPS):
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        tmp = f"{so}.{os.getpid()}"
        subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                        "-shared", "-I", CSRC, "-o", tmp, SRC], check=True)
        os.replace(tmp, so)
    lib = C.CDLL(so)
    fp, d, i = C.c_void_p, C.c_double, C.c_int
    lib.plan_constants.argtypes = [fp]
    lib.plan_make.argtypes = [i, d, d, i, fp, fp, fp, i]
    lib.plan_ray_box.argtypes = [i, d, d, fp, i, fp]
    lib.plan_raycast_runs.argtypes = [fp, C.c_longlong, i, i]
    lib.plan_polygon_tiles.argtypes = [fp, i, fp, i, d, fp]
    return lib


@functools.lru_cache(None)
def constants():
    """RT, RC_STRIDE, PT_X, PT_Y, PG_COLS, PG_ROWS"""
    v = np.zeros(6, np.int32)
    _lib().plan_constants(v.ctypes.data)
    return dict(zip(("RT", "RC_STRIDE", "PT_X", "PT_Y", "PG_COLS", "PG_ROWS"), (int(x) for x in v)))


_PLAN_FIELDS = ("n_steps", "n_tab", "span_cells", "off_t8", "off_t16", "off_steps", "off_bar", "rc_smem", "lut_p2",
                "cells_per_thread", "post_tma", "post_instance", "post_smem")


@functools.lru_cache(None)
def plan(W, resolution, max_ray_length, dilation=0):
    """make_plan of a W x W map: the FramePlan and DevCfg fields it decides, the march table (`steps`), and where
    k_raycast's coarse maps and march table sit ("gap" between the halves of the cell table, or "behind" it)."""
    out = np.zeros(len(_PLAN_FIELDS), np.int64)
    max_len16 = np.zeros(1, np.float32)
    steps = np.zeros(65535, np.float32)
    _lib().plan_make(W, resolution, max_ray_length, dilation, out.ctypes.data, max_len16.ctypes.data, steps.ctypes.data,
                     len(steps))
    p = dict(zip(_PLAN_FIELDS, (int(x) for x in out)))
    p["post_tma"] = bool(p["post_tma"])
    p["max_len16"] = float(max_len16[0])
    p["steps"] = steps[:p["n_steps"]].copy()
    p["where"] = "gap" if p["off_t8"] < 65536 else "behind"
    return p


def ray_box(W, resolution, max_ray_length, t_rel):
    """ray_box of a frame with sensors at t_rel (positions relative to the map centre): (r0, r1, c0, c1, ts, ta, tb)"""
    t = np.ascontiguousarray(np.asarray(t_rel, np.float32).reshape(-1, 3))
    out = np.zeros(7, np.int32)
    _lib().plan_ray_box(W, resolution, max_ray_length, t.ctypes.data, len(t), out.ctypes.data)
    return tuple(int(x) for x in out)


def raycast_runs(box, n_rays, n_steps, count_rays=False):
    """whether k_raycast runs for a sensor with n_rays rays in a frame with this ray box"""
    b = np.asarray(box, np.int32)
    return bool(_lib().plan_raycast_runs(b.ctypes.data, int(n_rays), int(n_steps), int(count_rays)))


def polygon_tiles(poly, center, W, resolution):
    """the tiles and the interior column window the batch polygon check gives a polygon: (tile rows, tile columns,
    col0, n_col)"""
    xy = np.ascontiguousarray(np.asarray(poly, np.float32).reshape(-1, 2))
    c = np.ascontiguousarray(np.asarray(center, np.float32)[:2])
    out = np.zeros(6, np.int32)
    _lib().plan_polygon_tiles(xy.ctypes.data, len(xy), c.ctypes.data, W, resolution, out.ctypes.data)
    tr0, n_tr, tc0, n_tc, col0, n_col = (int(x) for x in out)
    return range(tr0, tr0 + n_tr), range(tc0, tc0 + n_tc), col0, n_col
