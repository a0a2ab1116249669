"""Camera image fusion without a GPU: the NumPy restatement (tests/image_oracle.py) against the reference's own kernel
strings compiled for the host with contraction off (oracle/build_ref_image.py), and the library's host part
(image_camera in csrc/emap_image.cuh, compiled as the library is) against the restatement."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import image_oracle as IO          # noqa: E402

W, RES, TAG = 130, 0.04, "core130"
K = np.array([[320.0, 0, 319.5], [0, 320.0, 239.5], [0, 0, 1]], np.float32)
D_RADTAN = np.array([-0.28, 0.07, 1e-3, -2e-3, 0.01], np.float32)


def look_at(cam, target):
    """R (map -> camera optical: z forward, x right, y down), t = -R cam."""
    z = np.asarray(target, np.float64) - cam
    z /= np.linalg.norm(z)
    x = np.cross(z, [0, 0, 1.0])
    x = x / np.linalg.norm(x) if np.linalg.norm(x) > 1e-9 else np.array([1.0, 0, 0])
    y = np.cross(z, x)
    R = np.stack([x, y, z]).astype(np.float32)
    return R, (-R.astype(np.float64) @ cam).astype(np.float32)


def state(seed, nan_frac=0.0):
    rng = np.random.default_rng(seed)
    em = np.zeros((7, W, W), np.float32)
    xs = (np.arange(W) - W // 2) * RES
    em[0] = (0.3 * np.sin(xs[:, None] * 1.3) * np.cos(xs[None, :] * 0.9) + rng.normal(0, 0.02, (W, W))).astype(np.float32)
    em[0][rng.random((W, W)) < 0.01] += 1.0                                    # posts that occlude
    em[2] = (rng.random((W, W)) < 0.85).astype(np.float32)
    em[2][rng.random((W, W)) < 0.02] = 0.5                                     # nonzero, not 1: blocks, never fused
    if nan_frac:
        em[0][rng.random((W, W)) < nan_frac] = np.nan
    return em


CASES = {
    "pinhole": dict(cam=[-1.0, 0.3, 1.5], target=[1.5, 0.0, 0.0], model="plumb_bob", D=D_RADTAN),
    "radtan": dict(cam=[-1.0, -0.4, 1.2], target=[1.2, 0.5, 0.0], model="radtan", D=D_RADTAN),
    "radtan4": dict(cam=[0.5, 0.5, 2.0], target=[-1.0, -0.5, 0.0], model="radtan", D=D_RADTAN[:4]),
    "looking_away": dict(cam=[0.0, 0.0, 1.0], target=[0.0, 0.0, 3.0], model="radtan", D=D_RADTAN),
    "outside_map": dict(cam=[9.0, 4.0, 3.0], target=[0.0, 0.0, 0.0], model="radtan", D=D_RADTAN),
    "edge_cell": dict(cam=[-2.5, -2.5, 0.8], target=[0.0, 0.0, 0.0], model="none", D=np.zeros(0, np.float32)),
    "nan_cells": dict(cam=[-1.0, 0.3, 1.5], target=[1.5, 0.0, 0.0], model="radtan", D=D_RADTAN, nan=0.05),
}


def _ref_lib():
    so = os.path.join(ROOT, "oracle", "_ref", f"libref_image_cpu_{TAG}.so")
    if not os.path.exists(so):
        pytest.skip(f"{so} is built from the reference's source by build(); not present")
    lib = C.CDLL(so)
    fp = C.c_void_p
    lib.ref_image_corr.argtypes = [C.c_longlong, fp, C.c_float, C.c_float, C.c_float, fp, fp, fp, C.c_float, C.c_float,
                                   fp, fp, fp, C.c_int]
    for fn in (lib.ref_image_color, lib.ref_image_exponential):
        fn.argtypes = [C.c_longlong, fp, C.c_float, fp, fp, fp, C.c_float, C.c_float, fp, C.c_int]
    assert lib.ref_image_cell_n() == W
    return lib


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_matches_reference_source(case):
    lib = _ref_lib()
    cfg = CASES[case]
    center = np.array([0.12, -0.08, 0.05], np.float32)
    R, t = look_at(np.asarray(cfg["cam"], np.float64) + center, np.asarray(cfg["target"], np.float64) + center)
    em = state(7, cfg.get("nan", 0.0))
    if case == "edge_cell":
        em[2][0, :] = 1; em[2][:, 0] = 1; em[2][-1, :] = 1; em[2][:, -1] = 1
    H, Wi = 480, 640
    cam = IO.camera(K, cfg["D"], cfg["model"], R, t, center, W, RES)
    u, v, valid = IO.correspondence(em, cam, center, RES, H, Wi)
    p = lambda a: a.ctypes.data
    Dref = cam["D"].copy()
    uv = np.zeros((2, W, W), np.float32)
    vr = np.zeros((W, W), np.bool_)
    lib.ref_image_corr(W * W, p(em), cam["x1"], cam["y1"], cam["z1"], p(cam["P"]), p(K.reshape(-1).copy()), p(Dref),
                       float(H), float(Wi), p(center), p(uv), p(vr), 0)
    assert np.array_equal(vr, valid), f"{case}: {(vr != valid).sum()} cells differ in validity"
    assert np.array_equal(uv[0][valid].view(np.uint32), u[valid].view(np.uint32))
    assert np.array_equal(uv[1][valid].view(np.uint32), v[valid].view(np.uint32))
    if case == "looking_away":
        assert not valid.any()
    elif case == "outside_map":
        assert valid.any() and cam["x1"] > W
    else:
        assert valid.sum() > 100
    if case == "nan_cells":
        return        # int(NaN) is undefined on the host: the device rule of the pixel is checked on the GPU
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (4, H, Wi)).astype(np.float32)
    img[3] = rng.normal(0, 5, (H, Wi)).astype(np.float32)
    for kind, fn, plane in (("color", lib.ref_image_color, 0), ("exponential", lib.ref_image_exponential, 3)):
        sem = rng.normal(0, 1, (2, W, W)).astype(np.float32)
        new = np.zeros_like(sem)
        src = img if kind == "color" else np.ascontiguousarray(img[plane:plane + 1])
        fn(W * W, p(sem), 1.0, p(src), p(uv), p(vr), float(H), float(Wi), p(new), 0)
        want = IO.fuse(sem[1], kind, img, plane, u, v, valid)
        assert np.array_equal(new[1][valid].view(np.uint32), want[valid].view(np.uint32)), kind
        assert np.array_equal(new[1][~valid].view(np.uint32), sem[1][~valid].view(np.uint32)), kind


_HARNESS = r"""
#include <cstdio>
#include "emap_image.cuh"
int main() {
  float K[9], R[9], t[3], c[3], D[8];
  int n_D, W;
  double res;
  char model[32];
  while (std::scanf("%d %lf %d %31s", &W, &res, &n_D, model) == 4) {
    for (float* a : {K, R}) for (int k = 0; k < 9; k++) std::scanf("%a", &a[k]);
    for (float* a : {t, c}) for (int k = 0; k < 3; k++) std::scanf("%a", &a[k]);
    for (int k = 0; k < n_D; k++) std::scanf("%a", &D[k]);
    ImageCam cam;
    const int rc = image_camera(K, D, n_D, model, R, t, c, W, res, &cam);
    std::printf("%d", rc);
    if (rc == 0) {
      for (int k = 0; k < 12; k++) std::printf(" %a", cam.P[k]);
      for (int k = 0; k < 5; k++) std::printf(" %a", cam.D[k]);
      std::printf(" %d %a %a %a", cam.distort, cam.x1, cam.y1, cam.z1);
    }
    std::printf("\n");
  }
  return 0;
}
"""


def test_host_camera_matches_oracle(tmp_path):
    """image_camera (emap_image.cuh), the host part every caller of emap_input_image shares: P, the D rule, the camera
    cell and the rejections, against IO.camera for random poses, far cameras, D of every length and non-finite input."""
    import shutil
    import subprocess
    from elevation_mapping_cupy_b200 import build
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src, exe = tmp_path / "cam.cu", tmp_path / "cam"
    src.write_text(_HARNESS)
    subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", build.CSRC, "-o",
                    str(exe), str(src)], check=True)
    rng = np.random.default_rng(11)
    cases = []
    for k in range(400):
        Wc, res = [(130, 0.04), (202, 0.04), (1024, 0.04), (2048, 0.04), (511, 0.1)][k % 5]
        c = rng.uniform(-300, 300, 3).astype(np.float32)
        span = [2.0, 0.6 * Wc * res, 5e5, 4e6][k % 4]
        cam = c + rng.uniform(-span, span, 3)
        R, t = look_at(cam.astype(np.float64), c.astype(np.float64) + rng.uniform(-3, 3, 3))
        n_D = int(rng.integers(0, 7))
        D = rng.normal(0, 0.1, n_D).astype(np.float32)
        model = ["radtan", "plumb_bob", "equidistant", "none"][k % 4 if k % 3 else 0]
        Kc = K.copy()
        if k % 37 == 5:
            Kc[0, 0] = np.inf
        if k % 41 == 6:
            t = t.copy(); t[1] = np.nan
        cases.append((Wc, res, model, Kc, R, t, c, D))
    text = ""
    for Wc, res, model, Kc, R, t, c, D in cases:
        vals = list(Kc.reshape(-1)) + list(R.reshape(-1)) + list(t) + list(c) + list(D)
        text += f"{Wc} {res!r} {len(D)} {model} " + " ".join(float(np.float32(x)).hex() for x in vals) + "\n"
    out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(out) == len(cases)
    n_ok = n_far = 0
    for line, (Wc, res, model, Kc, R, t, c, D) in zip(out, cases):
        f = line.split()
        try:
            want = IO.camera(Kc, D, model, R, t, c, Wc, res)
        except ValueError as e:
            assert f[0] == ("1" if "finite" in str(e) else "2"), (line, str(e))
            n_far += f[0] == "2"
            continue
        assert f[0] == "0", line
        got = np.array([float.fromhex(x) for x in f[1:18]], np.float32)
        assert np.array_equal(got[:12].view(np.uint32), want["P"].view(np.uint32))
        assert np.array_equal(got[12:17].view(np.uint32), want["D"].view(np.uint32))
        assert int(f[18]) == int(want["distort"])
        rest = np.array([float.fromhex(x) for x in f[19:22]], np.float32)
        assert np.array_equal(rest.view(np.uint32), np.array([want["x1"], want["y1"], want["z1"]], np.float32).view(np.uint32))
        n_ok += 1
    assert n_ok > 150 and n_far > 20
