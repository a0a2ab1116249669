"""Builds libemap.so in-tree with nvcc for sm_90a (no JIT cache: the .so travels with the repo)."""
import os
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libemap.so")
SOURCES = ["emap_api.cu"]
HEADERS = ["emap_kernels.cuh", "emap_device.cuh", "emap_inpaint.cuh", "emap_semantic.cuh", os.path.join("..", "..", "include", "emap.h")]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-shared", "-cudart", "shared", "-Xptxas", "-v"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    cmd = ["nvcc"] + NVCC_FLAGS + ["-o", LIB] + [os.path.join(CSRC, f) for f in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode:
        print(" ".join(cmd))
        print(r.stdout)
        print(r.stderr)
    if r.returncode:
        raise RuntimeError("nvcc failed building libemap.so")
    with open(os.path.join(PKG, "libemap.ptxas.log"), "w") as f:
        f.write(r.stderr)
    return LIB


def build_variant(name, defines):
    """Experimental build with extra -D flags into libemap_<name>.so (selected at run time with EMAP_LIB=...)."""
    out = os.path.join(PKG, "libemap_%s.so" % name)
    cmd = ["nvcc"] + NVCC_FLAGS + ["-D" + d for d in defines] + ["-o", out] + [os.path.join(CSRC, f) for f in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        print(r.stderr)
        raise RuntimeError("nvcc failed building " + out)
    return out


if __name__ == "__main__":
    print(build(force=True, verbose=True))
