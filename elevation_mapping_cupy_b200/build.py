"""Builds libemap.so in-tree with nvcc for sm_90a (no JIT cache: the .so travels with the repo).

Each source is compiled on its own (in parallel, objects in a temporary directory) and the objects are linked once."""
import os
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libemap.so")
SOURCES = ["emap_api.cu", "emap_export_api.cu", "emap_polygon_api.cu", "emap_plugins_api.cu",
           "emap_terrain_query_api.cu"]
HEADERS = ["emap_handle.cuh", "emap_kernels.cuh", "emap_export.cuh", "emap_plugins.cuh", "emap_device.cuh",
           "emap_inpaint.cuh", "emap_semantic.cuh", "emap_polygon.cuh", "emap_semantic_plugins.cuh", "emap_image.cuh",
           "emap_submap.cuh", "emap_mapcloud.cuh", "emap_initialize.cuh", "emap_sources.cuh", "emap_plan.cuh",
           "emap_planes.cuh", "emap_regions.cuh", "emap_postprocess.cuh", "emap_terrain_query.cuh",
           "emap_grid.cuh", "emap_grid_lookup.cuh", "emap_resample.cuh", "emap_sdf.cuh", "emap_values_at.cuh", "emap_filters.cuh", os.path.join("..", "..", "include", "emap.h")]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMPILE_FLAGS = ["-O3", "-std=c++17"] + GENCODE + ["-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
LINK_FLAGS = GENCODE + ["-shared", "-cudart", "shared"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def _run(cmd, out, verbose):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode:
        print(" ".join(cmd))
        print(r.stdout)
        print(r.stderr)
    if r.returncode:
        raise RuntimeError("nvcc failed building " + out)
    return r.stderr


def _nvcc(out, defines=(), verbose=False):
    """Compiles every source to an object, in parallel, and links the objects into `out`; returns the ptxas report of
    every source, in SOURCES order."""
    with tempfile.TemporaryDirectory(prefix="emap_build_") as tmp:
        objs = [os.path.join(tmp, os.path.splitext(src)[0] + ".o") for src in SOURCES]
        cmds = [["nvcc"] + COMPILE_FLAGS + ["-D" + d for d in defines] + ["-c", os.path.join(CSRC, src), "-o", obj]
                for src, obj in zip(SOURCES, objs)]
        with ThreadPoolExecutor(max_workers=len(cmds)) as pool:
            logs = list(pool.map(lambda cmd: _run(cmd, out, verbose), cmds))
        _run(["nvcc"] + LINK_FLAGS + ["-o", out] + objs, out, verbose)
    return "".join(logs)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    log = _nvcc(LIB, verbose=verbose)
    with open(os.path.join(PKG, "libemap.ptxas.log"), "w") as f:
        f.write(log)
    return LIB


def build_variant(name, defines):
    """Experimental build with extra -D flags into libemap_<name>.so (selected at run time with EMAP_LIB=...)."""
    out = os.path.join(PKG, "libemap_%s.so" % name)
    _nvcc(out, defines)
    return out


if __name__ == "__main__":
    print(build(force=True, verbose=True))
