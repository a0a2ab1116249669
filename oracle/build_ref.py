"""oracle/build_ref.py -- TEST INFRASTRUCTURE ONLY.

Compiles the REFERENCE'S OWN kernel source for this path, from where it lies
under /root/reference, into oracle/_ref/ (git-ignored, travels to the GPU box):

  * `libref_cpu_<tag>.so`  -- the CUDA-C strings of
    elevation_mapping_cupy/script/elevation_mapping_cupy/kernels/custom_kernels.py
    (add_points_kernel, error_counting_kernel, average_map_kernel,
    dilation_filter_kernel, normal_filter_kernel) and plugins/min_filter.py,
    compiled for the host with g++ through a small shim header
    (oracle/ref_shim.h) that restates what CuPy supplies around an
    ElementwiseKernel body: `class float16` (cupy/_core/include/cupy/carray.cuh,
    third-party, not under /root/reference), CUDA's mixed-type min/max
    overloads, atomicAdd, and the `for i in range(size)` loop.
  * `libref_gpu_<tag>.so`  -- the same strings compiled by nvcc for sm_90a
    (128-thread blocks, one element per thread, as CuPy launches them), so that
    the GPU box can run the real reference kernels next to the new engine.

No reference source is copied into the repository: the strings are obtained at
build time by importing the reference module with a stub `cupy` whose
ElementwiseKernel records its arguments; the generated translation units live
only under oracle/_ref/.  Kernel constants are baked in at generation time
(the reference does the same through string.Template), so one library is built
per parameter set ("tag").
"""
import hashlib
import importlib.util
import json
import os
import subprocess
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = "/root/reference/elevation_mapping_cupy/script/elevation_mapping_cupy"
OUT = os.path.join(HERE, "_ref")


GENERATOR_VERSION = 2        # bump when the set of emitted kernels changes (prebuilt libraries are rebuilt)


class _Rec:
    def __init__(self, in_params, out_params, operation, name, preamble=""):
        self.in_params, self.out_params = in_params, out_params
        self.operation, self.name, self.preamble = operation, name, preamble


def _load_with_stub(path, modname):
    """Import a reference module with `cupy` replaced by a recorder."""
    stub = types.ModuleType("cupy")
    stub.ElementwiseKernel = lambda in_params, out_params, operation, name="k", preamble="", **kw: _Rec(
        in_params, out_params, operation, name, preamble)
    stub.ndarray = object
    stub.zeros = lambda *a, **k: None
    saved = {k: sys.modules.get(k) for k in ("cupy",)}
    sys.modules["cupy"] = stub
    try:
        spec = importlib.util.spec_from_file_location(modname, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return mod


def _min_filter_rec(cell_n, dilation_size):
    """plugins/min_filter.py builds its kernel inside MinFilter.__init__ and
    imports .plugin_manager (needs ruamel); pull the class out with stubs."""
    src = open(os.path.join(REF_ROOT, "plugins", "min_filter.py")).read()
    src = src.replace("from .plugin_manager import PluginBase", "class PluginBase:\n    def __init__(self, *a, **k):\n        pass\n")
    stub = types.ModuleType("cupy")
    stub.ElementwiseKernel = lambda in_params, out_params, operation, name="k", preamble="", **kw: _Rec(
        in_params, out_params, operation, name, preamble)
    stub.ndarray = object
    stub.zeros = lambda *a, **k: None
    saved = sys.modules.get("cupy")
    sys.modules["cupy"] = stub
    try:
        ns = {}
        exec(compile(src, "min_filter.py", "exec"), ns)
        obj = ns["MinFilter"](cell_n=cell_n, dilation_size=dilation_size, iteration_n=1)
    finally:
        if saved is None:
            sys.modules.pop("cupy", None)
        else:
            sys.modules["cupy"] = saved
    return obj.min_filter_kernel


def _plugin_rec(fname, cls, attr, **ctor):
    """Kernel built inside a plugin class constructor (the module imports .plugin_manager, which needs ruamel)."""
    src = open(os.path.join(REF_ROOT, "plugins", fname)).read()
    for imp in ("from .plugin_manager import PluginBase", "from elevation_mapping_cupy.plugins.plugin_manager import PluginBase"):
        src = src.replace(imp, "class PluginBase:\n    def __init__(self, *a, **k):\n        pass\n")
    stub = types.ModuleType("cupy")
    stub.ElementwiseKernel = lambda in_params, out_params, operation, name="k", preamble="", **kw: _Rec(
        in_params, out_params, operation, name, preamble)
    stub.ndarray = object
    stub.float32 = "float32"
    stub.zeros = lambda *a, **k: None
    saved = sys.modules.get("cupy")
    sys.modules["cupy"] = stub
    try:
        ns = {}
        exec(compile(src, fname, "exec"), ns)
        obj = ns[cls](**ctor)
    finally:
        if saved is None:
            sys.modules.pop("cupy", None)
        else:
            sys.modules["cupy"] = saved
    return getattr(obj, attr)


def _fusion_mod(fname):
    """fusion/<fname>: module-level kernel factories; imports .fusion_manager (FusionBase) and cupy."""
    src = open(os.path.join(REF_ROOT, "fusion", fname)).read()
    src = src.replace("from .fusion_manager import FusionBase", "class FusionBase:\n    pass\n")
    stub = types.ModuleType("cupy")
    stub.ElementwiseKernel = lambda in_params, out_params, operation, name="k", preamble="", **kw: _Rec(
        in_params, out_params, operation, name, preamble)
    stub.ndarray = object
    saved = sys.modules.get("cupy")
    sys.modules["cupy"] = stub
    try:
        ns = {}
        exec(compile(src, fname, "exec"), ns)
    finally:
        if saved is None:
            sys.modules.pop("cupy", None)
        else:
            sys.modules["cupy"] = saved
    return ns


def _params(rec):
    """'raw U a, raw T b' -> [('U','a'), ...] for in and out."""
    def parse(s):
        out = []
        for tok in s.split(","):
            parts = tok.split()
            assert parts[0] == "raw", tok
            out.append((parts[1], parts[2]))
        return out
    return parse(rec.in_params), parse(rec.out_params)


CTYPE = {"U": "float", "T": "float", "int16": "short"}


def _emit(rec, fn, gpu, types=None, carray=False):
    """types: C types of the kernel's other template letters (e.g. {"W": "int", "V": "unsigned int"}), as CuPy would
    deduce them from the arrays the caller passes.  carray: wrap the raw pointers in CArr (float-indexable, as CuPy's
    CArray is) inside the body."""
    ins, outs = _params(rec)
    CT = dict(CTYPE, **(types or {}))
    sfx = "_" if carray else ""
    args = ["long long size"] + [f"const {CT[t]}* {n}{sfx}" for t, n in ins] + [f"{CT[t]}* {n}{sfx}" for t, n in outs]
    names = [n for _, n in ins] + [n for _, n in outs]
    wrap = ""
    if carray:
        wrap = "".join(f"const CArr<const {CT[t]}> {n}{{{n}_}}; " for t, n in ins) + "".join(f"const CArr<{CT[t]}> {n}{{{n}_}}; " for t, n in outs) + "\n"
    extra_typedefs = "".join(f"typedef {c} {t}; " for t, c in (types or {}).items())
    body = wrap + rec.operation
    if gpu:
        s = f"namespace ns_{fn} {{\ntypedef float U; typedef float T; {extra_typedefs}\n{rec.preamble}\n"
        s += f"__global__ void kern({', '.join(args)}) {{\n"
        s += "  for (long long i_ = blockIdx.x * (long long)blockDim.x + threadIdx.x; i_ < size; i_ += (long long)gridDim.x * blockDim.x) {\n"
        s += "    const int i = (int)i_;\n" + body + "\n  }\n}\n}\n"
        s += f'extern "C" int ref_{fn}({", ".join(args)}, void* stream) {{\n'
        s += "  if (size <= 0) return 0;\n"
        s += f"  ns_{fn}::kern<<<(unsigned)((size + 127) / 128), 128, 0, (cudaStream_t)stream>>>(size, {', '.join(n + sfx for n in names)});\n"
        s += "  return (int)cudaGetLastError();\n}\n"
    else:
        s = f"namespace refshim {{ namespace ns_{fn} {{\ntypedef float U; typedef float T; {extra_typedefs}\n{rec.preamble}\n"
        s += f"static inline void body(const int i, {', '.join(args[1:])}) {{\n{body}\n}}\n}} }}\n"
        s += f'extern "C" int ref_{fn}({", ".join(args)}, int parallel) {{\n'
        s += "  if (parallel) {\n    _Pragma(\"omp parallel for schedule(dynamic, 512)\")\n"
        s += f"    for (long long i = 0; i < size; i++) refshim::ns_{fn}::body((int)i, {', '.join(n + sfx for n in names)});\n  }} else {{\n"
        s += f"    for (long long i = 0; i < size; i++) refshim::ns_{fn}::body((int)i, {', '.join(n + sfx for n in names)});\n  }}\n  return 0;\n}}\n"
    return s


def param_tag(P):
    return hashlib.sha1(json.dumps(P, sort_keys=True).encode()).hexdigest()[:12]


def generate(P, gpu):
    """P: dict of python-typed parameters exactly as ElevationMap.compile_kernels
    passes them (elevation_mapping.py:240-282)."""
    ck = _load_with_stub(os.path.join(REF_ROOT, "kernels", "custom_kernels.py"), "ref_custom_kernels")
    W = P["cell_n"]
    recs = {
        "add_points": ck.add_points_kernel(
            P["resolution"], W, W, P["sensor_noise_factor"], P["mahalanobis_thresh"], P["outlier_variance"],
            P["wall_num_thresh"], P["max_ray_length"], P["cleanup_step"], P["min_valid_distance"],
            P["max_height_range"], P["cleanup_cos_thresh"], P["ramped_height_range_a"],
            P["ramped_height_range_b"], P["ramped_height_range_c"], P["enable_edge_sharpen"],
            P["enable_visibility_cleanup"]),
        "error_counting": ck.error_counting_kernel(
            P["resolution"], W, W, P["sensor_noise_factor"], P["mahalanobis_thresh"],
            P["drift_compensation_variance_inlier"], P["traversability_inlier"], P["min_valid_distance"],
            P["max_height_range"], P["ramped_height_range_a"], P["ramped_height_range_b"],
            P["ramped_height_range_c"]),
        "average_map": ck.average_map_kernel(W, W, P["max_variance"], P["initial_variance"]),
        "dilation_filter": ck.dilation_filter_kernel(W, W, P["dilation_size"]),
        "normal_filter": ck.normal_filter_kernel(W, W, P["resolution"]),
        "min_filter": _min_filter_rec(W, P.get("min_filter_dilation_size", 1)),
        "max_filter": _plugin_rec("max_filter.py", "MaxFilter", "max_filter_kernel", cell_n=W,
                                  dilation_size=P.get("min_filter_dilation_size", 1), iteration_n=1),
        "base_elevation_thr": _plugin_rec("robot_centric_elevation.py", "RobotCentricElevation", "base_elevation_kernel",
                                          cell_n=W, resolution=P["resolution"], threshold=P.get("rce_threshold", 1.1),
                                          use_threshold=True),
        "base_elevation_raw": _plugin_rec("robot_centric_elevation.py", "RobotCentricElevation", "base_elevation_kernel",
                                          cell_n=W, resolution=P["resolution"], threshold=P.get("rce_threshold", 1.1),
                                          use_threshold=False),
    }
    src = '#include "ref_shim.h"\n'
    for fn, rec in recs.items():
        src += _emit(rec, fn, gpu)
    # semantic point-channel fusion (fusion/pointcloud_average.py, pointcloud_class_average.py, pointcloud_color.py)
    avg = _fusion_mod("pointcloud_average.py"); cavg = _fusion_mod("pointcloud_class_average.py"); col = _fusion_mod("pointcloud_color.py")
    alpha = P.get("average_weight", 0.5)
    sem = {
        "sem_sum": (avg["sum_kernel"](P["resolution"], W, W), {"W": "int"}),
        "sem_average": (avg["average_kernel"](W, W), {"W": "int", "V": "float"}),
        "sem_class_average": (cavg["class_average_kernel"](W, W, alpha), {"W": "int", "V": "float"}),
        "sem_add_color": (col["add_color_kernel"](W, W), {"W": "int", "V": "unsigned int"}),
        "sem_color_average": (col["color_average_kernel"](W, W), {"W": "int", "V": "unsigned int"}),
    }
    for fn, (rec, ty) in sem.items():
        src += _emit(rec, fn, gpu, ty, carray=True)
    src += f'extern "C" int ref_cell_n(void) {{ return {W}; }}\n'
    return src


def build(P, tag=None, gpu=False, verbose=False):
    """Returns the path of the built library (cached by parameter hash)."""
    tag = tag or param_tag(P)
    os.makedirs(OUT, exist_ok=True)
    kind = "gpu" if gpu else "cpu"
    so = os.path.join(OUT, f"libref_{kind}_{tag}.so")
    meta = os.path.join(OUT, f"libref_{kind}_{tag}.json")
    stamp = dict(P, _generator=GENERATOR_VERSION)
    if os.path.exists(so) and os.path.exists(meta) and json.load(open(meta)) == stamp:
        return so
    if not os.path.isdir(REF_ROOT):
        raise FileNotFoundError(f"{REF_ROOT} absent and {so} not prebuilt")
    ext = "cu" if gpu else "cc"
    src_path = os.path.join(OUT, f"ref_{kind}_{tag}.{ext}")
    with open(src_path, "w") as f:
        f.write(generate(P, gpu))
    if gpu:
        cmd = ["nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
               "-DREF_SHIM_GPU", "-I", HERE, "-shared", "-Xcompiler", "-fPIC", "-cudart", "shared",
               "-o", so, src_path]
    else:
        cmd = ["g++", "-O2", "-std=c++17", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-w", "-I", HERE,
               "-shared", "-fPIC", "-o", so, src_path]
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    json.dump(stamp, open(meta, "w"), sort_keys=True)
    return so


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    from oracle.configs import REF_CONFIGS
    for name, P in REF_CONFIGS.items():
        for gpu in (False, True):
            print(name, "gpu" if gpu else "cpu", build(P, tag=name, gpu=gpu, verbose=True))
