"""oracle/build_ref_semantic.py -- TEST INFRASTRUCTURE ONLY.

Compiles the reference's own kernels of the three remaining point-cloud fusions, from where they lie under
/root/reference, into oracle/_ref/ (git-ignored, travels to the GPU box), next to the frame kernels of
oracle/build_ref.py and through the same recipe (its recording `cupy` stub and its emitter; nothing is copied into the
repository):

  * `libref_semantic_cpu_<tag>.so` -- g++, contraction off, one element at a time in input order when `parallel` is 0;
  * `libref_semantic_gpu_<tag>.so` -- nvcc for sm_90a with its default FMA contraction (128-thread blocks, one element
    per thread, as CuPy launches an ElementwiseKernel).

Kernels:
  * `alpha_kernel` of fusion/pointcloud_class_bayesian.py                  -> ref_sem_alpha
  * `sum_compact_kernel` of fusion/pointcloud_bayesian_inference.py        -> ref_sem_sum_compact
  * `bayesian_inference_kernel` of fusion/pointcloud_bayesian_inference.py -> ref_sem_bayesian_inference
  * `sum_max_kernel` of fusion/pointcloud_class_max.py                     -> ref_sem_sum_max
Template letters: U = float (points_all, maps) and W = int (channel / layer index arrays), as the reference's callers bind
them.  The recipe fixes T = float, so sum_max_kernel's class ranks (`raw T max_id`) are passed as fp32 values; every rank
below 2^24 is exact and converts to the same int index.  Arguments follow the kernel's in_params then out_params, after
`size`, with a trailing `parallel` (host) or `stream` (device).
"""
import json
import os
import subprocess

from oracle import build_ref as B

GENERATOR_VERSION = 1        # bump when the emitted kernels change (prebuilt libraries are rebuilt)

TYPES = {"W": "int"}


def generate(P, gpu):
    W = P["cell_n"]
    cb = B._fusion_mod("pointcloud_class_bayesian.py")
    bi = B._fusion_mod("pointcloud_bayesian_inference.py")
    cm = B._fusion_mod("pointcloud_class_max.py")
    recs = {
        "sem_alpha": cb["alpha_kernel"](P["resolution"], W, W),
        "sem_sum_compact": bi["sum_compact_kernel"](P["resolution"], W, W),
        "sem_bayesian_inference": bi["bayesian_inference_kernel"](W, W),
        "sem_sum_max": cm["sum_max_kernel"](P["resolution"], W, W),
    }
    src = '#include "ref_shim.h"\n'
    for fn, rec in recs.items():
        src += B._emit(rec, fn, gpu, TYPES, carray=True)
    src += f'extern "C" int ref_semantic_cell_n(void) {{ return {W}; }}\n'
    return src


def build(P, tag, gpu=False, verbose=False):
    """Returns the path of the built library (rebuilt when P or the generator changes)."""
    os.makedirs(B.OUT, exist_ok=True)
    kind = "gpu" if gpu else "cpu"
    so = os.path.join(B.OUT, f"libref_semantic_{kind}_{tag}.so")
    meta = os.path.join(B.OUT, f"libref_semantic_{kind}_{tag}.json")
    stamp = dict(P, _generator=GENERATOR_VERSION)
    if os.path.exists(so) and os.path.exists(meta) and json.load(open(meta)) == stamp:
        return so
    if not os.path.isdir(B.REF_ROOT):
        raise FileNotFoundError(f"{B.REF_ROOT} absent and {so} not prebuilt")
    src_path = os.path.join(B.OUT, f"ref_semantic_{kind}_{tag}.{'cu' if gpu else 'cc'}")
    with open(src_path, "w") as f:
        f.write(generate(P, gpu))
    if gpu:
        cmd = ["nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
               "-DREF_SHIM_GPU", "-I", B.HERE, "-shared", "-Xcompiler", "-fPIC", "-cudart", "shared", "-o", so, src_path]
    else:
        cmd = ["g++", "-O2", "-std=c++17", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-w", "-I", B.HERE,
               "-shared", "-fPIC", "-o", so, src_path]
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    json.dump(stamp, open(meta, "w"), sort_keys=True)
    return so
