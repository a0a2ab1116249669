"""oracle/build_ref_image.py -- TEST INFRASTRUCTURE ONLY.

Compiles the reference's own camera-image kernels, from where they lie under /root/reference, into oracle/_ref/
(git-ignored, travels to the GPU box), next to the frame kernels of oracle/build_ref.py:

  * `libref_image_cpu_<tag>.so` -- g++, contraction off (what tests/image_oracle.py restates);
  * `libref_image_gpu_<tag>.so` -- nvcc for sm_90a with its default FMA contraction (128-thread blocks, one cell per
    thread, as CuPy launches an ElementwiseKernel), so that the GPU box runs the reference's kernels next to the engine.

Kernels (strings obtained through oracle/build_ref.py's recording `cupy` stub; nothing is copied into the repository):
  * `image_to_map_correspondence_kernel` of kernels/custom_image_kernels.py (tolerance_z_collision 0.10, as
    elevation_mapping.py:300-305 builds it);
  * `color_correspondences_to_map_kernel` of fusion/image_color.py;
  * `exponential_correspondences_to_map_kernel` of fusion/image_exponential.py with alpha 0.7 (ImageExponential).
CuPy binds the scalar arguments x1, y1, z1, image_height, image_width and map_idx as `raw U`, i.e. the map's fp32: they
are by-value floats here.  `raw B` (the valid mask) is bool.

Exported: ref_image_corr(size, map, x1, y1, z1, P, K, D, image_height, image_width, center, uv, valid, stream|parallel),
ref_image_color / ref_image_exponential(size, sem_map, map_idx, image, uv, valid, image_height, image_width, new_sem_map,
stream|parallel) and ref_image_cell_n().
"""
import json
import os
import subprocess

from oracle import build_ref as B

GENERATOR_VERSION = 1        # bump when the emitted kernels change (prebuilt libraries are rebuilt)

SCALARS = {"x1", "y1", "z1", "image_height", "image_width", "map_idx"}
CT = {"U": "float", "B": "bool"}


def _emit(rec, fn, gpu):
    ins, outs = B._params(rec)
    args = ["long long size"]
    for t, n in ins:
        args.append(f"float {n}" if n in SCALARS else f"const {CT[t]}* {n}")
    args += [f"{CT[t]}* {n}" for t, n in outs]
    names = [n for _, n in ins] + [n for _, n in outs]
    if gpu:
        s = f"namespace ns_{fn} {{\ntypedef float U; typedef bool B;\n{rec.preamble}\n"
        s += f"__global__ void kern({', '.join(args)}) {{\n"
        s += "  for (long long i_ = blockIdx.x * (long long)blockDim.x + threadIdx.x; i_ < size; i_ += (long long)gridDim.x * blockDim.x) {\n"
        s += "    const int i = (int)i_;\n" + rec.operation + "\n  }\n}\n}\n"
        s += f'extern "C" int ref_{fn}({", ".join(args)}, void* stream) {{\n'
        s += "  if (size <= 0) return 0;\n"
        s += f"  ns_{fn}::kern<<<(unsigned)((size + 127) / 128), 128, 0, (cudaStream_t)stream>>>(size, {', '.join(names)});\n"
        s += "  return (int)cudaGetLastError();\n}\n"
    else:
        s = f"namespace refshim {{ namespace ns_{fn} {{\ntypedef float U; typedef bool B;\n{rec.preamble}\n"
        s += f"static inline void body(const int i, {', '.join(args[1:])}) {{\n{rec.operation}\n}}\n}} }}\n"
        s += f'extern "C" int ref_{fn}({", ".join(args)}, int parallel) {{\n'
        s += "  if (parallel) {\n    _Pragma(\"omp parallel for schedule(dynamic, 512)\")\n"
        s += f"    for (long long i = 0; i < size; i++) refshim::ns_{fn}::body((int)i, {', '.join(names)});\n  }} else {{\n"
        s += f"    for (long long i = 0; i < size; i++) refshim::ns_{fn}::body((int)i, {', '.join(names)});\n  }}\n  return 0;\n}}\n"
    return s


def generate(P, gpu):
    W = P["cell_n"]
    cik = B._load_with_stub(os.path.join(B.REF_ROOT, "kernels", "custom_image_kernels.py"), "ref_custom_image_kernels")
    col = B._fusion_mod("image_color.py")
    exp = B._fusion_mod("image_exponential.py")
    recs = {
        "image_corr": cik.image_to_map_correspondence_kernel(P["resolution"], W, W, 0.10),
        "image_color": col["color_correspondences_to_map_kernel"](P["resolution"], W, W),
        "image_exponential": exp["exponential_correspondences_to_map_kernel"](P["resolution"], W, W, 0.7),
    }
    src = '#include "ref_shim.h"\n'
    for fn, rec in recs.items():
        src += _emit(rec, fn, gpu)
    src += f'extern "C" int ref_image_cell_n(void) {{ return {W}; }}\n'
    return src


def build(P, tag, gpu=False, verbose=False):
    """Returns the path of the built library (rebuilt when P or the generator changes)."""
    os.makedirs(B.OUT, exist_ok=True)
    kind = "gpu" if gpu else "cpu"
    so = os.path.join(B.OUT, f"libref_image_{kind}_{tag}.so")
    meta = os.path.join(B.OUT, f"libref_image_{kind}_{tag}.json")
    stamp = dict(P, _generator=GENERATOR_VERSION)
    if os.path.exists(so) and os.path.exists(meta) and json.load(open(meta)) == stamp:
        return so
    if not os.path.isdir(B.REF_ROOT):
        raise FileNotFoundError(f"{B.REF_ROOT} absent and {so} not prebuilt")
    src_path = os.path.join(B.OUT, f"ref_image_{kind}_{tag}.{'cu' if gpu else 'cc'}")
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
