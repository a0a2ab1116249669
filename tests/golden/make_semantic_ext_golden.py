"""Regenerates tests/golden/semantic_ext_core130.npz: the reference's class_bayesian, bayesian_inference and class_max
fusions on the seeded inputs of tests/semantic_ext_inputs.py, two frames.

The kernels are the reference's own strings (alpha_kernel, sum_compact_kernel, bayesian_inference_kernel,
sum_max_kernel), compiled for the host by oracle/build_ref_semantic.py and run one element at a time in input order,
launched over every (point, channel) and (cell, channel) pair (DESIGN §4d).  The array steps around them restate the
reference's __call__ bodies (fusion/pointcloud_class_bayesian.py:71-75, pointcloud_class_max.py:82-123) in NumPy, with
the class set U and id_max as DESIGN §4d defines them.  Needs the reference tree.  Usage: python
tests/golden/make_semantic_ext_golden.py
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from elevation_mapping_cupy_b200.parameter import core_parameter   # noqa: E402
from oracle import build_ref_semantic as BS                        # noqa: E402
from oracle import semantic_ext as X                               # noqa: E402
from oracle.configs import REF_CONFIGS                             # noqa: E402
import semantic_ext_inputs as SI                                   # noqa: E402


def main():
    W = SI.W
    p = core_parameter(W)
    L = C.CDLL(BS.build(REF_CONFIGS["core130"], tag="core130", gpu=False))
    fp = lambda a: a.ctypes.data_as(C.c_void_p)
    i32 = lambda v: np.array(v, np.int32)
    dummy = np.zeros(16, np.float32)
    sigma = np.ones((2, W, W), np.float32)
    sem_bi = np.zeros((2, W, W), np.float32)
    id_max = np.zeros((2, W, W), np.int32)
    out = {}
    for frame in range(2):
        idx, valid, inside, rows, feats, cnt = SI.frame_inputs(p, frame)
        N, ncol = rows.shape
        # class_bayesian (pointcloud_class_bayesian.py:62-75): new_map zeroed every frame
        new_map = np.zeros((3, W, W), np.float32)
        L.ref_sem_alpha(C.c_longlong(N * 3), fp(rows), fp(i32(SI.CB_COLS)), fp(i32([0, 1, 2])), fp(i32([ncol, 3])),
                        fp(new_map), 0)
        s = new_map[0] + new_map[1] + new_map[2]
        s[s == 0] = 1
        out[f"cb_{frame}"] = (new_map / s[None]).astype(np.float32)
        # bayesian_inference (pointcloud_bayesian_inference.py:101-122), variance persistent from 1.0
        sum_mean = np.zeros((2, W, W), np.float32)
        L.ref_sem_sum_compact(C.c_longlong(N * 2), fp(rows), fp(dummy), fp(dummy), fp(i32(SI.BI_COLS)), fp(i32([0, 1])),
                              fp(i32([ncol, 2])), fp(sum_mean), 0)
        new_el = np.zeros((7, W, W), np.float32); new_el[2] = cnt.reshape(W, W)
        L.ref_sem_bayesian_inference(C.c_longlong(W * W * 2), fp(i32(SI.BI_COLS)), fp(i32([0, 1])), fp(i32([ncol, 2])),
                                     fp(new_el), fp(sigma), fp(sum_mean), fp(sem_bi), 0)
        out[f"bi_{frame}"] = sem_bi.copy()
        out[f"bi_sigma_{frame}"] = sigma.copy()
        # class_max (pointcloud_class_max.py:81-123): sums per class rank by sum_max_kernel, then the rounds
        prob, cid = X.decode_max(feats[:, [c - 3 for c in SI.CM_COLS]])
        U = np.union1d(np.unique(cid), np.unique(id_max))
        rank = np.searchsorted(U, cid).astype(np.float32)
        prob_sum = np.zeros((len(U), W, W), np.float32)
        L.ref_sem_sum_max(C.c_longlong(N), fp(rows), fp(np.ascontiguousarray(prob)), fp(np.ascontiguousarray(rank)),
                          fp(i32(SI.CM_COLS)), fp(i32([0, 1])), fp(i32([ncol, 2, 2])), fp(prob_sum), 0)
        nm = np.zeros((2, W, W), np.float32)
        for k in range(2):
            am = np.argmax(prob_sum, axis=0)
            nm[k] = np.amax(prob_sum, axis=0)
            id_max[k] = U[am]
            prob_sum[am] = 0
        s = nm[0] + nm[1]
        s[s == 0] = 1
        out[f"cm_{frame}"] = (nm / s[None]).astype(np.float32)
        out[f"cm_id_{frame}"] = id_max.copy()
    np.savez_compressed(os.path.join(HERE, "semantic_ext_core130.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
