"""Test helper: the REFERENCE'S OWN CUDA kernels on the GPU.

oracle/build_ref.py compiles the CUDA-C strings of kernels/custom_kernels.py unmodified with nvcc for sm_90a
(oracle/_ref/libref_gpu_<tag>.so, 128-thread blocks, one element per thread, as CuPy launches them).  This class
drives them in the order of elevation_mapping.py:316-391 with torch tensors standing in for the CuPy arrays and
torch/cuDNN convolutions for traversability_filter.py:15-42 (that IS the reference's traversability path).
It is racy exactly like the original, so comparisons are made on order-independent cells only.
"""
import ctypes as C
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class RefGpuMap:
    def __init__(self, param, tag):
        so = os.path.join(ROOT, "oracle", "_ref", f"libref_gpu_{tag}.so")
        if not os.path.exists(so):
            raise FileNotFoundError(so)
        self.lib = C.CDLL(so)
        assert self.lib.ref_cell_n() == param.cell_n
        self.param = param
        W = self.cell_n = param.cell_n
        dev = "cuda"
        self.elevation_map = torch.zeros((7, W, W), dtype=torch.float32, device=dev)
        self.elevation_map[1] += param.initial_variance
        self.elevation_map[3] += 1.0
        self.new_map = torch.zeros((7, W, W), dtype=torch.float32, device=dev)
        self.normal_map = torch.zeros((3, W, W), dtype=torch.float32, device=dev)
        self.traversability_input = torch.zeros((W, W), dtype=torch.float32, device=dev)
        self.mask_dummy = torch.zeros((W, W), dtype=torch.float32, device=dev)
        self.zero = torch.zeros(1, dtype=torch.float32, device=dev)
        self.center = np.zeros(3, np.float32)
        self.mean_error = 0.0
        self.additive_mean_error = 0.0
        if not np.any(param.w1):
            param.load_weights(param.weight_file)
        f = lambda w: torch.from_numpy(np.ascontiguousarray(w, np.float32)).to(dev)
        self.w1, self.w2, self.w3, self.wo = f(param.w1), f(param.w2), f(param.w3), f(param.w_out)
        cell_range = int(np.clip(int(param.overlap_clear_range_xy / param.resolution), 0, W))
        self.cell_min, self.cell_max = W // 2 - cell_range // 2, W // 2 + cell_range // 2
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False

    @staticmethod
    def _p(t):
        return C.c_void_p(t.data_ptr())

    def set_state(self, em, nm, center):
        self.elevation_map.copy_(torch.from_numpy(np.ascontiguousarray(em)))
        self.normal_map.copy_(torch.from_numpy(np.ascontiguousarray(nm)))
        self.center = np.asarray(center, np.float32).copy()

    def input_pointcloud(self, pts, R, t, position_noise, orientation_noise, points_dev=None):
        """elevation_mapping.py:316-391; returns the per-point write-back (CK.py:260-262) as a device tensor"""
        pr, W, L, p_ = self.param, self.cell_n, self.lib, self._p
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.new_map.zero_()
        error = torch.zeros(1, dtype=torch.float32, device="cuda"); error_cnt = torch.zeros(1, dtype=torch.float32, device="cuda")
        points = points_dev.clone() if points_dev is not None else torch.from_numpy(np.ascontiguousarray(pts[:, :3], np.float32)).cuda()
        n = points.shape[0]
        Rd = torch.from_numpy(np.ascontiguousarray(R, np.float32).reshape(9)).cuda()
        td = torch.from_numpy((np.asarray(t, np.float32) - self.center).astype(np.float32)).cuda()
        em = self.elevation_map
        L.ref_error_counting(C.c_longlong(n), p_(em), p_(points), p_(self.zero), p_(self.zero), p_(Rd), p_(td),
                             p_(self.new_map), p_(error), p_(error_cnt), st)
        if (pr.enable_drift_compensation and float(error_cnt) > pr.min_height_drift_cnt        # host sync, as EM.py:346-353
                and (position_noise > pr.position_noise_thresh or orientation_noise > pr.orientation_noise_thresh)):
            self.mean_error = error / error_cnt
            self.additive_mean_error = self.additive_mean_error + self.mean_error
            if abs(float(self.mean_error)) < pr.max_drift:
                em[0] += self.mean_error * np.float32(pr.drift_compensation_alpha)
        L.ref_add_points(C.c_longlong(n), p_(self.zero), p_(self.zero), p_(Rd), p_(td), p_(self.normal_map),
                         p_(points), p_(em), p_(self.new_map), st)
        L.ref_average_map(C.c_longlong(W * W), p_(self.new_map), p_(em), st)
        if pr.enable_overlap_clearance:                                                       # EM.py:393-410
            hmin = td[2] - np.float32(pr.overlap_clear_range_z); hmax = td[2] + np.float32(pr.overlap_clear_range_z)
            near = em[:, self.cell_min:self.cell_max, self.cell_min:self.cell_max]
            ok = ~torch.logical_or(near[0] < hmin, near[0] > hmax)
            near[0] = torch.where(ok, near[0], torch.zeros_like(near[0]))
            near[1] = torch.where(ok, near[1], torch.full_like(near[1], pr.initial_variance))
            near[2] = torch.where(ok, near[2], torch.zeros_like(near[2]))
            ok = ~torch.logical_or(near[5] < hmin, near[5] > hmax)
            near[5] = torch.where(ok, near[5], torch.zeros_like(near[5]))
            near[6] = torch.where(ok, near[6], torch.zeros_like(near[6]))
        self.traversability_input.zero_()
        mask = em[2] + em[6]
        L.ref_dilation_filter(C.c_longlong(W * W), p_(em[5]), p_(mask), p_(self.traversability_input), p_(self.mask_dummy), st)
        import torch.nn.functional as F
        e = self.traversability_input.view(1, 1, W, W)                                        # TF.py:32-42
        o1 = F.conv2d(e, self.w1.view(4, 1, 3, 3), dilation=1)[:, :, 2:-2, 2:-2]
        o2 = F.conv2d(e, self.w2.view(4, 1, 3, 3), dilation=2)[:, :, 1:-1, 1:-1]
        o3 = F.conv2d(e, self.w3.view(4, 1, 3, 3), dilation=3)
        out = torch.exp(-F.conv2d(torch.cat((o1, o2, o3), 1).abs(), self.wo.view(1, 12, 1, 1)))
        em[3][3:-3, 3:-3] = out[0, 0]
        self.normal_map.zero_()
        L.ref_normal_filter(C.c_longlong(W * W), p_(self.traversability_input), p_(em[2]), p_(self.normal_map), st)
        return points
