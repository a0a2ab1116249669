"""One inpainting call on config D's map (2048^2, one 1M-point depth frame): the workload of DESIGN.md §4c."""
import os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from elevation_mapping_cupy_b200.parameter import core_parameter
from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
from elevation_mapping_cupy_b200 import workloads as wl
W = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
em = ElevationMap(core_parameter(W))
pts, R, t = wl.depth_camera_cloud(3, 0)
em.move_to(t, R)
em.input_pointcloud(torch.from_numpy(pts).cuda(), ["x", "y", "z"], R, t, 0.02, 0.02)
torch.cuda.synchronize()
for rep in range(2):
    t0 = time.perf_counter(); em.get_layer("inpaint"); torch.cuda.synchronize(); dt = time.perf_counter() - t0
import ctypes as C
r_, mj, nc = C.c_int32(), C.c_int32(), C.c_int32()
em._check(em._L.emap_inpaint_stats(em._h, C.byref(r_), C.byref(mj), C.byref(nc)))
print("inpaint ms", 1e3 * dt, "rounds", r_.value, "max jacobi", mj.value, "not converged", nc.value)
