// tests/native/planes_host.cpp -- TEST HELPER: the sliding-window fit of csrc/emap_planes.cuh (the same inline
// functions the kernels call) compiled for the CPU, so that the fit and the eigen solver can be checked without a GPU.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -I<cuda>/include -o tests/native/_build/libplanes_host.so tests/native/planes_host.cpp
#include "../../elevation_mapping_cupy_b200/csrc/emap_planes.cuh"

// out = (normal xyz, error) of the k x k window around (r, c)
extern "C" void planes_window_fit(const float* img, int rows, int cols, int r, int c, int k, double res, double* out) {
  const PlaneFit f = pl_window_fit(img, rows, cols, r, c, k, res);
  for (int i = 0; i < 3; i++) out[i] = f.n[i];
  out[3] = f.err;
}
