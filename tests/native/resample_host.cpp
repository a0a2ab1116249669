// tests/native/resample_host.cpp -- TEST HELPER: the geometry and the per-cell resampling of csrc/emap_resample.cuh
// (the same inline functions emap_plane_grid_geometry and k_rs_resample call) compiled for the CPU, so that they can
// be checked against inpainting.cpp's formula and the NumPy restatement without a device.
//   build: g++ -O2 -shared -fPIC -I<cuda>/include -o tests/native/_build/libresample_host.so tests/native/resample_host.cpp
#include "../../elevation_mapping_cupy_b200/csrc/emap_resample.cuh"

extern "C" void resample_geometry(int64_t rows, int64_t cols, double res, double new_res, int64_t* size,
                                  double* out_res) {
  rs_geometry(rows, cols, res, new_res, size, out_res);
}

extern "C" void resample_grid(const float* src, int R, int C, float* dst, int rows, int cols) {
  for (int r = 0; r < rows; r++)
    for (int c = 0; c < cols; c++) dst[(int64_t)r * cols + c] = rs_cell(src, R, C, rows, cols, r, c);
}
