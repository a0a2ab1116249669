// postprocess_host.cpp -- the host parts of csrc/emap_postprocess.cuh for tests/test_planar_terrain_cpu.py: the
// ellipse's row spans, the kernel sizes, the Gaussian coefficients and the slope offsets, compiled by g++.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -I<cuda>/include -o tests/native/_build/libpostprocess_host.so
//          tests/native/postprocess_host.cpp
#include "../../elevation_mapping_cupy_b200/csrc/emap_postprocess.cuh"

extern "C" {

// half[i] for the rows of a MORPH_ELLIPSE of odd size
void pp_ellipse_spans(int size, int* half) {
  for (int i = 0; i < size; i++) half[i] = rg_ellipse_half((size - 1) / 2, i);
}

int pp_kernel(double size, double res) { return pp_kernel_size(size, res); }

void pp_gauss(int k, float* out) { pp_gauss_coeffs(k, out); }

// the k x k offsets table, row-major
void pp_offsets(float slope, int k, float* out) {
  const int h = (k - 1) / 2;
  for (int a = 0; a < k; a++)
    for (int b = 0; b < k; b++) out[a * k + b] = pp_slope_offset(slope, a - h, b - h);
}
}
