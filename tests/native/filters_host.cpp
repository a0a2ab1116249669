// filters_host.cpp -- the host part of emap_grid_filter's Gaussian (pp_gauss_coeffs with a sigma, csrc/emap_postprocess.cuh)
// for tests/test_grid_filters_cpu.py, compiled by g++.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -I<cuda>/include -o tests/native/_build/libfilters_host.so
//          tests/native/filters_host.cpp
#include "../../elevation_mapping_cupy_b200/csrc/emap_postprocess.cuh"

extern "C" {

void gf_gauss(int k, double sigma, float* out) { pp_gauss_coeffs(k, out, sigma); }

}  // extern "C"
