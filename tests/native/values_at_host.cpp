// tests/native/values_at_host.cpp -- TEST HELPER: the per-point functions of csrc/emap_values_at.cuh (va_plan and
// va_value, the same inline functions k_values_at runs, over the same VaGridSrc) compiled for the CPU, so that they can
// be compared with tests/values_at_oracle.py.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -I<cuda>/include -o tests/native/_build/libvalues_at_host.so
//          tests/native/values_at_host.cpp
#include "../../elevation_mapping_cupy_b200/csrc/emap_values_at.cuh"

extern "C" {

// emap_grid_values_at's outputs for n_layers host layers of one geometry (data: the layers back to back, each rows x
// cols row-major), one point after the other
void vah_values_at(const float* data, int n_layers, int64_t rows, int64_t cols, const double* position, double res,
                   int method, int64_t n, const double* xy, float* values, int32_t* status) {
  VaGeom g;
  g.rows = (int)rows;
  g.cols = (int)cols;
  g.res = res;
  for (int a = 0; a < 2; a++) {
    g.pos[a] = position[a];
    g.len[a] = (double)(a ? cols : rows) * res;
  }
  VaGridSrc s;
  s.n = n_layers;
  s.cols = g.cols;
  for (int k = 0; k < VA_MAX_LAYERS; k++) s.data[k] = k < n_layers ? data + (int64_t)k * rows * cols : nullptr;
  for (int64_t i = 0; i < n; i++) {
    VaPoint p;
    va_plan(g, method, xy[2 * i], xy[2 * i + 1], p);
    status[i] = p.status;
    for (int l = 0; l < n_layers; l++) values[l * n + i] = s.value(p, l);
  }
}

// the cubic-convolution weights at t
void vah_cubic_weights(double t, double* w) { va_cubic_weights(t, w); }
}
