// tests/native/sdf_host.cpp -- TEST HELPER: the per-line and per-point functions of csrc/emap_sdf.cuh (the same inline
// functions the kernels call, one thread in place of a CTA) compiled for the CPU, so that envelopes, whole fields and
// queries can be compared with brute force and tests/sdf_oracle.py.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -I<cuda>/include -o tests/native/_build/libsdf_host.so
//          tests/native/sdf_host.cpp
#include <vector>

#include "../../elevation_mapping_cupy_b200/csrc/emap_sdf.cuh"

namespace {
struct Plain {
  const int32_t* f;
  int32_t operator()(int i) const { return f[i]; }
};

// One pass over a line of signed values, evaluated in `parts` contiguous parts as the CTA's threads split it
void line_pass(const int32_t* s, int n, int parts, int32_t* out) {
  std::vector<int16_t> va(n > 0 ? n : 1), vb(n > 0 ? n : 1);
  const int ma = sdf_envelope(SdfToOccupied{s}, n, va.data()), mb = sdf_envelope(SdfToFree{s}, n, vb.data());
  for (int p = 0; p < parts; p++) {
    const int q0 = (int)((int64_t)n * p / parts), q1 = (int)((int64_t)n * (p + 1) / parts);
    sdf_line_part(s, va.data(), ma, vb.data(), mb, q0, q1, [&](int q, int32_t v) { out[q] = v; });
  }
}
}  // namespace

extern "C" {

// min over p of (q - p)^2 + f[p] (f[p] = SDF_INF: not a site) for every q, in `parts` parts; returns the envelope's
// number of sites
int sdfh_envelope(const int32_t* f, int n, int parts, int32_t* out) {
  std::vector<int16_t> v(n > 0 ? n : 1);
  const Plain F{f};
  const int m = sdf_envelope(F, n, v.data());
  for (int p = 0; p < parts; p++) {
    const int q0 = (int)((int64_t)n * p / parts), q1 = (int)((int64_t)n * (p + 1) / parts);
    int k = sdf_envelope_find(F, v.data(), m, q0);
    for (int q = q0; q < q1; q++) out[q] = sdf_envelope_at(F, v.data(), m, q, k);
  }
  return m;
}

// one signed pass over a line (both fields)
void sdfh_line(const int32_t* s, int n, int parts, int32_t* out) { line_pass(s, n, parts, out); }

// the top slice of a column
int sdfh_top(float e, double z_min, double res, int n_z) { return sdf_top(e, z_min, res, n_z); }

// emap_signed_distance_field's volume for a host grid: the same three steps as the kernels, one line at a time
void sdfh_field(const float* grid, int rows, int cols, double z_min, int n_z, double res, float* out) {
  const int64_t cells = (int64_t)rows * cols;
  uint32_t key = SDF_KEY_NONE;
  for (int64_t i = 0; i < cells; i++)
    if (std::fabs(grid[i]) <= FLT_MAX && sdf_key(grid[i]) < key) key = sdf_key(grid[i]);
  const float fill = sdf_fill(key);
  int32_t* vol = (int32_t*)out;
  std::vector<int32_t> s(rows > cols ? rows : cols), o(rows > cols ? rows : cols);
  for (int k = 0; k < n_z; k++)
    for (int r = 0; r < rows; r++) {
      for (int c = 0; c < cols; c++) {
        float e = grid[(int64_t)r * cols + c];
        if (!(std::fabs(e) <= FLT_MAX)) e = fill;
        s[c] = sdf_z_value(sdf_top(e, z_min, res, n_z), k, n_z);
      }
      line_pass(s.data(), cols, SDF_LINE_THREADS, vol + ((int64_t)k * rows + r) * cols);
    }
  for (int k = 0; k < n_z; k++)
    for (int c = 0; c < cols; c++) {
      int32_t* col = vol + (int64_t)k * rows * cols + c;
      for (int r = 0; r < rows; r++) s[r] = col[(int64_t)r * cols];
      line_pass(s.data(), rows, SDF_LINE_THREADS, o.data());
      for (int r = 0; r < rows; r++) ((float*)col)[(int64_t)r * cols] = sdf_metres(o[r], (float)res);
    }
}

// emap_sdf_values' outputs (4 doubles per point)
void sdfh_values(const float* vol, int rows, int cols, int n_z, const double* position, double res, double z_min,
                 int64_t n, const double* points, double* out) {
  SdfVol f;
  f.data = vol;
  f.rows = rows;
  f.cols = cols;
  f.n_z = n_z;
  f.pos[0] = position[0];
  f.pos[1] = position[1];
  f.res = res;
  f.z_min = z_min;
  for (int64_t q = 0; q < n; q++) sdf_value(f, points[3 * q], points[3 * q + 1], points[3 * q + 2], out + 4 * q);
}
}
