// emap_export.cuh -- the map's exported values (sm_90a): one cell of any exportable layer (export_cell), the layer
// lists of the export calls (ExportList) and k_export_multi, which exports a list in one launch.  k_submap and the
// transformed windows (emap_submap.cuh) read their cells through export_cell.
#pragma once
#include "emap_device.cuh"

// export EM.py:579-670,720-775: NaN-fill, +center_z, crop the border ring, flip both axes.
// kind: 0 elevation, 1 variance, 2 traversability, 3 time, 4 upper_bound, 5 is_upper_bound, 6..8 normal xyz,
// 10 normal_color (normal_color_value)
// kind 9: arbitrary plane with flags (bit0 fill_nan, bit1 add_z) = process_map_for_publish (EM.py:579-596)
// export_cell: the value of state cell (r, cc); export_value: of exported cell o (row-major over the (W-2)^2 output).
// COLOUR: whether kind 10 can occur.  Only a call that asks for normal_color runs the COLOUR instantiation, so every
// other export runs the same code it ran before that kind existed.
#define EXPORT_KIND_PLANE 9
#define EXPORT_KIND_NORMAL_COLOR 10

// The bridge's addNormalColorLayer (WRAP:296-314) for one cell, restated from grid_map's colorVectorToValue
// (GridMapMath.cpp; not checked against a grid_map build): c = ((nx + 1) / 2, (ny + 1) / 2) in double, each rounded to
// float, and nz; channel = int(c * 255.0f) (float product, truncated toward zero); the value is the float whose bits
// are (r << 16) | (g << 8) | b.  A channel whose product is NaN is 0, one beyond the int32 range saturates (the
// reference's int cast is undefined there; the frame only writes unit normals, whose channels are in [-255, 255]).
__device__ __forceinline__ float normal_color_value(float nx, float ny, float nz) {
  const float cx = __double2float_rn(__dmul_rn(__dadd_rn((double)nx, 1.0), 0.5));   // x / 2.0 == x * 0.5, exactly
  const float cy = __double2float_rn(__dmul_rn(__dadd_rn((double)ny, 1.0), 0.5));
  const unsigned r = (unsigned)__float2int_rz(__fmul_rn(cx, 255.0f));
  const unsigned g = (unsigned)__float2int_rz(__fmul_rn(cy, 255.0f));
  const unsigned b = (unsigned)__float2int_rz(__fmul_rn(nz, 255.0f));
  return __uint_as_float((r << 16) | (g << 8) | b);
}
template <bool COLOUR = false>
__device__ __forceinline__ float export_cell(const DevCfg& c, const float* __restrict__ map, const float* __restrict__ normal,
                                             int r, int cc, int kind, float center_z, int only_above,
                                             const float* __restrict__ plane, int flags) {
  const int i = r * c.W + cc, C = c.C;
  const float nanv = __int_as_float(0x7fc00000);
  const float valid = map[2 * C + i], isup = map[6 * C + i], upper = map[5 * C + i];
  float v;
  switch (kind) {
    case 0: v = (valid > 0.5f) ? __fadd_rn(map[i], center_z) : nanv; break;
    case 1: v = map[C + i]; break;
    case 2: {   // EM.py:615-628: NaN where neither valid nor upper-bounded; only [3:-3] is ever defined
      const bool in33 = r >= 3 && r <= c.W - 4 && cc >= 3 && cc <= c.W - 4;
      v = (in33 && __fadd_rn(valid, isup) > 0.5f) ? map[3 * C + i] : nanv; break; }
    case 3: v = map[4 * C + i]; break;
    case 4: case 5: {
      const bool ok = only_above ? ((upper > 0.f && isup > 0.5f) || valid > 0.5f) : (valid > 0.5f || isup > 0.5f);
      v = ok ? (kind == 4 ? __fadd_rn(upper, center_z) : isup) : nanv; break; }
    case EXPORT_KIND_PLANE: {
      v = plane[i];
      if ((flags & 1) && !(valid > 0.5f)) v = nanv;
      if (flags & 2) v = __fadd_rn(v, center_z);
      break; }
    default:
      v = (COLOUR && kind == EXPORT_KIND_NORMAL_COLOR) ? normal_color_value(normal[i], normal[C + i], normal[2 * C + i])
                                                       : normal[(size_t)(kind - 6) * C + i];
      break;
  }
  return v;
}
template <bool COLOUR>
__device__ __forceinline__ float export_value(const DevCfg& c, const float* __restrict__ map, const float* __restrict__ normal,
                                              int o, int kind, float center_z, int only_above, const float* __restrict__ plane,
                                              int flags) {
  const int Wo = c.W - 2;
  const int orow = o / Wo, ocol = o - orow * Wo;
  const int r = Wo - 1 - orow + 1, cc = Wo - 1 - ocol + 1;         // flip(0), flip(1) of m[1:-1,1:-1]
  return export_cell<COLOUR>(c, map, normal, r, cc, kind, center_z, only_above, plane, flags);
}

// One launch exports a list of layers (WRAP:213-252 get_grid_map asks for several): blockIdx.y = layer.
#define EXPORT_MAX_LAYERS 24
struct ExportList { int n; int kind[EXPORT_MAX_LAYERS]; int flags[EXPORT_MAX_LAYERS]; const float* plane[EXPORT_MAX_LAYERS]; };
// Whether a list asks for normal_color: k_export_multi and k_submap run their COLOUR instantiation only then.
inline bool export_has_colour(const ExportList& L) {
  for (int k = 0; k < L.n; k++)
    if (L.kind[k] == EXPORT_KIND_NORMAL_COLOR) return true;
  return false;
}
template <bool COLOUR>
__global__ void __launch_bounds__(256)
k_export_multi(const DevCfg c, const float* __restrict__ map, const float* __restrict__ normal, float* __restrict__ out,
               const ExportList L, float center_z, int only_above) {
  const int Wo = c.W - 2;
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  const int l = blockIdx.y;
  if (o >= Wo * Wo) return;
  out[(size_t)l * Wo * Wo + o] =
      export_value<COLOUR>(c, map, normal, o, L.kind[l], center_z, only_above, L.plane[l], L.flags[l]);
}
