// emap_semantic.cuh -- point-channel semantic fusion of a frame (SURVEY 8(f)2), sm_90a.
//
// Reference: semantic_map.py:223-259 (update_layers_pointcloud, called from elevation_mapping.py:371 right after
// average_map_kernel), fusion/pointcloud_average.py:22-113, fusion/pointcloud_class_average.py, and
// fusion/pointcloud_color.py:15-152.  There, each fusion algorithm launches a scatter kernel over
// (point, channel) -- float atomicAdd of the feature into new_map[layer] for every valid + inside point, or r/g/b/count
// integer sums for a colour channel -- and a dense kernel over (cell, channel) that writes the layer from the sums and
// the frame's fused-point count new_map[2] (CK.py:185).
// Here: ONE scatter kernel over the frame's points for all channels of all three algorithms (it reads the packed
// (idx, valid, inside) record k_index_error left on the device and the feature columns of the caller's cloud), and ONE
// per-cell kernel, both inside the frame (after k_fuse, before k_finalize re-zeroes the counts).  Float sums are
// accumulated in 2^-32 fixed point like the height sums: order-independent, deterministic, within one rounding of any
// order of the reference's float atomics.
#pragma once
#include "emap_device.cuh"

enum { SEM_AVERAGE = 0, SEM_CLASS_AVERAGE = 1, SEM_COLOR = 2 };
#define SEM_MAX_CH 16

struct SemCfg {
  int n_ch;                      // channels fused this frame (0: semantic fusion off)
  int col[SEM_MAX_CH];           // column of the feature in a cloud row (>= 3)
  int kind[SEM_MAX_CH];          // SEM_*
  int layer[SEM_MAX_CH];         // layer of semantic_map the channel writes
  int slot[SEM_MAX_CH];          // scratch slot: i64 sum plane (average kinds) / first of 4 u32 planes (colour)
  double alpha;                  // parameter.py:163 average_weight (class_average)
};

// scatter: fusion/pointcloud_average.py:41-52 (sum_kernel), fusion/pointcloud_color.py:51-61 (add_color_kernel)
template <typename T>
__global__ void __launch_bounds__(256)
k_sem_sum(const DevCfg c, const SemCfg sc, const T* __restrict__ pts, const i64 n, const i64 stride,
          const int* __restrict__ pidx, i64* __restrict__ fsum, u32* __restrict__ csum) {
  const i64 i = blockIdx.x * (i64)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int rec = pidx[i];
  if ((rec & (PT_VALID | PT_INSIDE | PT_SKIP)) != (PT_VALID | PT_INSIDE)) return;     // `if (valid) if (inside)`
  const int idx = rec & PT_IDX_MASK;
  const T* row = pts + i * stride;
  const size_t C = (size_t)c.C;
  for (int k = 0; k < sc.n_ch; k++) {
    const float feat = (float)row[sc.col[k]];                     // points_all is float32 (EM.py:456)
    if (sc.kind[k] == SEM_COLOR) {
      const u32 color = __float_as_uint(feat);                    // pointcloud_color.py:56-60
      u32* p = csum + (size_t)sc.slot[k] * C + idx;
      atomicAdd(p, (color >> 16) & 0xffu);
      atomicAdd(p + C, (color >> 8) & 0xffu);
      atomicAdd(p + 2 * C, color & 0xffu);
      atomicAdd(p + 3 * C, 1u);
    } else {
      atomicAdd((u64*)(fsum + (size_t)sc.slot[k] * C + idx), (u64)fix32(feat));
    }
  }
}

// per cell: pointcloud_average.py:71-79 (average_kernel), pointcloud_class_average.py (class_average_kernel),
// pointcloud_color.py:97-116 (color_average_kernel); re-zeroes the scratch it consumed.
__global__ void __launch_bounds__(256)
k_sem_apply(const DevCfg c, const SemCfg sc, const u64* __restrict__ cnt_fo, i64* __restrict__ fsum, u32* __restrict__ csum,
            float* __restrict__ semantic_map) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const size_t C = (size_t)c.C;
  const float cnt = (float)(u32)cnt_fo[i];                        // new_elmap[get_map_idx(id, 2)]: the frame's fused count
  for (int k = 0; k < sc.n_ch; k++) {
    float* out = semantic_map + (size_t)sc.layer[k] * C + i;
    if (sc.kind[k] == SEM_COLOR) {
      u32* p = csum + (size_t)sc.slot[k] * C + i;
      const u32 n = p[3 * C];
      if (n > 0) {
        const u32 r = p[0] / n, g = p[C] / n, b = p[2 * C] / n;
        *out = __uint_as_float((r << 16) + (g << 8) + b);
        p[0] = 0; p[C] = 0; p[2 * C] = 0; p[3 * C] = 0;
      }
      continue;
    }
    i64* sp = fsum + (size_t)sc.slot[k] * C + i;
    const i64 sfix = *sp;
    if (sfix != 0) *sp = 0;
    if (!(cnt > 0.f)) continue;
    const float sum = (float)unfix32(sfix);                       // newmap[...] as the float the reference holds
    if (sc.kind[k] == SEM_AVERAGE) {
      *out = __fdiv_rn(sum, __fmul_rn(1.0f, cnt));                // newmap / (1*cnt)
    } else {
      const float prev = *out;
      if (prev == 0.f) *out = __fdiv_rn(sum, __fmul_rn(1.0f, cnt));
      else *out = (float)(sc.alpha * (double)prev + (1.0 - sc.alpha) * (double)sum / (double)cnt);   // literal alpha: double
    }
  }
}
