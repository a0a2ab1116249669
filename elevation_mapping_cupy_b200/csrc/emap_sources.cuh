// emap_sources.cuh -- where a frame's points come from (sm_90a).
//
// The frame kernels that read the caller's input (k_index_error, k_sem_sum, k_cm_count) are templated on a point
// source: row i of the frame is `load(i, x, y, z)` (false: the row is dropped, as a NaN row of a cloud) and its extra
// channel `col` (>= 3) is `feature(i, col)`.  Every later kernel reads only the frame's own xyzv / pidx buffers.
//   RowSource<T>  the caller's cloud: rows of `stride` elements of T, xyz first (emap_input_pointcloud / _sensors)
//   DepthSource   one depth camera, read pixel by pixel with no intermediate cloud (emap_input_depth_images)
#pragma once
#include "emap_device.cuh"

#define SEM_MAX_CH 16             // semantic channels of a frame (emap_semantic_configure)

// The semantic point channels a frame fuses (emap_semantic_configure): which column of a point goes into which layer,
// and how (emap_semantic.cuh).
enum { SEM_AVERAGE = 0, SEM_CLASS_AVERAGE = 1, SEM_COLOR = 2, SEM_CLASS_BAYESIAN = 3, SEM_BAYESIAN_INFERENCE = 4,
       SEM_CLASS_MAX = 5 };

struct SemCfg {
  int n_ch;                      // channels fused this frame (0: semantic fusion off)
  int col[SEM_MAX_CH];           // column of the feature in a cloud row (>= 3)
  int kind[SEM_MAX_CH];          // SEM_*
  int layer[SEM_MAX_CH];         // layer of semantic_map the channel writes
  int slot[SEM_MAX_CH];          // scratch slot: i64 sum plane (average and bayesian kinds) / first of 4 u32 planes
                                 // (colour) / position among the class_max channels
  double alpha;                  // parameter.py:163 average_weight (class_average)
  int n_max;                     // class_max channels
  float* sigma;                  // (n_layers, W, W) variance planes of bayesian_inference, caller-owned (or null)
  int* id_max;                   // (n_id_max, W, W) class id of every class_max round, caller-owned (or null)
  int n_id_max;
};

// One point's xyz.  fp32 rows padded to 4 floats (16-byte aligned): one 128-bit read-only load per point; other
// layouts: three scalar loads (a warp's rows are contiguous, so they coalesce into the same sectors).
template <typename T>
__device__ __forceinline__ void load_point(const T* __restrict__ pts, i64 i, i64 stride, float& x, float& y, float& z) {
  const T* p = pts + i * stride;
  x = (float)p[0]; y = (float)p[1]; z = (float)p[2];
}
template <>
__device__ __forceinline__ void load_point<float>(const float* __restrict__ pts, i64 i, i64 stride, float& x, float& y, float& z) {
  const float* p = pts + i * stride;
  if (stride == 4 && (reinterpret_cast<uintptr_t>(pts) & 15) == 0) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(p));
    x = v.x; y = v.y; z = v.z;
  } else {
    x = p[0]; y = p[1]; z = p[2];
  }
}

template <typename T>
struct RowSource {
  static constexpr bool kCountsKept = false;     // every row counts as a point of the frame (NaN rows included)
  const T* pts;
  i64 stride;
  __device__ __forceinline__ bool load(i64 i, float& x, float& y, float& z) const {
    load_point(pts, i, stride, x, y, z);
    return true;
  }
  __device__ __forceinline__ float feature(i64 i, int col) const { return (float)pts[i * stride + col]; }   // EM.py:456 fp32
};

// The semantic sensor node's cloud of one depth image (sensor_processing/semantic_sensor/.../pointcloud_node.py
// create_pcl_from_image, get_coordinates, process_image), pixel i = v * width + u being row i:
//  - kept iff isfinite(d) && d > 0 && d < max_depth && (no confidence || q >= conf_min);
//  - x = fp32(((double)u - cx) * (double)d / fx), y likewise with v, cy, fy, each operation rounded once in double
//    (NumPy 2 promotes the node's float32 coordinates against the float64 P), z = d;
//  - channel 3 + j: the packed colour (r << 16) | (g << 8) | b as fp32 bits, or a feature plane, bits as they are.
// Only the kept pixels are points of the frame: k_index_error counts them (FrameScalars::nkept).
struct DepthSource {
  static constexpr bool kCountsKept = true;
  const float* depth;             // (H, W) metres
  const float* conf;              // (H, W) or null
  const unsigned char* rgb;       // (H, W, 3) or null
  const float* feat;              // (n_features, H, W) or null
  i64 plane;                      // H * W
  int width;
  float conf_min, max_depth;
  double fx, fy, cx, cy;
  u64 src[2];                     // byte j (channel 3 + j): 0 colour, k + 1 feature plane k (words, not an array of
                                  // bytes: a kernel parameter indexed at run time would be copied to local memory)
  __device__ __forceinline__ bool load(i64 i, float& x, float& y, float& z) const {
    const float d = __ldg(depth + i);
    if (!(isfinite(d) && d > 0.f && d < max_depth)) return false;
    if (conf && !(__ldg(conf + i) >= conf_min)) return false;
    const int v = (int)(i / width), u = (int)(i - (i64)v * width);
    x = __double2float_rn(__ddiv_rn(__dmul_rn(__dsub_rn((double)u, cx), (double)d), fx));
    y = __double2float_rn(__ddiv_rn(__dmul_rn(__dsub_rn((double)v, cy), (double)d), fy));
    z = d;
    return true;
  }
  __device__ __forceinline__ float feature(i64 i, int col) const {
    const int j = col - 3;
    const int s = (int)(((j < 8 ? src[0] : src[1]) >> (8 * (j & 7))) & 0xffu) - 1;
    if (s < 0) {
      const unsigned char* p = rgb + 3 * i;
      return __uint_as_float(((u32)p[0] << 16) | ((u32)p[1] << 8) | (u32)p[2]);
    }
    return __ldg(feat + (size_t)s * plane + i);
  }
};
