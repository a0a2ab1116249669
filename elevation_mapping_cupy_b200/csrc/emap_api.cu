// emap_api.cu -- C ABI of libemap.so (see include/emap.h) and host-side orchestration.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 (see elevation_mapping_cupy_b200/build.py)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include <dlfcn.h>
#include <nvtx3/nvToolsExt.h>

#include "../../include/emap.h"
#include "emap_kernels.cuh"
#include "emap_inpaint.cuh"
#include "emap_semantic.cuh"

namespace {

thread_local std::string g_create_error;

struct StageTimer {
  cudaEvent_t ev[9];
  bool have = false;
};

}  // namespace

struct emap_handle {
  emap_config cfg;
  DevCfg dc;
  int device = 0;
  std::mutex mu;
  std::string err;
  cudaStream_t stream = nullptr, copy_stream = nullptr, own_stream = nullptr, side_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;     // side-stream fork / join of the deferred fusion pushes
  cudaEvent_t ev_order = nullptr;                       // emap_wait_for_stream / emap_stream_wait_for
  // state
  float* map = nullptr;       // (7,W,W)
  float* map_alt = nullptr;   // shift target
  CUtensorMap post_tm[2];     // TMA descriptors of the two state buffers as (W, W, 7) fp32 tensors, box = k_post's staged tile
  const float* post_tm_base[2] = {nullptr, nullptr};
  float* normal = nullptr;    // (3,W,W)
  float* trav_input = nullptr;
  float center[3] = {0, 0, 0};        // fp32 like EM.py:61
  float base_rotation[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  // scratch
  CellScratch sc{};
  u32* u32_block = nullptr;   // cnt_ai (2 x u32 per cell) | cnt_fo (2 x u32 per cell) | n_ray
  i64* i64_block = nullptr;   // SH | SV | DV
  int* ukey_x = nullptr;      // exchange copy of the upper-bound keys (sharded frames)
  FrameScalars* fs = nullptr;
  float* steps = nullptr;     // device march table: [0] dummy, [1 + k] = s_k, +inf padded to n_tab entries
  int n_tab = 0;
  std::vector<float> steps_host;
  unsigned short* lut = nullptr;   // cell of every fp16 bit pattern (k_build_lut)
  unsigned short* step_cnt = nullptr;   // march steps below every non-negative fp16 value (k_build_step_cnt)
  unsigned char* dirty = nullptr;  // per-cell dirty bytes of single-GPU frames (CellScratch::dirty)
  u32* tmap = nullptr;             // coarse ray map of the frame: RT x RT tile maxima of thr (keys)
  size_t rc_smem = 0;
  RcLayout rc_lay{};
  int span_cells = 0;              // cells (per axis) one 31-step warp iteration of the march can span
  // points
  void* d_in[2] = {nullptr, nullptr};
  size_t d_in_bytes[2] = {0, 0};
  cudaEvent_t in_free[2] = {nullptr, nullptr}, copy_done = nullptr;
  int in_sel = 0;
  float4* xyzv = nullptr;
  int* pidx = nullptr;
  Ray* rays = nullptr;        // compacted rays of the frame, one segment per sensor (at the sensor's point offset)
  int* ray_ctl = nullptr;     // per sensor: RC_CTL ints {ray count, work-queue counters}; zero between frames (k_finalize)
  int ray_ctl_cap = 0;        // sensors
  bool overlap_override = false;
  float overlap_z_override = 0.f;
  i64 pt_cap = 0;
  int n_sm = 132, rc_blocks_per_sm = 8;
  // last frame description
  std::vector<Pose> poses;
  std::vector<i64> offs;      // n_sensors + 1
  i64 n_points = 0, global_off = 0;
  float pos_noise = 0, ori_noise = 0;
  int phase = 0;              // sharded-frame state machine
  bool fused_drift = false;   // single-GPU frame: no k_drift launch (k_fuse decides, k_finalize resets)
  // multicast-attached scratch (sharded frames over NVLink multicast, emap_shard_attach)
  bool attached = false;
  std::vector<const void*> pend_pts;   // device pointers of the frame's clouds (index pass deferred to phase 0)
  std::vector<int64_t> pend_n;
  int64_t pend_stride = 0;
  int pend_dtype = 0, pend_host = 0;
  bool zero_copy_pending = false;      // the index pass reads the caller's pinned host buffer: sync before returning
  // export staging
  float* d_export = nullptr;
  size_t d_export_floats = 0;
  // plugin scratch
  float* pl[4] = {nullptr, nullptr, nullptr, nullptr};
  int* pl_cnt = nullptr;
  int pl_cnt_cap = 0;
  // C-side communicator of sharded frames (emap_comm_init): NCCL, loaded at run time
  void* nccl_comm = nullptr;
  int comm_rank = 0, comm_nranks = 1;
  // semantic point-channel fusion (emap_semantic_configure): caller-owned layers, library-owned per-frame sums
  SemCfg sem{};
  float* sem_map = nullptr;        // (n_layers, W, W) fp32, device, caller-owned
  i64* sem_fsum = nullptr;         // one 2^-32 fixed-point sum plane per averaged channel
  u32* sem_csum = nullptr;         // r, g, b, count planes per colour channel
  int sem_fslots = 0, sem_cslots = 0;
  // inpainting scratch (allocated on first use): one block, carved into the arrays of InpaintView + lists + control
  void* ip_block = nullptr;
  size_t ip_bytes = 0;
  int ip_grid = 0;
  // misc
  int64_t launches = 0;
  int count_rays = 0;
  int timing = 0;
  StageTimer st;
  float stage_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

namespace {

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e_);                        \
      return EMAP_ERR_CUDA;                                                               \
    }                                                                                     \
  } while (0)

#define LAUNCH_CHECK()                                                                    \
  do {                                                                                    \
    h->launches++;                                                                        \
    cudaError_t e_ = cudaGetLastError();                                                  \
    if (e_ != cudaSuccess) {                                                              \
      h->err = std::string("kernel launch: ") + cudaGetErrorString(e_);                   \
      return EMAP_ERR_CUDA;                                                               \
    }                                                                                     \
  } while (0)

// launch with programmatic stream serialisation (PDL), see pdl_trigger / pdl_wait in emap_kernels.cuh
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(std::forward<Args>(args))...);
}
#define PDL(kern, grid, block, smem, ...)                                                         \
  do {                                                                                            \
    cudaError_t le_ = launch_pdl(kern, dim3(grid), dim3(block), (size_t)(smem), h->stream, __VA_ARGS__); \
    if (le_ != cudaSuccess) { h->err = std::string("kernel launch: ") + cudaGetErrorString(le_); return EMAP_ERR_CUDA; } \
  } while (0)

inline float h16_host(float x) { return __half2float(__float2half_rn(x)); }

inline int cdiv(i64 a, int b) { return (int)((a + b - 1) / b); }

int fail(emap_handle* h, int code, const char* msg) {
  if (h) h->err = msg;
  return code;
}

void make_pose(const float* R, const float* t_rel, Pose* q) {
  for (int i = 0; i < 9; i++) q->R16[i] = h16_host(R[i]);
  for (int i = 0; i < 3; i++) { q->t16[i] = h16_host(t_rel[i]); q->t[i] = t_rel[i]; }
}

void fill_devcfg(const emap_config& c, DevCfg& d) {
  memset(&d, 0, sizeof(d));
  d.W = c.cell_n; d.C = c.cell_n * c.cell_n;
  d.dilation = c.dilation_size; d.edge_sharpen = c.enable_edge_sharpen; d.drift_en = c.enable_drift_compensation;
  d.visibility = c.enable_visibility_cleanup; d.overlap = c.enable_overlap_clearance;
  // EM.py:87-91
  int cell_range = (int)(c.overlap_clear_range_xy / c.resolution);
  if (cell_range < 0) cell_range = 0;
  if (cell_range > c.cell_n) cell_range = c.cell_n;
  d.cell_min = c.cell_n / 2 - cell_range / 2; d.cell_max = c.cell_n / 2 + cell_range / 2;
  d.resolution = c.resolution; d.half_w = 0.5 * (double)c.cell_n;
  d.snf = c.sensor_noise_factor; d.mahal = c.mahalanobis_thresh; d.outlier_var = c.outlier_variance;
  d.inlier_var_half = c.drift_compensation_variance_inlier / 2.0; d.trav_inlier = c.traversability_inlier;
  d.wall_thresh = c.wall_num_thresh; d.min_drift_cnt = c.min_height_drift_cnt;
  d.max_ray_length = c.max_ray_length; d.cleanup_step = c.cleanup_step; d.cos_thresh = c.cleanup_cos_thresh;
  d.mvd2 = c.min_valid_distance * c.min_valid_distance; d.max_height = c.max_height_range;
  d.ramp_a = c.ramped_height_range_a; d.ramp_b = c.ramped_height_range_b; d.ramp_c = c.ramped_height_range_c;
  d.max_variance = c.max_variance; d.pos_thresh = c.position_noise_thresh; d.ori_thresh = c.orientation_noise_thresh;
  d.inv_res_f = (float)(1.0 / c.resolution); d.half_w_f = (float)(0.5 * (double)c.cell_n);
  d.c_out = (float)c.outlier_variance; d.init_var = (float)c.initial_variance;
  d.max_drift_f = (float)c.max_drift; d.drift_alpha_f = (float)c.drift_compensation_alpha;
  d.max_len16 = h16_host((float)c.max_ray_length);
  d.w_plus_half_f = (float)c.cell_n + 0.5f;
  d.res_f = (float)c.resolution;
  d.overlap_z_f = (float)c.overlap_clear_range_z; d.time_var_f = (float)c.time_variance;
  d.time_int_f = (float)c.time_interval;
  // ray-march cell table: fp16 coordinates are clamped to [-LIM, LIM], LIM = the first fp16 value >= (W/2 + 1) * resolution;
  // every value at or beyond +-LIM maps to cell W-1 / 0, so only the bit patterns [0, P) and [0x8000, 0x8000 + P) are staged
  {
    const double want = (0.5 * (double)c.cell_n + 1.0) * c.resolution;
    __half hl = __float2half_ru((float)std::min(want, 60000.0));
    unsigned short bits = __half_as_ushort(hl);
    if (bits > 0x7bff) bits = 0x7bff;
    d.lut_lim2 = ((u32)bits << 16) | bits;
    d.lut_p2 = (int)(((size_t)(bits + 1) * 2 + 15) & ~(size_t)15);
  }
}

// CK.py:203,268: the fp16 march variable, identical for every ray
void build_steps(const emap_config& c, float max_len16, std::vector<float>& out) {
  const double ray_step = c.resolution / std::sqrt(2.0);
  out.clear();
  float s = h16_host((float)ray_step);
  while (s < max_len16 && out.size() < 65535) {
    out.push_back(s);
    float nx = h16_host((float)((double)s + ray_step));
    if (!(nx > s)) break;      // fp16 spacing exceeded the step: the reference would spin forever
    s = nx;
  }
}

int ensure_points(emap_handle* h, i64 n) {
  if (n <= h->pt_cap) return 0;
  i64 cap = n + n / 4 + 1024;
  CK(cudaStreamSynchronize(h->stream));
  if (h->xyzv) cudaFree(h->xyzv);
  if (h->pidx) cudaFree(h->pidx);
  if (h->rays) cudaFree(h->rays);
  h->xyzv = nullptr; h->pidx = nullptr; h->rays = nullptr; h->pt_cap = 0;
  CK(cudaMalloc(&h->xyzv, sizeof(float4) * cap));
  CK(cudaMalloc(&h->pidx, sizeof(int) * cap));
  CK(cudaMalloc(&h->rays, sizeof(Ray) * cap));
  h->pt_cap = cap;
  return 0;
}

int ensure_in(emap_handle* h, int b, size_t bytes) {
  if (bytes <= h->d_in_bytes[b]) return 0;
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaStreamSynchronize(h->copy_stream));
  if (h->d_in[b]) cudaFree(h->d_in[b]);
  h->d_in[b] = nullptr; h->d_in_bytes[b] = 0;
  size_t cap = bytes + bytes / 4 + 4096;
  CK(cudaMalloc(&h->d_in[b], cap));
  h->d_in_bytes[b] = cap;
  return 0;
}

// NVTX range around the launches of one frame stage (visible in nsys / ncu timelines; a no-op without a tool attached)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

int stage_mark(emap_handle* h, int k) {
  if (!h->timing) return 0;
  CK(cudaEventRecord(h->st.ev[k], h->stream));
  return 0;
}

template <typename T>
int launch_index(emap_handle* h, const Pose& q, const T* pts, i64 n, i64 stride, i64 off, int sensor) {
  if (n <= 0) return 0;
  PDL(k_index_error<T>, cdiv(n, 256), 256, 0, h->dc, q, pts, n, stride, h->xyzv + off, h->pidx + off, (const float*)h->map,
      h->sc, h->fs, h->rays + off, h->ray_ctl + RC_CTL * sensor, (const unsigned short*)h->step_cnt);
  LAUNCH_CHECK();
  return 0;
}

// phase 0: upload + index/error pass for every sensor
int frame_begin(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n, int64_t row_stride,
                int dtype, int is_device_ptr, const float* R, const float* t, int64_t global_off, float pn, float on,
                bool sharded) {
  h->sc.dirty = sharded ? nullptr : h->dirty;      // sharded frames derive the marker from the all-reduced counts
  h->fused_drift = !sharded;
  if (n_sensors < 1 || row_stride < 3 || (dtype != EMAP_F32 && dtype != EMAP_F64))
    return fail(h, EMAP_ERR_INVALID, "emap_input: n_sensors >= 1, row_stride >= 3, dtype f32/f64 required");
  const size_t esz = dtype == EMAP_F32 ? 4 : 8;
  h->offs.assign(n_sensors + 1, 0);
  for (int s = 0; s < n_sensors; s++) {
    if (n[s] < 0 || (n[s] > 0 && !points[s])) return fail(h, EMAP_ERR_INVALID, "emap_input: bad point array");
    h->offs[s + 1] = h->offs[s] + n[s];
  }
  const i64 N = h->offs[n_sensors];
  if (global_off + N >= (1ll << 31)) return fail(h, EMAP_ERR_INVALID, "emap_input: more than 2^31 points in a frame");
  h->n_points = N; h->global_off = global_off; h->pos_noise = pn; h->ori_noise = on;
  int rc = ensure_points(h, N);
  if (rc) return rc;
  h->poses.resize(n_sensors);
  for (int s = 0; s < n_sensors; s++) {
    float tr[3];
    for (int k = 0; k < 3; k++) tr[k] = t[3 * s + k] - h->center[k];      // EM.py:314,333 (fp32)
    make_pose(R + 9 * s, tr, &h->poses[s]);
  }
  // frame scalars: keep mean / additive error, zero the accumulators
  if (n_sensors > h->ray_ctl_cap) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->ray_ctl) cudaFree(h->ray_ctl);
    h->ray_ctl = nullptr; h->ray_ctl_cap = 0;
    CK(cudaMalloc(&h->ray_ctl, sizeof(int) * RC_CTL * (n_sensors + 8)));
    CK(cudaMemsetAsync(h->ray_ctl, 0, sizeof(int) * RC_CTL * (n_sensors + 8), h->stream));   // ordered before the frame's kernels
    h->ray_ctl_cap = n_sensors + 8;
  }
  h->overlap_override = false;
  if (stage_mark(h, 0)) return EMAP_ERR_CUDA;
  const void* dev_pts[64];
  std::vector<const void*> dev_vec;
  const void** dp = dev_pts;
  if (n_sensors > 64) { dev_vec.resize(n_sensors); dp = dev_vec.data(); }
  // Host clouds in page-locked memory (cudaHostAlloc / cudaHostRegister / torch pin_memory) are read by the index
  // kernel directly over PCIe (zero-copy): no staging copy, no copy-engine round trip.  Pageable memory is staged.
  bool zero_copy = false;
  if (!is_device_ptr) {
    zero_copy = true;
    for (int s = 0; s < n_sensors && zero_copy; s++) {
      if (n[s] == 0) { dp[s] = points[s]; continue; }
      cudaPointerAttributes at;
      if (cudaPointerGetAttributes(&at, points[s]) != cudaSuccess || at.type != cudaMemoryTypeHost || !at.devicePointer) {
        cudaGetLastError(); zero_copy = false;
      } else dp[s] = at.devicePointer;
    }
  }
  if (is_device_ptr) {
    for (int s = 0; s < n_sensors; s++) dp[s] = points[s];
  } else if (zero_copy) {
    is_device_ptr = 1;                       // nothing to stage; the caller's buffer is read until the index pass ends
    h->zero_copy_pending = true;
  } else {
    const int b = h->in_sel; h->in_sel ^= 1;
    size_t total = 0;
    for (int s = 0; s < n_sensors; s++) total += (size_t)n[s] * row_stride * esz;
    rc = ensure_in(h, b, total);
    if (rc) return rc;
    CK(cudaStreamWaitEvent(h->copy_stream, h->in_free[b], 0));
    size_t o = 0;
    for (int s = 0; s < n_sensors; s++) {
      const size_t bytes = (size_t)n[s] * row_stride * esz;
      if (bytes) CK(cudaMemcpyAsync((char*)h->d_in[b] + o, points[s], bytes, cudaMemcpyHostToDevice, h->copy_stream));
      dp[s] = (char*)h->d_in[b] + o;
      o += bytes;
    }
    CK(cudaEventRecord(h->copy_done, h->copy_stream));
    CK(cudaStreamWaitEvent(h->stream, h->copy_done, 0));
  }
  h->pend_pts.assign(dp, dp + n_sensors);
  h->pend_n.assign(n, n + n_sensors);
  h->pend_stride = row_stride; h->pend_dtype = dtype; h->pend_host = !is_device_ptr;
  h->phase = -1;                                                   // index pass pending
  return 0;
}

// index + error-count pass of every sensor (CK.py:280-345)
int frame_index(emap_handle* h) {
  NvtxRange nv("emap:index+error");
  const int n_sensors = (int)h->pend_pts.size();
  for (int s = 0; s < n_sensors; s++) {
    int rc = h->pend_dtype == EMAP_F32
                 ? launch_index<float>(h, h->poses[s], (const float*)h->pend_pts[s], h->pend_n[s], h->pend_stride, h->offs[s], s)
                 : launch_index<double>(h, h->poses[s], (const double*)h->pend_pts[s], h->pend_n[s], h->pend_stride, h->offs[s], s);
    if (rc) return rc;
  }
  if (h->pend_host) CK(cudaEventRecord(h->in_free[h->in_sel ^ 1], h->stream));
  if (h->zero_copy_pending) CK(cudaEventRecord(h->copy_done, h->stream));      // caller's buffer is free after this point
  if (stage_mark(h, 1)) return EMAP_ERR_CUDA;
  h->phase = 1;
  return 0;
}

int frame_fuse(emap_handle* h) {
  NvtxRange nv("emap:drift+fusion");
  const float overlap_tz = h->overlap_override ? h->overlap_z_override : h->poses[0].t[2];
  if (!h->fused_drift) {
    PDL(k_drift, 1, 256, 0, h->dc, h->fs, h->pos_noise, h->ori_noise, overlap_tz, 1, h->tmap);
    LAUNCH_CHECK();
  }
  if (stage_mark(h, 2)) return EMAP_ERR_CUDA;
  if (h->fused_drift) {
    // single GPU: the drift decision is derived inside k_fuse (launched even for an empty frame: it publishes the statistics)
    PDL((k_fuse<3, 1>), std::max(1, cdiv(h->n_points, 256)), 256, 0, h->dc, h->n_points, h->global_off, (const float4*)h->xyzv,
        (const int*)h->pidx, (const float*)h->map, h->sc, (const FrameScalars*)h->fs, h->fs, h->pos_noise, h->ori_noise, overlap_tz);
    LAUNCH_CHECK();
  } else if (h->n_points > 0) {
    if (h->attached) {
      // NVLink multicast: only the counts are on the critical path; sums + last-writer keys follow on the side stream
      // (frame_rays), under the ray-cast
      PDL((k_fuse<1, 0>), cdiv(h->n_points, 256), 256, 0, h->dc, h->n_points, h->global_off, (const float4*)h->xyzv,
          (const int*)h->pidx, (const float*)h->map, h->sc, (const FrameScalars*)h->fs, h->fs, 0.f, 0.f, 0.f);
    } else {
      PDL((k_fuse<3, 0>), cdiv(h->n_points, 256), 256, 0, h->dc, h->n_points, h->global_off, (const float4*)h->xyzv,
          (const int*)h->pidx, (const float*)h->map, h->sc, (const FrameScalars*)h->fs, h->fs, 0.f, 0.f, 0.f);
    }
    LAUNCH_CHECK();
  }
  if (stage_mark(h, 3)) return EMAP_ERR_CUDA;
  h->phase = 2;
  return 0;
}

// semantic point-channel fusion of the frame (semantic_map.py:223-259 after EM.py:369-371): needs the fused counts of
// k_fuse and must run before k_finalize re-zeroes them
template <typename T>
int launch_sem_sum(emap_handle* h, const T* pts, i64 n, i64 stride, i64 off) {
  if (n <= 0) return 0;
  k_sem_sum<T><<<cdiv(n, 256), 256, 0, h->stream>>>(h->dc, h->sem, pts, n, stride, (const int*)(h->pidx + off), h->sem_fsum, h->sem_csum);
  LAUNCH_CHECK();
  return 0;
}

int frame_semantic(emap_handle* h) {
  if (h->sem.n_ch <= 0 || !h->sem_map) return 0;
  NvtxRange nv("emap:semantic");
  for (size_t s = 0; s < h->pend_pts.size(); s++) {
    int rc = h->pend_dtype == EMAP_F32
                 ? launch_sem_sum<float>(h, (const float*)h->pend_pts[s], h->pend_n[s], h->pend_stride, h->offs[s])
                 : launch_sem_sum<double>(h, (const double*)h->pend_pts[s], h->pend_n[s], h->pend_stride, h->offs[s]);
    if (rc) return rc;
  }
  // the cloud (staging buffer or the caller's pinned memory) is free only now
  if (h->pend_host) CK(cudaEventRecord(h->in_free[h->in_sel ^ 1], h->stream));
  if (h->zero_copy_pending) CK(cudaEventRecord(h->copy_done, h->stream));
  k_sem_apply<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, h->sem, (const u64*)h->sc.cnt_fo, h->sem_fsum, h->sem_csum, h->sem_map);
  LAUNCH_CHECK();
  return 0;
}

// Cells a ray of this frame can reach.  A sample is t + ray*s with |ray| <= 1 per axis and s < len <= max_len16, so it
// lies within max_len16 of the sensor on each axis; its fp16 rounding moves it by at most 2^-11 of its magnitude.
// Rows [r0, r1) x columns [c0, c1), columns aligned to `align`; union over the frame's sensors, two cells of slack.
// Tile size 2^ts: at most RT tiles per axis, and a double-size tile at least half the span of one warp iteration
// (so that an iteration starting anywhere in a double tile stays inside the 3 x 3 block k_raycast tests).
RayGrid ray_grid(const emap_handle* h, int align) {
  const int W = h->dc.W;
  int r0 = W, r1 = 0, c0 = W, c1 = 0;
  const double L = (double)h->dc.max_len16;
  for (const Pose& q : h->poses) {
    for (int ax = 0; ax < 2; ax++) {
      const double tc = (double)q.t[ax];
      const double e = (std::fabs(tc) + L) * (1.0 / 2048.0) + 1e-4;
      double lo = std::floor((tc - L - e) / h->dc.resolution + h->dc.half_w) - 2.0;
      double hi = std::floor((tc + L + e) / h->dc.resolution + h->dc.half_w) + 3.0;
      if (!(lo == lo) || !(hi == hi)) { lo = 0; hi = W; }         // NaN pose: whole map
      const int a = (int)std::min(std::max(lo, 0.0), (double)W), b = (int)std::min(std::max(hi, 0.0), (double)W);
      if (ax == 0) { r0 = std::min(r0, a); r1 = std::max(r1, b); } else { c0 = std::min(c0, a); c1 = std::max(c1, b); }
    }
  }
  RayGrid g{0, 0, 0, 0, 3, 0, 0};
  if (r1 <= r0 || c1 <= c0) return g;
  c0 = (c0 / align) * align; c1 = std::min(W, ((c1 + align - 1) / align) * align);
  g.r0 = r0; g.r1 = r1; g.c0 = c0; g.c1 = c1;
  // tiles are aligned to the map (tile = cell >> ts) and the coarse maps start at a double-tile boundary at or before
  // (r0, c0): RT tiles per axis must reach the far edge of the box from there
  for (int ts = 2;; ts++) {
    const int al = 2 << ts;
    const int r0a = (r0 / al) * al, c0a = (c0 / al) * al;
    if ((RT << ts) >= std::max(r1 - r0a, c1 - c0a) && (4 << ts) >= h->span_cells + 1) {
      g.ts = ts; g.ta = r0a >> ts; g.tb = c0a >> ts;
      break;
    }
  }
  return g;
}

int frame_rays(emap_handle* h) {
  NvtxRange nv("emap:record+raycast");
  const bool deferred = h->attached && h->n_points > 0;
  if (deferred) {   // sums + last-writer keys of the fusion: multicast pushes on the side stream, under the ray-cast
    CK(cudaEventRecord(h->ev_fork, h->stream));
    CK(cudaStreamWaitEvent(h->side_stream, h->ev_fork, 0));
    k_fuse<2, 0><<<cdiv(h->n_points, 256), 256, 0, h->side_stream>>>(h->dc, h->n_points, h->global_off, (const float4*)h->xyzv,
                                                                       (const int*)h->pidx, (const float*)h->map, h->sc,
                                                                       (const FrameScalars*)h->fs, h->fs, 0.f, 0.f, 0.f);
    LAUNCH_CHECK();
    CK(cudaEventRecord(h->ev_join, h->side_stream));
  }
  if (h->dc.visibility) {
    const int V = (h->dc.W % 4 == 0) ? 4 : 1;
    const RayGrid box = ray_grid(h, V);
    const i64 nthreads = (i64)(box.r1 - box.r0) * ((box.c1 - box.c0) / V);
    if (nthreads > 0) {
      if (V == 4) PDL(k_record<4>, cdiv(nthreads, 256), 256, 0, h->dc, (const float*)h->map, h->sc, (const FrameScalars*)h->fs, box, h->tmap);
      else PDL(k_record<1>, cdiv(nthreads, 256), 256, 0, h->dc, (const float*)h->map, h->sc, (const FrameScalars*)h->fs, box, h->tmap);
      LAUNCH_CHECK();
    }
    if (stage_mark(h, 4)) return EMAP_ERR_CUDA;
    for (size_t s = 0; s + 1 < h->offs.size(); s++) {
      const i64 n = h->offs[s + 1] - h->offs[s];
      if (n <= 0 || h->dc.n_steps == 0) continue;
      // persistent grid: enough CTAs to fill every SM, never more than one warp per possible ray
      const int grid = (int)std::min<i64>((i64)h->n_sm * h->rc_blocks_per_sm, (n + RC_THREADS / 32 - 1) / (RC_THREADS / 32));
      if (h->count_rays)
        PDL(k_raycast<true>, grid, RC_THREADS, h->rc_smem, h->dc, h->poses[s], (const Ray*)(h->rays + h->offs[s]), h->ray_ctl + RC_CTL * (int)s,
            (const float*)h->map, (const float*)h->normal, h->sc, (const float*)h->steps, h->n_tab, (const unsigned short*)h->lut, box, (const u32*)h->tmap, h->rc_lay, h->fs);
      else
        PDL(k_raycast<false>, grid, RC_THREADS, h->rc_smem, h->dc, h->poses[s], (const Ray*)(h->rays + h->offs[s]), h->ray_ctl + RC_CTL * (int)s,
            (const float*)h->map, (const float*)h->normal, h->sc, (const float*)h->steps, h->n_tab, (const unsigned short*)h->lut, box, (const u32*)h->tmap, h->rc_lay, h->fs);
      LAUNCH_CHECK();
    }
  } else if (stage_mark(h, 4)) return EMAP_ERR_CUDA;
  if (deferred) CK(cudaStreamWaitEvent(h->stream, h->ev_join, 0));   // before the cross-rank barrier that follows this phase
  if (stage_mark(h, 5)) return EMAP_ERR_CUDA;
  h->phase = 3;
  return 0;
}

size_t post_smem(const DevCfg& d) {
  const int HL = d.dilation + 3, HLX = (HL + 3) & ~3;
  const size_t plane = (size_t)(((PT_Y + 2 * HL) * (PT_X + 2 * HLX) + 31) & ~31);
  return sizeof(float) * (3 * plane + (size_t)(PT_Y + 6) * (PT_X + 6) + 2) + sizeof(unsigned long long) * (size_t)(PT_Y + 2 * HL + 2);
}

// TMA descriptor of one state buffer for k_post: tensor (x = column, y = row, z = layer), box = staged tile + halo of one
// layer; out-of-range elements are filled with zeros.  cuTensorMapEncodeTiled is fetched from the driver at run time
// (no link-time dependency on libcuda).
int make_post_tm(emap_handle* h, int which, const float* base) {
  typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static encode_fn enc = nullptr;
  if (!enc) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn)
      return fail(h, EMAP_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
    enc = (encode_fn)fn;
  }
  memset(&h->post_tm[which], 0, sizeof(CUtensorMap));
  h->post_tm_base[which] = base;
  const int W = h->dc.W;
  const int HL = h->dc.dilation + 3, HLX = (HL + 3) & ~3;
  // plain loads instead when the row pitch is not a multiple of 16 bytes, or the map is smaller than one staged box
  h->dc.post_tma = (W % 4 == 0 && W >= PT_X + 2 * HLX && W >= PT_Y + 2 * HL) ? 1 : 0;
  if (!h->dc.post_tma) return 0;
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)W, 7};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)W * W * 4};
  const cuuint32_t box[3] = {(cuuint32_t)(PT_X + 2 * HLX), (cuuint32_t)(PT_Y + 2 * HL), 1};
  const cuuint32_t es[3] = {1, 1, 1};
  const CUresult r = enc(&h->post_tm[which], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)base, dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(h, EMAP_ERR_CUDA, "cuTensorMapEncodeTiled failed");
  return 0;
}

int launch_post(emap_handle* h) {
  dim3 grid(cdiv(h->dc.W, PT_X), cdiv(h->dc.W, PT_Y));
  const size_t sm = post_smem(h->dc);
  const CUtensorMap& tm = h->post_tm[h->post_tm_base[1] == h->map ? 1 : 0];
  switch (h->dc.dilation) {
    case 1: PDL(k_post<1>, grid, 256, sm, h->dc, h->map, h->trav_input, h->normal, tm); break;
    case 2: PDL(k_post<2>, grid, 256, sm, h->dc, h->map, h->trav_input, h->normal, tm); break;
    case 3: PDL(k_post<3>, grid, 256, sm, h->dc, h->map, h->trav_input, h->normal, tm); break;
    default: PDL(k_post<0>, grid, 256, sm, h->dc, h->map, h->trav_input, h->normal, tm); break;
  }
  LAUNCH_CHECK();
  return 0;
}

int frame_finish(emap_handle* h) {
  NvtxRange nv("emap:finalize+post");
  if (h->dc.W % 4 == 0) PDL(k_finalize<4>, cdiv(h->dc.C / 4, 256), 256, 0, h->dc, h->map, h->sc, (const FrameScalars*)h->fs, h->dc.visibility, h->ray_ctl, RC_CTL * h->ray_ctl_cap, h->fused_drift ? h->fs : nullptr, h->tmap);
  else PDL(k_finalize<1>, cdiv(h->dc.C, 256), 256, 0, h->dc, h->map, h->sc, (const FrameScalars*)h->fs, h->dc.visibility, h->ray_ctl, RC_CTL * h->ray_ctl_cap, h->fused_drift ? h->fs : nullptr, h->tmap);
  LAUNCH_CHECK();
  if (stage_mark(h, 6)) return EMAP_ERR_CUDA;
  int rc = launch_post(h);
  if (rc) return rc;
  if (stage_mark(h, 7)) return EMAP_ERR_CUDA;
  h->st.have = h->timing != 0;
  h->phase = 0;
  return 0;
}

int layer_index(const char* name) {
  static const char* names[] = {"elevation", "variance", "is_valid", "traversability", "time", "upper_bound", "is_upper_bound"};
  for (int i = 0; i < 7; i++) if (!strcmp(name, names[i])) return i;
  return -1;
}

int alloc_plugin_scratch(emap_handle* h) {
  for (int i = 0; i < 4; i++) if (!h->pl[i]) CK(cudaMalloc(&h->pl[i], sizeof(float) * h->dc.C));
  return 0;
}

// upper-bound keys of a sharded frame (NCCL mode): u32 keys <-> the s32 order an int32 MIN all-reduce needs
__global__ void k_ukey_extract(int C, const u32* __restrict__ ukv, int* __restrict__ x) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  x[i] = (int)(ukv[i] ^ 0x80000000u);                    // order-preserving u32 -> s32
}
__global__ void k_ukey_merge(int C, u32* __restrict__ ukv, const int* __restrict__ x) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  ukv[i] = ((u32)x[i]) ^ 0x80000000u;
}

}  // namespace

// =============================================================================================
extern "C" {

const char* emap_last_error(const emap_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int emap_create(const emap_config* cfg, int device, emap_handle** out) {
  if (!cfg || !out) { g_create_error = "emap_create: null argument"; return EMAP_ERR_INVALID; }
  if (cfg->abi_version != EMAP_ABI_VERSION) { g_create_error = "emap_create: abi_version mismatch"; return EMAP_ERR_INVALID; }
  if (cfg->cell_n < 8 || cfg->cell_n > 2049) {
    // beyond 2049 the reference's own clamp through float16 (CK.py:22-25,45-49) stops being exact
    g_create_error = "emap_create: cell_n must be in [8, 2049]"; return EMAP_ERR_INVALID;
  }
  if (!(cfg->resolution > 0) || cfg->dilation_size < 0 || cfg->dilation_size > 8) {
    g_create_error = "emap_create: resolution > 0 and 0 <= dilation_size <= 8 required"; return EMAP_ERR_INVALID;
  }
  emap_handle* h = new emap_handle();
  h->cfg = *cfg; h->device = device;
  auto bail = [&](const char* what, cudaError_t e) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(e);
    emap_destroy(h);
    return (int)EMAP_ERR_CUDA;
  };
  cudaError_t e;
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  fill_devcfg(*cfg, h->dc);
  build_steps(*cfg, h->dc.max_len16, h->steps_host);
  h->dc.n_steps = (int)h->steps_host.size();
  h->dc.first_step = h->steps_host.empty() ? INFINITY : h->steps_host[0];
  const size_t C = (size_t)h->dc.C;
  if ((e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  h->stream = h->own_stream;
  if ((e = cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  for (int b = 0; b < 2; b++) {
    if ((e = cudaEventCreateWithFlags(&h->in_free[b], cudaEventDisableTiming)) != cudaSuccess) return bail("event", e);
    if ((e = cudaEventRecord(h->in_free[b], h->stream)) != cudaSuccess) return bail("event", e);
  }
  if ((e = cudaEventCreateWithFlags(&h->copy_done, cudaEventDisableTiming)) != cudaSuccess) return bail("event", e);
  if ((e = cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  if ((e = cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming)) != cudaSuccess) return bail("event", e);
  if ((e = cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming)) != cudaSuccess) return bail("event", e);
  if ((e = cudaEventCreateWithFlags(&h->ev_order, cudaEventDisableTiming)) != cudaSuccess) return bail("event", e);
  for (int k = 0; k < 9; k++) if ((e = cudaEventCreate(&h->st.ev[k])) != cudaSuccess) return bail("event", e);
#define ALLOC(p, bytes) if ((e = cudaMalloc(&(p), (bytes))) != cudaSuccess) return bail("cudaMalloc", e)
#define TRY(call) if ((e = (call)) != cudaSuccess) return bail(#call, e)
  ALLOC(h->map, sizeof(float) * 7 * C);
  ALLOC(h->map_alt, sizeof(float) * 7 * C);
  ALLOC(h->normal, sizeof(float) * 3 * C);
  ALLOC(h->trav_input, sizeof(float) * C);
  ALLOC(h->u32_block, sizeof(u32) * 5 * C);
  ALLOC(h->i64_block, sizeof(i64) * 3 * C);
  ALLOC(h->sc.last, sizeof(u64) * C);
  ALLOC(h->sc.rec, sizeof(uint2) * C);
  ALLOC(h->sc.thr, sizeof(float) * C);
  ALLOC(h->sc.ukv, sizeof(u32) * C);
  ALLOC(h->dirty, C + 16);
  ALLOC(h->ukey_x, sizeof(int) * C);
  ALLOC(h->fs, sizeof(FrameScalars));
  ALLOC(h->lut, sizeof(unsigned short) * 65536);
  ALLOC(h->tmap, sizeof(u32) * RT * RT);
  ALLOC(h->step_cnt, sizeof(unsigned short) * (0x7c00 + 8));
  ALLOC(h->d_export, sizeof(float) * C);
  h->d_export_floats = C;
  // march table as k_raycast reads it: [0] unused (lane 0 of the first warp iteration), [1 + k] = s_k, +inf padding up to
  // a whole number of 31-step warp iterations + one warp of over-read
  h->n_tab = (int)(((h->steps_host.size() + RC_STRIDE - 1) / RC_STRIDE) * RC_STRIDE + 64) & ~1;
  ALLOC(h->steps, sizeof(float) * h->n_tab);
#undef ALLOC
  h->sc.cnt_ai = (u64*)h->u32_block; h->sc.cnt_fo = (u64*)(h->u32_block + 2 * C); h->sc.n_ray = h->u32_block + 4 * C;
  h->sc.SH = h->i64_block; h->sc.SV = h->i64_block + C; h->sc.DV = h->i64_block + 2 * C;
  h->sc.dirty = h->dirty;
  TRY(cudaMemsetAsync(h->u32_block, 0, sizeof(u32) * 5 * C, h->stream));
  TRY(cudaMemsetAsync(h->i64_block, 0, sizeof(i64) * 3 * C, h->stream));
  TRY(cudaMemsetAsync(h->sc.last, 0, sizeof(u64) * C, h->stream));
  TRY(cudaMemsetAsync(h->sc.rec, 0, sizeof(uint2) * C, h->stream));
  TRY(cudaMemsetAsync(h->sc.thr, 0, sizeof(float) * C, h->stream));
  TRY(cudaMemsetAsync(h->sc.ukv, 0xff, sizeof(u32) * C, h->stream));      // UKEY_NONE
  TRY(cudaMemsetAsync(h->dirty, 0, C + 16, h->stream));
  TRY(cudaMemsetAsync(h->tmap, 0, sizeof(u32) * RT * RT, h->stream));
  TRY(cudaMemsetAsync(h->normal, 0, sizeof(float) * 3 * C, h->stream));
  TRY(cudaMemsetAsync(h->trav_input, 0, sizeof(float) * C, h->stream));
  TRY(cudaMemsetAsync(h->fs, 0, sizeof(FrameScalars), h->stream));
  {
    std::vector<float> tab((size_t)h->n_tab, INFINITY);
    tab[0] = NAN;       // "step -1" of lane 0 in a ray's first warp iteration: NaN -> cell (0, 0), see k_raycast
    for (size_t k = 0; k < h->steps_host.size(); k++) tab[1 + k] = h->steps_host[k];
    // pageable source: the copy is staged before the call returns, and the stream is synchronised below
    TRY(cudaMemcpyAsync(h->steps, tab.data(), sizeof(float) * tab.size(), cudaMemcpyHostToDevice, h->stream));
    TRY(cudaStreamSynchronize(h->stream));
  }
  k_build_lut<<<256, 256, 0, h->stream>>>(h->dc, h->lut);
  k_build_step_cnt<<<cdiv(0x7c01, 256), 256, 0, h->stream>>>((const float*)(h->steps + 1), h->dc.n_steps, h->step_cnt);
  k_init<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, h->map);
  h->launches += 2;
  if (make_post_tm(h, 0, h->map) || make_post_tm(h, 1, h->map_alt)) {
    g_create_error = h->err; emap_destroy(h); return EMAP_ERR_CUDA;
  }
  if (post_smem(h->dc) > 48 * 1024)
    TRY(cudaFuncSetAttribute(k_post<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)post_smem(h->dc)));
  {
    {   // one warp iteration of the march: 30 steps between its first and last new sample, in cells (+1: fp16 coordinates)
      double span = 0;
      const std::vector<float>& st = h->steps_host;
      for (size_t k = 0; k + 1 < st.size(); k++) {
        const size_t e = std::min(st.size() - 1, k + RC_STRIDE - 1);
        span = std::max(span, ((double)st[e] - (double)st[k]) / cfg->resolution);
      }
      h->span_cells = (int)std::ceil(span) + 2;
    }
    {   // shared-memory layout of k_raycast: coarse maps + march table in the gap between the two halves of the cell
        // table when they fit there, else behind the second half
      const size_t P2 = (size_t)h->dc.lut_p2;
      const size_t need = sizeof(float) * (RT * RT + (RT / 2) * (RT / 2) + (size_t)h->n_tab) + 16;
      size_t base = (P2 + 15) & ~(size_t)15, end = 65536 + P2;
      if (base + need > 65536) { base = (end + 15) & ~(size_t)15; end = base + need; }
      h->rc_lay.off_t8 = (int)base;
      h->rc_lay.off_t16 = (int)(base + sizeof(float) * RT * RT);
      h->rc_lay.off_steps = (int)(base + sizeof(float) * (RT * RT + (RT / 2) * (RT / 2)));
      h->rc_lay.off_bar = (int)((base + need - 16 + 7) & ~(size_t)7);
      h->rc_smem = end;
    }
    TRY(cudaFuncSetAttribute(k_raycast<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->rc_smem));
    TRY(cudaFuncSetAttribute(k_raycast<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->rc_smem));
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->n_sm = prop.multiProcessorCount;
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_raycast<false>, RC_THREADS, h->rc_smem) == cudaSuccess && nb > 0)
      h->rc_blocks_per_sm = nb;
    else h->rc_blocks_per_sm = 1;
  }
  TRY(cudaStreamSynchronize(h->stream));
  TRY(cudaGetLastError());
#undef TRY
  *out = h;
  return EMAP_OK;
}

static void comm_release(emap_handle* h);

int emap_destroy(emap_handle* h) {
  if (!h) return EMAP_OK;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->copy_stream) cudaStreamSynchronize(h->copy_stream);
  comm_release(h);
  if (h->attached) { h->u32_block = nullptr; h->i64_block = nullptr; h->sc.last = nullptr; h->sc.rec = nullptr; h->sc.ukv = nullptr; h->fs = nullptr; }
  void* ptrs[] = {h->map, h->map_alt, h->normal, h->trav_input, h->u32_block, h->i64_block, h->sc.last, h->sc.rec,
                  h->sc.ukv, h->ukey_x, h->fs, h->steps, h->d_export, h->d_in[0], h->d_in[1], h->xyzv, h->pidx, h->pl[0], h->pl[1],
                  h->pl[2], h->pl[3], h->pl_cnt, h->rays, h->ray_ctl, h->sc.thr, h->dirty, h->lut, h->step_cnt, h->tmap, h->ip_block, h->sem_fsum, h->sem_csum};
  for (void* p : ptrs) if (p) cudaFree(p);
  for (int b = 0; b < 2; b++) if (h->in_free[b]) cudaEventDestroy(h->in_free[b]);
  if (h->copy_done) cudaEventDestroy(h->copy_done);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  if (h->ev_order) cudaEventDestroy(h->ev_order);
  if (h->side_stream) { cudaStreamSynchronize(h->side_stream); cudaStreamDestroy(h->side_stream); }
  for (int k = 0; k < 9; k++) if (h->st.ev[k]) cudaEventDestroy(h->st.ev[k]);
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  delete h;
  return EMAP_OK;
}

#define ENTER(h)                                               \
  if (!(h)) return EMAP_ERR_INVALID;                           \
  std::lock_guard<std::mutex> lock_((h)->mu);                  \
  {                                                            \
    cudaError_t e_ = cudaSetDevice((h)->device);               \
    if (e_ != cudaSuccess) { (h)->err = cudaGetErrorString(e_); return EMAP_ERR_CUDA; } \
  }

int emap_set_traversability_weights(emap_handle* h, const float* w1, const float* w2, const float* w3, const float* w_out) {
  ENTER(h);
  if (!w1 || !w2 || !w3 || !w_out) return fail(h, EMAP_ERR_INVALID, "null weights");
  const float* wl[3] = {w1, w2, w3};
  for (int l = 0; l < 3; l++)
    for (int cp = 0; cp < 2; cp++)
      for (int j = 0; j < 9; j++) h->dc.wp[l][cp][j] = make_float2(wl[l][(2 * cp) * 9 + j], wl[l][(2 * cp + 1) * 9 + j]);
  memcpy(h->dc.wout, w_out, sizeof(float) * 12);
  return EMAP_OK;
}

int emap_input_sensors(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n, int64_t row_stride,
                       int dtype, int is_device_ptr, const float* R, const float* t, float pn, float on) {
  ENTER(h);
  if (!points || !n || !R || !t) return fail(h, EMAP_ERR_INVALID, "emap_input: null argument");
  if (h->attached) return fail(h, EMAP_ERR_STATE, "handle is attached to a sharded scratch: use the emap_shard_* calls");
  int rc = frame_begin(h, n_sensors, points, n, row_stride, dtype, is_device_ptr, R, t, 0, pn, on, false);
  if (rc) return rc;
  if ((rc = frame_index(h))) return rc;
  if ((rc = frame_fuse(h))) return rc;
  if ((rc = frame_semantic(h))) return rc;
  if ((rc = frame_rays(h))) return rc;
  if ((rc = frame_finish(h))) return rc;
  if (!is_device_ptr || h->zero_copy_pending) CK(cudaEventSynchronize(h->copy_done));   // caller may reuse its host buffers on return
  h->zero_copy_pending = false;
  return EMAP_OK;
}

int emap_input_pointcloud(emap_handle* h, const void* points, int64_t n, int64_t row_stride, int dtype, int is_device_ptr,
                          const float R[9], const float t[3], float pn, float on) {
  const void* p[1] = {points};
  int64_t nn[1] = {n};
  return emap_input_sensors(h, 1, p, nn, row_stride, dtype, is_device_ptr, R, t, pn, on);
}

// ---- semantic point-channel fusion ------------------------------------------------------------
int emap_semantic_configure(emap_handle* h, int32_t n_channels, const int32_t* column, const int32_t* kind, const int32_t* layer,
                            float* semantic_map_device, int32_t n_layers, double average_weight) {
  ENTER(h);
  if (n_channels <= 0) { h->sem.n_ch = 0; h->sem_map = nullptr; return EMAP_OK; }
  if (n_channels > SEM_MAX_CH || !column || !kind || !layer || !semantic_map_device || n_layers < 1)
    return fail(h, EMAP_ERR_INVALID, "emap_semantic_configure: 1..16 channels, non-null arrays and layer buffer");
  SemCfg c;
  memset(&c, 0, sizeof(c));
  c.n_ch = n_channels; c.alpha = average_weight;
  int nf = 0, nc = 0;
  for (int k = 0; k < n_channels; k++) {
    if (column[k] < 3 || layer[k] < 0 || layer[k] >= n_layers || kind[k] < SEM_AVERAGE || kind[k] > SEM_COLOR)
      return fail(h, EMAP_ERR_INVALID, "emap_semantic_configure: column >= 3, 0 <= layer < n_layers, kind 0..2 required");
    c.col[k] = column[k]; c.kind[k] = kind[k]; c.layer[k] = layer[k];
    c.slot[k] = (kind[k] == SEM_COLOR) ? 4 * nc++ : nf++;
  }
  const size_t C = (size_t)h->dc.C;
  if (nf > h->sem_fslots) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->sem_fsum) cudaFree(h->sem_fsum);
    h->sem_fsum = nullptr; h->sem_fslots = 0;
    CK(cudaMalloc(&h->sem_fsum, sizeof(i64) * C * nf));
    CK(cudaMemsetAsync(h->sem_fsum, 0, sizeof(i64) * C * nf, h->stream));
    h->sem_fslots = nf;
  }
  if (nc > h->sem_cslots) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->sem_csum) cudaFree(h->sem_csum);
    h->sem_csum = nullptr; h->sem_cslots = 0;
    CK(cudaMalloc(&h->sem_csum, sizeof(u32) * C * 4 * nc));
    CK(cudaMemsetAsync(h->sem_csum, 0, sizeof(u32) * C * 4 * nc, h->stream));
    h->sem_cslots = nc;
  }
  h->sem = c; h->sem_map = semantic_map_device;
  return EMAP_OK;
}

// device-resident write-back of the last frame (CK.py:260-262): packed (cell index | flags) per input row, see
// PT_* in emap_device.cuh: bits 0..23 cell index, bit 28 valid, bit 29 inside, bit 30 row skipped (NaN)
int emap_point_record_device_ptr(emap_handle* h, const int32_t** packed, int64_t* n) {
  ENTER(h);
  if (!packed || !n) return fail(h, EMAP_ERR_INVALID, "null argument");
  *packed = (const int32_t*)h->pidx; *n = h->n_points;
  return EMAP_OK;
}

// ---- sharded frame ---------------------------------------------------------------------------

int emap_shard_begin(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n, int64_t row_stride,
                     int dtype, int is_device_ptr, const float* R, const float* t, int64_t global_point_offset, float pn,
                     float on) {
  ENTER(h);
  if (!points || !n || !R || !t) return fail(h, EMAP_ERR_INVALID, "emap_shard_begin: null argument");
  int rc = frame_begin(h, n_sensors, points, n, row_stride, dtype, is_device_ptr, R, t, global_point_offset, pn, on, true);
  if (rc) return rc;
  if (!is_device_ptr && !h->zero_copy_pending) CK(cudaEventSynchronize(h->copy_done));   // staged copy done: host buffers reusable
  // multicast mode: every rank must have reset its frame scalars before anyone pushes -> the caller runs a
  // cross-rank barrier and then emap_shard_phase(h, 0); NCCL mode: index right away
  if (h->attached) return 0;
  rc = frame_index(h);
  if (!rc && h->zero_copy_pending) { CK(cudaEventSynchronize(h->copy_done)); h->zero_copy_pending = false; }
  return rc;
}

static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

int64_t emap_shard_scratch_bytes(const emap_handle* h) {
  if (!h) return EMAP_ERR_INVALID;
  const size_t C = (size_t)h->dc.C;
  return (int64_t)(al256(4 * 5 * C) + al256(8 * 3 * C) + al256(8 * C) + al256(8 * C) + al256(4 * C) + al256(sizeof(FrameScalars)));
}

int emap_shard_attach(emap_handle* h, void* local_base, void* multicast_base, int64_t bytes) {
  ENTER(h);
  if (!local_base || !multicast_base || bytes < emap_shard_scratch_bytes(h))
    return fail(h, EMAP_ERR_INVALID, "emap_shard_attach: need local + multicast base of >= emap_shard_scratch_bytes()");
  CK(cudaStreamSynchronize(h->stream));
  const size_t C = (size_t)h->dc.C;
  char* b = (char*)local_base;
  FrameScalars keep;
  CK(cudaMemcpy(&keep, h->fs, sizeof(keep), cudaMemcpyDeviceToHost));
  // the library's own scratch is released; the symmetric block (owned by the caller) replaces it
  void* old[] = {h->u32_block, h->i64_block, h->sc.last, h->sc.rec, h->sc.ukv, h->fs};
  for (void* p : old) if (p && !h->attached) cudaFree(p);
  h->u32_block = (u32*)b; b += al256(4 * 5 * C);
  h->i64_block = (i64*)b; b += al256(8 * 3 * C);
  h->sc.last = (u64*)b; b += al256(8 * C);
  h->sc.rec = (uint2*)b; b += al256(8 * C);
  h->sc.ukv = (u32*)b; b += al256(4 * C);
  h->fs = (FrameScalars*)b;
  h->sc.cnt_ai = (u64*)h->u32_block; h->sc.cnt_fo = (u64*)(h->u32_block + 2 * C); h->sc.n_ray = h->u32_block + 4 * C;
  h->sc.SH = h->i64_block; h->sc.SV = h->i64_block + C; h->sc.DV = h->i64_block + 2 * C;
  h->sc.mc_off = (i64)((char*)multicast_base - (char*)local_base);
  CK(cudaMemsetAsync(local_base, 0, (size_t)emap_shard_scratch_bytes(h), h->stream));
  CK(cudaMemsetAsync(h->sc.ukv, 0xff, sizeof(u32) * C, h->stream));
  CK(cudaMemcpyAsync(h->fs, &keep, sizeof(keep), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->attached = true;
  return EMAP_OK;
}

int emap_shard_set_overlap_z(emap_handle* h, float z_abs) {
  ENTER(h);
  if (h->phase != 1 && h->phase != -1) return fail(h, EMAP_ERR_STATE, "emap_shard_set_overlap_z must follow emap_shard_begin");
  h->overlap_override = true; h->overlap_z_override = z_abs - h->center[2];     // consumed by k_drift (phase 1)
  return EMAP_OK;
}

int emap_shard_exchange(emap_handle* h, int32_t phase, emap_exchange* out, int32_t* n_out) {
  ENTER(h);
  if (!out || !n_out || *n_out < 3) return fail(h, EMAP_ERR_INVALID, "emap_shard_exchange: need capacity >= 3");
  const i64 C = h->dc.C;
  if (phase == 1) {          // after begin: counts (CK.py:334,336) and the drift statistics (CK.py:332-333)
    if (h->phase != 1) return fail(h, EMAP_ERR_STATE, "exchange 1 must follow emap_shard_begin");
    out[0] = {h->sc.cnt_ai, 2 * C, 3};          // two 32-bit counters per cell: an int32 SUM keeps them apart
    out[1] = {&h->fs->E, 2, 0};
    *n_out = 2;
  } else if (phase == 2) {   // after fusion: sums, counts, last-writer keys
    if (h->phase != 2) return fail(h, EMAP_ERR_STATE, "exchange 2 must follow phase 1");
    out[0] = {h->sc.SH, 2 * C, 0};
    out[1] = {h->sc.cnt_fo, 2 * C, 3};
    out[2] = {h->sc.last, C, 1};
    *n_out = 3;
  } else if (phase == 3) {   // after the ray-cast: decrements, counts, upper-bound keys
    if (h->phase != 3) return fail(h, EMAP_ERR_STATE, "exchange 3 must follow phase 2");
    if (h->dc.visibility) {
      k_ukey_extract<<<cdiv(C, 256), 256, 0, h->stream>>>((int)C, h->sc.ukv, h->ukey_x);
      LAUNCH_CHECK();
      out[0] = {h->sc.DV, C, 0};
      out[1] = {h->sc.n_ray, C, 3};
      out[2] = {h->ukey_x, C, 2};
      *n_out = 3;
      h->phase = 4;
    } else *n_out = 0;
  } else return fail(h, EMAP_ERR_INVALID, "emap_shard_exchange: phase must be 1..3");
  return EMAP_OK;
}

int emap_shard_phase(emap_handle* h, int32_t phase) {
  ENTER(h);
  if (phase == 0) {
    if (h->phase != -1) return fail(h, EMAP_ERR_STATE, "phase 0 must follow emap_shard_begin on an attached handle");
    int rc0 = frame_index(h);
    if (!rc0 && h->zero_copy_pending) { CK(cudaEventSynchronize(h->copy_done)); h->zero_copy_pending = false; }
    return rc0;
  }
  if (phase == 1) {
    if (h->phase != 1) return fail(h, EMAP_ERR_STATE, "phase 1 must follow emap_shard_begin");
    return frame_fuse(h);
  }
  if (phase == 2) {
    if (h->phase != 2) return fail(h, EMAP_ERR_STATE, "phase 2 must follow phase 1");
    return frame_rays(h);
  }
  if (phase == 3) {
    if (h->phase != 3 && h->phase != 4) return fail(h, EMAP_ERR_STATE, "phase 3 must follow phase 2");
    if (h->phase == 4) {
      k_ukey_merge<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc.C, h->sc.ukv, h->ukey_x);
      LAUNCH_CHECK();
    }
    return frame_finish(h);
  }
  return fail(h, EMAP_ERR_INVALID, "emap_shard_phase: phase must be 0..3");
}

// ---- sharded frames without a host framework: NCCL through the C ABI ---------------------------------------------
// NCCL is loaded at run time (dlopen: no build- or load-time dependency); only the entry points and enum values used
// below are declared, as nccl.h 2.x defines them.
namespace {
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, emap_nccl_id, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok() const { return lib && GetUniqueId && CommInitRank && CommDestroy && AllReduce; }
};
NcclApi& nccl_api() {
  static NcclApi a;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { a.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (a.lib) break; }
    if (!a.lib) return;
    a.GetUniqueId = (int (*)(void*))dlsym(a.lib, "ncclGetUniqueId");
    a.CommInitRank = (int (*)(void**, int, emap_nccl_id, int))dlsym(a.lib, "ncclCommInitRank");
    a.CommDestroy = (int (*)(void*))dlsym(a.lib, "ncclCommDestroy");
    a.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(a.lib, "ncclAllReduce");
    a.GetErrorString = (const char* (*)(int))dlsym(a.lib, "ncclGetErrorString");
  });
  return a;
}
enum { kNcclSum = 0, kNcclMax = 2, kNcclMin = 3, kNcclInt32 = 2, kNcclInt64 = 4 };
}  // namespace

static void comm_release(emap_handle* h) {
  if (h->nccl_comm && nccl_api().ok()) { nccl_api().CommDestroy(h->nccl_comm); h->nccl_comm = nullptr; }
}

int emap_comm_unique_id(emap_nccl_id* out) {
  if (!out) return EMAP_ERR_INVALID;
  NcclApi& a = nccl_api();
  if (!a.ok()) { g_create_error = "emap_comm_unique_id: libnccl.so.2 could not be loaded"; return EMAP_ERR_STATE; }
  return a.GetUniqueId(out) == 0 ? EMAP_OK : EMAP_ERR_CUDA;
}

int emap_comm_init(emap_handle* h, const emap_nccl_id* id, int32_t rank, int32_t nranks) {
  ENTER(h);
  if (!id || nranks < 1 || rank < 0 || rank >= nranks) return fail(h, EMAP_ERR_INVALID, "emap_comm_init: bad argument");
  NcclApi& a = nccl_api();
  if (!a.ok()) return fail(h, EMAP_ERR_STATE, "emap_comm_init: libnccl.so.2 could not be loaded");
  if (h->nccl_comm) { a.CommDestroy(h->nccl_comm); h->nccl_comm = nullptr; }
  const int r = a.CommInitRank(&h->nccl_comm, nranks, *id, rank);
  if (r != 0) { h->err = std::string("ncclCommInitRank: ") + (a.GetErrorString ? a.GetErrorString(r) : "error"); h->nccl_comm = nullptr; return EMAP_ERR_CUDA; }
  h->comm_rank = rank; h->comm_nranks = nranks;
  return EMAP_OK;
}

static int comm_exchange(emap_handle* h, int phase) {
  emap_exchange ex[4];
  int32_t n = 4;
  // (emap_shard_exchange takes the handle lock itself: this helper runs with it held, so build the list directly)
  const i64 C = h->dc.C;
  if (phase == 1) { ex[0] = {h->sc.cnt_ai, 2 * C, 3}; ex[1] = {&h->fs->E, 2, 0}; n = 2; }
  else if (phase == 2) { ex[0] = {h->sc.SH, 2 * C, 0}; ex[1] = {h->sc.cnt_fo, 2 * C, 3}; ex[2] = {h->sc.last, C, 1}; n = 3; }
  else {
    if (!h->dc.visibility) return 0;
    k_ukey_extract<<<cdiv(C, 256), 256, 0, h->stream>>>((int)C, h->sc.ukv, h->ukey_x);
    LAUNCH_CHECK();
    ex[0] = {h->sc.DV, C, 0}; ex[1] = {h->sc.n_ray, C, 3}; ex[2] = {h->ukey_x, C, 2}; n = 3;
    h->phase = 4;
  }
  NcclApi& a = nccl_api();
  for (int k = 0; k < n; k++) {
    const int dt = (ex[k].kind == 0 || ex[k].kind == 1) ? kNcclInt64 : kNcclInt32;
    const int op = ex[k].kind == 1 ? kNcclMax : ex[k].kind == 2 ? kNcclMin : kNcclSum;
    const int r = a.AllReduce(ex[k].ptr, ex[k].ptr, (size_t)ex[k].count, dt, op, h->nccl_comm, h->stream);
    if (r != 0) { h->err = std::string("ncclAllReduce: ") + (a.GetErrorString ? a.GetErrorString(r) : "error"); return EMAP_ERR_CUDA; }
  }
  return 0;
}

// One sharded frame, collective over the communicator of emap_comm_init: this rank's sensors are fused into the
// replicated grid together with every other rank's (integer NCCL all-reduces between the phases; replicas stay bit-identical).
int emap_input_sensors_sharded(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n, int64_t row_stride,
                               int dtype, int is_device_ptr, const float* R, const float* t, int64_t global_point_offset,
                               float overlap_sensor_z_absolute, float pn, float on) {
  ENTER(h);
  if (!h->nccl_comm) return fail(h, EMAP_ERR_STATE, "emap_input_sensors_sharded: call emap_comm_init first");
  if (h->attached) return fail(h, EMAP_ERR_STATE, "handle is attached to a multicast scratch: use the emap_shard_* calls");
  if (!points || !n || !R || !t) return fail(h, EMAP_ERR_INVALID, "emap_input_sensors_sharded: null argument");
  int rc = frame_begin(h, n_sensors, points, n, row_stride, dtype, is_device_ptr, R, t, global_point_offset, pn, on, true);
  if (rc) return rc;
  if (!is_device_ptr && !h->zero_copy_pending) CK(cudaEventSynchronize(h->copy_done));
  if ((rc = frame_index(h))) return rc;
  if (h->zero_copy_pending) { CK(cudaEventSynchronize(h->copy_done)); h->zero_copy_pending = false; }
  h->overlap_override = true; h->overlap_z_override = overlap_sensor_z_absolute - h->center[2];
  if ((rc = comm_exchange(h, 1))) return rc;
  if ((rc = frame_fuse(h))) return rc;
  if ((rc = comm_exchange(h, 2))) return rc;
  if ((rc = frame_rays(h))) return rc;
  if ((rc = comm_exchange(h, 3))) return rc;
  if (h->phase == 4) {
    k_ukey_merge<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc.C, h->sc.ukv, h->ukey_x);
    LAUNCH_CHECK();
  }
  return frame_finish(h);
}

// ---- read-backs ------------------------------------------------------------------------------
int emap_get_point_record(emap_handle* h, int32_t* idx, uint8_t* valid, uint8_t* inside, int64_t n) {
  ENTER(h);
  if (n > h->n_points) n = h->n_points;
  std::vector<int> rec((size_t)(n > 0 ? n : 0));
  if (n > 0) CK(cudaMemcpyAsync(rec.data(), h->pidx, sizeof(int) * n, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int64_t i = 0; i < n; i++) {
    const int r = rec[i];
    if (idx) idx[i] = (r & PT_SKIP) ? -1 : (r & PT_IDX_MASK);
    if (valid) valid[i] = (r & PT_VALID) ? 1 : 0;
    if (inside) inside[i] = (r & PT_INSIDE) ? 1 : 0;
  }
  return EMAP_OK;
}

int emap_get_frame_stats(emap_handle* h, emap_frame_stats* out) {
  ENTER(h);
  if (!out) return fail(h, EMAP_ERR_INVALID, "null out");
  FrameScalars f;
  CK(cudaMemcpyAsync(&f, h->fs, sizeof(f), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  out->mean_error = f.mean_error; out->additive_mean_error = f.additive_mean_error; out->shift_applied = f.shift;
  out->error_sum = f.error_sum; out->error_cnt = f.ecnt_last; out->drift_applied = f.applied; out->drift_evaluated = f.evaluated;
  out->n_points = h->n_points; out->n_valid_points = f.nvalid_last; out->ray_steps = f.ray_steps; out->ray_visits = f.ray_visits;
  return EMAP_OK;
}

int emap_set_ray_counting(emap_handle* h, int enable) { ENTER(h); h->count_rays = enable ? 1 : 0; return EMAP_OK; }

// ---- pose / time -----------------------------------------------------------------------------
static int shift_map(emap_handle* h, int sx, int sy, double dz) {
  const int nb = cdiv(h->dc.C, 256);
  if (sx == 0 && sy == 0) {                                    // EM.py:208-209 early return, then shift_map_z
    k_shift_z<<<nb, 256, 0, h->stream>>>(h->dc, h->map, dz);
    LAUNCH_CHECK();
    return 0;
  }
  k_shift<<<nb, 256, 0, h->stream>>>(h->dc, h->map, h->map_alt, sx, sy, dz);
  LAUNCH_CHECK();
  float* t = h->map; h->map = h->map_alt; h->map_alt = t;
  return 0;
}

int emap_move_to(emap_handle* h, const double position[3], const float R[9]) {
  ENTER(h);
  if (!position) return fail(h, EMAP_ERR_INVALID, "null position");
  if (R) memcpy(h->base_rotation, R, sizeof(float) * 9);       // EM.py:162
  double delta[3];
  for (int k = 0; k < 3; k++) delta[k] = position[k] - (double)h->center[k];      // EM.py:164
  const double px = std::nearbyint(delta[0] / h->cfg.resolution), py = std::nearbyint(delta[1] / h->cfg.resolution);
  h->center[0] = (float)((double)h->center[0] + px * h->cfg.resolution);          // EM.py:165-168
  h->center[1] = (float)((double)h->center[1] + py * h->cfg.resolution);
  h->center[2] = (float)((double)h->center[2] + delta[2]);
  return shift_map(h, -(int)px, -(int)py, -delta[2]);                              // EM.py:169-170
}

int emap_move(emap_handle* h, const double d[3]) {
  ENTER(h);
  if (!d) return fail(h, EMAP_ERR_INVALID, "null delta");
  const double px = std::nearbyint(d[0] / h->cfg.resolution), py = std::nearbyint(d[1] / h->cfg.resolution);   // EM.py:147
  h->center[0] = (float)((double)h->center[0] + px * h->cfg.resolution);
  h->center[1] = (float)((double)h->center[1] + py * h->cfg.resolution);
  h->center[2] = (float)((double)h->center[2] + d[2]);
  return shift_map(h, (int)px, (int)py, -d[2]);                                    // EM.py:151-152
}

int emap_clear(emap_handle* h) {
  ENTER(h);
  k_clear<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, h->map);
  LAUNCH_CHECK();
  CK(cudaMemsetAsync(&h->fs->mean_error, 0, 2 * sizeof(float), h->stream));     // EM.py:127-128
  return EMAP_OK;
}

int emap_update_variance(emap_handle* h) {
  ENTER(h);
  k_update_variance<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, h->map);
  LAUNCH_CHECK();
  return EMAP_OK;
}

int emap_update_time(emap_handle* h) {
  ENTER(h);
  k_update_time<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, h->map);
  LAUNCH_CHECK();
  return EMAP_OK;
}

int emap_update_normal(emap_handle* h, const float* dilated) {
  ENTER(h);
  k_normal<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, dilated ? dilated : h->trav_input, h->map + 2 * (size_t)h->dc.C, h->normal);
  LAUNCH_CHECK();
  return EMAP_OK;
}

// EM.py:913-922: the device half of initialize_map, after the caller wrote the interpolated planes (emap_set_state):
// `iterations` Jacobi passes of the initialiser dilation, then upper_bound <- elevation on valid cells.
int emap_initialize_map_finish(emap_handle* h, int32_t dilation_size, int32_t iterations) {
  ENTER(h);
  if (dilation_size < 0 || dilation_size > 64 || iterations < 0 || iterations > 16)
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map_finish: 0 <= dilation_size <= 64, 0 <= iterations <= 16");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  const size_t B = sizeof(float) * (size_t)h->dc.C;
  const int nb = cdiv(h->dc.C, 256);
  const int passes = dilation_size > 0 ? iterations : 0;
  for (int it = 0; it < std::max(passes, 1); it++) {
    CK(cudaMemcpyAsync(h->pl[0], h->map, B, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaMemcpyAsync(h->pl[1], h->map + 2 * (size_t)h->dc.C, B, cudaMemcpyDeviceToDevice, h->stream));
    k_init_dilate<<<nb, 256, 0, h->stream>>>(h->dc, h->pl[0], h->pl[1], h->map, passes ? dilation_size : 0,
                                              it == std::max(passes, 1) - 1);
    LAUNCH_CHECK();
  }
  return EMAP_OK;
}

int emap_get_position(emap_handle* h, double out[3]) {
  ENTER(h);
  for (int k = 0; k < 3; k++) out[k] = h->center[k];
  return EMAP_OK;
}

// ---- export ----------------------------------------------------------------------------------
int emap_get_map_with_name(emap_handle* h, const char* name, float* out_host, int64_t n_out) {
  ENTER(h);
  if (!name || !out_host) return fail(h, EMAP_ERR_INVALID, "null argument");
  static const char* names[] = {"elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
                                "normal_x", "normal_y", "normal_z"};
  int kind = -1;
  for (int i = 0; i < 9; i++) if (!strcmp(name, names[i])) kind = i;
  if (kind < 0) { h->err = std::string("Layer ") + name + " is not in the map"; return EMAP_ERR_NOLAYER; }
  const int Wo = h->dc.W - 2;
  if (n_out != (int64_t)Wo * Wo) return fail(h, EMAP_ERR_INVALID, "output must hold (cell_n-2)^2 floats");
  k_export<<<cdiv((i64)Wo * Wo, 256), 256, 0, h->stream>>>(h->dc, h->map, h->normal, h->d_export, kind, h->center[2],
                                                              h->cfg.use_only_above_for_upper_bound, nullptr, 0);
  LAUNCH_CHECK();
  CK(cudaMemcpyAsync(out_host, h->d_export, sizeof(float) * Wo * Wo, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

int emap_export_plane(emap_handle* h, const float* plane, int fill_nan, int add_z, float* out_host, int64_t n_out) {
  ENTER(h);
  if (!plane || !out_host) return fail(h, EMAP_ERR_INVALID, "null argument");
  const int Wo = h->dc.W - 2;
  if (n_out != (int64_t)Wo * Wo) return fail(h, EMAP_ERR_INVALID, "output must hold (cell_n-2)^2 floats");
  k_export<<<cdiv((i64)Wo * Wo, 256), 256, 0, h->stream>>>(h->dc, h->map, h->normal, h->d_export, 9, h->center[2], 0, plane,
                                                              (fill_nan ? 1 : 0) | (add_z ? 2 : 0));
  LAUNCH_CHECK();
  CK(cudaMemcpyAsync(out_host, h->d_export, sizeof(float) * Wo * Wo, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

// Several layers in one launch, one device-to-host copy and one synchronisation (WRAP:213-252 get_grid_map exports a list
// of layers per call).  names[k]: a basic layer name, or NULL / a plugin layer name together with planes[k] != NULL (a (W,W)
// device plane, exported like emap_export_plane with flags[k]: bit 0 fill_nan, bit 1 add the centre height).
int emap_get_layers(emap_handle* h, int32_t n, const char* const* names, const float* const* planes, const int32_t* flags,
                    float* out_host, int64_t n_out_total) {
  ENTER(h);
  if (n < 1 || n > EXPORT_MAX_LAYERS || !out_host) return fail(h, EMAP_ERR_INVALID, "emap_get_layers: 1..24 layers, non-null output");
  static const char* basic[] = {"elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
                                "normal_x", "normal_y", "normal_z"};
  const int Wo = h->dc.W - 2;
  const size_t per = (size_t)Wo * Wo;
  if (n_out_total != (int64_t)(per * n)) return fail(h, EMAP_ERR_INVALID, "output must hold n * (cell_n-2)^2 floats");
  ExportList L;
  memset(&L, 0, sizeof(L));
  L.n = n;
  for (int k = 0; k < n; k++) {
    if (planes && planes[k]) { L.kind[k] = 9; L.plane[k] = planes[k]; L.flags[k] = flags ? flags[k] : 0; continue; }
    int kind = -1;
    if (names && names[k]) for (int i = 0; i < 9; i++) if (!strcmp(names[k], basic[i])) kind = i;
    if (kind < 0) { h->err = std::string("Layer ") + (names && names[k] ? names[k] : "(null)") + " is not in the map"; return EMAP_ERR_NOLAYER; }
    L.kind[k] = kind;
  }
  if (h->d_export_floats < per * n) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->d_export) cudaFree(h->d_export);
    h->d_export = nullptr; h->d_export_floats = 0;
    CK(cudaMalloc(&h->d_export, sizeof(float) * per * n));
    h->d_export_floats = per * n;
  }
  k_export_multi<<<dim3(cdiv((i64)per, 256), n), 256, 0, h->stream>>>(h->dc, h->map, h->normal, h->d_export, L, h->center[2],
                                                                       h->cfg.use_only_above_for_upper_bound);
  LAUNCH_CHECK();
  CK(cudaMemcpyAsync(out_host, h->d_export, sizeof(float) * per * n, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

int emap_layer_device_ptr(emap_handle* h, const char* name, void** ptr) {
  ENTER(h);
  if (!name || !ptr) return fail(h, EMAP_ERR_INVALID, "null argument");
  const size_t C = (size_t)h->dc.C;
  int li = layer_index(name);
  if (li >= 0) { *ptr = h->map + li * C; return EMAP_OK; }
  if (!strcmp(name, "elevation_map")) { *ptr = h->map; return EMAP_OK; }
  if (!strcmp(name, "normal_map") || !strcmp(name, "normal_x")) { *ptr = h->normal; return EMAP_OK; }
  if (!strcmp(name, "normal_y")) { *ptr = h->normal + C; return EMAP_OK; }
  if (!strcmp(name, "normal_z")) { *ptr = h->normal + 2 * C; return EMAP_OK; }
  if (!strcmp(name, "traversability_input")) { *ptr = h->trav_input; return EMAP_OK; }
  h->err = std::string("Layer ") + name + " is not in the map";
  return EMAP_ERR_NOLAYER;
}

int emap_exists_layer(const emap_handle* h, const char* name) {
  if (!h || !name) return 0;
  return layer_index(name) >= 0 ? 1 : 0;
}

int emap_get_state(emap_handle* h, float* map_host, float* normal_host) {
  ENTER(h);
  const size_t C = (size_t)h->dc.C;
  if (map_host) CK(cudaMemcpyAsync(map_host, h->map, sizeof(float) * 7 * C, cudaMemcpyDeviceToHost, h->stream));
  if (normal_host) CK(cudaMemcpyAsync(normal_host, h->normal, sizeof(float) * 3 * C, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

int emap_set_state(emap_handle* h, const float* map_host, const float* normal_host, const double center[3]) {
  ENTER(h);
  const size_t C = (size_t)h->dc.C;
  if (map_host) CK(cudaMemcpyAsync(h->map, map_host, sizeof(float) * 7 * C, cudaMemcpyHostToDevice, h->stream));
  if (normal_host) CK(cudaMemcpyAsync(h->normal, normal_host, sizeof(float) * 3 * C, cudaMemcpyHostToDevice, h->stream));
  if (center) for (int k = 0; k < 3; k++) h->center[k] = (float)center[k];
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

// ---- plugins ---------------------------------------------------------------------------------
static int minmax_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k,
                         int32_t iteration_n, int32_t* iterations_run, int is_max);

int emap_min_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                    int32_t* iterations_run) {
  ENTER(h);
  return minmax_filter(h, elevation, is_valid, out, k, iteration_n, iterations_run, 0);
}

int emap_max_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                    int32_t* iterations_run) {
  ENTER(h);
  return minmax_filter(h, elevation, is_valid, out, k, iteration_n, iterations_run, 1);
}

int emap_erode(emap_handle* h, const float* layer, float* out, int32_t kernel_size, int32_t iterations, int32_t reverse) {
  ENTER(h);
  if (!layer || !out || kernel_size < 1 || kernel_size > 31 || iterations < 1 || iterations > 64)
    return fail(h, EMAP_ERR_INVALID, "emap_erode: bad argument");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  if (h->pl_cnt_cap < 2) {
    if (h->pl_cnt) cudaFree(h->pl_cnt);
    h->pl_cnt = nullptr; h->pl_cnt_cap = 0;
    CK(cudaMalloc(&h->pl_cnt, sizeof(int) * 32));
    h->pl_cnt_cap = 32;
  }
  const u32 init[2] = {0xffffffffu, 0u};
  CK(cudaMemcpyAsync(h->pl_cnt, init, sizeof(init), cudaMemcpyHostToDevice, h->stream));
  const int nb = cdiv(h->dc.C, 256);
  k_layer_minmax<<<nb, 256, 0, h->stream>>>(h->dc, layer, reverse, (u32*)h->pl_cnt);
  LAUNCH_CHECK();
  const int ks = kernel_size + (iterations - 1) * (kernel_size - 1), anchor = (kernel_size / 2) * iterations;
  const float* src = layer;
  if (layer == out) {        // in-place call: erode from a copy
    CK(cudaMemcpyAsync(h->pl[0], layer, sizeof(float) * (size_t)h->dc.C, cudaMemcpyDeviceToDevice, h->stream));
    src = h->pl[0];
  }
  k_erode<<<nb, 256, 0, h->stream>>>(h->dc, src, out, ks, anchor, reverse, (const u32*)h->pl_cnt);
  LAUNCH_CHECK();
  return EMAP_OK;
}

int emap_robot_centric_elevation(emap_handle* h, const float* elevation, const float* is_valid, const float R[9], float* out,
                                 double resolution, double threshold, int32_t use_threshold) {
  ENTER(h);
  if (!elevation || !is_valid || !R || !out) return fail(h, EMAP_ERR_INVALID, "null argument");
  k_robot_centric<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, elevation, is_valid, out, R[6], R[7], R[8], resolution,
                                                              threshold, use_threshold);
  LAUNCH_CHECK();
  return EMAP_OK;
}

static int minmax_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k,
                         int32_t iteration_n, int32_t* iterations_run, int is_max) {
  if (!elevation || !is_valid || !out || k < 0 || k > 16 || iteration_n < 1)
    return fail(h, EMAP_ERR_INVALID, "emap_min_filter: bad argument");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  if (h->pl_cnt_cap < iteration_n + 1) {
    if (h->pl_cnt) cudaFree(h->pl_cnt);
    h->pl_cnt = nullptr; h->pl_cnt_cap = 0;
    CK(cudaMalloc(&h->pl_cnt, sizeof(int) * (iteration_n + 1)));
    h->pl_cnt_cap = iteration_n + 1;
  }
  const size_t B = sizeof(float) * (size_t)h->dc.C;
  float *hA = h->pl[0], *mA = h->pl[1], *hB = h->pl[2], *mB = h->pl[3];
  CK(cudaMemsetAsync(h->pl_cnt, 0, sizeof(int) * (iteration_n + 1), h->stream));
  CK(cudaMemcpyAsync(hA, elevation, B, cudaMemcpyDeviceToDevice, h->stream));      // min_filter.py:105-106
  CK(cudaMemcpyAsync(mA, is_valid, B, cudaMemcpyDeviceToDevice, h->stream));
  const int nb = cdiv(h->dc.C, 256);
  for (int it = 0; it < iteration_n; it++) {
    const bool even = (it & 1) == 0;
    k_min_filter_iter<<<nb, 256, 0, h->stream>>>(h->dc, k, is_valid, even ? hA : hB, even ? mA : mB, even ? hB : hA,
                                                  even ? mB : mA, h->pl_cnt, it, is_max);
    LAUNCH_CHECK();
  }
  k_min_filter_final<<<nb, 256, 0, h->stream>>>(h->dc, hA, mA, hB, mB, h->pl_cnt, iteration_n, out, h->pl_cnt + iteration_n);
  LAUNCH_CHECK();
  if (iterations_run) {
    CK(cudaMemcpyAsync(iterations_run, h->pl_cnt + iteration_n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}

int emap_smooth_filter(emap_handle* h, const float* in, float* out) {
  ENTER(h);
  if (!in || !out) return fail(h, EMAP_ERR_INVALID, "null argument");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  const int nb = cdiv(h->dc.C, 256);
  k_box3<<<nb, 256, 0, h->stream>>>(h->dc, in, h->pl[0], 0); LAUNCH_CHECK();
  k_box3<<<nb, 256, 0, h->stream>>>(h->dc, h->pl[0], h->pl[1], 1); LAUNCH_CHECK();
  k_box3<<<nb, 256, 0, h->stream>>>(h->dc, h->pl[1], h->pl[0], 0); LAUNCH_CHECK();
  k_box3<<<nb, 256, 0, h->stream>>>(h->dc, h->pl[0], out, 1); LAUNCH_CHECK();
  return EMAP_OK;
}

// plugins/inpainting.py:53-63: 8-bit normalisation, cv.inpaint(h, mask, 1, INPAINT_TELEA), de-normalisation -- OpenCV's
// fast-marching fill replayed on the device in parallel (emap_inpaint.cuh), bit-identical to cv2's result.
int emap_inpaint(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t method) {
  ENTER(h);
  NvtxRange nv("emap:inpaint");
  if (!elevation || !is_valid || !out) return fail(h, EMAP_ERR_INVALID, "emap_inpaint: null argument");
  if (method != 0) return fail(h, EMAP_ERR_INVALID, "emap_inpaint: only method 0 (telea) is implemented; 'ns' (Navier-Stokes) is not");
  const int W = h->dc.W, rows = W + 2, cols = W + 2;
  const size_t N = (size_t)rows * cols, C = (size_t)W * W;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  // f, ck, vc0, vc1 (u8 N) | img (u8 C) | T, Tc0, Tc1 (f32 N) | ord (u32 N) | heapA, heapB, children (int N) | ctl | em (u32 N)
  const size_t need = 4 * al(N) + al(C) + 3 * al(4 * N) + al(4 * N) + 3 * al(4 * N) + al(sizeof(InpaintCtl)) + al(4 * N);
  if (h->ip_bytes < need) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->ip_block) cudaFree(h->ip_block);
    h->ip_block = nullptr; h->ip_bytes = 0;
    CK(cudaMalloc(&h->ip_block, need));
    // once: the march loads a pixel's child fields (ck, Tc, vc) speculatively, before it knows the pixel is a child of the
    // running round; the values of non-children are never used, but they should not be uninitialised memory
    CK(cudaMemsetAsync(h->ip_block, 0, need, h->stream));
    h->ip_bytes = need;
    int nb = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_ip_march, IP_MARCH_THREADS, 0));
    if (nb < 1) return fail(h, EMAP_ERR_CUDA, "emap_inpaint: the cooperative kernel does not fit on an SM");
    h->ip_grid = h->n_sm;          // one CTA per SM: the fronts are thin, and a grid barrier costs less with fewer CTAs
  }
  char* b = (char*)h->ip_block;
  InpaintView v;
  v.rows = rows; v.cols = cols;
  v.f = (uint8_t*)b; b += al(N);
  v.ck = (uint8_t*)b; b += al(N);
  v.vc[0] = (uint8_t*)b; b += al(N);
  v.vc[1] = (uint8_t*)b; b += al(N);
  v.img = (uint8_t*)b; b += al(C);
  v.T = (float*)b; b += al(4 * N);
  v.Tc[0] = (float*)b; b += al(4 * N);
  v.Tc[1] = (float*)b; b += al(4 * N);
  v.ord = (uint32_t*)b; b += al(4 * N);
  int* heapA = (int*)b; b += al(4 * N);
  int* heapB = (int*)b; b += al(4 * N);
  int* children = (int*)b; b += al(4 * N);
  InpaintCtl* ctl = (InpaintCtl*)b; b += al(sizeof(InpaintCtl));
  v.em = (uint32_t*)b;
  InpaintCtl init;
  memset(&init, 0, sizeof(init));
  init.mm[0] = 0xffffffffu; init.mm[1] = 0u;
  CK(cudaMemcpyAsync(ctl, &init, sizeof(init), cudaMemcpyHostToDevice, h->stream));     // pageable: staged before return
  const int nbC = cdiv((i64)C, 256), nbN = cdiv((i64)N, 256);
  k_ip_minmax<<<nbC, 256, 0, h->stream>>>((int)C, elevation, is_valid, ctl); LAUNCH_CHECK();
  k_ip_init<<<nbN, 256, 0, h->stream>>>(W, elevation, is_valid, v, (const InpaintCtl*)ctl); LAUNCH_CHECK();
  k_ip_band<<<nbN, 256, 0, h->stream>>>(v, heapA, ctl); LAUNCH_CHECK();
  k_ip_band_flag<<<nbN, 256, 0, h->stream>>>(v, (const int*)heapA, ctl); LAUNCH_CHECK();
  {
    int cap = 4096;
    void* args[] = {(void*)&v, (void*)&heapA, (void*)&heapB, (void*)&children, (void*)&ctl, (void*)&cap};
    CK(cudaLaunchCooperativeKernel((const void*)k_ip_march, dim3(h->ip_grid), dim3(IP_MARCH_THREADS), args, 0, h->stream));
    h->launches++;
  }
  k_ip_finish<<<nbC, 256, 0, h->stream>>>((int)C, (const uint8_t*)v.img, elevation, out, (const InpaintCtl*)ctl); LAUNCH_CHECK();
  return EMAP_OK;
}

// rounds / Jacobi statistics of the last emap_inpaint call (diagnostics)
int emap_inpaint_stats(emap_handle* h, int32_t* rounds, int32_t* max_jacobi, int32_t* not_converged) {
  ENTER(h);
  if (!h->ip_block) return fail(h, EMAP_ERR_STATE, "emap_inpaint has not run");
  const int W = h->dc.W;
  const size_t N = (size_t)(W + 2) * (W + 2), C = (size_t)W * W;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t off = 4 * al(N) + al(C) + 3 * al(4 * N) + al(4 * N) + 3 * al(4 * N);
  InpaintCtl c;
  CK(cudaMemcpyAsync(&c, (char*)h->ip_block + off, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (rounds) *rounds = c.rounds;
  if (max_jacobi) *max_jacobi = c.max_jacobi;
  if (not_converged) *not_converged = c.not_converged;
  return EMAP_OK;
}

// ---- plumbing --------------------------------------------------------------------------------
int emap_sync(emap_handle* h) {
  ENTER(h);
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

int emap_stream(emap_handle* h, void** s) { if (!h || !s) return EMAP_ERR_INVALID; *s = (void*)h->stream; return EMAP_OK; }
int emap_set_stream(emap_handle* h, void* s) {
  ENTER(h);
  CK(cudaStreamSynchronize(h->stream));
  h->stream = s ? (cudaStream_t)s : h->own_stream;
  return EMAP_OK;
}
int emap_wait_for_stream(emap_handle* h, void* s) {
  ENTER(h);
  if ((cudaStream_t)s == h->stream) return EMAP_OK;
  CK(cudaEventRecord(h->ev_order, (cudaStream_t)s));
  CK(cudaStreamWaitEvent(h->stream, h->ev_order, 0));
  return EMAP_OK;
}
int emap_stream_wait_for(emap_handle* h, void* s) {
  ENTER(h);
  if ((cudaStream_t)s == h->stream) return EMAP_OK;
  CK(cudaEventRecord(h->ev_order, h->stream));
  CK(cudaStreamWaitEvent((cudaStream_t)s, h->ev_order, 0));
  return EMAP_OK;
}
int emap_cell_n(const emap_handle* h) { return h ? h->dc.W : EMAP_ERR_INVALID; }
int64_t emap_launch_count(const emap_handle* h) { return h ? h->launches : 0; }

int emap_enable_stage_timing(emap_handle* h, int enable) { ENTER(h); h->timing = enable ? 1 : 0; h->st.have = false; return EMAP_OK; }

int emap_get_stage_ms(emap_handle* h, float out[8]) {
  ENTER(h);
  if (!out) return fail(h, EMAP_ERR_INVALID, "null out");
  if (!h->st.have) return fail(h, EMAP_ERR_STATE, "no timed frame (emap_enable_stage_timing first)");
  CK(cudaStreamSynchronize(h->stream));
  for (int k = 0; k < 7; k++) CK(cudaEventElapsedTime(&out[k], h->st.ev[k], h->st.ev[k + 1]));
  CK(cudaEventElapsedTime(&out[7], h->st.ev[0], h->st.ev[7]));
  return EMAP_OK;
}

}  // extern "C"
