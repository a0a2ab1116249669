// emap_handle.cuh -- the handle and the host plumbing every host source of libemap.so shares (library-internal: the C
// ABI is include/emap.h).  The host sources split the ABI by area: emap_api.cu (handle, frames, sharding, pose and
// state), emap_export_api.cu (layers, windows, planes, map clouds), emap_polygon_api.cu (polygon checks) and
// emap_plugins_api.cu (plugins, inpainting, PCA, image fusion, map initialisation).  Each includes the kernel headers of
// its own area only, so that every kernel is compiled into exactly one module; this header includes none.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include <cuda.h>                 // CUtensorMap (type only; the encoder is fetched at run time, make_post_tm)
#include <nvtx3/nvToolsExt.h>

#include "../../include/emap.h"
#include "emap_plan.cuh"
#include "emap_sources.cuh"

struct emap_handle;

// Owner of one allocation of n elements of T, in device memory or (PINNED) in page-locked host memory: freed with its
// owner; grown by replacing it (grow() below for device memory).  Reads as a T* in kernel launches and pointer arithmetic.
template <typename T, bool PINNED = false>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { reset(); }
  operator T*() const { return p_; }
  size_t size() const { return n_; }
  cudaError_t alloc(size_t n) {
    reset();
    const cudaError_t e = PINNED ? cudaHostAlloc((void**)&p_, sizeof(T) * n, cudaHostAllocDefault)
                                 : cudaMalloc(&p_, sizeof(T) * n);
    if (e == cudaSuccess) n_ = n; else p_ = nullptr;
    return e;
  }
  void reset() {
    if (p_) PINNED ? cudaFreeHost(p_) : cudaFree(p_);
    p_ = nullptr; n_ = 0;
  }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

template <typename T>
using PinnedBuf = DevBuf<T, true>;

// Owner of one stream or event: destroyed with its owner.  Reads as the raw cudaStream_t / cudaEvent_t.
template <typename H, cudaError_t (*Create)(H*, unsigned), cudaError_t (*Destroy)(H)>
class CudaHandle {
 public:
  CudaHandle() = default;
  CudaHandle(const CudaHandle&) = delete;
  CudaHandle& operator=(const CudaHandle&) = delete;
  ~CudaHandle() { if (h_) Destroy(h_); }
  operator H() const { return h_; }
  cudaError_t create(unsigned flags) { return Create(&h_, flags); }

 private:
  H h_ = nullptr;
};
using Stream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;
using Event = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;

struct StageTimer {
  Event ev[9];
  bool have = false;
};

// A host-to-device upload through pinned staging, each buffer grown to the largest upload: the device copy kernels
// read, its staging, and the event after which the staging may be overwritten.
struct StagedUpload {
  DevBuf<char> dev;
  PinnedBuf<char> host;
  Event staged;
  int room(emap_handle* h, size_t n);      // both buffers hold n bytes, and the previous upload has left the staging
  int send(emap_handle* h, size_t n);      // queues the upload of the first n staged bytes on the handle's stream
};

// The per-call scratch of one call family: the device block its kernels carve, the upload of its host inputs
// (stage_inputs, or room / send where a call builds its upload in the staging) and the pinned staging its host outputs
// come back through (read_back).  Each buffer grows to the family's largest call.
struct Staging {
  DevBuf<char> block;
  StagedUpload up;
  PinnedBuf<char> down;
};

// The input of a frame: where its kernels read every sensor's points, and when the caller may reuse its host memory.
// A frame describes it (kind, rows, the caller's buffers); stage() makes the buffers readable by the kernels, each()
// hands every sensor's point source to a launch, read_done() follows each pass that reads them, and wait_free()
// returns once the caller may reuse them.
struct FrameInput {
  enum Kind { F32_ROWS, F64_ROWS, DEPTH };
  enum Residence { DEVICE, STAGED, ZERO_COPY };    // the caller's device memory, a staged copy, page-locked host memory
  DevBuf<char> staging[2];                         // used by alternate staged frames
  Event staging_free[2], copied, host_free;        // staging block b reusable; staged copies done; zero-copy input read
  int buf = 1;                                     // staging block of the last staged frame
  Kind kind = F32_ROWS;                // the current frame's kind and residence
  Residence res = DEVICE;
  bool read = false, held = false;     // read_done() has run; wait_free() has yet to wait
  std::vector<int64_t> n;              // rows of sensor s
  // bytes[k] bytes at bufs[k] as the caller passed them (rows: sensor s's at k = s; DEPTH: camera s's depth,
  // confidence, rgb and feature planes at k = 4s .. 4s + 3), read by the kernels at readable[k] (stage)
  std::vector<const void*> bufs, readable;
  std::vector<size_t> bytes;
  int64_t stride = 0;                  // rows: elements from one row to the next
  std::vector<DepthSource> cams;       // DEPTH: camera s, pointed at its planes by stage() (a null conf stays null)
  int stage(emap_handle* h, int is_device_ptr);
  int read_done(emap_handle* h);
  int wait_free(emap_handle* h);
  template <typename F>     // f(src, s) for the point source of every sensor s (float or double rows, or a camera)
  int each(F&& f) const {   // until one returns non-zero
    for (int s = 0; s < (int)n.size(); s++) {
      const int rc = kind == DEPTH ? f(cams[s], s)
                   : kind == F32_ROWS ? f(RowSource<float>{(const float*)readable[s], stride}, s)
                                      : f(RowSource<double>{(const double*)readable[s], stride}, s);
      if (rc) return rc;
    }
    return 0;
  }
};

// How far the current frame has come (a sharded frame's caller drives it one call at a time): none, input staged, the
// index / fusion / ray-cast pass queued, or exchange 3 took the upper-bound keys (the finish merges them back first)
enum class Progress { IDLE, BEGUN, INDEXED, FUSED, RAYS_CAST, KEYS_EXCHANGED };

// sizes of the polygon check's device block (carve_polygon): partials, column extremes, read-back bytes
struct PolySizes {
  size_t items = 0, cols = 0, down = 0;
};

struct emap_handle {
  ~emap_handle();
  emap_config cfg;
  DevCfg dc;
  FramePlan plan;             // make_plan: march table, kernel variants, shared-memory layouts
  int device = 0;
  std::mutex mu;
  std::string err;
  cudaStream_t stream = nullptr;                        // own_stream or the caller's (emap_set_stream)
  Stream own_stream, copy_stream, side_stream;
  Event ev_fork, ev_join;                               // side-stream fork / join of the deferred fusion pushes
  Event ev_order;                                       // emap_wait_for_stream / emap_stream_wait_for
  // state
  DevBuf<float> map;          // (7,W,W); the same buffer for the handle's lifetime (captured frames bind it)
  DevBuf<float> map_alt;      // shift target, copied back into map
  CUtensorMap post_tm;        // TMA descriptor of map as a (W, W, 7) fp32 tensor, box = k_post's staged tile
  DevBuf<float> normal;       // (3,W,W)
  DevBuf<float> trav_input;
  float center[3] = {0, 0, 0};        // fp32 like EM.py:61
  float base_rotation[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  // scratch
  CellScratch sc{};
  FrameScalars* fs = nullptr;
  DevBuf<char> xscratch;      // the library's exchange scratch (carve_exchange): sc's per-cell arrays + fs; empty once attached
  DevBuf<int> ukey_x;         // exchange copy of the upper-bound keys (sharded frames)
  DevBuf<float> steps;        // device march table: [0] dummy, [1 + k] = s_k, +inf padded to plan.n_tab entries
  DevBuf<unsigned short> lut;        // cell of every fp16 bit pattern (k_build_lut)
  DevBuf<unsigned short> step_cnt;   // march steps below every non-negative fp16 value (k_build_step_cnt)
  DevBuf<unsigned char> dirty;       // two marker bytes per cell of single-GPU frames, points and rays (CellScratch::dirty)
  DevBuf<float> thr;                 // CellScratch::thr
  DevBuf<u32> tmap;                  // coarse ray map of the frame: RT x RT tile maxima of thr (keys)
  // points
  FrameInput in;
  DevBuf<float4> xyzv;
  DevBuf<int> pidx;
  DevBuf<Ray> rays;           // compacted rays of the frame, one segment per sensor (at the sensor's point offset)
  DevBuf<int> ray_ctl;        // per sensor: RC_CTL ints {ray count, work-queue counters}; zero between frames (k_finalize)
  bool overlap_override = false;
  float overlap_z_override = 0.f;
  int n_sm = 132, rc_blocks_per_sm = 8;
  // last frame description
  std::vector<Pose> poses;
  std::vector<i64> offs;      // n_sensors + 1
  i64 n_points = 0, global_off = 0;
  float pos_noise = 0, ori_noise = 0;
  Progress progress = Progress::IDLE;
  bool fused_drift = false;   // single-GPU frame: no k_drift launch (k_fuse decides, k_finalize resets)
  // multicast-attached scratch (sharded frames over NVLink multicast, emap_shard_attach): the caller's symmetric block,
  // the exchange scratch then the semantic sum planes (carve_sem)
  bool attached = false;
  char* attach_base = nullptr;
  int64_t attach_bytes = 0;
  // C-side communicator of sharded frames (emap_comm_init): NCCL, loaded at run time
  void* nccl_comm = nullptr;
  int comm_rank = 0, comm_nranks = 1;
  // semantic point-channel fusion (emap_semantic_configure): caller-owned layers, library-owned per-frame sums
  SemCfg sem{};
  float* sem_map = nullptr;        // (n_layers, W, W) fp32, device, caller-owned
  DevBuf<i64> sem_fsum;            // one 2^-32 fixed-point sum plane per averaged channel
  DevBuf<u32> sem_csum;            // r, g, b, count planes per colour channel
  int sem_nf = 0, sem_nc = 0;      // the configuration's averaged and colour channels (its sum planes: sem_fsum, sem_csum)
  // class_max scratch (SemMax): per-cell words (cnt, off, occ), control words + bitmaps + U list, the per-record table
  DevBuf<u32> cm_cell, cm_ctl, cm_key, cm_flag;
  DevBuf<i64> cm_sum;
  // The per-call scratch of the other calls.  Each member belongs to one call family, is allocated on first use and is
  // grown by that family only, so a call's growth (and the host synchronisation it costs) never depends on another's.
  DevBuf<float> d_export;          // host-bound layers and windows, staged on the device (grown to the largest call)
  struct {                         // emap_get_transformed_submaps' per-cell keys (grown to the largest call, zero
    DevBuf<u32> key1;              // between calls: k_tsub_gather resets them)
    DevBuf<u64> key2;
  } tsub;
  Staging planes;                  // emap_segment_planes, the planar regions and terrain, emap_plane_decomposition:
                                   // the block carved by carve_planes, a host grid, the host outputs (carve_plane_out)
  DevBuf<char> regions;            // emap_extract_planar_regions' scratch (carve_regions), grown to the largest window
  struct {                         // emap_get_map_points / emap_get_normal_arrows: the count and offset tables, the
    DevBuf<int> table;             // kept cells' payload (grown to the largest call) and a pinned word for the count
    DevBuf<char> out;
    PinnedBuf<int> count;
  } mapcloud;
  Staging poly;                    // the polygon checks: the block carved by carve_polygon for poly_cap, the poison
  PolySizes poly_cap;              // counts, descriptors and clipped vertices (PolyStage), the results and rings
  struct {                         // min / max filter, erode, smooth and the map initialiser's dilation: four planes
    DevBuf<float> plane[4];        // and the per-iteration counters
    DevBuf<int> cnt;
  } plugin;
  struct {                         // emap_inpaint: one block carved by inpaint_scratch (zeroed once), and the
    DevBuf<char> block;            // cooperative march's grid
    int grid = 0;
  } inpaint;
  Staging inpaint_image;           // emap_inpaint_image / emap_nonlinear_interpolation: inpaint_scratch's block (and a
                                   // host-bound grid), a host image and mask or grid, the host output
  Staging filters;                 // emap_grid_filter: the block carved by carve_filter (and a host-bound output), a
                                   // host grid and mask, the host output
  DevBuf<char> pca_block;          // emap_features_pca: one device block carved by carve_pca
  Staging query;                   // emap_project_to_planar_regions: the block carved by carve_query, host tables and
                                   // queries, the host outputs
  Staging lookup;                  // the grid lookups, the point values and the distance field: the block (the
                                   // lookups' and point values' outputs, the field's fill key and host-bound volume),
                                   // host grids or a field and queries, the host outputs
  DevBuf<double> line_rows;        // emap_values_between's host-bound line offsets, then its rows
  StagedUpload img_up;             // emap_input_image with a host image
  StagedUpload init_up;            // emap_initialize_map's arrays
  // misc
  int64_t launches = 0;
  int count_rays = 0;
  int timing = 0;
  StageTimer st;
  float stage_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

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

// plain launch of a per-cell kernel (one thread per map cell) on the handle's stream
#define PER_CELL(kern, ...)                                                                       \
  do {                                                                                            \
    kern<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(__VA_ARGS__);                                 \
    LAUNCH_CHECK();                                                                               \
  } while (0)

// the head of every entry point that takes a handle: the handle's lock and device
#define ENTER(h)                                               \
  if (!(h)) return EMAP_ERR_INVALID;                           \
  std::lock_guard<std::mutex> lock_((h)->mu);                  \
  {                                                            \
    cudaError_t e_ = cudaSetDevice((h)->device);               \
    if (e_ != cudaSuccess) { (h)->err = cudaGetErrorString(e_); return EMAP_ERR_CUDA; } \
  }

inline int cdiv(i64 a, int b) { return (int)((a + b - 1) / b); }

inline int fail(emap_handle* h, int code, const char* msg) {
  if (h) h->err = msg;
  return code;
}

// Makes b hold at least n elements.  A smaller buffer is replaced by one of n + slack elements (zero-filled on the
// handle's stream if `zero`), once every stream of the handle is idle: no queued kernel or copy still uses the old one.
template <typename T>
int grow(emap_handle* h, DevBuf<T>& b, size_t n, size_t slack, bool zero) {
  if (n <= b.size()) return 0;
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaStreamSynchronize(h->copy_stream));
  CK(cudaStreamSynchronize(h->side_stream));
  CK(b.alloc(n + slack));
  if (zero) CK(cudaMemsetAsync(b, 0, sizeof(T) * b.size(), h->stream));
  return 0;
}

// Waits only for the previous upload (a staged event that was never recorded is complete; one not yet created is
// created here) and when a buffer grows.
inline int StagedUpload::room(emap_handle* h, size_t n) {
  if (!(cudaEvent_t)staged) CK(staged.create(cudaEventDisableTiming));
  CK(cudaEventSynchronize(staged));
  if (host.size() < n) CK(host.alloc(n));
  return grow(h, dev, n, 0, false);
}

inline int StagedUpload::send(emap_handle* h, size_t n) {
  CK(cudaMemcpyAsync(dev, host, n, cudaMemcpyHostToDevice, h->stream));
  CK(cudaEventRecord(staged, h->stream));
  return 0;
}

// Sequential carving of one device block into 256-byte aligned arrays (`align` bytes: packed behind the previous one).
// With a null base only the size is added up.
struct Carver {
  uintptr_t base;
  size_t bytes = 0;
  template <typename T>
  T* take(size_t n, size_t align = 256) {
    T* p = (T*)(base + bytes);
    bytes = (bytes + sizeof(T) * n + align - 1) & ~(align - 1);
    return p;
  }
};

// A call's host inputs uploaded through `up` in one copy.  The arguments are (pointer, bytes) pairs, one per input, with
// 0 bytes for an input already on the device.  The host inputs are laid out by Carver, copied into the staging and sent,
// and each of their pointers is repointed at its device copy; the caller may reuse its buffers once this returns.
inline void stage_each(Carver&, size_t&, char*, char*) {}
template <typename T, typename... More>
void stage_each(Carver& c, size_t& end, char* host, char* dev, const T*& p, size_t bytes, More&&... more) {
  if (bytes) {
    const size_t o = (size_t)c.take<char>(bytes);
    end = o + bytes;
    if (host) {
      memcpy(host + o, p, bytes);
      p = (const T*)(dev + o);
    }
  }
  stage_each(c, end, host, dev, more...);
}
template <typename... Inputs>
int stage_inputs(emap_handle* h, StagedUpload& up, Inputs&&... in) {
  Carver layout{0};
  size_t end = 0;
  stage_each(layout, end, nullptr, nullptr, in...);
  if (!end) return 0;
  if (int rc = up.room(h, end)) return rc;
  Carver c{0};
  stage_each(c, end, up.host, up.dev, in...);
  return up.send(h, end);
}

// stage_inputs for a list of n inputs known at run time: p[k] and bytes[k] as the (pointer, bytes) pairs above.
template <typename T>
int stage_input_list(emap_handle* h, StagedUpload& up, int n, const T** p, const size_t* bytes) {
  Carver layout{0};
  size_t end = 0;
  for (int k = 0; k < n; k++)
    if (bytes[k]) end = (size_t)layout.take<char>(bytes[k]) + bytes[k];
  if (!end) return 0;
  if (int rc = up.room(h, end)) return rc;
  Carver c{0};
  for (int k = 0; k < n; k++)
    if (bytes[k]) {
      const size_t o = (size_t)c.take<char>(bytes[k]);
      memcpy(up.host + o, p[k], bytes[k]);
      p[k] = (const T*)(up.dev + o);
    }
  return up.send(h, end);
}

// A call's host outputs: `bytes` of device memory at src back into s.down (grown to hold at least `room` bytes) in one
// copy and one synchronisation.  The caller takes its pieces out of s.down.
inline int read_back(emap_handle* h, Staging& s, const void* src, size_t bytes, size_t room = 0) {
  room = std::max(room, bytes);
  if (s.down.size() < room) CK(s.down.alloc(room));
  CK(cudaMemcpyAsync(s.down, src, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return 0;
}

// NVTX range around the launches of one stage or call (visible in nsys / ncu timelines; a no-op without a tool attached)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// Called across the host sources (emap_api.cu).
int clear_map(emap_handle* h);             // EM.py:119-128 clear
