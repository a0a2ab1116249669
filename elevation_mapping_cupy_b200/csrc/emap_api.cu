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
#include "emap_polygon.cuh"
#include "emap_semantic_plugins.cuh"
#include "emap_image.cuh"
#include "emap_submap.cuh"
#include "emap_planes.cuh"
#include "emap_mapcloud.cuh"
#include "emap_initialize.cuh"

static_assert(EMAP_DEPTH_MAX_CHANNELS == SEM_MAX_CH, "emap.h and the semantic kernels disagree on the channel count");

namespace {

thread_local std::string g_create_error;

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

// sizes of the polygon check's scratch (carve_polygon): upload bytes, partials, column extremes, read-back bytes
struct PolySizes {
  size_t up = 0, items = 0, cols = 0, down = 0;
};

}  // namespace

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
  DevBuf<unsigned char> dirty;       // per-cell dirty bytes of single-GPU frames (CellScratch::dirty)
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
  // multicast-attached scratch (sharded frames over NVLink multicast, emap_shard_attach)
  bool attached = false;
  // export staging
  DevBuf<float> d_export;
  // emap_get_transformed_submaps' per-cell keys (grown to the largest call, zero between calls: k_tsub_gather resets)
  DevBuf<u32> ts_key1;
  DevBuf<u64> ts_key2;
  // emap_segment_planes' scratch (grown to the largest window): one device block carved by carve_planes
  DevBuf<char> pl_block;
  PinnedBuf<char> pl_host;    // its host output's staging: info, plane table and layers, as one copy of the block's tail
  // plugin scratch
  DevBuf<float> pl[4];
  DevBuf<int> pl_cnt;
  // C-side communicator of sharded frames (emap_comm_init): NCCL, loaded at run time
  void* nccl_comm = nullptr;
  int comm_rank = 0, comm_nranks = 1;
  // semantic point-channel fusion (emap_semantic_configure): caller-owned layers, library-owned per-frame sums
  SemCfg sem{};
  float* sem_map = nullptr;        // (n_layers, W, W) fp32, device, caller-owned
  DevBuf<i64> sem_fsum;            // one 2^-32 fixed-point sum plane per averaged channel
  DevBuf<u32> sem_csum;            // r, g, b, count planes per colour channel
  // class_max scratch (SemMax): per-cell words (cnt, off, occ), control words + bitmaps + U list, the per-record table
  DevBuf<u32> cm_cell, cm_ctl, cm_key, cm_flag;
  DevBuf<i64> cm_sum;
  // inpainting scratch (allocated on first use): one block, carved by inpaint_scratch
  DevBuf<char> ip_block;
  int ip_grid = 0;
  // polygon safety check scratch (allocated on first use, grown to the largest call): one device block carved by
  // carve_polygon, and its pinned host staging (the upload region on the way in, the read-back region on the way out)
  DevBuf<char> pg_block;
  PolySizes pg_cap{};
  PinnedBuf<char> pg_host;
  // features_pca scratch (allocated on first use): one device block carved by carve_pca
  DevBuf<char> pca_block;
  // emap_input_image with a host image (allocated on first use)
  StagedUpload img_up;
  // emap_get_map_points / emap_get_normal_arrows (allocated on first use): the count and offset tables, the kept cells'
  // payload (grown to the largest call) and a pinned word for the count
  DevBuf<int> mc_table;
  DevBuf<char> mc_out;
  PinnedBuf<int> mc_count_host;
  // emap_initialize_map's arrays (allocated on first use)
  StagedUpload init_up;
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

// plain launch of a per-cell kernel (one thread per map cell) on the handle's stream
#define PER_CELL(kern, ...)                                                                       \
  do {                                                                                            \
    kern<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(__VA_ARGS__);                                 \
    LAUNCH_CHECK();                                                                               \
  } while (0)

inline int cdiv(i64 a, int b) { return (int)((a + b - 1) / b); }

int fail(emap_handle* h, int code, const char* msg) {
  if (h) h->err = msg;
  return code;
}

void make_pose(const float* R, const float* t_rel, Pose* q) {
  for (int i = 0; i < 9; i++) q->R16[i] = h16_host(R[i]);
  for (int i = 0; i < 3; i++) { q->t16[i] = h16_host(t_rel[i]); q->t[i] = t_rel[i]; }
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

// Waits only for the previous upload (a staged event that was never recorded is complete) and when a buffer grows.
int StagedUpload::room(emap_handle* h, size_t n) {
  CK(cudaEventSynchronize(staged));
  if (host.size() < n) CK(host.alloc(n));
  return grow(h, dev, n, 0, false);
}

int StagedUpload::send(emap_handle* h, size_t n) {
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

// The per-cell exchange scratch of a frame, one block: what the ranks of a sharded frame reduce.  Carves the block at
// `base` into sc's exchanged arrays and fs; returns its size.
size_t carve_exchange(size_t C, void* base, CellScratch& sc, FrameScalars*& fs) {
  Carver b{(uintptr_t)base};
  sc.cnt_ai = b.take<u64>(C, 8); sc.cnt_fo = b.take<u64>(C, 8); sc.n_ray = b.take<u32>(C);
  sc.SH = b.take<i64>(C, 8); sc.SV = b.take<i64>(C, 8); sc.DV = b.take<i64>(C);
  sc.last = b.take<u64>(C);
  sc.rec = b.take<uint2>(C);
  sc.ukv = b.take<u32>(C);
  fs = b.take<FrameScalars>(1);
  return b.bytes;
}

size_t exchange_bytes(size_t C) {
  CellScratch sc;
  FrameScalars* fs;
  return carve_exchange(C, nullptr, sc, fs);
}

// Moves the exchange scratch of h to `base` in its between-frames state: all zero, upper-bound keys UKEY_NONE.
cudaError_t place_exchange(emap_handle* h, void* base) {
  const size_t C = (size_t)h->dc.C;
  carve_exchange(C, base, h->sc, h->fs);
  cudaError_t e = cudaMemsetAsync(base, 0, exchange_bytes(C), h->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(h->sc.ukv, 0xff, sizeof(u32) * C, h->stream);
  return e;
}

// The inpainting scratch of a W x W map, one block; N = (W + 2)^2 padded pixels.
struct InpaintScratch {
  InpaintView v;
  int* heap[2];
  int* children;
  InpaintCtl* ctl;
  size_t bytes;
};

InpaintScratch inpaint_scratch(int W, void* base) {
  const size_t N = (size_t)(W + 2) * (W + 2);
  Carver b{(uintptr_t)base};
  InpaintScratch s;
  s.v.rows = s.v.cols = W + 2;
  s.v.f = b.take<uint8_t>(N); s.v.ck = b.take<uint8_t>(N); s.v.vc[0] = b.take<uint8_t>(N); s.v.vc[1] = b.take<uint8_t>(N);
  s.v.img = b.take<uint8_t>((size_t)W * W);
  s.v.T = b.take<float>(N); s.v.Tc[0] = b.take<float>(N); s.v.Tc[1] = b.take<float>(N);
  s.v.ord = b.take<uint32_t>(N);
  s.heap[0] = b.take<int>(N); s.heap[1] = b.take<int>(N); s.children = b.take<int>(N);
  s.ctl = b.take<InpaintCtl>(1);
  s.v.em = b.take<uint32_t>(N);
  s.bytes = b.bytes;
  return s;
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

template <typename Src>
int launch_index(emap_handle* h, const Src& src, int s) {
  const i64 n = h->in.n[s], off = h->offs[s];
  if (n <= 0) return 0;
  PDL(k_index_error<Src>, cdiv(n, 256), 256, 0, h->dc, h->poses[s], src, n, h->xyzv + off, h->pidx + off,
      (const float*)h->map, h->sc, h->fs, h->rays + off, h->ray_ctl + RC_CTL * s, (const unsigned short*)h->step_cnt);
  LAUNCH_CHECK();
  return 0;
}

// Makes the frame's buffers readable by its kernels at readable[k], and points the depth cameras there.  Device
// memory is read in place.  Host buffers that are all page-locked (cudaHostAlloc / cudaHostRegister / torch pin_memory)
// are read by the kernels directly over PCIe (zero-copy): no staging copy, no copy-engine round trip.  Otherwise every
// buffer is staged, 256-byte aligned, into the staging block the last staged frame did not use, on the copy stream.
int FrameInput::stage(emap_handle* h, int is_device_ptr) {
  readable = bufs;
  res = is_device_ptr ? DEVICE : ZERO_COPY; read = false; held = !is_device_ptr;
  for (size_t k = 0; k < bufs.size() && res == ZERO_COPY; k++) {
    if (bytes[k] == 0) continue;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, bufs[k]) != cudaSuccess || at.type != cudaMemoryTypeHost || !at.devicePointer) {
      cudaGetLastError(); res = STAGED;
    } else readable[k] = at.devicePointer;
  }
  if (res == STAGED) {
    buf ^= 1;
    const auto aligned = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t total = 0;
    for (size_t b : bytes) total += aligned(b);
    if (int rc = grow(h, staging[buf], total, total / 4 + 4096, false)) return rc;
    CK(cudaStreamWaitEvent(h->copy_stream, staging_free[buf], 0));
    size_t o = 0;
    for (size_t k = 0; k < bufs.size(); k++) {
      if (bytes[k]) CK(cudaMemcpyAsync((char*)staging[buf] + o, bufs[k], bytes[k], cudaMemcpyHostToDevice, h->copy_stream));
      readable[k] = (char*)staging[buf] + o;
      o += aligned(bytes[k]);
    }
    CK(cudaEventRecord(copied, h->copy_stream));
    CK(cudaStreamWaitEvent(h->stream, copied, 0));
  }
  for (size_t s = 0; kind == DEPTH && s < cams.size(); s++) {
    const void* const* p = &readable[4 * s];
    DepthSource& d = cams[s];
    d.depth = (const float*)p[0]; d.conf = d.conf ? (const float*)p[1] : nullptr;
    d.rgb = (const unsigned char*)p[2]; d.feat = (const float*)p[3];
  }
  return 0;
}

// After a pass that reads the input: its staging block or the caller's page-locked memory is free from here on the stream
int FrameInput::read_done(emap_handle* h) {
  if (res == STAGED) CK(cudaEventRecord(staging_free[buf], h->stream));
  else if (res == ZERO_COPY) CK(cudaEventRecord(host_free, h->stream));
  read = true;
  return 0;
}

// Returns once the caller may reuse its host memory: staged input once its copy has finished, zero-copy input once its
// last reader is queued (read_done) and has run, device input at once.  No wait while the stream is captured: the
// graph reads the caller's page-locked memory at every replay.  After one wait, the frame's later calls return at once.
int FrameInput::wait_free(emap_handle* h) {
  if (!held || (res == ZERO_COPY && !read)) return 0;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CK(cudaStreamIsCapturing(h->stream, &cs));
  if (cs == cudaStreamCaptureStatusNone) CK(cudaEventSynchronize(res == STAGED ? copied : host_free));
  held = false;
  return 0;
}

// Starts a frame on the input that h->in describes: the row offsets, sensor poses and per-row buffers, then the input
// staged, with the index pass pending.  The caller has validated the rows (every n[s] >= 0, fewer than 2^31 in all).
int frame_start(emap_handle* h, int is_device_ptr, const float* R, const float* t, int64_t global_off, float pn,
                float on, bool sharded) {
  const int n_sensors = (int)h->in.n.size();
  h->sc.dirty = sharded ? nullptr : (unsigned char*)h->dirty;      // sharded frames derive the marker from the all-reduced counts
  h->fused_drift = !sharded;
  h->offs.assign(n_sensors + 1, 0);
  for (int s = 0; s < n_sensors; s++) h->offs[s + 1] = h->offs[s] + h->in.n[s];
  const i64 N = h->offs[n_sensors];
  h->n_points = N; h->global_off = global_off; h->pos_noise = pn; h->ori_noise = on;
  int rc;
  if ((rc = grow(h, h->xyzv, N, N / 4 + 1024, false)) || (rc = grow(h, h->pidx, N, N / 4 + 1024, false)) ||
      (rc = grow(h, h->rays, N, N / 4 + 1024, false)))
    return rc;
  h->poses.resize(n_sensors);
  for (int s = 0; s < n_sensors; s++) {
    float tr[3];
    for (int k = 0; k < 3; k++) tr[k] = t[3 * s + k] - h->center[k];      // EM.py:314,333 (fp32)
    make_pose(R + 9 * s, tr, &h->poses[s]);
  }
  // zero-filled on the stream: ordered before the frame's kernels
  if ((rc = grow(h, h->ray_ctl, (size_t)RC_CTL * n_sensors, RC_CTL * 8, true))) return rc;
  h->overlap_override = false;
  if (stage_mark(h, 0)) return EMAP_ERR_CUDA;
  if ((rc = h->in.stage(h, is_device_ptr))) return rc;
  h->progress = Progress::BEGUN;
  return 0;
}

// A frame of point clouds: sensor s has n[s] rows of row_stride elements of dtype at points[s]
int frame_begin(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n, int64_t row_stride,
                int dtype, int is_device_ptr, const float* R, const float* t, int64_t global_off, float pn, float on,
                bool sharded) {
  if (n_sensors < 1 || row_stride < 3 || (dtype != EMAP_F32 && dtype != EMAP_F64))
    return fail(h, EMAP_ERR_INVALID, "emap_input: n_sensors >= 1, row_stride >= 3, dtype f32/f64 required");
  const size_t esz = dtype == EMAP_F32 ? 4 : 8;
  i64 N = 0;
  for (int s = 0; s < n_sensors; s++) {
    if (n[s] < 0 || (n[s] > 0 && !points[s])) return fail(h, EMAP_ERR_INVALID, "emap_input: bad point array");
    N += n[s];
  }
  if (global_off + N >= (1ll << 31)) return fail(h, EMAP_ERR_INVALID, "emap_input: more than 2^31 points in a frame");
  FrameInput& in = h->in;
  in.kind = dtype == EMAP_F32 ? FrameInput::F32_ROWS : FrameInput::F64_ROWS; in.stride = row_stride;
  in.n.assign(n, n + n_sensors); in.bufs.assign(points, points + n_sensors); in.bytes.resize(n_sensors);
  for (int s = 0; s < n_sensors; s++) in.bytes[s] = (size_t)n[s] * row_stride * esz;
  return frame_start(h, is_device_ptr, R, t, global_off, pn, on, sharded);
}

// index + error-count pass of every sensor (CK.py:280-345)
int frame_index(emap_handle* h) {
  NvtxRange nv("emap:index+error");
  if (int rc = h->in.each([h](auto pts, int s) { return launch_index(h, pts, s); })) return rc;
  if (int rc = h->in.read_done(h)) return rc;
  if (stage_mark(h, 1)) return EMAP_ERR_CUDA;
  h->progress = Progress::INDEXED;
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
  h->progress = Progress::FUSED;
  return 0;
}

// semantic point-channel fusion of the frame (semantic_map.py:223-259 after EM.py:369-371): needs the fused counts of
// k_fuse and must run before k_finalize re-zeroes them
// the class_max scratch as the kernels see it (pointers into the handle's buffers)
SemMax sem_max(emap_handle* h) {
  const size_t C = (size_t)h->dc.C;
  SemMax m;
  m.cnt = h->cm_cell; m.off = h->cm_cell + C; m.occ = h->cm_cell + 2 * C;
  m.ctl = h->cm_ctl; m.ulist = h->cm_ctl + CM_CTL + (1 + SEM_MAX_CH) * CM_WORDS;
  m.key = h->cm_key; m.flag = h->cm_flag; m.sum = h->cm_sum;
  return m;
}

template <typename Src>
int launch_sem_sum(emap_handle* h, const Src& src, int s) {
  const i64 n = h->in.n[s];
  if (n <= 0) return 0;
  k_sem_sum<Src><<<cdiv(n, 256), 256, 0, h->stream>>>(h->dc, h->sem, src, n, (const int*)(h->pidx + h->offs[s]),
                                                       h->sem_fsum, h->sem_csum, sem_max(h));
  LAUNCH_CHECK();
  return 0;
}

// class_max before the scatter: U and the records per cell over every cloud (id_max read once, with the first cloud)
template <typename Src>
int launch_cm_count(emap_handle* h, const Src& src, int s) {
  const i64 n = h->in.n[s], n_idm = s == 0 ? (i64)h->sem.n_id_max * h->dc.C : 0;
  const i64 work = std::max(n, n_idm);
  if (work <= 0) return 0;
  const int grid = (int)std::min<i64>(cdiv(work, 256), (i64)h->n_sm * 4);
  k_cm_count<Src><<<grid, 256, 0, h->stream>>>(h->sem, src, n, (const int*)(h->pidx + h->offs[s]),
                                               (const int*)h->sem.id_max, n_idm, sem_max(h));
  LAUNCH_CHECK();
  return 0;
}

int frame_semantic(emap_handle* h) {
  if (h->sem.n_ch <= 0 || !h->sem_map) return 0;
  NvtxRange nv("emap:semantic");
  const int n_max = h->sem.n_max;
  if (n_max > 0) {
    // table slots: n_max per valid + inside point at most (grown like the frame's other point buffers)
    const size_t slots = (size_t)h->n_points * n_max;
    int rc;
    if ((rc = grow(h, h->cm_key, slots, slots / 4 + 1024, true)) || (rc = grow(h, h->cm_flag, slots, slots / 4 + 1024, true)) ||
        (rc = grow(h, h->cm_sum, slots, slots / 4 + 1024, true)))
      return rc;
    CK(cudaMemsetAsync(h->cm_ctl, 0, sizeof(u32) * (CM_CTL + (1 + n_max) * CM_WORDS), h->stream));
    if ((rc = h->in.each([h](auto pts, int s) { return launch_cm_count(h, pts, s); }))) return rc;
    PER_CELL(k_cm_alloc, h->dc.C, sem_max(h));
    k_cm_ulist<<<1, 1024, 0, h->stream>>>(sem_max(h));
    LAUNCH_CHECK();
  }
  if (int rc = h->in.each([h](auto pts, int s) { return launch_sem_sum(h, pts, s); })) return rc;
  if (int rc = h->in.read_done(h)) return rc;      // the input is free only now
  if (n_max > 0) {
    // occupied cells: at most one per valid + inside point
    const int grid = std::max(1, cdiv(std::min<i64>(h->dc.C, h->n_points), 256));
    for (int k = 0, j = 0; k < h->sem.n_ch; k++) {
      if (h->sem.kind[k] != SEM_CLASS_MAX) continue;
      k_cm_round<<<grid, 256, 0, h->stream>>>(h->dc.C, j, j == n_max - 1, sem_max(h), h->sem_map + (size_t)h->sem.layer[k] * h->dc.C,
                                              h->sem.id_max + (size_t)j * h->dc.C);
      LAUNCH_CHECK();
      j++;
    }
  }
  PER_CELL(k_sem_apply, h->dc, h->sem, (const u64*)h->sc.cnt_fo, h->sem_fsum, h->sem_csum, h->sem_map, sem_max(h));
  return 0;
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
    const int V = h->plan.cells_per_thread;
    const RayGrid box = ray_box(h->dc, h->plan, h->poses.data(), (int)h->poses.size());
    const i64 nthreads = (i64)(box.r1 - box.r0) * ((box.c1 - box.c0) / V);
    if (nthreads > 0) {
      if (V == 4) PDL(k_record<4>, cdiv(nthreads, 256), 256, 0, h->dc, (const float*)h->map, h->sc, (const FrameScalars*)h->fs, box, h->tmap);
      else PDL(k_record<1>, cdiv(nthreads, 256), 256, 0, h->dc, (const float*)h->map, h->sc, (const FrameScalars*)h->fs, box, h->tmap);
      LAUNCH_CHECK();
    }
    if (stage_mark(h, 4)) return EMAP_ERR_CUDA;
    for (size_t s = 0; s + 1 < h->offs.size(); s++) {
      const i64 n = h->offs[s + 1] - h->offs[s];
      if (!raycast_runs(box, n, h->dc.n_steps, h->count_rays != 0)) continue;
      // persistent grid: enough CTAs to fill every SM, never more than one warp per possible ray
      const int grid = (int)std::min<i64>((i64)h->n_sm * h->rc_blocks_per_sm, (n + RC_THREADS / 32 - 1) / (RC_THREADS / 32));
      if (h->count_rays)
        PDL(k_raycast<true>, grid, RC_THREADS, h->plan.rc_smem, h->dc, h->poses[s], (const Ray*)(h->rays + h->offs[s]), h->ray_ctl + RC_CTL * (int)s,
            (const float*)h->map, (const float*)h->normal, h->sc, (const float*)h->steps, h->plan.n_tab, (const unsigned short*)h->lut, box, (const u32*)h->tmap, h->plan.rc_lay, h->fs);
      else
        PDL(k_raycast<false>, grid, RC_THREADS, h->plan.rc_smem, h->dc, h->poses[s], (const Ray*)(h->rays + h->offs[s]), h->ray_ctl + RC_CTL * (int)s,
            (const float*)h->map, (const float*)h->normal, h->sc, (const float*)h->steps, h->plan.n_tab, (const unsigned short*)h->lut, box, (const u32*)h->tmap, h->plan.rc_lay, h->fs);
      LAUNCH_CHECK();
    }
  } else if (stage_mark(h, 4)) return EMAP_ERR_CUDA;
  if (deferred) CK(cudaStreamWaitEvent(h->stream, h->ev_join, 0));   // before the cross-rank barrier that follows this phase
  if (stage_mark(h, 5)) return EMAP_ERR_CUDA;
  h->progress = Progress::RAYS_CAST;
  return 0;
}

// TMA descriptor of the state buffer for k_post: tensor (x = column, y = row, z = layer), box = staged tile + halo of one
// layer; out-of-range elements are filled with zeros.  Encoded only when the plan stages k_post's tiles with TMA.
// cuTensorMapEncodeTiled is fetched from the driver at run time (no link-time dependency on libcuda).
int make_post_tm(emap_handle* h) {
  memset(&h->post_tm, 0, sizeof(CUtensorMap));
  if (!h->dc.post_tma) return 0;
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
  const int W = h->dc.W;
  const int HL = h->dc.dilation + 3, HLX = (HL + 3) & ~3;
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)W, 7};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4, (cuuint64_t)W * W * 4};
  const cuuint32_t box[3] = {(cuuint32_t)(PT_X + 2 * HLX), (cuuint32_t)(PT_Y + 2 * HL), 1};
  const cuuint32_t es[3] = {1, 1, 1};
  const CUresult r = enc(&h->post_tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)(float*)h->map, dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(h, EMAP_ERR_CUDA, "cuTensorMapEncodeTiled failed");
  return 0;
}

int launch_post(emap_handle* h) {
  dim3 grid(cdiv(h->dc.W, PT_X), cdiv(h->dc.W, PT_Y));
  const size_t sm = h->plan.post_smem;
  const CUtensorMap& tm = h->post_tm;
  switch (h->plan.post_instance) {
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
  if (h->plan.cells_per_thread == 4) PDL(k_finalize<4>, cdiv(h->dc.C / 4, 256), 256, 0, h->dc, h->map, h->sc, (const FrameScalars*)h->fs, h->dc.visibility, h->ray_ctl, (int)h->ray_ctl.size(), h->fused_drift ? h->fs : nullptr, h->tmap);
  else PDL(k_finalize<1>, cdiv(h->dc.C, 256), 256, 0, h->dc, h->map, h->sc, (const FrameScalars*)h->fs, h->dc.visibility, h->ray_ctl, (int)h->ray_ctl.size(), h->fused_drift ? h->fs : nullptr, h->tmap);
  LAUNCH_CHECK();
  if (stage_mark(h, 6)) return EMAP_ERR_CUDA;
  int rc = launch_post(h);
  if (rc) return rc;
  if (stage_mark(h, 7)) return EMAP_ERR_CUDA;
  h->st.have = h->timing != 0;
  h->progress = Progress::IDLE;
  return 0;
}

int layer_index(const char* name) {
  static const char* names[] = {"elevation", "variance", "is_valid", "traversability", "time", "upper_bound", "is_upper_bound"};
  for (int i = 0; i < 7; i++) if (!strcmp(name, names[i])) return i;
  return -1;
}

int alloc_plugin_scratch(emap_handle* h) {
  for (int i = 0; i < 4; i++) {
    int rc = grow(h, h->pl[i], h->dc.C, 0, false);
    if (rc) return rc;
  }
  return 0;
}

// emap_min_filter / emap_max_filter: `iteration_n` Jacobi passes ping-ponging between two plane pairs, then the select
template <bool MAX>
int minmax_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                  int32_t* iterations_run) {
  if (!elevation || !is_valid || !out || k < 0 || k > 16 || iteration_n < 1)
    return fail(h, EMAP_ERR_INVALID, "emap_min_filter: bad argument");
  int rc;
  if ((rc = alloc_plugin_scratch(h)) || (rc = grow(h, h->pl_cnt, (size_t)iteration_n + 1, 0, false))) return rc;
  const size_t B = sizeof(float) * (size_t)h->dc.C;
  float *hA = h->pl[0], *mA = h->pl[1], *hB = h->pl[2], *mB = h->pl[3];
  CK(cudaMemsetAsync(h->pl_cnt, 0, sizeof(int) * (iteration_n + 1), h->stream));
  CK(cudaMemcpyAsync(hA, elevation, B, cudaMemcpyDeviceToDevice, h->stream));      // min_filter.py:105-106
  CK(cudaMemcpyAsync(mA, is_valid, B, cudaMemcpyDeviceToDevice, h->stream));
  for (int it = 0; it < iteration_n; it++) {
    const bool even = (it & 1) == 0;
    PER_CELL(k_fill_filter_iter<MAX>, h->dc, k, is_valid, even ? hA : hB, even ? mA : mB, even ? hB : hA, even ? mB : mA,
             h->pl_cnt, it);
  }
  PER_CELL(k_min_filter_final, h->dc, hA, mA, hB, mB, h->pl_cnt, iteration_n, out, h->pl_cnt + iteration_n);
  if (iterations_run) {
    CK(cudaMemcpyAsync(iterations_run, h->pl_cnt + iteration_n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
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

// The arrays the ranks of a sharded frame reduce after phase 1..3 (kinds: see emap_exchange in emap.h).  Phase 3 first
// extracts the upper-bound keys in s32 order; without visibility cleanup it exchanges nothing.
int exchange_list(emap_handle* h, int phase, emap_exchange out[3], int32_t* n_out) {
  const i64 C = h->dc.C;
  if (phase == 1) {          // after begin: counts (CK.py:334,336) and the drift statistics (CK.py:332-333)
    out[0] = {h->sc.cnt_ai, 2 * C, 3};          // two 32-bit counters per cell: an int32 SUM keeps them apart
    out[1] = {&h->fs->E, 2, 0};
    *n_out = 2;
  } else if (phase == 2) {   // after fusion: sums, counts, last-writer keys
    out[0] = {h->sc.SH, 2 * C, 0};
    out[1] = {h->sc.cnt_fo, 2 * C, 3};
    out[2] = {h->sc.last, C, 1};
    *n_out = 3;
  } else if (h->dc.visibility) {   // after the ray-cast: decrements, counts, upper-bound keys
    k_ukey_extract<<<cdiv(C, 256), 256, 0, h->stream>>>((int)C, h->sc.ukv, h->ukey_x);
    LAUNCH_CHECK();
    out[0] = {h->sc.DV, C, 0};
    out[1] = {h->sc.n_ray, C, 3};
    out[2] = {h->ukey_x, C, 2};
    *n_out = 3;
    h->progress = Progress::KEYS_EXCHANGED;
  } else *n_out = 0;
  return 0;
}

// last phase of a sharded frame: the reduced upper-bound keys back to u32 (if phase 3 exchanged them), then finalize
int shard_finish(emap_handle* h) {
  if (h->progress == Progress::KEYS_EXCHANGED) {
    k_ukey_merge<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc.C, h->sc.ukv, h->ukey_x);
    LAUNCH_CHECK();
  }
  return frame_finish(h);
}

// export_value's named kinds: kExportNames[k] is kind k, except the last, normal_color (kind EXPORT_KIND_PLANE is a
// caller plane)
const char* const kExportNames[] = {"elevation", "variance", "traversability", "time", "upper_bound", "is_upper_bound",
                                    "normal_x", "normal_y", "normal_z", "normal_color"};
constexpr int kNumExportNames = sizeof(kExportNames) / sizeof(kExportNames[0]);
static_assert(kNumExportNames == EXPORT_KIND_PLANE + 1, "kinds 0..8 are named in order, then normal_color");
inline int export_kind(int name_index) {
  return name_index == kNumExportNames - 1 ? EXPORT_KIND_NORMAL_COLOR : name_index;
}

// The n (<= EXPORT_MAX_LAYERS) layers of an export call.  names[k]: a name of kExportNames, or planes[k] != NULL: a (W,W)
// device plane exported with flags[k] (bit 0 fill_nan, bit 1 add the centre height).  Returns false, with the message
// in h->err, for an unknown name.
bool export_list(emap_handle* h, int32_t n, const char* const* names, const float* const* planes, const int32_t* flags,
                 ExportList& L) {
  memset(&L, 0, sizeof(L));
  L.n = n;
  for (int k = 0; k < n; k++) {
    if (planes && planes[k]) {
      L.kind[k] = EXPORT_KIND_PLANE; L.plane[k] = planes[k]; L.flags[k] = flags ? flags[k] : 0;
      continue;
    }
    int kind = -1;
    if (names && names[k])
      for (int i = 0; i < kNumExportNames; i++) if (!strcmp(names[k], kExportNames[i])) kind = export_kind(i);
    if (kind < 0) { h->err = std::string("Layer ") + (names && names[k] ? names[k] : "(null)") + " is not in the map"; return false; }
    L.kind[k] = kind;
  }
  return true;
}

// Layers by one k_export_multi launch, one device-to-host copy and one synchronisation (layers as export_list).
int export_layers(emap_handle* h, int32_t n, const char* const* names, const float* const* planes, const int32_t* flags,
                  float* out_host, int64_t n_out_total) {
  if (n < 1 || n > EXPORT_MAX_LAYERS || !out_host) return fail(h, EMAP_ERR_INVALID, "emap_get_layers: 1..24 layers, non-null output");
  const int Wo = h->dc.W - 2;
  const size_t per = (size_t)Wo * Wo;
  if (n_out_total != (int64_t)(per * n)) return fail(h, EMAP_ERR_INVALID, "output must hold n * (cell_n-2)^2 floats");
  ExportList L;
  if (!export_list(h, n, names, planes, flags, L)) return EMAP_ERR_NOLAYER;
  int rc = grow(h, h->d_export, per * n, 0, false);
  if (rc) return rc;
  const auto kern = export_has_colour(L) ? k_export_multi<true> : k_export_multi<false>;
  kern<<<dim3(cdiv((i64)per, 256), n), 256, 0, h->stream>>>(h->dc, h->map, h->normal, h->d_export, L, h->center[2],
                                                             h->cfg.use_only_above_for_upper_bound);
  LAUNCH_CHECK();
  CK(cudaMemcpyAsync(out_host, h->d_export, sizeof(float) * per * n, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

// emap_get_map_points (ARROWS false) / emap_get_normal_arrows (true): the count pass and the scan, one synchronisation
// for the total; then, if the caller's capacity holds it, the write pass, the payload's copies and one more
// synchronisation.  Nothing reaches the caller's rows when the capacity is too small.
template <bool ARROWS>
int map_cloud(emap_handle* h, int64_t* n_rows, float* xyz, int32_t* ids, double* seg) {
  const int Wo = h->dc.W - 2;
  const int n_chunks = cdiv(Wo, MC_TILE), n_tiles = cdiv(Wo, MC_TILE);
  const int n = Wo * n_chunks, span = MC_TILE * n_chunks;      // count entries; entries of one scan CTA
  static_assert(MC_TILE % 4 == 0, "k_mapcloud_scan reads whole spans as int4");
  // cell_n <= 2049 (emap_create): at most 64 chunks, a span of at most 2048 entries, two per scan thread
  if (span > 2 * 1024) return fail(h, EMAP_ERR_INVALID, "map point cloud: cell_n too large for k_mapcloud_scan");
  int rc = grow(h, h->mc_table, 2 * (size_t)n + 1, 0, false);
  if (rc) return rc;
  if (!h->mc_count_host) CK(h->mc_count_host.alloc(1));
  int* cnt = h->mc_table;
  int* off = cnt + n;
  const dim3 grid(n_tiles, n_chunks);
  const MapCloudGeom g = {(double)h->center[0], (double)h->center[1], h->cfg.resolution};
  MapCloudOut o = {nullptr, nullptr, nullptr};
  k_mapcloud<ARROWS, false><<<grid, MC_THREADS, 0, h->stream>>>(h->dc, h->map, h->normal, h->center[2], cnt, nullptr, g, o);
  LAUNCH_CHECK();
  k_mapcloud_scan<<<cdiv(n, span), 1024, 0, h->stream>>>(cnt, off, n, span);
  LAUNCH_CHECK();
  CK(cudaMemcpyAsync(h->mc_count_host, off + n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  const int64_t total = *h->mc_count_host;
  if (total > *n_rows) {
    *n_rows = total;
    return fail(h, EMAP_ERR_INVALID, "map point cloud: capacity too small (needed rows in the count argument)");
  }
  *n_rows = total;
  if (!total) return EMAP_OK;
  const size_t id_bytes = ARROWS ? (sizeof(int32_t) * (size_t)total + 255) & ~(size_t)255 : 0;
  const size_t row_bytes = ARROWS ? 6 * sizeof(double) : 3 * sizeof(float);
  rc = grow(h, h->mc_out, id_bytes + row_bytes * (size_t)total, 0, false);
  if (rc) return rc;
  char* base = h->mc_out;
  o.xyz = (float*)base; o.ids = (int32_t*)base; o.seg = (double*)(base + id_bytes);
  k_mapcloud<ARROWS, true><<<grid, MC_THREADS, 0, h->stream>>>(h->dc, h->map, h->normal, h->center[2], cnt, off, g, o);
  LAUNCH_CHECK();
  if (ARROWS) {
    CK(cudaMemcpyAsync(ids, o.ids, sizeof(int32_t) * total, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(seg, o.seg, 6 * sizeof(double) * total, cudaMemcpyDeviceToHost, h->stream));
  } else {
    CK(cudaMemcpyAsync(xyz, o.xyz, 3 * sizeof(float) * total, cudaMemcpyDeviceToHost, h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  return EMAP_OK;
}

// ---- polygon safety check --------------------------------------------------------------------
constexpr int kRingHead = 256;     // ring vertices of a single call read back with its result
constexpr size_t kBatchRingHead = 4096;    // ring rows of a batch read back with its results
// (longer rings take a second copy)

struct PolyScratch {
  char* up;                        // upload region: poison counts, descriptors, clipped vertices (PolyStage)
  PolyPartial* part;               // one per k_polygon work item
  int *col_min, *col_max;          // the polygons' column windows, back to back
  char* down;                      // read-back region: one PolyResult per polygon, then the rings (PolyStage)
};

// One call's layout of the upload and read-back regions, the same in device and in pinned host memory, so that each
// region moves in one copy.  The two poison counts sit at offset 0 of the upload, the results at offset 0 of the read-back.
struct PolyStage {
  size_t desc, xy, up_bytes;
  size_t ring, down_bytes;
};

PolyStage poly_stage(size_t n_poly, size_t n_vert, size_t ring_rows) {
  PolyStage s;
  s.desc = 16;
  s.xy = s.desc + sizeof(PolyDesc) * n_poly;
  s.up_bytes = s.xy + sizeof(float2) * n_vert;
  s.ring = sizeof(PolyResult) * n_poly;
  s.down_bytes = s.ring + sizeof(double2) * ring_rows;
  return s;
}

dim3 polygon_grid(int W) { return dim3(cdiv(W, PG_COLS), cdiv(W, PG_ROWS)); }
size_t ring_capacity(int W) { return 2 * (size_t)(W - 2) + 1; }

size_t carve_polygon(const PolySizes& z, void* base, PolyScratch& s) {
  Carver b{(uintptr_t)base};
  s.up = b.take<char>(z.up);
  s.part = b.take<PolyPartial>(z.items);
  s.col_min = b.take<int>(z.cols);
  s.col_max = b.take<int>(z.cols);
  s.down = b.take<char>(z.down);
  return b.bytes;
}

// Carves the scratch of a call of sizes z, growing the device block and the pinned staging (upload region, then
// read-back region) to the largest call so far.
int alloc_polygon_scratch(emap_handle* h, const PolySizes& z, PolyScratch& s) {
  PolySizes& c = h->pg_cap;
  if (!h->pg_block || z.up > c.up || z.items > c.items || z.cols > c.cols || z.down > c.down) {
    // the read-back region follows the upload region in pinned memory: keep it aligned for its double2 rings
    c.up = std::max(c.up, (z.up + 255) & ~(size_t)255); c.items = std::max(c.items, z.items);
    c.cols = std::max(c.cols, z.cols); c.down = std::max(c.down, z.down);
    CK(h->pg_block.alloc(carve_polygon(c, nullptr, s)));
    carve_polygon(c, h->pg_block, s);
    CK(cudaMemsetAsync(s.col_min, 0x7f, sizeof(int) * c.cols, h->stream));    // "no cell yet": k_hull restores it
    CK(cudaMemsetAsync(s.col_max, 0xff, sizeof(int) * c.cols, h->stream));
  }
  if (h->pg_host.size() < c.up + c.down) CK(h->pg_host.alloc(c.up + c.down));
  carve_polygon(c, h->pg_block, s);
  return 0;
}

// The device part of a call whose n_poly polygons (n_items work items) are staged in the upload region of h->pg_host:
// one upload copy, k_poly_poison (with `poison`), k_polygon, k_hull, one copy of the results and the first `head` ring
// rows into the read-back region of h->pg_host, one synchronisation; one more copy and synchronisation only if a ring
// ends beyond `head`.
int run_polygons(emap_handle* h, const PolyScratch& s, const PolyStage& st, int n_poly, int n_items, bool poison,
                 const float* checker_plane, double safe_thresh, double safe_min_thresh, int32_t max_unsafe_n,
                 float* mask, bool hulls, size_t head) {
  const int W = h->dc.W;
  const size_t C = (size_t)h->dc.C;
  const dim3 g = polygon_grid(W);
  const float* valid = h->map + L_VALID * C;
  const float* checker = checker_plane ? checker_plane : h->map + L_TRAV * C;
  PolyArgs a;
  a.poly = (const PolyDesc*)(s.up + st.desc); a.n_poly = n_poly; a.xy = (const float2*)(s.up + st.xy);
  a.cx = h->center[0]; a.cy = h->center[1];
  a.thr_over = (float)(1.0 - safe_thresh); a.thr_max = (float)(1.0 - safe_min_thresh);    // traversability_polygon.py:25-26
  a.max_unsafe_n = max_unsafe_n;
  a.poison = poison ? (const int*)s.up : nullptr;
  memcpy(&a.one, h->pg_host + st.desc, sizeof(PolyDesc));
  CK(cudaMemcpyAsync(s.up, h->pg_host, st.up_bytes, cudaMemcpyHostToDevice, h->stream));
  if (poison) {
    k_poly_poison<<<std::min(cdiv((i64)C, 256), 4 * h->n_sm), 256, 0, h->stream>>>(W, valid, checker, (int*)s.up);
    LAUNCH_CHECK();
  }
  (poison ? k_polygon<true> : k_polygon<false>)<<<n_items, PG_THREADS, 0, h->stream>>>(
      W, h->dc.res_f, a, valid, checker, mask, s.part, hulls ? s.col_min : nullptr, hulls ? s.col_max : nullptr);
  LAUNCH_CHECK();
  k_hull<<<n_poly, HULL_THREADS, 0, h->stream>>>(W, h->cfg.resolution, a, (int)g.x, (int)g.y, s.part, s.col_min,
                                                 s.col_max, (PolyResult*)s.down,
                                                 hulls ? (double2*)(s.down + st.ring) : nullptr);
  LAUNCH_CHECK();
  char* back = h->pg_host + h->pg_cap.up;
  head = std::min(head, (st.down_bytes - st.ring) / sizeof(double2));
  CK(cudaMemcpyAsync(back, s.down, st.ring + sizeof(double2) * head, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  const PolyResult* r = (const PolyResult*)back;
  const PolyDesc* d = (const PolyDesc*)(h->pg_host + st.desc);
  size_t end = 0;
  for (int i = 0; i < n_poly; i++)
    if (r[i].n_ring) end = std::max(end, (size_t)d[i].ring_off + r[i].n_ring);
  if (end > head) {
    const size_t off = st.ring + sizeof(double2) * head;
    CK(cudaMemcpyAsync(back + off, s.down + off, sizeof(double2) * (end - head), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}

// ---- features_pca ------------------------------------------------------------------------------
struct PcaScratch {
  PcaResult* res;
  double* part;                    // pca_entries(PCA_MAX_F) per k_pca_stats CTA
  double* proj;                    // 3 planes of C projections
};

int pca_stats_grid(emap_handle* h) { return std::min(cdiv(h->dc.C, 32), 2 * h->n_sm); }   // 32 <= tile cells

size_t carve_pca(emap_handle* h, void* base, PcaScratch& s) {
  Carver b{(uintptr_t)base};
  s.res = b.take<PcaResult>(1);
  s.part = b.take<double>((size_t)pca_stats_grid(h) * PCA_MAX_ENTRIES);
  s.proj = b.take<double>(3 * (size_t)h->dc.C);
  return b.bytes;
}

// the planes of a semantic plugin call: a non-null host array of n non-null device pointers
bool planes_ok(int32_t n, const float* const* planes) {
  if (n > 0 && !planes) return false;
  for (int l = 0; l < n; l++) if (!planes[l]) return false;
  return true;
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
    delete h;
    return (int)EMAP_ERR_CUDA;
  };
  cudaError_t e;
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  make_plan(*cfg, h->dc, h->plan);
  const size_t C = (size_t)h->dc.C;
  for (Stream* s : {&h->own_stream, &h->copy_stream, &h->side_stream})
    if ((e = s->create(cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  h->stream = h->own_stream;
  for (Event* ev : {&h->in.staging_free[0], &h->in.staging_free[1], &h->in.copied, &h->in.host_free, &h->ev_fork,
                    &h->ev_join, &h->ev_order, &h->img_up.staged, &h->init_up.staged})
    if ((e = ev->create(cudaEventDisableTiming)) != cudaSuccess) return bail("event", e);
  for (Event& ev : h->st.ev) if ((e = ev.create(cudaEventDefault)) != cudaSuccess) return bail("event", e);
#define ALLOC(buf, n) if ((e = (buf).alloc(n)) != cudaSuccess) return bail("cudaMalloc", e)
#define TRY(call) if ((e = (call)) != cudaSuccess) return bail(#call, e)
  ALLOC(h->map, 7 * C);
  ALLOC(h->map_alt, 7 * C);
  ALLOC(h->normal, 3 * C);
  ALLOC(h->trav_input, C);
  ALLOC(h->xscratch, exchange_bytes(C));
  ALLOC(h->thr, C);
  ALLOC(h->dirty, C + 16);
  ALLOC(h->ukey_x, C);
  ALLOC(h->lut, 65536);
  ALLOC(h->tmap, RT * RT);
  ALLOC(h->step_cnt, 0x7c00 + 8);
  ALLOC(h->steps, h->plan.n_tab);
#undef ALLOC
  h->sc.thr = h->thr;
  h->sc.dirty = h->dirty;
  TRY(place_exchange(h, h->xscratch));
  TRY(cudaMemsetAsync(h->thr, 0, sizeof(float) * C, h->stream));
  TRY(cudaMemsetAsync(h->dirty, 0, C + 16, h->stream));
  TRY(cudaMemsetAsync(h->tmap, 0, sizeof(u32) * RT * RT, h->stream));
  TRY(cudaMemsetAsync(h->normal, 0, sizeof(float) * 3 * C, h->stream));
  TRY(cudaMemsetAsync(h->trav_input, 0, sizeof(float) * C, h->stream));
  {
    std::vector<float> tab((size_t)h->plan.n_tab, INFINITY);
    tab[0] = NAN;       // "step -1" of lane 0 in a ray's first warp iteration: NaN -> cell (0, 0), see k_raycast
    for (size_t k = 0; k < h->plan.steps.size(); k++) tab[1 + k] = h->plan.steps[k];
    // pageable source: the copy is staged before the call returns, and the stream is synchronised below
    TRY(cudaMemcpyAsync(h->steps, tab.data(), sizeof(float) * tab.size(), cudaMemcpyHostToDevice, h->stream));
    TRY(cudaStreamSynchronize(h->stream));
  }
  k_build_lut<<<256, 256, 0, h->stream>>>(h->dc, h->lut);
  k_build_step_cnt<<<cdiv(0x7c01, 256), 256, 0, h->stream>>>((const float*)(h->steps + 1), h->dc.n_steps, h->step_cnt);
  k_init<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc, h->map);
  h->launches += 2;
  if (make_post_tm(h)) {
    g_create_error = h->err; delete h; return EMAP_ERR_CUDA;
  }
  if (h->plan.post_smem > 48 * 1024)
    TRY(cudaFuncSetAttribute(k_post<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->plan.post_smem));
  TRY(cudaFuncSetAttribute(k_raycast<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->plan.rc_smem));
  TRY(cudaFuncSetAttribute(k_raycast<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->plan.rc_smem));
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->n_sm = prop.multiProcessorCount;
  int nb = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_raycast<false>, RC_THREADS, h->plan.rc_smem) == cudaSuccess && nb > 0)
    h->rc_blocks_per_sm = nb;
  else h->rc_blocks_per_sm = 1;
  TRY(cudaStreamSynchronize(h->stream));
  TRY(cudaGetLastError());
#undef TRY
  *out = h;
  return EMAP_OK;
}

int emap_destroy(emap_handle* h) {
  delete h;
  return EMAP_OK;
}

static void comm_release(emap_handle* h);

}  // extern "C"

// The members release the memory, streams and events after this body, once no queued work uses them (emap_set_stream
// synchronises the stream it replaces, so the current one holds everything queued on the handle's behalf).
emap_handle::~emap_handle() {
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);
  if (copy_stream) cudaStreamSynchronize(copy_stream);
  if (side_stream) cudaStreamSynchronize(side_stream);
  comm_release(this);
}

// EM.py:119-128 clear
int clear_map(emap_handle* h) {
  PER_CELL(k_clear, h->dc, h->map);
  CK(cudaMemsetAsync(&h->fs->mean_error, 0, 2 * sizeof(float), h->stream));     // EM.py:127-128
  return EMAP_OK;
}

// EM.py:913-922 after the interpolation: `iterations` Jacobi passes of the initialiser dilation, then
// upper_bound <- elevation on valid cells
int initialize_finish(emap_handle* h, int32_t dilation_size, int32_t iterations) {
  if (dilation_size < 0 || dilation_size > 64 || iterations < 0 || iterations > 16)
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map_finish: 0 <= dilation_size <= 64, 0 <= iterations <= 16");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  const size_t B = sizeof(float) * (size_t)h->dc.C;
  const int passes = dilation_size > 0 ? iterations : 0;
  for (int it = 0; it < std::max(passes, 1); it++) {
    CK(cudaMemcpyAsync(h->pl[0], h->map, B, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaMemcpyAsync(h->pl[1], h->map + 2 * (size_t)h->dc.C, B, cudaMemcpyDeviceToDevice, h->stream));
    PER_CELL(k_init_dilate, h->dc, h->pl[0], h->pl[1], h->map, passes ? dilation_size : 0, it == std::max(passes, 1) - 1);
  }
  return EMAP_OK;
}

// The frame after frame_start: every pass, then the wait after which the caller may reuse its host memory
int frame_run(emap_handle* h) {
  int rc;
  if ((rc = frame_index(h)) || (rc = frame_fuse(h)) || (rc = frame_semantic(h)) || (rc = frame_rays(h)) ||
      (rc = frame_finish(h)))
    return rc;
  return h->in.wait_free(h);
}

extern "C" {

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
  const int rc = frame_begin(h, n_sensors, points, n, row_stride, dtype, is_device_ptr, R, t, 0, pn, on, false);
  return rc ? rc : frame_run(h);
}

int emap_input_pointcloud(emap_handle* h, const void* points, int64_t n, int64_t row_stride, int dtype, int is_device_ptr,
                          const float R[9], const float t[3], float pn, float on) {
  const void* p[1] = {points};
  int64_t nn[1] = {n};
  return emap_input_sensors(h, 1, p, nn, row_stride, dtype, is_device_ptr, R, t, pn, on);
}

int emap_input_depth_images(emap_handle* h, int32_t n_cameras, const emap_depth_camera* cams, int is_device_ptr,
                            int32_t n_channels, const int32_t* channel_source, int32_t n_features,
                            float confidence_threshold, float max_depth, float pn, float on) {
  ENTER(h);
  if (h->attached) return fail(h, EMAP_ERR_STATE, "handle is attached to a sharded scratch: use the emap_shard_* calls");
  if (!cams || n_cameras < 1 || n_cameras > EMAP_DEPTH_MAX_CAMERAS)
    return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: 1 <= n_cameras <= EMAP_DEPTH_MAX_CAMERAS cameras required");
  if (n_channels < 0 || n_channels > SEM_MAX_CH || (n_channels > 0 && !channel_source) || n_features < 0 ||
      n_features > EMAP_DEPTH_MAX_FEATURES)
    return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: 0..16 channels with their sources, 0..255 feature planes required");
  int n_color = 0, n_feat_used = 0;
  for (int j = 0; j < n_channels; j++) {
    if (channel_source[j] < -1 || channel_source[j] >= n_features)
      return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: a channel source outside [-1, n_features)");
    n_color += channel_source[j] == -1;
    n_feat_used += channel_source[j] >= 0;
  }
  if (n_color > 1) return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: more than one colour channel");
  if (h->sem.n_ch > 0 && h->sem_map)
    for (int k = 0; k < h->sem.n_ch; k++)
      if (h->sem.col[k] >= 3 + n_channels)
        return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: a configured semantic column beyond 3 + n_channels");
  int64_t n[EMAP_DEPTH_MAX_CAMERAS];      // at most 16 * 2^24 = 2^28 pixels: below the frame's 2^31 rows
  float R[9 * EMAP_DEPTH_MAX_CAMERAS], t[3 * EMAP_DEPTH_MAX_CAMERAS];
  for (int s = 0; s < n_cameras; s++) {
    const emap_depth_camera& c = cams[s];
    bool finite = std::isfinite(c.fx) && std::isfinite(c.fy) && c.fx != 0.0 && c.fy != 0.0 && std::isfinite(c.cx) &&
                  std::isfinite(c.cy);
    for (int k = 0; k < 9; k++) finite = finite && std::isfinite(c.R[k]);
    for (int k = 0; k < 3; k++) finite = finite && std::isfinite(c.t[k]);
    if (!c.depth || c.height <= 0 || c.width <= 0 || (i64)c.height * c.width > (1ll << 24))
      return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: a depth image, 0 < height * width <= 2^24 required");
    if (!finite) return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: non-finite or zero fx / fy, or non-finite cx, cy, R, t");
    if ((n_color && !c.rgb) || (n_feat_used && !c.features))
      return fail(h, EMAP_ERR_INVALID, "emap_input_depth_images: a colour channel needs rgb, a feature channel the feature planes");
    n[s] = (i64)c.height * c.width;
    memcpy(R + 9 * s, c.R, sizeof(c.R));
    memcpy(t + 3 * s, c.t, sizeof(c.t));
  }
  // per camera: depth, confidence, rgb, feature planes (the ones the channels read)
  FrameInput& in = h->in;
  in.kind = FrameInput::DEPTH; in.n.assign(n, n + n_cameras);
  in.bufs.resize(4 * n_cameras); in.bytes.resize(4 * n_cameras); in.cams.assign(n_cameras, DepthSource{});
  for (int s = 0; s < n_cameras; s++) {
    const emap_depth_camera& c = cams[s];
    const size_t P = (size_t)n[s];
    in.bufs[4 * s] = c.depth; in.bytes[4 * s] = 4 * P;
    in.bufs[4 * s + 1] = c.confidence; in.bytes[4 * s + 1] = c.confidence ? 4 * P : 0;
    in.bufs[4 * s + 2] = c.rgb; in.bytes[4 * s + 2] = n_color ? 3 * P : 0;
    in.bufs[4 * s + 3] = c.features; in.bytes[4 * s + 3] = n_feat_used ? 4 * P * n_features : 0;
    DepthSource& d = in.cams[s];
    d.conf = c.confidence; d.plane = n[s]; d.width = c.width;
    d.conf_min = confidence_threshold; d.max_depth = max_depth;
    d.fx = c.fx; d.fy = c.fy; d.cx = c.cx; d.cy = c.cy;
    for (int j = 0; j < n_channels; j++) d.src[j / 8] |= (u64)(channel_source[j] + 1) << (8 * (j % 8));
  }
  const int rc = frame_start(h, is_device_ptr, R, t, 0, pn, on, false);
  return rc ? rc : frame_run(h);
}

int emap_input_depth_image(emap_handle* h, const emap_depth_camera* camera, int is_device_ptr, int32_t n_channels,
                           const int32_t* channel_source, int32_t n_features, float confidence_threshold, float max_depth,
                           float pn, float on) {
  return emap_input_depth_images(h, 1, camera, is_device_ptr, n_channels, channel_source, n_features, confidence_threshold,
                                 max_depth, pn, on);
}

// ---- semantic point-channel fusion ------------------------------------------------------------
namespace {
int semantic_configure(emap_handle* h, const char* fn, int max_kind, int32_t n_channels, const int32_t* column,
                       const int32_t* kind, const int32_t* layer, float* semantic_map_device, int32_t n_layers,
                       double average_weight, float* variance_device, int32_t* id_max_device, int32_t n_id_max) {
  char msg[200];
  if (n_channels <= 0) { h->sem.n_ch = 0; h->sem_map = nullptr; return EMAP_OK; }
  if (n_channels > SEM_MAX_CH || !column || !kind || !layer || !semantic_map_device || n_layers < 1) {
    snprintf(msg, sizeof(msg), "%s: 1..16 channels, non-null arrays and layer buffer", fn);
    return fail(h, EMAP_ERR_INVALID, msg);
  }
  SemCfg c;
  memset(&c, 0, sizeof(c));
  c.n_ch = n_channels; c.alpha = average_weight;
  int nf = 0, nc = 0, nm = 0, nb = 0;
  for (int k = 0; k < n_channels; k++) {
    if (column[k] < 3 || layer[k] < 0 || layer[k] >= n_layers || kind[k] < SEM_AVERAGE || kind[k] > max_kind) {
      snprintf(msg, sizeof(msg), "%s: column >= 3, 0 <= layer < n_layers, kind 0..%d required", fn, max_kind);
      return fail(h, EMAP_ERR_INVALID, msg);
    }
    c.col[k] = column[k]; c.kind[k] = kind[k]; c.layer[k] = layer[k];
    c.slot[k] = (kind[k] == SEM_COLOR) ? 4 * nc++ : (kind[k] == SEM_CLASS_MAX) ? nm++ : nf++;
    nb += kind[k] == SEM_BAYESIAN_INFERENCE;
  }
  if (nb > 0 && !variance_device)
    return fail(h, EMAP_ERR_INVALID, "emap_semantic_configure_ext: bayesian_inference needs the variance planes");
  if (nm > 0 && (!id_max_device || n_id_max < nm))
    return fail(h, EMAP_ERR_INVALID, "emap_semantic_configure_ext: class_max needs id_max with one plane per class_max channel");
  c.n_max = nm; c.sigma = nb ? variance_device : nullptr;
  c.id_max = nm ? id_max_device : nullptr; c.n_id_max = nm ? n_id_max : 0;
  const size_t C = (size_t)h->dc.C;
  int rc;
  if ((rc = grow(h, h->sem_fsum, C * nf, 0, true)) || (rc = grow(h, h->sem_csum, C * 4 * nc, 0, true))) return rc;
  if (nm > 0 && ((rc = grow(h, h->cm_cell, 3 * C, 0, true)) ||
                 (rc = grow(h, h->cm_ctl, (size_t)CM_CTL + (1 + SEM_MAX_CH) * CM_WORDS + 65536, 0, true))))
    return rc;
  h->sem = c; h->sem_map = semantic_map_device;
  return EMAP_OK;
}
}  // namespace

int emap_semantic_configure(emap_handle* h, int32_t n_channels, const int32_t* column, const int32_t* kind, const int32_t* layer,
                            float* semantic_map_device, int32_t n_layers, double average_weight) {
  ENTER(h);
  return semantic_configure(h, "emap_semantic_configure", SEM_COLOR, n_channels, column, kind, layer, semantic_map_device,
                            n_layers, average_weight, nullptr, nullptr, 0);
}

int emap_semantic_configure_ext(emap_handle* h, int32_t n_channels, const int32_t* column, const int32_t* kind,
                                const int32_t* layer, float* semantic_map_device, int32_t n_layers, double average_weight,
                                float* variance_device, int32_t* id_max_device, int32_t n_id_max) {
  ENTER(h);
  return semantic_configure(h, "emap_semantic_configure_ext", SEM_CLASS_MAX, n_channels, column, kind, layer,
                            semantic_map_device, n_layers, average_weight, variance_device, id_max_device, n_id_max);
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
  if (rc || (rc = h->in.wait_free(h))) return rc;
  // multicast mode: every rank must have reset its frame scalars before anyone pushes -> the caller runs a
  // cross-rank barrier and then emap_shard_phase(h, 0); NCCL mode: index right away
  if (h->attached) return 0;
  return (rc = frame_index(h)) ? rc : h->in.wait_free(h);
}

int64_t emap_shard_scratch_bytes(const emap_handle* h) {
  if (!h) return EMAP_ERR_INVALID;
  return (int64_t)exchange_bytes((size_t)h->dc.C);
}

int emap_shard_attach(emap_handle* h, void* local_base, void* multicast_base, int64_t bytes) {
  ENTER(h);
  if (!local_base || !multicast_base || bytes < emap_shard_scratch_bytes(h))
    return fail(h, EMAP_ERR_INVALID, "emap_shard_attach: need local + multicast base of >= emap_shard_scratch_bytes()");
  CK(cudaStreamSynchronize(h->stream));
  FrameScalars keep;
  CK(cudaMemcpy(&keep, h->fs, sizeof(keep), cudaMemcpyDeviceToHost));
  // the library's own scratch is released; the symmetric block (owned by the caller) replaces it
  h->xscratch.reset();
  CK(place_exchange(h, local_base));
  h->sc.mc_off = (i64)((char*)multicast_base - (char*)local_base);
  CK(cudaMemcpyAsync(h->fs, &keep, sizeof(keep), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->attached = true;
  return EMAP_OK;
}

int emap_shard_set_overlap_z(emap_handle* h, float z_abs) {
  ENTER(h);
  if (h->progress != Progress::BEGUN && h->progress != Progress::INDEXED)
    return fail(h, EMAP_ERR_STATE, "emap_shard_set_overlap_z must follow emap_shard_begin");
  h->overlap_override = true; h->overlap_z_override = z_abs - h->center[2];     // consumed by k_drift (phase 1)
  return EMAP_OK;
}

int emap_shard_exchange(emap_handle* h, int32_t phase, emap_exchange* out, int32_t* n_out) {
  ENTER(h);
  if (!out || !n_out || *n_out < 3) return fail(h, EMAP_ERR_INVALID, "emap_shard_exchange: need capacity >= 3");
  if (phase < 1 || phase > 3) return fail(h, EMAP_ERR_INVALID, "emap_shard_exchange: phase must be 1..3");
  static const char* order[] = {"", "exchange 1 must follow emap_shard_begin", "exchange 2 must follow phase 1",
                                "exchange 3 must follow phase 2"};
  static const Progress after[] = {Progress::IDLE, Progress::INDEXED, Progress::FUSED, Progress::RAYS_CAST};
  if (h->progress != after[phase]) return fail(h, EMAP_ERR_STATE, order[phase]);
  return exchange_list(h, phase, out, n_out);
}

int emap_shard_phase(emap_handle* h, int32_t phase) {
  ENTER(h);
  if (phase == 0) {
    if (h->progress != Progress::BEGUN) return fail(h, EMAP_ERR_STATE, "phase 0 must follow emap_shard_begin on an attached handle");
    const int rc = frame_index(h);
    return rc ? rc : h->in.wait_free(h);
  }
  if (phase == 1) {
    if (h->progress != Progress::INDEXED) return fail(h, EMAP_ERR_STATE, "phase 1 must follow emap_shard_begin");
    return frame_fuse(h);
  }
  if (phase == 2) {
    if (h->progress != Progress::FUSED) return fail(h, EMAP_ERR_STATE, "phase 2 must follow phase 1");
    return frame_rays(h);
  }
  if (phase == 3) {
    if (h->progress != Progress::RAYS_CAST && h->progress != Progress::KEYS_EXCHANGED) return fail(h, EMAP_ERR_STATE, "phase 3 must follow phase 2");
    return shard_finish(h);
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
  emap_exchange ex[3];
  int32_t n = 0;
  int rc = exchange_list(h, phase, ex, &n);
  if (rc) return rc;
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
  if (rc || (rc = h->in.wait_free(h)) || (rc = frame_index(h)) || (rc = h->in.wait_free(h))) return rc;
  h->overlap_override = true; h->overlap_z_override = overlap_sensor_z_absolute - h->center[2];
  if ((rc = comm_exchange(h, 1))) return rc;
  if ((rc = frame_fuse(h))) return rc;
  if ((rc = comm_exchange(h, 2))) return rc;
  if ((rc = frame_rays(h))) return rc;
  if ((rc = comm_exchange(h, 3))) return rc;
  return shard_finish(h);
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
  out->n_points = h->in.kind == FrameInput::DEPTH ? f.nkept_last : h->n_points; out->n_valid_points = f.nvalid_last; out->ray_steps = f.ray_steps; out->ray_visits = f.ray_visits;
  return EMAP_OK;
}

int emap_set_ray_counting(emap_handle* h, int enable) { ENTER(h); h->count_rays = enable ? 1 : 0; return EMAP_OK; }

// ---- pose / time -----------------------------------------------------------------------------
static int shift_map(emap_handle* h, int sx, int sy, double dz) {
  if (sx == 0 && sy == 0) {                                    // EM.py:208-209 early return, then shift_map_z
    PER_CELL(k_shift_z, h->dc, h->map, dz);
    return 0;
  }
  // shifted into map_alt and copied back: map keeps its address, which captured frames and the caller's views hold
  PER_CELL(k_shift, h->dc, h->map, h->map_alt, sx, sy, dz);
  CK(cudaMemcpyAsync(h->map, h->map_alt, sizeof(float) * 7 * (size_t)h->dc.C, cudaMemcpyDeviceToDevice, h->stream));
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
  return clear_map(h);
}

int emap_update_variance(emap_handle* h) {
  ENTER(h);
  PER_CELL(k_update_variance, h->dc, h->map);
  return EMAP_OK;
}

int emap_update_time(emap_handle* h) {
  ENTER(h);
  PER_CELL(k_update_time, h->dc, h->map);
  return EMAP_OK;
}

int emap_update_normal(emap_handle* h, const float* dilated) {
  ENTER(h);
  PER_CELL(k_normal, h->dc, dilated ? dilated : h->trav_input, h->map + 2 * (size_t)h->dc.C, h->normal);
  return EMAP_OK;
}

// EM.py:913-922: the device half of initialize_map, after the caller wrote the interpolated planes (emap_set_state):
// `iterations` Jacobi passes of the initialiser dilation, then upper_bound <- elevation on valid cells.
int emap_initialize_map_finish(emap_handle* h, int32_t dilation_size, int32_t iterations) {
  ENTER(h);
  return initialize_finish(h, dilation_size, iterations);
}

// EM.py:899-922 + map_initializer.py:25-62 on the device (include/emap.h, csrc/emap_initialize.cuh): clear, snap, the
// host part (triangulation, gradients, coefficients, tile lists), one upload, one interpolation kernel, then the
// dilation passes and the upper-bound fill of emap_initialize_map_finish.
int emap_initialize_map(emap_handle* h, const float* xyz_host, int32_t n_points, int32_t method,
                        const int32_t* triangles_host, int32_t n_triangles, const double* gradients_host,
                        double initialized_variance, int32_t dilation_size_initialize) {
  ENTER(h);
  NvtxRange nv("emap:initialize_map");
  int rc = clear_map(h);                 // EM.py:906: every failure below leaves the map cleared
  if (rc) return rc;
  if (!xyz_host) return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: null points");
  if (n_points <= 3) return fail(h, EMAP_ERR_INVALID, "Initialization points must be more than 3.");
  if (n_points > EMAP_INIT_MAX_POINTS)
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: more than EMAP_INIT_MAX_POINTS points");
  if (method < 0 || method > 2) return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: method must be 0 (nearest), 1 (linear) or 2 (cubic)");
  if (triangles_host && (n_triangles < 1 || n_triangles > 2 * EMAP_INIT_MAX_POINTS))
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: 1 to 2 * EMAP_INIT_MAX_POINTS triangles required");
  if (dilation_size_initialize < 0 || dilation_size_initialize > 64 || !std::isfinite(initialized_variance))
    return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: 0 <= dilation_size_initialize <= 64 and a finite variance required");
  // transform_to_map_index as elevation_mapping.py applies it, in fp32: ((xy - center) / res + W / 2), truncated
  const int W = h->dc.W, n = n_points;
  const float res_f = (float)h->cfg.resolution, half_f = (float)(0.5 * W);
  std::vector<long long> xy(2 * (size_t)n);
  std::vector<double> z(n);
  bool narrow = true;
  for (int i = 0; i < n; i++) {
    const float* q = xyz_host + 3 * (size_t)i;
    if (!std::isfinite(q[0]) || !std::isfinite(q[1]) || !std::isfinite(q[2]))
      return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: non-finite point");
    for (int d = 0; d < 2; d++) {
      const float v = (q[d] - h->center[d]) / res_f;
      const float c = v + half_f;
      if (!(c >= -2147483648.f && c < 2147483648.f))
        return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: a point's cell index is outside the int32 range");
      xy[2 * i + d] = (long long)(int32_t)c;
      narrow &= std::llabs(xy[2 * i + d]) <= INIT_NARROW;
    }
    z[i] = (double)(float)(q[2] - h->center[2]);
  }
  InitArgs a;
  memset(&a, 0, sizeof(a));
  a.W = W; a.C = h->dc.C; a.tiles_x = (W + INIT_TILE - 1) / INIT_TILE;
  a.var = (float)initialized_variance;
  // the upload: one block, 256-byte aligned arrays, the same layout in pinned and in device memory
  std::vector<int> tri, nb, off, list;
  std::vector<double> grad, coef;
  Carver up{0};           // base 0: take() returns byte offsets
  size_t o_pxy = 0, o_pz = 0, o_txy = 0, o_coef = 0, o_off = 0, o_list = 0;
  if (method == 0) {
    a.n = n;
    o_pxy = (size_t)up.take<int2>(n);
    o_pz = (size_t)up.take<float>(n);
  } else {
    if (triangles_host) {
      tri.assign(triangles_host, triangles_host + 3 * (size_t)n_triangles);
      for (int t = 0; t < n_triangles; t++) {
        int* v = &tri[3 * (size_t)t];
        if (v[0] < 0 || v[0] >= n || v[1] < 0 || v[1] >= n || v[2] < 0 || v[2] >= n)
          return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: triangle index outside [0, n_points)");
        const int o = init_host::orient_sign(&xy[2 * (size_t)v[0]], &xy[2 * (size_t)v[1]], &xy[2 * (size_t)v[2]]);
        if (o == 0) return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: a triangle of zero area");
        if (o < 0) std::swap(v[1], v[2]);
      }
    } else if (!init_host::delaunay(xy, tri)) {
      return fail(h, EMAP_ERR_INVALID, "emap_initialize_map: the points are collinear (no triangulation)");
    }
    const int T = (int)(tri.size() / 3);
    a.n = T;
    if (method == 2) {
      init_host::neighbours(tri, nb);
      if (!gradients_host) init_host::estimate_gradients(xy, z, tri, grad);
      coef.resize((size_t)INIT_CT * T);
      init_host::ct_coefficients(xy, z, gradients_host ? gradients_host : grad.data(), tri, nb, coef.data());
    } else {
      coef.resize(3 * (size_t)T);
      for (size_t k = 0; k < coef.size(); k++) coef[k] = z[tri[k]];
    }
    init_host::bin_tiles(W, xy, tri, off, list);
    o_txy = (size_t)up.take<int>(6 * (size_t)T);
    o_coef = (size_t)up.take<double>(coef.size());
    o_off = (size_t)up.take<int>(off.size());
    o_list = (size_t)up.take<int>(std::max<size_t>(list.size(), 1));
  }
  if ((rc = h->init_up.room(h, up.bytes))) return rc;
  char* hb = h->init_up.host;
  char* db = h->init_up.dev;
  if (method == 0) {
    int2* pxy = (int2*)(hb + o_pxy);
    float* pz = (float*)(hb + o_pz);
    for (int i = 0; i < n; i++) { pxy[i] = make_int2((int)xy[2 * i], (int)xy[2 * i + 1]); pz[i] = (float)z[i]; }
    a.pxy = (const int2*)(db + o_pxy); a.pz = (const float*)(db + o_pz);
  } else {
    int* txy = (int*)(hb + o_txy);
    for (size_t k = 0; k < tri.size(); k++) { txy[2 * k] = (int)xy[2 * (size_t)tri[k]]; txy[2 * k + 1] = (int)xy[2 * (size_t)tri[k] + 1]; }
    memcpy(hb + o_coef, coef.data(), sizeof(double) * coef.size());
    memcpy(hb + o_off, off.data(), sizeof(int) * off.size());
    if (!list.empty()) memcpy(hb + o_list, list.data(), sizeof(int) * list.size());
    a.txy = (const int*)(db + o_txy); a.coef = (const double*)(db + o_coef);
    a.tile_off = (const int*)(db + o_off); a.tile_tri = (const int*)(db + o_list);
  }
  if ((rc = h->init_up.send(h, up.bytes))) return rc;
  const int grid = a.tiles_x * a.tiles_x;
  if (method == 0) {
    if (narrow) k_init_nearest<long long><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
    else k_init_nearest<__int128><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
  } else if (method == 1) {
    if (narrow) k_init_interp<long long, false><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
    else k_init_interp<__int128, false><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
  } else {
    if (narrow) k_init_interp<long long, true><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
    else k_init_interp<__int128, true><<<grid, INIT_THREADS, 0, h->stream>>>(a, h->map);
  }
  LAUNCH_CHECK();
  return initialize_finish(h, dilation_size_initialize, 2);
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
  return export_layers(h, 1, &name, nullptr, nullptr, out_host, n_out);
}

// Several layers in one launch, one device-to-host copy and one synchronisation (WRAP:213-252 get_grid_map exports a list
// of layers per call).
int emap_get_layers(emap_handle* h, int32_t n, const char* const* names, const float* const* planes, const int32_t* flags,
                    float* out_host, int64_t n_out_total) {
  ENTER(h);
  return export_layers(h, n, names, planes, flags, out_host, n_out_total);
}

static_assert(EMAP_SUBMAP_MAX_WINDOWS == SUBMAP_MAX_WINDOWS && EMAP_SUBMAP_MAX_LAYERS == EXPORT_MAX_LAYERS,
              "emap.h states the kernel's limits");

static bool submap_lengths_ok(int64_t n, const double* windows) {
  for (int64_t w = 0; w < n; w++)
    for (int a = 2; a < 4; a++)
      if (!(std::isfinite(windows[4 * w + a]) && windows[4 * w + a] >= 0.0)) return false;
  return true;
}

// The host part of emap_get_submaps on its own (no handle, no device): submap_window for every request.
int emap_submap_windows(int32_t cell_n, double resolution, const double center[2], int32_t n_windows,
                        const double* windows, int32_t* info, double* centres) {
  if (!center || !windows || !info || !centres || cell_n < 3 || !(std::isfinite(resolution) && resolution > 0.0) ||
      n_windows < 0 || !submap_lengths_ok(n_windows, windows))
    return EMAP_ERR_INVALID;
  for (int32_t w = 0; w < n_windows; w++) submap_window(cell_n, resolution, center, windows + 4 * w, info + 5 * w, centres + 2 * w);
  return EMAP_OK;
}

// Appends the successful window q = submap_window's info to k_submap's table: its first work item is `tiles` and its
// first output float `total`, both advanced past it.
static void submap_add(SubmapArgs& a, int W, const int32_t q[5], int n_layers, int& tiles, long long& total) {
  SubmapWin& s = a.win[a.n_win++];
  s.r0 = (int16_t)(W - 2 - q[1]); s.c0 = (int16_t)(W - 2 - q[2]);
  s.rows = (int16_t)q[3]; s.cols = (int16_t)q[4];
  s.tile0 = tiles; s.off = total;
  tiles += cdiv(q[3], SUBMAP_ROWS);
  total += (long long)n_layers * q[3] * q[4];
}

// The get_raw_submap service (elevation_mapping_ros.cpp:507-553) for a batch of windows: the windows on the host
// (submap_window), every (window, layer, row) of the batch in one k_submap launch whose table is its parameters.  Host
// output: one device-to-host copy and one synchronisation; device output: stream-ordered, no synchronisation.  Every
// check runs before anything is written or launched.
int emap_get_submaps(emap_handle* h, int32_t n_windows, const double* windows, int32_t n_layers, const char* const* names,
                     const float* const* planes_device, const int32_t* flags, float* out, int32_t out_is_device,
                     int64_t out_floats, int32_t* info, double* centres) {
  ENTER(h);
  NvtxRange nv("emap:get_submaps");
  if (!windows || !names || !out || !info || !centres) return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: null argument");
  if (n_windows < 1 || n_windows > EMAP_SUBMAP_MAX_WINDOWS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: 1 to EMAP_SUBMAP_MAX_WINDOWS windows required");
  if (n_layers < 1 || n_layers > EMAP_SUBMAP_MAX_LAYERS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: 1 to EMAP_SUBMAP_MAX_LAYERS layers required");
  if (!submap_lengths_ok(n_windows, windows))
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: lengths must be finite and >= 0");
  SubmapArgs a;
  if (!export_list(h, n_layers, names, planes_device, flags, a.L)) return EMAP_ERR_INVALID;
  const int W = h->dc.W;
  const double m[2] = {h->center[0], h->center[1]};
  std::vector<int32_t> inf(5 * (size_t)n_windows);
  std::vector<double> cen(2 * (size_t)n_windows);
  a.n_win = 0;
  int tiles = 0;
  long long total = 0;
  for (int w = 0; w < n_windows; w++) {
    const int32_t* q = &inf[5 * w];
    submap_window(W, h->cfg.resolution, m, windows + 4 * w, &inf[5 * w], &cen[2 * w]);
    if (q[0]) submap_add(a, W, q, n_layers, tiles, total);
  }
  if (total > out_floats)
    return fail(h, EMAP_ERR_INVALID, "emap_get_submaps: out_floats is below the layers times the windows' cells");
  memcpy(info, inf.data(), sizeof(int32_t) * inf.size());
  memcpy(centres, cen.data(), sizeof(double) * cen.size());
  if (!a.n_win) return EMAP_OK;
  float* dst = out;
  if (!out_is_device) {
    const int rc = grow(h, h->d_export, (size_t)total, 0, false);
    if (rc) return rc;
    dst = h->d_export;
  }
  const auto kern = export_has_colour(a.L) ? k_submap<true> : k_submap<false>;
  kern<<<dim3(tiles, n_layers), dim3(32, SUBMAP_ROWS), 0, h->stream>>>(h->dc, h->map, h->normal, dst, a, h->center[2],
                                                                       h->cfg.use_only_above_for_upper_bound);
  LAUNCH_CHECK();
  if (!out_is_device) {
    CK(cudaMemcpyAsync(out, dst, sizeof(float) * total, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}

static_assert(EMAP_TRANSFORM_TOLERANCE == TSUB_ORTHO_TOL && EMAP_TRANSFORMED_WINDOWS_PER_LAUNCH == TSUB_MAX_WINDOWS,
              "emap.h states the transformed windows' limits");

static bool transforms_ok(int64_t n, const double* transforms) {
  for (int64_t w = 0; w < n; w++)
    if (!tsub_transform_ok(transforms + 12 * w)) return false;
  return true;
}

// The host part of emap_get_transformed_submaps on its own (no handle, no device): transformed_window for every request.
int emap_transformed_submap_windows(int32_t cell_n, double resolution, const double center[2], int32_t n_windows,
                                    const double* windows, const double* transforms, int32_t* info, double* geometry) {
  if (!center || !windows || !transforms || !info || !geometry || cell_n < 3 ||
      !(std::isfinite(resolution) && resolution > 0.0) || n_windows < 0 || !submap_lengths_ok(n_windows, windows) ||
      !transforms_ok(n_windows, transforms))
    return EMAP_ERR_INVALID;
  for (int32_t w = 0; w < n_windows; w++) {
    TSubGeom g;
    transformed_window(cell_n, resolution, center, windows + 4 * w, transforms + 12 * w, g);
    info[3 * w] = g.win[0]; info[3 * w + 1] = g.size[0]; info[3 * w + 2] = g.size[1];
    for (int a = 0; a < 2; a++) { geometry[4 * w + a] = g.pos[a]; geometry[4 * w + 2 + a] = g.len[a]; }
  }
  return EMAP_OK;
}

// get_raw_submap with a request frame other than the map frame (elevation_mapping_ros.cpp:507-553 with grid_map's
// getTransformedMap): the geometry on the host (transformed_window), then per launch of up to TSUB_MAX_WINDOWS windows
// the two scatter passes and the gather (csrc/emap_submap.cuh), each launch's table in its parameters.  Output, stream
// and graph rules as emap_get_submaps; every check runs before anything is written or launched.
int emap_get_transformed_submaps(emap_handle* h, int32_t n_windows, const double* windows, const double* transforms,
                                 double sample_ratio, int32_t n_layers, const char* const* names,
                                 const float* const* planes_device, const int32_t* flags, float* out,
                                 int32_t out_is_device, int64_t out_floats, int32_t* info, double* geometry) {
  ENTER(h);
  NvtxRange nv("emap:get_transformed_submaps");
  if (!windows || !transforms || !names || !out || !info || !geometry)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: null argument");
  if (n_windows < 1 || n_windows > EMAP_SUBMAP_MAX_WINDOWS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: 1 to EMAP_SUBMAP_MAX_WINDOWS windows required");
  if (n_layers < 1 || n_layers > EMAP_SUBMAP_MAX_LAYERS)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: 1 to EMAP_SUBMAP_MAX_LAYERS layers required");
  if (!submap_lengths_ok(n_windows, windows))
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: lengths must be finite and >= 0");
  if (!transforms_ok(n_windows, transforms))
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: a transform is not finite or its R is not "
                                     "orthonormal within EMAP_TRANSFORM_TOLERANCE");
  if (!(std::isfinite(sample_ratio) && sample_ratio >= 0.0))
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: sample_ratio must be finite and >= 0");
  ExportList L;
  if (!export_list(h, n_layers, names, planes_device, flags, L)) return EMAP_ERR_INVALID;
  const int W = h->dc.W;
  const double res = h->cfg.resolution;
  const double m[2] = {h->center[0], h->center[1]};
  std::vector<TSubGeom> g(n_windows);
  long long cells = 0;
  for (int w = 0; w < n_windows; w++) {
    transformed_window(W, res, m, windows + 4 * w, transforms + 12 * w, g[w]);
    const long long n = (long long)g[w].size[0] * g[w].size[1];
    if (n > INT32_MAX - TSUB_THREADS)
      return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: a new map of 2^31 cells or more");
    cells += n;
  }
  if (n_layers * cells > out_floats)
    return fail(h, EMAP_ERR_INVALID, "emap_get_transformed_submaps: out_floats is below the layers times the new maps' cells");
  for (int w = 0; w < n_windows; w++) {
    info[3 * w] = g[w].win[0]; info[3 * w + 1] = g[w].size[0]; info[3 * w + 2] = g[w].size[1];
    for (int a = 0; a < 2; a++) { geometry[4 * w + a] = g[w].pos[a]; geometry[4 * w + 2 + a] = g[w].len[a]; }
  }
  if (!cells) return EMAP_OK;
  int rc;
  if ((rc = grow(h, h->ts_key1, (size_t)cells, 0, true)) || (rc = grow(h, h->ts_key2, (size_t)cells, 0, true))) return rc;
  float* dst = out;
  if (!out_is_device) {
    if ((rc = grow(h, h->d_export, (size_t)(n_layers * cells), 0, false))) return rc;
    dst = h->d_export;
  }
  const bool colour = export_has_colour(L);
  TSubArgs a;
  a.L = L;
  a.n_samples = sample_ratio > 0.0 ? 5 : 1;
  a.res = res;
  a.s = res * sample_ratio;
  long long cell0 = 0;
  for (int w0 = 0; w0 < n_windows;) {
    a.n_win = 0;
    int blk_src = 0, blk_dst = 0;
    for (; w0 < n_windows && a.n_win < TSUB_MAX_WINDOWS; w0++) {
      const TSubGeom& q = g[w0];
      if (!q.win[0] || !q.size[0] || !q.size[1]) continue;
      TSubWin& s = a.win[a.n_win++];
      for (int k = 0; k < 9; k++) s.R[k] = transforms[12 * w0 + k];
      for (int k = 0; k < 3; k++) s.t[k] = transforms[12 * w0 + 9 + k];
      s.x0 = q.centre[0] + (0.5 * (q.win[3] * res) - 0.5 * res);
      s.y0 = q.centre[1] + (0.5 * (q.win[4] * res) - 0.5 * res);
      for (int k = 0; k < 2; k++) { s.pos[k] = q.pos[k]; s.len[k] = q.len[k]; }
      s.r0 = (int16_t)(W - 2 - q.win[1]); s.c0 = (int16_t)(W - 2 - q.win[2]);
      s.rows = (int16_t)q.win[3]; s.cols = (int16_t)q.win[4];
      s.nrows = q.size[0]; s.ncols = q.size[1];
      s.blk_src = blk_src; s.blk_dst = blk_dst; s.cell0 = cell0;
      blk_src += cdiv((i64)q.win[3] * q.win[4], TSUB_THREADS);
      blk_dst += cdiv((i64)q.size[0] * q.size[1], TSUB_THREADS);
      cell0 += (long long)q.size[0] * q.size[1];
    }
    if (!a.n_win) continue;
    k_tsub_scatter<1><<<blk_src, TSUB_THREADS, 0, h->stream>>>(h->dc, h->map, h->ts_key1, h->ts_key2, a, h->center[2]);
    LAUNCH_CHECK();
    k_tsub_scatter<2><<<blk_src, TSUB_THREADS, 0, h->stream>>>(h->dc, h->map, h->ts_key1, h->ts_key2, a, h->center[2]);
    LAUNCH_CHECK();
    const auto gather = colour ? k_tsub_gather<true> : k_tsub_gather<false>;
    gather<<<blk_dst, TSUB_THREADS, 0, h->stream>>>(h->dc, h->map, h->normal, h->ts_key1, h->ts_key2, dst, a,
                                                    h->center[2], h->cfg.use_only_above_for_upper_bound);
    LAUNCH_CHECK();
  }
  if (!out_is_device) {
    CK(cudaMemcpyAsync(out, dst, sizeof(float) * n_layers * cells, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return EMAP_OK;
}

// ---- plane segmentation of one window (emap_segment_planes, csrc/emap_planes.cuh) ----------------------------------

// The scratch of a window of n cells with `slots` label slots, one block: the window, two image planes (fill / median
// ping-pong), union-find parents, flags and ranks, fill keys, the planarity masks, scan block sums, the header words,
// the label statistics and decisions, and the host output's staging (info, plane table, layers).
namespace {

struct PlaneScratch {
  float *raw, *img[2];
  int *parent, *flag, *rank, *lab, *bsum, *hdr, *keep;
  unsigned* key;
  unsigned char *bin, *tmp, *bg;
  unsigned long long* st;
  int32_t* info;
  double* planes;
  float* layers;
};

size_t carve_planes(int64_t n, int64_t slots, int64_t plane_rows, bool host_out, void* base, PlaneScratch& s) {
  Carver c{(uintptr_t)base};
  const int64_t m = std::max(n, slots);
  s.raw = c.take<float>(n); s.img[0] = c.take<float>(n); s.img[1] = c.take<float>(n);
  s.parent = c.take<int>(n); s.flag = c.take<int>(m); s.rank = c.take<int>(m); s.lab = c.take<int>(n);
  s.bsum = c.take<int>(m / PL_SCAN + 1); s.hdr = c.take<int>(8); s.keep = c.take<int>(slots);
  s.key = c.take<unsigned>(n);
  s.bin = c.take<unsigned char>(n); s.tmp = c.take<unsigned char>(n); s.bg = c.take<unsigned char>(slots);
  s.st = c.take<unsigned long long>(slots * PL_STAT);
  s.info = c.take<int32_t>(host_out ? 8 : 0);
  s.planes = c.take<double>(host_out ? 7 * plane_rows : 0);
  s.layers = c.take<float>(host_out ? 4 * n : 0);
  return c.bytes;
}

// Raster-order ranks of the n flags in s.flag into s.rank, the count into *total (three launches).
int plane_scan(emap_handle* h, const PlaneScratch& s, int64_t n, int* total) {
  const int nb = cdiv(n, PL_SCAN);
  k_pl_scan_blocks<<<nb, PL_SCAN, 0, h->stream>>>(s.flag, (int)n, s.bsum);
  LAUNCH_CHECK();
  k_pl_scan_top<<<1, PL_SCAN, 0, h->stream>>>(s.bsum, nb, total);
  LAUNCH_CHECK();
  k_pl_scan_rank<<<nb, PL_SCAN, 0, h->stream>>>(s.flag, (int)n, s.bsum, s.rank);
  LAUNCH_CHECK();
  return 0;
}

// Union-find merge and flatten of the cells whose parent is >= 0.
int plane_components(emap_handle* h, const PlaneScratch& s, int rows, int cols, int conn8) {
  const int64_t n = (int64_t)rows * cols;
  k_pl_uf_merge<<<cdiv(n, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.parent, rows, cols, conn8);
  LAUNCH_CHECK();
  k_pl_uf_flatten<<<cdiv(n, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.parent, (int)n);
  LAUNCH_CHECK();
  return 0;
}

}  // namespace

static_assert(EMAP_PLANE_EIGEN_MIN == PL_EIG_MIN, "emap.h states the fit's threshold");

// Why p is rejected (nullptr: accepted) for a map of resolution `res`.
static const char* plane_params_error(const emap_plane_params& p, double res) {
  if (p.ransac) return "emap_segment_planes: RANSAC refinement is not supported (ransac must be 0)";
  const int mk = std::max(1, std::min(p.median_kernel, 5));
  if (mk != 1 && mk != 3 && mk != 5) return "emap_segment_planes: the median kernel must clamp to 1, 3 or 5";
  if (p.median_repeats < 0 || p.median_repeats > EMAP_PLANE_MAX_REPEATS)
    return "emap_segment_planes: median_repeats must be in [0, EMAP_PLANE_MAX_REPEATS]";
  if (std::isnan(p.resolution) || (p.resolution > 0.0 && !(std::fabs(res - p.resolution) < 1e-6)))
    return "emap_segment_planes: resampling is not supported (resolution must be <= 0 or the map's)";
  if (p.kernel_size < 3 || p.kernel_size % 2 == 0 || p.kernel_size > EMAP_PLANE_MAX_KERNEL)
    return "emap_segment_planes: kernel_size must be odd, >= 3 and <= EMAP_PLANE_MAX_KERNEL";
  if (p.opening < 0 || p.opening > EMAP_PLANE_MAX_OPENING)
    return "emap_segment_planes: opening must be in [0, EMAP_PLANE_MAX_OPENING]";
  if (p.connectivity != 4 && p.connectivity != 8) return "emap_segment_planes: connectivity must be 4 or 8";
  if (!std::isfinite(p.plane_inclination_cos) || !std::isfinite(p.local_inclination_cos) ||
      !std::isfinite(p.patch_error))
    return "emap_segment_planes: the inclination cosines and the patch error must be finite";
  return nullptr;
}

int64_t emap_plane_capacity(int64_t rows, int64_t cols, const emap_plane_params* params) {
  if (!params || rows < 0 || cols < 0) return -1;
  return rows * cols / std::max(params->min_points, 3);
}

// The plane decomposition node's segmented planes map for one window (ConvexPlaneDecompositionRos.cpp:115-149 up to
// SlidingWindowPlaneExtractor, without RANSAC): the window by k_submap, then the passes of csrc/emap_planes.cuh.  Host
// output: the copies and one synchronisation; device output: stream-ordered, no synchronisation.  Every check runs
// before anything is written or launched.
int emap_segment_planes(emap_handle* h, const double window[4], const emap_plane_params* params, float* layers_out,
                        int32_t out_is_device, int64_t out_floats, double* planes_out, int64_t planes_capacity,
                        int32_t* info) {
  ENTER(h);
  NvtxRange nv("emap:segment_planes");
  if (!window || !params || !layers_out || !planes_out || !info)
    return fail(h, EMAP_ERR_INVALID, "emap_segment_planes: null argument");
  if (!submap_lengths_ok(1, window)) return fail(h, EMAP_ERR_INVALID, "emap_segment_planes: lengths must be finite and >= 0");
  const emap_plane_params p = *params;
  const double res = h->cfg.resolution;
  if (const char* e = plane_params_error(p, res)) return fail(h, EMAP_ERR_INVALID, e);
  const int W = h->dc.W;
  const double m[2] = {h->center[0], h->center[1]};
  int32_t q[5];
  double centre[2];
  submap_window(W, res, m, window, q, centre);
  const int rows = q[3], cols = q[4];
  const int64_t n = (int64_t)rows * cols;
  if (q[0] && out_floats < 4 * n)
    return fail(h, EMAP_ERR_INVALID, "emap_segment_planes: out_floats is below 4 * rows * cols");
  const int64_t plane_rows = emap_plane_capacity(rows, cols, &p);
  if (q[0] && planes_capacity < plane_rows)
    return fail(h, EMAP_ERR_INVALID, "emap_segment_planes: planes_capacity is below emap_plane_capacity()");
  if (!q[0]) {
    if (out_is_device) CK(cudaMemsetAsync(info, 0, 5 * sizeof(int32_t), h->stream));
    else memset(info, 0, 5 * sizeof(int32_t));
    return EMAP_OK;
  }
  // labels are at most ceil(n / 2) (a 4-connected checkerboard), plus 0.  The statistics are sized and zeroed for that
  // worst case (128 bytes a slot) because the label count is known only on the device.
  const int64_t slots = n / 2 + 2;
  PlaneScratch s;
  int rc = grow(h, h->pl_block, carve_planes(n, slots, plane_rows, !out_is_device, nullptr, s), 0, false);
  if (rc) return rc;
  const size_t used = carve_planes(n, slots, plane_rows, !out_is_device, h->pl_block, s);
  float* dst = out_is_device ? layers_out : s.layers;
  double* dst_planes = out_is_device ? planes_out : s.planes;
  int32_t* dst_info = out_is_device ? info : s.info;
  // the window: k_submap's elevation layer into s.raw
  SubmapArgs a;
  const char* elevation = "elevation";
  if (!export_list(h, 1, &elevation, nullptr, nullptr, a.L)) return EMAP_ERR_CUDA;
  a.n_win = 0;
  int tiles = 0;
  long long total = 0;
  submap_add(a, W, q, 1, tiles, total);
  k_submap<false><<<dim3(tiles, 1), dim3(32, SUBMAP_ROWS), 0, h->stream>>>(h->dc, h->map, h->normal, s.raw, a, h->center[2],
                                                                           h->cfg.use_only_above_for_upper_bound);
  LAUNCH_CHECK();
  CK(cudaMemsetAsync(s.hdr, 0, 8 * sizeof(int), h->stream));
  CK(cudaMemsetAsync(s.st, 0, sizeof(unsigned long long) * slots * PL_STAT, h->stream));
  const int cb = cdiv(n, PL_THREADS);
  // fill: minValues' fixed point per NaN component
  k_pl_fill_init<<<cb, PL_THREADS, 0, h->stream>>>(s.raw, s.parent, s.key, s.hdr, (int)n);
  LAUNCH_CHECK();
  if ((rc = plane_components(h, s, rows, cols, 0))) return rc;
  k_pl_fill_min<<<cb, PL_THREADS, 0, h->stream>>>(s.raw, s.parent, s.key, rows, cols);
  LAUNCH_CHECK();
  k_pl_fill_write<<<cb, PL_THREADS, 0, h->stream>>>(s.raw, s.parent, s.key, s.img[0], (int)n);
  LAUNCH_CHECK();
  // median, numberOfRepeats times
  const int mk = std::max(1, std::min(p.median_kernel, 5));
  int cur = 0;
  if (mk > 1)
    for (int r = 0; r < p.median_repeats; r++, cur ^= 1) {
      (mk == 3 ? k_pl_median<3> : k_pl_median<5>)<<<cb, PL_THREADS, 0, h->stream>>>(s.img[cur], s.img[cur ^ 1], rows, cols);
      LAUNCH_CHECK();
    }
  const float* img = s.img[cur];
  // sliding-window planarity, opening, labels
  k_pl_fit<<<cb, PL_THREADS, 0, h->stream>>>(img, s.bin, rows, cols, p.kernel_size, res, p.patch_error * p.patch_error,
                                             p.local_inclination_cos);
  LAUNCH_CHECK();
  if (p.opening > 0) {
    k_pl_morph<false><<<cb, PL_THREADS, 0, h->stream>>>(s.bin, s.tmp, rows, cols, p.opening);
    LAUNCH_CHECK();
    k_pl_morph<true><<<cb, PL_THREADS, 0, h->stream>>>(s.tmp, s.bin, rows, cols, p.opening);
    LAUNCH_CHECK();
  }
  k_pl_cc_init<<<cb, PL_THREADS, 0, h->stream>>>(s.bin, s.parent, s.key, s.flag, (int)n);
  LAUNCH_CHECK();
  const bool conn8 = p.connectivity == 8;
  if ((rc = plane_components(h, s, rows, cols, conn8))) return rc;
  (conn8 ? k_pl_first<2> : k_pl_first<1>)<<<cb, PL_THREADS, 0, h->stream>>>(s.parent, s.key, rows, cols);
  LAUNCH_CHECK();
  k_pl_first_flag<<<cb, PL_THREADS, 0, h->stream>>>(s.parent, s.key, s.flag, (int)n);
  LAUNCH_CHECK();
  const int64_t n_blocks = conn8 ? (int64_t)cdiv(rows, 2) * cdiv(cols, 2) : n;
  if ((rc = plane_scan(h, s, n_blocks, s.hdr + 1))) return rc;
  k_pl_label<<<cb, PL_THREADS, 0, h->stream>>>(s.parent, s.key, s.rank, s.lab, (int)n);
  LAUNCH_CHECK();
  // per-label planes
  k_pl_stats<<<cdiv(cdiv(n, PL_RUN), PL_THREADS), PL_THREADS, 0, h->stream>>>(img, s.lab, s.st, rows, cols);
  LAUNCH_CHECK();
  const PlaneLabelArgs la = {centre[0] + (0.5 * (rows * res) - 0.5 * res), centre[1] + (0.5 * (cols * res) - 0.5 * res),
                             res, p.plane_inclination_cos, p.min_points};
  k_pl_decide<<<cdiv(slots, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.st, s.hdr, s.flag, s.bg, (int)slots, la);
  LAUNCH_CHECK();
  if ((rc = plane_scan(h, s, slots, s.hdr + 2))) return rc;
  k_pl_planes<<<cdiv(slots, PL_THREADS), PL_THREADS, 0, h->stream>>>(s.st, s.rank, s.hdr, dst_planes, (int)slots, la);
  LAUNCH_CHECK();
  k_pl_out<<<cb, PL_THREADS, 0, h->stream>>>(s.raw, img, s.lab, s.bg, s.hdr, dst, dst_info, rows, cols);
  LAUNCH_CHECK();
  if (!out_is_device) {
    // info, the plane table and the layers are the block's tail: one copy, one synchronisation, and the caller's
    // buffers take the layers and planes only when the window had a finite cell
    const size_t off = (char*)s.info - (char*)h->pl_block, bytes = used - off;
    if (h->pl_host.size() < bytes) CK(h->pl_host.alloc(bytes));
    CK(cudaMemcpyAsync(h->pl_host, s.info, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    PlaneScratch t;
    carve_planes(n, slots, plane_rows, true, (char*)h->pl_host - off, t);
    memcpy(info, t.info, 5 * sizeof(int32_t));
    if (info[0]) {
      memcpy(planes_out, t.planes, sizeof(double) * 7 * info[4]);
      memcpy(layers_out, t.layers, sizeof(float) * 4 * n);
    }
  }
  return EMAP_OK;
}

// The node's publishAsPointCloud (elevation_mapping_ros.cpp:501-505): the points of the exported elevation (map_cloud).
int emap_get_map_points(emap_handle* h, float* xyz_host, int64_t* n_points) {
  ENTER(h);
  NvtxRange nv("emap:get_map_points");
  if (!n_points || *n_points < 0 || (*n_points > 0 && !xyz_host))
    return fail(h, EMAP_ERR_INVALID, "emap_get_map_points: null argument or negative capacity");
  return map_cloud<false>(h, n_points, xyz_host, nullptr, nullptr);
}

// The node's publishNormalAsArrow (elevation_mapping_ros.cpp:751-778): the arrows of the exported normals (map_cloud).
int emap_get_normal_arrows(emap_handle* h, int32_t* ids_host, double* segments_host, int64_t* n_arrows) {
  ENTER(h);
  NvtxRange nv("emap:get_normal_arrows");
  if (!n_arrows || *n_arrows < 0 || (*n_arrows > 0 && (!ids_host || !segments_host)))
    return fail(h, EMAP_ERR_INVALID, "emap_get_normal_arrows: null argument or negative capacity");
  return map_cloud<true>(h, n_arrows, nullptr, ids_host, segments_host);
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

// EM.py:837-889 get_polygon_traversability (WRAP:254-281): area, clip and bounding box on the host in fp32, then a
// batch of one polygon whose work items are every tile of the grid (the mask is written everywhere, and the statistics
// need no poison pass), one device-to-host copy and one synchronisation.
int emap_polygon_traversability(emap_handle* h, const float* polygon_xy, int32_t n_vertices, const float* checker_plane,
                                double safe_thresh, double safe_min_thresh, int32_t max_unsafe_n, double result[3],
                                double* hull_xy, int32_t* n_hull, float* mask) {
  ENTER(h);
  if (!polygon_xy || !result || !n_hull || *n_hull < 0 || (*n_hull > 0 && !hull_xy))
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability: null argument or negative hull capacity");
  if (n_vertices < 3 || n_vertices > EMAP_POLYGON_MAX_VERTICES)
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability: 3 to EMAP_POLYGON_MAX_VERTICES vertices required");
  const int W = h->dc.W;
  const dim3 g = polygon_grid(W);
  const PolyStage st = poly_stage(1, n_vertices, ring_capacity(W));
  PolySizes z;
  z.up = st.up_bytes; z.items = (size_t)g.x * g.y; z.cols = W - 2; z.down = st.down_bytes;
  PolyScratch s;
  int rc = alloc_polygon_scratch(h, z, s);
  if (rc) return rc;
  const float area = shoelace_f32(polygon_xy, n_vertices);
  PolyDesc d = {};
  float2* xy = (float2*)(h->pg_host + st.xy);
  clip_polygon(W, h->cfg.resolution, h->center, polygon_xy, n_vertices, xy, d.bbox);
  const float clipped_area = shoelace_f32((const float*)xy, n_vertices);
  d.v0 = 0; d.n = n_vertices; d.item0 = 0;
  d.tr0 = 0; d.tc0 = 0; d.n_tr = g.y; d.n_tc = g.x;
  d.col0 = 0; d.n_col = W - 2; d.col_off = 0; d.ring_off = 0;
  memcpy(h->pg_host + st.desc, &d, sizeof(d));
  rc = run_polygons(h, s, st, 1, (int)z.items, false, checker_plane, safe_thresh, safe_min_thresh, max_unsafe_n, mask,
                    true, kRingHead);
  if (rc) return rc;
  const char* back = h->pg_host + h->pg_cap.up;
  PolyResult r;
  memcpy(&r, back, sizeof(r));
  const double2* ring = (const double2*)(back + st.ring);
  // EM.py:884-887: a polygon (almost) entirely outside the map is unsafe
  result[0] = (r.is_safe && !(clipped_area < 0.001f)) ? 1.0 : 0.0;
  result[1] = r.t;
  result[2] = (double)area;
  if (r.n_ring > *n_hull) {
    *n_hull = r.n_ring;
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability: hull capacity too small (needed length in *n_hull)");
  }
  for (int k = 0; k < r.n_ring; k++) { hull_xy[2 * k] = ring[k].x; hull_xy[2 * k + 1] = ring[k].y; }
  *n_hull = r.n_ring;
  return EMAP_OK;
}

// The check_safety service (CheckSafety.srv) in one call: every polygon's answer is emap_polygon_traversability's.  The
// work items are only the tiles of each polygon's cell bounding box; k_poly_poison carries the map-wide NaN rule to
// the cells outside them.  One upload, one read-back copy and one synchronisation (plus one for long rings).
int emap_polygon_traversability_batch(emap_handle* h, int32_t n_polygons, const int32_t* n_vertices,
                                      const float* polygon_xy, const float* checker_plane, double safe_thresh,
                                      double safe_min_thresh, int32_t max_unsafe_n, double* results, double* hull_xy,
                                      int64_t* hull_offsets, int64_t* hull_rows) {
  ENTER(h);
  if (n_polygons < 1 || n_polygons > EMAP_POLYGON_MAX_BATCH)
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability_batch: 1 to EMAP_POLYGON_MAX_BATCH polygons required");
  if (!n_vertices || !polygon_xy || !results || (hull_xy && (!hull_offsets || !hull_rows)) ||
      (hull_rows && *hull_rows < 0))
    return fail(h, EMAP_ERR_INVALID, "emap_polygon_traversability_batch: null argument or negative hull capacity");
  size_t n_vert = 0;
  for (int i = 0; i < n_polygons; i++) {
    if (n_vertices[i] < 3 || n_vertices[i] > EMAP_POLYGON_MAX_VERTICES)
      return fail(h, EMAP_ERR_INVALID,
                  "emap_polygon_traversability_batch: 3 to EMAP_POLYGON_MAX_VERTICES vertices required per polygon");
    n_vert += n_vertices[i];
  }
  const bool hulls = hull_xy != nullptr;
  // traversability_polygon.py:25 compares the whole interior: with fp32(1 - safe_thresh) < 0 the masked 0 of every cell
  // outside a polygon is over too, so its count and hull take the whole map.  Every polygon then brings every tile and
  // the whole column window, as the single call does.
  const bool whole_map = (float)(1.0 - safe_thresh) < 0.0f;
  const dim3 g = polygon_grid(h->dc.W);
  // each polygon's tiles (its work items and partials), column window and ring slot
  std::vector<PolyDesc> desc(n_polygons);
  size_t items = 0, cols = 0, rows = 0, v0 = 0;
  for (int i = 0; i < n_polygons; i++) {
    PolyDesc& d = desc[i];
    clip_polygon(h->dc.W, h->cfg.resolution, h->center, polygon_xy + 2 * v0, n_vertices[i], nullptr, d.bbox);
    polygon_tiles(h->dc.W, h->cfg.resolution, h->center, d);
    if (whole_map) {
      d.tr0 = 0; d.tc0 = 0; d.n_tr = g.y; d.n_tc = g.x;
      d.col0 = 0; d.n_col = h->dc.W - 2;
    }
    if (!hulls) d.n_col = 0;
    d.v0 = (int)v0; d.n = n_vertices[i]; d.item0 = (int)items; d.col_off = (int)cols; d.ring_off = (int)rows;
    items += (size_t)d.n_tr * d.n_tc;
    cols += d.n_col;
    rows += d.n_col ? 2 * (size_t)d.n_col + 1 : 0;
    v0 += n_vertices[i];
  }
  const PolyStage st = poly_stage(n_polygons, n_vert, rows);
  PolySizes z;
  z.up = st.up_bytes; z.items = items; z.cols = cols; z.down = st.down_bytes;
  PolyScratch s;
  int rc = alloc_polygon_scratch(h, z, s);
  if (rc) return rc;
  memset(h->pg_host, 0, st.desc);                                   // the poison counts start at zero
  memcpy(h->pg_host + st.desc, desc.data(), sizeof(PolyDesc) * n_polygons);
  float2* xy = (float2*)(h->pg_host + st.xy);
  std::vector<float> area(n_polygons), clipped_area(n_polygons);
  for (int i = 0; i < n_polygons; i++) {
    const PolyDesc& d = desc[i];
    area[i] = shoelace_f32(polygon_xy + 2 * (size_t)d.v0, d.n);
    float bbox[4];
    clip_polygon(h->dc.W, h->cfg.resolution, h->center, polygon_xy + 2 * (size_t)d.v0, d.n, xy + d.v0, bbox);
    clipped_area[i] = shoelace_f32((const float*)(xy + d.v0), d.n);
  }
  rc = run_polygons(h, s, st, n_polygons, (int)items, true, checker_plane, safe_thresh, safe_min_thresh, max_unsafe_n,
                    nullptr, hulls, kBatchRingHead);
  if (rc) return rc;
  const char* back = h->pg_host + h->pg_cap.up;
  const PolyResult* r = (const PolyResult*)back;
  const double2* ring = (const double2*)(back + st.ring);
  int64_t total = 0;
  for (int i = 0; i < n_polygons; i++) {
    // EM.py:884-887: a polygon (almost) entirely outside the map is unsafe
    results[3 * i] = (r[i].is_safe && !(clipped_area[i] < 0.001f)) ? 1.0 : 0.0;
    results[3 * i + 1] = r[i].t;
    results[3 * i + 2] = (double)area[i];
    if (hull_offsets) hull_offsets[i] = total;
    total += r[i].n_ring;
  }
  if (hull_offsets) hull_offsets[n_polygons] = total;
  if (!hulls) {
    if (hull_rows) *hull_rows = 0;
    return EMAP_OK;
  }
  if (total > *hull_rows) {
    *hull_rows = total;
    return fail(h, EMAP_ERR_INVALID,
                "emap_polygon_traversability_batch: hull capacity too small (needed rows in *hull_rows)");
  }
  for (int i = 0; i < n_polygons; i++) {
    const double2* src = ring + desc[i].ring_off;
    double* dst = hull_xy + 2 * hull_offsets[i];
    for (int k = 0; k < r[i].n_ring; k++) { dst[2 * k] = src[k].x; dst[2 * k + 1] = src[k].y; }
  }
  *hull_rows = total;
  return EMAP_OK;
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
int emap_min_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                    int32_t* iterations_run) {
  ENTER(h);
  return minmax_filter<false>(h, elevation, is_valid, out, k, iteration_n, iterations_run);
}

int emap_max_filter(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t k, int32_t iteration_n,
                    int32_t* iterations_run) {
  ENTER(h);
  return minmax_filter<true>(h, elevation, is_valid, out, k, iteration_n, iterations_run);
}

int emap_erode(emap_handle* h, const float* layer, float* out, int32_t kernel_size, int32_t iterations, int32_t reverse) {
  ENTER(h);
  if (!layer || !out || kernel_size < 1 || kernel_size > 31 || iterations < 1 || iterations > 64)
    return fail(h, EMAP_ERR_INVALID, "emap_erode: bad argument");
  int rc;
  if ((rc = alloc_plugin_scratch(h)) || (rc = grow(h, h->pl_cnt, 2, 30, false))) return rc;
  u32* const mm = (u32*)(int*)h->pl_cnt;      // min / max of the layer
  const u32 init[2] = {0xffffffffu, 0u};
  CK(cudaMemcpyAsync(mm, init, sizeof(init), cudaMemcpyHostToDevice, h->stream));
  PER_CELL(k_layer_minmax, h->dc, layer, reverse, mm);
  const int ks = kernel_size + (iterations - 1) * (kernel_size - 1), anchor = (kernel_size / 2) * iterations;
  const float* src = layer;
  if (layer == out) {        // in-place call: erode from a copy
    CK(cudaMemcpyAsync(h->pl[0], layer, sizeof(float) * (size_t)h->dc.C, cudaMemcpyDeviceToDevice, h->stream));
    src = h->pl[0];
  }
  PER_CELL(k_erode, h->dc, src, out, ks, anchor, reverse, (const u32*)mm);
  return EMAP_OK;
}

int emap_robot_centric_elevation(emap_handle* h, const float* elevation, const float* is_valid, const float R[9], float* out,
                                 double resolution, double threshold, int32_t use_threshold) {
  ENTER(h);
  if (!elevation || !is_valid || !R || !out) return fail(h, EMAP_ERR_INVALID, "null argument");
  PER_CELL(k_robot_centric, h->dc, elevation, is_valid, out, R[6], R[7], R[8], resolution, threshold, use_threshold);
  return EMAP_OK;
}

int emap_smooth_filter(emap_handle* h, const float* in, float* out) {
  ENTER(h);
  if (!in || !out) return fail(h, EMAP_ERR_INVALID, "null argument");
  int rc = alloc_plugin_scratch(h);
  if (rc) return rc;
  PER_CELL(k_box3, h->dc, in, h->pl[0], 0);
  PER_CELL(k_box3, h->dc, h->pl[0], h->pl[1], 1);
  PER_CELL(k_box3, h->dc, h->pl[1], h->pl[0], 0);
  PER_CELL(k_box3, h->dc, h->pl[0], out, 1);
  return EMAP_OK;
}

// plugins/inpainting.py:53-63: 8-bit normalisation, cv.inpaint(h, mask, 1, INPAINT_TELEA), de-normalisation -- OpenCV's
// fast-marching fill replayed on the device in parallel (emap_inpaint.cuh), bit-identical to cv2's result.
int emap_inpaint(emap_handle* h, const float* elevation, const float* is_valid, float* out, int32_t method) {
  ENTER(h);
  NvtxRange nv("emap:inpaint");
  if (!elevation || !is_valid || !out) return fail(h, EMAP_ERR_INVALID, "emap_inpaint: null argument");
  if (method != 0) return fail(h, EMAP_ERR_INVALID, "emap_inpaint: only method 0 (telea) is implemented; 'ns' (Navier-Stokes) is not");
  const int W = h->dc.W;
  const size_t N = (size_t)(W + 2) * (W + 2), C = (size_t)W * W;
  // zero-filled once: the march loads a pixel's child fields (ck, Tc, vc) speculatively, before it knows the pixel is a
  // child of the running round; the values of non-children are never used, but they should not be uninitialised memory
  int rc = grow(h, h->ip_block, inpaint_scratch(W, nullptr).bytes, 0, true);
  if (rc) return rc;
  if (!h->ip_grid) {
    int nb = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_ip_march, IP_MARCH_THREADS, 0));
    if (nb < 1) return fail(h, EMAP_ERR_CUDA, "emap_inpaint: the cooperative kernel does not fit on an SM");
    h->ip_grid = h->n_sm;          // one CTA per SM: the fronts are thin, and a grid barrier costs less with fewer CTAs
  }
  InpaintScratch s = inpaint_scratch(W, h->ip_block);
  InpaintView& v = s.v;
  InpaintCtl* ctl = s.ctl;
  InpaintCtl init;
  memset(&init, 0, sizeof(init));
  init.mm[0] = 0xffffffffu; init.mm[1] = 0u;
  CK(cudaMemcpyAsync(ctl, &init, sizeof(init), cudaMemcpyHostToDevice, h->stream));     // pageable: staged before return
  const int nbN = cdiv((i64)N, 256);
  PER_CELL(k_ip_minmax, (int)C, elevation, is_valid, ctl);
  k_ip_init<<<nbN, 256, 0, h->stream>>>(W, elevation, is_valid, v, (const InpaintCtl*)ctl); LAUNCH_CHECK();
  k_ip_band<<<nbN, 256, 0, h->stream>>>(v, s.heap[0], ctl); LAUNCH_CHECK();
  k_ip_band_flag<<<nbN, 256, 0, h->stream>>>(v, (const int*)s.heap[0], ctl); LAUNCH_CHECK();
  {
    int cap = 4096;
    void* args[] = {(void*)&v, (void*)&s.heap[0], (void*)&s.heap[1], (void*)&s.children, (void*)&ctl, (void*)&cap};
    CK(cudaLaunchCooperativeKernel((const void*)k_ip_march, dim3(h->ip_grid), dim3(IP_MARCH_THREADS), args, 0, h->stream));
    h->launches++;
  }
  PER_CELL(k_ip_finish, (int)C, (const uint8_t*)v.img, elevation, out, (const InpaintCtl*)ctl);
  return EMAP_OK;
}

// plugins/semantic_filter.py:89-133: argmax over the planes, palette entry of the class id (bits)
int emap_semantic_filter(emap_handle* h, int32_t n_layers, const float* const* planes, float* out) {
  ENTER(h);
  if (!out || n_layers < 0 || n_layers > EMAP_SEMANTIC_FILTER_MAX_LAYERS || !planes_ok(n_layers, planes))
    return fail(h, EMAP_ERR_INVALID, "emap_semantic_filter: 0 to EMAP_SEMANTIC_FILTER_MAX_LAYERS non-null planes and a non-null output required");
  SemFilterArgs a;
  memset(&a, 0, sizeof(a));
  a.n = n_layers;
  for (int l = 0; l < n_layers; l++) a.plane[l] = planes[l];
  PER_CELL(k_semantic_filter, h->dc.C, a, (u32*)out);
  return EMAP_OK;
}

// plugins/semantic_traversability.py:59-83: per-layer threshold votes (fp64 comparisons), fp32(0.1) or 1
int emap_semantic_traversability(emap_handle* h, int32_t n_layers, const float* const* planes, const double* thresholds,
                                 const int32_t* is_traversability_type, float* out) {
  ENTER(h);
  if (!out || n_layers < 0 || n_layers > EMAP_SEMANTIC_TRAVERSABILITY_MAX_LAYERS || !planes_ok(n_layers, planes) ||
      (n_layers > 0 && (!thresholds || !is_traversability_type)))
    return fail(h, EMAP_ERR_INVALID, "emap_semantic_traversability: 0 to EMAP_SEMANTIC_TRAVERSABILITY_MAX_LAYERS non-null planes, "
                                     "thresholds, types and a non-null output required");
  SemTravArgs a;
  memset(&a, 0, sizeof(a));
  a.n = n_layers;
  for (int l = 0; l < n_layers; l++) {
    a.plane[l] = planes[l];
    a.thr[l] = thresholds[l];
    if (is_traversability_type[l]) a.is_trav[l >> 5] |= 1u << (l & 31);
  }
  PER_CELL(k_semantic_traversability, h->dc.C, a, out);
  return EMAP_OK;
}

// plugins/features_pca.py:44-96: exact 3-component PCA of the clipped features on the device, packed to colour bits.
// Four launches and one synchronisation, at the end, to read the NaN flag.
int emap_features_pca(emap_handle* h, int32_t n_features, const float* const* planes, float* out) {
  ENTER(h);
  NvtxRange nv("emap:features_pca");
  if (!out || n_features < 3 || n_features > EMAP_PCA_MAX_FEATURES || !planes_ok(n_features, planes))
    return fail(h, EMAP_ERR_INVALID, "emap_features_pca: 3 to EMAP_PCA_MAX_FEATURES non-null planes and a non-null output required");
  PcaScratch s;
  int rc = grow(h, h->pca_block, carve_pca(h, nullptr, s), 0, false);
  if (rc) return rc;
  carve_pca(h, h->pca_block, s);
  const int C = h->dc.C, F = n_features;
  PcaArgs a;
  memset(&a, 0, sizeof(a));
  a.F = F;
  for (int f = 0; f < F; f++) a.plane[f] = planes[f];
  const size_t eig_smem = sizeof(double) * 2 * F * (F + 1);
  CK(cudaFuncSetAttribute(k_pca_eigen, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eig_smem));
  CK(cudaMemsetAsync(&s.res->nan, 0, sizeof(int), h->stream));
  const int grid = pca_stats_grid(h);
  k_pca_stats<<<grid, PCA_THREADS, 0, h->stream>>>(C, a, s.part, s.res);
  LAUNCH_CHECK();
  k_pca_eigen<<<1, PCA_THREADS, eig_smem, h->stream>>>(C, F, grid, s.part, s.res);
  LAUNCH_CHECK();
  PER_CELL(k_pca_project, C, a, s.res, s.proj);
  PER_CELL(k_pca_pack, C, (const PcaResult*)s.res, (const double*)s.proj, (u32*)out);
  int nan = 0;
  CK(cudaMemcpyAsync(&nan, &s.res->nan, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (nan) return fail(h, EMAP_ERR_INVALID, "emap_features_pca: NaN in the input features");
  return EMAP_OK;
}

// EM.py:468-562 input_image + semantic_map.py:261-309 update_layers_image: the host part (image_camera) and one
// k_image_fuse launch.  A host image is copied into pinned staging and from there, once, to the device; a device image
// is read in place, with no host synchronisation.
int emap_input_image(emap_handle* h, int32_t n_planes, const float* image, int is_device_ptr, int32_t height, int32_t width,
                     const float K[9], const float* D, int32_t n_D, const char* distortion_model, const float R[9],
                     const float t[3], int32_t n_fused, const int32_t* plane, const int32_t* kind, const int32_t* layer,
                     float* semantic_map_device, int32_t n_layers) {
  ENTER(h);
  NvtxRange nv("emap:input_image");
  if (!image || !K || !R || !t || !distortion_model || (n_D > 0 && !D) || n_D < 0 ||
      (n_fused > 0 && (!plane || !kind || !layer || !semantic_map_device)))
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: null argument");
  if (n_planes < 1 || height < 1 || width < 1 || (int64_t)height * width > (1ll << 24))
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: n_planes >= 1 and 1 <= height * width <= 2^24 required");
  if (n_fused < 0 || n_fused > EMAP_IMAGE_MAX_CHANNELS)
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: 0 to EMAP_IMAGE_MAX_CHANNELS fused channels required");
  ImageArgs a;
  memset(&a, 0, sizeof(a));
  for (int k = 0; k < n_fused; k++) {
    if (kind[k] != EMAP_IMAGE_COLOR && kind[k] != EMAP_IMAGE_EXPONENTIAL)
      return fail(h, EMAP_ERR_INVALID, "emap_input_image: kind must be EMAP_IMAGE_COLOR or EMAP_IMAGE_EXPONENTIAL");
    if (plane[k] < 0 || plane[k] >= n_planes || (kind[k] == EMAP_IMAGE_COLOR && n_planes < 3))
      return fail(h, EMAP_ERR_INVALID, "emap_input_image: plane outside the image, or a colour channel with fewer than 3 planes");
    if (layer[k] < 0 || layer[k] >= n_layers)
      return fail(h, EMAP_ERR_INVALID, "emap_input_image: layer outside [0, n_layers)");
    a.plane[k] = plane[k];
    a.kind[k] = kind[k] == EMAP_IMAGE_COLOR ? IMG_COLOR : IMG_EXPONENTIAL;
    a.layer[k] = layer[k];
  }
  const int cam = image_camera(K, D, n_D, distortion_model, R, t, h->center, h->dc.W, h->cfg.resolution, &a.cam);
  if (cam == IMG_CAM_NONFINITE) return fail(h, EMAP_ERR_INVALID, "emap_input_image: non-finite K, R or t");
  if (cam == IMG_CAM_OUTSIDE)
    return fail(h, EMAP_ERR_INVALID, "emap_input_image: camera cell cell_n / 2 + t / resolution outside [0, 2^24)");
  if (n_fused == 0) return EMAP_OK;       // the correspondence alone changes nothing
  const size_t plane_sz = (size_t)height * width, n_img = plane_sz * n_planes;
  const float* img = image;
  if (!is_device_ptr) {
    const size_t bytes = sizeof(float) * n_img;
    if (int rc = h->img_up.room(h, bytes)) return rc;
    memcpy(h->img_up.host, image, bytes);                // the caller's buffer is free from here on
    if (int rc = h->img_up.send(h, bytes)) return rc;
    img = (const float*)(char*)h->img_up.dev;
  }
  for (int k = 0; k < 3; k++) a.center[k] = h->center[k];
  a.res = h->cfg.resolution;
  a.W = h->dc.W; a.C = h->dc.C;
  a.img_w = (float)width; a.img_h = (float)height;
  a.n_img = (long long)n_img; a.plane_sz = (long long)plane_sz;
  a.image = img; a.sem = semantic_map_device; a.n = n_fused;
  PER_CELL(k_image_fuse, a, (const float*)h->map);
  return EMAP_OK;
}

// rounds / Jacobi statistics of the last emap_inpaint call (diagnostics)
int emap_inpaint_stats(emap_handle* h, int32_t* rounds, int32_t* max_jacobi, int32_t* not_converged) {
  ENTER(h);
  if (!h->ip_block) return fail(h, EMAP_ERR_STATE, "emap_inpaint has not run");
  InpaintCtl c;
  CK(cudaMemcpyAsync(&c, inpaint_scratch(h->dc.W, h->ip_block).ctl, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
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
