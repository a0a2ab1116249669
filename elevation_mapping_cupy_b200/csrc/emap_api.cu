// emap_api.cu -- C ABI of libemap.so (see include/emap.h): the handle, frames (point clouds, depth images, sharded
// frames and their NCCL exchange), semantic configuration, read-backs, pose, time and state, streams and stage timing.
// The other calls are in emap_export_api.cu, emap_polygon_api.cu and emap_plugins_api.cu (see emap_handle.cuh).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 (see elevation_mapping_cupy_b200/build.py)
#include <dlfcn.h>

#include "emap_handle.cuh"
#include "emap_kernels.cuh"
#include "emap_semantic.cuh"

static_assert(EMAP_DEPTH_MAX_CHANNELS == SEM_MAX_CH, "emap.h and the semantic kernels disagree on the channel count");

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

namespace {

thread_local std::string g_create_error;

void make_pose(const float* R, const float* t_rel, Pose* q) {
  for (int i = 0; i < 9; i++) q->R16[i] = h16_host(R[i]);
  for (int i = 0; i < 3; i++) { q->t16[i] = h16_host(t_rel[i]); q->t[i] = t_rel[i]; }
}

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

bool sem_on(const emap_handle* h) { return h->sem.n_ch > 0 && h->sem_map; }

// The semantic sum planes of h's configuration carved at `base`: the 2^-32 fixed-point planes, then the r, g, b, count
// planes of each colour channel.  Returns their size (0 without a configuration).
size_t carve_sem(const emap_handle* h, uintptr_t base, i64*& fsum, u32*& csum) {
  const size_t C = (size_t)h->dc.C;
  const bool on = sem_on(h);
  Carver b{base};
  fsum = b.take<i64>(on ? C * h->sem_nf : 0);
  csum = b.take<u32>(on ? 4 * C * h->sem_nc : 0);
  return b.bytes;
}

// Where the frame's semantic sums are: the handle's planes, or behind the exchange scratch of an attached block (where
// every rank's k_sem_sum adds into all replicas)
void sem_sums(emap_handle* h, i64*& fsum, u32*& csum) {
  if (h->attached) carve_sem(h, (uintptr_t)h->attach_base + exchange_bytes((size_t)h->dc.C), fsum, csum);
  else { fsum = h->sem_fsum; csum = h->sem_csum; }
}

// Moves the exchange scratch of h to `base` in its between-frames state: all zero, upper-bound keys UKEY_NONE.
cudaError_t place_exchange(emap_handle* h, void* base) {
  const size_t C = (size_t)h->dc.C;
  carve_exchange(C, base, h->sc, h->fs);
  cudaError_t e = cudaMemsetAsync(base, 0, exchange_bytes(C), h->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(h->sc.ukv, 0xff, sizeof(u32) * C, h->stream);
  return e;
}

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
  i64* fsum;
  u32* csum;
  sem_sums(h, fsum, csum);
  if (h->sc.mc_off)
    k_sem_sum<Src, true><<<cdiv(n, 256), 256, 0, h->stream>>>(h->dc, h->sem, src, n, (const int*)(h->pidx + h->offs[s]),
                                                              fsum, csum, sem_max(h), h->sc.mc_off);
  else
    k_sem_sum<Src, false><<<cdiv(n, 256), 256, 0, h->stream>>>(h->dc, h->sem, src, n, (const int*)(h->pidx + h->offs[s]),
                                                               fsum, csum, sem_max(h), (i64)0);
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

// The arrays the ranks of a sharded frame reduce after phase 1..3 (kinds: see emap_exchange in emap.h); returns their
// count.  Phase 3 lists the upper-bound keys in s32 order (exchange_keys); without visibility cleanup it lists nothing.
int exchange_list(emap_handle* h, int phase, emap_exchange out[EMAP_SHARD_MAX_EXCHANGES]) {
  const i64 C = h->dc.C;
  if (phase == 1) {          // after begin: counts (CK.py:334,336) and the drift statistics (CK.py:332-333)
    out[0] = {h->sc.cnt_ai, 2 * C, 3};          // two 32-bit counters per cell: an int32 SUM keeps them apart
    out[1] = {&h->fs->E, 2, 0};
    return 2;
  }
  if (phase == 2) {          // after fusion: sums, counts (listed second: the only array phase 2 reads), last-writer keys
    out[0] = {h->sc.SH, 2 * C, 0};
    out[1] = {h->sc.cnt_fo, 2 * C, 3};
    out[2] = {h->sc.last, C, 1};
    int n = 3;
    if (sem_on(h)) {         // the semantic sums of phase 1, read in phase 3 like the height sums
      i64* fsum;
      u32* csum;
      sem_sums(h, fsum, csum);
      if (h->sem_nf) out[n++] = {fsum, h->sem_nf * C, 0};
      if (h->sem_nc) out[n++] = {csum, 4 * h->sem_nc * C, 3};
    }
    return n;
  }
  if (!h->dc.visibility) return 0;
  out[0] = {h->sc.DV, C, 0};   // after the ray-cast: decrements, counts, upper-bound keys
  out[1] = {h->sc.n_ray, C, 3};
  out[2] = {h->ukey_x, C, 2};
  return 3;
}

// Before exchange 3: the upper-bound keys in the s32 order an int32 MIN all-reduce needs (shard_finish merges them back)
int exchange_keys(emap_handle* h) {
  if (!h->dc.visibility) return 0;
  k_ukey_extract<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc.C, h->sc.ukv, h->ukey_x);
  LAUNCH_CHECK();
  h->progress = Progress::KEYS_EXCHANGED;
  return 0;
}

// A sharded frame's semantic passes: this rank's sums in phase 1, after which the caller may reuse its host input, and
// the layers from the reduced sums and counts in phase 3, before k_finalize re-zeroes the counts
int shard_sem_sum(emap_handle* h) {
  if (!sem_on(h)) return 0;
  NvtxRange nv("emap:semantic");
  int rc;
  if ((rc = h->in.each([h](auto pts, int s) { return launch_sem_sum(h, pts, s); })) || (rc = h->in.read_done(h))) return rc;
  return h->in.wait_free(h);
}

int shard_sem_apply(emap_handle* h) {
  if (!sem_on(h)) return 0;
  i64* fsum;
  u32* csum;
  sem_sums(h, fsum, csum);
  PER_CELL(k_sem_apply, h->dc, h->sem, (const u64*)h->sc.cnt_fo, fsum, csum, h->sem_map, sem_max(h));
  return 0;
}

// last phase of a sharded frame: the reduced upper-bound keys back to u32 (if phase 3 exchanged them), then finalize
int shard_finish(emap_handle* h) {
  if (h->progress == Progress::KEYS_EXCHANGED) {
    k_ukey_merge<<<cdiv(h->dc.C, 256), 256, 0, h->stream>>>(h->dc.C, h->sc.ukv, h->ukey_x);
    LAUNCH_CHECK();
  }
  const int rc = shard_sem_apply(h);
  return rc ? rc : frame_finish(h);
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
                    &h->ev_join, &h->ev_order, &h->img_up.staged, &h->init_up.staged,
                    &h->query.up.staged, &h->lookup.up.staged})
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
  ALLOC(h->dirty, 2 * (C + 16));
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
  TRY(cudaMemsetAsync(h->dirty, 0, 2 * (C + 16), h->stream));
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

int clear_map(emap_handle* h) {
  PER_CELL(k_clear, h->dc, h->map);
  CK(cudaMemsetAsync(&h->fs->mean_error, 0, 2 * sizeof(float), h->stream));     // EM.py:127-128
  return EMAP_OK;
}

// A frame of depth cameras (emap_input_depth_images, its sharded twins): the argument checks, then the frame's input.
// Its rows are the pixels, camera after camera, so a sharded frame's global_off counts the pixels of lower ranks.
int depth_begin(emap_handle* h, const char* fn, int32_t n_cameras, const emap_depth_camera* cams, int is_device_ptr,
                int32_t n_channels, const int32_t* channel_source, int32_t n_features, float confidence_threshold,
                float max_depth, int64_t global_off, float pn, float on, bool sharded) {
  char msg[200];
#define DMSG(text) (snprintf(msg, sizeof(msg), "%s: " text, fn), msg)
  if (!cams || n_cameras < 1 || n_cameras > EMAP_DEPTH_MAX_CAMERAS)
    return fail(h, EMAP_ERR_INVALID, DMSG("1 <= n_cameras <= EMAP_DEPTH_MAX_CAMERAS cameras required"));
  if (n_channels < 0 || n_channels > SEM_MAX_CH || (n_channels > 0 && !channel_source) || n_features < 0 ||
      n_features > EMAP_DEPTH_MAX_FEATURES)
    return fail(h, EMAP_ERR_INVALID, DMSG("0..16 channels with their sources, 0..255 feature planes required"));
  int n_color = 0, n_feat_used = 0;
  for (int j = 0; j < n_channels; j++) {
    if (channel_source[j] < -1 || channel_source[j] >= n_features)
      return fail(h, EMAP_ERR_INVALID, DMSG("a channel source outside [-1, n_features)"));
    n_color += channel_source[j] == -1;
    n_feat_used += channel_source[j] >= 0;
  }
  if (n_color > 1) return fail(h, EMAP_ERR_INVALID, DMSG("more than one colour channel"));
  if (h->sem.n_ch > 0 && h->sem_map)
    for (int k = 0; k < h->sem.n_ch; k++)
      if (h->sem.col[k] >= 3 + n_channels)
        return fail(h, EMAP_ERR_INVALID, DMSG("a configured semantic column beyond 3 + n_channels"));
  int64_t n[EMAP_DEPTH_MAX_CAMERAS];      // at most 16 * 2^24 = 2^28 pixels: below the frame's 2^31 rows
  float R[9 * EMAP_DEPTH_MAX_CAMERAS], t[3 * EMAP_DEPTH_MAX_CAMERAS];
  for (int s = 0; s < n_cameras; s++) {
    const emap_depth_camera& c = cams[s];
    bool finite = std::isfinite(c.fx) && std::isfinite(c.fy) && c.fx != 0.0 && c.fy != 0.0 && std::isfinite(c.cx) &&
                  std::isfinite(c.cy);
    for (int k = 0; k < 9; k++) finite = finite && std::isfinite(c.R[k]);
    for (int k = 0; k < 3; k++) finite = finite && std::isfinite(c.t[k]);
    if (!c.depth || c.height <= 0 || c.width <= 0 || (i64)c.height * c.width > (1ll << 24))
      return fail(h, EMAP_ERR_INVALID, DMSG("a depth image, 0 < height * width <= 2^24 required"));
    if (!finite) return fail(h, EMAP_ERR_INVALID, DMSG("non-finite or zero fx / fy, or non-finite cx, cy, R, t"));
    if ((n_color && !c.rgb) || (n_feat_used && !c.features))
      return fail(h, EMAP_ERR_INVALID, DMSG("a colour channel needs rgb, a feature channel the feature planes"));
    n[s] = (i64)c.height * c.width;
    memcpy(R + 9 * s, c.R, sizeof(c.R));
    memcpy(t + 3 * s, c.t, sizeof(c.t));
  }
  i64 N = 0;
  for (int s = 0; s < n_cameras; s++) N += n[s];
  if (global_off + N >= (1ll << 31)) return fail(h, EMAP_ERR_INVALID, DMSG("more than 2^31 rows up to this rank's last pixel"));
#undef DMSG
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
  return frame_start(h, is_device_ptr, R, t, global_off, pn, on, sharded);
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
  const int rc = depth_begin(h, "emap_input_depth_images", n_cameras, cams, is_device_ptr, n_channels, channel_source,
                             n_features, confidence_threshold, max_depth, 0, pn, on, false);
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
  if (n_channels <= 0) { h->sem.n_ch = 0; h->sem_map = nullptr; h->sem_nf = h->sem_nc = 0; return EMAP_OK; }
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
  // an attached handle keeps its sums in the symmetric block (sem_sums)
  if (!h->attached && ((rc = grow(h, h->sem_fsum, C * nf, 0, true)) || (rc = grow(h, h->sem_csum, C * 4 * nc, 0, true))))
    return rc;
  if (nm > 0 && ((rc = grow(h, h->cm_cell, 3 * C, 0, true)) ||
                 (rc = grow(h, h->cm_ctl, (size_t)CM_CTL + (1 + SEM_MAX_CH) * CM_WORDS + 65536, 0, true))))
    return rc;
  h->sem = c; h->sem_map = semantic_map_device; h->sem_nf = nf; h->sem_nc = nc;
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
namespace {
// What a sharded frame refuses before anything is queued: a class_max channel (its per-cell tables and class set do not
// reduce as fixed-size sums), and an attached block too small for the sums of the semantic configuration
int shard_check(emap_handle* h, const char* fn) {
  char msg[200];
  if (sem_on(h) && h->sem.n_max > 0) {
    snprintf(msg, sizeof(msg), "%s: class_max channels are not fused by sharded frames", fn);
    return fail(h, EMAP_ERR_INVALID, msg);
  }
  if (h->attached && h->attach_bytes < emap_shard_scratch_bytes(h)) {
    snprintf(msg, sizeof(msg), "%s: the semantic configuration outgrew the attached block: attach a block of "
             "emap_shard_scratch_bytes()", fn);
    return fail(h, EMAP_ERR_STATE, msg);
  }
  return 0;
}

// A sharded frame after its input is described and staged: NCCL mode indexes at once, an attached handle in phase 0
// (after the caller's barrier).  The caller may reuse its host input on return, or after phase 1 when the semantic sums
// read it there.
int shard_begun(emap_handle* h) {
  int rc = h->in.wait_free(h);
  if (rc || h->attached || (rc = frame_index(h))) return rc;
  return sem_on(h) ? 0 : h->in.wait_free(h);
}
}  // namespace

int emap_shard_begin(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n, int64_t row_stride,
                     int dtype, int is_device_ptr, const float* R, const float* t, int64_t global_point_offset, float pn,
                     float on) {
  ENTER(h);
  if (!points || !n || !R || !t) return fail(h, EMAP_ERR_INVALID, "emap_shard_begin: null argument");
  int rc;
  if ((rc = shard_check(h, "emap_shard_begin")) ||
      (rc = frame_begin(h, n_sensors, points, n, row_stride, dtype, is_device_ptr, R, t, global_point_offset, pn, on, true)))
    return rc;
  // multicast mode: every rank must have reset its frame scalars before anyone pushes -> the caller runs a
  // cross-rank barrier and then emap_shard_phase(h, 0); NCCL mode: index right away
  return shard_begun(h);
}

int emap_shard_begin_depth_images(emap_handle* h, int32_t n_cameras, const emap_depth_camera* cams, int is_device_ptr,
                                  int32_t n_channels, const int32_t* channel_source, int32_t n_features,
                                  float confidence_threshold, float max_depth, int64_t global_point_offset, float pn,
                                  float on) {
  ENTER(h);
  const char* fn = "emap_shard_begin_depth_images";
  int rc;
  if ((rc = shard_check(h, fn)) ||
      (rc = depth_begin(h, fn, n_cameras, cams, is_device_ptr, n_channels, channel_source, n_features,
                        confidence_threshold, max_depth, global_point_offset, pn, on, true)))
    return rc;
  return shard_begun(h);
}

int64_t emap_shard_scratch_bytes(const emap_handle* h) {
  if (!h) return EMAP_ERR_INVALID;
  i64* fsum;
  u32* csum;
  return (int64_t)(exchange_bytes((size_t)h->dc.C) + carve_sem(h, 0, fsum, csum));
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
  const size_t xb = exchange_bytes((size_t)h->dc.C);       // the semantic sum planes: zero between frames
  CK(cudaMemsetAsync((char*)local_base + xb, 0, (size_t)bytes - xb, h->stream));
  h->attach_base = (char*)local_base; h->attach_bytes = bytes;
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
  emap_exchange ex[EMAP_SHARD_MAX_EXCHANGES];
  const int n = exchange_list(h, phase, ex);
  if (*n_out < n) {
    *n_out = n;
    return fail(h, EMAP_ERR_INVALID, "emap_shard_exchange: capacity below the listed arrays (*n_out: the count needed)");
  }
  if (phase == 3) if (int rc = exchange_keys(h)) return rc;
  std::copy(ex, ex + n, out);
  *n_out = n;
  return 0;
}

int emap_shard_phase(emap_handle* h, int32_t phase) {
  ENTER(h);
  if (phase == 0) {
    if (h->progress != Progress::BEGUN) return fail(h, EMAP_ERR_STATE, "phase 0 must follow emap_shard_begin on an attached handle");
    const int rc = frame_index(h);
    return rc || sem_on(h) ? rc : h->in.wait_free(h);
  }
  if (phase == 1) {
    if (h->progress != Progress::INDEXED) return fail(h, EMAP_ERR_STATE, "phase 1 must follow emap_shard_begin");
    const int rc = frame_fuse(h);
    return rc ? rc : shard_sem_sum(h);
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
  emap_exchange ex[EMAP_SHARD_MAX_EXCHANGES];
  const int n = exchange_list(h, phase, ex);
  if (phase == 3) if (int rc = exchange_keys(h)) return rc;
  NcclApi& a = nccl_api();
  for (int k = 0; k < n; k++) {
    const int dt = (ex[k].kind == 0 || ex[k].kind == 1) ? kNcclInt64 : kNcclInt32;
    const int op = ex[k].kind == 1 ? kNcclMax : ex[k].kind == 2 ? kNcclMin : kNcclSum;
    const int r = a.AllReduce(ex[k].ptr, ex[k].ptr, (size_t)ex[k].count, dt, op, h->nccl_comm, h->stream);
    if (r != 0) { h->err = std::string("ncclAllReduce: ") + (a.GetErrorString ? a.GetErrorString(r) : "error"); return EMAP_ERR_CUDA; }
  }
  return 0;
}

// The phases of a sharded frame after its begin, collective over the communicator of emap_comm_init (integer NCCL
// all-reduces between them; the replicas stay bit-identical)
static int comm_frame(emap_handle* h, float overlap_sensor_z_absolute) {
  int rc;
  h->overlap_override = true; h->overlap_z_override = overlap_sensor_z_absolute - h->center[2];
  if ((rc = comm_exchange(h, 1)) || (rc = frame_fuse(h)) || (rc = shard_sem_sum(h)) || (rc = comm_exchange(h, 2)) ||
      (rc = frame_rays(h)) || (rc = comm_exchange(h, 3)))
    return rc;
  return shard_finish(h);
}

static int comm_check(emap_handle* h, const char* fn) {
  char msg[200];
  snprintf(msg, sizeof(msg), "%s: call emap_comm_init first", fn);
  if (!h->nccl_comm) return fail(h, EMAP_ERR_STATE, msg);
  if (h->attached) return fail(h, EMAP_ERR_STATE, "handle is attached to a multicast scratch: use the emap_shard_* calls");
  return shard_check(h, fn);
}

// One sharded frame: this rank's sensors are fused into the replicated grid together with every other rank's.
int emap_input_sensors_sharded(emap_handle* h, int32_t n_sensors, const void* const* points, const int64_t* n, int64_t row_stride,
                               int dtype, int is_device_ptr, const float* R, const float* t, int64_t global_point_offset,
                               float overlap_sensor_z_absolute, float pn, float on) {
  ENTER(h);
  int rc;
  if ((rc = comm_check(h, "emap_input_sensors_sharded"))) return rc;
  if (!points || !n || !R || !t) return fail(h, EMAP_ERR_INVALID, "emap_input_sensors_sharded: null argument");
  if ((rc = frame_begin(h, n_sensors, points, n, row_stride, dtype, is_device_ptr, R, t, global_point_offset, pn, on, true)) ||
      (rc = shard_begun(h)))
    return rc;
  return comm_frame(h, overlap_sensor_z_absolute);
}

// One sharded frame of this rank's depth cameras (global_point_offset: the pixels of the lower ranks' cameras)
int emap_input_depth_images_sharded(emap_handle* h, int32_t n_cameras, const emap_depth_camera* cams, int is_device_ptr,
                                    int32_t n_channels, const int32_t* channel_source, int32_t n_features,
                                    float confidence_threshold, float max_depth, int64_t global_point_offset,
                                    float overlap_sensor_z_absolute, float pn, float on) {
  ENTER(h);
  const char* fn = "emap_input_depth_images_sharded";
  int rc;
  if ((rc = comm_check(h, fn)) ||
      (rc = depth_begin(h, fn, n_cameras, cams, is_device_ptr, n_channels, channel_source, n_features,
                        confidence_threshold, max_depth, global_point_offset, pn, on, true)) ||
      (rc = shard_begun(h)))
    return rc;
  return comm_frame(h, overlap_sensor_z_absolute);
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
int emap_get_position(emap_handle* h, double out[3]) {
  ENTER(h);
  for (int k = 0; k < 3; k++) out[k] = h->center[k];
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
