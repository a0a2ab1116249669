// emap_kernels.cuh -- the per-frame kernels of the fusion path (sm_90a).
//
// Frame = elevation_mapping.py:316-391 (update_map_with_kernel) executed under the canonical
// serialisation of SURVEY.md 8(c):
//   k_index_error   CK.py:280-345   per point: geometry, cell, drift-inlier statistics, counts
//   k_drift         EM.py:346-357   one thread: mean error, shift decision (no host sync)
//   k_fuse          CK.py:168-197   per point: Kalman update against the pre-frame snapshot
//   k_record        --              per cell: pack the post-fusion state a ray needs into 16 B
//   k_raycast       CK.py:198-259   per point: visibility cleanup / upper-bound carving
//   k_finalize      CK.py:348-389 + EM.py:393-410   per cell: apply all side effects, average, overlap clear
//   k_post          CK.py:392-449, traversability_filter.py:15-42, CK.py:452-506  dilation + CNN + normals
// Order-dependent float accumulations of the reference (atomicAdd of new_h, new_v, validity
// decrements, drift errors) are accumulated exactly in 2^-32 fixed point (int64 atomics), which
// makes every result independent of thread order, run-to-run deterministic and bit-identical to
// oracle/emap_oracle.c; they are within one fp32 rounding of some order of the reference atomics.
#pragma once
#include <cuda.h>                 // CUtensorMap (type only; the encoder is fetched at run time, make_post_tm)
#include "emap_plan.cuh"         // RT, RayGrid, RC_STRIDE, RcLayout, PT_X, PT_Y
#include "emap_sources.cuh"

// accumulate into the per-cell scratch: local L2 atomic, or one in-switch multicast reduction
__device__ __forceinline__ void red_add(u32* p, u32 v, i64 mc) {
  if (mc) asm volatile("multimem.red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"((char*)p + mc), "r"(v) : "memory");
  else atomicAdd(p, v);
}
__device__ __forceinline__ void red_add(u64* p, u64 v, i64 mc) {
  if (mc) asm volatile("multimem.red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"((char*)p + mc), "l"(v) : "memory");
  else atomicAdd(p, v);
}
__device__ __forceinline__ void red_max(u64* p, u64 v, i64 mc) {
  if (mc) asm volatile("multimem.red.relaxed.sys.global.max.u64 [%0], %1;" ::"l"((char*)p + mc), "l"(v) : "memory");
  else atomicMax(p, v);
}
__device__ __forceinline__ void red_min(u32* p, u32 v, i64 mc) {
  if (mc) asm volatile("multimem.red.relaxed.sys.global.min.u32 [%0], %1;" ::"l"((char*)p + mc), "r"(v) : "memory");
  else atomicMin(p, v);
}

// Programmatic dependent launch (PDL): every frame kernel is launched with programmatic stream serialisation, lets
// its successor start launching right away (pdl_trigger) and waits for its predecessor's results only where it first
// needs them (pdl_wait).  With the attribute absent both are no-ops.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Bulk copies (TMA) into shared memory that complete on one mbarrier: one thread arms the barrier with the bytes the
// copies will deliver (bar_expect) and issues them; the CTA waits for the barrier's phase (bar_wait) only after every
// thread can see the initialised barrier (a __syncthreads in between).
__device__ __forceinline__ void bar_expect(u32 bar, u32 bytes) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_wait(u32 bar, u32 parity) {
  u32 ok = 0;
  while (!ok)
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
}
// `bytes` (a multiple of 16) from global `src` to shared `dst` (both 16-byte aligned)
__device__ __forceinline__ void bulk_copy(u32 dst, const void* src, u32 bytes, u32 bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// the box of tensor map `tm` at element coordinates (x, y, z) to shared `dst`; elements outside the tensor arrive as zeros
__device__ __forceinline__ void tensor_copy_3d(u32 dst, const CUtensorMap* tm, int x, int y, int z, u32 bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(dst), "l"(tm), "r"(x), "r"(y), "r"(z), "r"(bar) : "memory");
}

#ifndef FUSE_AGG
#define FUSE_AGG 1                // single-GPU frames: warp-aggregate the per-cell atomics of a warp that has runs (0: never)
#endif

// ---- warp aggregation of pushes over RUNS of adjacent lanes that hit the same cell (scan-ordered
// clouds put consecutive points in the same cell).  Every accumulation is an integer sum / max, so
// pre-reducing a run in registers and pushing once is exactly equivalent; it is what keeps the number of
// NVLink multicast reductions per frame (one per update, applied by the switch to every replica) down.
struct RunInfo { u32 run_mask; bool tail; };
__device__ __forceinline__ RunInfo run_of(int key, int lane) {
  const int prev = __shfl_up_sync(0xffffffffu, key, 1);
  const u32 heads = __ballot_sync(0xffffffffu, lane == 0 || key != prev);
  const u32 below = heads & ((2u << lane) - 1u);                     // heads at or below this lane
  const int start = 31 - __clz(below);
  const u32 above = heads & ~((2u << lane) - 1u);                    // heads above this lane
  const int end = above ? (__ffs(above) - 1) : 32;                   // one past the run
  RunInfo r;
  r.run_mask = (end == 32 ? 0xffffffffu : ((1u << end) - 1u)) & ~((1u << start) - 1u);
  r.tail = lane == end - 1;
  return r;
}
// inclusive sum of v over the lanes of the run that are at or below this lane (the tail lane gets the run total)
__device__ __forceinline__ i64 run_sum(i64 v, int lane, u32 run_mask) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const i64 o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d && ((run_mask >> (lane - d)) & 1u)) v += o;
  }
  return v;
}

// number of entries of the increasing table t[0..n) that are < x (binary search; NaN x -> 0)
__device__ __forceinline__ int count_below(const float* __restrict__ t, int n, float x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(t + mid) < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------
// Src: a point source of emap_sources.cuh (the caller's cloud rows, or a depth image read pixel by pixel)
template <typename Src>
__global__ void __launch_bounds__(256)
k_index_error(const DevCfg c, const Pose q, const Src src, const i64 n,
              float4* __restrict__ xyzv, int* __restrict__ pidx, const float* __restrict__ map,
              const CellScratch s, FrameScalars* fs, Ray* __restrict__ rays, int* __restrict__ ray_ctl,
              const unsigned short* __restrict__ step_cnt) {
  pdl_trigger(); pdl_wait();
  const i64 i = blockIdx.x * (i64)blockDim.x + threadIdx.x;
  i64 e = 0; int ec = 0, nv = 0, nk = 0;
  Ray ray; ray.len = -1.f; ray.counts = 0;
  int cell_key = -1 - (int)(threadIdx.x & 31);                    // cell receiving this point's count (unique negative: none)
  bool is_inl = false;
  if (i < n) {
    float px, py, pz;                                             // EM.py:456 cast to fp32
    const bool kept = src.load(i, px, py, pz);
    int rec;
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!kept || px != px || py != py || pz != pz) {              // EM.py:458 drop NaN rows (and masked pixels)
      rec = PT_SKIP | PT_IDX_MASK;
    } else {
      nk = 1;
      Geom g; point_geom(c, q, px, py, pz, g);
      const int idx = g.ix * c.W + g.iy;
      rec = idx | (g.valid ? PT_VALID : 0) | (g.inside ? PT_INSIDE : 0);
      o = make_float4(g.x, g.y, g.z, g.v);
      nv = g.valid;
      if (g.valid && c.visibility) {
        // ray_vector CK.py:83-101 and the per-ray constants of CK.py:199-201,250
        const float vx = h16(h16(g.x) - q.t16[0]), vy = h16(h16(g.y) - q.t16[1]), vz = h16(h16(g.z) - q.t16[2]);
        const float norm = h16(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), __fmul_rn(vz, vz))));
        ray.rx = ray.ry = ray.rz = 0.f;
        if (norm > 0.f) { ray.rx = h16(__fdiv_rn(vx, norm)); ray.ry = h16(__fdiv_rn(vy, norm)); ray.rz = h16(__fdiv_rn(vz, norm)); }
        ray.x = g.x; ray.y = g.y; ray.z = g.z;
        ray.len = fminf(norm, c.max_len16);                       // CK.py:201
        // Bound used to skip the `d < 0.1` test of CK.py:225-226 far from the end point p.  With u = p - t,
        // the fp16 roundings of p, t and their difference move v by at most sqrt(3)*2^-11*(2m + |v|) (m = largest
        // coordinate magnitude), the fp16 direction and norm by at most 9.2e-4*s, and |v| >= norm*(1 - 2^-11), so
        // |p - (t + dir*s)| >= (norm - s)(1 - 2^-11) - 1e-3*(2m + 2 norm).  d >= 0.1003 (no fp16 rounding can
        // bring it under 0.1) is therefore guaranteed for s < norm - (0.325 + 1e-3*(2m + 2 norm)).
        const float m = fmaxf(fmaxf(fmaxf(fabsf(g.x), fabsf(g.y)), fabsf(g.z)),
                              fmaxf(fmaxf(fabsf(q.t[0]), fabsf(q.t[1])), fabsf(q.t[2])));
        const float len_far = norm - (0.325f + 1e-3f * (2.f * m + 2.f * norm));
        // number of march steps below len / len_far, from the per-handle table over the non-negative fp16 values
        // (k_build_step_cnt).  len is an fp16 value: exact.  len_far is rounded DOWN to fp16 first: the count can only
        // get smaller, i.e. the `d < 0.1` test is evaluated for a few more samples than necessary -- same results.
        const u32 n_act = __ldg(step_cnt + __half_as_ushort(__float2half_rn(ray.len)));
        u32 k_far = 0;
        if (len_far > 0.f) k_far = __ldg(step_cnt + min((u32)__half_as_ushort(__float2half_rd(len_far)), 0x7c00u));
        ray.counts = n_act | (k_far << 16);
      }
      if (g.valid && g.inside) {                                  // CK.py:318-323
        const float mh = __ldg(map + idx), mv = __ldg(map + c.C + idx);
        const float mvalid = __ldg(map + 2 * c.C + idx), mt = __ldg(map + 3 * c.C + idx);
        if (mvalid > 0.5f && (double)fabsf(mh - g.z) < (double)mv * c.mahal
            && (double)mv < c.inlier_var_half && (double)mt > c.trav_inlier) {   // CK.py:328-330
          e = fix32(g.z - mh); ec = 1;
          is_inl = true;
        }
        cell_key = idx;
        if (s.dirty) s.dirty[2 * idx] = 1;                        // points marker: exactly the cells k_fuse may touch
      }
    }
    xyzv[i] = o; pidx[i] = rec;
  }
  {   // per-cell counts (CK.py:334,336).  Sharded frame: one multicast reduction per run of lanes in the same cell.
      // Single GPU: one atomic per point, or per run when the warp has runs at all (scan-ordered clouds)
    const int lane = threadIdx.x & 31;
    const int below = __shfl_up_sync(0xffffffffu, cell_key, 1);
    const bool agg = s.mc_off || (FUSE_AGG && __any_sync(0xffffffffu, lane > 0 && cell_key >= 0 && cell_key == below));
    if (!agg) {
      if (cell_key >= 0) atomicAdd(s.cnt_ai + cell_key, is_inl ? 0x100000001ull : 1ull);
    } else {
      const RunInfo ri = run_of(cell_key, lane);
      const u32 inl = __ballot_sync(0xffffffffu, is_inl) & ri.run_mask;
      if (ri.tail && cell_key >= 0)
        red_add(s.cnt_ai + cell_key, (u64)__popc(ri.run_mask) | ((u64)__popc(inl) << 32), s.mc_off);
    }
  }
  // compact the rays that have at least one march step (s_0 < len) into the sensor's ray list: one
  // atomic per CTA; the list order is irrelevant (every ray effect is a commutative integer atomic)
  __shared__ int s_rc[9];
  const bool has_ray = (ray.counts & 0xffffu) != 0;               // at least one march step: s_0 < len
  const u32 ray_bal = __ballot_sync(0xffffffffu, has_ray);
  if ((threadIdx.x & 31) == 0) s_rc[threadIdx.x >> 5] = __popc(ray_bal);
  // block reduction -> one integer atomic per block (order independent)
  if (Src::kCountsKept) nv |= nk << 16;                           // a block has 256 rows: both counts fit in one int
  for (int o = 16; o > 0; o >>= 1) {
    e += __shfl_down_sync(0xffffffffu, e, o);
    ec += __shfl_down_sync(0xffffffffu, ec, o);
    nv += __shfl_down_sync(0xffffffffu, nv, o);
  }
  __shared__ i64 s_e[8]; __shared__ int s_c[8], s_v[8];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_e[w] = e; s_c[w] = ec; s_v[w] = nv; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; k++) { e += s_e[k]; ec += s_c[k]; nv += s_v[k]; }
    if (e != 0) red_add((u64*)&fs->E, (u64)e, s.mc_off);
    if (ec) red_add((u64*)&fs->ecnt, (u64)ec, s.mc_off);
    if (Src::kCountsKept) {
      if (nv >> 16) atomicAdd((u64*)&fs->nkept, (u64)(nv >> 16));
      nv &= 0xffff;
    }
    if (nv) atomicAdd((u64*)&fs->nvalid, (u64)nv);
    int tot = 0;
    for (int k = 0; k < 8; k++) tot += s_rc[k];
    s_rc[8] = tot ? atomicAdd(ray_ctl, tot) : 0;
  }
  __syncthreads();
  if (has_ray) {
    int base = s_rc[8];
    for (int k = 0; k < w; k++) base += s_rc[k];
    float4* dst = reinterpret_cast<float4*>(rays + base + __popc(ray_bal & ((1u << l) - 1u)));
    dst[0] = make_float4(ray.x, ray.y, ray.z, ray.len);
    dst[1] = make_float4(ray.rx, ray.ry, ray.rz, __uint_as_float(ray.counts));
  }
}

// overlap-clear reference of a sharded frame (emap_shard_set_overlap_z)
__global__ void k_set_overlap(FrameScalars* fs, float overlap_tz) {
  if (threadIdx.x == 0 && blockIdx.x == 0) fs->overlap_tz = overlap_tz;
}

// EM.py:346-357: the drift decision of a frame from the accumulated inlier statistics
struct DriftDecision { int applied, evaluated; float shift, mean, error_sum; };
__device__ __forceinline__ DriftDecision drift_decide(const DevCfg& c, const i64 E, const i64 ecnt, const float position_noise,
                                                      const float orientation_noise) {
  DriftDecision d;
  d.applied = 0; d.evaluated = 0; d.shift = 0.f; d.mean = 0.f;
  d.error_sum = (float)unfix32(E);
  if (c.drift_en && (double)(float)ecnt > c.min_drift_cnt
      && ((double)position_noise > c.pos_thresh || (double)orientation_noise > c.ori_thresh)) {
    d.mean = __fdiv_rn(d.error_sum, (float)ecnt);
    d.evaluated = 1;
    if (fabsf(d.mean) < c.max_drift_f) { d.shift = __fmul_rn(d.mean, c.drift_alpha_f); d.applied = 1; }
  }
  return d;
}
// one thread: publish the decision and the frame statistics (emap_get_frame_stats), reset the ray-march counters
__device__ __forceinline__ void drift_publish(FrameScalars* fs, const DriftDecision& d, const i64 ecnt, const float overlap_tz,
                                              const int set_overlap) {
  fs->nvalid_last = fs->nvalid; fs->nkept_last = fs->nkept;
  fs->ray_steps = 0; fs->ray_visits = 0;
  fs->ecnt_last = ecnt;
  if (set_overlap) fs->overlap_tz = overlap_tz;
  fs->error_sum = d.error_sum; fs->shift = d.shift; fs->applied = d.applied; fs->evaluated = d.evaluated;
  if (d.evaluated) { fs->mean_error = d.mean; fs->additive_mean_error = __fadd_rn(fs->additive_mean_error, d.mean); }
}

// Sharded frames (the statistics arrive from all ranks between the index pass and the fusion): one thread decides.
// Also the frame's housekeeping: the drift accumulators are consumed here and zeroed for the NEXT frame, and the coarse
// ray map is reset.  (Single-GPU frames have no k_drift launch: every k_fuse thread derives the decision itself, see there.)
__global__ void k_drift(const DevCfg c, FrameScalars* fs, float position_noise, float orientation_noise,
                        float overlap_tz, int set_overlap, u32* __restrict__ tmap) {
  pdl_trigger(); pdl_wait();
  for (int k = threadIdx.x; k < RT * RT; k += blockDim.x) tmap[k] = 0u;       // below every key: fkey(-inf) = 0x007fffff
  if (threadIdx.x || blockIdx.x) return;
  const i64 ecnt = fs->ecnt;
  const DriftDecision d = drift_decide(c, fs->E, ecnt, position_noise, orientation_noise);
  drift_publish(fs, d, ecnt, overlap_tz, set_overlap);
  fs->E = 0; fs->ecnt = 0; fs->nvalid = 0; fs->nkept = 0;
}

// CK.py:168-197 fusion half; every load is of the pre-frame snapshot (+ drift shift)
// PUSH: bit 0 = the counts (cnt_fo: needed by the ray-cast), bit 1 = the sums and last-writer keys (needed only by
// k_finalize).  Single GPU: 3.  Sharded frames over NVLink multicast launch it twice: <1> on the critical path and <2>
// on a side stream under the ray-cast, so that three of the four multicast reductions per run leave the critical path.
// DRIFT = 1 (single-GPU frames): there is no k_drift launch.  The inlier statistics are complete when this kernel starts, so
// every thread derives the drift decision itself (two broadcast loads, a handful of flops) and thread 0 publishes it for
// the later kernels; the accumulators are re-zeroed by k_finalize, after the last reader.
template <int PUSH, int DRIFT>
__global__ void __launch_bounds__(256)
k_fuse(const DevCfg c, const i64 n, const i64 global_off, const float4* __restrict__ xyzv,
       const int* __restrict__ pidx, const float* __restrict__ map, const CellScratch s,
       const FrameScalars* fs, FrameScalars* fsw, const float position_noise, const float orientation_noise,
       const float overlap_tz) {
  pdl_trigger(); pdl_wait();
  const i64 i = blockIdx.x * (i64)blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  int applied; float shift;
  if (DRIFT) {
    const i64 ecnt = fs->ecnt;
    const DriftDecision d = drift_decide(c, fs->E, ecnt, position_noise, orientation_noise);
    applied = d.applied; shift = d.shift;
    if (blockIdx.x == 0 && threadIdx.x == 0) drift_publish(fsw, d, ecnt, overlap_tz, 1);
  } else {
    applied = fs->applied; shift = fs->shift;
  }
  int idx = -1 - lane;                    // unique negative key: this lane pushes nothing
  bool is_out = false, is_fused = false;
  i64 fh = 0, fv = 0;
  u64 key = 0;
  if (i < n) {
    const int rec = pidx[i];
    if ((rec & (PT_VALID | PT_INSIDE | PT_SKIP)) == (PT_VALID | PT_INSIDE)) {
      idx = rec & PT_IDX_MASK;
      const float4 g = xyzv[i];
      const float z = g.z, v = g.w;
      float mh = __ldg(map + idx);
      if (applied) mh = __fadd_rn(mh, shift);                     // EM.py:357 applied lazily
      const float mv = __ldg(map + c.C + idx);
      const float num_points = (float)(u32)s.cnt_ai[idx];         // CK.py:172
      if ((double)fabsf(mh - z) > (double)mv * c.mahal) {
        is_out = true;                                            // CK.py:174
      } else if (c.edge_sharpen && (double)num_points > c.wall_thresh
                 && (double)z < (double)mh - (double)mv * c.mahal / (double)num_points) {
        // CK.py:177-179 edge sharpening: skip
      } else {
        const float den = __fadd_rn(mv, v);
        const float new_h = __fdiv_rn(__fmaf_rn(mh, v, __fmul_rn(z, mv)), den);   // CK.py:181 (nvcc contraction)
        const float new_v = __fdiv_rn(__fmul_rn(mv, v), den);                     // CK.py:182
        is_fused = true; fh = fix32(new_h); fv = fix32(new_v);
        key = ((u64)(u32)(global_off + i) << 32) | (u64)__float_as_uint(new_h);   // CK.py:191: last writer in input order
      }
    }
  }
  if (!s.mc_off) {
    // single GPU: plain L2 atomics -- unless some lane shares its cell with the lane below it (scan-ordered clouds:
    // LiDAR rings, depth-image rows), in which case the warp takes the run-aggregated path below (one atomic per run
    // and quantity instead of one per point; exact, every accumulation is an integer sum / max)
    const int below = __shfl_up_sync(0xffffffffu, idx, 1);
    const bool agg = FUSE_AGG && __any_sync(0xffffffffu, lane > 0 && idx >= 0 && idx == below);
    if (!agg) {
      if ((PUSH & 1) && (is_out || is_fused)) atomicAdd(s.cnt_fo + idx, is_out ? 0x100000000ull : 1ull);
      if ((PUSH & 2) && is_fused) {
        atomicAdd((u64*)(s.SH + idx), (u64)fh);
        atomicAdd((u64*)(s.SV + idx), (u64)fv);
        atomicMax(s.last + idx, key);
      }
      return;
    }
  }
  // pre-reduce each run of lanes in the same cell: one atomic (sharded frame: one multicast reduction) per quantity
  const RunInfo ri = run_of(idx, lane);
  const u32 outs = __ballot_sync(0xffffffffu, is_out) & ri.run_mask;
  const u32 fus = __ballot_sync(0xffffffffu, is_fused) & ri.run_mask;
  const i64 sh = run_sum(fh, lane, ri.run_mask), sv = run_sum(fv, lane, ri.run_mask);
  const u64 top_key = __shfl_sync(0xffffffffu, key, fus ? 31 - __clz(fus) : lane);   // highest fused lane = latest point
  if (ri.tail && idx >= 0) {
    if ((PUSH & 1) && (outs | fus)) red_add(s.cnt_fo + idx, (u64)__popc(fus) | ((u64)__popc(outs) << 32), s.mc_off);
    if ((PUSH & 2) && fus) {
      red_add((u64*)(s.SH + idx), (u64)sh, s.mc_off);
      red_add((u64*)(s.SV + idx), (u64)sv, s.mc_off);
      red_max(s.last + idx, top_key, s.mc_off);
    }
  }
}

// V consecutive elements (V = 4: one 16-byte access, needs C % 4 == 0; V = 1: any cell_n)
template <int V, typename T> __device__ __forceinline__ void ldv(const T* p, T (&a)[V]) {
  if (V == 2) { const uint2 t = *reinterpret_cast<const uint2*>(p); a[0] = ((const T*)&t)[0]; a[1 % V] = ((const T*)&t)[1]; }
  else if (V == 4) { const uint4 t = *reinterpret_cast<const uint4*>(p); a[0] = ((const T*)&t)[0]; a[1 % V] = ((const T*)&t)[1]; a[2 % V] = ((const T*)&t)[2]; a[3 % V] = ((const T*)&t)[3]; }
  else { for (int j = 0; j < V; j++) a[j] = p[j]; }
}
template <int V, typename T> __device__ __forceinline__ void stv(T* p, const T (&a)[V]) {
  if (V == 2) { uint2 t; ((T*)&t)[0] = a[0]; ((T*)&t)[1] = a[1 % V]; *reinterpret_cast<uint2*>(p) = t; }
  else if (V == 4) { uint4 t; ((T*)&t)[0] = a[0]; ((T*)&t)[1] = a[1 % V]; ((T*)&t)[2] = a[2 % V]; ((T*)&t)[3] = a[3 % V]; *reinterpret_cast<uint4*>(p) = t; }
  else { for (int j = 0; j < V; j++) p[j] = a[j]; }
}
template <int V> __device__ __forceinline__ void ldv64(const u64* p, u64 (&a)[V]) {     // V u64: 16-byte accesses when V is even
  if (V % 2 == 0) { for (int j = 0; j < V; j += 2) { const uint4 t = *reinterpret_cast<const uint4*>(p + j); a[j] = ((u64)t.y << 32) | t.x; a[(j + 1) % V] = ((u64)t.w << 32) | t.z; } }
  else { for (int j = 0; j < V; j++) a[j] = p[j]; }
}
template <int V, typename T> __device__ __forceinline__ bool anyv(const T (&a)[V]) { bool r = false; for (int j = 0; j < V; j++) r |= (a[j] != (T)0); return r; }
template <int V, typename T> __device__ __forceinline__ bool diffv(const T (&a)[V], const T (&b)[V]) { bool r = false; for (int j = 0; j < V; j++) r |= (a[j] != b[j]); return r; }

// n sequential fp32 additions of the constant c (the atomicAdds of CK.py:174 / CK.py:251)
__device__ __forceinline__ float add_n_times(float v, float c, u32 n) {
  for (u32 k = 0; k < n; k++) v = __fadd_rn(v, c);
  return v;
}

// Post-fusion state of a cell as a ray sees it (SURVEY 8(c) step 3 -> 4), in two levels:
//   thr (4 B)  first level.  A ray sample at height nz can act on the cell only if !(nz > thr):
//                invalid cell              thr = its upper bound (+inf if unbounded): a sample carves only below it, CK.py:230
//                valid, time < 0.5, border thr = -inf: CK.py:237 / CK.py:211, never
//                valid otherwise           thr = h' + 0.06 (and fl(thr - 0.05f) > h' checked), so nz > thr implies the
//                                          far-below rejection `h' < nz - 0.05f` the second level would take (CK.py:239)
//   rec (8 B)  second level, read only by the few samples that pass: .x = bits(h' = h (+ drift shift)) for valid
//              cells / upper-bound key for invalid ones, .y = RF_* flags.
// The variance a ray needs (CK.py:239) is rebuilt on the second level from map[1] and n_out.
// Only the cells a ray of this frame can reach are recorded: box = sensor cell +- (max_ray_length / resolution + slack),
// rows [box.x, box.y) x columns [box.z, box.w) (columns a multiple of V), computed on the host (ray_box in emap_plan.cuh).
// Also reduces thr to the coarse map tmap: max over each 2^ts x 2^ts tile (order-preserving keys, atomicMax; zeroed
// by k_drift) -- a ray above a tile's maximum cannot act on any of its cells (k_raycast).
template <int V>
__global__ void __launch_bounds__(256)
k_record(const DevCfg c, const float* __restrict__ map, const CellScratch s, const FrameScalars* __restrict__ fs, const RayGrid g,
         u32* __restrict__ tmap) {
  pdl_trigger(); pdl_wait();
  const int ncg = (g.c1 - g.c0) / V;                              // column groups per row
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ncg * (g.r1 - g.r0)) return;
  const int rr = g.r0 + t / ncg, cc0 = g.c0 + (t % ncg) * V;
  const int i0 = rr * c.W + cc0;
  const size_t C = (size_t)c.C;
  float h4[V], va4[V], ti4[V], up4[V], iu4[V];
  u32 cf4[V], ci4[V];
  ldv<V>(map + i0, h4); ldv<V>(map + 2 * C + i0, va4); ldv<V>(map + 4 * C + i0, ti4);
  ldv<V>(map + 5 * C + i0, up4); ldv<V>(map + 6 * C + i0, iu4);
  {
    u64 fo[V], ai[V];
    ldv64<V>(s.cnt_fo + i0, fo); ldv64<V>(s.cnt_ai + i0, ai);
    for (int j = 0; j < V; j++) { cf4[j] = (u32)fo[j]; ci4[j] = (u32)(ai[j] >> 32); }
  }
  const int applied = fs->applied; const float shift = fs->shift;
  const float inf = __int_as_float(0x7f800000);
  u32 oa[V], ofl[V]; float ot[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    float valid = va4[j], time = ti4[j];
    const bool hit = cf4[j] > 0;
    if (hit) { valid = 1.f; time = 0.f; }                                    // CK.py:187-192
    u32 fl = (time < 0.5f ? RF_T05 : 0u) | (time < 1.0f ? RF_T10 : 0u)
           | ((double)(float)ci4[j] > c.wall_thresh ? RF_WALL : 0u);
    u32 a; float th;
    if (valid < 0.5f) {
      const bool unbounded = hit || iu4[j] < 0.5f;
      a = unbounded ? UKEY_NONE : fkey(up4[j]);
      th = unbounded ? inf : up4[j];                                         // NaN bound: `nz > NaN` never skips
    } else {
      fl |= RF_VALID;
      float h = h4[j];
      if (applied) h = __fadd_rn(h, shift);
      a = __float_as_uint(h);
      th = __fadd_rn(h, 0.06f);
      if (!(__fsub_rn(th, 0.05f) > h)) th = inf;                             // huge / NaN heights: never skip
      if (fl & RF_T05) th = -inf;
    }
    {   // border ring: make every ray skip the cell (see RF_* in emap_device.cuh)
      const int cc = cc0 + j;
      if (rr == 0 || rr == c.W - 1 || cc == 0 || cc == c.W - 1) { fl = RF_VALID | RF_T05 | RF_T10; th = -inf; }
    }
    oa[j] = a; ofl[j] = fl; ot[j] = th;
  }
  stv<V>(s.thr + i0, ot);
  {   // V cells of one row lie in one tile (V <= 4 <= 2^ts, cc0 - c0 a multiple of V)
    float m = -inf;
#pragma unroll
    for (int j = 0; j < V; j++) m = fmaxf(m, (ot[j] != ot[j]) ? inf : ot[j]);     // NaN threshold: never cull
    if (m > -inf) atomicMax(tmap + (((rr >> g.ts) - g.ta) * RT + ((cc0 >> g.ts) - g.tb)), fkey(m));
  }
  if (V == 4) {
    uint4* dst = reinterpret_cast<uint4*>(s.rec + i0);
    dst[0] = make_uint4(oa[0], ofl[0], oa[1 % V], ofl[1 % V]);
    dst[1] = make_uint4(oa[2 % V], ofl[2 % V], oa[3 % V], ofl[3 % V]);
  } else {
    for (int j = 0; j < V; j++) s.rec[i0 + j] = make_uint2(oa[j], ofl[j]);
  }
}

// step_cnt[b] = number of march steps s_k < x for the non-negative fp16 value x with bit pattern b (0 .. 0x7c00 = +inf)
__global__ void __launch_bounds__(256) k_build_step_cnt(const float* __restrict__ steps, int n_steps, unsigned short* __restrict__ step_cnt) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > 0x7c00) return;
  step_cnt[b] = (unsigned short)count_below(steps, n_steps, __half2float(__ushort_as_half((unsigned short)b)));
}

// fill the per-handle cell table (all 65536 fp16 bit patterns, CK.py:22-33 in its exact double form)
__global__ void __launch_bounds__(256) k_build_lut(const DevCfg c, unsigned short* __restrict__ lut) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= 65536) return;
  lut[b] = (unsigned short)axis_cell_exact(c, __half2float(__ushort_as_half((unsigned short)b)));
}

// CK.py:198-259 ray-cast half as a persistent kernel.  The rays of the frame were set up and compacted
// by k_index_error; every WARP pulls the next ray from a global work counter (dynamic balancing: ray
// lengths differ by 100x) and marches it with its 32 lanes on consecutive steps of the fp16 march
// variable s_k (shared table: s_0 = half(step), s_{k+1} = half(float(double(s_k) + step)), CK.py:203).
//   * cell of a sample: the fp16 coordinates half(t + ray*s_k) (CK.py:205-207,26-33) index a shared-memory
//     table of the exact cell of every fp16 value (TMA bulk copy of the handle's table, issued before the
//     dependency wait); coordinates are first clamped to [-LIM, LIM] (packed half2 min/max), beyond which
//     every value maps to cell 0 / W-1 anyway, so only the patterns [0, P) and [0x8000, 0x8000 + P) are staged.
//   * "same cell as the previous step" (CK.py:209-210) is a shuffle with the neighbouring lane; warp iterations
//     overlap by one step (lane 0 re-derives the last cell of the previous iteration and never visits).
//   * first level: one 4-byte load decides whether the sample can act at all (see k_record); the few that can
//     take the exact second level.  The effects of a visit are commutative integer atomics, so neither lane
//     nor ray order matters.
#define RC_THREADS 768
#define RC_CTL 64                 // ints of control state per sensor: [0] ray count, [32] the work counter (128 B apart)
#ifndef RC_BATCH
#define RC_BATCH 4                // rays a warp draws from the work counter at a time
#endif

// cell of the sample t + ray*s (CK.py:205-207 -> 26-33) through the staged table; all lanes must pass in-range addresses
__device__ __forceinline__ void rc_cell(const u32 s_lut, const u32 lim2, const u32 nlim2, const float nx, const float ny,
                                        u32& ix, u32& iy) {
  u32 xy;                                                         // {half(nx), half(ny)} clamped to [-LIM, LIM] (NaN -> -LIM -> cell 0)
  asm("{ .reg .b32 t; cvt.rn.f16x2.f32 t, %2, %1; max.f16x2 t, t, %3; min.f16x2 %0, t, %4; }"
      : "=r"(xy) : "f"(nx), "f"(ny), "r"(nlim2), "r"(lim2));
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(ix) : "r"(s_lut + ((xy & 0xffffu) << 1)));
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(iy) : "r"(s_lut + ((xy >> 16) << 1)));
}

template <bool COUNT>
__global__ void __launch_bounds__(RC_THREADS, 2)
k_raycast(const DevCfg c, const Pose q, const Ray* __restrict__ rays, int* __restrict__ ray_ctl,
          const float* __restrict__ map, const float* __restrict__ normal,
          const CellScratch s, const float* __restrict__ steps_tab, const int n_tab,
          const unsigned short* __restrict__ lut, const RayGrid g, const u32* __restrict__ tmap, const RcLayout lay,
          FrameScalars* fs) {
  // shared: [0, P2) cells of the non-negative fp16 patterns | [65536, 65536 + P2) negative patterns; in the gap between
  // them (or behind, if it is too small): coarse maps t8 (RT x RT) and t16 (RT/2 x RT/2), the march table
  // (n_tab floats: [0] dummy, [1 + k] = s_k, +inf padded) and the mbarrier of the bulk copies
  extern __shared__ __align__(128) unsigned char s_raw[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int P2 = c.lut_p2;
  float* s_steps = reinterpret_cast<float*>(s_raw + lay.off_steps);
  float* s_t8 = reinterpret_cast<float*>(s_raw + lay.off_t8);
  float* s_t16 = reinterpret_cast<float*>(s_raw + lay.off_t16);
  const u32 s_lut = (u32)__cvta_generic_to_shared(s_raw);
  const u32 sbar = s_lut + (u32)lay.off_bar;
  pdl_trigger();
  // static tables (written once at emap_create): staged before the dependency wait, under the previous kernel's tail
  if (tid == 0) {
    bar_expect(sbar, 2 * P2);
    bulk_copy(s_lut, lut, P2, sbar);
    bulk_copy(s_lut + 65536u, lut + 32768, P2, sbar);
  }
  for (int k = tid; k < n_tab; k += RC_THREADS) s_steps[k] = steps_tab[k];
  pdl_wait();
  // coarse maps of this frame (k_record): t8[a][b] = max thr over fine tile (a, b); t16[A][B] = max over the 3 x 3 block
  // of double-size tiles whose first one is (A, B), i.e. fine tiles [2A, 2A+6) x [2B, 2B+6): a warp iteration (31 steps,
  // < 22 cells per axis) whose first-corner tile is (A, B) stays inside that block.
  for (int k = tid; k < RT * RT; k += RC_THREADS) s_t8[k] = funkey(tmap[k] ? tmap[k] : 0x007fffffu);
  __syncthreads();
  for (int k = tid; k < (RT / 2) * (RT / 2); k += RC_THREADS) {
    const int A = k / (RT / 2), B = k - A * (RT / 2);
    float m = __int_as_float(0xff800000);                         // k_record never stores a NaN key
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++)
        if (2 * A + i < RT && 2 * B + j < RT) m = fmaxf(m, s_t8[(2 * A + i) * RT + 2 * B + j]);
    s_t16[k] = m;
  }
  __syncthreads();
  bar_wait(sbar, 0);
  const int n_rays = ray_ctl[0];
  const int W = c.W, C = c.C;
  const float tx = q.t[0], ty = q.t[1], tz = q.t[2];
  const u32 lim2 = c.lut_lim2, nlim2 = c.lut_lim2 ^ 0x80008000u;
  const u32 s_steps_a = s_lut + (u32)lay.off_steps;               // shared-space address of s_tab[0]
  const u32 s_t8_a = s_lut + (u32)lay.off_t8, s_t16_a = s_lut + (u32)lay.off_t16;
  const int ts = g.ts;
  const u32 s_t8_o = s_t8_a - 4u * (u32)(g.ta * RT + g.tb);      // address of the (virtual) entry of tile (0, 0)
  int n_steps_done = 0, n_visits = 0;
  // Work queue: one global counter; a warp draws RC_BATCH consecutive rays per atomic (all warps hammering ONE address
  // serialise at ~0.8 ns per atomic, which bounded the kernel at one ray per atomic) and draws its next batch when it
  // starts the last ray of the current one, so the atomic's latency is hidden by that ray's march.  Drawing at the start
  // of the batch instead reserved a whole batch ahead: when the queue ran dry, warps still held up to 2 batches and
  // finished over the last ~22 us of the kernel (per-warp %globaltimer stamps: 17 % of warp time idle at the end).
  // (Measured and dropped: several queues with rays dealt round-robin -- 4 % to 20 % slower, consecutive rays share cells
  // and belong in one warp; batches of 8 -- 11 % slower at config B, the tail gets ragged; a two-level queue, CTA chunks
  // from the global counter + shared-memory atomics per warp -- 2 % slower at B, 15 % at D: the prefetched global atomic
  // below hides its latency under the march, a shared-memory draw at the start of every batch does not.
  // On one H100 80GB HBM3 at 400 W, config B, raycast stage in bench.py: parent (draw at the batch start) 69.7-70.2 us,
  // this draw 63.8-64.0 us.  Two march iterations in flight per warp (two thr gathers per lane, 58-60 registers, one
  // 1024-thread CTA per SM) with this draw: 68.5-69.5 us at B and 325 us against 284 us at config D -- fewer warps cost
  // more latency hiding than the second gather gives; with the draw at the batch start 73.8-74.3 us (512 x 2: 77.3-78.2).
  // Loading a batch's four direction records at once and the next batch's after its first ray: no gain at B, and the
  // extra registers spill at 768 x 2.  Batches of 2 with this draw: 81.5-81.8 us, the single counter saturates.)
  int* next = ray_ctl + 32;
  int pend = 0;
  if (lane == 0) pend = atomicAdd(next, RC_BATCH);
  int rbase = __shfl_sync(0xffffffffu, pend, 0);
  while (rbase < n_rays) {
   for (int r = rbase; r < min(rbase + RC_BATCH, n_rays); r++) {
    if (lane == 0 && (r + 1 == rbase + RC_BATCH || r + 1 == n_rays)) pend = atomicAdd(next, RC_BATCH);   // next batch
    const float4 rb = __ldg(reinterpret_cast<const float4*>(rays + r) + 1);
    const float rx = rb.x, ry = rb.y, rz = rb.z;
    const int n_act = (int)(__float_as_uint(rb.w) & 0xffffu), k_far = (int)(__float_as_uint(rb.w) >> 16);
    const int n_it = (n_act + RC_STRIDE - 1) / RC_STRIDE;
    for (int it0 = 0; it0 < n_it; it0 += 32) {
      // ---- which of the next 32 warp iterations can act at all: lane L decides iteration it0 + L from the cells of its
      // first and last step (coordinates are monotone along the ray, so they bound the iteration's cells) and the lower of
      // the two sample heights, against the 3 x 3-block maximum of the coarse map
      u32 todo;
      {
        const int it = it0 + lane;
        bool live = it < n_it;
        const int ka = min(it * RC_STRIDE, n_act - 1), kb = min(it * RC_STRIDE + RC_STRIDE - 1, n_act - 1);
        float sa, sb;
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(sa) : "r"(s_steps_a + 4u * (u32)(max(ka, 0) + 1)));
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(sb) : "r"(s_steps_a + 4u * (u32)(max(kb, 0) + 1)));
        u32 ixa, iya, ixb, iyb;
        rc_cell(s_lut, lim2, nlim2, __fmaf_rn(rx, sa, tx), __fmaf_rn(ry, sa, ty), ixa, iya);
        rc_cell(s_lut, lim2, nlim2, __fmaf_rn(rx, sb, tx), __fmaf_rn(ry, sb, ty), ixb, iyb);
        const float zmin = fminf(__fmaf_rn(rz, sa, tz), __fmaf_rn(rz, sb, tz));
        const int A = (int)(min(ixa, ixb) >> (ts + 1)) - (g.ta >> 1), B = (int)(min(iya, iyb) >> (ts + 1)) - (g.tb >> 1);
        if (live && !COUNT && (unsigned)A < RT / 2 && (unsigned)B < RT / 2) {
          float m;
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(m) : "r"(s_t16_a + 4u * (u32)(A * (RT / 2) + B)));
          if (zmin > m) live = false;                             // NaN on either side: stays live
        }
        todo = __ballot_sync(0xffffffffu, live);
      }
      while (todo) {
        const int it = it0 + __ffs(todo) - 1;
        todo &= todo - 1;
        // lane l handles step k = it*31 + l - 1 (k = -1: none); lane 0 only supplies the previous cell
        const int k = it * RC_STRIDE + lane - 1;
        // lanes past the ray's end repeat its last step (same cell as their predecessor: skipped by CK.py:209 below); lane 0
        // of the first iteration reads the table's NaN entry -> cell (0, 0), a border cell no ray acts on
        const int kc = min(k, n_act - 1);
        float sk;
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(sk) : "r"(s_steps_a + 4u * (u32)(kc + 1)));
        const float nx = __fmaf_rn(rx, sk, tx);                   // t + ray*s: product exact (CK.py:205-207)
        const float ny = __fmaf_rn(ry, sk, ty);
        u32 ix, iy;
        rc_cell(s_lut, lim2, nlim2, nx, ny, ix, iy);
        const int nidx = (int)(ix * (u32)W + iy);
        const int prev = __shfl_up_sync(0xffffffffu, nidx, 1);    // lane 0 gets its own value back: never visits
        if (COUNT) n_steps_done += ((unsigned)k < (unsigned)n_act) && lane != 0;
        if (nidx == prev) continue;                               // CK.py:209 (CK.py:211: border cells are skipped via thr = -inf)
        const float nz = __fmaf_rn(rz, sk, tz);
        if (!COUNT) {   // coarse level: the fine tile's maximum (every cell a ray reaches lies in the tiled box: frame_rays
                        // launches no march when that box is empty)
          float m;
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(m) : "r"(s_t8_o + (ix >> ts) * (4u * RT) + ((iy >> ts) << 2)));
          if (nz > m) continue;
        }
        if (COUNT) {   // statistics mode: count the cells examined past the skips of CK.py:209-226, as the oracle does
          bool near = false;
          if (k >= k_far) {
            const float4 ra = __ldg(reinterpret_cast<const float4*>(rays + r));
            const float ddx = ra.x - nx, ddy = ra.y - ny, ddz = ra.z - nz;
            float d = __fmul_rn(ddy, ddy); d = __fmaf_rn(ddx, ddx, d); d = __fmaf_rn(ddz, ddz, d);
            near = h16(d) < 0.1f;
          }
          if (!near && cell_inside(W, (int)ix, (int)iy)) n_visits++;   // border cells are skipped first (CK.py:211)
        }
        if (nz > __ldg(s.thr + nidx)) continue;                   // first level: the sample cannot act on this cell
        // ---- second level (rare): the exact tests of CK.py:225-256
        const float4 ra = __ldg(reinterpret_cast<const float4*>(rays + r));      // end point, march length
        if (k >= k_far) {
          // CK.py:225-226 `d < 0.1` (d = fp16 of the squared distance to the end point); cannot fire for k < k_far
          // (bound derived where the ray is set up, k_index_error)
          const float ddx = ra.x - nx, ddy = ra.y - ny, ddz = ra.z - nz;
          float d = __fmul_rn(ddy, ddy); d = __fmaf_rn(ddx, ddx, d); d = __fmaf_rn(ddz, ddz, d);
          d = h16(d);
          if (d < 0.1f) continue;    // `d < 0.1` in double: no fp16 value lies in [0.1, 0.1f)
        }
        const uint2 rc = s.rec[nidx];
        if (!(rc.y & RF_VALID)) {                                 // CK.py:229-235 carve the upper bound
          const u32 key = fkey(nz);
          if (key < rc.x && key < __ldcg(s.ukv + nidx)) {
            red_min(s.ukv + nidx, key, s.mc_off);                 // true min over all rays (and ranks)
            if (s.dirty) s.dirty[2 * nidx + 1] = 1;
          }
          continue;
        }
        if (rc.y & RF_T05) continue;                              // CK.py:237
        const float nh = __uint_as_float(rc.x);
        // CK.py:239 needs nh > nz + 0.01 - min(v,1)*0.05 >= nz - 0.04: reject far-below cells in fp32
        if (nh < nz - 0.05f) continue;
        const float nv = add_n_times(__ldg(map + C + nidx), c.c_out, (u32)(s.cnt_fo[nidx] >> 32));
        const double rhs = fma(-fmin((double)nv, 1.0), 0.05, (double)nz + 0.01);   // CK.py:239 (nvcc contraction)
        if (!((double)nh > rhs)) continue;
        const float n0 = h16(__ldg(normal + nidx)), n1 = h16(__ldg(normal + C + nidx)), n2 = h16(__ldg(normal + 2 * C + nidx));
        const float product = __fadd_rn(__fadd_rn(__fmul_rn(rx, n0), __fmul_rn(ry, n1)), __fmul_rn(rz, n2));   // CK.py:103-108
        if ((double)fabsf(product) < c.cos_thresh) continue;      // CK.py:245
        if ((rc.y & RF_WALL) && (rc.y & RF_T10)) continue;        // CK.py:246-247
        const i64 dec_fix = fix32((float)(-c.cleanup_step / ((double)ra.w / c.max_ray_length)));   // CK.py:250
        red_add((u64*)(s.DV + nidx), (u64)dec_fix, s.mc_off);     // CK.py:250
        red_add(s.n_ray + nidx, 1u, s.mc_off);                    // CK.py:251
        red_min(s.ukv + nidx, fkey(nz), s.mc_off);                // CK.py:253-256
        if (s.dirty) s.dirty[2 * nidx + 1] = 1;
      }
    }
   }
    rbase = __shfl_sync(0xffffffffu, pend, 0);
  }
  if (COUNT) {
    for (int o = 16; o > 0; o >>= 1) {
      n_steps_done += __shfl_down_sync(0xffffffffu, n_steps_done, o);
      n_visits += __shfl_down_sync(0xffffffffu, n_visits, o);
    }
    if (lane == 0) {
      atomicAdd((u64*)&fs->ray_steps, (u64)n_steps_done);
      atomicAdd((u64*)&fs->ray_visits, (u64)n_visits);
    }
  }
}

// Apply every side effect of the frame to the state planes, then average_map_kernel
// (CK.py:362-384) and clear_overlap_map (EM.py:393-410); re-zero the consumed scratch.
// One cell, full path: everything the frame may have done to it.  The scratch falls into two groups, each written by one
// side of the frame: `pts` (cnt_fo, cnt_ai, SH, SV, last: the point passes) and `rays` (n_ray, ukv, DV: the ray-cast).  A
// group whose flag is clear still holds its between-frames value (zero; UKEY_NONE for ukv), so it is neither read nor
// re-zeroed.  cnt_ai is re-zeroed without being read: it is non-zero exactly where `pts` is set.  An overlap-window cell
// with neither flag reads only the map planes.
__device__ __forceinline__ void finalize_cell(const DevCfg& c, float* __restrict__ map, const CellScratch& s, const int i,
                                              const int applied, const float shift,
                                              const float hmin, const float hmax, const bool pts, const bool rays) {
  const size_t C = (size_t)c.C;
  // every load the flagged groups need up front, also the ones only some of their cells need (last / sums: fused points;
  // DV: rays that decrement): the kernel is bound by dependent round trips to L2 / DRAM, not by bytes, so one wave of loads
  // beats two dependent ones
  u64 fo = 0, last_key = 0;
  i64 sh_fix = 0, sv_fix = 0;
  if (pts) { fo = s.cnt_fo[i]; last_key = s.last[i]; sh_fix = s.SH[i]; sv_fix = s.SV[i]; }
  u32 nr = 0, kv = UKEY_NONE;
  i64 dv_fix = 0;
  if (rays) { nr = s.n_ray[i]; kv = s.ukv[i]; dv_fix = s.DV[i]; }
  const u32 cf = (u32)fo, no = (u32)(fo >> 32);
  const float h0 = map[i], v0 = map[C + i], va0 = map[2 * C + i], ti0 = map[4 * C + i], up0 = map[5 * C + i], iu0 = map[6 * C + i];
  float h = h0, v = v0, valid = va0, time = ti0, upper = up0, isup = iu0;
  if (applied) h = __fadd_rn(h, shift);                           // EM.py:357 applied lazily
  v = add_n_times(v, c.c_out, no);                                // CK.py:174
  if (cf > 0) {                                                   // CK.py:187-192
    valid = 1.f; time = 0.f; isup = 0.f;
    upper = __uint_as_float((u32)(last_key & 0xffffffffull));
  }
  if (rays) {
    const u32 key0 = (isup < 0.5f) ? UKEY_NONE : fkey(upper);
    if (nr > 0) {
      valid = __fadd_rn(valid, (float)unfix32(dv_fix));           // CK.py:250
      v = add_n_times(v, c.c_out, nr);                            // CK.py:251
    }
    // true min over rays (CK.py:230-233,253-256) of the keys carved into the cell
    const u32 ukey = min(key0, kv);
    if (ukey != key0) { upper = funkey(ukey); isup = 1.f; }
  }
  // average_map_kernel CK.py:362-384
  const float valid_in = valid;
  if (cf > 0) {
    const double cnt = (double)cf;
    const float mean_v = (float)(unfix32(sv_fix) / cnt);
    if ((double)mean_v > c.max_variance) { h = 0.f; v = c.init_var; valid = 0.f; }
    else { h = (float)(unfix32(sh_fix) / cnt); v = mean_v; valid = 1.f; }
  }
  if (valid_in < 0.5f) { h = 0.f; v = c.init_var; valid = 0.f; }
  // clear_overlap_map EM.py:393-410
  const int rr = (int)((u32)i / (u32)c.W), cc = i - rr * c.W;
  if (c.overlap && rr >= c.cell_min && rr < c.cell_max && cc >= c.cell_min && cc < c.cell_max) {
    if (h < hmin || h > hmax) { h = 0.f; v = c.init_var; valid = 0.f; }
    if (upper < hmin || upper > hmax) { upper = 0.f; isup = 0.f; }
  }
  if (applied || h != h0) map[i] = h;
  if (v != v0) map[C + i] = v;
  if (valid != va0) map[2 * C + i] = valid;
  if (time != ti0) map[4 * C + i] = time;
  if (upper != up0) map[5 * C + i] = upper;
  if (isup != iu0) map[6 * C + i] = isup;
  // re-zero the consumed scratch
  if (cf) { s.SH[i] = 0; s.SV[i] = 0; s.last[i] = 0; }
  if (fo) s.cnt_fo[i] = 0;
  if (nr) { s.DV[i] = 0; s.n_ray[i] = 0; }
  if (pts) s.cnt_ai[i] = 0;                                       // every point that sets the flag counts into cnt_ai
  if (kv != UKEY_NONE) s.ukv[i] = UKEY_NONE;
}

// V consecutive cells per thread.  A frame touches few cells (< 15 % at config B): the two markers of a cell (a points
// byte set by k_index_error, a rays byte set by k_raycast; in sharded frames derived from the all-reduced cnt_all / ukv)
// select the full path and which scratch groups it reads; everywhere else only the drift shift (EM.py:357) and the reset
// of invalid cells (CK.py:380-384) remain: 3 planes read, at most 3 written, as vectors.  The cells that need the full
// path are compacted per warp (shared-memory list, index << 2 | group flags) and then finalised one per LANE, so the rare
// path runs converged.
#ifndef FIN_MINB
#define FIN_MINB 4
#endif
template <int V>
__global__ void __launch_bounds__(256, FIN_MINB)
k_finalize(const DevCfg c, float* __restrict__ map, const CellScratch s, const FrameScalars* __restrict__ fs,
           const int rays_ran, int* __restrict__ ray_ctl, const int n_ctl, FrameScalars* fs_reset, u32* __restrict__ tmap) {
  __shared__ int s_list[8][32 * V];
  pdl_trigger(); pdl_wait();
  if (blockIdx.x == 0) for (int k = threadIdx.x; k < n_ctl; k += blockDim.x) ray_ctl[k] = 0;   // consumed by k_raycast: next frame's
  if (fs_reset && blockIdx.x == 1 % gridDim.x) {     // frames without k_drift: the housekeeping it would do for the next frame
    for (int k = threadIdx.x; k < RT * RT; k += blockDim.x) tmap[k] = 0u;
    if (threadIdx.x == 0) { fs_reset->E = 0; fs_reset->ecnt = 0; fs_reset->nvalid = 0; fs_reset->nkept = 0; }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // blocks in centre-first order (bmid, bmid + 1, bmid - 1, bmid + 2, ...): the map is centred on the robot, so the rows the
  // frame touches (the points near the sensor, the overlap window) are the middle ones, and their blocks, which take the
  // full path, start in the first wave instead of finishing the last
  const int bmid = gridDim.x / 2, boff = (blockIdx.x + 1) / 2;
  const int blk = (blockIdx.x & 1) ? bmid - boff : bmid + boff;
  const int i0 = (blk * blockDim.x + threadIdx.x) * V;
  const size_t C = (size_t)c.C;
  const int applied = fs->applied;
  const float shift = fs->shift;
  static_assert(V == 1 || V == 4, "k_finalize: 1 or 4 cells per thread");
  u32 full = 0, pm = 0, rm = 0;      // bit j: cell i0 + j takes the full path / its points group / its rays group is read
  int r = 0, col0 = 0;
  if (i0 < c.C) {
    r = i0 / c.W; col0 = i0 - r * c.W;                             // V == 4 only when W % 4 == 0: one row per thread
    if (s.dirty) {
      unsigned char* mk = s.dirty + 2 * (size_t)i0;                // the V cells' markers: one 8-byte (V = 4) or 2-byte load
      const u64 d = V == 4 ? *reinterpret_cast<const u64*>(mk) : (u64)*reinterpret_cast<const unsigned short*>(mk);
      if (d) {
        if (V == 4) *reinterpret_cast<u64*>(mk) = 0ull; else *reinterpret_cast<unsigned short*>(mk) = 0;
#pragma unroll
        for (int j = 0; j < V; j++) {
          if ((d >> (16 * j)) & 0xffu) pm |= 1u << j;
          if ((d >> (16 * j + 8)) & 0xffu) rm |= 1u << j;
        }
      }
    } else {
      // DV and n_ray are only ever accumulated together with a red_min on ukv: ukv != UKEY_NONE covers the rays group
      u64 ca[V]; u32 kv[V];
      ldv64<V>(s.cnt_ai + i0, ca); ldv<V>(s.ukv + i0, kv);
      for (int j = 0; j < V; j++) {
        if (ca[j] != 0ull) pm |= 1u << j;
        if (kv[j] != UKEY_NONE) rm |= 1u << j;
      }
    }
    if (!rays_ran) rm = 0;
    full = pm | rm;
    if (c.overlap && r >= c.cell_min && r < c.cell_max)            // clear_overlap_map window (EM.py:393-410)
      for (int j = 0; j < V; j++) if (col0 + j >= c.cell_min && col0 + j < c.cell_max) full |= 1u << j;
    if (full != (1u << V) - 1u) {
      float h0[V], v0[V], va0[V], h4[V], v4[V], va4[V];
      ldv<V>(map + i0, h0); ldv<V>(map + C + i0, v0); ldv<V>(map + 2 * C + i0, va0);
#pragma unroll
      for (int j = 0; j < V; j++) {
        const bool inval = va0[j] < 0.5f;                         // CK.py:380-384
        h4[j] = inval ? 0.f : (applied ? __fadd_rn(h0[j], shift) : h0[j]);
        v4[j] = inval ? c.init_var : v0[j];
        va4[j] = inval ? 0.f : va0[j];
      }
      if (full == 0) {
        if (applied || diffv<V>(h4, h0)) stv<V>(map + i0, h4);
        if (diffv<V>(v4, v0)) stv<V>(map + C + i0, v4);
        if (diffv<V>(va4, va0)) stv<V>(map + 2 * C + i0, va4);
      } else {
#pragma unroll
        for (int j = 0; j < V; j++) {
          if ((full >> j) & 1u) continue;                         // finalised below by whichever lane picks it up
          if (applied || h4[j] != h0[j]) map[i0 + j] = h4[j];
          if (v4[j] != v0[j]) map[C + i0 + j] = v4[j];
          if (va4[j] != va0[j]) map[2 * C + i0 + j] = va4[j];
        }
      }
    }
  }
  // warp-level compaction of the full-path cells
  const int nfull = __popc(full);
  int incl = nfull;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += o; }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  if (total == 0) return;
  int pos = incl - nfull;
  for (int j = 0; j < V; j++)      // C <= 2049^2 < 2^23: the index shifted by 2 fits an int
    if ((full >> j) & 1u) s_list[wid][pos++] = ((i0 + j) << 2) | (int)((pm >> j) & 1u) | (int)(((rm >> j) & 1u) << 1);
  __syncwarp();
  const float hmin = __fsub_rn(fs->overlap_tz, c.overlap_z_f), hmax = __fadd_rn(fs->overlap_tz, c.overlap_z_f);
  for (int e = lane; e < total; e += 32) {
    const int ent = s_list[wid][e];
    finalize_cell(c, map, s, ent >> 2, applied, shift, hmin, hmax, ent & 1, (ent >> 1) & 1);
  }
}

// ------------------------------------------------------------------------------------------
// k_post: dilation (CK.py:392-449) of upper_bound with mask = is_valid + is_upper_bound
// (EM.py:376-383) -> traversability_input; traversability CNN (traversability_filter.py:15-42)
// -> map[3][3:-3,3:-3] (EM.py:385-388); normals of the dilated map (CK.py:452-506, EM.py:564-577).
// One CTA per PT_Y x PT_X tile; the (tile + halo) of the two input planes is staged in shared
// memory once, the dilated tile (+3 halo) stays in shared memory for the CNN and the normals.  The tile size and the
// shared-memory size are in emap_plan.cuh.

// two channels' taps: acc.{x,y} = fma(w.{x,y}, t, acc.{x,y}), each IEEE round-to-nearest.  Hopper has no paired
// fp32 FMA, so this is two scalar FFMAs (the same rounding, so the same bits).
__device__ __forceinline__ void ffma2(float2& acc, const float2 w, const float t) {
  acc.x = __fmaf_rn(w.x, t, acc.x);
  acc.y = __fmaf_rn(w.y, t, acc.y);
}

// K = dilation_size as a compile-time constant (0 = use c.dilation at run time).
template <int KT>
__global__ void __launch_bounds__(256)
k_post(const DevCfg c, float* __restrict__ map, float* __restrict__ trav_input, float* __restrict__ normal,
       const __grid_constant__ CUtensorMap tm) {
  extern __shared__ __align__(128) float smem[];
  pdl_trigger(); pdl_wait();
  const int W = c.W, C = c.C;
  const int K = KT ? KT : c.dilation;
  const int HL = K + 3;                          // row halo of the staged inputs
  const int HLX = (HL + 3) & ~3;                 // column halo rounded up to 16 bytes: every staged row segment
                                                 // starts on a 16-byte boundary, as the TMA bulk copy needs
  const int A = PT_Y + 2 * HL, B = PT_X + 2 * HLX;
  constexpr int DA = PT_Y + 6, DB = PT_X + 6;
  const int PS = (A * B + 31) & ~31;             // plane stride in floats: every staged plane starts on a 128-byte boundary (TMA)
  float* s_up = smem;                            // A*B   upper_bound
  float* s_mask = s_up + PS;                     // A*B   is_valid, then the raw mask = is_valid + is_upper_bound (CK.py:424)
  float* s_iu = s_mask + PS;                     // A*B   is_upper_bound (TMA path only)
  float* s_dil = s_iu + PS;                      // DA*DB dilated tile (+3 halo)
  unsigned long long* s_rowsel = reinterpret_cast<unsigned long long*>(s_dil + DA * DB + ((DA * DB) & 1));   // A words
  unsigned long long* s_bar = s_rowsel + A;      // mbarrier of the tensor copies
  const float* up = map + 5 * C; const float* valid = map + 2 * C; const float* isup = map + 6 * C;
  const int r0 = blockIdx.y * PT_Y, c0 = blockIdx.x * PT_X;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  // Stage upper_bound / is_valid / is_upper_bound for the tile + halo: three TMA tensor copies (cp.async.bulk.tensor.3d
  // of a B x A x 1 box of the (W, W, 7) state tensor; elements outside the map arrive as zeros) completing on one
  // mbarrier.  Maps whose row pitch is not a multiple of 16 bytes cannot be described to the TMA unit: plain loads.
  const bool bulk = c.post_tma != 0;
  if (bulk) {
    const u32 sbar = (u32)__cvta_generic_to_shared(s_bar);
    if (tid == 0) {
      bar_expect(sbar, 3 * A * B * 4);
#pragma unroll
      for (int pl = 0; pl < 3; pl++)
        tensor_copy_3d((u32)__cvta_generic_to_shared(pl == 0 ? s_up : pl == 1 ? s_mask : s_iu), &tm, c0 - HLX, r0 - HL,
                       pl == 0 ? 5 : pl == 1 ? 2 : 6, sbar);
    }
    __syncthreads();                             // the barrier is initialised before anyone polls it
    bar_wait(sbar, 0);
  }
  // raw mask + per staged row one 64-bit word whose bit b says "cell (a,b) may be SELECTED as a neighbour"
  // (CK.py:432-434: is_inside && mask > 0.5), built with warp ballots (B <= 64)
  int any_sel = 0;
  for (int a = ty; a < A; a += 8) {
    const int r = r0 - HL + a;
    u32 bits[2];
#pragma unroll
    for (int ch = 0; ch < 2; ch++) {
      const int b = tx + 32 * ch;
      const int cc = c0 - HLX + b;
      float m = 0.f;
      const bool in_stage = b < B;
      if (bulk) {
        if (in_stage) { m = __fadd_rn(s_mask[a * B + b], s_iu[a * B + b]); s_mask[a * B + b] = m; }
      } else {
        float u = 0.f;
        if (in_stage && r >= 0 && r < W && cc >= 0 && cc < W) {
          const int gi = r * W + cc;
          u = __ldg(up + gi);
          m = __fadd_rn(__ldg(valid + gi), __ldg(isup + gi));
        }
        if (in_stage) { s_up[a * B + b] = u; s_mask[a * B + b] = m; }
      }
      const bool sel = in_stage && r > 0 && r < W - 1 && cc > 0 && cc < W - 1 && m > 0.5f;
      bits[ch] = __ballot_sync(0xffffffffu, sel);
    }
    if (tx == 0) s_rowsel[a] = ((unsigned long long)bits[1] << 32) | bits[0];
    any_sel |= (bits[0] | bits[1]) != 0;
  }
  any_sel = __syncthreads_or(any_sel);
  for (int e = tid; e < DA * DB; e += 256) {
    const int a = e / DB, b = e - a * DB;
    const int r = r0 - 3 + a, cc = c0 - 3 + b;
    float out = 0.f;
    if (r >= 0 && r < W && cc >= 0 && cc < W) {
      if (cc >= K - 1 && cc <= W - K) {          // no wrapped neighbour can be selected: shared-memory path
        const int sa = a + K, sb = b + HLX - 3;  // position in the staged planes (HL - 3 == K rows, HLX - 3 columns)
        out = s_up[sa * B + sb];
        if (any_sel && s_mask[sa * B + sb] < 0.5f) {
          // windows of selectable neighbours, one (2K+1)-bit word per row; first hit in
          // (dx+dy ascending, dy ascending) order == the reference's strict-< scan (CK.py:429-438)
          // Row dy's (2K+1)-bit window of selectable neighbours, shifted left by (dy+K), puts the
          // neighbour (dy,dx) at bit s' = (dx+K)+(dy+K): the reference's strict-< scan (CK.py:429-438)
          // picks the smallest dx+dy, ties to the smallest dy == lowest set bit of the OR, then the
          // first row that has it.  Branch-free, all lanes.
          if (KT) {
            // compile-time K: the shifted row windows stay in registers; the winner row is the first whose term has bit s'
            constexpr int KK = KT ? KT : 1;
            const u32 wmask = (1u << (2 * KK + 1)) - 1u;
            u32 term[2 * KK + 1], any = 0;
#pragma unroll
            for (int i = 0; i <= 2 * KK; i++) {
              term[i] = ((u32)(s_rowsel[sa + i - KK] >> (sb - KK)) & wmask) << i;
              any |= term[i];
            }
            if (any) {
              const int sp = __ffs(any) - 1;                     // s' of the winner
              int iw = 2 * KK;
#pragma unroll
              for (int i = 2 * KK - 1; i >= 0; i--) if ((term[i] >> sp) & 1u) iw = i;
              out = s_up[(sa + iw - KK) * B + sb + (sp - iw - KK)];
            }
          } else {
            const u64 wmask = (1ull << (2 * K + 1)) - 1ull;      // s' reaches 4K = 32 at K = 8: 64-bit words
            u64 any = 0;
            for (int dy = -K; dy <= K; dy++)
              any |= ((s_rowsel[sa + dy] >> (sb - K)) & wmask) << (dy + K);
            if (any) {
              const int sp = __ffsll((long long)any) - 1;
              int dyw = K;
              for (int dy = K; dy >= -K; dy--) {
                const int dx = sp - (dy + K) - K;
                if (dx >= -K && dx <= K && ((s_rowsel[sa + dy] >> (sb + dx)) & 1ull)) dyw = dy;
              }
              out = s_up[(sa + dyw) * B + sb + (sp - (dyw + K) - K)];
            }
          }
        }
      }
      // else: one of the K-1 outermost columns -> filled below, one warp per cell
    }
    s_dil[e] = out;
  }
  // Border columns (cc <= K-2 or cc >= W-K+1): the flat-index window of CK.py:403-407 wraps into the adjacent
  // row there.  Rare (2(K-1) columns of the map), so: one WARP per cell, lanes over the (2K+1)^2 candidates,
  // priority key = (dx+dy, dy) as in the scan of CK.py:429-438, warp-min picks the winner.
  if (K >= 2 && (c0 - 3 < K - 1 || c0 + PT_X + 3 > W - K)) {       // block-uniform condition
    __syncthreads();     // the loop above stored a placeholder for these cells from OTHER threads: order the two writes
    const int lane = tid & 31, warp = tid >> 5, side = 2 * K + 1;
    // the border columns this tile (+3 halo) covers: [la, la + nl) on the left edge, [ra, ra + nr) on the right edge
    const int la = max(c0 - 3, 0), nl = max(0, min(c0 - 3 + DB - 1, K - 2) - la + 1);
    const int ra = max(max(c0 - 3, W - K + 1), K - 1), nr = max(0, min(c0 - 3 + DB - 1, W - 1) - ra + 1);
    const int nc = nl + nr;
    for (int e2 = warp; e2 < DA * nc; e2 += 8) {
      const int a = e2 / nc, j = e2 - a * nc;
      const int r = r0 - 3 + a, cc = j < nl ? la + j : ra + (j - nl);
      const int e = a * DB + (cc - (c0 - 3));
      if (r < 0 || r >= W) continue;                                                           // warp-uniform
      const int i = r * W + cc;
      float out = up[i];
      if (__fadd_rn(valid[i], isup[i]) < 0.5f) {
        // row and column of the flat index i + W*dy + dx of for_window: one wrap step finds them, as |dx| <= K <= 8 <= W
        auto wrap = [&](int dy, int dx) {
          int rr = r + dy, c2 = cc + dx;
          if (c2 < 0) { c2 += W; rr -= 1; } else if (c2 >= W) { c2 -= W; rr += 1; }
          return make_int2(rr, c2);
        };
        u32 best = 0xffffffffu;
        for (int cand = lane; cand < side * side; cand += 32) {
          const int dy = cand / side - K, dx = cand - (dy + K) * side - K;
          const int2 n = wrap(dy, dx);
          if (n.x <= 0 || n.x >= W - 1 || n.y <= 0 || n.y >= W - 1) continue;
          const int idx = n.x * W + n.y;
          if (__fadd_rn(valid[idx], isup[idx]) > 0.5f) best = min(best, (u32)((dx + dy + 2 * K) << 8 | (dy + K)));
        }
        best = __reduce_min_sync(0xffffffffu, best);
        if (best != 0xffffffffu) {
          const int dy = (int)(best & 255u) - K, dx = (int)(best >> 8) - 2 * K - dy;
          const int2 n = wrap(dy, dx);
          out = up[n.x * W + n.y];
        }
      }
      if (lane == 0) s_dil[e] = out;
    }
  }
  __syncthreads();
#pragma unroll
  for (int half = 0; half < PT_Y / 8; half++) {
    const int a = ty + half * 8, b = tx;
    const int r = r0 + a, cc = c0 + b;
    if (r >= W || cc >= W) continue;
    const int gi = r * W + cc;
    const float* d = s_dil + (a + 3) * DB + (b + 3);
    const float h = d[0];
    trav_input[gi] = h;
    // traversability CNN; summation order = oracle_traversability
    if (r >= 3 && r <= W - 4 && cc >= 3 && cc <= W - 4) {
      float acc = 0.f;
#pragma unroll
      for (int l = 0; l < 3; l++) {
        const int dil = l + 1;
        float t[9];
#pragma unroll
        for (int p = 0; p < 3; p++)
#pragma unroll
          for (int qq = 0; qq < 3; qq++) t[p * 3 + qq] = d[(p - 1) * dil * DB + (qq - 1) * dil];
#pragma unroll
        for (int cp = 0; cp < 2; cp++) {                           // channels 2cp, 2cp+1 of each tap
          float2 s2 = make_float2(0.f, 0.f);
#pragma unroll
          for (int j = 0; j < 9; j++) ffma2(s2, c.wp[l][cp][j], t[j]);
          acc = __fmaf_rn(c.wout[l * 4 + 2 * cp], fabsf(s2.x), acc);
          acc = __fmaf_rn(c.wout[l * 4 + 2 * cp + 1], fabsf(s2.y), acc);
        }
      }
      map[3 * C + gi] = expf(-acc);
    }
    // normals CK.py:486-501 (normal_map is cleared first, EM.py:571)
    float3 n = make_float3(0.f, 0.f, 0.f);
    if (__ldg(valid + gi) > 0.5f && r >= 1 && r <= W - 3 && cc >= 1 && cc <= W - 3) n = surface_normal(h, d[1], d[DB], c.res_f);
    normal[gi] = n.x; normal[C + gi] = n.y; normal[2 * C + gi] = n.z;
  }
}

// EM.py:564-577 update_normal(dilated_map) with an arbitrary device plane
__global__ void __launch_bounds__(256)
k_normal(const DevCfg c, const float* __restrict__ dil, const float* __restrict__ valid, float* __restrict__ normal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const int W = c.W, r = i / W, cc = i - r * W;
  float3 n = make_float3(0.f, 0.f, 0.f);
  if (valid[i] > 0.5f && r >= 1 && r <= W - 3 && cc >= 1 && cc <= W - 3) n = surface_normal(dil[i], dil[i + 1], dil[i + W], c.res_f);
  normal[i] = n.x; normal[c.C + i] = n.y; normal[2 * c.C + i] = n.z;
}

// ------------------------------------------------------------------------------------------
// pose / time
// EM.py:200-226: roll by (sx, sy) cells, pad the vacated strips (0, variance = initial), add dz to
// elevation and upper_bound (float32 plane + float64 scalar -> computed in double, stored fp32).
__global__ void __launch_bounds__(256)
k_shift(const DevCfg c, const float* __restrict__ src, float* __restrict__ dst, int sx, int sy, double dz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const int W = c.W, r = i / W, cc = i - r * W;
  const size_t C = (size_t)c.C;
  const bool pad = (sx > 0 && r < sx) || (sx < 0 && r >= W + sx) || (sy > 0 && cc < sy) || (sy < 0 && cc >= W + sy);
  float v[7];
  if (pad) {
#pragma unroll
    for (int l = 0; l < 7; l++) v[l] = (l == L_V) ? c.init_var : 0.f;
  } else {
    int rs = r - sx, cs = cc - sy;
    rs = ((rs % W) + W) % W; cs = ((cs % W) + W) % W;
    const size_t si = (size_t)rs * W + cs;
#pragma unroll
    for (int l = 0; l < 7; l++) v[l] = __ldg(src + l * C + si);     // one index computation, seven loads in flight
  }
  v[L_H] = (float)((double)v[L_H] + dz); v[L_UPPER] = (float)((double)v[L_UPPER] + dz);
#pragma unroll
  for (int l = 0; l < 7; l++) dst[l * C + i] = v[l];
}
__global__ void __launch_bounds__(256) k_shift_z(const DevCfg c, float* __restrict__ map, double dz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  map[i] = (float)((double)map[i] + dz);
  map[5 * c.C + i] = (float)((double)map[5 * c.C + i] + dz);
}
__global__ void __launch_bounds__(256) k_clear(const DevCfg c, float* __restrict__ map) {   // EM.py:119-125
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  for (int l = 0; l < 7; l++) map[(size_t)l * c.C + i] = (l == L_V) ? c.init_var : 0.f;
}
__global__ void __launch_bounds__(256) k_init(const DevCfg c, float* __restrict__ map) {    // EM.py:68-85
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  for (int l = 0; l < 7; l++) map[(size_t)l * c.C + i] = (l == L_V) ? c.init_var : (l == L_TRAV ? 1.f : 0.f);
}
__global__ void __launch_bounds__(256) k_update_variance(const DevCfg c, float* __restrict__ map) {   // EM.py:420-422
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  map[c.C + i] = __fadd_rn(map[c.C + i], __fmul_rn(c.time_var_f, map[2 * c.C + i]));
}
__global__ void __launch_bounds__(256) k_update_time(const DevCfg c, float* __restrict__ map) {       // EM.py:424-426
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  map[4 * c.C + i] = __fadd_rn(map[4 * c.C + i], c.time_int_f);
}
