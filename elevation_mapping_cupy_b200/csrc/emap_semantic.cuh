// emap_semantic.cuh -- point-channel semantic fusion of a frame (SURVEY 8(f)2), sm_90a.
//
// Reference: semantic_map.py:223-259 (update_layers_pointcloud, called from elevation_mapping.py:371 right after
// average_map_kernel), fusion/pointcloud_average.py:22-113, fusion/pointcloud_class_average.py, and
// fusion/pointcloud_color.py:15-152.  There, each fusion algorithm launches a scatter kernel over
// (point, channel) -- float atomicAdd of the feature into new_map[layer] for every valid + inside point, or r/g/b/count
// integer sums for a colour channel -- and a dense kernel over (cell, channel) that writes the layer from the sums and
// the frame's fused-point count new_map[2] (CK.py:185).
// Here: ONE scatter kernel over the frame's points for all channels of all algorithms (it reads the packed
// (idx, valid, inside) record k_index_error left on the device and the feature columns of the frame's point source), and ONE
// per-cell kernel, both inside the frame (after k_fuse, before k_finalize re-zeroes the counts).  Float sums are
// accumulated in 2^-32 fixed point like the height sums: order-independent, deterministic, within one rounding of any
// order of the reference's float atomics.
// class_bayesian (fusion/pointcloud_class_bayesian.py) and bayesian_inference (pointcloud_bayesian_inference.py) ride on
// the same two kernels.  class_max (pointcloud_class_max.py) needs rounds across cells (a class that wins at any cell is
// zeroed everywhere for the later rounds), so it adds its own passes between them, see "class_max" below.  DESIGN §4d
// defines all three where the reference crashes or degenerates.
#pragma once
#include "emap_kernels.cuh"       // red_add
#include "emap_sources.cuh"

// ---- class_max scratch ------------------------------------------------------------------------------------------------
// U = the class ids of the frame's non-dropped rows and of id_max: one 65 536-bit bitmap.  Every valid + inside point
// brings n_max (id, fp16 probability) records to its cell; cell c owns the table slots [off[c], off[c] + cnt[c]) and
// hashes its ids into them (open addressing, one slot per record, so a cell's distinct ids always fit).  A slot sums its
// id's probabilities in 2^-24 fixed point (exact for fp16) and flags the non-finite ones.  Memory: O(C) per-cell words
// and O(N * n_max) slots; nothing grows with the number of classes.
#define CM_WORDS 2048                  // 65 536 ids / 32
enum { CM_TOTAL = 0, CM_OCC = 1, CM_UMIN = 2, CM_NU = 3, CM_CTL = 8 };
enum { CM_POS_INF = 1, CM_NEG_INF = 2, CM_NAN = 4 };

struct SemMax {
  u32* cnt;       // (C) records of the cell this frame; zero between frames (k_sem_apply)
  u32* off;       // (C) first table slot of the cell (valid where cnt > 0)
  u32* occ;       // cells with records, in no particular order
  u32* ctl;       // CM_CTL words: slots handed out, occupied cells, smallest id of U, |U|; then the bitmaps:
                  // U at ctl + CM_CTL, the winners of round k at ctl + CM_CTL + (1 + k) * CM_WORDS
  u32* ulist;     // the ids of U, ascending
  u32* key;       // table: id + 1 (0: empty)
  u32* flag;      // table: CM_* of the non-finite probabilities
  i64* sum;       // table: 2^-24 fixed-point sum of the finite probabilities
};

__device__ __forceinline__ u32 cm_hash(u32 id, u32 m) { return (id * 2654435761u) % m; }

// the fp32 value of a slot: NaN if a NaN or both infinities were summed, else the infinity, else the fixed-point sum
__device__ __forceinline__ float cm_value(u32 f, i64 s) {
  if ((f & CM_NAN) || (f & (CM_POS_INF | CM_NEG_INF)) == (CM_POS_INF | CM_NEG_INF)) return __int_as_float(0x7fffffff);
  if (f & CM_POS_INF) return __int_as_float(0x7f800000);
  if (f & CM_NEG_INF) return __int_as_float(0xff800000);
  return __fmul_rn(__ll2float_rn(s), 5.9604644775390625e-08f);          // * 2^-24: exact
}

// scatter: fusion/pointcloud_average.py:41-52 (sum_kernel), fusion/pointcloud_color.py:51-61 (add_color_kernel)
// fusion/pointcloud_class_bayesian.py alpha_kernel (theta >= 0 only), pointcloud_bayesian_inference.py
// sum_compact_kernel and pointcloud_class_max.py sum_max_kernel (into the cell's hash table), every (point, channel).
// MC (sharded frames on a multicast-attached block): the sums go to every rank's replica through red_add at mc_off;
// otherwise mc_off is unused and the sums are local atomics.
template <typename Src, bool MC>
__global__ void __launch_bounds__(256)
k_sem_sum(const DevCfg c, const SemCfg sc, const Src src, const i64 n,
          const int* __restrict__ pidx, i64* __restrict__ fsum, u32* __restrict__ csum, const SemMax ms, const i64 mc_off) {
  const i64 mc = MC ? mc_off : 0;
  const i64 i = blockIdx.x * (i64)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int rec = pidx[i];
  if ((rec & (PT_VALID | PT_INSIDE | PT_SKIP)) != (PT_VALID | PT_INSIDE)) return;     // `if (valid) if (inside)`
  const int idx = rec & PT_IDX_MASK;
  const size_t C = (size_t)c.C;
  for (int k = 0; k < sc.n_ch; k++) {
    const float feat = src.feature(i, sc.col[k]);
    if (sc.kind[k] == SEM_COLOR) {
      const u32 color = __float_as_uint(feat);                    // pointcloud_color.py:56-60
      u32* p = csum + (size_t)sc.slot[k] * C + idx;
      red_add(p, (color >> 16) & 0xffu, mc);
      red_add(p + C, (color >> 8) & 0xffu, mc);
      red_add(p + 2 * C, color & 0xffu, mc);
      red_add(p + 3 * C, 1u, mc);
    } else if (sc.kind[k] == SEM_CLASS_MAX) {
      const u32 bits = __float_as_uint(feat);                     // decode_max: fp16 probability | class id << 16
      const u32 id = bits >> 16;
      const float prob = __half2float(__ushort_as_half((unsigned short)(bits & 0xffffu)));
      const u32 m = ms.cnt[idx], base = ms.off[idx];
      u32 s = cm_hash(id, m);
      for (;;) {
        const u32 kk = atomicCAS(ms.key + base + s, 0u, id + 1);
        if (kk == 0u || kk == id + 1) break;
        if (++s == m) s = 0;
      }
      if (prob != prob) atomicOr(ms.flag + base + s, (u32)CM_NAN);
      else if (isinf(prob)) atomicOr(ms.flag + base + s, (u32)(prob > 0.f ? CM_POS_INF : CM_NEG_INF));
      else atomicAdd((u64*)(ms.sum + base + s), (u64)__float2ll_rn(__fmul_rn(prob, 16777216.0f)));
    } else {
      if (sc.kind[k] == SEM_CLASS_BAYESIAN && !(feat >= 0.f)) continue;     // alpha_kernel: `if (theta >= theta_max)`
      red_add((u64*)(fsum + (size_t)sc.slot[k] * C + idx), (u64)fix32(feat), mc);
    }
  }
}

// class_max, before the scatter: U (ids of every non-dropped row, and of the first n_idm entries of id_max) and the
// records per cell.  Grid-stride; each block ORs into a shared bitmap and flushes its non-zero words once.
template <typename Src>
__global__ void __launch_bounds__(256)
k_cm_count(const SemCfg sc, const Src src, const i64 n, const int* __restrict__ pidx,
           const int* __restrict__ idm, const i64 n_idm, const SemMax ms) {
  __shared__ u32 bm[CM_WORDS];
  for (int w = threadIdx.x; w < CM_WORDS; w += blockDim.x) bm[w] = 0;
  __syncthreads();
  const i64 step = (i64)gridDim.x * blockDim.x;
  for (i64 i = blockIdx.x * (i64)blockDim.x + threadIdx.x; i < n; i += step) {
    const int rec = pidx[i];
    if (rec & PT_SKIP) continue;                                  // EM.py:458 dropped the row: not in points_all
    for (int k = 0; k < sc.n_ch; k++) {
      if (sc.kind[k] != SEM_CLASS_MAX) continue;
      const u32 id = __float_as_uint(src.feature(i, sc.col[k])) >> 16;
      atomicOr(bm + (id >> 5), 1u << (id & 31));
    }
    if ((rec & (PT_VALID | PT_INSIDE)) == (PT_VALID | PT_INSIDE)) atomicAdd(ms.cnt + (rec & PT_IDX_MASK), (u32)sc.n_max);
  }
  for (i64 j = blockIdx.x * (i64)blockDim.x + threadIdx.x; j < n_idm; j += step) {
    const u32 id = (u32)idm[j] & 0xffffu;
    atomicOr(bm + (id >> 5), 1u << (id & 31));
  }
  __syncthreads();
  for (int w = threadIdx.x; w < CM_WORDS; w += blockDim.x)
    if (bm[w]) atomicOr(ms.ctl + CM_CTL + w, bm[w]);
}

// class_max, per cell: the cell's table slots and its place in the list of occupied cells (one atomic per warp each)
__global__ void __launch_bounds__(256) k_cm_alloc(const int C, const SemMax ms) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const u32 m = i < C ? ms.cnt[i] : 0u;
  const int lane = threadIdx.x & 31;
  u32 incl = m;                                                   // inclusive warp prefix of the record counts
  for (int d = 1; d < 32; d <<= 1) {
    const u32 v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  const u32 occ = __ballot_sync(0xffffffffu, m > 0);
  u32 base = 0, obase = 0;
  if (lane == 31 && incl) { base = atomicAdd(ms.ctl + CM_TOTAL, incl); obase = atomicAdd(ms.ctl + CM_OCC, (u32)__popc(occ)); }
  base = __shfl_sync(0xffffffffu, base, 31);
  obase = __shfl_sync(0xffffffffu, obase, 31);
  if (m > 0) {
    ms.off[i] = base + incl - m;
    ms.occ[obase + __popc(occ & ((1u << lane) - 1))] = (u32)i;
  }
}

// class_max: U as an ascending id list, its smallest id and its size (one block of 1024 threads, two words each)
__global__ void __launch_bounds__(1024) k_cm_ulist(const SemMax ms) {
  __shared__ u32 wsum[32];
  const u32* U = ms.ctl + CM_CTL;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const u32 w0 = U[2 * t], w1 = U[2 * t + 1];
  const u32 own = __popc(w0) + __popc(w1);
  u32 incl = own;
  for (int d = 1; d < 32; d <<= 1) {
    const u32 v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  u32 before = 0;
  for (int w = 0; w < warp; w++) before += wsum[w];
  u32 r = before + incl - own;
  for (int h = 0; h < 2; h++) {
    u32 w = h ? w1 : w0;
    while (w) {
      const int b = __ffs(w) - 1;
      w &= w - 1;
      const u32 id = (u32)(64 * t + 32 * h + b);
      if (r == 0) ms.ctl[CM_UMIN] = id;
      ms.ulist[r++] = id;
    }
  }
  if (t == 1023) ms.ctl[CM_NU] = before + incl;
}

__device__ __forceinline__ bool cm_zeroed(const u32* __restrict__ ctl, int k, u32 id) {
  for (int j = 0; j < k; j++)
    if ((ctl[CM_CTL + (1 + j) * CM_WORDS + (id >> 5)] >> (id & 31)) & 1u) return true;
  return false;
}

// class_max round k (pointcloud_class_max.py:115-118), per occupied cell: the maximum over U of the cell's sums, an id
// absent here or won in an earlier round counting 0; ties to the smallest id, a NaN is the maximum.  Writes the maximum
// to the channel's layer (normalised by k_sem_apply) and the id to id_max[k], and marks the id as won.  Cells without
// records are left to k_sem_apply: every id is 0 there, so U's smallest id wins, and it is marked won here when such a
// cell exists.  The last round empties the cell's table slots for the next frame.
__global__ void __launch_bounds__(256)
k_cm_round(const int C, const int k, const bool last, const SemMax ms, float* __restrict__ out, int* __restrict__ id_out) {
  const u32* ctl = ms.ctl;
  u32* wins = ms.ctl + CM_CTL + (1 + k) * CM_WORDS;
  const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0 && ctl[CM_OCC] < (u32)C) {
    const u32 u = ctl[CM_UMIN];
    atomicOr(wins + (u >> 5), 1u << (u & 31));
  }
  if (t >= ctl[CM_OCC]) return;
  const u32 cell = ms.occ[t];
  const u32 m = ms.cnt[cell], base = ms.off[cell];
  bool have = false;
  float bv = 0.f;
  u32 bid = 0;
  for (u32 s = 0; s < m; s++) {
    const u32 key = ms.key[base + s];
    if (!key) continue;
    const u32 id = key - 1;
    if (cm_zeroed(ctl, k, id)) continue;
    const float v = cm_value(ms.flag[base + s], ms.sum[base + s]);
    bool take;
    if (!have) take = true;
    else if (bv != bv) take = (v != v) && id < bid;
    else if (v != v) take = true;
    else take = v > bv || (v == bv && id < bid);
    if (take) { have = true; bv = v; bid = id; }
  }
  if (!have || (bv == bv && bv <= 0.f)) {
    // the smallest id of U that counts 0 here: absent from the cell's table, or won in an earlier round
    const u32 nu = ctl[CM_NU];
    for (u32 r = 0; r < nu; r++) {
      const u32 u = ms.ulist[r];
      bool present = false;
      u32 s = cm_hash(u, m);
      for (u32 probe = 0; probe < m; probe++) {
        const u32 key = ms.key[base + s];
        if (key == 0) break;
        if (key == u + 1) { present = true; break; }
        if (++s == m) s = 0;
      }
      if (present && !cm_zeroed(ctl, k, u)) continue;
      if (!have || bv < 0.f || u < bid) { bv = 0.f; bid = u; }
      have = true;
      break;
    }
  }
  out[cell] = bv;
  id_out[cell] = (int)bid;
  u32* w = wins + (bid >> 5);
  const u32 b = 1u << (bid & 31);
  if (!(*(volatile u32*)w & b)) atomicOr(w, b);
  if (last)
    for (u32 s = 0; s < m; s++) { ms.key[base + s] = 0; ms.flag[base + s] = 0; ms.sum[base + s] = 0; }
}

// per cell: pointcloud_average.py:71-79 (average_kernel), pointcloud_class_average.py (class_average_kernel),
// pointcloud_color.py:97-116 (color_average_kernel), pointcloud_bayesian_inference.py (bayesian_inference_kernel), and
// the normalisation of class_bayesian / class_max (`semantic_map[layers] = new_map[layers] / sum`, every cell); re-zeroes
// the scratch it consumed.
__global__ void __launch_bounds__(256)
k_sem_apply(const DevCfg c, const SemCfg sc, const u64* __restrict__ cnt_fo, i64* __restrict__ fsum, u32* __restrict__ csum,
            float* __restrict__ semantic_map, const SemMax ms) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.C) return;
  const size_t C = (size_t)c.C;
  const float cnt = (float)(u32)cnt_fo[i];                        // new_elmap[get_map_idx(id, 2)]: the frame's fused count
  // the normalisers, summed in ascending channel order; a zero sum divides by 1
  const bool cm_rec = sc.n_max > 0 && ms.cnt[i] > 0;              // class_max: the rounds wrote this cell's maxima
  float tot_cb = 0.f, tot_cm = 0.f;
  for (int k = 0; k < sc.n_ch; k++) {
    if (sc.kind[k] == SEM_CLASS_BAYESIAN) tot_cb = __fadd_rn(tot_cb, (float)unfix32(fsum[(size_t)sc.slot[k] * C + i]));
    else if (sc.kind[k] == SEM_CLASS_MAX && cm_rec) tot_cm = __fadd_rn(tot_cm, semantic_map[(size_t)sc.layer[k] * C + i]);
  }
  if (tot_cb == 0.f) tot_cb = 1.f;
  if (tot_cm == 0.f) tot_cm = 1.f;
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
    if (sc.kind[k] == SEM_CLASS_MAX) {
      // a cell without records: every id is 0, U's smallest id wins every round
      if (!cm_rec) sc.id_max[(size_t)sc.slot[k] * C + i] = (int)ms.ctl[CM_UMIN];
      *out = cm_rec ? __fdiv_rn(*out, tot_cm) : 0.f;
      continue;
    }
    i64* sp = fsum + (size_t)sc.slot[k] * C + i;
    const i64 sfix = *sp;
    if (sfix != 0) *sp = 0;
    const float sum = (float)unfix32(sfix);                       // newmap[...] as the float the reference holds
    if (sc.kind[k] == SEM_CLASS_BAYESIAN) {
      *out = __fdiv_rn(sum, tot_cb);
      continue;
    }
    if (!(cnt > 0.f)) continue;
    if (sc.kind[k] == SEM_AVERAGE) {
      *out = __fdiv_rn(sum, __fmul_rn(1.0f, cnt));                // newmap / (1*cnt)
    } else if (sc.kind[k] == SEM_BAYESIAN_INFERENCE) {
      // bayesian_inference_kernel as nvcc compiles it for sm_90a (its SASS: no contraction, sigma * x folded to x)
      float* sp2 = sc.sigma + (size_t)sc.layer[k] * C + i;
      const float feat_ml = __fdiv_rn(sum, cnt);
      const float feat_old = *out, sigma_old = *sp2;
      const float cs = __fmul_rn(cnt, sigma_old);
      const float d = __fadd_rn(cs, 1.0f);
      *out = __fadd_rn(__fdiv_rn(feat_old, d), __fdiv_rn(__fmul_rn(cs, feat_ml), d));
      *sp2 = __fdiv_rn(sigma_old, d);
    } else {
      const float prev = *out;
      if (prev == 0.f) *out = __fdiv_rn(sum, __fmul_rn(1.0f, cnt));
      else *out = (float)(sc.alpha * (double)prev + (1.0 - sc.alpha) * (double)sum / (double)cnt);   // literal alpha: double
    }
  }
  if (cm_rec) ms.cnt[i] = 0;
}
