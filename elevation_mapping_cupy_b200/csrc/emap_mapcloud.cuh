// emap_mapcloud.cuh -- the exported map as a point cloud and as normal arrows (emap_get_map_points,
// emap_get_normal_arrows), sm_90a.
//
// Reference: the ROS node's map timer (elevation_mapping_ros.cpp:687-702) turns grid_map's copy of the exported layers
// (WRAP:213-252) into a point cloud (publishAsPointCloud, :501-505, GridMapRosConverter::toPointCloud) and into normal
// arrows (publishNormalAsArrow, :751-778), with host loops over every cell.  Both are one ordered stream compaction of
// the exported map in grid_map's storage order, which is column-major: output rank c * (W-2) + r for exported cell
// (r, c).  The state is row-major, so a thread per output position would read down state columns.  Instead:
//   k_mapcloud<.., false>  one CTA per 32 x 32 tile of the exported map (an exported row chunk k of 32 rows by 32
//                          columns): warps stage tile rows with coalesced loads through export_cell into shared
//                          memory, then each warp walks tile columns (lane = row) and writes the kept-cell count of
//                          every (exported column c, row chunk k) to cnt[c * n_chunks + k];
//   k_mapcloud_scan        the exclusive prefix of cnt in that (column-major) order, and the total;
//   k_mapcloud<.., true>   the same tiles again: a kept cell's row is its column chunk's offset plus its rank among the
//                          chunk's kept lanes (a ballot), so each warp writes consecutive rows.
// Nothing is ordered by atomics: the output is the same on every run.  Scratch: the count and offset tables
// (2 (W-2) n_chunks + 1 ints) and the payload of the kept cells only.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "emap_export.cuh"

#define MC_TILE 32                 // exported rows of a chunk = exported columns of a tile (one warp's lanes)
#define MC_THREADS 256             // 8 warps: each stages 4 tile rows, then walks 4 tile columns

// Geometry of the exported map (get_grid_map's setGeometry, WRAP:223-228, with grid_map's getPositionFromIndex and
// buffer start (0, 0)): exported cell (r, c) lies at x = (cx + (0.5 * L - 0.5 * res)) - res * r,
// y = (cy + (0.5 * L - 0.5 * res)) - res * c, in double, L = (W - 2) * res, (cx, cy) the fp32 centre widened.  The device
// evaluates it with explicit roundings (mc_position), so no compiler contracts it into a fused multiply-add.
struct MapCloudGeom {
  double cx, cy, res;
};

__device__ __forceinline__ double mc_position(double centre, double res, int Wo, int index) {
  const double L = __dmul_rn((double)Wo, res);
  const double first = __dadd_rn(centre, __dsub_rn(__dmul_rn(0.5, L), __dmul_rn(0.5, res)));
  return __dsub_rn(first, __dmul_rn(res, (double)index));
}

// Payload of k_mapcloud<.., true>.  Points: xyz[3 * row ..] = float (x, y, z).  Arrows: ids[row] = c * (W-2) + r,
// seg[6 * row ..] = double (start, end).
struct MapCloudOut {
  float* xyz;
  int32_t* ids;
  double* seg;
};

// publishNormalAsArrow skips a cell when Eigen's normal.norm() < 0.1, norm = sqrt((nx^2 + ny^2) + nz^2) in double.  The
// test is written as the reference's skip test, so a normal that is not a number keeps its arrow as it does there
// (the frame never writes one).
__device__ __forceinline__ bool mc_arrow_kept(float nx, float ny, float nz) {
  const double x = nx, y = ny, z = nz;
  const double n2 = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
  return !(__dsqrt_rn(n2) < 0.1);
}

// One kept cell's output row `row` (exported cell (r, col), elevation e, normal n).
template <bool ARROWS>
__device__ __forceinline__ void mc_write(const MapCloudGeom& g, const MapCloudOut& o, float e, float nx, float ny,
                                         float nz, int row, int r, int col, int Wo) {
  const double x = mc_position(g.cx, g.res, Wo, r), y = mc_position(g.cy, g.res, Wo, col);
  if (!ARROWS) {
    float* p = o.xyz + 3 * (size_t)row;
    p[0] = __double2float_rn(x); p[1] = __double2float_rn(y); p[2] = e;
  } else {
    const double z = e;
    double* q = o.seg + 6 * (size_t)row;
    q[0] = x; q[1] = y; q[2] = z;
    q[3] = __dadd_rn(x, __dmul_rn((double)nx, 0.1));                      // start + normal * 0.1
    q[4] = __dadd_rn(y, __dmul_rn((double)ny, 0.1));
    q[5] = __dadd_rn(z, __dmul_rn((double)nz, 0.1));
    o.ids[row] = col * Wo + r;
  }
}

template <bool ARROWS, bool WRITE>
__global__ void __launch_bounds__(MC_THREADS)
k_mapcloud(const DevCfg c, const float* __restrict__ map, const float* __restrict__ normal, float center_z,
           int* __restrict__ cnt, const int* __restrict__ off, const MapCloudGeom g, const MapCloudOut o) {
  constexpr int NP = ARROWS ? 4 : 1;                 // staged planes: elevation (+ normal x, y, z)
  __shared__ float s[NP][MC_TILE][MC_TILE + 1];
  const int Wo = c.W - 2, n_chunks = gridDim.y;
  const int c0 = blockIdx.x * MC_TILE, k = blockIdx.y, r0 = k * MC_TILE;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float nanv = __int_as_float(0x7fc00000);
  // stage: warp w loads tile rows w, w + 8, ...; lane l reads exported column c0 + l = state column Wo - c0 - l, so a
  // warp's 32 addresses are one 128-byte span (run backwards)
  const int oc = c0 + lane;
#pragma unroll
  for (int j = 0; j < MC_TILE / 8; j++) {
    const int rl = warp + 8 * j, orow = r0 + rl;
    float v[NP];
#pragma unroll
    for (int p = 0; p < NP; p++) v[p] = nanv;
    if (orow < Wo && oc < Wo) {
      const int sr = Wo - orow, sc = Wo - oc;        // flip(0), flip(1) of m[1:-1, 1:-1]
#pragma unroll
      for (int p = 0; p < NP; p++) v[p] = export_cell(c, map, normal, sr, sc, p ? 5 + p : 0, center_z, 0, nullptr, 0);
    }
#pragma unroll
    for (int p = 0; p < NP; p++) s[p][rl][lane] = v[p];
  }
  __syncthreads();
  // walk: warp w takes tile columns w, w + 8, ...; lane = tile row, so the kept lanes of a column are consecutive rows
  // of the output (cells outside the map were staged as NaN and are never kept)
#pragma unroll 1
  for (int j = 0; j < MC_TILE / 8; j++) {
    const int cl = warp + 8 * j, col = c0 + cl;
    if (col >= Wo) break;                            // the same for the whole warp
    const float e = s[0][lane][cl];
    const float nx = s[ARROWS ? 1 : 0][lane][cl], ny = s[ARROWS ? 2 : 0][lane][cl], nz = s[ARROWS ? 3 : 0][lane][cl];
    const bool keep = isfinite(e) && (!ARROWS || mc_arrow_kept(nx, ny, nz));
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    const int item = col * n_chunks + k;
    if (!WRITE) {
      if (lane == 0) cnt[item] = __popc(m);
    } else if (keep) {
      mc_write<ARROWS>(g, o, e, nx, ny, nz, off[item] + __popc(m & ((1u << lane) - 1u)), r0 + lane, col, Wo);
    }
  }
}

// Inclusive scan of one value per thread across a CTA of blockDim.x (a multiple of 32, at most 1024) threads; `tot`
// receives the CTA's total.
__device__ __forceinline__ int mc_block_scan(int v, int* warp_sums, int& tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += u;
  }
  if (lane == 31) warp_sums[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int w = lane < n_warps ? warp_sums[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += u;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  tot = warp_sums[31];
  const int r = v + (warp ? warp_sums[warp - 1] : 0);
  __syncthreads();                                   // warp_sums may be reused
  return r;
}

// off[i] = cnt[0] + ... + cnt[i - 1] for the n entries of cnt, off[n] = the total.  One CTA per segment of `seg`
// entries (a tile column's chunks, at most 2 * blockDim.x): it sums every entry before its segment (coalesced, in
// parallel) and scans its own, so no CTA waits for another and the sums are the same on every run.
__global__ void __launch_bounds__(1024)
k_mapcloud_scan(const int* __restrict__ cnt, int* __restrict__ off, int n, int seg) {
  __shared__ int warp_sums[32];
  const int s0 = blockIdx.x * seg, s1 = min(s0 + seg, n);
  int before = 0;
  const int4* cnt4 = reinterpret_cast<const int4*>(cnt);           // seg is a multiple of 4: s0 is 16-byte aligned
#pragma unroll 4
  for (int i = threadIdx.x; i < s0 / 4; i += blockDim.x) {
    const int4 q = cnt4[i];
    before += (q.x + q.y) + (q.z + q.w);
  }
  int tot;
  mc_block_scan(before, warp_sums, tot);
  before = tot;
  const int i0 = s0 + 2 * (int)threadIdx.x;
  const int a = i0 < s1 ? cnt[i0] : 0, b = i0 + 1 < s1 ? cnt[i0 + 1] : 0;
  const int incl = mc_block_scan(a + b, warp_sums, tot);
  const int ex = before + incl - (a + b);
  if (i0 < s1) off[i0] = ex;
  if (i0 + 1 < s1) off[i0 + 1] = ex + a;
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) off[n] = before + tot;
}
