// emap_planes.cuh -- plane segmentation of one map window (emap_segment_planes), sm_90a.
//
// Reference: plane_segmentation's convex_plane_decomposition node up to its segmented planes map: grid_map_filters_rsl's
// inpainting::minValues and smoothing::median (GridMapPreprocessing), then SlidingWindowPlaneExtractor without RANSAC.
// include/emap.h states the contract; DESIGN.md §4l the parallel restatement of each step.  The window itself is cut
// by k_submap (emap_submap.cuh).  The fit and the eigen solver are __host__ __device__ so that a native test can run
// them on the CPU.
#pragma once
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#if !defined(__CUDACC__)
using std::fabs;
using std::floor;
using std::isfinite;
using std::rint;
using std::sqrt;
#endif

#define PL_THREADS 256
#define PL_SCAN 1024               // elements per scan block (one thread each)
#define PL_RUN 64                  // cells per thread of k_pl_stats
#define PL_STAT 16                 // u64 words per label: n, Σr, Σc, Σrr, Σcc, Σrc, 4 x int128 (Σh, Σhh, Σrh, Σch)
#define PL_EIG_MIN 1e-8            // the middle eigenvalue below which a normal is not defined

#if defined(__CUDACC__)
#define PL_HD __host__ __device__ __forceinline__
#else
#define PL_HD inline
#endif

// cv::getStructuringElement(MORPH_ELLIPSE, (2 r + 1)^2): row i covers columns r - w .. r + w, w = the half width.  The
// region erosions (emap_regions.cuh) and the post-processing's grey morphology (emap_postprocess.cuh) share it.  r = 0
// is OpenCV's 1 x 1 element (it switches to MORPH_RECT there; the formula would divide by 0).
PL_HD int rg_ellipse_half(int r, int i) {
  if (r == 0) return 0;
  const int dy = i - r;
  const double inv_r2 = 1.0 / ((double)r * r);
  return (int)rint(r * sqrt((double)(r * r - dy * dy) * inv_r2));
}

// A fit's result: the unit normal (z >= 0) and the squared error (the smallest eigenvalue, clamped at 0), or
// (UnitZ, 1e30) when it is not defined.
struct PlaneFit {
  double n[3];
  double err;
};

// Eigen-decomposition of the symmetric 3 x 3 matrix A (row-major, 9 entries) by cyclic Jacobi rotations in double:
// w ascending, column k of V (V[3 r + k]) the unit eigenvector of w[k].
PL_HD void pl_eigen3(const double A[9], double w[3], double V[9]) {
  double a[3][3], v[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) { a[i][j] = A[3 * i + j]; v[i][j] = i == j ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 64; sweep++) {
    if (a[0][1] == 0.0 && a[0][2] == 0.0 && a[1][2] == 0.0) break;
    for (int pq = 0; pq < 3; pq++) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double apq = a[p][q];
      if (apq == 0.0) continue;
      const double g = 100.0 * fabs(apq);
      if (sweep > 3 && fabs(a[p][p]) + g == fabs(a[p][p]) && fabs(a[q][q]) + g == fabs(a[q][q])) {
        a[p][q] = a[q][p] = 0.0;
        continue;
      }
      const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
      double t = fabs(theta) > 1e150 ? 0.5 / theta : 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
      if (theta < 0.0 && fabs(theta) <= 1e150) t = -t;
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      a[p][p] -= t * apq;
      a[q][q] += t * apq;
      a[p][q] = a[q][p] = 0.0;
      const int r = 3 - p - q;
      const double arp = a[r][p], arq = a[r][q];
      a[r][p] = a[p][r] = c * arp - s * arq;
      a[r][q] = a[q][r] = s * arp + c * arq;
      for (int k = 0; k < 3; k++) {
        const double vkp = v[k][p], vkq = v[k][q];
        v[k][p] = c * vkp - s * vkq;
        v[k][q] = s * vkp + c * vkq;
      }
    }
  }
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 3; i++)
    for (int j = i + 1; j < 3; j++)
      if (a[o[j]][o[j]] < a[o[i]][o[i]]) { const int x = o[i]; o[i] = o[j]; o[j] = x; }
  for (int k = 0; k < 3; k++) {
    w[k] = a[o[k]][o[k]];
    for (int r = 0; r < 3; r++) V[3 * r + k] = v[r][o[k]];
  }
}

// normalAndErrorFromCovariance: cov = S / n - mean mean^T (S: the six sums of products xx, xy, xz, yy, yz, zz), its
// smallest eigenvalue's eigenvector flipped to z >= 0 and that eigenvalue clamped at 0, or (UnitZ, 1e30) when the
// middle eigenvalue is <= PL_EIG_MIN.
PL_HD PlaneFit pl_fit_cov(const double cov[9]) {
  double w[3], V[9];
  pl_eigen3(cov, w, V);
  PlaneFit f;
  if (!(w[1] > PL_EIG_MIN)) {
    f.n[0] = f.n[1] = 0.0; f.n[2] = 1.0; f.err = 1e30;
    return f;
  }
  const double sg = V[6] < 0.0 ? -1.0 : 1.0;
  for (int r = 0; r < 3; r++) f.n[r] = sg * V[3 * r];
  f.err = w[0] > 0.0 ? w[0] : 0.0;
  return f;
}

PL_HD PlaneFit pl_fit_sums(double n, const double sum[3], const double S[6]) {
  const double m[3] = {sum[0] / n, sum[1] / n, sum[2] / n};
  const double cov[9] = {S[0] / n - m[0] * m[0], S[1] / n - m[0] * m[1], S[2] / n - m[0] * m[2],
                         S[1] / n - m[1] * m[0], S[3] / n - m[1] * m[1], S[4] / n - m[1] * m[2],
                         S[2] / n - m[2] * m[0], S[4] / n - m[2] * m[1], S[5] / n - m[2] * m[2]};
  return pl_fit_cov(cov);
}

// computeNormalAndErrorForWindow at cell (r, c) of a rows x cols image: the k x k window centred there, cells outside
// the image and non-finite heights skipped, points (-kr * res, -kc * res, h) for window row kr, column kc (0 .. k-1),
// visited column by column and accumulated in double; fewer than 3 points: (UnitZ, 1e30).
PL_HD PlaneFit pl_window_fit(const float* img, int rows, int cols, int r, int c, int k, double res) {
  const int half = (k - 1) / 2;
  int n = 0;
  double sum[3] = {0.0, 0.0, 0.0}, S[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int kc = 0; kc < k; kc++) {
    const int cc = c - half + kc;
    if (cc < 0 || cc >= cols) continue;
    for (int kr = 0; kr < k; kr++) {
      const int rr = r - half + kr;
      if (rr < 0 || rr >= rows) continue;
      const float h = img[(long long)rr * cols + cc];
      if (!isfinite(h)) continue;
      const double p[3] = {-kr * res, -kc * res, (double)h};
      n++;
      for (int a = 0; a < 3; a++) sum[a] += p[a];
      S[0] += p[0] * p[0]; S[1] += p[0] * p[1]; S[2] += p[0] * p[2];
      S[3] += p[1] * p[1]; S[4] += p[1] * p[2]; S[5] += p[2] * p[2];
    }
  }
  if (n < 3) {
    PlaneFit f;
    f.n[0] = f.n[1] = 0.0; f.n[2] = 1.0; f.err = 1e30;
    return f;
  }
  return pl_fit_sums((double)n, sum, S);
}

// ---- per-label statistics in exact integer arithmetic ---------------------------------------------------------------
// A label's sums are order independent, so they are deterministic however the cells are visited: the row and column
// sums are integers, and each h-term (h, h^2, r h, c h: exact in double) is added as a signed 128-bit fixed-point value
// with 64 fractional bits (its bits below 2^-64 are truncated).  Stored as (lo, hi) u64 pairs.
struct PlI128 {
  unsigned long long lo;
  long long hi;
};

PL_HD PlI128 pl_i128(double v) {
  const double a = fabs(v), ip = floor(a);
  PlI128 x;
  x.hi = (long long)ip;
  x.lo = (unsigned long long)((a - ip) * 18446744073709551616.0);
  if (v < 0.0) {
    x.lo = ~x.lo + 1ull;
    x.hi = ~x.hi + (x.lo == 0ull ? 1 : 0);
  }
  return x;
}

PL_HD void pl_i128_add(PlI128& s, PlI128 v) {
  const unsigned long long lo = s.lo + v.lo;
  s.hi += v.hi + (lo < s.lo ? 1 : 0);
  s.lo = lo;
}

PL_HD double pl_i128_value(unsigned long long lo, unsigned long long hi) {
  return (double)(long long)hi + (double)lo * 5.421010862427522170e-20;   // 2^-64
}

// A label's plane from its statistics st[PL_STAT]: support = the mean of (origin_x - r res, origin_y - c res, h), the
// normal of pl_fit_sums on S / n - mean mean^T (computed here from the centred integer moments).  Returns false when the
// label has fewer than max(min_points, 3) points.
PL_HD bool pl_label_plane(const unsigned long long* st, double ox, double oy, double res, int min_points,
                          double support[3], PlaneFit& f) {
  const double n = (double)st[0];
  if (st[0] < 3ull || (min_points > 0 && st[0] < (unsigned long long)min_points)) return false;
  const double mr = (double)st[1] / n, mc = (double)st[2] / n;
  const double sh = pl_i128_value(st[6], st[7]), shh = pl_i128_value(st[8], st[9]);
  const double srh = pl_i128_value(st[10], st[11]), sch = pl_i128_value(st[12], st[13]);
  const double mh = sh / n;
  support[0] = ox - res * mr;
  support[1] = oy - res * mc;
  support[2] = mh;
  const double vrr = (double)st[3] / n - mr * mr, vcc = (double)st[4] / n - mc * mc, vrc = (double)st[5] / n - mr * mc;
  const double vrh = srh / n - mr * mh, vch = sch / n - mc * mh, vhh = shh / n - mh * mh;
  // x = ox - res r, y = oy - res c: cov(x, h) = -res cov(r, h), cov(x, y) = res^2 cov(r, c)
  const double r2 = res * res;
  const double cov[9] = {r2 * vrr, r2 * vrc, -res * vrh, r2 * vrc, r2 * vcc, -res * vch, -res * vrh, -res * vch, vhh};
  f = pl_fit_cov(cov);
  return true;
}

#if defined(__CUDACC__)
// ---- device passes --------------------------------------------------------------------------------------------------
// Header words of the scratch (hdr): [0] the window has a finite cell, [1] highest_label, [2] n_planes.

// Union-find over cells whose parent is >= 0 (the mask): roots carry their component's minimum linear index.
__device__ __forceinline__ int pl_find(const int* parent, int a) {
  int p = ((volatile const int*)parent)[a];
  while (p != a) { a = p; p = ((volatile const int*)parent)[a]; }
  return a;
}

__device__ __forceinline__ void pl_union(int* parent, int a, int b) {
  for (;;) {
    a = pl_find(parent, a); b = pl_find(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&parent[a], b);
    if (old == a) return;
    a = old;
  }
}

// Fill's mask: the NaN cells; also flags whether any cell is finite.
__global__ void k_pl_fill_init(const float* __restrict__ raw, int* __restrict__ parent, unsigned* __restrict__ key,
                               int* __restrict__ hdr, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float h = raw[i];
  parent[i] = isnan(h) ? i : -1;
  key[i] = 0xffffffffu;
  if (isfinite(h)) hdr[0] = 1;
}

// Planar cells' mask; clears the first-block keys and the block flags.
__global__ void k_pl_cc_init(const unsigned char* __restrict__ bin, int* __restrict__ parent, unsigned* __restrict__ key,
                             int* __restrict__ flag, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  parent[i] = bin[i] ? i : -1;
  key[i] = 0xffffffffu;
  flag[i] = 0;
}

// Merges every masked cell with its masked neighbours above and to the left (and, with 8-connectivity, above-left and
// above-right).
__global__ void k_pl_uf_merge(int* parent, int rows, int cols, int conn8) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || parent[i] < 0) return;
  const int r = i / cols, c = i - r * cols;
  if (c > 0 && parent[i - 1] >= 0) pl_union(parent, i, i - 1);
  if (r > 0) {
    if (parent[i - cols] >= 0) pl_union(parent, i, i - cols);
    if (conn8) {
      if (c > 0 && parent[i - cols - 1] >= 0) pl_union(parent, i, i - cols - 1);
      if (c + 1 < cols && parent[i - cols + 1] >= 0) pl_union(parent, i, i - cols + 1);
    }
  }
}

// Points every masked cell at its root.
__global__ void k_pl_uf_flatten(int* parent, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && parent[i] >= 0) parent[i] = pl_find(parent, i);
}

// cv::connectedComponents numbers components in the order its scan meets them: by first cell in raster order with
// 4-connectivity (SAUF), by first 2 x 2 block in raster order of the blocks with 8-connectivity (Spaghetti; the cells
// of one block are 8-connected, so no two components share a first block).  key[root] = the component's first block
// (B = 1 or 2), then flag[block] = 1 for every first block.
template <int B>
__global__ void k_pl_first(const int* __restrict__ parent, unsigned* key, int rows, int cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || parent[i] < 0) return;
  const int r = i / cols, c = i - r * cols;
  atomicMin(&key[parent[i]], (unsigned)((r / B) * ((cols + B - 1) / B) + c / B));
}

__global__ void k_pl_first_flag(const int* __restrict__ parent, const unsigned* __restrict__ key, int* __restrict__ flag,
                                int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && parent[i] == i) flag[key[i]] = 1;
}

// minValues' fixed point: each NaN component's minimum over the non-NaN 4-neighbours of its cells, one atomicMin of an
// order-preserving key per (non-NaN cell, NaN neighbour).
__global__ void k_pl_fill_min(const float* __restrict__ raw, const int* __restrict__ parent, unsigned* key, int rows,
                              int cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols || parent[i] >= 0) return;
  const int r = i / cols, c = i - r * cols;
  const unsigned k = tsub_fkey(raw[i]);
  if (c > 0 && parent[i - 1] >= 0) atomicMin(&key[parent[i - 1]], k);
  if (c + 1 < cols && parent[i + 1] >= 0) atomicMin(&key[parent[i + 1]], k);
  if (r > 0 && parent[i - cols] >= 0) atomicMin(&key[parent[i - cols]], k);
  if (r + 1 < rows && parent[i + cols] >= 0) atomicMin(&key[parent[i + cols]], k);
}

__global__ void k_pl_fill_write(const float* __restrict__ raw, const int* __restrict__ parent,
                                const unsigned* __restrict__ key, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = parent[i] >= 0 ? tsub_funkey(key[parent[i]]) : raw[i];
}

// cv::medianBlur on CV_32F: the exact median of the K x K values around each cell, border replicated.  With KEEP_NAN a
// NaN cell stays NaN, as in cv2 (emap_grid_filter); the fminf / fmaxf network itself passes over NaN operands.
template <int K, bool KEEP_NAN = false>
__global__ void k_pl_median(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  float v[K * K];
#pragma unroll
  for (int dr = 0; dr < K; dr++)
#pragma unroll
    for (int dc = 0; dc < K; dc++) {
      const int rr = min(max(r + dr - K / 2, 0), rows - 1), cc = min(max(c + dc - K / 2, 0), cols - 1);
      v[dr * K + dc] = src[rr * cols + cc];
    }
#pragma unroll
  for (int a = 1; a < K * K; a++)
#pragma unroll
    for (int b = a; b > 0; b--) {
      const float x = v[b - 1], y = v[b];
      v[b - 1] = fminf(x, y);
      v[b] = fmaxf(x, y);
    }
  dst[i] = KEEP_NAN && isnan(src[i]) ? src[i] : v[K * K / 2];
}

// runSlidingWindowDetector: planar iff the centre is finite, error < thr2 and n.z > cos_local.
__global__ void k_pl_fit(const float* __restrict__ img, unsigned char* __restrict__ bin, int rows, int cols, int k,
                         double res, double thr2, double cos_local) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  unsigned char p = 0;
  if (isfinite(img[i])) {
    const PlaneFit f = pl_window_fit(img, rows, cols, r, c, k, res);
    p = f.err < thr2 && f.n[2] > cos_local;
  }
  bin[i] = p;
}

// One half of MORPH_OPEN with a (2 rad + 1) cross, border replicated: erosion (MAX false) or dilation (MAX true).
template <bool MAX>
__global__ void k_pl_morph(const unsigned char* __restrict__ src, unsigned char* __restrict__ dst, int rows, int cols,
                           int rad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  int v = src[i];
  for (int d = 1; d <= rad; d++) {
    const int a = src[min(r + d, rows - 1) * cols + c], b = src[max(r - d, 0) * cols + c];
    const int e = src[r * cols + min(c + d, cols - 1)], g = src[r * cols + max(c - d, 0)];
    v = MAX ? max(max(v, a), max(max(b, e), g)) : min(min(v, a), min(min(b, e), g));
  }
  dst[i] = (unsigned char)v;
}

// Exclusive block scan of one int per thread (blockDim.x == PL_SCAN); returns the prefix, `total` the block's sum.
__device__ __forceinline__ int pl_block_scan(int v, int& total) {
  __shared__ int warp_sum[PL_SCAN / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = warp_sum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_sum[lane] = s;
  }
  __syncthreads();
  total = warp_sum[PL_SCAN / 32 - 1];
  const int r = x - v + (wid ? warp_sum[wid - 1] : 0);
  __syncthreads();
  return r;
}

// Raster-order ranks of the flagged elements in three launches: block sums, the scan of the block sums (one CTA, which
// also stores the total), and the ranks (rank[i] = number of flagged elements before i; unflagged: -1).
__global__ void __launch_bounds__(PL_SCAN) k_pl_scan_blocks(const int* __restrict__ flag, int n, int* __restrict__ bsum) {
  const int i = blockIdx.x * PL_SCAN + threadIdx.x;
  int total;
  pl_block_scan(i < n ? flag[i] : 0, total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(PL_SCAN) k_pl_scan_top(int* bsum, int nb, int* __restrict__ total_out) {
  const int per = (nb + PL_SCAN - 1) / PL_SCAN, b0 = threadIdx.x * per;
  int s = 0;
  for (int b = b0; b < min(b0 + per, nb); b++) s += bsum[b];
  int total;
  int run = pl_block_scan(s, total);
  for (int b = b0; b < min(b0 + per, nb); b++) {
    const int x = bsum[b];
    bsum[b] = run;
    run += x;
  }
  if (threadIdx.x == 0) *total_out = total;
}

__global__ void __launch_bounds__(PL_SCAN) k_pl_scan_rank(const int* __restrict__ flag, int n,
                                                          const int* __restrict__ bsum, int* __restrict__ rank) {
  const int i = blockIdx.x * PL_SCAN + threadIdx.x;
  const int f = i < n ? flag[i] : 0;
  int total;
  const int p = pl_block_scan(f, total);
  if (i < n) rank[i] = f ? bsum[blockIdx.x] + p : -1;
}

// cv::connectedComponents' labels: 1 + the rank of the component's first block, 0 for background.
__global__ void k_pl_label(const int* __restrict__ parent, const unsigned* __restrict__ key, const int* __restrict__ rank,
                           int* __restrict__ lab, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) lab[i] = parent[i] >= 0 ? rank[key[parent[i]]] + 1 : 0;
}

__device__ __forceinline__ void pl_flush(unsigned long long* st, const unsigned long long u[6], const PlI128 x[4]) {
  for (int k = 0; k < 6; k++) atomicAdd(&st[k], u[k]);
  for (int k = 0; k < 4; k++) {
    unsigned long long* w = st + 6 + 2 * k;
    const unsigned long long old = atomicAdd(&w[0], x[k].lo);
    atomicAdd(&w[1], (unsigned long long)x[k].hi + (old + x[k].lo < old ? 1ull : 0ull));
  }
}

// Per-label statistics of the finite cells: each thread sums PL_RUN consecutive cells in registers and adds each run
// of one label to the label's words with integer atomics.
__global__ void k_pl_stats(const float* __restrict__ img, const int* __restrict__ lab, unsigned long long* st, int rows,
                           int cols) {
  const long long n = (long long)rows * cols;
  const long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * PL_RUN;
  if (i0 >= n) return;
  const long long i1 = min(i0 + PL_RUN, n);
  int cur = 0;
  unsigned long long u[6] = {0, 0, 0, 0, 0, 0};
  PlI128 x[4] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}};
  for (long long i = i0; i < i1; i++) {
    const int l = lab[i];
    const float h = img[i];
    if (l <= 0 || !isfinite(h)) continue;
    if (l != cur) {
      if (cur) pl_flush(st + (long long)cur * PL_STAT, u, x);
      cur = l;
      for (int k = 0; k < 6; k++) u[k] = 0;
      for (int k = 0; k < 4; k++) x[k] = PlI128{0, 0};
    }
    const unsigned long long r = (unsigned long long)(i / cols), c = (unsigned long long)(i % cols);
    const double hd = (double)h;
    u[0] += 1; u[1] += r; u[2] += c; u[3] += r * r; u[4] += c * c; u[5] += r * c;
    pl_i128_add(x[0], pl_i128(hd));
    pl_i128_add(x[1], pl_i128(hd * hd));
    pl_i128_add(x[2], pl_i128((double)r * hd));
    pl_i128_add(x[3], pl_i128((double)c * hd));
  }
  if (cur) pl_flush(st + (long long)cur * PL_STAT, u, x);
}

// extractPlaneParametersFromLabeledImage's decisions per label L (1 .. highest_label): keep[L] = 1 for a plane,
// bg[L] = 1 for a label set to background; labels with too few points keep their label and get no plane.
struct PlaneLabelArgs {
  double ox, oy, res, cos_plane;
  int min_points;
};

__global__ void k_pl_decide(const unsigned long long* __restrict__ st, const int* __restrict__ hdr,
                            int* __restrict__ keep, unsigned char* __restrict__ bg, int slots, PlaneLabelArgs a) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= slots) return;
  int k = 0;
  unsigned char b = 0;
  double support[3];
  PlaneFit f;
  if (l >= 1 && l <= hdr[1] && pl_label_plane(st + (long long)l * PL_STAT, a.ox, a.oy, a.res, a.min_points, support, f)) {
    k = f.n[2] > a.cos_plane;
    b = !k;
  }
  keep[l] = k;
  bg[l] = b;
}

// The plane table, labels ascending: row rank[L] = (L, support, normal).
__global__ void k_pl_planes(const unsigned long long* __restrict__ st, const int* __restrict__ rank,
                            const int* __restrict__ hdr, double* __restrict__ planes, int slots, PlaneLabelArgs a) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= slots || !hdr[0] || rank[l] < 0) return;
  double support[3];
  PlaneFit f;
  pl_label_plane(st + (long long)l * PL_STAT, a.ox, a.oy, a.res, a.min_points, support, f);
  double* row = planes + 7ll * rank[l];
  row[0] = l;
  for (int k = 0; k < 3; k++) { row[1 + k] = support[k]; row[4 + k] = f.n[k]; }
}

// The four output layers and info {success, rows, cols, highest_label, n_planes}; nothing but info when the window has
// no finite cell.  raw == nullptr leaves layer 0 unwritten (a caller's grid is its own elevation_raw).
__global__ void k_pl_out(const float* __restrict__ raw, const float* __restrict__ img, const int* __restrict__ lab,
                         const unsigned char* __restrict__ bg, const int* __restrict__ hdr, float* __restrict__ out,
                         int32_t* __restrict__ info, int rows, int cols) {
  const int n = rows * cols;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int ok = hdr[0];
  if (i == 0) {
    info[0] = ok; info[1] = rows; info[2] = cols;
    info[3] = ok ? hdr[1] : 0; info[4] = ok ? hdr[2] : 0;
  }
  if (i >= n || !ok) return;
  int l = lab[i];
  if (l > 0 && bg[l]) l = 0;
  if (raw) out[i] = raw[i];
  out[n + i] = img[i];
  out[2 * n + i] = (float)l;
  out[3 * n + i] = l > 0 ? 1.f : 0.f;
}
#endif
