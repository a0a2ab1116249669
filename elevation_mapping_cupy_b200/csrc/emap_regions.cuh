// emap_regions.cuh -- planar region extraction of one segmented window (emap_extract_planar_regions), sm_90a.
//
// Reference: plane_segmentation's convex_plane_decomposition ContourExtraction::extractPlanarRegions (upsampling,
// margin erosion, boundaries and insets by cv::findContours(RETR_CCOMP, CHAIN_APPROX_SIMPLE), the cross-erosion
// fallback, the projection to the plane frame) and Postprocessing::addHeightOffset.  include/emap.h states the
// contract; DESIGN.md §4l the parallel restatement.  The upsampling index, the start-pixel rule and the border
// following with CHAIN_APPROX_SIMPLE's compression (and the structuring element, rg_ellipse_half in emap_planes.cuh)
// are __host__ __device__ so that a native test can check them against cv2.
#pragma once
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#include "emap_planes.cuh"

#define RG_MAX_MARGIN 4            // emap.h's EMAP_REGION_MAX_MARGIN: the margin ellipse is at most 11 x 11
#define RG_KMAX (2 * (1 + RG_MAX_MARGIN) + 1)
#define RG_ROW 17                  // doubles per region row: label, 3 x 4 plane-to-world transform, bbox
#define RG_POLY 5                  // int32 per polygon row: region, role, inset, first_vertex, n_vertices
#define RG_BITS 26                 // pixel indices fit in 26 bits (6137^2 < 2^26)
#define RG_LOW ((1ull << RG_BITS) - 1ull)

// Upsampled row (column) u -> source row (column) of a source with m >= 2 rows: the first and last source rows take 2
// upsampled rows each, every inner one 3 (Upsampling.cpp), so the upsampled size is 3 m - 2.
PL_HD int rg_src(int u, int m) {
  const int s = u < 2 ? 0 : (u - 2) / 3 + 1;
  return s < m - 1 ? s : m - 1;
}

// Border-following start of pixel i of a binary image in Suzuki-Abe's scan (8-connected foreground, 4-connected
// background, zero outside): 1 = an outer border (i is the raster-first pixel of its foreground component), 2 = a hole
// border (the pixel right of i is the raster-first pixel of a background component that does not touch the image
// edge), 0 = none.  root_* are component roots, each the component's least index; frame is the root of the background
// that touches the edge (-1: none).
PL_HD int rg_start(int i, bool fg, int root, bool has_right, bool fg_right, int root_right, int frame) {
  if (!fg) return 0;
  if (root == i) return 1;
  return has_right && !fg_right && root_right == i + 1 && root_right != frame ? 2 : 0;
}

// Follows the border that starts at (x0, y0) as cv::findContours does (hole: the start's background is on its right,
// else on its left) and calls emit(x, y) for every point CHAIN_APPROX_SIMPLE keeps: a pixel where the chain's
// direction changes, and a lone pixel once.  nz(x, y) reads the image (0 outside).  Returns the number of points.
// Directions: 0 = +x, then counter-clockwise on the screen (y down): 1 = (+1, -1), 2 = (0, -1), ... 7 = (+1, +1).
template <class NZ, class EMIT>
PL_HD int rg_trace(const NZ& nz, int x0, int y0, bool hole, EMIT& emit) {
  const int DX[8] = {1, 1, 0, -1, -1, -1, 0, 1}, DY[8] = {0, -1, -1, -1, 0, 1, 1, 1};
  const int s0 = hole ? 0 : 4;
  int s = s0, x1, y1;
  do {
    s = (s - 1) & 7;
    x1 = x0 + DX[s];
    y1 = y0 + DY[s];
  } while (!nz(x1, y1) && s != s0);
  if (s == s0) {
    emit(x0, y0);
    return 1;
  }
  int n = 0, x3 = x0, y3 = y0, prev = s ^ 4;
  for (;;) {
    // the 8 neighbours in one go (independent reads), then the first foreground one counter-clockwise after s; the
    // pixel the chain came from (direction s) is foreground, so the search ends
    unsigned nb = 0;
    for (int d = 0; d < 8; d++) nb |= (unsigned)(bool)nz(x3 + DX[d], y3 + DY[d]) << d;
    int k = s;
    do {
      k++;
    } while (!((nb >> (k & 7)) & 1u));
    k &= 7;
    const int x4 = x3 + DX[k], y4 = y3 + DY[k];
    if (k != prev) {
      emit(x3, y3);
      n++;
      prev = k;
    }
    if (x4 == x0 && y4 == y0 && x3 == x1 && y3 == y1) return n;
    x3 = x4;
    y3 = y4;
    s = (k + 4) & 7;
  }
}

// getTransformLocalToGlobal(support, normal) as a 3 x 4 row-major [R | t] (PlanarRegion.cpp).
PL_HD void rg_plane_transform(const double support[3], const double normal[3], double T[12]) {
  const double nn = sqrt(normal[0] * normal[0] + normal[1] * normal[1] + normal[2] * normal[2]);
  const double z[3] = {normal[0] / nn, normal[1] / nn, normal[2] / nn};
  double y[3] = {0.0, z[2], -z[1]};                       // z x UnitX
  const double y2 = y[0] * y[0] + y[1] * y[1] + y[2] * y[2];
  if (y2 > 1e-3) {
    const double q = sqrt(y2);
    for (int k = 0; k < 3; k++) y[k] /= q;
  } else {
    const double u[3] = {z[2], 0.0, -z[0]};               // UnitY x z
    double w[3] = {z[1] * u[2] - z[2] * u[1], z[2] * u[0] - z[0] * u[2], z[0] * u[1] - z[1] * u[0]};
    const double q = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    for (int k = 0; k < 3; k++) y[k] = w[k] / q;
  }
  const double x[3] = {y[1] * z[2] - y[2] * z[1], y[2] * z[0] - y[0] * z[2], y[0] * z[1] - y[1] * z[0]};
  for (int r = 0; r < 3; r++) {
    T[4 * r + 0] = x[r];
    T[4 * r + 1] = y[r];
    T[4 * r + 2] = z[r];
    T[4 * r + 3] = support[r];
  }
}

// projectToPlaneAlongGravity of world (wx, wy) with T from rg_plane_transform.
PL_HD void rg_project(const double T[12], double wx, double wy, double& px, double& py) {
  const double dx = wx - T[3], dy = wy - T[7];
  const double dz = (-dx * T[2] - dy * T[6]) / T[10];
  px = T[0] * dx + T[4] * dy + T[8] * dz;
  py = T[1] * dx + T[5] * dy + T[9] * dz;
}

#if defined(__CUDACC__)
// ---- device passes --------------------------------------------------------------------------------------------------
// The upsampled image (UR x UC = (3R - 2) x (3C - 2) pixels) is never stored as labels: a pixel's plane row is pr[] of
// its source cell.  One mask byte per pixel holds four binary images: bit 0 the margin-eroded planes, bit 1 its
// inset, bit 2 the fallback (cross-eroded) planes of the labels the first pass left empty, bit 3 its inset.  After
// either erosion, pixels of two labels are never 8-adjacent, so all labels share one image per bit.

struct RgKernel {
  int r;                 // radius
  int half[RG_KMAX];     // half width of row i (dy = i - r)
};

struct RgGeom {
  int R, C, UR, UC;      // source and upsampled sizes
};

__device__ __forceinline__ int rg_pr(const int* pr, const RgGeom& g, int y, int x) {
  y = min(max(y, 0), g.UR - 1);
  x = min(max(x, 0), g.UC - 1);
  return pr[rg_src(y, g.R) * g.C + rg_src(x, g.C)];
}

// Plane row of every source cell: rank[] of its label after the plane decisions (-1: background or no plane).
__global__ void k_rg_rows(const int* __restrict__ lab, const int* __restrict__ rank, int* __restrict__ pr, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pr[i] = lab[i] > 0 ? rank[lab[i]] : -1;
}

// Bit 2 ph: (up == label) eroded once by the kernel with BORDER_REPLICATE, for every plane row (pass 0) or for the
// plane rows that pass 0 left without a region (pass 1, ok[row] == 0).
__global__ void k_rg_erode(const int* __restrict__ pr, const int* __restrict__ ok, unsigned char* __restrict__ mask,
                           RgGeom g, RgKernel k, int ph) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.UR * g.UC) return;
  const int y = i / g.UC, x = i - y * g.UC;
  const int L = rg_pr(pr, g, y, x);
  bool v = L >= 0 && (ph == 0 || !ok[L]);
  for (int a = 0; a <= 2 * k.r && v; a++)
    for (int b = -k.half[a]; b <= k.half[a] && v; b++) v = rg_pr(pr, g, y + a - k.r, x + b) == L;
  mask[i] = ph == 0 ? (unsigned char)v : (unsigned char)(mask[i] | (v ? 4 : 0));
}

// Bit 2 ph + 1: the inset, bit 2 ph eroded by the 3 x 3 cross and the image's first and last rows and columns cleared.
__global__ void k_rg_inset(unsigned char* mask, RgGeom g, int ph) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.UR * g.UC) return;
  const int y = i / g.UC, x = i - y * g.UC;
  const int b = 1 << (2 * ph);
  bool v = (mask[i] & b) && y > 0 && x > 0 && y < g.UR - 1 && x < g.UC - 1;
  v = v && (mask[i - 1] & b) && (mask[i + 1] & b) && (mask[i - g.UC] & b) && (mask[i + g.UC] & b);
  if (v) mask[i] |= (unsigned char)(b << 1);
}

// Union-find over every pixel of one bit image, foreground 8-connected and background 4-connected; background pixels
// on the edge join the extra node n, so that parent[n] ends as the root of the edge-touching background.
__global__ void k_rg_uf_init(int* parent, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n) parent[i] = i;
}

// pl_find with path halving: each visited node is pointed at its grandparent.  A node's parent only ever moves to an
// ancestor in its tree (or, in rg_union's race, to another tree that the same union then merges), so the halving keeps
// every tree's membership; it keeps the chains of the image-wide background components short.
__device__ __forceinline__ int rg_find(int* parent, int a) {
  volatile int* p = parent;
  int q = p[a];
  while (q != a) {
    const int r = p[q];
    if (r != q) p[a] = r;
    a = q;
    q = r;
  }
  return a;
}

__device__ __forceinline__ void rg_union(int* parent, int a, int b) {
  for (;;) {
    a = rg_find(parent, a);
    b = rg_find(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&parent[a], b);
    if (old == a) return;
    a = old;
  }
}

__global__ void k_rg_uf_merge(const unsigned char* __restrict__ mask, int bit, int* parent, RgGeom g) {
  const int n = g.UR * g.UC;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = i / g.UC, x = i - y * g.UC;
  const bool v = mask[i] & bit;
  if (x > 0 && (bool)(mask[i - 1] & bit) == v) rg_union(parent, i, i - 1);
  if (y > 0) {
    if ((bool)(mask[i - g.UC] & bit) == v) rg_union(parent, i, i - g.UC);
    if (v && x > 0 && (mask[i - g.UC - 1] & bit)) rg_union(parent, i, i - g.UC - 1);
    if (v && x + 1 < g.UC && (mask[i - g.UC + 1] & bit)) rg_union(parent, i, i - g.UC + 1);
  }
  if (!v && (x == 0 || y == 0 || x == g.UC - 1 || y == g.UR - 1)) {
    // one pixel per run of edge background joins node n (every other pixel of the run reaches it through its edge
    // predecessor), so that the threads of the edge do not all contend for n's chain
    const bool row_edge = y == 0 || y == g.UR - 1;
    const bool first = row_edge ? x == 0 || (mask[i - 1] & bit) : (bool)(mask[i - g.UC] & bit);
    if (first) rg_union(parent, i, n);
  }
}

struct RgNz {
  const unsigned char* mask;
  int bit, UR, UC;
  __device__ bool operator()(int x, int y) const {
    return x >= 0 && y >= 0 && x < UC && y < UR && (mask[y * UC + x] & bit);
  }
};

struct RgCount {
  __device__ void operator()(int, int) {}
};

// The start kind of pixel i in the boundary image (bit bo) and in the inset image (bit bn): 1 / 2 outer / hole of
// the boundary image, 3 / 4 outer / hole of the inset image, 0 none.  No pixel starts in both: a boundary start has a
// background 4-neighbour, and an inset pixel has none.
__device__ __forceinline__ int rg_kind(const unsigned char* mask, const int* pa, const int* pb, int bo, int bn, int i,
                                       const RgGeom& g) {
  const int n = g.UR * g.UC, x = i % g.UC;
  const bool r = x + 1 < g.UC;
  const int ko = rg_start(i, mask[i] & bo, pa[i], r, r && (mask[i + 1] & bo), r ? pa[i + 1] : -1, pa[n]);
  if (ko) return ko;
  const int kn = rg_start(i, mask[i] & bn, pb[i], r, r && (mask[i + 1] & bn), r ? pb[i + 1] : -1, pb[n]);
  return kn ? kn + 2 : 0;
}

// cnt[i] = the number of points of the border that starts at i (0: none).
__global__ void k_rg_count(const unsigned char* __restrict__ mask, const int* __restrict__ pa,
                           const int* __restrict__ pb, int* __restrict__ cnt, RgGeom g, int ph) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.UR * g.UC) return;
  const int bo = 1 << (2 * ph), bn = bo << 1;
  const int k = rg_kind(mask, pa, pb, bo, bn, i, g);
  int c = 0;
  if (k) {
    RgNz nz{mask, k <= 2 ? bo : bn, g.UR, g.UC};
    RgCount e;
    c = rg_trace(nz, i % g.UC, i / g.UC, !(k & 1), e);
  }
  cnt[i] = c;
}

// have[b] = 1 for every boundary b (its outer start pixel) that holds the first vertex of an inset with > 1 point: the
// inset's start pixel lies in b's component (proof in DESIGN.md §4l).
__global__ void k_rg_have(const unsigned char* __restrict__ mask, const int* __restrict__ pa,
                          const int* __restrict__ pb, const int* __restrict__ cnt, int* __restrict__ have, RgGeom g,
                          int ph) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.UR * g.UC) return;
  const int bo = 1 << (2 * ph);
  if (cnt[i] > 1 && rg_kind(mask, pa, pb, bo, bo << 1, i, g) == 3) have[pa[i]] = 1;
}

// flag[i] = 1 for the start of a kept polygon: its boundary has > 1 point and an inset, and an inset contour's inset
// has > 1 point.  Pass 0 marks ok[row] for every plane row that keeps a boundary.
__global__ void k_rg_keep(const unsigned char* __restrict__ mask, const int* __restrict__ pa,
                          const int* __restrict__ pb, const int* __restrict__ cnt, const int* __restrict__ have,
                          const int* __restrict__ pr, int* __restrict__ flag, int* __restrict__ ok, RgGeom g, int ph) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.UR * g.UC) return;
  const int bo = 1 << (2 * ph);
  const int k = rg_kind(mask, pa, pb, bo, bo << 1, i, g);
  int f = 0;
  if (k) {
    const int b = pa[i];
    f = cnt[b] > 1 && have[b] && (k <= 2 || cnt[k == 3 ? i : pb[i]] > 1);
    if (f && k == 1 && ph == 0) ok[rg_pr(pr, g, i / g.UC, i % g.UC)] = 1;
  }
  flag[i] = f;
}

// Appends the kept polygons of pass ph (raster order of their start) to the records: a sort key, the point count and
// (start pixel, pass).  Key: (plane row, boundary start descending, part), part = boundary outer < its holes (start
// descending) < each inset (start descending) with its outer before its holes (start descending): the reference's
// order (labels ascending, cv::findContours' RETR_CCOMP order within a label).  Counts polygons and regions per row.
__global__ void k_rg_append(const unsigned char* __restrict__ mask, const int* __restrict__ pa,
                            const int* __restrict__ pb, const int* __restrict__ cnt, const int* __restrict__ pr,
                            const int* __restrict__ flag, const int* __restrict__ rank, const int* __restrict__ hdr,
                            unsigned long long* __restrict__ khi, unsigned long long* __restrict__ klo,
                            int* __restrict__ rn, int* __restrict__ rcode, int* lcnt, int* lreg, RgGeom g, int ph) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.UR * g.UC || !flag[i]) return;
  const int bo = 1 << (2 * ph);
  const int k = rg_kind(mask, pa, pb, bo, bo << 1, i, g);
  const int L = rg_pr(pr, g, i / g.UC, i % g.UC);
  const unsigned long long b = RG_LOW - (unsigned long long)pa[i], own = RG_LOW - (unsigned long long)i;
  unsigned long long part, lo;
  if (k == 1) { part = 0; lo = 0; }
  else if (k == 2) { part = 1; lo = own; }
  else if (k == 3) { part = 2; lo = own << (RG_BITS + 1); }
  else { part = 2; lo = ((RG_LOW - (unsigned long long)pb[i]) << (RG_BITS + 1)) | (1ull << RG_BITS) | own; }
  const int id = (ph ? hdr[0] : 0) + rank[i];
  khi[id] = ((unsigned long long)L << (RG_BITS + 2)) | (b << 2) | part;
  klo[id] = lo;
  rn[id] = cnt[i];
  rcode[id] = 2 * i + ph;
  atomicAdd(&lcnt[L], 1);
  if (k == 1) atomicAdd(&lreg[L], 1);
}

// Counting sort into plane-row buckets (slot order within a bucket is arbitrary; k_rg_rank orders it).
__global__ void k_rg_bucket(const unsigned long long* __restrict__ khi, const int* __restrict__ hdr,
                            const int* __restrict__ loff, int* lfill, int* __restrict__ bucket, int cap) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= cap || id >= hdr[0] + hdr[1]) return;
  const int L = (int)(khi[id] >> (RG_BITS + 2));
  bucket[loff[L] + atomicAdd(&lfill[L], 1)] = id;
}

__device__ __forceinline__ bool rg_less(unsigned long long ah, unsigned long long al, unsigned long long bh,
                                        unsigned long long bl) {
  return ah < bh || (ah == bh && al < bl);
}

// Each record's output position (the keys are unique, so position = the number of smaller keys in its bucket), its
// region index and its inset index, found by one pass over its bucket.
__global__ void k_rg_rank(const unsigned long long* __restrict__ khi, const unsigned long long* __restrict__ klo,
                          const int* __restrict__ rn, const int* __restrict__ hdr, const int* __restrict__ lcnt,
                          const int* __restrict__ loff, const int* __restrict__ roff, const int* __restrict__ bucket,
                          int* __restrict__ s_n, int* __restrict__ s_id, int* __restrict__ s_reg,
                          int* __restrict__ s_ins, int cap) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= cap || id >= hdr[0] + hdr[1]) return;
  const unsigned long long h = khi[id], l = klo[id];
  const int L = (int)(h >> (RG_BITS + 2)), part = (int)(h & 3);
  const bool inset_hole = part == 2 && ((l >> RG_BITS) & 1);
  int pos = 0, reg = 0, ins = 0;
  for (int j = loff[L], e = loff[L] + lcnt[L]; j < e; j++) {
    const int o = bucket[j];
    const unsigned long long oh = khi[o], ol = klo[o];
    if (!rg_less(oh, ol, h, l)) continue;
    pos++;
    if ((oh & 3) == 0) reg++;
    if ((oh & 3) == 2 && (oh >> 2) == (h >> 2) && !((ol >> RG_BITS) & 1)) ins++;
  }
  const int p = loff[L] + pos;
  s_n[p] = rn[id];
  s_id[p] = id;
  s_reg[p] = roff[L] + reg - (part == 0 ? 0 : 1);
  s_ins[p] = part == 2 ? ins - (inset_hole ? 1 : 0) : -1;
}

// info[5 .. 8] = {n_regions, n_polygons, n_vertices, complete}; hdr[5] = complete for k_rg_write.
__global__ void k_rg_info(int* hdr, int32_t* __restrict__ info, long long cap_r, long long cap_p, long long cap_v) {
  const int np = hdr[0] + hdr[1];
  const int ok = hdr[3] <= cap_r && np <= cap_p && hdr[4] <= cap_v;
  info[5] = hdr[3]; info[6] = np; info[7] = hdr[4]; info[8] = ok;
  hdr[5] = ok;
}

// info[from .. 7] = 0 and complete = 1: a window outside the map (from 0) or without 2 x 2 cells (from 5).
__global__ void k_rg_none(int32_t* info, int from) {
  for (int k = from; k < 8; k++) info[k] = 0;
  info[8] = 1;
}

struct RgOut {
  double* regions;
  int32_t* polys;
  double* verts;
  const double* planes;  // the plane table: (label, support, normal) per row
  double ox, oy, res3, offset;
};

struct RgWrite {
  double* v;
  const double* T;
  double ox, oy, res3;
  double lo[2], hi[2];
  int n;
  __device__ void operator()(int x, int y) {
    double px, py;
    rg_project(T, ox - res3 * y, oy - res3 * x, px, py);
    v[2 * n] = px;
    v[2 * n + 1] = py;
    lo[0] = n ? fmin(lo[0], px) : px; lo[1] = n ? fmin(lo[1], py) : py;
    hi[0] = n ? fmax(hi[0], px) : px; hi[1] = n ? fmax(hi[1], py) : py;
    n++;
  }
};

// One thread per polygon in output order: its row, its points (traced again) in the plane frame, and for a boundary
// outer its region row.  Nothing when the output is incomplete.
__global__ void k_rg_write(const unsigned char* __restrict__ mask, const unsigned long long* __restrict__ khi,
                           const unsigned long long* __restrict__ klo, const int* __restrict__ rcode,
                           const int* __restrict__ hdr, const int* __restrict__ s_n, const int* __restrict__ s_id,
                           const int* __restrict__ s_reg, const int* __restrict__ s_ins,
                           const int* __restrict__ s_first, RgOut o, RgGeom g, int cap) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= cap || p >= hdr[0] + hdr[1] || !hdr[5]) return;
  const int id = s_id[p], code = rcode[id], i = code >> 1, ph = code & 1;
  const unsigned long long h = khi[id];
  const int L = (int)(h >> (RG_BITS + 2)), part = (int)(h & 3);
  const int role = part == 0 ? 0 : part == 1 ? 1 : ((klo[id] >> RG_BITS) & 1) ? 3 : 2;
  const int first = s_n[p] ? s_first[p] : 0;
  int32_t* row = o.polys + (long long)RG_POLY * p;
  row[0] = s_reg[p]; row[1] = role; row[2] = s_ins[p]; row[3] = first; row[4] = s_n[p];
  const double* pl = o.planes + 7ll * L;
  double T[12];
  rg_plane_transform(pl + 1, pl + 4, T);
  const int bo = 1 << (2 * ph);
  RgNz nz{mask, role < 2 ? bo : bo << 1, g.UR, g.UC};
  RgWrite w{o.verts + 2ll * first, T, o.ox, o.oy, o.res3, {0, 0}, {0, 0}, 0};
  rg_trace(nz, i % g.UC, i / g.UC, role & 1, w);
  if (role == 0) {
    double* r = o.regions + (long long)RG_ROW * s_reg[p];
    r[0] = pl[0];
    for (int k = 0; k < 12; k++) r[1 + k] = T[k];
    r[1 + 11] += o.offset;
    r[13] = w.lo[0]; r[14] = w.lo[1]; r[15] = w.hi[0]; r[16] = w.hi[1];
  }
}
#endif
