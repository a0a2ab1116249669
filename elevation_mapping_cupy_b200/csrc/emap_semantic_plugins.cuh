// emap_semantic_plugins.cuh -- the plugins that consume semantic layers (sm_90a): plugins/semantic_filter.py:13-133,
// plugins/semantic_traversability.py:12-83 and plugins/features_pca.py:13-96 of the reference.
//
// k_semantic_filter: per cell, numpy.argmax over L stacked planes (first maximum wins, a NaN is the maximum and the first
// NaN wins), then the palette entry of that class id, stored as bits.  About half the palette words are fp32 denormals:
// they are only ever moved as integers.
// k_semantic_traversability: per cell, the number of layers whose value passes its threshold (<= for the traversability
// type, >= otherwise, compared in fp64); fp32(0.1) if none passes, else 1.
// features_pca: exact 3-component PCA of F clipped feature planes, four kernels and no mid-call host synchronisation:
//   k_pca_stats  per-feature sums and the F x F Gram matrix in fp64, one partial per CTA, and the NaN flag;
//   k_pca_eigen  one CTA: sums the partials in a fixed order, centres, cyclic Jacobi (parallel round-robin ordering) in
//                fp64, the top 3 eigenvectors with sklearn's svd_flip(u_based_decision=False) sign rule;
//   k_pca_project (x - mean) . v_k in fp64 per cell, min / max per component (exact, so atomics keep it deterministic);
//   k_pca_pack   uint8(trunc((p - min) / (max - min) * 255)) per channel, packed r << 16 | g << 8 | b.
#pragma once
#include "emap_device.cuh"

#define SEMF_MAX_LAYERS 255       // == EMAP_SEMANTIC_FILTER_MAX_LAYERS
#define SEMT_MAX_LAYERS 128       // == EMAP_SEMANTIC_TRAVERSABILITY_MAX_LAYERS (pointers + thresholds fit the 4 KB of kernel
                                  // parameters)
#define PCA_MAX_F 64              // == EMAP_PCA_MAX_FEATURES
#define PCA_THREADS 512           // k_pca_stats and k_pca_eigen
#define PCA_TILE_FLOATS 8192      // k_pca_stats' shared tile: (F + 1) rows of TC + 1 floats
#define PCA_MAX_ENTRIES ((PCA_MAX_F * (PCA_MAX_F + 1)) / 2 + PCA_MAX_F)   // Gram triangle + feature sums
#define PCA_ENTRIES_PER_THREAD ((PCA_MAX_ENTRIES + PCA_THREADS - 1) / PCA_THREADS)
#define PCA_MAX_SWEEPS 40

struct SemFilterArgs {
  int n;
  const float* plane[SEMF_MAX_LAYERS];
};

struct SemTravArgs {
  int n;
  u32 is_trav[(SEMT_MAX_LAYERS + 31) / 32];   // bit l: layer l is of the "traversability" type
  const float* plane[SEMT_MAX_LAYERS];
  double thr[SEMT_MAX_LAYERS];
};

struct PcaArgs {
  int F;
  const float* plane[PCA_MAX_F];
};

struct PcaResult {                 // written by k_pca_eigen, read by the projection and pack kernels
  double mean[PCA_MAX_F];
  double comp[3][PCA_MAX_F];
  unsigned long long lo[3], hi[3]; // ordered keys of the per-component min / max (pca_key)
  int nan;                         // an input value was NaN
  int sweeps;                      // Jacobi sweeps run (diagnostics)
};

// plugins/semantic_filter.py:30-58 color_map(255): the VOC-style map with bit 0/1/2 of the index interleaved into r/g/b from
// the top bit down, rows 1 and 2 set to (81, 113, 162), row 3 to (188, 63, 59), row 0 dropped (class id k takes row k + 1);
// transform_color (:60-75) packs r << 16 | g << 8 | b.  Built once, at compile time.
struct SemPalette {
  u32 rgb[SEMF_MAX_LAYERS];
};
constexpr u32 sem_palette_row(int i) {
  if (i == 1 || i == 2) return (81u << 16) | (113u << 8) | 162u;
  if (i == 3) return (188u << 16) | (63u << 8) | 59u;
  u32 r = 0, g = 0, b = 0;
  int c = i;
  for (int j = 0; j < 8; j++) {
    r |= (u32)(c & 1) << (7 - j);
    g |= (u32)((c >> 1) & 1) << (7 - j);
    b |= (u32)((c >> 2) & 1) << (7 - j);
    c >>= 3;
  }
  return (r << 16) | (g << 8) | b;
}
constexpr SemPalette make_sem_palette() {
  SemPalette p{};
  for (int k = 0; k < SEMF_MAX_LAYERS; k++) p.rgb[k] = sem_palette_row(k + 1);
  return p;
}
__device__ const SemPalette g_sem_palette = make_sem_palette();

__global__ void __launch_bounds__(256) k_semantic_filter(int C, SemFilterArgs a, u32* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  int id = 0;
  if (a.n > 0) {
    float best = __ldg(a.plane[0] + i);
    for (int l = 1; l < a.n && !isnan(best); l++) {
      const float v = __ldg(a.plane[l] + i);
      if (isnan(v) || v > best) { best = v; id = l; }
    }
  }
  out[i] = __ldg(&g_sem_palette.rgb[id]);
}

__global__ void __launch_bounds__(256) k_semantic_traversability(int C, SemTravArgs a, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  int score = 0;
  for (int l = 0; l < a.n; l++) {
    const double v = (double)__ldg(a.plane[l] + i);    // exact: the comparison is the fp64 one
    const bool trav = (a.is_trav[l >> 5] >> (l & 31)) & 1u;
    score += trav ? (v <= a.thr[l]) : (v >= a.thr[l]);  // false for NaN
  }
  out[i] = score == 0 ? 0.1f : 1.0f;                    // semantic_traversability.py:80: sum <= 0.9 ? 0.1 : 1
}

// ---- features_pca ----------------------------------------------------------------------------------------------------
// cells per k_pca_stats tile: (F + 1) rows of TC + 1 floats fit PCA_TILE_FLOATS; TC a multiple of 32
__host__ __device__ inline int pca_tile_cells(int F) {
  int tc = (PCA_TILE_FLOATS / (F + 1) - 1) & ~31;
  return tc > 1024 ? 1024 : tc;
}
__host__ __device__ inline int pca_entries(int F) { return F * (F + 1) / 2 + F; }

// order-preserving map of a non-NaN double to u64 (exact min / max through integer atomics)
__device__ __forceinline__ unsigned long long pca_key(double d) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(d);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double pca_unkey(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// Entry e of the accumulated set: e < F(F+1)/2 is the Gram entry (a, b), a <= b, row-major over the upper triangle;
// the last F entries are the feature sums (a, F): row F of the tile holds 1 for every real cell.
__device__ __forceinline__ void pca_entry_ab(int F, int e, int& a, int& b) {
  const int T = F * (F + 1) / 2;
  if (e >= T) { a = e - T; b = F; return; }
  a = 0;
  int row = F;
  while (e >= row) { e -= row; row--; a++; }
  b = a + e;
}

// One partial (pca_entries(F) doubles) per CTA over tiles blockIdx.x, blockIdx.x + gridDim.x, ...: the partition and the
// summation order depend only on C, F and the grid, so the result is the same every run.  With E <= PCA_THREADS entries,
// G = PCA_THREADS / E thread groups each take one entry per thread and every G-th cell of a tile, and their sums are
// added in group order at the end; with more entries every thread takes J = ceil(E / PCA_THREADS) of them.
__global__ void __launch_bounds__(PCA_THREADS) k_pca_stats(int C, PcaArgs a, double* __restrict__ part,
                                                           PcaResult* __restrict__ res) {
  __shared__ __align__(16) float s[PCA_TILE_FLOATS];
  __shared__ int s_nan;
  const int F = a.F, TC = pca_tile_cells(F), TP = TC + 1, E = pca_entries(F);
  const int G = E <= PCA_THREADS ? PCA_THREADS / E : 1, J = (E + PCA_THREADS - 1) / PCA_THREADS;
  const int g = G > 1 ? (int)threadIdx.x / E : 0, e0 = G > 1 ? (int)threadIdx.x % E : (int)threadIdx.x;
  const bool active = g < G;
  if (threadIdx.x == 0) s_nan = 0;
  int ea[PCA_ENTRIES_PER_THREAD], eb[PCA_ENTRIES_PER_THREAD];
  double acc[PCA_ENTRIES_PER_THREAD];
#pragma unroll
  for (int j = 0; j < PCA_ENTRIES_PER_THREAD; j++) {
    const int e = e0 + j * PCA_THREADS;
    ea[j] = eb[j] = 0;
    if (j < J && e < E) pca_entry_ab(F, e, ea[j], eb[j]);
    ea[j] *= TP; eb[j] *= TP;
    acc[j] = 0.0;
  }
  int nan = 0;
  const int n_tiles = (C + TC - 1) / TC;
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int c0 = t * TC;
    __syncthreads();                                       // the previous tile is consumed
    for (int k = threadIdx.x; k < (F + 1) * TC; k += PCA_THREADS) {
      const int f = k / TC, c = k - f * TC, i = c0 + c;
      float v = 0.f;
      if (i < C) {
        if (f < F) {
          v = __ldg(a.plane[f] + i);
          nan |= isnan(v);
          v = fminf(fmaxf(v, -1.f), 1.f);                  // features_pca.py:75 np.clip(data, -1, 1), in fp32
        } else v = 1.f;
      }
      s[f * TP + c] = v;
    }
    __syncthreads();
    if (active) {
      if (J == 1) {
        for (int c = g; c < TC; c += G) acc[0] = fma((double)s[ea[0] + c], (double)s[eb[0] + c], acc[0]);  // exact product
      } else {
        for (int c = 0; c < TC; c++) {
#pragma unroll
          for (int j = 0; j < PCA_ENTRIES_PER_THREAD; j++)
            if (j < J) acc[j] = fma((double)s[ea[j] + c], (double)s[eb[j] + c], acc[j]);
        }
      }
    }
  }
  if (nan) s_nan = 1;                                      // benign race: every writer stores 1
  __syncthreads();                                         // the tile is consumed: its memory takes the group sums
  double* red = (double*)s;                                // G * E <= PCA_THREADS doubles
  if (G > 1) {
    if (active) red[g * E + e0] = acc[0];
    __syncthreads();
    if ((int)threadIdx.x < E) {
      double sum = red[threadIdx.x];
      for (int k = 1; k < G; k++) sum += red[k * E + threadIdx.x];
      part[(size_t)blockIdx.x * E + threadIdx.x] = sum;
    }
  } else {
#pragma unroll
    for (int j = 0; j < PCA_ENTRIES_PER_THREAD; j++) {
      const int e = e0 + j * PCA_THREADS;
      if (j < J && e < E) part[(size_t)blockIdx.x * E + e] = acc[j];
    }
  }
  if (threadIdx.x == 0 && s_nan) res->nan = 1;
}

// Jacobi rotation of the pair (p, q) that zeroes A[p][q] (Golub & Van Loan, sym.schur2): J = [[c, s], [-s, c]].
__device__ __forceinline__ void pca_rotation(double app, double aqq, double apq, double& c, double& s) {
  if (apq == 0.0) { c = 1.0; s = 0.0; return; }
  const double tau = (aqq - app) / (2.0 * apq);
  const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
  c = 1.0 / sqrt(1.0 + t * t);
  s = t * c;
}

// One CTA.  Dynamic shared memory: A and V, F x (F + 1) doubles each.
__global__ void __launch_bounds__(PCA_THREADS) k_pca_eigen(int C, int F, int n_part, const double* __restrict__ part,
                                                           PcaResult* __restrict__ res) {
  extern __shared__ double sm[];
  const int LD = F + 1;
  double* A = sm;
  double* V = sm + F * LD;
  __shared__ double s_sum[PCA_MAX_F];
  __shared__ double s_rc[PCA_MAX_F / 2], s_rs[PCA_MAX_F / 2];
  __shared__ int s_rp[PCA_MAX_F / 2], s_rq[PCA_MAX_F / 2];
  __shared__ double s_row[PCA_MAX_F];
  __shared__ int s_done;
  const int E = pca_entries(F), T = F * (F + 1) / 2;
  const int tid = threadIdx.x;
  // partials in CTA order, then the centred scatter matrix (its scale does not change the eigenvectors)
  for (int e = tid; e < E; e += PCA_THREADS) {
    double g = 0.0;
    for (int b = 0; b < n_part; b++) g += part[(size_t)b * E + e];
    if (e >= T) s_sum[e - T] = g;
    else {
      int ia, ib;
      pca_entry_ab(F, e, ia, ib);
      A[ia * LD + ib] = g;
    }
  }
  for (int k = tid; k < F * F; k += PCA_THREADS) V[(k / F) * LD + k % F] = (k / F == k % F) ? 1.0 : 0.0;
  __syncthreads();
  const double n = (double)C;                              // divisions, not a reciprocal: exact where the data allow
  for (int k = tid; k < F * F; k += PCA_THREADS) {
    const int i = k / F, j = k % F;
    if (i <= j) {
      const double v = A[i * LD + j] - s_sum[i] * s_sum[j] / n;
      A[i * LD + j] = v;
      if (i != j) A[j * LD + i] = v;
    }
  }
  if (tid < F) res->mean[tid] = s_sum[tid] / n;
  if (tid == 0) s_done = res->nan;                         // NaN input: the call fails, skip the iteration
  __syncthreads();
  // cyclic Jacobi, round-robin ordering: m / 2 disjoint pairs per round, m - 1 rounds per sweep (m = F rounded up to even;
  // pairs with the padding index are skipped)
  const int m = (F + 1) & ~1, half = m / 2;
  int sweep = 0;
  for (; sweep < PCA_MAX_SWEEPS && !s_done; sweep++) {
    for (int r = 0; r < m - 1; r++) {
      if (tid < half) {
        const int pp = tid, qq = m - 1 - tid;
        const int p = pp == 0 ? 0 : 1 + (pp - 1 + r) % (m - 1);
        const int q = 1 + (qq - 1 + r) % (m - 1);
        double c = 1.0, s = 0.0;
        if (p < F && q < F) pca_rotation(A[p * LD + p], A[q * LD + q], A[p * LD + q], c, s);
        s_rp[tid] = p < F && q < F ? p : -1; s_rq[tid] = q; s_rc[tid] = c; s_rs[tid] = s;
      }
      __syncthreads();
      for (int k = tid; k < F * half; k += PCA_THREADS) {  // A <- A J, V <- V J (columns p, q of row i)
        const int i = k / half, pr = k % half, p = s_rp[pr];
        if (p < 0 || s_rs[pr] == 0.0) continue;
        const int q = s_rq[pr];
        const double c = s_rc[pr], s = s_rs[pr];
        const double ap = A[i * LD + p], aq = A[i * LD + q], vp = V[i * LD + p], vq = V[i * LD + q];
        A[i * LD + p] = c * ap - s * aq; A[i * LD + q] = s * ap + c * aq;
        V[i * LD + p] = c * vp - s * vq; V[i * LD + q] = s * vp + c * vq;
      }
      __syncthreads();
      for (int k = tid; k < F * half; k += PCA_THREADS) {  // A <- J^T A (rows p, q of column j)
        const int j = k / half, pr = k % half, p = s_rp[pr];
        if (p < 0 || s_rs[pr] == 0.0) continue;
        const int q = s_rq[pr];
        const double c = s_rc[pr], s = s_rs[pr];
        const double ap = A[p * LD + j], aq = A[q * LD + j];
        A[p * LD + j] = c * ap - s * aq; A[q * LD + j] = s * ap + c * aq;
      }
      __syncthreads();
    }
    // converged when the off-diagonal mass is below 1e-26 of the diagonal's (|off| ~ 1e-13 |diag|): fixed-order sums
    if (tid < F) {
      double off = 0.0;
      for (int j = 0; j < F; j++) if (j != tid) off += A[tid * LD + j] * A[tid * LD + j];
      s_row[tid] = off;
    }
    __syncthreads();
    if (tid == 0) {
      double off = 0.0, dia = 0.0;
      for (int i = 0; i < F; i++) { off += s_row[i]; dia += A[i * LD + i] * A[i * LD + i]; }
      s_done = !(off > 1e-26 * dia);
    }
    __syncthreads();
  }
  if (tid == 0) {
    // the 3 largest eigenvalues, descending; equal eigenvalues keep the lower index first
    int pick[3];
    for (int k = 0; k < 3; k++) {
      int best = -1;
      for (int i = 0; i < F; i++) {
        bool used = false;
        for (int j = 0; j < k; j++) used |= pick[j] == i;
        if (!used && (best < 0 || A[i * LD + i] > A[best * LD + best])) best = i;
      }
      pick[k] = best;
    }
    for (int k = 0; k < 3; k++) {
      // sklearn svd_flip(u_based_decision=False): the entry of largest |value| (the first on ties) is made positive
      int arg = 0;
      for (int i = 1; i < F; i++) if (fabs(V[i * LD + pick[k]]) > fabs(V[arg * LD + pick[k]])) arg = i;
      const double sg = V[arg * LD + pick[k]] < 0.0 ? -1.0 : 1.0;
      for (int i = 0; i < F; i++) res->comp[k][i] = sg * V[i * LD + pick[k]];
      res->lo[k] = ~0ull;
      res->hi[k] = 0ull;
    }
    res->sweeps = sweep;
  }
}

// p[k * C + i] = (x_i - mean) . v_k in fp64 over the clipped fp32 features; min / max per component into res->lo / hi.
__global__ void __launch_bounds__(256) k_pca_project(int C, PcaArgs a, PcaResult* __restrict__ res, double* __restrict__ p) {
  __shared__ double s_m[PCA_MAX_F], s_v[3][PCA_MAX_F];
  __shared__ unsigned long long s_lo[3], s_hi[3];
  const int F = a.F;
  for (int k = threadIdx.x; k < F; k += blockDim.x) {
    s_m[k] = res->mean[k];
    s_v[0][k] = res->comp[0][k]; s_v[1][k] = res->comp[1][k]; s_v[2][k] = res->comp[2][k];
  }
  if (threadIdx.x < 3) { s_lo[threadIdx.x] = ~0ull; s_hi[threadIdx.x] = 0ull; }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long lo[3] = {~0ull, ~0ull, ~0ull}, hi[3] = {0ull, 0ull, 0ull};
  if (i < C) {
    double q[3] = {0.0, 0.0, 0.0};
    for (int f = 0; f < F; f++) {
      const double x = (double)fminf(fmaxf(__ldg(a.plane[f] + i), -1.f), 1.f) - s_m[f];
      q[0] = fma(x, s_v[0][f], q[0]); q[1] = fma(x, s_v[1][f], q[1]); q[2] = fma(x, s_v[2][f], q[2]);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
      p[(size_t)k * C + i] = q[k];
      lo[k] = hi[k] = pca_key(q[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < 3; k++) {
    for (int o = 16; o; o >>= 1) {
      lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
      hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; k++) { atomicMin(&s_lo[k], lo[k]); atomicMax(&s_hi[k], hi[k]); }
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    atomicMin(&res->lo[threadIdx.x], s_lo[threadIdx.x]);
    atomicMax(&res->hi[threadIdx.x], s_hi[threadIdx.x]);
  }
}

// features_pca.py:83-93: channel = uint8(trunc((p - min) / (max - min) * 255)) in fp64; a component of range 0 gives 0
__global__ void __launch_bounds__(256) k_pca_pack(int C, const PcaResult* __restrict__ res, const double* __restrict__ p,
                                                  u32* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  u32 rgb = 0;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const double lo = pca_unkey(res->lo[k]), range = pca_unkey(res->hi[k]) - lo;
    u32 ch = 0;
    if (range > 0.0) ch = (u32)__double2int_rz((p[(size_t)k * C + i] - lo) / range * 255.0);
    rgb = (rgb << 8) | (ch & 0xffu);
  }
  out[i] = rgb;
}
