// emap_initialize.cuh -- the map initialiser's interpolation (emap_initialize_map), sm_90a.
//
// Reference: EM.py:899-922 + map_initializer.py:25-62, SciPy's griddata over every cell from a handful of points.  The
// host part snaps the points to cells, builds the Delaunay triangulation when the caller passes none, estimates the
// cubic's vertex gradients when the caller passes none, turns them into per-triangle coefficients and bins the
// triangles into 32 x 32 cell tiles.  One kernel then writes elevation / variance / is_valid of every cell where the
// interpolant is defined.  include/emap.h states the rules.
//
// Every predicate is exact on integer cell indices (__int128 where products can pass 63 bits).  Kernel arithmetic is
// fp64 with explicit round-to-nearest operations (no contraction), in the order of tests/initialize_oracle.py.
#pragma once
#include <algorithm>
#include <array>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>
#include <cuda_runtime.h>

#define INIT_TILE 32              // cells per tile side
#define INIT_THREADS 256          // 8 warps: each thread takes 4 rows of one tile column
#define INIT_CHUNK 256            // triangles / point candidates staged in shared memory at a time
#define INIT_CT 19                // Clough-Tocher ordinates per triangle
#define INIT_NARROW (1ll << 29)   // cell indices within +-2^29: every kernel product fits in 63 bits

struct InitArgs {
  int W, C, tiles_x, n;               // n: points (nearest) or triangles
  float var;                          // initialized_variance
  const int* txy;                     // (T, 6) counter-clockwise vertices x0 y0 x1 y1 x2 y2
  const double* coef;                 // (T, 3) vertex heights (linear) or (T, INIT_CT) ordinates (cubic)
  const int* tile_off;                // (tiles + 1) CSR offsets of the tile triangle lists, ascending triangle order
  const int* tile_tri;
  const int2* pxy;                    // (n) point cells (nearest)
  const float* pz;                    // (n) point heights (nearest)
};

// ---- exact integer predicates ----------------------------------------------------------------------------------------
// D: long long when every coordinate is narrow (|x| <= 2^29), __int128 otherwise.
template <typename D>
__host__ __device__ __forceinline__ D orient2(D ax, D ay, D bx, D by, D cx, D cy) {
  return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
}

__host__ __device__ __forceinline__ double i128_to_double(__int128 v) {
  const bool neg = v < 0;
  const unsigned __int128 u = neg ? (unsigned __int128)(-(v + 1)) + 1 : (unsigned __int128)v;
  const double d = (double)(unsigned long long)(u >> 64) * 18446744073709551616.0 + (double)(unsigned long long)u;
  return neg ? -d : d;
}
__host__ __device__ __forceinline__ double to_double(long long v) { return (double)v; }
__host__ __device__ __forceinline__ double to_double(__int128 v) { return i128_to_double(v); }

namespace init_host {

// > 0 when d lies strictly inside the circumcircle of the counter-clockwise triangle (a, b, c).  Differences take 33
// bits, lifts 66 and cross terms 66, so a lift is split at bit 32 and the sum kept as H * 2^32 + L.
inline int incircle(const long long* a, const long long* b, const long long* c, const long long* d) {
  const __int128 ax = a[0] - d[0], ay = a[1] - d[1], bx = b[0] - d[0], by = b[1] - d[1], cx = c[0] - d[0], cy = c[1] - d[1];
  const __int128 lift[3] = {ax * ax + ay * ay, bx * bx + by * by, cx * cx + cy * cy};
  const __int128 cross[3] = {bx * cy - cx * by, cx * ay - ax * cy, ax * by - bx * ay};
  __int128 H = 0, L = 0;
  for (int k = 0; k < 3; k++) {
    H += (lift[k] >> 32) * cross[k];
    L += (lift[k] & (__int128)0xffffffff) * cross[k];
  }
  const __int128 carry = L >> 32;             // floor: leaves 0 <= L < 2^32
  H += carry;
  L -= carry * ((__int128)1 << 32);
  return H > 0 ? 1 : (H < 0 ? -1 : (L > 0 ? 1 : 0));
}

inline int orient_sign(const long long* a, const long long* b, const long long* c) {
  const __int128 o = orient2<__int128>(a[0], a[1], b[0], b[1], c[0], c[1]);
  return o > 0 ? 1 : (o < 0 ? -1 : 0);
}

struct Tri {
  int v[3];       // counter-clockwise; v[2] == -1 for a ghost (hull edge v[0] -> v[1], outside on its left)
  int n[3];       // the triangle across the edge opposite v[k]
  int stamp;      // insertion that put it in a cavity (dead) or 0
};

// The library's Delaunay triangulation (tests/initialize_oracle.py delaunay): Bowyer-Watson with exact predicates and
// ghost triangles, inserting in input order from the seed (point 0, the first point that differs from it, the first
// point not collinear with those two).  A point equal to an earlier one is skipped.  A point on a circumcircle does not
// break the triangle, so among cocircular points the triangles of the earlier ones stay.  Returns false when all points
// are collinear.  `out` gets the triangles in canonical order: each rotated to start at its lowest vertex, sorted.
inline bool delaunay(const std::vector<long long>& xy, std::vector<int>& out) {
  const int n = (int)(xy.size() / 2);
  auto P = [&](int i) { return &xy[2 * (size_t)i]; };
  int i1 = -1, i2 = -1;
  for (int i = 1; i < n && i1 < 0; i++)
    if (xy[2 * i] != xy[0] || xy[2 * i + 1] != xy[1]) i1 = i;
  if (i1 < 0) return false;
  for (int i = 1; i < n && i2 < 0; i++)
    if (orient_sign(P(0), P(i1), P(i)) != 0) i2 = i;
  if (i2 < 0) return false;
  int a = 0, b = i1, c = i2;
  if (orient_sign(P(a), P(b), P(c)) < 0) std::swap(b, c);
  std::vector<Tri> T;
  T.reserve(8 * (size_t)n);
  // solid 0 = (a, b, c); ghosts across its edges: opposite a (edge b-c) -> (c, b, inf), opposite b -> (a, c, inf),
  // opposite c -> (b, a, inf); each ghost's solid neighbour sits opposite its inf vertex (n[2])
  T.push_back({{a, b, c}, {1, 2, 3}, 0});
  T.push_back({{c, b, -1}, {3, 2, 0}, 0});
  T.push_back({{a, c, -1}, {1, 3, 0}, 0});
  T.push_back({{b, a, -1}, {2, 1, 0}, 0});
  std::unordered_map<unsigned long long, int> seen;
  auto key = [&](int i) { return ((unsigned long long)(uint32_t)xy[2 * i] << 32) | (uint32_t)xy[2 * i + 1]; };
  seen[key(0)] = 0; seen[key(i1)] = i1; seen[key(i2)] = i2;
  auto conflict = [&](const Tri& t, int p) {
    if (t.v[2] >= 0) return incircle(P(t.v[0]), P(t.v[1]), P(t.v[2]), P(p)) > 0;
    const long long *u = P(t.v[0]), *v = P(t.v[1]), *q = P(p);
    const int o = orient_sign(u, v, q);
    if (o != 0) return o > 0;
    const __int128 d0 = (__int128)(q[0] - u[0]) * (v[0] - u[0]) + (__int128)(q[1] - u[1]) * (v[1] - u[1]);
    const __int128 d1 = (__int128)(q[0] - v[0]) * (u[0] - v[0]) + (__int128)(q[1] - v[1]) * (u[1] - v[1]);
    return d0 > 0 && d1 > 0;
  };
  struct Edge { int x, y, out, tri; };
  std::vector<int> stack, fresh;
  std::vector<Edge> bnd;
  int last = 0;
  for (int p = 0, stamp = 1; p < n; p++) {
    if (p == 0 || p == i1 || p == i2) continue;
    if (!seen.emplace(key(p), p).second) continue;
    stamp++;
    // visibility walk from the last new triangle to one whose circle holds p (Delaunay: the walk terminates; a bound
    // guards it all the same, with a scan of every live triangle behind it)
    int t = last;
    if (T[t].v[2] < 0) t = T[t].n[2];
    for (long long steps = 0; T[t].v[2] >= 0 && steps <= 4ll * (long long)T.size(); steps++) {
      int next = -1;
      for (int k = 0; k < 3 && next < 0; k++)
        if (orient_sign(P(T[t].v[(k + 1) % 3]), P(T[t].v[(k + 2) % 3]), P(p)) < 0) next = T[t].n[k];
      if (next < 0) break;
      t = next;
    }
    if (!conflict(T[t], p)) t = -1;
    for (int s = 0; s < (int)T.size() && t < 0; s++)
      if (!T[s].stamp && conflict(T[s], p)) t = s;
    if (t < 0) return false;
    // the cavity: every triangle whose circle holds p, connected; its boundary edges face p
    stack.assign(1, t);
    T[t].stamp = stamp;
    bnd.clear();
    while (!stack.empty()) {
      const int s = stack.back();
      stack.pop_back();
      for (int k = 0; k < 3; k++) {
        const int o = T[s].n[k];
        if (T[o].stamp == stamp) continue;
        if (!T[o].stamp && conflict(T[o], p)) { T[o].stamp = stamp; stack.push_back(o); continue; }
        bnd.push_back({T[s].v[(k + 1) % 3], T[s].v[(k + 2) % 3], o, -1});
      }
    }
    fresh.clear();
    for (Edge& e : bnd) {
      Tri nt = {{e.x, e.y, p}, {-2, -2, e.out}, 0};
      const int r = e.x < 0 ? 1 : (e.y < 0 ? 2 : 0);       // rotate so a ghost's inf vertex comes last
      Tri rt;
      for (int k = 0; k < 3; k++) { rt.v[k] = nt.v[(k + r) % 3]; rt.n[k] = nt.n[(k + r) % 3]; }
      rt.stamp = 0;
      e.tri = (int)T.size();
      for (int k = 0; k < 3; k++)                    // the outside triangle now faces the new one
        if (T[e.out].n[k] >= 0 && T[T[e.out].n[k]].stamp == stamp) {
          const int* ov = T[e.out].v;
          if ((ov[(k + 1) % 3] == e.y && ov[(k + 2) % 3] == e.x)) T[e.out].n[k] = e.tri;
        }
      T.push_back(rt);
      fresh.push_back(e.tri);
    }
    for (int f : fresh)                              // link the new triangles around p to one another
      for (int k = 0; k < 3; k++) {
        if (T[f].n[k] != -2) continue;
        const int x = T[f].v[(k + 1) % 3], y = T[f].v[(k + 2) % 3];
        for (int g : fresh)
          for (int j = 0; j < 3; j++)
            if (T[g].v[(j + 1) % 3] == y && T[g].v[(j + 2) % 3] == x) T[f].n[k] = g;
      }
    last = fresh.back();
  }
  out.clear();
  std::vector<std::array<int, 3>> tris;
  for (const Tri& t : T) {
    if (t.stamp || t.v[2] < 0) continue;
    const int r = (t.v[0] < t.v[1] && t.v[0] < t.v[2]) ? 0 : (t.v[1] < t.v[2] ? 1 : 2);
    tris.push_back({t.v[r], t.v[(r + 1) % 3], t.v[(r + 2) % 3]});
  }
  std::sort(tris.begin(), tris.end());
  for (const auto& t : tris) out.insert(out.end(), t.begin(), t.end());
  return true;
}

// (T, 3): the triangle across the edge opposite vertex k of each counter-clockwise triangle, -1 on the hull
inline void neighbours(const std::vector<int>& tri, std::vector<int>& nb) {
  const int T = (int)(tri.size() / 3);
  std::unordered_map<unsigned long long, int> at;
  at.reserve(3 * (size_t)T);
  auto ek = [](int x, int y) { return ((unsigned long long)(uint32_t)x << 32) | (uint32_t)y; };
  for (int t = 0; t < T; t++)
    for (int k = 0; k < 3; k++) at[ek(tri[3 * t + (k + 1) % 3], tri[3 * t + (k + 2) % 3])] = t;
  nb.assign(3 * (size_t)T, -1);
  for (int t = 0; t < T; t++)
    for (int k = 0; k < 3; k++) {
      auto it = at.find(ek(tri[3 * t + (k + 2) % 3], tri[3 * t + (k + 1) % 3]));
      if (it != at.end()) nb[3 * t + k] = it->second;
    }
}

// SciPy's estimate_gradients_2d_global (tol 1e-6, maxiter 400): Gauss-Seidel sweeps over the vertices in index order,
// each vertex's neighbours in ascending order.  A point on no triangle keeps gradient (0, 0).
inline void estimate_gradients(const std::vector<long long>& xy, const std::vector<double>& z, const std::vector<int>& tri,
                               std::vector<double>& y) {
  const int n = (int)z.size();
  std::vector<std::vector<int>> nb(n);
  for (size_t t = 0; t < tri.size(); t += 3)
    for (int k = 0; k < 3; k++) {
      nb[tri[t + k]].push_back(tri[t + (k + 1) % 3]);
      nb[tri[t + k]].push_back(tri[t + (k + 2) % 3]);
    }
  for (auto& v : nb) { std::sort(v.begin(), v.end()); v.erase(std::unique(v.begin(), v.end()), v.end()); }
  y.assign(2 * (size_t)n, 0.0);
  for (int iter = 0; iter < 400; iter++) {
    double err = 0;
    for (int i = 0; i < n; i++) {
      if (nb[i].empty()) continue;
      double q0 = 0, q1 = 0, q3 = 0, s0 = 0, s1 = 0;
      for (int j : nb[i]) {
        const double ex = (double)xy[2 * j] - (double)xy[2 * i], ey = (double)xy[2 * j + 1] - (double)xy[2 * i + 1];
        const double L = std::sqrt(ex * ex + ey * ey), L3 = L * L * L;
        const double df2 = -ex * y[2 * j] - ey * y[2 * j + 1];
        q0 += 4 * ex * ex / L3;
        q1 += 4 * ex * ey / L3;
        q3 += 4 * ey * ey / L3;
        s0 += (6 * (z[i] - z[j]) - 2 * df2) * ex / L3;
        s1 += (6 * (z[i] - z[j]) - 2 * df2) * ey / L3;
      }
      const double det = q0 * q3 - q1 * q1;
      const double r0 = (q3 * s0 - q1 * s1) / det, r1 = (-q1 * s0 + q0 * s1) / det;
      double change = std::max(std::fabs(y[2 * i] + r0), std::fabs(y[2 * i + 1] + r1));
      y[2 * i] = -r0;
      y[2 * i + 1] = -r1;
      change /= std::max(1.0, std::max(std::fabs(r0), std::fabs(r1)));
      err = std::max(err, change);
    }
    if (err < 1e-6) break;
  }
}

// SciPy's Clough-Tocher element (CloughTocher2DInterpolator) of each triangle as 19 Bezier ordinates, in the order
// of tests/initialize_oracle.py CT_NAMES; the cross-boundary directions point at the neighbours' centroids.
inline void ct_coefficients(const std::vector<long long>& xy, const std::vector<double>& z, const double* grad,
                            const std::vector<int>& tri, const std::vector<int>& nb, double* out) {
  const int T = (int)(tri.size() / 3);
  auto X = [&](int v) { return (double)xy[2 * v]; };
  auto Y = [&](int v) { return (double)xy[2 * v + 1]; };
  for (int t = 0; t < T; t++) {
    const int* v = &tri[3 * t];
    const double p0[2] = {X(v[0]), Y(v[0])}, p1[2] = {X(v[1]), Y(v[1])}, p2[2] = {X(v[2]), Y(v[2])};
    const double e12x = p1[0] - p0[0], e12y = p1[1] - p0[1], e23x = p2[0] - p1[0], e23y = p2[1] - p1[1];
    const double e31x = p0[0] - p2[0], e31y = p0[1] - p2[1];
    const double f1 = z[v[0]], f2 = z[v[1]], f3 = z[v[2]];
    const double* d0 = grad + 2 * (size_t)v[0];
    const double* d1 = grad + 2 * (size_t)v[1];
    const double* d2 = grad + 2 * (size_t)v[2];
    const double df12 = +(d0[0] * e12x + d0[1] * e12y), df21 = -(d1[0] * e12x + d1[1] * e12y);
    const double df23 = +(d1[0] * e23x + d1[1] * e23y), df32 = -(d2[0] * e23x + d2[1] * e23y);
    const double df31 = +(d2[0] * e31x + d2[1] * e31y), df13 = -(d0[0] * e31x + d0[1] * e31y);
    const double c3000 = f1, c0300 = f2, c0030 = f3;
    const double c2100 = (df12 + 3 * c3000) / 3, c2010 = (df13 + 3 * c3000) / 3;
    const double c1200 = (df21 + 3 * c0300) / 3, c0210 = (df23 + 3 * c0300) / 3;
    const double c1020 = (df31 + 3 * c0030) / 3, c0120 = (df32 + 3 * c0030) / 3;
    const double c2001 = (c2100 + c2010 + c3000) / 3, c0201 = (c1200 + c0300 + c0210) / 3;
    const double c0021 = (c1020 + c0120 + c0030) / 3;
    double g[3] = {-0.5, -0.5, -0.5};
    const double a = (p1[0] - p0[0]) * (p2[1] - p0[1]) - (p1[1] - p0[1]) * (p2[0] - p0[0]);
    for (int k = 0; k < 3; k++) {
      const int o = nb[3 * t + k];
      if (o < 0) continue;
      const int* w = &tri[3 * o];
      const double s[2] = {X(w[0]) + X(w[1]) + X(w[2]), Y(w[0]) + Y(w[1]) + Y(w[2])};     // 3 x the centroid
      const double q[3][2] = {{3 * p0[0], 3 * p0[1]}, {3 * p1[0], 3 * p1[1]}, {3 * p2[0], 3 * p2[1]}};
      const double l0 = (q[1][0] - s[0]) * (q[2][1] - s[1]) - (q[1][1] - s[1]) * (q[2][0] - s[0]);
      const double l1 = (q[2][0] - s[0]) * (q[0][1] - s[1]) - (q[2][1] - s[1]) * (q[0][0] - s[0]);
      const double l2 = (q[0][0] - s[0]) * (q[1][1] - s[1]) - (q[0][1] - s[1]) * (q[1][0] - s[0]);
      const double c[3] = {l0 / (9 * a), l1 / (9 * a), l2 / (9 * a)};
      if (k == 0) g[k] = (2 * c[2] + c[1] - 1) / (2 - 3 * c[2] - 3 * c[1]);
      else if (k == 1) g[k] = (2 * c[0] + c[2] - 1) / (2 - 3 * c[0] - 3 * c[2]);
      else g[k] = (2 * c[1] + c[0] - 1) / (2 - 3 * c[1] - 3 * c[0]);
    }
    const double c0111 = (g[0] * (-c0300 + 3 * c0210 - 3 * c0120 + c0030) + (-c0300 + 2 * c0210 - c0120 + c0021 + c0201)) / 2;
    const double c1011 = (g[1] * (-c0030 + 3 * c1020 - 3 * c2010 + c3000) + (-c0030 + 2 * c1020 - c2010 + c2001 + c0021)) / 2;
    const double c1101 = (g[2] * (-c3000 + 3 * c2100 - 3 * c1200 + c0300) + (-c3000 + 2 * c2100 - c1200 + c2001 + c0201)) / 2;
    const double c1002 = (c1101 + c1011 + c2001) / 3, c0102 = (c1101 + c0111 + c0201) / 3;
    const double c0012 = (c1011 + c0111 + c0021) / 3, c0003 = (c1002 + c0102 + c0012) / 3;
    const double all[INIT_CT] = {c3000, c0300, c0030, c2100, c2010, c1200, c0210, c1020, c0120, c2001,
                                 c0201, c0021, c0111, c1011, c1101, c1002, c0102, c0012, c0003};
    memcpy(out + (size_t)INIT_CT * t, all, sizeof(all));
  }
}

// CSR lists of the triangles whose bounding box meets each INIT_TILE x INIT_TILE tile, in ascending triangle order
inline void bin_tiles(int W, const std::vector<long long>& xy, const std::vector<int>& tri, std::vector<int>& off,
                      std::vector<int>& list) {
  const int tx = (W + INIT_TILE - 1) / INIT_TILE, T = (int)(tri.size() / 3);
  off.assign((size_t)tx * tx + 1, 0);
  list.clear();
  for (int pass = 0; pass < 2; pass++) {
    std::vector<int> fill(off.begin(), off.end() - 1);
    if (pass) list.resize(off.back());
    for (int t = 0; t < T; t++) {
      long long lo[2] = {LLONG_MAX, LLONG_MAX}, hi[2] = {LLONG_MIN, LLONG_MIN};
      for (int k = 0; k < 3; k++)
        for (int d = 0; d < 2; d++) {
          lo[d] = std::min(lo[d], xy[2 * tri[3 * t + k] + d]);
          hi[d] = std::max(hi[d], xy[2 * tri[3 * t + k] + d]);
        }
      if (hi[0] < 0 || hi[1] < 0 || lo[0] >= W || lo[1] >= W) continue;
      const int r0 = (int)std::max(lo[0], 0ll) / INIT_TILE, r1 = (int)std::min(hi[0], (long long)W - 1) / INIT_TILE;
      const int c0 = (int)std::max(lo[1], 0ll) / INIT_TILE, c1 = (int)std::min(hi[1], (long long)W - 1) / INIT_TILE;
      for (int r = r0; r <= r1; r++)
        for (int c = c0; c <= c1; c++) {
          if (pass) list[fill[r * tx + c]++] = t;
          else off[r * tx + c + 1]++;
        }
    }
    if (!pass)
      for (size_t k = 1; k < off.size(); k++) off[k] += off[k - 1];
  }
}

}  // namespace init_host

// ---- kernels ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }

// the cubic Bezier patch over one sub-triangle at (u, v, w), w for the centroid; ordinates A..J as in
// tests/initialize_oracle.py _bezier, in its operation order
__device__ __forceinline__ double bezier(double u, double v, double w, const double* c, int A, int B, int Cc, int D, int E,
                                         int F, int G, int H, int I) {
  const double uu = dm(u, u), vv = dm(v, v), ww = dm(w, w);
  double s = dm(dm(uu, u), c[A]);
  s = da(s, dm(dm(dm(3.0, uu), v), c[B]));
  s = da(s, dm(dm(dm(3.0, u), vv), c[Cc]));
  s = da(s, dm(dm(vv, v), c[D]));
  s = da(s, dm(dm(dm(3.0, uu), w), c[E]));
  s = da(s, dm(dm(dm(dm(6.0, u), v), w), c[F]));
  s = da(s, dm(dm(dm(3.0, vv), w), c[G]));
  s = da(s, dm(dm(dm(3.0, u), ww), c[H]));
  s = da(s, dm(dm(dm(3.0, v), ww), c[I]));
  return da(s, dm(dm(ww, w), c[18]));
}

// Linear (CUBIC false) or Clough-Tocher (CUBIC true): one CTA per tile stages the tile's triangle list in shared memory;
// each cell takes the lowest-index triangle that holds it (closed, exact orientation tests), evaluates in fp64 and
// stores fp32.  Cells outside every triangle keep what they hold (the cleared map).
template <typename D, bool CUBIC>
__global__ void __launch_bounds__(INIT_THREADS) k_init_interp(const InitArgs a, float* __restrict__ map) {
  __shared__ int s_xy[INIT_CHUNK][6];
  __shared__ int s_id[INIT_CHUNK];
  const int tile = blockIdx.x, i0 = (tile / a.tiles_x) * INIT_TILE, j = (tile % a.tiles_x) * INIT_TILE + (threadIdx.x & 31);
  const int row = threadIdx.x >> 5;
  int owner[INIT_TILE / 8];
#pragma unroll
  for (int r = 0; r < INIT_TILE / 8; r++) owner[r] = -1;
  const int beg = a.tile_off[tile], end = a.tile_off[tile + 1];
  for (int base = beg; base < end; base += INIT_CHUNK) {
    const int m = min(INIT_CHUNK, end - base);
    __syncthreads();
    for (int t = threadIdx.x; t < m; t += INIT_THREADS) {
      const int id = a.tile_tri[base + t];
      s_id[t] = id;
#pragma unroll
      for (int k = 0; k < 6; k++) s_xy[t][k] = a.txy[6 * (size_t)id + k];
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < INIT_TILE / 8; r++) {
      const D ci = i0 + row + 8 * r, cj = j;
      if (owner[r] >= 0 || ci >= a.W || cj >= a.W) continue;
      for (int t = 0; t < m; t++) {
        const int* p = s_xy[t];
        if (orient2<D>(p[2], p[3], p[4], p[5], ci, cj) >= 0 && orient2<D>(p[4], p[5], p[0], p[1], ci, cj) >= 0 &&
            orient2<D>(p[0], p[1], p[2], p[3], ci, cj) >= 0) {
          owner[r] = s_id[t];
          break;
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < INIT_TILE / 8; r++) {
    if (owner[r] < 0) continue;
    const int ci = i0 + row + 8 * r, t = owner[r];
    const int* p = a.txy + 6 * (size_t)t;
    const D o0 = orient2<D>(p[2], p[3], p[4], p[5], ci, j), o1 = orient2<D>(p[4], p[5], p[0], p[1], ci, j);
    const D o2 = orient2<D>(p[0], p[1], p[2], p[3], ci, j);
    const double s = to_double(o0 + o1 + o2);
    const double b0 = __ddiv_rn(to_double(o0), s), b1 = __ddiv_rn(to_double(o1), s), b2 = __ddiv_rn(to_double(o2), s);
    double v;
    if (!CUBIC) {
      const double* z = a.coef + 3 * (size_t)t;
      v = da(da(dm(b0, z[0]), dm(b1, z[1])), dm(b2, z[2]));
    } else {
      const double* c = a.coef + (size_t)INIT_CT * t;
      const double mn = fmin(fmin(b0, b1), b2);
      const double e1 = b0 - mn, e2 = b1 - mn, e3 = b2 - mn, e4 = dm(3.0, mn);
      // ordinate indices: tests/initialize_oracle.py CT_NAMES
      if (b0 == mn) v = bezier(e2, e3, e4, c, 1, 6, 8, 2, 10, 12, 11, 16, 17);
      else if (b1 == mn) v = bezier(e3, e1, e4, c, 2, 7, 4, 0, 11, 13, 9, 17, 15);
      else v = bezier(e1, e2, e4, c, 0, 3, 5, 1, 9, 14, 10, 15, 16);
    }
    if (isnan(v)) continue;
    const size_t cell = (size_t)ci * a.W + j;
    map[cell] = (float)v;
    map[a.C + cell] = a.var;
    map[2 * (size_t)a.C + cell] = 1.f;
  }
}

template <typename D>
__device__ __forceinline__ D dmin(D a, D b) { return b < a ? b : a; }
template <typename D>
__device__ __forceinline__ D dmax(D a, D b) { return b > a ? b : a; }

// Nearest: per tile, the least over all points of the greatest squared distance to the tile bounds the candidates
// (a point whose least distance to the tile is above it is never nearest there); candidates are staged in shared
// memory and each cell keeps the least squared distance, the lowest input index on a tie.
template <typename D>
__global__ void __launch_bounds__(INIT_THREADS) k_init_nearest(const InitArgs a, float* __restrict__ map) {
  __shared__ D s_red[INIT_THREADS];
  __shared__ int s_n;
  __shared__ int s_i[INIT_THREADS], s_x[INIT_THREADS], s_y[INIT_THREADS];
  const int tile = blockIdx.x, i0 = (tile / a.tiles_x) * INIT_TILE, j0 = (tile % a.tiles_x) * INIT_TILE;
  const int i1 = min(i0 + INIT_TILE, a.W) - 1, j1 = min(j0 + INIT_TILE, a.W) - 1;
  const int j = j0 + (threadIdx.x & 31), row = threadIdx.x >> 5;
  auto far2 = [&](int2 p) {
    const D dx = dmax((D)p.x - i0, (D)i1 - p.x), dy = dmax((D)p.y - j0, (D)j1 - p.y);
    return dx * dx + dy * dy;
  };
  auto near2 = [&](int2 p) {
    const D dx = p.x < i0 ? (D)i0 - p.x : (p.x > i1 ? (D)p.x - i1 : (D)0);
    const D dy = p.y < j0 ? (D)j0 - p.y : (p.y > j1 ? (D)p.y - j1 : (D)0);
    return dx * dx + dy * dy;
  };
  D bound = far2(a.pxy[0]);
  for (int k = threadIdx.x; k < a.n; k += INIT_THREADS) bound = dmin(bound, far2(a.pxy[k]));
  s_red[threadIdx.x] = bound;
  for (int h = INIT_THREADS / 2; h > 0; h >>= 1) {
    __syncthreads();
    if (threadIdx.x < h) s_red[threadIdx.x] = dmin(s_red[threadIdx.x], s_red[threadIdx.x + h]);
  }
  __syncthreads();
  bound = s_red[0];
  D best[INIT_TILE / 8];
  int bi[INIT_TILE / 8];
#pragma unroll
  for (int r = 0; r < INIT_TILE / 8; r++) { best[r] = 0; bi[r] = -1; }
  for (int base = 0; base < a.n; base += INIT_THREADS) {
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const int k = base + threadIdx.x;
    if (k < a.n) {
      const int2 p = a.pxy[k];
      if (near2(p) <= bound) {
        const int slot = atomicAdd(&s_n, 1);
        s_i[slot] = k; s_x[slot] = p.x; s_y[slot] = p.y;
      }
    }
    __syncthreads();
    const int m = s_n;
#pragma unroll
    for (int r = 0; r < INIT_TILE / 8; r++) {
      const D ci = i0 + row + 8 * r;
      for (int c = 0; c < m; c++) {
        const D dx = ci - s_x[c], dy = (D)j - s_y[c];
        const D d = dx * dx + dy * dy;
        if (bi[r] < 0 || d < best[r] || (d == best[r] && s_i[c] < bi[r])) { best[r] = d; bi[r] = s_i[c]; }
      }
    }
  }
  if (j > j1) return;
#pragma unroll
  for (int r = 0; r < INIT_TILE / 8; r++) {
    const int ci = i0 + row + 8 * r;
    if (ci > i1) continue;
    const size_t cell = (size_t)ci * a.W + j;
    map[cell] = a.pz[bi[r]];
    map[a.C + cell] = a.var;
    map[2 * (size_t)a.C + cell] = 1.f;
  }
}
