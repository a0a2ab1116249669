// tests/native/regions_host.cpp -- TEST HELPER: the border-start rule, the border following and CHAIN_APPROX_SIMPLE's
// compression of csrc/emap_regions.cuh (the same inline functions the kernels call) compiled for the CPU, over a
// sequential union-find, so that they can be checked against cv2.findContours(RETR_CCOMP, CHAIN_APPROX_SIMPLE).
//   build: g++ -O2 -shared -fPIC -I<cuda>/include -o tests/native/_build/libregions_host.so tests/native/regions_host.cpp
#include <algorithm>
#include <vector>

#include "../../elevation_mapping_cupy_b200/csrc/emap_regions.cuh"

namespace {

int find(std::vector<int>& p, int a) {
  while (p[a] != a) a = p[a] = p[p[a]];
  return a;
}

void unite(std::vector<int>& p, int a, int b) {
  a = find(p, a);
  b = find(p, b);
  if (a != b) p[std::max(a, b)] = std::min(a, b);
}

struct Nz {
  const unsigned char* img;
  int rows, cols;
  bool operator()(int x, int y) const { return x >= 0 && y >= 0 && x < cols && y < rows && img[y * cols + x]; }
};

struct Collect {
  std::vector<int>* xy;
  void operator()(int x, int y) {
    xy->push_back(x);
    xy->push_back(y);
  }
};

}  // namespace

// The contours of a rows x cols 0/1 image in the order the kernels emit them: top-level contours by start pixel
// descending, each followed by its holes by start pixel descending.  Writes per contour (parent, n_points) into meta
// (parent -1 for an outer, else the index of its outer) and the points as (x, y) into xy; returns the number of
// contours (-1: a capacity is too small).
extern "C" int regions_contours(const unsigned char* img, int rows, int cols, int* meta, int meta_cap, int* xy,
                                int xy_cap, int* ellipse_half, int margin) {
  const int n = rows * cols;
  std::vector<int> p(n + 1);
  for (int i = 0; i <= n; i++) p[i] = i;
  for (int i = 0; i < n; i++) {
    const int y = i / cols, x = i % cols;
    const bool v = img[i];
    if (x > 0 && (bool)img[i - 1] == v) unite(p, i, i - 1);
    if (y > 0) {
      if ((bool)img[i - cols] == v) unite(p, i, i - cols);
      if (v && x > 0 && img[i - cols - 1]) unite(p, i, i - cols - 1);
      if (v && x + 1 < cols && img[i - cols + 1]) unite(p, i, i - cols + 1);
    }
    if (!v && (x == 0 || y == 0 || x == cols - 1 || y == rows - 1)) unite(p, i, n);
  }
  for (int i = 0; i <= n; i++) p[i] = find(p, i);
  std::vector<int> outers, holes;
  for (int i = 0; i < n; i++) {
    const int x = i % cols;
    const bool r = x + 1 < cols;
    const int k = rg_start(i, img[i], p[i], r, r && img[i + 1], r ? p[i + 1] : -1, p[n]);
    if (k == 1) outers.push_back(i);
    if (k == 2) holes.push_back(i);
  }
  std::reverse(outers.begin(), outers.end());
  std::reverse(holes.begin(), holes.end());
  Nz nz{img, rows, cols};
  int nc = 0, nxy = 0;
  std::vector<int> pts;
  auto emit = [&](int start, bool hole, int parent) {
    pts.clear();
    Collect c{&pts};
    const int np = rg_trace(nz, start % cols, start / cols, hole, c);
    if (nc >= meta_cap || nxy + (int)pts.size() > xy_cap || np * 2 != (int)pts.size()) return false;
    meta[2 * nc] = parent;
    meta[2 * nc + 1] = np;
    std::copy(pts.begin(), pts.end(), xy + nxy);
    nxy += (int)pts.size();
    nc++;
    return true;
  };
  for (int o : outers) {
    const int me = nc;
    if (!emit(o, false, -1)) return -1;
    for (int h : holes)
      if (p[h] == o && !emit(h, true, me)) return -1;
  }
  for (int r = 0; r <= 2 * (1 + margin); r++) ellipse_half[r] = rg_ellipse_half(1 + margin, r);
  return nc;
}

// rg_src for every upsampled index of a size-m source.
extern "C" void regions_src(int m, int* out) {
  for (int u = 0; u < 3 * m - 2; u++) out[u] = rg_src(u, m);
}
