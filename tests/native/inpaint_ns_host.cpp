// tests/native/inpaint_ns_host.cpp -- TEST HELPER: replays the device's Navier-Stokes inpainting (csrc/emap_inpaint.cuh,
// ip_eval_child_ns / ip_eval_child_ns_fast, the same inline functions k_ip_march<IP_NS> calls) on the CPU, one "thread"
// at a time with the kernel's pass structure, so that the NS estimate on the shared round / event-order machinery can be
// pinned against cv2.inpaint(INPAINT_NS) and tests/ns_inpaint_oracle.py without a GPU.  Any H x W image, H, W >= 1.
//   build: g++ -O2 -ffp-contract=off -shared -fPIC -o tests/native/_build/libinpaint_ns_host.so tests/native/inpaint_ns_host.cpp
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../elevation_mapping_cupy_b200/csrc/emap_inpaint.cuh"

// max_jacobi < 0: the border-aware evaluation everywhere (cross-check of the two paths)
extern "C" int inpaint_ns_host(const uint8_t* img_in, const uint8_t* mask, int H, int W, uint8_t* out, int max_jacobi,
                               int* rounds_out, int* max_iters_out, int* not_converged_out) {
  const bool use_fast = max_jacobi >= 0;
  if (max_jacobi < 0) max_jacobi = -max_jacobi;
  const int rows = H + 2, cols = W + 2, N = rows * cols;
  std::vector<uint8_t> f(N, IP_KNOWN), ck(N, 0), vc0(N, 0), vc1(N, 0), img(img_in, img_in + (size_t)H * W);
  std::vector<float> T(N, IP_TBIG), Tc0(N, 0.f), Tc1(N, 0.f);
  std::vector<uint32_t> ord(N, IP_ROOT), em(N, 0u);
  InpaintView v{rows, cols, f.data(), T.data(), ord.data(), img.data(), ck.data(), {Tc0.data(), Tc1.data()}, {vc0.data(), vc1.data()}, em.data()};
  // k_ip_image_init, k_ip_band, k_ip_band_flag
  for (int i = 1; i < rows - 1; i++)
    for (int j = 1; j < cols - 1; j++)
      if (mask[(i - 1) * W + (j - 1)]) f[i * cols + j] = IP_INSIDE;
  std::vector<int> band;
  for (int i = 1; i < rows - 1; i++)
    for (int j = 1; j < cols - 1; j++) {
      const int p = i * cols + j;
      if (f[p] != IP_KNOWN) continue;
      if (f[p - cols] == IP_INSIDE || f[p + cols] == IP_INSIDE || f[p - 1] == IP_INSIDE || f[p + 1] == IP_INSIDE) band.push_back(p);
    }
  for (int p : band) { f[p] = IP_BAND; T[p] = 0.f; }
  std::vector<int> heap(band), children;
  int round = 0, max_iters = 0, not_conv = 0;
  while (!heap.empty()) {
    round++;
    float tcur = IP_TBIG * 4;
    for (int p : heap) tcur = std::min(tcur, T[p]);
    // pass A: children of the round (claimed), then their first poppers
    children.clear();
    for (int q : heap) {
      if (!ip_in_round(v, q, tcur)) continue;
      const int nb[4] = {q - cols, q - 1, q + cols, q + 1};
      for (int k = 0; k < 4; k++) {
        const int c = nb[k];
        const int ci = c / cols, cj = c - ci * cols;
        if (ci <= 0 || cj <= 0 || ci >= rows - 1 || cj >= cols - 1) continue;
        if (f[c] == IP_INSIDE) { f[c] = IP_CHILD; children.push_back(c); }
      }
    }
    for (int c : children) {
      ck[c] = (uint8_t)ip_find_popper(v, c, tcur);
      Tc0[c] = IP_TBIG; vc0[c] = 0; Tc1[c] = IP_TBIG; vc1[c] = 0;
    }
    // Jacobi iterations to the fixed point
    int cur = 0, it = 0;
    for (;; it++) {
      bool changed = false;
      for (int c : children) {
        float t; uint8_t val;
        if (use_fast && ip_interior(v, c)) changed |= ip_eval_child_ns_fast(v, c, cur, it == 0, &t, &val);
        else changed |= ip_eval_child_ns(v, c, cur, &t, &val);
        v.Tc[cur ^ 1][c] = t; v.vc[cur ^ 1][c] = val;
      }
      cur ^= 1;
      if (!changed) break;
      if (it + 1 >= max_jacobi) { not_conv++; break; }
    }
    max_iters = std::max(max_iters, it + 1);
    // commit
    std::vector<int> next;
    for (int q : heap) {
      if (ip_in_round(v, q, tcur)) f[q] = IP_KNOWN; else next.push_back(q);
    }
    for (int c : children) {
      T[c] = v.Tc[cur][c];
      const int ci = c / cols, cj = c - ci * cols;
      img[(ci - 1) * W + (cj - 1)] = v.vc[cur][c];
      ord[c] = ((uint32_t)round << 3) | ck[c];
    }
    for (int c : children) { f[c] = IP_BAND; next.push_back(c); }
    heap.swap(next);
  }
  memcpy(out, img.data(), (size_t)H * W);
  if (rounds_out) *rounds_out = round;
  if (max_iters_out) *max_iters_out = max_iters;
  if (not_converged_out) *not_converged_out = not_conv;
  return 0;
}
