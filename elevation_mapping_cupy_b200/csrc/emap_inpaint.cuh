// emap_inpaint.cuh -- plugins/inpainting.py:53-63 on the device: OpenCV's Telea inpainting (radius 1, one channel) as a
// PARALLEL discrete-event replay of its fast-marching sweep.
//
// cv2.inpaint(INPAINT_TELEA) pops pixels from a priority queue ordered by (T, push order) and fills each unknown
// 4-neighbour of the popped pixel once, from whatever is known at that moment -- a sequential algorithm whose result
// depends on the pop order.  The order is nevertheless LOCALLY determined:
//   * a pixel filled when q is popped gets T > T(q) + 0.707 (the eikonal update adds at least 1/sqrt(2) to the smallest
//     known neighbour, and q -- the first neighbour to be popped -- is the smallest), so all queue entries with
//     T in [Tmin, Tmin + 0.7) are popped before any pixel they create: one ROUND handles them together;
//   * inside a round, the event "c is filled" happens at key E(c) = (T(q), S(q), k) of its first popper q (k = which
//     neighbour of q it is); a neighbour x of c is known at that moment iff it was known before the round or is itself
//     filled in this round with E(x) < E(c);
//   * push order S is (round, E) -- comparable between two pixels by walking their popper chains.
// Every pixel of a round is evaluated concurrently; pixels that depend on earlier pixels of the same round (chains
// along the front) are iterated to their fixed point (Jacobi), which reproduces the sequential result exactly.
// The arithmetic below follows inpaint.cpp (icvTeleaInpaintFMM / FastMarching_solve) operation for operation, with
// the float / double widths the x86-64 build uses; it is pinned against cv2 4.x by the tests (which also hold a sequential
// restatement of the OpenCV routine).  Host code may include this header: tests/native/inpaint_host.cpp replays the same
// rounds on the CPU with these very functions.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#if defined(__CUDACC__)
#define IP_HD __host__ __device__ __forceinline__
#else
#define IP_HD inline
#endif

enum { IP_KNOWN = 0, IP_BAND = 1, IP_INSIDE = 2, IP_CHILD = 3 };
#define IP_TBIG 1.0e6f
#define IP_DELTA 0.70f            // round width in T; must stay below 1/sqrt(2)
#define IP_ROOT 4                 // ord.k of an initial band pixel (no popper)
#define IP_CMP_DEPTH 24            // popper-chain levels walked on a (T, round) tie before falling back to the pixel index;
                                   // random images need the deep walk (a cap of 2 changes results), regular fronts tie all the way

struct InpaintView {
  int rows, cols;                 // padded: image is (rows-2) x (cols-2), pixel (i,j) of the image = padded (i+1, j+1)
  uint8_t* f;                     // [rows*cols] IP_* state
  float* T;                       // [rows*cols]
  uint32_t* ord;                  // [rows*cols] push order of a queue pixel: round << 3 | k
  uint8_t* img;                   // [(rows-2)*(cols-2)] the 8-bit image being filled
  // children of the running round (valid where f == IP_CHILD)
  uint8_t* ck;                    // popper direction k of the child (0: popper is below, 1: right, 2: above, 3: left)
  float* Tc[2];                   // double-buffered T iterate
  uint8_t* vc[2];                 // double-buffered value iterate
  uint32_t* em;                   // [rows*cols] per interior child: which of its 12 stencil pixels are known at its event
                                  // (bits 0..12) / are same-round children filled EARLIER (bits 16..28); see ip_child_masks
};

// no FMA contraction anywhere: the reference build is plain SSE2
#if defined(__CUDA_ARCH__)
#define IP_FMUL(a, b) __fmul_rn((a), (b))
#define IP_FADD(a, b) __fadd_rn((a), (b))
#define IP_FSUB(a, b) __fsub_rn((a), (b))
#define IP_FDIV(a, b) __fdiv_rn((a), (b))
#define IP_DMUL(a, b) __dmul_rn((a), (b))
#define IP_DADD(a, b) __dadd_rn((a), (b))
#define IP_DSUB(a, b) __dsub_rn((a), (b))
#define IP_DDIV(a, b) __ddiv_rn((a), (b))
#define IP_DSQRT(a) __dsqrt_rn((a))
#define IP_FSQRT(a) __fsqrt_rn((a))
#else
#define IP_FMUL(a, b) ((float)((float)(a) * (float)(b)))
#define IP_FADD(a, b) ((float)((float)(a) + (float)(b)))
#define IP_FSUB(a, b) ((float)((float)(a) - (float)(b)))
#define IP_FDIV(a, b) ((float)((float)(a) / (float)(b)))
#define IP_DMUL(a, b) ((double)(a) * (double)(b))
#define IP_DADD(a, b) ((double)(a) + (double)(b))
#define IP_DSUB(a, b) ((double)(a) - (double)(b))
#define IP_DDIV(a, b) ((double)(a) / (double)(b))
#define IP_DSQRT(a) sqrt((double)(a))
#define IP_FSQRT(a) sqrtf((float)(a))
#endif

// popper of a child with direction k (the popped pixel q saw the child as its k-th neighbour: up, left, down, right)
IP_HD int ip_popper(int cols, int p, int k) {
  return k == 0 ? p + cols : k == 1 ? p + 1 : k == 2 ? p - cols : p - 1;
}

// strict order of two QUEUE pixels (f == BAND, before or while they are popped): (T, push order)
IP_HD bool ip_key_less(const InpaintView& v, int a, int b) {
  // T and push order of a level are fetched together: one memory round trip per level of the popper chains
  const float ta = v.T[a], tb = v.T[b];
  uint32_t oa = v.ord[a], ob = v.ord[b];
  if (ta != tb) return ta < tb;
  for (int depth = 0; depth < IP_CMP_DEPTH; depth++) {
    if (a == b) return false;
    const uint32_t ra = oa >> 3, rb = ob >> 3;
    if (ra != rb) return ra < rb;                                 // pushed in an earlier round
    const int ka = (int)(oa & 7u), kb = (int)(ob & 7u);
    if (ka == IP_ROOT || kb == IP_ROOT) return a < b;             // initial band: row-major (both are roots: same round 0)
    const int qa = ip_popper(v.cols, a, ka), qb = ip_popper(v.cols, b, kb);
    if (qa == qb) return ka < kb;
    const float tqa = v.T[qa], tqb = v.T[qb];
    const uint32_t oqa = v.ord[qa], oqb = v.ord[qb];
    if (tqa != tqb) return tqa < tqb;
    a = qa; b = qb; oa = oqa; ob = oqb;                           // same T: their own push order decides
  }
  return a < b;
}

// event order of two CHILDREN of the running round (popper directions in v.ck)
IP_HD bool ip_event_less(const InpaintView& v, int c1, int c2) {
  const int k1 = v.ck[c1], k2 = v.ck[c2];
  const int q1 = ip_popper(v.cols, c1, k1), q2 = ip_popper(v.cols, c2, k2);
  if (q1 == q2) return k1 < k2;
  return ip_key_less(v, q1, q2);
}

// is queue pixel q popped in the round that starts at tcur?
IP_HD bool ip_in_round(const InpaintView& v, int q, float tcur) { return v.f[q] == IP_BAND && v.T[q] < tcur + IP_DELTA; }

// First popper of an INSIDE pixel p in this round: direction k (0..3) or -1 if none of its neighbours is popped.
IP_HD int ip_find_popper(const InpaintView& v, int p, float tcur) {
  int best = -1, bq = -1;
  for (int k = 0; k < 4; k++) {
    const int q = ip_popper(v.cols, p, k);
    if (!ip_in_round(v, q, tcur)) continue;
    // between two poppers the earlier key wins; the same popper cannot appear twice
    if (best < 0 || ip_key_less(v, q, bq)) { best = k; bq = q; }
  }
  return best;
}

struct IpNb { bool known; float T; };

// state of pixel x as child c sees it at the moment c is filled; `cur` selects the iterate of same-round children
IP_HD IpNb ip_at_event(const InpaintView& v, int c, int x, int cur) {
  IpNb n;
  const uint8_t fx = v.f[x];
  if (fx == IP_KNOWN || fx == IP_BAND) { n.known = true; n.T = v.T[x]; return n; }
  if (fx == IP_CHILD && x != c && ip_event_less(v, x, c)) { n.known = true; n.T = v.Tc[cur][x]; return n; }
  n.known = false; n.T = IP_TBIG;
  return n;
}

IP_HD float ip_solve(const IpNb& n1, const IpNb& n2) {           // FastMarching_solve
  const double a11 = (double)n1.T, a22 = (double)n2.T;
  const double m12 = a11 < a22 ? a11 : a22;
  double sol;
  if (n1.known) {
    if (n2.known) {
      const double d = IP_DSUB(a11, a22);
      if (fabs(d) >= 1.0) sol = IP_DADD(1.0, m12);
      else sol = IP_DMUL(IP_DADD(IP_DADD(a11, a22), IP_DSQRT(IP_DSUB(2.0, IP_DMUL(d, d)))), 0.5);
    } else sol = IP_DADD(1.0, a11);
  } else if (n2.known) sol = IP_DADD(1.0, a22);
  else sol = IP_DADD(1.0, m12);
  return (float)sol;
}

// value of image pixel (padded coordinates) as seen at c's event: same-round EARLIER children read their iterate,
// everything else the image (for a pixel not yet filled that is its original content, which the reference also reads
// through its shifted border indices)
IP_HD int ip_val(const InpaintView& v, int c, int prow, int pcol, int cur) {
  const int x = prow * v.cols + pcol;
  if (v.f[x] == IP_CHILD && x != c && ip_event_less(v, x, c)) return v.vc[cur][x];
  return v.img[(prow - 1) * (v.cols - 2) + (pcol - 1)];
}

// One evaluation of child c (padded index): new T and value from the state at its event.  Returns true if either
// differs from the current iterate.
IP_HD bool ip_eval_child(const InpaintView& v, int c, int cur, float* t_out, uint8_t* val_out) {
  const int cols = v.cols, rows = v.rows;
  const int i = c / cols, j = c - i * cols;
  const IpNb up = ip_at_event(v, c, c - cols, cur), dn = ip_at_event(v, c, c + cols, cur);
  const IpNb lf = ip_at_event(v, c, c - 1, cur), rt = ip_at_event(v, c, c + 1, cur);
  float dist = ip_solve(up, lf);
  { const float d2 = ip_solve(dn, lf); if (d2 < dist) dist = d2; }
  { const float d3 = ip_solve(up, rt); if (d3 < dist) dist = d3; }
  { const float d4 = ip_solve(dn, rt); if (d4 < dist) dist = d4; }
  // gradT
  float gtx, gty;
  if (rt.known) gtx = lf.known ? IP_FMUL(IP_FSUB(rt.T, lf.T), 0.5f) : IP_FSUB(rt.T, dist);
  else gtx = lf.known ? IP_FSUB(dist, lf.T) : 0.f;
  if (dn.known) gty = up.known ? IP_FMUL(IP_FSUB(dn.T, up.T), 0.5f) : IP_FSUB(dn.T, dist);
  else gty = up.known ? IP_FSUB(dist, up.T) : 0.f;
  float Ia = 0.f, Jx = 0.f, Jy = 0.f, s = 1.0e-20f;
  // cross neighbours in the loop order of the reference: (i-1,j), (i,j-1), (i,j+1), (i+1,j)   [(i,j) itself is INSIDE]
  const int dk[4] = {-1, 0, 0, 1}, dl[4] = {0, -1, 1, 0};
  for (int n = 0; n < 4; n++) {
    const int k = i + dk[n], l = j + dl[n];
    if (!(k > 0 && l > 0 && k < rows - 1 && l < cols - 1)) continue;
    const IpNb& nb = (n == 0) ? up : (n == 1) ? lf : (n == 2) ? rt : dn;
    if (!nb.known) continue;
    const int km = k - 1 + (k == 1), kp = k - 1 - (k == rows - 2);
    const int lm = l - 1 + (l == 1), lp = l - 1 - (l == cols - 2);
    const float ry = (float)(i - k), rx = (float)(j - l);
    // |r| = 1: dst = 1 / (|r|^2 sqrt(|r|^2)) = 1
    const float lev = (float)IP_DDIV(1.0, IP_DADD(1.0, fabs(IP_DSUB((double)nb.T, (double)dist))));
    float dir = IP_FADD(IP_FMUL(rx, gtx), IP_FMUL(ry, gty));
    if (fabs((double)dir) <= 0.01) dir = 0.000001f;
    const float w = fabsf(IP_FMUL(lev, dir));
    // gradI at (k,l): its own neighbours as known at c's event; image rows/cols in UNPADDED coordinates (km, lm, ...)
    const int x = k * cols + l;
    const bool r_kn = ip_at_event(v, c, x + 1, cur).known, l_kn = ip_at_event(v, c, x - 1, cur).known;
    const bool d_kn = ip_at_event(v, c, x + cols, cur).known, u_kn = ip_at_event(v, c, x - cols, cur).known;
    float gix, giy;
    if (r_kn) {
      if (l_kn) gix = IP_FMUL((float)(ip_val(v, c, km + 1, lp + 2, cur) - ip_val(v, c, km + 1, lm, cur)), 2.0f);
      else gix = (float)(ip_val(v, c, km + 1, lp + 2, cur) - ip_val(v, c, km + 1, lm + 1, cur));
    } else gix = l_kn ? (float)(ip_val(v, c, km + 1, lp + 1, cur) - ip_val(v, c, km + 1, lm, cur)) : 0.f;
    if (d_kn) {
      if (u_kn) giy = IP_FMUL((float)(ip_val(v, c, kp + 2, lm + 1, cur) - ip_val(v, c, km, lm + 1, cur)), 2.0f);
      else giy = (float)(ip_val(v, c, kp + 2, lm + 1, cur) - ip_val(v, c, km + 1, lm + 1, cur));
    } else giy = u_kn ? (float)(ip_val(v, c, kp + 1, lm + 1, cur) - ip_val(v, c, km, lm + 1, cur)) : 0.f;
    Ia = IP_FADD(Ia, IP_FMUL(w, (float)ip_val(v, c, k, l, cur)));
    Jx = IP_FSUB(Jx, IP_FMUL(w, IP_FMUL(gix, rx)));
    Jy = IP_FSUB(Jy, IP_FMUL(w, IP_FMUL(giy, ry)));
    s = IP_FADD(s, w);
  }
  // all in float (sqrt resolves to its float overload, 1.0e-20f / 0.5f are float literals)
  const float jn = IP_FSQRT(IP_FADD(IP_FMUL(Jx, Jx), IP_FMUL(Jy, Jy)));
  const float sat = IP_FADD(IP_FADD(IP_FDIV(Ia, s), IP_FDIV(IP_FADD(Jx, Jy), IP_FADD(jn, 1.0e-20f))), 0.5f);
  // cv::saturate_cast<uchar>(float) = cvRound (nearest even) then clamp
  int iv;
  if (!(sat == sat)) iv = 0;
  else { const float rn = rintf(sat < -1.0e6f ? -1.0e6f : (sat > 1.0e6f ? 1.0e6f : sat)); iv = (int)rn; }
  iv = iv < 0 ? 0 : (iv > 255 ? 255 : iv);
  const bool changed = (dist != v.Tc[cur][c]) || ((uint8_t)iv != v.vc[cur][c]);
  *t_out = dist; *val_out = (uint8_t)iv;
  return changed;
}

// ---------------------------------------------------------------------------------------------
// Same evaluation for a child at least 3 pixels away from the image border (none of the reference's shifted border
// indices apply), written as GATHER-THEN-COMPUTE: the state of the 13 pixels within distance 2 is fetched with
// independent loads (two waves: the pixels, then the poppers of those that are children of this round), so that a
// device thread waits for a few memory round trips instead of a long chain of dependent ones.  Bit-identical to
// ip_eval_child by construction (same operations in the same order); the host harness cross-checks both.
//   stencil slots: 0 c | 1 up 2 left 3 right 4 down | 5 up-up 6 up-left 7 up-right 8 left-left 9 right-right
//                  10 down-left 11 down-right 12 down-down
IP_HD bool ip_interior(const InpaintView& v, int c) {
  const int i = c / v.cols, j = c - i * v.cols;
  return i >= 3 && j >= 3 && i <= v.rows - 4 && j <= v.cols - 4;
}

// Which pixels of c's stencil are known at c's event, and which of those are children of the same round filled earlier.
// The event order of a round is fixed once its children and their first poppers are chosen (pass A): it depends on the
// queue pixels only, not on the fixed-point iterate.  So the (possibly deep: popper-chain walks on T ties, which regular
// fronts produce all the time) comparisons are made ONCE per child and round, in the first fixed-point iteration, and
// cached in v.em; the later iterations read two bit masks.
IP_HD uint32_t ip_child_masks(const InpaintView& v, int c) {
  const int cols = v.cols;
  const int off[13] = {0, -cols, -1, 1, cols, -2 * cols, -cols - 1, -cols + 1, -2, 2, cols - 1, cols + 1, 2 * cols};
  uint8_t F[13], K[13];
#pragma unroll
  for (int n = 0; n < 13; n++) { const int x = c + off[n]; F[n] = v.f[x]; K[n] = v.ck[x]; }       // wave 1
  int Q[13]; float TQ[13]; uint32_t OQ[13];
#pragma unroll
  for (int n = 0; n < 13; n++) {                                   // wave 2: poppers of the children among them
    const bool ch = F[n] == IP_CHILD;
    Q[n] = ch ? ip_popper(cols, c + off[n], K[n]) : c;
    TQ[n] = v.T[Q[n]]; OQ[n] = v.ord[Q[n]];
  }
  uint32_t m = 0, tie = 0;
#pragma unroll
  for (int n = 1; n < 13; n++) {
    bool known = false, earlier = false;
    if (F[n] == IP_KNOWN || F[n] == IP_BAND) known = true;
    else if (F[n] == IP_CHILD) {
      // ip_event_less(x, c)
      if (Q[n] == Q[0]) earlier = K[n] < K[0];
      else if (TQ[n] != TQ[0]) earlier = TQ[n] < TQ[0];
      else if ((OQ[n] >> 3) != (OQ[0] >> 3)) earlier = (OQ[n] >> 3) < (OQ[0] >> 3);
      else tie |= 1u << n;                                         // equal T and round: the popper chains decide (below)
    }
    if (known || earlier) m |= 1u << n;
    if (earlier) m |= 1u << (16 + n);
  }
  if (tie) {
    // ip_key_less(Q[n], Q[0]) for every tied n AT ONCE: all comparisons share the chain of c's own popper, and the loads of
    // one level (T and push order of every chain's next popper) are independent -- one memory round trip per level for the
    // whole stencil instead of two per level and neighbour.  Operation for operation the loop of ip_key_less.
    int a[13]; uint32_t oa[13];
#pragma unroll
    for (int n = 1; n < 13; n++) { a[n] = Q[n]; oa[n] = OQ[n]; }
    int b = Q[0]; uint32_t ob = OQ[0];
    for (int depth = 0; depth < IP_CMP_DEPTH && tie; depth++) {
      const uint32_t rb = ob >> 3;
      const int kb = (int)(ob & 7u);
      const int qb = kb == IP_ROOT ? b : ip_popper(cols, b, kb);
      int qa[13];
#pragma unroll
      for (int n = 1; n < 13; n++) {
        qa[n] = b;
        if (!((tie >> n) & 1u)) continue;
        bool done = true, earlier = false;
        const uint32_t ra = oa[n] >> 3;
        const int ka = (int)(oa[n] & 7u);
        if (a[n] == b) earlier = false;
        else if (ra != rb) earlier = ra < rb;
        else if (ka == IP_ROOT || kb == IP_ROOT) earlier = a[n] < b;
        else {
          qa[n] = ip_popper(cols, a[n], ka);
          if (qa[n] == qb) earlier = ka < kb; else done = false;
        }
        if (done) { tie &= ~(1u << n); if (earlier) m |= (1u << n) | (1u << (16 + n)); }
      }
      if (!tie) break;
      const float tqb = v.T[qb]; const uint32_t oqb = v.ord[qb];
      float tqa[13]; uint32_t oqa[13];
#pragma unroll
      for (int n = 1; n < 13; n++) { tqa[n] = v.T[qa[n]]; oqa[n] = v.ord[qa[n]]; }            // one wave
#pragma unroll
      for (int n = 1; n < 13; n++) {
        if (!((tie >> n) & 1u)) continue;
        if (tqa[n] != tqb) { tie &= ~(1u << n); if (tqa[n] < tqb) m |= (1u << n) | (1u << (16 + n)); }
        else { a[n] = qa[n]; oa[n] = oqa[n]; }
      }
      b = qb; ob = oqb;
    }
#pragma unroll
    for (int n = 1; n < 13; n++)                                   // depth cap: the pixel index decides, as in ip_key_less
      if (((tie >> n) & 1u) && a[n] < b) m |= (1u << n) | (1u << (16 + n));
  }
  return m;
}

// `first`: this is the first fixed-point iteration of the round (compute and cache the masks of c).
IP_HD bool ip_eval_child_fast(const InpaintView& v, int c, int cur, bool first, float* t_out, uint8_t* val_out) {
  const int cols = v.cols, W = cols - 2;
  const int off[13] = {0, -cols, -1, 1, cols, -2 * cols, -cols - 1, -cols + 1, -2, 2, cols - 1, cols + 1, 2 * cols};
  uint8_t VC[13], IM[13];
  float TT[13], TC[13];
  const int ci = c / cols, cj = c - ci * cols;
  const int cimg = (ci - 1) * W + (cj - 1);
  const int offi[13] = {0, -W, -1, 1, W, -2 * W, -W - 1, -W + 1, -2, 2, W - 1, W + 1, 2 * W};
#pragma unroll
  for (int n = 0; n < 13; n++) {                                   // one wave of independent loads
    const int x = c + off[n];
    TT[n] = v.T[x]; TC[n] = v.Tc[cur][x]; VC[n] = v.vc[cur][x]; IM[n] = v.img[cimg + offi[n]];
  }
  uint32_t m;
  if (first) { m = ip_child_masks(v, c); v.em[c] = m; } else m = v.em[c];
  bool kn[13]; float Tn[13]; int val[13];
  kn[0] = false; Tn[0] = IP_TBIG; val[0] = IM[0];
#pragma unroll
  for (int n = 1; n < 13; n++) {
    const bool earlier = (m >> (16 + n)) & 1u;
    kn[n] = (m >> n) & 1u;
    Tn[n] = (kn[n] && !earlier) ? TT[n] : (earlier ? TC[n] : IP_TBIG);
    val[n] = earlier ? (int)VC[n] : (int)IM[n];
  }
  IpNb up, lf, rt, dn;
  up.known = kn[1]; up.T = Tn[1]; lf.known = kn[2]; lf.T = Tn[2]; rt.known = kn[3]; rt.T = Tn[3]; dn.known = kn[4]; dn.T = Tn[4];
  float dist = ip_solve(up, lf);
  { const float d2 = ip_solve(dn, lf); if (d2 < dist) dist = d2; }
  { const float d3 = ip_solve(up, rt); if (d3 < dist) dist = d3; }
  { const float d4 = ip_solve(dn, rt); if (d4 < dist) dist = d4; }
  float gtx, gty;
  if (rt.known) gtx = lf.known ? IP_FMUL(IP_FSUB(rt.T, lf.T), 0.5f) : IP_FSUB(rt.T, dist);
  else gtx = lf.known ? IP_FSUB(dist, lf.T) : 0.f;
  if (dn.known) gty = up.known ? IP_FMUL(IP_FSUB(dn.T, up.T), 0.5f) : IP_FSUB(dn.T, dist);
  else gty = up.known ? IP_FSUB(dist, up.T) : 0.f;
  float Ia = 0.f, Jx = 0.f, Jy = 0.f, s = 1.0e-20f;
  // per cross neighbour n (order up, left, right, down): slots of ITS left / right / up / down pixel, and r = c - n
  const int nL[4] = {6, 8, 0, 10}, nR[4] = {7, 0, 9, 11}, nU[4] = {5, 6, 7, 0}, nD[4] = {0, 10, 11, 12};
  const float rxs[4] = {0.f, 1.f, -1.f, 0.f}, rys[4] = {1.f, 0.f, 0.f, -1.f};
#pragma unroll
  for (int n = 0; n < 4; n++) {
    const int sl = n + 1;
    if (!kn[sl]) continue;
    const float rx = rxs[n], ry = rys[n];
    const float lev = (float)IP_DDIV(1.0, IP_DADD(1.0, fabs(IP_DSUB((double)Tn[sl], (double)dist))));
    float dir = IP_FADD(IP_FMUL(rx, gtx), IP_FMUL(ry, gty));
    if (fabs((double)dir) <= 0.01) dir = 0.000001f;
    const float w = fabsf(IP_FMUL(lev, dir));
    const bool r_kn = kn[nR[n]], l_kn = kn[nL[n]], d_kn = kn[nD[n]], u_kn = kn[nU[n]];
    float gix, giy;
    if (r_kn) gix = l_kn ? IP_FMUL((float)(val[nR[n]] - val[nL[n]]), 2.0f) : (float)(val[nR[n]] - val[sl]);
    else gix = l_kn ? (float)(val[sl] - val[nL[n]]) : 0.f;
    if (d_kn) giy = u_kn ? IP_FMUL((float)(val[nD[n]] - val[nU[n]]), 2.0f) : (float)(val[nD[n]] - val[sl]);
    else giy = u_kn ? (float)(val[sl] - val[nU[n]]) : 0.f;
    Ia = IP_FADD(Ia, IP_FMUL(w, (float)val[sl]));
    Jx = IP_FSUB(Jx, IP_FMUL(w, IP_FMUL(gix, rx)));
    Jy = IP_FSUB(Jy, IP_FMUL(w, IP_FMUL(giy, ry)));
    s = IP_FADD(s, w);
  }
  const float jn = IP_FSQRT(IP_FADD(IP_FMUL(Jx, Jx), IP_FMUL(Jy, Jy)));
  const float sat = IP_FADD(IP_FADD(IP_FDIV(Ia, s), IP_FDIV(IP_FADD(Jx, Jy), IP_FADD(jn, 1.0e-20f))), 0.5f);
  int iv;
  if (!(sat == sat)) iv = 0;
  else { const float rn = rintf(sat < -1.0e6f ? -1.0e6f : (sat > 1.0e6f ? 1.0e6f : sat)); iv = (int)rn; }
  iv = iv < 0 ? 0 : (iv > 255 ? 255 : iv);
  const bool changed = (dist != TC[0]) || ((uint8_t)iv != VC[0]);
  *t_out = dist; *val_out = (uint8_t)iv;
  return changed;
}

// ---------------------------------------------------------------------------------------------
// cv2.inpaint(INPAINT_NS) at radius 1 (icvNSInpaintFMM, one 8-bit channel).  The sweep is Telea's -- the same queue and
// the same FastMarching_solve T update, and at radius 1 Telea's march outside the mask covers no pixel -- so the rounds,
// children and event order above carry over unchanged; only the per-pixel estimate differs.  It reads T nowhere: each
// known 4-neighbour n of the filled pixel adds w * value(n) with w = dst * dir, dst = 1 / (|r|^4 + 1), and dir the
// alignment of r with n's image-gradient estimate (sums of absolute differences of its known 4-neighbours' values).
// Those neighbours lie within distance 2 of the filled pixel: the same 13-pixel stencil and cached event masks as Telea.
// Restated from the published routine and pinned against the cv2 binary by tests/test_inpaint_ns_cpu.py (the sequential
// restatement is tests/ns_inpaint_oracle.py).
enum { IP_TELEA = 0, IP_NS = 1 };

// One known neighbour n's term: r = (rx, ry) from the filled pixel to n; kd / ku / kr / kl: n's down / up / right / left
// pixel is known at the event.  The 8-bit values are the ones the reference reads: a, b, cc down the image column lm at
// rows kp+1, kp, km-1 (its gradI.x), d, e, g along the image row km at columns lp+1, lm, lm-1 (its gradI.y), and n's own
// value `val`.  Float arithmetic of the x86-64 build (sqrt and fabs resolve to their float overloads).
IP_HD void ip_ns_term(float rx, float ry, bool kd, bool ku, bool kr, bool kl, int a, int b, int cc, int d, int e, int g,
                      int val, float& Ia, float& s) {
  const float vl = IP_FADD(IP_FMUL(rx, rx), IP_FMUL(ry, ry));                     // VectorLength: the SQUARED length
  const float dst = IP_FDIV(1.0f, IP_FADD(IP_FMUL(vl, vl), 1.0f));
  float gx, gy;
  if (kd) gx = ku ? (float)(abs(a - b) + abs(b - cc)) : IP_FMUL((float)abs(a - b), 2.0f);
  else gx = ku ? IP_FMUL((float)abs(b - cc), 2.0f) : 0.f;
  if (kr) gy = kl ? (float)(abs(d - e) + abs(e - g)) : IP_FMUL((float)abs(d - e), 2.0f);
  else gy = kl ? IP_FMUL((float)abs(e - g), 2.0f) : 0.f;
  gx = -gx;
  float dir = IP_FADD(IP_FMUL(rx, gx), IP_FMUL(ry, gy));
  if (fabs((double)dir) <= 0.01) dir = 0.000001f;
  else dir = fabsf(IP_FDIV(dir, IP_FSQRT(IP_FMUL(vl, IP_FADD(IP_FMUL(gx, gx), IP_FMUL(gy, gy))))));
  const float w = IP_FMUL(dst, dir);
  Ia = IP_FADD(Ia, IP_FMUL(w, (float)val));
  s = IP_FADD(s, w);
}

// saturate_cast<uchar>((double)Ia / s): cvRound (nearest even) of the double quotient, clamped
IP_HD uint8_t ip_ns_round(float Ia, float s) {
  int iv = (int)rint(IP_DDIV((double)Ia, (double)s));                               // Ia / s lies in [0, 255]
  return (uint8_t)(iv < 0 ? 0 : (iv > 255 ? 255 : iv));
}

// 8-bit value of IMAGE pixel (row, col) as child c sees it, the coordinates clamped to the image.  Only a one-row or
// one-column image needs the clamp: the reference's shifted indices then leave the image and it reads memory outside it
// (its result is not even repeatable between calls there), which this replaces by the nearest image row / column.
IP_HD int ip_ns_val(const InpaintView& v, int c, int row, int col, int cur) {
  row = row < 0 ? 0 : (row > v.rows - 3 ? v.rows - 3 : row);
  col = col < 0 ? 0 : (col > v.cols - 3 ? v.cols - 3 : col);
  return ip_val(v, c, row + 1, col + 1, cur);
}

// Border-aware evaluation of child c (any position): the reference's loop over (k, l) in the 3x3 window, of which only
// the 4-neighbours are within radius 1.
IP_HD bool ip_eval_child_ns(const InpaintView& v, int c, int cur, float* t_out, uint8_t* val_out) {
  const int cols = v.cols, rows = v.rows;
  const int i = c / cols, j = c - i * cols;
  const IpNb up = ip_at_event(v, c, c - cols, cur), dn = ip_at_event(v, c, c + cols, cur);
  const IpNb lf = ip_at_event(v, c, c - 1, cur), rt = ip_at_event(v, c, c + 1, cur);
  float dist = ip_solve(up, lf);
  { const float d2 = ip_solve(dn, lf); if (d2 < dist) dist = d2; }
  { const float d3 = ip_solve(up, rt); if (d3 < dist) dist = d3; }
  { const float d4 = ip_solve(dn, rt); if (d4 < dist) dist = d4; }
  float Ia = 0.f, s = 1.0e-20f;
  const int dk[4] = {-1, 0, 0, 1}, dl[4] = {0, -1, 1, 0};
  for (int n = 0; n < 4; n++) {
    const int k = i + dk[n], l = j + dl[n];
    if (!(k > 0 && l > 0 && k < rows - 1 && l < cols - 1)) continue;
    const IpNb& nb = (n == 0) ? up : (n == 1) ? lf : (n == 2) ? rt : dn;
    if (!nb.known) continue;
    // image rows / columns of the reference (UNPADDED coordinates, shifted next to the border)
    const int km = k - 1 + (k == 1), kp = k - 1 - (k == rows - 2);
    const int lm = l - 1 + (l == 1), lp = l - 1 - (l == cols - 2);
    const int x = k * cols + l;
    const bool kd = ip_at_event(v, c, x + cols, cur).known, ku = ip_at_event(v, c, x - cols, cur).known;
    const bool kr = ip_at_event(v, c, x + 1, cur).known, kl = ip_at_event(v, c, x - 1, cur).known;
    ip_ns_term((float)(l - j), (float)(k - i), kd, ku, kr, kl, ip_ns_val(v, c, kp + 1, lm, cur),
               ip_ns_val(v, c, kp, lm, cur), ip_ns_val(v, c, km - 1, lm, cur), ip_ns_val(v, c, km, lp + 1, cur),
               ip_ns_val(v, c, km, lm, cur), ip_ns_val(v, c, km, lm - 1, cur), ip_val(v, c, k, l, cur), Ia, s);
  }
  const uint8_t iv = ip_ns_round(Ia, s);
  const bool changed = (dist != v.Tc[cur][c]) || (iv != v.vc[cur][c]);
  *t_out = dist; *val_out = iv;
  return changed;
}

// The same for a child at least 3 pixels from the border (no shifted index applies), gather-then-compute over the 13
// stencil slots and the cached event masks of ip_eval_child_fast.  Bit-identical to ip_eval_child_ns by construction;
// tests/native/inpaint_ns_host.cpp cross-checks both.
IP_HD bool ip_eval_child_ns_fast(const InpaintView& v, int c, int cur, bool first, float* t_out, uint8_t* val_out) {
  const int cols = v.cols, W = cols - 2;
  const int off[13] = {0, -cols, -1, 1, cols, -2 * cols, -cols - 1, -cols + 1, -2, 2, cols - 1, cols + 1, 2 * cols};
  uint8_t VC[13], IM[13];
  float TT[13], TC[13];
  const int ci = c / cols, cj = c - ci * cols;
  const int cimg = (ci - 1) * W + (cj - 1);
  const int offi[13] = {0, -W, -1, 1, W, -2 * W, -W - 1, -W + 1, -2, 2, W - 1, W + 1, 2 * W};
#pragma unroll
  for (int n = 0; n < 13; n++) {                                   // one wave of independent loads
    const int x = c + off[n];
    TT[n] = v.T[x]; TC[n] = v.Tc[cur][x]; VC[n] = v.vc[cur][x]; IM[n] = v.img[cimg + offi[n]];
  }
  uint32_t m;
  if (first) { m = ip_child_masks(v, c); v.em[c] = m; } else m = v.em[c];
  bool kn[13]; float Tn[13]; int val[13];
  kn[0] = false; Tn[0] = IP_TBIG; val[0] = IM[0];
#pragma unroll
  for (int n = 1; n < 13; n++) {
    const bool earlier = (m >> (16 + n)) & 1u;
    kn[n] = (m >> n) & 1u;
    Tn[n] = (kn[n] && !earlier) ? TT[n] : (earlier ? TC[n] : IP_TBIG);
    val[n] = earlier ? (int)VC[n] : (int)IM[n];
  }
  IpNb up, lf, rt, dn;
  up.known = kn[1]; up.T = Tn[1]; lf.known = kn[2]; lf.T = Tn[2]; rt.known = kn[3]; rt.T = Tn[3]; dn.known = kn[4]; dn.T = Tn[4];
  float dist = ip_solve(up, lf);
  { const float d2 = ip_solve(dn, lf); if (d2 < dist) dist = d2; }
  { const float d3 = ip_solve(up, rt); if (d3 < dist) dist = d3; }
  { const float d4 = ip_solve(dn, rt); if (d4 < dist) dist = d4; }
  float Ia = 0.f, s = 1.0e-20f;
  // per cross neighbour n (order up, left, right, down): slots of ITS left / right / up / down pixel, and r = n - c
  const int nL[4] = {6, 8, 0, 10}, nR[4] = {7, 0, 9, 11}, nU[4] = {5, 6, 7, 0}, nD[4] = {0, 10, 11, 12};
  const float rxs[4] = {0.f, -1.f, 1.f, 0.f}, rys[4] = {-1.f, 0.f, 0.f, 1.f};
#pragma unroll
  for (int n = 0; n < 4; n++) {
    const int sl = n + 1;
    if (!kn[sl]) continue;
    ip_ns_term(rxs[n], rys[n], kn[nD[n]], kn[nU[n]], kn[nR[n]], kn[nL[n]], val[nD[n]], val[sl], val[nU[n]], val[nR[n]],
               val[sl], val[nL[n]], val[sl], Ia, s);
  }
  const uint8_t iv = ip_ns_round(Ia, s);
  const bool changed = (dist != TC[0]) || (iv != VC[0]);
  *t_out = dist; *val_out = iv;
  return changed;
}

// =============================================================================================
#if defined(__CUDACC__)
#include <cooperative_groups.h>

#include "emap_grid.cuh"

// device-resident control block of one inpainting run
struct InpaintCtl {
  int heap_cnt[2];                // entries of the two heap lists (ping-pong)
  int tmin_bits[2];               // min T (bits of a non-negative float) over the list of the same index
  int child_cnt;
  int chg[3];                     // "some child changed" flags of Jacobi iterations, rotating
  int rounds, max_jacobi, not_converged;
  unsigned int mm[2];             // min / max keys of the valid heights
  int n_valid;
};

// plugins/inpainting.py:54-56: min / max of the valid cells' heights (order-preserving keys)
__global__ void __launch_bounds__(256)
k_ip_minmax(int C, const float* __restrict__ h, const float* __restrict__ valid, InpaintCtl* ctl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned int lo = 0xffffffffu, hi = 0u; int nv = 0;
  if (i < C && !(valid[i] < 0.5f)) {                               // mask = is_valid < 0.5
    const unsigned int u = __float_as_uint(h[i]);
    lo = hi = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    nv = 1;
  }
  lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi); nv = __reduce_add_sync(0xffffffffu, nv);
  if ((threadIdx.x & 31) == 0 && nv) { atomicMin(&ctl->mm[0], lo); atomicMax(&ctl->mm[1], hi); atomicAdd(&ctl->n_valid, nv); }
}

__device__ __forceinline__ float ip_unkey(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// plugins/inpainting.py:57: ((h - h_min) * 255 / (h_max - h_min)).astype(uint8) in float32 (python float scalars take the
// array's dtype; a CUDA float -> uint8 conversion saturates), and the fast-marching state: INSIDE where the cell is
// invalid, everything else (padding ring included) KNOWN with T = 1e6.
__global__ void __launch_bounds__(256)
k_ip_init(int W, const float* __restrict__ h, const float* __restrict__ valid, InpaintView v, const InpaintCtl* __restrict__ ctl) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= v.rows * v.cols) return;
  const int i = p / v.cols, j = p - i * v.cols;
  uint8_t f = IP_KNOWN;
  if (i >= 1 && j >= 1 && i <= W && j <= W) {
    const int ci = (i - 1) * W + (j - 1);
    const float mn = ip_unkey(ctl->mm[0]), mx = ip_unkey(ctl->mm[1]);
    const float span = (float)((double)mx - (double)mn);
    const float q = __fdiv_rn(__fmul_rn(__fsub_rn(h[ci], mn), 255.0f), span);
    int iq = (q != q) ? 0 : __float2int_rz(fminf(fmaxf(q, -1.0f), 256.0f));
    v.img[ci] = (uint8_t)min(max(iq, 0), 255);
    if (valid[ci] < 0.5f) f = IP_INSIDE;
  }
  v.f[p] = f; v.T[p] = IP_TBIG; v.ord[p] = IP_ROOT;
}

// initial band: known pixels (not on the ring) with an INSIDE 4-neighbour; T = 0, queued (list order is irrelevant:
// the push order of the initial band is row-major BY INDEX, see ip_key_less)
__global__ void __launch_bounds__(256)
k_ip_band(InpaintView v, int* __restrict__ heap0, InpaintCtl* ctl) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= v.rows * v.cols) return;
  const int i = p / v.cols, j = p - i * v.cols;
  if (i < 1 || j < 1 || i > v.rows - 2 || j > v.cols - 2 || v.f[p] != IP_KNOWN) return;
  // f is only read here for INSIDE; BAND is written to a separate pass-local decision (T) to avoid racing with readers
  if (v.f[p - v.cols] == IP_INSIDE || v.f[p + v.cols] == IP_INSIDE || v.f[p - 1] == IP_INSIDE || v.f[p + 1] == IP_INSIDE) {
    v.T[p] = 0.f;
    heap0[atomicAdd(&ctl->heap_cnt[0], 1)] = p;
  }
}
__global__ void __launch_bounds__(256) k_ip_band_flag(InpaintView v, const int* __restrict__ heap0, InpaintCtl* ctl) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < ctl->heap_cnt[0]) v.f[heap0[e]] = IP_BAND;
  if (e == 0) { ctl->tmin_bits[0] = 0; }
}

// claim an INSIDE pixel for this round (byte compare-and-swap through its 32-bit word)
__device__ __forceinline__ bool ip_claim(uint8_t* f, int c) {
  unsigned int* w = reinterpret_cast<unsigned int*>(f + (c & ~3));
  const int sh = (c & 3) * 8;
  unsigned int old = *reinterpret_cast<volatile unsigned int*>(w);
  while (true) {
    if (((old >> sh) & 0xffu) != IP_INSIDE) return false;
    const unsigned int nw = (old & ~(0xffu << sh)) | ((unsigned int)IP_CHILD << sh);
    const unsigned int prev = atomicCAS(w, old, nw);
    if (prev == old) return true;
    old = prev;
  }
}

// The whole fast-marching replay: one cooperative launch, grid barriers between the passes of a round.  METHOD selects
// the per-pixel estimate (IP_TELEA or IP_NS); the rounds are the same for both.
#define IP_MARCH_THREADS 256
template <int METHOD>
__global__ void __launch_bounds__(IP_MARCH_THREADS, 1)
k_ip_march(InpaintView v, int* __restrict__ heapA, int* __restrict__ heapB, int* __restrict__ children, InpaintCtl* ctl,
           int jacobi_cap) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  const int W = v.cols - 2;
  int p = 0, round = 0, max_j = 0, not_conv = 0;
  while (true) {
    int* const hcur = p ? heapB : heapA;
    int* const hnext = p ? heapA : heapB;
    const int nheap = ctl->heap_cnt[p];
    if (nheap == 0) break;
    round++;
    const float tcur = __int_as_float(ctl->tmin_bits[p]);
    // ---- pass A: children of the round, their first popper
    if (gtid == 0) { ctl->heap_cnt[p ^ 1] = 0; ctl->tmin_bits[p ^ 1] = 0x7f7fffff; ctl->chg[0] = 0; ctl->chg[1] = 0; ctl->chg[2] = 0; }
    for (int e = gtid; e < nheap; e += gsz) {
      const int q = hcur[e];
      if (!ip_in_round(v, q, tcur)) continue;
      const int nb[4] = {q - v.cols, q - 1, q + v.cols, q + 1};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int c = nb[k];
        const int ci = c / v.cols, cj = c - ci * v.cols;
        if (ci <= 0 || cj <= 0 || ci >= v.rows - 1 || cj >= v.cols - 1) continue;
        if (v.f[c] != IP_INSIDE || !ip_claim(v.f, c)) continue;
        v.ck[c] = (uint8_t)ip_find_popper(v, c, tcur);
        v.Tc[0][c] = IP_TBIG; v.Tc[1][c] = IP_TBIG; v.vc[0][c] = 0; v.vc[1][c] = 0;
        children[atomicAdd(&ctl->child_cnt, 1)] = c;
      }
    }
    grid.sync();
    const int nchild = ctl->child_cnt;
    // ---- Jacobi iterations to the fixed point of the round
    int cur = 0, it = 0;
    for (;; it++) {
      bool changed = false;
      for (int e = gtid; e < nchild; e += gsz) {
        const int c = children[e];
        float t; uint8_t val;
        if (METHOD == IP_NS)
          changed |= ip_interior(v, c) ? ip_eval_child_ns_fast(v, c, cur, it == 0, &t, &val) : ip_eval_child_ns(v, c, cur, &t, &val);
        else
          changed |= ip_interior(v, c) ? ip_eval_child_fast(v, c, cur, it == 0, &t, &val) : ip_eval_child(v, c, cur, &t, &val);
        v.Tc[cur ^ 1][c] = t; v.vc[cur ^ 1][c] = val;
      }
      if (changed) atomicOr(&ctl->chg[it % 3], 1);
      if (gtid == 0) ctl->chg[(it + 1) % 3] = 0;
      grid.sync();
      cur ^= 1;
      if (!ctl->chg[it % 3]) break;
      if (it + 1 >= jacobi_cap) { not_conv++; break; }
    }
    max_j = max(max_j, it + 1);
    // ---- commit: popped pixels become KNOWN, children join the queue
    for (int e = gtid; e < nheap; e += gsz) {
      const int q = hcur[e];
      if (ip_in_round(v, q, tcur)) v.f[q] = IP_KNOWN;
      else {
        hnext[atomicAdd(&ctl->heap_cnt[p ^ 1], 1)] = q;
        atomicMin(&ctl->tmin_bits[p ^ 1], __float_as_int(v.T[q]));
      }
    }
    for (int e = gtid; e < nchild; e += gsz) {
      const int c = children[e];
      const float t = v.Tc[cur][c];
      v.T[c] = t;
      const int ci = c / v.cols, cj = c - ci * v.cols;
      v.img[(ci - 1) * W + (cj - 1)] = v.vc[cur][c];
      v.ord[c] = ((uint32_t)round << 3) | v.ck[c];
      hnext[atomicAdd(&ctl->heap_cnt[p ^ 1], 1)] = c;
      atomicMin(&ctl->tmin_bits[p ^ 1], __float_as_int(t));
      v.f[c] = IP_BAND;            // byte store; nobody reads a child's state in this pass (in-round tests look at queue pixels)
    }
    if (gtid == 0) ctl->child_cnt = 0;
    grid.sync();
    p ^= 1;
  }
  if (gtid == 0) { ctl->rounds = round; ctl->max_jacobi = max_j; ctl->not_converged = not_conv; }
}

// cv2.inpaint's setup for an 8-bit image (rows x cols) and its mask: the image copied in, INSIDE where the mask is
// non-zero, everything else (padding ring included) KNOWN with T = 1e6.  The control block is zeroed before.
__global__ void __launch_bounds__(256)
k_ip_image_init(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask, InpaintView v) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= v.rows * v.cols) return;
  const int i = p / v.cols, j = p - i * v.cols, W = v.cols - 2;
  uint8_t f = IP_KNOWN;
  if (i >= 1 && j >= 1 && i <= v.rows - 2 && j <= W) {
    const int ci = (i - 1) * W + (j - 1);
    v.img[ci] = img[ci];
    if (mask[ci]) f = IP_INSIDE;
  }
  v.f[p] = f; v.T[p] = IP_TBIG; v.ord[p] = IP_ROOT;
}

// ---- inpainting::nonlinearInterpolation (grid_map_filters_rsl inpainting.cpp:205-242) on a rows x cols grid
// minCoeffOfFinites / maxCoeffOfFinites and the count of finite cells, into a zeroed control block: mm[0] holds the
// complement of the lowest order-preserving key (so that 0 means "none", as for mm[1])
__global__ void __launch_bounds__(256)
k_ip_finite_range(int C, const float* __restrict__ h, InpaintCtl* ctl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned int lo_c = 0u, hi = 0u; int nv = 0;
  if (i < C && isfinite(h[i])) {
    const unsigned int u = __float_as_uint(h[i]);
    hi = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    lo_c = ~hi;
    nv = 1;
  }
  lo_c = __reduce_max_sync(0xffffffffu, lo_c); hi = __reduce_max_sync(0xffffffffu, hi); nv = __reduce_add_sync(0xffffffffu, nv);
  if ((threadIdx.x & 31) == 0 && nv) { atomicMax(&ctl->mm[0], lo_c); atomicMax(&ctl->mm[1], hi); atomicAdd(&ctl->n_valid, nv); }
}

__device__ __forceinline__ void ip_grid_range(const InpaintCtl* ctl, float& lo, float& hi) {
  lo = ip_unkey(~ctl->mm[0]); hi = ip_unkey(ctl->mm[1]);
}

// grid_map_cv's toImage<uchar, 1>(lo, hi) and the inpainting mask (isnan): a NaN cell is INSIDE with image value 0,
// every other cell is clamped to [lo, hi] and quantised in float, truncated (a NaN quotient -- lo == hi, or an
// infinite hi - lo -- converts to 0 as on x86).  Nothing finite: lo / hi are +-FLT_MAX, as in the reference.
__global__ void __launch_bounds__(256)
k_ip_grid_init(const float* __restrict__ h, InpaintView v, const InpaintCtl* __restrict__ ctl) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= v.rows * v.cols) return;
  const int i = p / v.cols, j = p - i * v.cols, W = v.cols - 2;
  uint8_t f = IP_KNOWN;
  if (i >= 1 && j >= 1 && i <= v.rows - 2 && j <= W) {
    const int ci = (i - 1) * W + (j - 1);
    float lo = 3.402823466e38f, hi = -3.402823466e38f;
    if (ctl->n_valid) ip_grid_range(ctl, lo, hi);
    const float x = h[ci];
    uint8_t q = 0;
    if (x != x) f = IP_INSIDE;
    else q = grid_to_u8(x, lo, hi);
    v.img[ci] = q;
  }
  v.f[p] = f; v.T[p] = IP_TBIG; v.ord[p] = IP_ROOT;
}

// convertTo(CV_32F, (hi - lo) / 255, lo) -- fused multiply-add, as cv::Mat::convertTo's x86 path computes it -- copied
// into the NaN cells only; every other cell is the input bit for bit.  Nothing finite: the input.
__global__ void __launch_bounds__(256)
k_ip_grid_out(int C, const uint8_t* __restrict__ img, const float* __restrict__ h, float* __restrict__ out,
              const InpaintCtl* __restrict__ ctl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  const float x = h[i];
  if (x == x || ctl->n_valid == 0) { out[i] = x; return; }
  float lo, hi;
  ip_grid_range(ctl, lo, hi);
  out[i] = grid_from_u8(img[i], lo, hi);
}

// plugins/inpainting.py:60: dst.astype(float32) * (h_max - h_min) / 255 + h_min
__global__ void __launch_bounds__(256)
k_ip_finish(int C, const uint8_t* __restrict__ img, const float* __restrict__ h_in, float* __restrict__ out,
            const InpaintCtl* __restrict__ ctl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  if (ctl->n_valid == 0) { out[i] = h_in[i]; return; }            // inpainting.py:62-63: nothing valid -> the layer itself
  const float mn = ip_unkey(ctl->mm[0]), mx = ip_unkey(ctl->mm[1]);
  const float span = (float)((double)mx - (double)mn);
  out[i] = __fadd_rn(__fdiv_rn(__fmul_rn((float)img[i], span), 255.0f), mn);
}
#endif  // __CUDACC__
