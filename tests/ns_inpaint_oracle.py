"""tests/ns_inpaint_oracle.py -- TEST INFRASTRUCTURE ONLY.

Sequential restatement of OpenCV's `cv2.inpaint(img_u8, mask, radius, INPAINT_NS)` for one 8-bit channel
(modules/photo/src/inpaint.cpp: icvNSInpaintFMM over the same FastMarching_solve and CvPriorityQueueFloat as Telea).
OpenCV's source is not in this tree, so the routine is restated from its published description and pinned bit for bit
against the cv2 binary by tests/test_inpaint_ns_cpu.py.  It reuses oracle/telea_seq.py's queue and T update: the sweep is
Telea's, only the per-pixel estimate differs.

Per filled pixel (i, j) (padded coordinates; the image is padded by one known ring) and per known pixel (k, l) with
|(k, l) - (i, j)|^2 <= range^2 (k, l not on the ring), all in float unless noted:
  * r = (l - j, k - i), |r|^2 = r.x^2 + r.y^2, dst = 1 / (|r|^2 |r|^2 + 1);
  * an image-gradient magnitude estimate of the 8-bit values around (k, l) from sums of absolute differences, over the
    image rows and columns km = k-1+(k==1), kp = k-1-(k==rows-2), lm = l-1+(l==1), lp = l-1-(l==cols-2) -- the shifted
    indices are how the reference reads the image next to its border (they are part of the pinned result).  On a
    1-row (1-column) image they leave the image; the reference then reads memory outside it and is not even repeatable
    between its own calls, so this restatement (and the device) clamps such reads to the image;
  * gradI.x = -gradI.x; dir = r . gradI, and |dir| <= 0.01 -> 1e-6, else |r . gradI / sqrt(|r|^2 |gradI|^2)|;
  * w = dst * dir; Ia += w * img[k-1, l-1] (unshifted); s += w (s starts at 1e-20);
and the pixel becomes saturate_cast<uchar>((double) Ia / s): round half to even in double, clamped to [0, 255].
"""
import numpy as np

from oracle.telea_seq import BAND, INSIDE, KNOWN, _Heap, _solve

F32 = np.float32


def cv_radius(radius):
    """cv::inpaint's radius: cvRound (half to even), at least 1 (and at most 100)."""
    r = int(np.rint(float(radius)))
    return min(max(r, 1), 100)


def _ns_value(f, out, i, j, rng, rows, cols):
    Ia = F32(0); s = F32(1.0e-20)
    for k in range(i - rng, i + rng + 1):
        km = k - 1 + (k == 1); kp = k - 1 - (k == rows - 2)
        for l in range(j - rng, j + rng + 1):
            lm = l - 1 + (l == 1); lp = l - 1 - (l == cols - 2)
            if not (k > 0 and l > 0 and k < rows - 1 and l < cols - 1):
                continue
            if f[k, l] == INSIDE or (l - j) * (l - j) + (k - i) * (k - i) > rng * rng:
                continue
            ry = F32(k - i); rx = F32(l - j)
            vl = F32(F32(rx * rx) + F32(ry * ry))
            dst = F32(F32(1) / F32(F32(vl * vl) + F32(1)))
            o = lambda a, b: int(out[min(max(a, 0), rows - 3), min(max(b, 0), cols - 3)])
            if f[k + 1, l] != INSIDE:
                if f[k - 1, l] != INSIDE:
                    gx = F32(abs(o(kp + 1, lm) - o(kp, lm)) + abs(o(kp, lm) - o(km - 1, lm)))
                else:
                    gx = F32(F32(abs(o(kp + 1, lm) - o(kp, lm))) * F32(2))
            else:
                gx = F32(F32(abs(o(kp, lm) - o(km - 1, lm))) * F32(2)) if f[k - 1, l] != INSIDE else F32(0)
            if f[k, l + 1] != INSIDE:
                if f[k, l - 1] != INSIDE:
                    gy = F32(abs(o(km, lp + 1) - o(km, lm)) + abs(o(km, lm) - o(km, lm - 1)))
                else:
                    gy = F32(F32(abs(o(km, lp + 1) - o(km, lm))) * F32(2))
            else:
                gy = F32(F32(abs(o(km, lm) - o(km, lm - 1))) * F32(2)) if f[k, l - 1] != INSIDE else F32(0)
            gx = F32(-gx)
            d = F32(F32(rx * gx) + F32(ry * gy))
            if abs(float(d)) <= 0.01:
                d = F32(0.000001)
            else:
                gl = F32(F32(gx * gx) + F32(gy * gy))
                d = F32(abs(F32(d / F32(np.sqrt(F32(vl * gl))))))
            w = F32(dst * d)
            Ia = F32(Ia + F32(w * F32(out[k - 1, l - 1])))
            s = F32(s + w)
    return np.uint8(min(max(int(np.rint(float(Ia) / float(s))), 0), 255))


def ns_inpaint(img, mask, radius=1, return_state=False):
    """img (H, W) uint8, mask (H, W) nonzero = to inpaint.  Returns what cv2.inpaint(img, mask, radius, INPAINT_NS) does."""
    H, W = img.shape
    rows, cols = H + 2, W + 2
    rng = cv_radius(radius)
    f = np.zeros((rows, cols), np.uint8)
    t = np.full((rows, cols), 1.0e6, np.float32)
    m = np.zeros((rows, cols), np.uint8)
    m[1:-1, 1:-1] = (mask != 0)
    out = img.copy()
    band = m.copy()                           # dilate(mask, cross) - mask, off the ring
    band[1:, :] |= m[:-1, :]; band[:-1, :] |= m[1:, :]; band[:, 1:] |= m[:, :-1]; band[:, :-1] |= m[:, 1:]
    band &= 1 - m
    band[0, :] = 0; band[-1, :] = 0; band[:, 0] = 0; band[:, -1] = 0
    heap = _Heap()
    for i in range(rows):
        for j in range(cols):
            if band[i, j]:
                heap.push(i, j, 0.0)
    f[band != 0] = BAND
    f[m != 0] = INSIDE
    t[band != 0] = 0
    order = []
    while True:
        it = heap.pop()
        if it is None:
            break
        ii, jj = it
        f[ii, jj] = KNOWN
        for i, j in ((ii - 1, jj), (ii, jj - 1), (ii + 1, jj), (ii, jj + 1)):
            if i <= 0 or j <= 0 or i >= rows - 1 or j >= cols - 1 or f[i, j] != INSIDE:
                continue
            dist = min(_solve(f, t, i - 1, j, i, j - 1), _solve(f, t, i + 1, j, i, j - 1),
                       _solve(f, t, i - 1, j, i, j + 1), _solve(f, t, i + 1, j, i, j + 1))
            t[i, j] = dist
            out[i - 1, j - 1] = _ns_value(f, out, i, j, rng, rows, cols)
            f[i, j] = BAND
            heap.push(i, j, dist)
            order.append((i, j))
    if return_state:
        return out, t, order
    return out


# ---- grid_map_filters_rsl's inpainting::nonlinearInterpolation (inpainting.cpp:205-242) ----------------------------
FLT_MAX = np.float32(3.4028234663852886e38)


def fma_f32(x, a, b):
    """fl(x * a + b) rounded once (cv::Mat::convertTo's fused x86 path) for uint8 x and float32 a, b: exact rational
    arithmetic over the 256 possible x, rounded to the nearest float32 (ties to even)."""
    from fractions import Fraction
    a, b = np.float32(a), np.float32(b)
    table = np.empty(256, np.float32)
    for v in range(256):
        if not (np.isfinite(a) and np.isfinite(b)):
            with np.errstate(all="ignore"):
                table[v] = np.float32(np.float64(v) * np.float64(a) + np.float64(b))
            continue
        e = Fraction(v) * Fraction(float(a)) + Fraction(float(b))
        f = np.float32(float(e))
        cands = [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
        cands = [c for c in cands if np.isfinite(c)]
        best = min(cands, key=lambda c: (abs(Fraction(float(c)) - e), int(np.float32(c).view(np.uint32)) & 1))
        table[v] = best
    return table[np.asarray(x, np.uint8)]


def to_image_u8(h, lo, hi):
    """grid_map_cv's toImage<uchar, 1>(lo, hi) (restated from its published source, not checked against a grid_map
    build): NaN -> 0; else clamp to [lo, hi] and (uchar)(((v - lo) / (hi - lo)) * 255.0f) in float, truncated, a NaN
    quotient converting to 0 as on x86."""
    h = np.asarray(h, np.float32)
    lo, hi = np.float32(lo), np.float32(hi)
    x = np.where(h < lo, lo, np.where(h > hi, hi, h)).astype(np.float32)
    with np.errstate(all="ignore"):
        r = ((x - lo) / (hi - lo)).astype(np.float32) * np.float32(255.0)
    return np.where(np.isnan(r), np.float32(0), r).astype(np.uint8)


def nonlinear_interpolation(h, resolution, inpaint_radius, inpaint=None):
    """h (rows, cols) float32.  `inpaint(img, mask, radius_px)` fills the 8-bit image (default: ns_inpaint)."""
    h = np.asarray(h, np.float32)
    mask = np.isnan(h)
    fin = h[np.isfinite(h)]
    if fin.size == 0:
        return h.copy()
    lo, hi = np.float32(fin.min()), np.float32(fin.max())
    img = to_image_u8(h, lo, hi)
    radius_px = float(inpaint_radius) / float(resolution)
    filled = (inpaint or ns_inpaint)(img, mask.astype(np.uint8), radius_px)
    with np.errstate(all="ignore"):
        scale = np.float32(np.float32(hi - lo) / np.float32(255.0))
    out = h.copy()
    out[mask] = fma_f32(filled, scale, lo)[mask]
    return out
