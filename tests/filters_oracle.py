"""NumPy restatement of emap_grid_filter (include/emap.h): grid_map_filters_rsl's minValues, median, boxBlur,
gaussianBlur, dilate, erode and outline on one rows x cols float32 layer.  boxBlur is OpenCV's running-sum box filter
(double row sums, double column sums, BORDER_REFLECT_101) written out; dilate, erode and outline are processing.cpp with
its clamped window corner; minValues is plane_segmentation_oracle's fixed point.  tests/test_grid_filters_cpu.py holds
each one to cv2 or to a literal transliteration of the reference."""
import math

import numpy as np

import ns_inpaint_oracle as NS
import plane_segmentation_oracle as PO
from planar_terrain_oracle import _corners

F32 = np.float32

MIN_VALUES, MEDIAN, BOX_BLUR, GAUSSIAN_BLUR, DILATE, ERODE, OUTLINE = range(7)


def reflect101(p, n):
    """cv::borderInterpolate(p, n, BORDER_REFLECT_101): reflected about the edge cells, as often as needed."""
    if n == 1:
        return 0
    while not 0 <= p < n:
        p = -p if p < 0 else 2 * (n - 1) - p
    return p


def _reflect_index(n, k):
    h = k // 2
    return np.array([reflect101(j - h, n) for j in range(n + k - 1)])


def box_blur_once(img, k):
    """cv::blur(img, (k, k)) on CV_32F: RowSum<float, double> then ColumnSum<double, float>, BORDER_REFLECT_101.  Rows:
    k <= 5 sum each window directly, left to right; other k keep a running sum s += x[i + k] - x[i].  Columns: one
    running sum per column from the top border row to the bottom one, s0 = sum + new row, out = float(s0 * (1 / k^2)),
    sum = s0 - oldest row."""
    a = np.asarray(img, F32).astype(np.float64)
    R, C = a.shape
    E = a[:, _reflect_index(C, k)]
    rs = np.empty((R, C), np.float64)
    with np.errstate(all="ignore"):
        if k <= 5:
            rs = E[:, 0: C].copy()
            for j in range(1, k):
                rs = rs + E[:, j: j + C]
        else:
            s = np.zeros(R)
            for j in range(k):
                s = s + E[:, j]
            rs[:, 0] = s
            for i in range(C - 1):
                s = s + (E[:, i + k] - E[:, i])
                rs[:, i + 1] = s
        X = rs[_reflect_index(R, k), :]
        out = np.empty((R, C), F32)
        acc = np.zeros(C)
        for j in range(k - 1):
            acc = acc + X[j]
        scale = 1.0 / (k * k)
        for y in range(R):
            s0 = acc + X[y + k - 1]
            out[y] = (s0 * scale).astype(F32)
            acc = s0 - X[y]
    return out


def box_blur(img, k, repeats=1):
    out = np.asarray(img, F32)
    for _ in range(repeats):
        out = box_blur_once(out, k)
    return out


def min_values(img):
    """minValues' fixed point (plane_segmentation_oracle.fill_min_values), with -0.0 ordered before +0.0 as the device's
    keys order them; a grid with no non-NaN cell is returned as it is."""
    out = PO.fill_min_values(img)
    a = np.asarray(img, F32)
    if np.isnan(a).all():
        return a.copy()
    zero = (out == 0) & np.isnan(a)
    if zero.any():
        # a component touching both -0.0 and +0.0 takes -0.0; recompute the sign on the zero-filled components
        from scipy import ndimage
        lab, _ = ndimage.label(np.isnan(a), structure=[[0, 1, 0], [1, 1, 1], [0, 1, 0]])
        neg = np.zeros(lab.max() + 1, bool)
        R, C = a.shape
        for dr, dc in ((0, 1), (0, -1), (1, 0), (-1, 0)):
            rr, cc = np.nonzero(np.isnan(a))
            r2, c2 = rr + dr, cc + dc
            ok = (r2 >= 0) & (r2 < R) & (c2 >= 0) & (c2 < C)
            v = a[r2[ok], c2[ok]]
            hit = (v == 0) & np.signbit(v)
            neg[lab[rr[ok][hit], cc[ok][hit]]] = True
        out[zero & neg[lab]] = F32(-0.0)
    return out


def _median_network(stack):
    """The device's float median: an insertion network of fminf / fmaxf (np.fmin / np.fmax) over the K^2 window values,
    the middle slot."""
    v = list(stack)
    for a in range(1, len(v)):
        for b in range(a, 0, -1):
            x, y = v[b - 1], v[b]
            v[b - 1], v[b] = np.fmin(x, y), np.fmax(x, y)
    return v[len(v) // 2]


def median_float(img, k):
    """One cv::medianBlur(k) on CV_32F for k = 3 or 5 as the device computes it: the K x K window (border replicated)
    through the fminf / fmaxf network, and a NaN cell kept NaN."""
    a = np.asarray(img, F32)
    if k == 1:
        return a.copy()
    R, C = a.shape
    h = k // 2
    rr = np.clip(np.arange(R)[:, None] + np.arange(-h, h + 1)[None, :], 0, R - 1)
    cc = np.clip(np.arange(C)[:, None] + np.arange(-h, h + 1)[None, :], 0, C - 1)
    stack = [a[rr[:, dr][:, None], cc[:, dc][None, :]] for dr in range(k) for dc in range(k)]
    out = _median_network(stack).astype(F32)
    return np.where(np.isnan(a), a, out).astype(F32)


def median_u8(img, k):
    """cv::medianBlur on CV_8U: the exact median of the k x k window, border replicated."""
    a = np.asarray(img, np.uint8)
    R, C = a.shape
    h = k // 2
    p = np.pad(a, h, mode="edge")
    win = np.lib.stride_tricks.sliding_window_view(p, (k, k)).reshape(R, C, k * k)
    return np.sort(win, axis=2)[:, :, (k * k) // 2].astype(np.uint8)


def median(img, kernel, delta=2, repeats=1):
    """smoothing::median: float medianBlur while kernel + delta (repeats - 1) <= 5, else toImage<uchar, 1> between the
    finite minimum and maximum, the 8-bit medianBlur repeats and convertTo (fused multiply-add) into every cell."""
    a = np.asarray(img, F32)
    if kernel + delta * (repeats - 1) <= 5:
        out = a.copy()
        for r in range(repeats):
            out = median_float(out, kernel + delta * r)
        return out
    fin = a[np.isfinite(a)]
    lo, hi = (fin.min(), fin.max()) if fin.size else (F32(3.402823466e38), F32(-3.402823466e38))
    u = NS.to_image_u8(a, lo, hi)
    for r in range(repeats):
        u = median_u8(u, kernel + delta * r)
    with np.errstate(all="ignore"):
        scale = F32((F32(hi) - F32(lo)) / F32(255.0))
    return NS.fma_f32(u, scale, lo)


def gauss_coeffs(k, sigma):
    """cv::getGaussianKernel(k, sigma, CV_32F) as the device's host code computes it (csrc/emap_postprocess.cuh)."""
    if sigma <= 0:
        import cv2
        return cv2.getGaussianKernel(k, 0, cv2.CV_32F).ravel().astype(F32)
    x = np.arange(k) - (k - 1) * 0.5
    w = np.exp((-0.5 / (sigma * sigma)) * x * x)
    s = 0.0
    for v in w:
        s += v
    return (w * (1.0 / s)).astype(F32)


def gauss_kernel_size(sigma):
    """cv::GaussianBlur's kernel size from sigma on a float image: cvRound(sigma * 4 * 2 + 1) | 1."""
    return int(np.rint(sigma * 4 * 2 + 1)) | 1


def _gauss_pass(x, c, axis):
    h = len(c) // 2
    n = x.shape[axis]
    idx = lambda d: np.array([reflect101(i + d, n) for i in range(n)])
    take = lambda d: np.take(x, idx(d), axis=axis)
    with np.errstate(all="ignore"):
        s = (c[h] * x).astype(F32)
        for j in range(1, h + 1):
            s = (s + (c[h + j] * (take(j) + take(-j)).astype(F32)).astype(F32)).astype(F32)
    return s


def gaussian_blur(img, k, sigma):
    """The device's GaussianBlur(k, sigma), BORDER_REFLECT_101: rows then columns, c0 x0 + sum c_j (x_+j + x_-j) with
    every operation rounded to fp32."""
    a = np.asarray(img, F32)
    if k == 0:
        k = gauss_kernel_size(sigma)
    if k == 1:
        return a.copy()
    c = gauss_coeffs(k, sigma)
    return _gauss_pass(_gauss_pass(a, c, 1), c, 0)


def finites_op(a, b, maximum):
    """grid_map's scalar_max_of_finites_op / scalar_min_of_finites_op, written out for two Python floats: the finite
    operand when only one is finite, else std::max(a, b) = (a < b) ? b : a or std::min(a, b) = (b < a) ? b : a."""
    fa, fb = math.isfinite(a), math.isfinite(b)
    if fa != fb:
        return a if fa else b
    return (b if a < b else a) if maximum else (b if b < a else a)


def morph(img, k, mask=None, inpaint=True, maximum=True):
    """processing.cpp's dilate (maximum) or erode, vectorised: the k x k window with the clamped corner on img * mask,
    folded with finites_op in Eigen's column-major order (the first extreme finite value, so the sign of a zero is the
    earliest one's; with no finite value the functor's fold of the non-finite cells), the cell's own value where that is
    NaN; NaN cells stay NaN unless `inpaint`."""
    a = np.asarray(img, F32)
    with np.errstate(invalid="ignore"):
        m = a if mask is None else (a * np.asarray(mask, F32)).astype(F32)
    R, C = a.shape
    r0, c0 = _corners(R, k), _corners(C, k)
    best = np.full((R, C), np.nan, F32)       # fold of the finite values
    nf = None                                 # fold of every value (used where nothing is finite)
    with np.errstate(invalid="ignore"):
        for j in range(k):
            for i in range(k):
                v = m[(r0 + i)[:, None], (c0 + j)[None, :]]
                fin = np.isfinite(v)
                better = (best < v) if maximum else (v < best)
                best = np.where(fin & (np.isnan(best) | better), v, best)
                if nf is None:
                    nf = v.copy()
                else:
                    nf = np.where((nf < v) if maximum else (v < nf), v, nf)
    res = np.where(np.isnan(best), nf, best)
    out = np.where(np.isnan(res), a, res).astype(F32)
    if not inpaint:
        out = np.where(np.isnan(a), a, out).astype(F32)
    return out


def morph_literal(img, k, mask=None, inpaint=True, maximum=True):
    """processing.cpp:15-105 transliterated cell by cell, with block(...).maxCoeffOfFinites() (minCoeffOfFinites) as
    Eigen's redux folds the functor: the block's first cell, then down each column, column after column."""
    a = np.asarray(img, F32)
    with np.errstate(invalid="ignore"):
        m = a if mask is None else (a * np.asarray(mask, F32)).astype(F32)
    R, C = a.shape
    h = (k - 1) // 2
    out = np.empty((R, C), F32)
    for col in range(C):
        for row in range(R):
            cc, rr = max(col - h, 0), max(row - h, 0)
            cc = C - k if cc + k > C else cc
            rr = R - k if rr + k > R else rr
            if inpaint or not np.isnan(a[row, col]):
                blk = m[rr: rr + k, cc: cc + k]
                cells = [float(blk[i, j]) for j in range(k) for i in range(k)]     # column-major
                res = cells[0]
                for x in cells[1:]:
                    res = finites_op(res, x, maximum)
                out[row, col] = a[row, col] if math.isnan(res) else F32(res)
            else:
                out[row, col] = np.nan
    return out


def outline(img):
    """processing.cpp's outline: a cell keeps its value where its clamped 3 x 3 window has a NaN, else NaN."""
    a = np.asarray(img, F32)
    R, C = a.shape
    r0, c0 = _corners(R, 3), _corners(C, 3)
    has = np.zeros((R, C), bool)
    for i in range(3):
        for j in range(3):
            has |= np.isnan(a[(r0 + i)[:, None], (c0 + j)[None, :]])
    return np.where(has, a, F32(np.nan)).astype(F32)


def apply(op, img, kernel=3, delta=2, repeats=1, sigma=0.0, inpaint=True, mask=None):
    """emap_grid_filter's result for one filter description."""
    if op == MIN_VALUES:
        return min_values(img)
    if op == MEDIAN:
        return median(img, kernel, delta, repeats)
    if op == BOX_BLUR:
        return box_blur(img, kernel, repeats)
    if op == GAUSSIAN_BLUR:
        return gaussian_blur(img, kernel, sigma)
    if op in (DILATE, ERODE):
        return morph(img, kernel, mask, inpaint, op == DILATE)
    if op == OUTLINE:
        return outline(img)
    raise ValueError(op)
