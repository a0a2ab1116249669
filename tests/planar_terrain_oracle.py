"""NumPy + cv2 restatement of emap_planar_terrain's post-processing (include/emap.h): the plane decomposition node's
Postprocessing::postprocess on one window's pre-processed elevation E and plane classification M.  cv2 does the grey
morphology, the box filter and the Gaussian; the minValues fill is plane_segmentation_oracle.fill_min_values; the sloped
dilation is grid_map_filters_rsl's applyKernelFunction, vectorised (sloped_dilation_literal is its loop).  Also the
library's own restatements of boxFilter and GaussianBlur (box_restated, gauss_restated), which the tests hold to cv2."""
import math

import numpy as np

import plane_segmentation_oracle as PO

F32 = np.float32


def std_round(q):
    """std::round on a double: halves away from zero.  Python's round rounds halves to even (2.5 -> 2), and
    floor(q + 0.5) is wrong for q = 0.49999999999999994, where q + 0.5 rounds up to 1.0; q - floor(q) is exact."""
    a = abs(q)
    f = math.floor(a)
    return math.copysign(f + (1.0 if a - f >= 0.5 else 0.0), q)


def kernel_size(size, res):
    """kernelSizeInPixels: 2 * (int)std::round(size / res) + 1 (0.1 / 0.04 = 2.5 gives 7)."""
    return 2 * int(std_round(size / res)) + 1


def slope_offsets(k, res):
    """offsets(i, j) = slope * std::sqrt(dx * dx + dy * dy) with float slope and int dx, dy: double, then float."""
    h = (k - 1) // 2
    d = np.arange(k) - h
    d2 = (d[:, None] ** 2 + d[None, :] ** 2).astype(np.float64)
    return (np.float64(F32(res)) * np.sqrt(d2)).astype(F32)


def _corners(n, k):
    h = (k - 1) // 2
    c = np.maximum(np.arange(n) - h, 0)
    return np.where(c + k > n, n - k, c)


def sloped_dilation(img, k, res):
    """applyKernelFunction(k, (data - offsets).maxCoeffOfFinites()) with the clamped window corner, vectorised."""
    R, C = img.shape
    off = slope_offsets(k, res)
    r0, c0 = _corners(R, k), _corners(C, k)
    best = np.full((R, C), -np.inf, F32)
    found = np.zeros((R, C), bool)
    for a in range(k):
        for b in range(k):
            v = (img[(r0 + a)[:, None], (c0 + b)[None, :]] - off[a, b]).astype(F32)
            fin = np.isfinite(v)
            best = np.where(fin, np.maximum(best, v), best)
            found |= fin
    return np.where(found, best, F32(np.nan)).astype(F32)


def sloped_dilation_literal(img, k, res):
    """processing.cpp:145-177 with the lambda of Postprocessing.cpp:126-128, transliterated cell by cell."""
    R, C = img.shape
    h = (k - 1) // 2
    off = slope_offsets(k, res)
    out = np.empty((R, C), F32)
    for col in range(C):
        for row in range(R):
            cc, rr = max(col - h, 0), max(row - h, 0)
            if cc + k > C:
                cc = C - k
            if rr + k > R:
                rr = R - k
            best = None
            for i in range(k):
                for j in range(k):
                    v = F32(img[rr + i, cc + j]) - off[i, j]
                    if np.isfinite(v):
                        best = v if best is None else max(best, v)
            out[row, col] = F32(np.nan) if best is None else best
    return out


def ellipse(size):
    import cv2
    return cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (size, size))


def box(img, k):
    import cv2
    return cv2.boxFilter(img, -1, (k, k), normalize=True, borderType=cv2.BORDER_REPLICATE)


def gauss(img, k):
    import cv2
    return cv2.GaussianBlur(img, (k, k), 0, 0, borderType=cv2.BORDER_REPLICATE)


def box_restated(img, k):
    """The library's box filter: the window's sum in double times the double 1 / k^2, rounded to float."""
    h = k // 2
    p = np.pad(img.astype(np.float64), h, mode="edge")
    R, C = img.shape
    s = np.zeros((R, C))
    for a in range(k):
        for b in range(k):
            s += p[a:a + R, b:b + C]
    return (s * (1.0 / (k * k))).astype(F32)


def _gauss_pass(x, c, axis):
    h = len(c) // 2
    p = np.pad(x, [(h, h) if a == axis else (0, 0) for a in range(2)], mode="edge")
    n = x.shape[axis]
    at = lambda d: p[:, d:d + n] if axis == 1 else p[d:d + n, :]  # noqa: E731
    s = (c[h] * at(h)).astype(F32)
    for j in range(1, h + 1):
        s = (s + (c[h + j] * (at(h + j) + at(h - j)).astype(F32)).astype(F32)).astype(F32)
    return s


def gauss_restated(img, k):
    """The library's Gaussian: cv2.getGaussianKernel's coefficients, rows then columns, c0 x0 + sum c_j (x_+j + x_-j)
    with every operation rounded to fp32."""
    import cv2
    c = cv2.getGaussianKernel(k, 0, cv2.CV_32F).ravel().astype(F32)
    return _gauss_pass(_gauss_pass(img.astype(F32), c, 1), c, 0)


def gauss_ulps_bound(k):
    """include/emap.h's EMAP_POST_GAUSS_ULPS(k): 4 k + 1 units in the last place of the largest magnitude."""
    return 4 * k + 1


def ulps(a, b, scale):
    """The largest difference between two fp32 arrays in units of the last place of `scale` (the largest magnitude of
    the filtered layer); NaN positions must agree."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    ok = ~np.isnan(a)
    d = np.abs(a[ok].astype(np.float64) - b[ok].astype(np.float64)).max(initial=0.0)
    return float(d / np.spacing(F32(abs(scale))))


def postprocess(E, M, res, p):
    """Postprocessing::postprocess on the map layers: E the pre-processed elevation, M the plane classification (0.0
    or 1.0), res the map resolution, p a PlaneSegmentationParams.  Returns the layers 4 .. 9 of emap_planar_terrain by
    their names, and the kernel sizes."""
    import cv2
    E, M = np.asarray(E, F32), np.asarray(M, F32)
    dil = kernel_size(p.smoothing_dilation_size, res)
    kb = kernel_size(p.smoothing_box_kernel_size, res)
    kg = kernel_size(p.smoothing_gauss_kernel_size, res)
    out = {"sizes": (dil, kb, kg)}
    out["elevationWithNaN"] = np.where(M == 1.0, E, F32(np.nan)).astype(F32)
    out["elevationWithNaN_i"] = PO.fill_min_values(out["elevationWithNaN"])
    out["elevationWithNaNClosed"] = cv2.morphologyEx(out["elevationWithNaN_i"], cv2.MORPH_CLOSE, ellipse(dil),
                                                     borderType=cv2.BORDER_REPLICATE)
    out["elevationWithNaNClosedDilated"] = sloped_dilation(out["elevationWithNaNClosed"], dil, res)
    out["smooth_planar"] = gauss(box(out["elevationWithNaNClosedDilated"], kb), kg)
    e = E.copy()
    off = int(p.nonplanar_horizontal_offset)
    if off > 0:
        d = cv2.dilate(E, ellipse(2 * off + 1), borderType=cv2.BORDER_REPLICATE)
        e = (M * e + (F32(1.0) - M) * d).astype(F32)
    ext, nonpl = float(p.extracted_planes_height_offset), float(p.nonplanar_height_offset)
    if ext != 0.0 or nonpl != 0.0:
        e = (e + F32(ext + nonpl)).astype(F32)          # Eigen narrows the double scalar to float first
        if nonpl != 0.0:
            e = (e - F32(nonpl) * M).astype(F32)
    out["elevation"] = e
    return out
