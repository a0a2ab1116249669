"""NumPy + cv2 restatement of emap_segment_planes (include/emap.h): the plane decomposition node's preprocessing
(grid_map_filters_rsl inpainting::minValues, smoothing::median) and SlidingWindowPlaneExtractor without RANSAC, on one
window.  cv2 does the median, the opening and the labels; numpy.linalg.eigh the fits.  Every decision also reports its
distance from its threshold, so that a scene can be checked to hold no decision a rounding error could flip."""
import numpy as np
from scipy import ndimage

EIG_MIN = 1e-8


def fill_min_values(h):
    """minValues' fixed point: each NaN cell takes the minimum of the non-NaN 4-neighbours of its 4-connected NaN
    component (a window with no non-NaN cell is returned as it is)."""
    out = h.astype(np.float32).copy()
    nan = np.isnan(out)
    if nan.all() or not nan.any():
        return out
    lab, n = ndimage.label(nan, structure=[[0, 1, 0], [1, 1, 1], [0, 1, 0]])
    best = np.full(n + 1, np.inf, np.float64)
    has = np.zeros(n + 1, bool)
    R, C = out.shape
    for dr, dc in ((0, 1), (0, -1), (1, 0), (-1, 0)):
        src = np.full((R, C), np.nan, np.float32)         # the neighbour's value at (r, c)
        l2 = np.zeros((R, C), lab.dtype)
        rs, cs = slice(max(dr, 0), R + min(dr, 0)), slice(max(dc, 0), C + min(dc, 0))
        rd, cd = slice(max(-dr, 0), R + min(-dr, 0)), slice(max(-dc, 0), C + min(-dc, 0))
        src[rd, cd] = out[rs, cs]
        l2[rd, cd] = lab[rd, cd]
        ok = (l2 > 0) & ~np.isnan(src)
        np.minimum.at(best, l2[ok], src[ok].astype(np.float64))
        has[l2[ok]] = True
    out[nan] = best[lab[nan]].astype(np.float32)
    return out


def fill_min_values_literal(h):
    """grid_map_filters_rsl inpainting.cpp:25-94, transliterated: the in-place loop over columns, then rows."""
    H_in = h.astype(np.float32)
    H = H_in.copy()
    R, C = H.shape
    has_value, changed = True, True
    while changed and has_value:
        has_value, changed = False, False
        for c in range(C):
            for r in range(R):
                if np.isnan(H_in[r, c]):
                    for rr, cc in ((r, c - 1), (r, c + 1), (r - 1, c), (r + 1, c)):
                        if 0 <= rr < R and 0 <= cc < C:
                            v = H[rr, cc]
                            if not np.isnan(v) and (v < H[r, c] or np.isnan(H[r, c])):
                                H[r, c] = v
                                changed = True
                else:
                    has_value = True
    return H


def median(img, kernel, repeats):
    import cv2
    k = max(1, min(int(kernel), 5))
    out = img.astype(np.float32).copy()
    if k == 1:
        return out
    for _ in range(int(repeats)):
        out = cv2.medianBlur(out, k)
    return out


def fit_cov(cov):
    """normalAndErrorFromCovariance on a batch of (3, 3) covariances: (normal (n, 3), error (n,))."""
    w, V = np.linalg.eigh(cov)
    n = V[..., :, 0].copy()
    n[n[:, 2] < 0] *= -1
    err = np.maximum(w[:, 0], 0.0)
    bad = ~(w[:, 1] > EIG_MIN)
    n[bad] = (0.0, 0.0, 1.0)
    err[bad] = 1e30
    return n, err, w


def window_fits(img, k, res):
    """computeNormalAndErrorForWindow at every cell, vectorised: sums over the window offsets in the reference's order
    (columns outer, rows inner).  Returns (normal (R, C, 3), error (R, C))."""
    R, C = img.shape
    half = (k - 1) // 2
    pad = np.full((R + 2 * half, C + 2 * half), np.nan, np.float64)
    pad[half:half + R, half:half + C] = img
    n = np.zeros((R, C))
    s = np.zeros((R, C, 3))
    S = np.zeros((R, C, 6))
    for kc in range(k):
        for kr in range(k):
            h = pad[kr:kr + R, kc:kc + C]
            ok = np.isfinite(h)
            p = (-kr * res, -kc * res)
            hz = np.where(ok, h, 0.0)
            n += ok
            s[..., 0] += np.where(ok, p[0], 0.0); s[..., 1] += np.where(ok, p[1], 0.0); s[..., 2] += hz
            S[..., 0] += np.where(ok, p[0] * p[0], 0.0); S[..., 1] += np.where(ok, p[0] * p[1], 0.0)
            S[..., 2] += np.where(ok, p[0], 0.0) * hz; S[..., 3] += np.where(ok, p[1] * p[1], 0.0)
            S[..., 4] += np.where(ok, p[1], 0.0) * hz; S[..., 5] += hz * hz
    return _fit_sums(n.reshape(-1), s.reshape(-1, 3), S.reshape(-1, 6), (R, C))


def _fit_sums(n, s, S, shape):
    nn = np.maximum(n, 1)[:, None]
    m = s / nn
    Sq = S / nn
    idx = ((0, 1, 2), (1, 3, 4), (2, 4, 5))
    cov = np.empty((len(n), 3, 3))
    for i in range(3):
        for j in range(3):
            cov[:, i, j] = Sq[:, idx[i][j]] - m[:, i] * m[:, j]
    cov = np.nan_to_num(cov)
    normal, err, _ = fit_cov(cov)
    few = n < 3
    normal[few] = (0.0, 0.0, 1.0)
    err[few] = 1e30
    return normal.reshape(shape + (3,)), err.reshape(shape)


def window_fits_literal(img, k, res):
    """The same per cell, one window at a time (SlidingWindowPlaneExtractor.cpp:79-113)."""
    R, C = img.shape
    half = (k - 1) // 2
    normal = np.zeros((R, C, 3))
    err = np.zeros((R, C))
    for r in range(R):
        for c in range(C):
            n, s, S = 0, np.zeros(3), np.zeros((3, 3))
            for kc in range(k):
                for kr in range(k):
                    rr, cc = r - half + kr, c - half + kc
                    if not (0 <= rr < R and 0 <= cc < C) or not np.isfinite(img[rr, cc]):
                        continue
                    p = np.array([-kr * res, -kc * res, float(img[rr, cc])])
                    n += 1
                    s += p
                    S += np.outer(p, p)
            if n < 3:
                normal[r, c], err[r, c] = (0, 0, 1), 1e30
                continue
            m = s / n
            nv, e, _ = fit_cov((S / n - np.outer(m, m))[None])
            normal[r, c], err[r, c] = nv[0], e[0]
    return normal, err


def segment(window, res, origin, p):
    """The whole pipeline on one window (float32, NaN = missing) with PlaneSegmentationParams p.  Returns a dict with
    success, elevation, segmentation (int32), classification, highest_label, planes (n, 7) and margin: the smallest
    relative distance of any decision value from its threshold."""
    import cv2
    window = np.asarray(window, np.float32)
    if not np.isfinite(window).any():
        return {"success": False}
    filled = fill_min_values(window)
    img = median(filled, p.median_kernel, p.median_repeats)
    normal, err = window_fits(img.astype(np.float64), p.kernel_size, res)
    thr2 = p.plane_patch_error_threshold ** 2
    finite = np.isfinite(img)
    planar = finite & (err < thr2) & (normal[..., 2] > p.local_plane_inclination_cos)
    margins = [np.inf]
    fitted = finite & (err < 1e29)
    if fitted.any():
        margins.append(np.min(np.abs(err[fitted] - thr2)) / thr2)
        margins.append(np.min(np.abs(normal[..., 2][fitted] - p.local_plane_inclination_cos)))
    binary = planar.astype(np.uint8)
    r = int(p.planarity_opening_filter)
    if r > 0:
        kern = cv2.getStructuringElement(cv2.MORPH_CROSS, (2 * r + 1, 2 * r + 1))
        binary = cv2.morphologyEx(binary, cv2.MORPH_OPEN, kern, anchor=(-1, -1), iterations=1,
                                  borderType=cv2.BORDER_REPLICATE)
    n_lab, labels = cv2.connectedComponents(binary, connectivity=int(p.connectivity), ltype=cv2.CV_32S)
    labels = labels.astype(np.int32)
    R, C = img.shape
    rows, cols = np.meshgrid(np.arange(R, dtype=np.float64), np.arange(C, dtype=np.float64), indexing="ij")
    planes = []
    out_labels = labels.copy()
    # the cells of every label, column-major as the reference visits them
    order = np.argsort(labels.T.reshape(-1), kind="stable")
    lab_cm = labels.T.reshape(-1)[order]
    starts = np.searchsorted(lab_cm, np.arange(n_lab + 1))
    x_cm = (origin[0] - rows * res).T.reshape(-1)[order]
    y_cm = (origin[1] - cols * res).T.reshape(-1)[order]
    h_cm = img.T.reshape(-1).astype(np.float64)[order]
    for L in range(1, n_lab):
        a, b = starts[L], starts[L + 1]
        ok = np.isfinite(h_cm[a:b])
        P = np.stack([x_cm[a:b][ok], y_cm[a:b][ok], h_cm[a:b][ok]], 1)
        n = len(P)
        if n < p.min_number_points_per_label or n < 3:
            continue
        s = P.sum(0)
        S = P.T @ P
        m = s / n
        nv, _, w = fit_cov((S / n - np.outer(m, m))[None])
        margins.append(abs(nv[0, 2] - p.plane_inclination_cos))
        if w[0, 1] > 0:
            margins.append(abs(w[0, 1] - EIG_MIN) / EIG_MIN)
        if nv[0, 2] > p.plane_inclination_cos:
            planes.append([L, *m, *nv[0]])
        else:
            out_labels[labels == L] = 0
    return {"success": True, "elevation": img, "planar": binary, "segmentation": out_labels,
            "classification": (out_labels > 0).astype(np.float32), "highest_label": n_lab - 1,
            "planes": np.array(planes, np.float64).reshape(-1, 7), "margin": float(min(margins))}
