"""NumPy restatement of the three semantic plugins as this package specifies them (INTEGRATION.md section 4).

Reference lines restated (elevation_mapping_cupy/script/elevation_mapping_cupy/plugins/):
  semantic_filter.py:30-58    color_map(N): bit-interleaved VOC palette, rows 1-3 overridden, row 0 dropped
  semantic_filter.py:60-75    transform_color: r << 16 | g << 8 | b as uint32 bits
  semantic_filter.py:116-133  argmax over the selected layers, palette lookup (zeros -> id 0 with no layer)
  semantic_traversability.py:59-83  per-layer threshold vote, `where(sum <= 0.9, 0.1, 1)`
  features_pca.py:66-96       clip to [-1, 1], PCA(3) (sklearn; here exact fp64 with svd_flip(u_based_decision=False)),
                              min-max scaling, uint8 cast, r << 16 | g << 8 | b
"""
import numpy as np

PCA_MAX_FEATURES = 64
FILTER_MAX_LAYERS = 255


def color_map(N=255):
    """semantic_filter.py:30-58 with normalized=False: (N, 3) uint8, row k is class id k."""
    cmap = np.zeros((N + 1, 3), dtype=np.uint8)
    for i in range(N + 1):
        r = g = b = 0
        c = i
        for j in range(8):
            r |= ((c >> 0) & 1) << (7 - j)
            g |= ((c >> 1) & 1) << (7 - j)
            b |= ((c >> 2) & 1) << (7 - j)
            c >>= 3
        cmap[i] = (r, g, b)
    cmap[1] = (81, 113, 162)
    cmap[2] = (81, 113, 162)
    cmap[3] = (188, 63, 59)
    return cmap[1:]


def palette():
    """semantic_filter.py:60-75: the packed uint32 words of color_map(255)."""
    c = color_map(255).astype(np.uint32)
    return (c[:, 0] << 16) | (c[:, 1] << 8) | c[:, 2]


def class_ids(stack):
    """numpy.argmax over axis 0 stated as a rule: the first maximum wins; a NaN is the maximum and the first NaN wins.
    stack: (L, ...) fp32; L = 0 gives id 0."""
    stack = np.asarray(stack, np.float32)
    if len(stack) == 0:
        return np.zeros(stack.shape[1:], np.int64)
    best = stack[0].copy()
    ids = np.zeros(stack.shape[1:], np.int64)
    for l in range(1, len(stack)):
        v = stack[l]
        take = ~np.isnan(best) & (np.isnan(v) | (v > best))
        best = np.where(take, v, best)
        ids = np.where(take, l, ids)
    return ids


def semantic_filter(stack, shape=None):
    """uint32 bits of the output plane; stack (L, W, W) fp32 (L may be 0 with `shape` given)."""
    stack = np.asarray(stack, np.float32)
    if len(stack) == 0:
        stack = np.zeros((0,) + tuple(shape), np.float32)
    if len(stack) > FILTER_MAX_LAYERS:
        raise ValueError("more than 255 layers")
    return palette()[class_ids(stack)]


def semantic_traversability(stack, thresholds, types, shape=None):
    """fp32 output plane.  A layer votes where v <= thr (type 'traversability') or v >= thr (other types); the comparison
    is made in fp64 (the fp32 value widened, the threshold as given); NaN never votes.  fp32(0.1) where no layer votes."""
    stack = np.asarray(stack, np.float32)
    score = np.zeros(stack.shape[1:] if len(stack) else tuple(shape), np.int64)
    for v, thr, typ in zip(stack, thresholds, types):
        v = v.astype(np.float64)
        score += (v <= float(thr)) if typ == "traversability" else (v >= float(thr))
    return np.where(score <= 0.9, np.float32(0.1), np.float32(1.0)).astype(np.float32)


def _rows(stack, chunk=1 << 17):
    F = len(stack)
    flat = stack.reshape(F, -1)
    for s in range(0, flat.shape[1], chunk):
        yield np.clip(flat[:, s:s + chunk].T, np.float32(-1), np.float32(1)).astype(np.float64)   # features_pca.py:75


def pca_fit(stack):
    """(mean (F,), components (3, F), eigenvalues (F,) descending) of the clipped features in fp64, every cell a sample.
    Each component's entry of largest |value| (the first on ties) is positive: sklearn's svd_flip(u_based_decision=False)."""
    stack = np.asarray(stack, np.float32)
    F = len(stack)
    if F < 3 or F > PCA_MAX_FEATURES:
        raise ValueError(f"3 to {PCA_MAX_FEATURES} feature layers required, got {F}")
    if np.isnan(stack).any():
        raise ValueError("Input contains NaN")
    n = stack[0].size
    s = np.zeros(F)
    G = np.zeros((F, F))
    for x in _rows(stack):
        s += x.sum(0)
        G += x.T @ x
    mean = s / n
    cov = G - np.outer(s, s) / n
    w, V = np.linalg.eigh(cov)
    order = np.argsort(-w, kind="stable")
    comps = V[:, order[:3]].T.copy()
    for k in range(3):
        arg = int(np.argmax(np.abs(comps[k])))
        if comps[k, arg] < 0:
            comps[k] = -comps[k]
    return mean, comps, w[order]


def pca_project(stack, mean, comps):
    """(3, W, W) fp64 projections (x - mean) . v_k"""
    stack = np.asarray(stack, np.float32)
    out = np.concatenate([(x - mean) @ comps.T for x in _rows(stack)], 0)
    return out.T.reshape((3,) + stack.shape[1:])


def pca_scaled(proj):
    """(p - min) / (max - min) * 255 per component in fp64 (features_pca.py:83-87); 0 where the range is 0"""
    lo = proj.min(axis=(1, 2), keepdims=True)
    rng = proj.max(axis=(1, 2), keepdims=True) - lo
    with np.errstate(invalid="ignore", divide="ignore"):
        sc = (proj - lo) / rng * 255.0
    return np.where(rng > 0, sc, 0.0)


def pack(channels):
    """(3, W, W) uint8 -> uint32 bits r << 16 | g << 8 | b (features_pca.py:89-93)"""
    c = channels.astype(np.uint32)
    return (c[0] << 16) | (c[1] << 8) | c[2]


def features_pca(stack, shape=None):
    """(uint32 bits of the output plane, fp64 scaled values (3, W, W) or None).  No layer gives zeros."""
    stack = np.asarray(stack, np.float32)
    if len(stack) == 0:
        return np.zeros(tuple(shape), np.uint32), None
    mean, comps, _ = pca_fit(stack)
    sc = pca_scaled(pca_project(stack, mean, comps))
    return pack(np.trunc(sc).astype(np.uint8)), sc


def gapped_features(F, W, seed, scales=(0.30, 0.22, 0.16, 0.10)):
    """(F, W, W) fp32 features with a known spectrum: independent components of std `scales` (then 0.05 * 0.9^k) in a
    random orthonormal basis, centred at a random offset; few values reach the clip at +-1.  Eigenvalue gaps >= 10 %."""
    rng = np.random.default_rng(seed)
    std = np.array([scales[k] if k < len(scales) else 0.05 * 0.9 ** (k - len(scales)) for k in range(F)])
    Q, _ = np.linalg.qr(rng.standard_normal((F, F)))
    z = rng.standard_normal((W * W, F)).astype(np.float32) * std.astype(np.float32)
    x = z @ Q.T.astype(np.float32) + rng.uniform(-0.2, 0.2, F).astype(np.float32)
    return np.ascontiguousarray(x.T.reshape(F, W, W)).astype(np.float32)
