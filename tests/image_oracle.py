"""NumPy restatement of camera image fusion (ElevationMap.input_image), operation by operation in fp32 / fp64 with no
contraction, so that it matches the reference's kernel strings built for the host with contraction off
(oracle/build_ref_image.py, libref_image_cpu_<tag>.so).

  * `camera`          -- the host part, EM.py:468-530: D rule, P = K [R | t], camera cell (what image_camera() in
                         csrc/emap_image.cuh computes; fp32 products, left-to-right sums, NumPy 2 promotion);
  * `correspondence`  -- kernels/custom_image_kernels.py:9-157: uv and valid per cell;
  * `fuse`            -- fusion/image_color.py and fusion/image_exponential.py (alpha 0.7) applied to a layer.

A float -> integer conversion of NaN gives 0 here, as the device's truncating conversion does (the host's is undefined).
"""
import numpy as np

f32 = np.float32


def camera(K, D, model, R, t, center, cell_n, resolution):
    """dict(P (12,), fx, fy, cx, cy, D (5,), distort, x1, y1, z1); raises ValueError where emap_input_image rejects."""
    K = np.asarray(K, f32).reshape(3, 3); R = np.asarray(R, f32).reshape(3, 3); t = np.asarray(t, f32).reshape(3)
    if not (np.isfinite(K).all() and np.isfinite(R).all() and np.isfinite(t).all()):
        raise ValueError("non-finite K, R or t")
    D = np.asarray(D, f32).reshape(-1)
    Dp = np.zeros(5, f32)
    if len(D) >= 4 and model == "radtan":
        Dp[:min(5, len(D))] = D[:5]
    Rt = np.concatenate([R, t[:, None]], 1)
    P = np.zeros((3, 4), f32)
    for r in range(3):
        for c in range(4):
            P[r, c] = (K[r, 0] * Rt[0, c] + K[r, 1] * Rt[1, c]) + K[r, 2] * Rt[2, c]
    center = np.asarray(center, f32)
    tc = np.zeros(3, f32)
    for c in range(3):
        tc[c] = ((-R[0, c]) * t[0] + (-R[1, c]) * t[1]) + (-R[2, c]) * t[2] - center[c]
    cell = []
    for k in range(2):
        s = f32(cell_n / 2) + tc[k] / f32(resolution)
        if not (s >= 0) or s >= f32(2 ** 24):
            raise ValueError("camera cell outside [0, 2^24)")
        cell.append(f32(np.uint32(s)))
    return dict(P=P.reshape(12), fx=K[0, 0], fy=K[1, 1], cx=K[0, 2], cy=K[1, 2], D=Dp, distort=bool((Dp != 0).any()),
                x1=cell[0], y1=cell[1], z1=tc[2])


def _trunc(a):
    """float -> int32 truncation as the device converts (NaN -> 0, saturating)."""
    a = np.asarray(a, np.float64)
    return np.where(np.isnan(a), 0, np.clip(np.trunc(np.nan_to_num(a)), -2 ** 31, 2 ** 31 - 1)).astype(np.int64)


def correspondence(em, cam, center, resolution, img_h, img_w, tolerance=0.10):
    """em: (>=3, W, W) fp32 state (elevation plane 0, is_valid plane 2).  Returns (u, v, valid) as (W, W) arrays; u / v
    are NaN-free only where valid."""
    W = em.shape[-1]
    elev, isv = em[0].reshape(-1).astype(f32), em[2].reshape(-1).astype(f32)
    i = np.arange(W * W)
    x0, y0 = i // W, i % W
    center = np.asarray(center, f32)
    with np.errstate(all="ignore"):
        p1 = ((x0 - W // 2).astype(np.float64) * resolution + np.float64(center[0])).astype(f32)
        p2 = ((y0 - W // 2).astype(np.float64) * resolution + np.float64(center[1])).astype(f32)
        z0 = elev
        p3 = z0 + center[2]
        P = cam["P"]
        row = lambda r: ((p1 * P[4 * r] + p2 * P[4 * r + 1]) + p3 * P[4 * r + 2]) + P[4 * r + 3]
        u, v, d = row(0), row(1), row(2)
        go = (isv == f32(1)) & ~(d <= 0)
        u = u / d
        v = v / d
        if cam["distort"]:
            k1, k2, q1, q2, k3 = cam["D"]
            x = (u - cam["cx"]) / cam["fx"]
            y = (v - cam["cy"]) / cam["fy"]
            r2 = x * x + y * y
            radial = ((f32(1) + k1 * r2) + (k2 * r2) * r2) + ((k3 * r2) * r2) * r2
            uc = (x * radial + ((f32(2) * q1) * x) * y) + q2 * (r2 + (f32(2) * x) * x)
            vc = (y * radial + ((f32(2) * q2) * x) * y) + q1 * (r2 + (f32(2) * y) * y)
            u = cam["fx"] * uc + cam["cx"]
            v = cam["fy"] * vc + cam["cy"]
        go &= ~((u < 0) | (v < 0) | (u >= f32(img_w)) | (v >= f32(img_h)))
        x1, y1 = int(cam["x1"]), int(cam["y1"])
        ddx, ddy = (x0 - x1).astype(f32), (y0 - y1).astype(f32)
        total = np.sqrt(ddx * ddx + ddy * ddy)
        dz = cam["z1"] - z0
        dx = np.abs(x1 - x0); sx = np.where(x0 < x1, 1, -1)
        dy = -np.abs(y1 - y0); sy = np.where(y0 < y1, 1, -1)
        err = dx + dy
        x, y = x0.copy(), y0.copy()
        ok = np.ones(W * W, bool)
        act = go.copy()
        while act.any():
            act &= ~((x == x1) & (y == y1))
            inside = (x >= 0) & (x < W) & (y >= 0) & (y < W)
            act &= inside                               # a line that has left the map never comes back
            c = np.flatnonzero(act)
            idx = y[c] + x[c] * W
            blk = isv[idx] != 0
            fx_, fy_ = (x0[c] - x[c]).astype(f32), (y0[c] - y[c]).astype(f32)
            dis = np.sqrt(fx_ * fx_ + fy_ * fy_)
            ray = z0[c] + (dis / total[c]) * dz[c]
            hit = blk & (elev[idx].astype(np.float64) - tolerance > ray.astype(np.float64))
            ok[c[hit]] = False
            act[c[hit]] = False
            e2 = 2 * err
            a = act & (e2 >= dy)
            stop = a & (x == x1)
            act &= ~stop
            a &= ~stop
            err[a] += dy[a]; x[a] += sx[a]
            b = act & (e2 <= dx)
            stop = b & (y == y1)
            act &= ~stop
            b &= ~stop
            err[b] += dx[b]; y[b] += sy[b]
    valid = go & ok
    return u.reshape(W, W), v.reshape(W, W), valid.reshape(W, W)


def pixel(u, v, img_w):
    """int(u) + int(v) * width in fp32 (fusion/image_*.py), NaN -> 0."""
    return _trunc(_trunc(v).astype(f32) * f32(img_w) + _trunc(u).astype(f32))


def fuse(layer, kind, image, plane, u, v, valid):
    """One channel: the layer after fusion/image_color.py (kind "color", planes 0, 1, 2) or fusion/image_exponential.py
    (kind "exponential", plane `plane`).  image: (C, H, W) fp32."""
    _, H, Wi = image.shape
    out = layer.copy()
    pix = pixel(u[valid], v[valid], Wi)
    flat = image.reshape(-1)
    if kind == "color":
        hw = f32(Wi) * f32(H)
        ig = _trunc(hw + pix.astype(f32))
        ib = _trunc(pix.astype(f32) + hw * f32(2))
        r, g, b = (_trunc(flat[k]).astype(np.uint32) for k in (pix, ig, ib))
        out[valid] = ((r << 16) + (g << 8) + b).astype(np.uint32).view(f32)
    else:
        img = flat[plane * H * Wi + pix].astype(np.float64)
        out[valid] = (layer[valid].astype(np.float64) * (1 - 0.7) + 0.7 * img).astype(f32)
    return out
