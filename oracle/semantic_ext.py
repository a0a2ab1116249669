"""oracle/semantic_ext.py -- NumPy definition of the point-channel fusions as the engine computes them (DESIGN §4d).

All six kinds of `emap_semantic_configure_ext`: `average`, `class_average`, `color` (fusion/pointcloud_average.py,
pointcloud_class_average.py, pointcloud_color.py) and `class_bayesian`, `bayesian_inference`, `class_max`
(pointcloud_class_bayesian.py, pointcloud_bayesian_inference.py, pointcloud_class_max.py), with the engine's exact sums:
a float feature is summed in 2^-32 fixed point (each term rounded once, |x| saturated at 2^20, NaN adds 0), an fp16
class_max probability in 2^-24 fixed point (exact).  So this is bit for bit what the device writes, and each float sum is
within one fp32 rounding of some order of the reference's float atomics.

`fuse` runs one frame; `decode_max` / `encode_max` are the class_max channel format; `class_max_rounds` is the
cross-cell round rule on its own, for hand-built cases.
"""
from fractions import Fraction

import numpy as np

KINDS = ("average", "class_average", "color", "class_bayesian", "bayesian_inference", "class_max")


def fix32(x):
    """float32 -> int64 2^-32 fixed point, as fix32 in csrc/emap_device.cuh (llrintf of the fp32 product)."""
    x = np.asarray(x, np.float32)
    x = np.where(np.isnan(x), np.float32(0), np.clip(x, np.float32(-1048576.0), np.float32(1048576.0))).astype(np.float32)
    return np.rint((x * np.float32(4294967296.0)).astype(np.float64)).astype(np.int64)


def unfix32(s):
    """(float)((double)s * 2^-32)"""
    return (np.asarray(s, np.int64).astype(np.float64) * (1.0 / 4294967296.0)).astype(np.float32)


def cell_sum_fix(cells, values, C):
    out = np.zeros(C, np.int64)
    np.add.at(out, cells, values)
    return out


def decode_max(f):
    """pointcloud_class_max.py decode_max: (fp16 probability as fp32, class id) of float32 channel values."""
    bits = np.asarray(f, np.float32).view(np.uint32)
    prob = (bits & 0xFFFF).astype(np.uint16).view(np.float16).astype(np.float32)
    return prob, (bits >> 16).astype(np.int64)


def encode_max(prob, ids):
    """The inverse: float32 values whose bits hold fp16(prob) | id << 16."""
    p = np.asarray(prob, np.float16).view(np.uint16).astype(np.uint32)
    return (p | (np.asarray(ids, np.uint32) << 16)).view(np.float32)


def _fma_double(a, b, c):
    """fp64 a*b + c rounded once (DFMA), element-wise."""
    out = a * b + c
    for j in np.flatnonzero(np.isfinite(a) & np.isfinite(b) & np.isfinite(c)):
        out[j] = float(Fraction(float(a[j])) * Fraction(float(b[j])) + Fraction(float(c[j])))
    return out


def _slot_values(fix, flags):
    """class_max sums: NaN if a NaN or both infinities were summed, else the infinity, else the fixed-point sum."""
    v = (fix.astype(np.float64).astype(np.float32) * np.float32(2.0 ** -24)).astype(np.float32)
    pos, neg = (flags & 1) > 0, (flags & 2) > 0
    v[pos] = np.inf
    v[neg] = -np.inf
    v[((flags & 4) > 0) | (pos & neg)] = np.nan
    return v


def class_max_rounds(C, U, entries, n_rounds):
    """The class_max round rule.  U: ids of the class set; entries: {cell: (ids ascending, fp32 sums)} for the cells with
    records.  Returns (values (n_rounds, C) fp32, ids (n_rounds, C) int32): in round k each cell takes the maximum over U
    (absent or earlier-won ids count 0, ties to the smallest id, NaN is the maximum); every id that won at any cell counts
    0 in the later rounds."""
    U = np.unique(np.asarray(U, np.int64))
    vals = np.zeros((n_rounds, C), np.float32)
    ids = np.full((n_rounds, C), U[0], np.int32)          # a cell without records: every id is 0, U's smallest wins
    zeroed = set()
    for k in range(n_rounds):
        won = set() if len(entries) == C else {int(U[0])}
        for cell, (eid, ev) in entries.items():
            live = np.array([int(i) not in zeroed for i in eid], bool)
            have = bool(live.any())
            if have:
                j = int(np.argmax(ev[live]))                   # first maximum / first NaN, ids ascending
                bv, bid = np.float32(ev[live][j]), int(eid[live][j])
            if not have or (not np.isnan(bv) and bv <= 0):
                present = {int(i) for i, l in zip(eid, live) if l}
                u0 = next((int(u) for u in U if int(u) not in present), None)
                if u0 is not None and (not have or bv < 0 or u0 < bid):
                    bv, bid, have = np.float32(0.0), u0, True
            vals[k, cell] = bv
            ids[k, cell] = bid
            won.add(bid)
        zeroed |= won
    return vals, ids


def fuse(W, idx, valid, inside, dropped, feats, kinds, layers, sem, cnt_fused, alpha=0.5, sigma=None, id_max=None):
    """One frame of point-channel fusion, in place.  idx / valid / inside / dropped: the frame's point record (all
    clouds, in order; dropped = a NaN x, y or z); feats (N, n_ch): the channel values as fp32; kinds / layers per channel;
    sem (n_layers, W, W) fp32; cnt_fused (W*W,): the frame's fused count per cell (new_map[2]); sigma (n_layers, W, W)
    fp32 variance planes (bayesian_inference); id_max (n_id_max, W, W) int32 (class_max)."""
    C = W * W
    feats = np.asarray(feats, np.float32)
    dropped = np.asarray(dropped, bool)
    sel = (np.asarray(valid) > 0) & (np.asarray(inside) > 0) & ~dropped
    cells = np.asarray(idx)[sel].astype(np.int64)
    cnt = np.asarray(cnt_fused).reshape(-1).astype(np.float32)
    m = cnt > 0
    planes = sem.reshape(len(sem), C)
    sums = {}
    for k, kind in enumerate(kinds):
        if kind in ("average", "class_average", "bayesian_inference", "class_bayesian"):
            f = feats[sel, k]
            if kind == "class_bayesian":
                keep = f >= 0                                  # alpha_kernel: theta >= 0 (NaN never)
                sums[k] = unfix32(cell_sum_fix(cells[keep], fix32(f[keep]), C))
            else:
                sums[k] = unfix32(cell_sum_fix(cells, fix32(f), C))
    tot_cb = np.zeros(C, np.float32)
    for k, kind in enumerate(kinds):
        if kind == "class_bayesian":
            tot_cb = (tot_cb + sums[k]).astype(np.float32)
    tot_cb[tot_cb == 0] = 1
    cm = [k for k, kind in enumerate(kinds) if kind == "class_max"]
    if cm:
        prob, cid = decode_max(feats[:, cm])
        U = np.union1d(np.unique(cid[~dropped]), np.unique(id_max.reshape(-1).astype(np.int64) & 0xFFFF))
        p, i = prob[sel].reshape(-1), cid[sel].reshape(-1)
        c = np.repeat(cells, len(cm))
        key = c * 65536 + i
        uk, inv = np.unique(key, return_inverse=True)
        fin = np.isfinite(p)
        fix = np.zeros(len(uk), np.int64)
        np.add.at(fix, inv[fin], np.rint(p[fin].astype(np.float64) * 2.0 ** 24).astype(np.int64))
        flags = np.zeros(len(uk), np.int64)
        np.bitwise_or.at(flags, inv[~fin], np.where(np.isnan(p[~fin]), 4, np.where(p[~fin] > 0, 1, 2)))
        v = _slot_values(fix, flags)
        ucell, start = np.unique(uk // 65536, return_index=True)
        end = np.append(start[1:], len(uk))
        entries = {int(cc): ((uk[a:b] % 65536), v[a:b]) for cc, a, b in zip(ucell, start, end)}
        cm_vals, cm_ids = class_max_rounds(C, U, entries, len(cm))
        tot_cm = np.zeros(C, np.float32)
        for j in range(len(cm)):
            tot_cm = (tot_cm + cm_vals[j]).astype(np.float32)
        tot_cm[tot_cm == 0] = 1
        idm = id_max.reshape(len(id_max), C)
        for j, k in enumerate(cm):
            planes[layers[k]] = (cm_vals[j] / tot_cm).astype(np.float32)
            idm[j] = cm_ids[j]
    for k, kind in enumerate(kinds):
        layer = planes[layers[k]]
        if kind == "color":
            col = feats[sel, k].view(np.uint32).astype(np.int64)
            n = np.bincount(cells, minlength=C)
            r = cell_sum_fix(cells, (col >> 16) & 0xFF, C)
            g = cell_sum_fix(cells, (col >> 8) & 0xFF, C)
            b = cell_sum_fix(cells, col & 0xFF, C)
            h = n > 0
            rgb = ((r[h] // n[h]) << 16) + ((g[h] // n[h]) << 8) + (b[h] // n[h])
            layer[h] = rgb.astype(np.uint32).view(np.float32)
        elif kind == "class_bayesian":
            layer[:] = (sums[k] / tot_cb).astype(np.float32)
        elif kind == "average":
            layer[m] = sums[k][m] / (np.float32(1) * cnt[m])
        elif kind == "class_average":
            prev = layer.copy()
            first = m & (prev == 0)
            layer[first] = sums[k][first] / (np.float32(1) * cnt[first])
            later = m & (prev != 0)
            q = (1.0 - alpha) * sums[k][later].astype(np.float64) / cnt[later].astype(np.float64)
            layer[later] = _fma_double(np.full(q.shape, alpha), prev[later].astype(np.float64), q).astype(np.float32)
        elif kind == "bayesian_inference":
            sg = sigma.reshape(len(sigma), C)[layers[k]]
            s, n = sums[k][m], cnt[m]
            feat_ml = (s / n).astype(np.float32)
            cs = (n * sg[m]).astype(np.float32)
            d = (cs + np.float32(1)).astype(np.float32)
            layer[m] = ((layer[m] / d).astype(np.float32) + ((cs * feat_ml).astype(np.float32) / d)).astype(np.float32)
            sg[m] = (sg[m] / d).astype(np.float32)
    return sem
