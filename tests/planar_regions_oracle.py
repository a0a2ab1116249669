"""NumPy + cv2 restatement of the plane decomposition node's contour extraction (convex_plane_decomposition's
ContourExtraction::extractPlanarRegions and Postprocessing::addHeightOffset), the oracle of
ElevationMap.extract_planar_regions.  Each label is cut to its bounding box plus the margin kernel's radius plus 1
before the erosions and findContours (crop=False runs on the whole upsampled image; the tests check both agree), so that
a 2047^2 window finishes in reasonable time.  Points inside polygons with holes use exact integer arithmetic."""
import math

import cv2
import numpy as np
import scipy.ndimage

CROSS = cv2.getStructuringElement(cv2.MORPH_CROSS, (3, 3))


def upsample_literal(image):
    """Upsampling.cpp's loops, transliterated."""
    rows, cols = image.shape
    ur, uc = 4 + 3 * (rows - 2), 4 + 3 * (cols - 2)
    out = np.zeros((ur, uc), image.dtype)

    def column(col, target_col):
        for row in range(rows):
            v = image[row, col]
            if row == 0:
                out[0, target_col] = v
                out[1, target_col] = v
            elif row + 1 == rows:
                out[ur - 2, target_col] = v
                out[ur - 1, target_col] = v
            else:
                t = 2 + 3 * (row - 1)
                out[t:t + 3, target_col] = v

    for col in range(cols):
        if col == 0:
            column(0, 0)
            out[:, 1] = out[:, 0]
        elif col + 1 == cols:
            column(col, uc - 2)
            out[:, uc - 1] = out[:, uc - 2]
        else:
            t = 2 + 3 * (col - 1)
            column(col, t)
            out[:, t + 1] = out[:, t]
            out[:, t + 2] = out[:, t + 1]
    return out


def source_index(m):
    """Upsampled index -> source index for a size-m axis."""
    u = np.arange(3 * m - 2)
    return np.minimum(np.where(u < 2, 0, (u - 2) // 3 + 1), m - 1)


def upsample(image):
    return image[np.ix_(source_index(image.shape[0]), source_index(image.shape[1]))]


def _on_segment(p, a, b):
    (px, py), (ax, ay), (bx, by) = p, a, b
    if (bx - ax) * (py - ay) - (by - ay) * (px - ax) != 0:
        return False
    return min(ax, bx) <= px <= max(ax, bx) and min(ay, by) <= py <= max(ay, by)


def bounded_side(p, poly):
    """1 inside, 0 on the boundary, -1 outside, for an integer point and a closed polygon of integer vertices."""
    n = len(poly)
    for k in range(n):
        if _on_segment(p, poly[k], poly[(k + 1) % n]):
            return 0
    px, py = p
    inside = False
    for k in range(n):
        (ax, ay), (bx, by) = poly[k], poly[(k + 1) % n]
        if (ay > py) != (by > py):
            # the edge crosses the horizontal line y = py at x = ax + (py - ay) (bx - ax) / (by - ay): compare exactly
            num = (py - ay) * (bx - ax)
            den = by - ay
            lhs = (px - ax) * den
            if (lhs < num) if den > 0 else (lhs > num):
                inside = not inside
    return 1 if inside else -1


def inside_with_holes(p, outer, holes):
    """CGAL's isInside on a polygon with holes: on the outer edge or a hole's edge counts as inside."""
    if bounded_side(p, outer) < 0:
        return False
    return all(bounded_side(p, h) <= 0 for h in holes)


def polygons(binary):
    """extractPolygonsFromBinaryImage: [(outer, [holes])] with integer (x, y) points."""
    contours, hierarchy = cv2.findContours(binary, cv2.RETR_CCOMP, cv2.CHAIN_APPROX_SIMPLE)
    out = []
    if hierarchy is None:
        return out
    h = hierarchy[0]
    for i, c in enumerate(contours):
        if h[i][3] < 0 and len(c) > 1:
            holes = []
            child = h[i][2]
            while child > 0:
                holes.append(contours[child].reshape(-1, 2))
                child = h[child][0]
            out.append((c.reshape(-1, 2), holes))
    return out


def boundary_and_inset(binary):
    boundaries = polygons(binary)
    er = cv2.erode(binary, CROSS, iterations=1, borderType=cv2.BORDER_REPLICATE)
    er[0, :] = 0
    er[-1, :] = 0
    er[:, 0] = 0
    er[:, -1] = 0
    insets = polygons(er)
    out = []
    for outer, holes in boundaries:
        assigned = [ins for ins in insets if inside_with_holes(tuple(ins[0][0]), [tuple(q) for q in outer],
                                                               [[tuple(q) for q in hh] for hh in holes])]
        if assigned:
            out.append(((outer, holes), assigned))
    return out


def plane_transform(support, normal):
    """getTransformLocalToGlobal as a 4 x 4 matrix."""
    z = np.asarray(normal, np.float64) / math.sqrt(float(np.dot(normal, normal)))
    y = np.cross(z, [1.0, 0.0, 0.0])
    y2 = float(np.dot(y, y))
    if y2 > 1e-3:
        y = y / math.sqrt(y2)
    else:
        y = np.cross(z, np.cross([0.0, 1.0, 0.0], z))
        y = y / math.sqrt(float(np.dot(y, y)))
    T = np.eye(4)
    T[:3, 0] = np.cross(y, z)
    T[:3, 1] = y
    T[:3, 2] = z
    T[:3, 3] = support
    return T


def project(T, wx, wy):
    dx, dy = wx - T[0, 3], wy - T[1, 3]
    dz = (-dx * T[0, 2] - dy * T[1, 2]) / T[2, 2]
    v = np.stack([dx, dy, dz])
    return np.stack([T[:3, 0] @ v, T[:3, 1] @ v], axis=-1)


def extract(labels, planes, origin, res, margin=1, height_offset=0.0, crop=True):
    """The planar regions of a segmentation (labels: (R, C) label image; planes: the (n, 7) plane table; origin: the
    centre of cell (0, 0)) as extract_planar_regions returns them."""
    labels = np.asarray(labels)
    if labels.shape[0] < 2 or labels.shape[1] < 2:
        return []
    si_r, si_c = source_index(labels.shape[0]), source_index(labels.shape[1])
    ur, uc = len(si_r), len(si_c)
    r = 1 + margin
    margin_kernel = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2 * r + 1, 2 * r + 1))
    res3 = res / 3.0
    int_labels = np.where(labels > 0, labels, 0).astype(np.int64)
    boxes = scipy.ndimage.find_objects(int_labels) if crop else None
    regions = []
    for row in planes:
        label = int(row[0])
        y0, y1, x0, x1 = 0, ur, 0, uc
        if crop:
            if label > len(boxes) or boxes[label - 1] is None:
                continue
            br, bc = boxes[label - 1]
            pad = r + 1
            y0 = max(int(np.searchsorted(si_r, br.start, "left")) - pad, 0)
            y1 = min(int(np.searchsorted(si_r, br.stop - 1, "right")) + pad, ur)
            x0 = max(int(np.searchsorted(si_c, bc.start, "left")) - pad, 0)
            x1 = min(int(np.searchsorted(si_c, bc.stop - 1, "right")) + pad, uc)
        full = np.ascontiguousarray((labels[np.ix_(si_r[y0:y1], si_c[x0:x1])] == label).astype(np.uint8))
        er = cv2.erode(full, margin_kernel, iterations=1, borderType=cv2.BORDER_REPLICATE)
        found = boundary_and_inset(er)
        if not found:
            er = cv2.erode(full, CROSS, iterations=1, borderType=cv2.BORDER_REPLICATE)
            found = boundary_and_inset(er)
        T = plane_transform(row[1:4], row[4:7])

        def to_plane(pts):
            x = pts[:, 0].astype(np.float64) + x0
            y = pts[:, 1].astype(np.float64) + y0
            return project(T, origin[0] - res3 * y, origin[1] - res3 * x)

        Tout = T.copy()
        Tout[2, 3] += height_offset
        for (outer, holes), insets in found:
            o = to_plane(outer)
            regions.append({"label": label, "transform": Tout,
                            "bbox": np.array([o[:, 0].min(), o[:, 1].min(), o[:, 0].max(), o[:, 1].max()]),
                            "boundary": {"outer": o, "holes": [to_plane(h) for h in holes]},
                            "insets": [{"outer": to_plane(io), "holes": [to_plane(h) for h in ih]}
                                       for io, ih in insets]})
    return regions
