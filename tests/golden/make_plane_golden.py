"""Writes tests/golden/planes_golden.npz: the reference's demo terrains (tests/golden/planes/*.png, from
convex_plane_decomposition_ros/data) as grey images, and, for every scene the plane segmentation tests run without a
live oracle, the expected outputs of tests/plane_segmentation_oracle.py (NumPy + cv2): digests of the window, the
elevation and the segmentation layers, highest_label and the plane table.  Scenes: the five terrains, the default 8 m
map after four LiDAR frames (built by the C oracle map, bit-identical to the device's), and a seeded 2047^2 window;
each with connectivity 4 and 8.  Asserts that no decision lies within 1e-9 of its threshold.
  python tests/golden/make_plane_golden.py   (needs cv2 and the built library and oracle)"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
sys.path.insert(0, os.path.dirname(TESTS))
import plane_scenes as S                   # noqa: E402
import plane_segmentation_oracle as PO     # noqa: E402

CASES = {"conn4": {}, "conn8": {"connectivity": 8}}


def window(img, pos, ln, center=(0.0, 0.0)):
    import ctypes as C
    from elevation_mapping_cupy_b200 import _lib
    L = _lib.load()
    W = img.shape[0] + 2
    req = np.array(list(pos) + list(ln), np.float64)
    info = np.zeros(5, np.int32)
    centre = np.zeros(2)
    c = np.array(center, np.float64)
    assert L.emap_submap_windows(W, S.RES, c.ctypes.data, 1, req.ctypes.data, info.ctypes.data,
                                 centre.ctypes.data) == 0
    _, r0, c0, rows, cols = info.tolist()
    origin = centre + (0.5 * (np.array([rows, cols]) * S.RES) - 0.5 * S.RES)
    return img[r0:r0 + rows, c0:c0 + cols], origin


def scenes(out):
    """(name, exported image, window position, window length, map centre)"""
    import cv2
    for name, (png, scale, pos, ln) in S.TERRAINS.items():
        grey = cv2.imread(os.path.join(HERE, "planes", png), cv2.IMREAD_GRAYSCALE)
        out["grey__" + name] = grey
        yield name, S.terrain_image(grey, scale, seed=5 if name == "holes" else None), pos, ln, (0.0, 0.0)
    from elevation_mapping_cupy_b200.parameter import core_parameter
    from oracle import oracle as O
    om = O.OracleElevationMap(core_parameter(S.LIDAR_W), nthreads=0)
    S.lidar_frames(om)
    yield "lidar", S.oracle_export(om), S.lidar_window(om.center), (3.0, 3.0), om.center[:2].astype(np.float64)
    yield "big", S.big_image(), (0.0, 0.0), (100.0, 100.0), (0.0, 0.0)


def main():
    out = {}
    for name, img, pos, ln, centre in scenes(out):
        raw, origin = window(img, pos, ln, centre)
        for case, kw in CASES.items():
            o = PO.segment(raw, S.RES, origin, S.params(**kw))
            assert o["success"] and o["margin"] > 1e-9, (name, case, o.get("margin"))
            k = f"{name}__{case}__"
            out[k + "raw"] = np.array(S.digest(raw))
            out[k + "elevation"] = np.array(S.digest(o["elevation"]))
            out[k + "segmentation"] = np.array(S.digest(o["segmentation"]))
            out[k + "highest_label"] = np.array(o["highest_label"])
            out[k + "planes"] = o["planes"]
            print(name, case, raw.shape, o["highest_label"], len(o["planes"]), "%.1e" % o["margin"])
    np.savez_compressed(S.GOLDEN, **out)


if __name__ == "__main__":
    main()
