"""Generates tests/golden/polygon_core130.npz: the masks that the REFERENCE'S OWN polygon_mask_kernel source
(CK.py:509-654, compiled for the host through oracle/ref_shim.h, see tests/polygon_oracle.py) computes for the seeded
polygons of polygon_oracle.mask_cases on the core130 map.  Needs the reference checkout; run

    python tests/golden/make_polygon_golden.py

Inputs are regenerated from seeds by the tests, so only the masks are stored (bit-packed, W*W bits each).
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.configs import REF_CONFIGS            # noqa: E402
import polygon_oracle as PO                        # noqa: E402


def polygon_case(tag="core130"):
    W, res = REF_CONFIGS[tag]["cell_n"], REF_CONFIGS[tag]["resolution"]
    out = {}
    with tempfile.TemporaryDirectory() as d:
        lib = PO.build_ref_mask(W, res, d)
        for name, poly, center in PO.mask_cases(W, res):
            clipped, bbox = PO.clip_polygon(poly, center, W, res)
            m = PO.ref_polygon_mask(lib, clipped, bbox, center, W)
            assert set(np.unique(m)) <= {0.0, 1.0}, name
            out[name] = np.packbits(m.reshape(-1) > 0.5)
    return out


if __name__ == "__main__":
    path = os.path.join(HERE, "polygon_core130.npz")
    np.savez_compressed(path, **polygon_case())
    print(path, os.path.getsize(path))
