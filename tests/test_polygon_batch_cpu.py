"""The batch polygon check's work list (no GPU needed): emap_polygon_traversability_batch gives each polygon only the
k_polygon tiles (PG_COLS = 32 columns by PG_ROWS = 64 rows, aligned to the map) that meet its cell bounding box, and
keeps its column extremes over the box's interior columns.  The library's enumeration (clip_polygon and polygon_tiles in
emap_polygon.cuh, through tests/plan_host.py) must hold every cell of the oracle's mask, so that no polygon loses a cell
to a tile it was not given."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import plan_host as ph               # noqa: E402
import polygon_oracle as PO          # noqa: E402


def _polygons(W, resolution, rng):
    L = 0.5 * (W - 2) * resolution
    out = [(p, c) for _, p, c in PO.mask_cases(W, resolution)]
    for _ in range(12):
        o = rng.uniform(-1.1 * L, 1.1 * L, 2)
        c = np.array([rng.uniform(-500, 500), rng.uniform(-500, 500), 0], np.float32)
        out.append((PO.star(rng, int(rng.integers(3, 20)), 0.01 * L, rng.uniform(0.02, 0.6) * L, c[0] + o[0], c[1] + o[1]),
                    c))
    k = np.array([[-64, -32], [64, -32], [64, 32], [-64, 32]], np.float64) * resolution    # on tile lines
    out.append((k.astype(np.float32), np.zeros(3, np.float32)))
    return out


@pytest.mark.parametrize("W", [130, 202, 1024, 2048, 2049])
def test_enumerated_tiles_hold_every_mask_cell(W):
    resolution = 0.04
    rng = np.random.default_rng(W)
    k = ph.constants()
    PG_COLS, PG_ROWS = k["PG_COLS"], k["PG_ROWS"]
    n_cells = 0
    for poly, center in _polygons(W, resolution, rng):
        clipped, bbox = PO.clip_polygon(poly, center, W, resolution)
        mask = PO.polygon_mask(clipped, bbox, center, resolution, W)
        rows, cols, col0, n_col = ph.polygon_tiles(poly, center, W, resolution)
        cover = np.zeros((W, W), bool)
        for r in rows:
            for c in cols:
                cover[r * PG_ROWS:(r + 1) * PG_ROWS, c * PG_COLS:(c + 1) * PG_COLS] = True
        assert not (mask.astype(bool) & ~cover).any()
        # the column window holds every interior column of the mask (the only columns of over-threshold cells)
        inner = np.flatnonzero(mask[1:-1, 1:-1].any(axis=0))
        assert ((inner >= col0) & (inner < col0 + n_col)).all()
        assert n_col <= W - 2
        n_cells += int(mask.sum())
    assert n_cells > 0


_HARNESS = r"""
#include <cstdio>
#include "emap_polygon.cuh"
int main() {
  float v, c, r;
  int W;
  while (std::scanf("%a %a %a %d", &v, &c, &r, &W) == 4) std::printf("%d\n", poly_axis_cell(v, c, r, W));
  return 0;
}
"""


def test_host_axis_cell_matches_the_device_sequence(tmp_path):
    """The host branch of poly_axis_cell (emap_polygon.cuh), which picks each polygon's tiles, compiled as the library
    is and run on the host: it must give the cells of CK.py:580-603's sequence (PO.vertex_cells) for coordinates near
    cell boundaries, far from the centre, clipped, NaN and infinite."""
    import shutil
    import subprocess
    from elevation_mapping_cupy_b200 import build
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src, exe = tmp_path / "axis.cu", tmp_path / "axis"
    src.write_text(_HARNESS)
    subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", build.CSRC, "-o",
                    str(exe), str(src)], check=True)
    rng = np.random.default_rng(5)
    cases = []
    for W, res in ((130, 0.04), (202, 0.04), (1024, 0.04), (2048, 0.04), (2049, 0.04), (256, 0.1), (512, 0.02)):
        L = 0.5 * W * res
        for c in (0.0, 12.3, -517.9, 1031.3):
            edges = (np.arange(-W // 2 - 2, W // 2 + 3) * res).astype(np.float64)
            v = np.concatenate([edges, np.nextafter(edges, -np.inf), np.nextafter(edges, np.inf),
                                rng.uniform(-1.3 * L, 1.3 * L, 200)]) + c
            cases += [(np.float32(x), np.float32(c), np.float32(res), W) for x in v]
        cases += [(np.float32(x), np.float32(0.0), np.float32(res), W) for x in (np.nan, np.inf, -np.inf, 7e4, -7e4)]
    text = "".join(f"{float(v).hex()} {float(c).hex()} {float(r).hex()} {W}\n" for v, c, r, W in cases)
    out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.split()
    got = np.array(out, np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        want = np.array([PO.vertex_cells(np.array([v]), c, r, W)[0] for v, c, r, W in cases])
    # NaN: the device's truncation gives 0 (vertex_cells' NumPy casts leave it unspecified)
    nan = np.array([np.isnan(v) for v, _, _, _ in cases])
    assert (got[nan] == 0).all()
    assert np.array_equal(got[~nan], want[~nan])
