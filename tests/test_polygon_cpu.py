"""The polygon safety check's yardstick (tests/polygon_oracle.py) against the reference's own mask kernel source, and the
properties of its hull, area and clip.  No GPU."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import polygon_oracle as PO          # noqa: E402

F = np.float32


def _wr(tag):
    from oracle.configs import REF_CONFIGS
    return REF_CONFIGS[tag]["cell_n"], REF_CONFIGS[tag]["resolution"]


def test_oracle_mask_matches_reference_golden():
    W, res = _wr("core130")
    gold = np.load(os.path.join(HERE, "golden", "polygon_core130.npz"))
    cases = PO.mask_cases(W, res)
    assert sorted(gold.files) == sorted(name for name, _, _ in cases)
    for name, poly, center in cases:
        clipped, bbox = PO.clip_polygon(poly, center, W, res)
        ref = np.unpackbits(gold[name])[:W * W].reshape(W, W)
        assert np.array_equal(PO.polygon_mask(clipped, bbox, center, res, W), ref), name
    # the reference test's triangle (test_elevation_mapping.py:101-106)
    assert int(np.unpackbits(gold["triangle"]).sum()) == 1326


@pytest.mark.skipif(not PO.ref_mask_available(), reason="needs the reference checkout to build its mask kernel")
@pytest.mark.parametrize("tag", ["core130", "default202"])
def test_oracle_mask_matches_reference_source(tag, tmp_path):
    W, res = _wr(tag)
    lib = PO.build_ref_mask(W, res, str(tmp_path))
    rng = np.random.default_rng(11)
    L = 0.5 * (W - 2) * res
    cases = PO.mask_cases(W, res)
    for k in range(12):                       # random polygons, some on cell boundaries, some past the map's edge
        poly = PO.star(rng, int(rng.integers(3, 40)), 0.05 * L, 1.3 * L, *rng.uniform(-0.5 * L, 0.5 * L, 2))
        if k % 3 == 0:
            poly = (np.round(poly / res) * res).astype(np.float32)
        cases.append((f"random{k}", poly, np.array([rng.uniform(-3, 3), rng.uniform(-3, 3), 0], np.float32)))
    for name, poly, center in cases:
        if name.startswith("random"):
            poly = (poly + center[:2]).astype(np.float32)
        clipped, bbox = PO.clip_polygon(poly, center, W, res)
        ref = PO.ref_polygon_mask(lib, clipped, bbox, center, W)
        assert np.array_equal(PO.polygon_mask(clipped, bbox, center, res, W), ref.astype(np.uint8)), name


def _inside_or_on(ring, pts):
    """Every point inside or on the closed counter-clockwise ring (integer cross products)."""
    a, b = ring[:-1], ring[1:]
    for p in pts:
        cr = (b[:, 0] - a[:, 0]) * (p[1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (p[0] - a[:, 0])
        if (cr < 0).any():
            return False
    return True


@pytest.mark.parametrize("seed", range(8))
def test_hull_properties_on_random_sets(seed):
    rng = np.random.default_rng(seed)
    n = [3, 5, 20, 200, 2000, 40, 7, 500][seed]
    pts = rng.integers(0, [30, 60, 128, 200, 1000, 8, 3, 2046][seed], (n, 2))
    ring = PO.convex_ring(pts)
    assert ring is not None
    assert np.array_equal(ring[0], ring[-1]) and len(ring) >= 4                     # closed, >= 3 vertices
    verts = ring[:-1]
    assert len({tuple(v) for v in verts}) == len(verts)
    assert {tuple(v) for v in verts} <= {tuple(p) for p in pts}                      # every vertex is an input cell
    assert tuple(verts[0]) == min(tuple(v) for v in verts)                           # starts at the smallest (row, col)
    a, b, c = verts, np.roll(verts, -1, 0), np.roll(verts, -2, 0)
    turn = (b[:, 0] - a[:, 0]) * (c[:, 1] - b[:, 1]) - (b[:, 1] - a[:, 1]) * (c[:, 0] - b[:, 0])
    assert (turn > 0).all()                                                          # strictly convex, counter-clockwise
    assert _inside_or_on(ring, pts)


def test_hull_degenerate_cases():
    assert PO.convex_ring(np.zeros((0, 2))) is None
    assert PO.convex_ring([[4, 5]]) is None
    assert PO.convex_ring([[4, 5], [4, 5]]) is None
    assert PO.convex_ring([[1, 1], [2, 2], [3, 3], [7, 7]]) is None                  # collinear: a line
    assert PO.convex_ring([[0, 3], [0, 9], [0, 4]]) is None
    r = PO.convex_ring([[0, 0], [0, 2], [2, 0], [1, 1], [0, 1]])                       # collinear points dropped
    assert r.tolist() == [[0, 0], [2, 0], [0, 2], [0, 0]]


def test_area_and_clip_match_fp32_restatement():
    from elevation_mapping_cupy_b200.elevation_mapping import _clipped_area
    rng = np.random.default_rng(3)
    W, res = 202, 0.04
    for k in range(20):
        poly = PO.star(rng, int(rng.integers(3, 30)), 0.1, 6.0, *rng.uniform(-3, 3, 2))
        center = np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), 0], np.float32)
        area = F(0)
        for i in range(len(poly)):                     # traversability_polygon.py:46-51 as CuPy evaluates it in fp32
            p1, p2 = poly[i - 1], poly[i]
            area = (area + (p1[0] * p2[1] - p1[1] * p2[0]) / F(2.0)).astype(np.float32)
        assert PO.shoelace_f32(poly) == abs(area)
        pmin = (center[:2] - F(4.0)) + F(res)          # EM.py:847-851, fp32
        pmax = (center[:2] + F(4.0)) - F(res)
        clipped, bbox = PO.clip_polygon(poly, center, W, res)
        assert np.array_equal(clipped, np.clip(poly, pmin, pmax))
        assert np.array_equal(bbox, np.concatenate([clipped.min(0), clipped.max(0)]))
        assert _clipped_area(poly, center, W, res) == PO.shoelace_f32(clipped)
    # a polygon entirely outside the map is clipped onto the map's edge: (nearly) zero area
    clipped, _ = PO.clip_polygon(np.array([[9, 9], [10, 9], [10, 10]], np.float32), np.zeros(3, np.float32), W, res)
    assert PO.shoelace_f32(clipped) < F(0.001)
