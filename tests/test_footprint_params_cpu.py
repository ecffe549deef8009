"""Properties of the oracle's footprint sweeps that test_footprint_params_gpu.py relies on, so that its oracle means what the
reference means: a non-finite traversability_default reaches exactly the footprints that hold an invalid cell, and
radius_is_integer_norm matters only where the first blocked cell lies beyond the inner radius in the exact norm."""
import math

import numpy as np
import pytest

import far_geometry as fg
from footprint_cases import BUILT_GAP, LAYERS, built_map, chain_map
from helpers import YAML, te_footprint_params


def circle(oracle, m, res, **kw):
    og = oracle.Geometry.make(*m["traversability"].shape, res)
    return oracle.footprint(og, te_footprint_params(oracle, **kw), *(m[k] for k in LAYERS))[0]


def polygon(oracle, m, res, **kw):
    og = oracle.Geometry.make(*m["traversability"].shape, res)
    return oracle.footprint_polygon(og, te_footprint_params(oracle, **kw), [v[:2] for v in YAML], 0.7854, *(m[k] for k in LAYERS))[1]


def maps(oracle):
    return [("built", built_map(), BUILT_GAP), ("chain", chain_map(oracle), {})]


@pytest.mark.parametrize("sweep", [circle, polygon], ids=["circle", "polygon"])
def test_non_finite_default_reaches_the_cells_a_finite_default_moves(oracle, sweep):
    for name, m, kw in maps(oracle):
        a, b = sweep(oracle, m, 0.02, traversability_default=0.3, **kw), sweep(oracle, m, 0.02, traversability_default=0.7, **kw)
        moved = a != b
        assert moved.sum() > 50 and (~moved & (a != 0)).sum() > 50, name
        for d in (float("nan"), float("inf"), -float("inf")):
            got = sweep(oracle, m, 0.02, traversability_default=d, **kw)
            assert np.array_equal(~np.isfinite(got), moved), (name, d)
            assert np.array_equal(got[~moved], a[~moved]), (name, d)   # every other cell is the finite default's
            if not math.isnan(d):
                assert (got[moved] == d).all(), (name, d)


def first_blocked_norm(oracle, m, res, rmax):
    """Per cell, the exact index-space norm of the first blocked cell the SpiralIterator visits (inf: none)."""
    rows, cols = m["traversability"].shape
    blocked = m["slope"] == 0
    X, Y = fg.cell_tables(rows, cols, res, (0.0, 0.0))
    I, J = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    out = np.full((rows, cols), np.inf)
    di, dj = oracle.spiral_offsets(rmax, res)
    for a, b in zip(di.tolist(), dj.tolist()):
        A, B = I + a, J + b
        ok = (A >= 0) & (A < rows) & (B >= 0) & (B < cols) & np.isinf(out)
        Ac, Bc = np.clip(A, 0, rows - 1), np.clip(B, 0, cols - 1)
        ok &= fg.circle_inside(X[Ac], Y[Bc], X[I], Y[J], rmax * rmax) & blocked[Ac, Bc]
        out[ok] = math.sqrt(a * a + b * b)
    return out


@pytest.mark.parametrize("res", [0.02, 0.03])
def test_integer_norm_matters_only_beyond_the_inner_radius(oracle, res):
    m = built_map(res, spacing=40)
    radius, offset = 0.30, 0.15
    kw = dict(radius=radius, offset=offset, **BUILT_GAP)
    exact = circle(oracle, m, res, radius_is_integer_norm=0, **kw)
    integer = circle(oracle, m, res, radius_is_integer_norm=1, **kw)
    norm = first_blocked_norm(oracle, m, res, radius + offset)
    differ = exact != integer
    assert differ.sum() > 50
    assert not (differ & ~(norm * res > radius)).any()
    # between the norms: the exact one gives the ring factor, the integer one 0
    band = np.isfinite(norm) & (np.floor(norm) * res <= radius) & (norm * res > radius)
    assert band.sum() > 50 and (integer[band] == 0).all() and (exact[band] != 0).all()
