"""Properties of the path-check oracle that test_paths_params_gpu.py relies on, so that its oracle means what the reference means:
a walk that stores a NaN or an infinity leaves its cell uncached, so the next check there walks again with its own radius and
flag; radius_is_integer_norm changes a circle's answer only where a blocked cell lies beyond the inner radius; a polygon that
covers no cell centre answers the default."""
import math

import numpy as np
import pytest

import paths_oracle as po
import paths_params_cases as pc
from helpers import footprint_arrays, te_footprint_params

INF, NAN = float("inf"), float("nan")


def run(oracle, m, kw, R, cache=None):
    rows, cols = m["traversability"].shape
    og = oracle.Geometry.make(rows, cols, pc.RES)
    fb, fx = footprint_arrays(R, R["fps"])
    return po.check_request(og, te_footprint_params(oracle, **kw), m, R["begin"], R["poses"], R["radius"], fb, fx,
                            conservative=R["cons"], cup=R["cup"], cache=cache)


def empty(m):
    return np.full(m["traversability"].shape, np.nan, np.float32, order="F")


@pytest.mark.parametrize("case", ["nan", "inf", "-inf", "offset0"])
def test_a_non_finite_store_is_walked_again(oracle, case):
    """The first check stores a non-finite float and is traversable; the second, at the same cell without the polygon flag,
    answers as it does on an empty cache (a walk), not as a read of that float would (traversable)."""
    m, kw, R = pc.ring_case(0) if case == "offset0" else pc.nan_case(float(case))
    cache = empty(m)
    safe, trav = run(oracle, m, kw, R, cache)[:2]
    assert safe.tolist() == [1, 0] and trav[1] == 0.0
    stored = cache[pc.CENTRE, pc.CENTRE]
    assert not math.isfinite(trav[0]) and not math.isfinite(stored)
    assert (math.isnan(trav[0]) and math.isnan(stored)) if case == "nan" else trav[0] == stored == (-INF if case == "-inf" else INF)
    alone = run(oracle, m, kw, pc.request([(R["poses"][1:2, :2], R["radius"][1], -1, 0, 0)]), empty(m))
    assert alone[0].tolist() == [0]
    # the same cell with a finite store is read: the second path reads the first one's float
    if case == "offset0":
        finite = run(oracle, *pc.ring_case(1), empty(m))   # the integer norm puts the blocker on the inner radius: 0 stored
        assert finite[0].tolist() == [0, 0] and finite[1].tolist() == [0.0, 0.0]
    else:
        finite = run(oracle, m, dict(kw, traversability_default=0.3), R, empty(m))
        assert finite[0].tolist() == [1, 1] and finite[1][1] == float(np.float32(finite[1][0])) != finite[1][0]


def test_a_finite_store_after_non_finite_ones_is_read(oracle):
    for d in (NAN, INF):
        m, kw, R = pc.mixed_case(d)
        cache = empty(m)
        safe, trav = run(oracle, m, kw, R, cache)[:2]
        assert safe.all() and not np.isfinite(trav[:2]).any()
        assert (trav[2:] == 0.5).all() and cache[pc.CENTRE, pc.CENTRE] == 0.5


def test_radius_alone_decides_the_revisit(oracle):
    """Two visits that differ only in radius: radius 0.26 puts the blocker inside its inner radius and blocks."""
    m, kw, R = pc.nan_case(NAN, cups=(1, 1), radii=(0.2, 0.26))
    cache = empty(m)
    safe, trav, _, count = run(oracle, m, kw, R, cache)[:4]
    assert safe.tolist() == [1, 0] and math.isnan(trav[0]) and count[1] > 0 and cache[pc.CENTRE, pc.CENTRE] == 0.0


def norm_request(m, radius):
    """Single circular poses at every other cell centre of rows / columns 10 .. n-10, radius `radius`, the polygon flag set (without
    it a blocker beyond the inner radius ends the walk untraversable under either norm)."""
    rows, cols = m["traversability"].shape
    X, Y = pc.fg.cell_tables(rows, cols, pc.RES, (0.0, 0.0))
    idx = [(a, b) for a in range(10, rows - 10, 2) for b in range(10, cols - 10, 2)]
    R = pc.request([([(float(X[a]), float(Y[b]))], radius, -1, 0, 1) for a, b in idx])
    return R, idx


def test_norm_matters_only_beyond_the_inner_radius(oracle):
    """A circle whose disk holds no blocked cell beyond the inner radius (exact norm) answers the same under both norms."""
    from footprint_cases import BUILT_GAP, built_map
    m = built_map(spacing=24)
    radius, offset = 0.2, 0.15
    R, idx = norm_request(m, radius)
    got = [run(oracle, m, dict(BUILT_GAP, offset=offset, radius_is_integer_norm=n), R)[:2] for n in (0, 1)]
    differ = (got[0][0] != got[1][0]) | (got[0][1].view(np.uint64) != got[1][1].view(np.uint64))
    rows, cols = m["traversability"].shape
    X, Y = pc.fg.cell_tables(rows, cols, pc.RES, (0.0, 0.0))
    blocked = np.argwhere(m["slope"] == 0)
    beyond = np.zeros(len(idx), bool)
    for k, (a, b) in enumerate(idx):
        d = blocked - [a, b]
        inside = (X[blocked[:, 0]] - X[a]) ** 2 + (Y[blocked[:, 1]] - Y[b]) ** 2 <= (radius + offset) ** 2
        beyond[k] = (inside & (np.sqrt((d * d).sum(1)) * pc.RES > radius)).any()
    assert differ.sum() > 20 and beyond.sum() > differ.sum()
    assert not (differ & ~beyond).any()


@pytest.mark.parametrize("default", [0.3, 0.0, NAN, -INF])
def test_polygon_covering_no_cell_centre_answers_the_default(oracle, default):
    m = pc.flat_map()
    tiny = np.asarray([(0.004, 0.004, 0.0), (0.009, 0.004, 0.0), (0.004, 0.009, 0.0)], np.float32)
    c = pc.centre_xy()
    R = pc.request([([c], math.nan, 0, 0, 0), ([c, (c[0] + 0.001, c[1])], math.nan, 0, 0, 0)], fps=[tiny])
    safe, trav, area = run(oracle, m, dict(traversability_default=default), R)[:3]
    assert safe.tolist() == [int(default != 0.0)] * 2
    if default != 0.0:
        assert np.array_equal(trav, [default] * 2, equal_nan=True) and (area > 0).all()
