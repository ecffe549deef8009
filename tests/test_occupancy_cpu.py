"""The CPU restatement of GridMapRosConverter::toOccupancyGrid (tests/occupancy_oracle.cpp) on hand-worked cases, against an
independent numpy float32 restatement over a value sweep, and te_occupancy_grid_info (host arithmetic) against its MapMetaData."""
import ctypes as C

import numpy as np
import pytest

import occupancy_oracle as oo

BAD_ARG = -1


def test_hand_checked_3x2_with_start_index():
    # map cell (i, j) in default order; (1, 0) maps v to trunc((1 - v) * 100) up to float32 rounding
    U = np.array([[1.0, 0.0], [np.nan, 0.5], [0.25, 0.3]], dtype=np.float32)
    buffered = np.roll(U, (1, 1), axis=(0, 1))                          # the same map stored with start index (1, 1)
    got = oo.occupancy_grid(buffered, 1.0, 0.0, start=(1, 1))
    # data[5 - (j * 3 + i)]: cell (0, 0) lands last, cell (2, 1) first
    assert got[5] == 0 and got[4] == -1 and got[3] == 75 and got[2] == 100 and got[1] == 50
    assert got[0] == oo.occupancy_numpy(U, 1.0, 0.0)[0]
    assert np.array_equal(got, oo.occupancy_numpy(U, 1.0, 0.0))
    assert np.array_equal(got, oo.occupancy_grid(U, 1.0, 0.0))


def test_reversed_and_plain_ranges():
    col = np.array([[1.0], [0.0], [np.nan], [0.5], [-7.0], [9.0]], dtype=np.float32)
    assert oo.occupancy_grid(col, 1.0, 0.0)[::-1].tolist() == [0, 100, -1, 50, 100, 0]
    assert oo.occupancy_grid(col, 0.0, 1.0)[::-1].tolist() == [100, 0, -1, 50, 0, 100]
    # equal bounds: +-Inf clamps to 100 / 0, v == data_min is 0 / 0 = NaN
    assert oo.occupancy_grid(col, 0.5, 0.5)[::-1].tolist() == [100, 0, -1, -1, 0, 100]


@pytest.mark.parametrize("rng_", oo.RANGES)
def test_oracle_equals_numpy_over_the_sweep(rng_):
    v = oo.sweep_values()
    assert len(v) > 5000
    layer = np.asfortranarray(v.reshape(-1, 1))
    got = oo.occupancy_grid(layer, *rng_)
    want = oo.occupancy_numpy(layer, *rng_)
    assert np.array_equal(got, want), int((got != want).sum())
    if rng_ == (1.0, 0.0):                                               # the sweep reaches both sides of integers
        assert len(np.unique(got)) == 102


def test_truncation_near_integers():
    # 0.3f with (1, 0): (0.3f - 1) / -1 * 100 in float32, then truncated: the oracle follows float32, not decimal arithmetic
    f = np.float32
    for x in (0.3, 0.07, 0.29, 0.57, 0.58):
        want = int(np.trunc(f(0) + ((f(x) - f(1)) / (f(0) - f(1))) * f(100)))
        assert oo.occupancy_grid(np.array([[x]], np.float32), 1.0, 0.0)[0] == want


def test_start_index_changes_nothing():
    rng = np.random.default_rng(3)
    rows, cols = 17, 23
    U = rng.normal(0.5, 0.6, (rows, cols)).astype(np.float32)
    U[rng.random(U.shape) < 0.1] = np.nan
    want = oo.occupancy_grid(U, 1.0, 0.0)
    for s in [(0, 0), (1, 0), (0, 1), (16, 22), (5, 11), (16, 0)]:
        assert np.array_equal(oo.occupancy_grid(np.roll(U, s, axis=(0, 1)), 1.0, 0.0, start=s), want), s


def _info(te, g, positions=None):
    return te.capi.occupancy_grid_info(g, positions)


def test_grid_info_against_the_oracle(te):
    g = te.Geometry.make(100, 133, 0.03, (2.5, -1.25))
    rec = _info(te, g)[0]
    w, h, res, ox, oy = oo.occupancy_info(100, 133, 0.03, (g.length_x, g.length_y), (2.5, -1.25))
    assert (rec["width"], rec["height"]) == (w, h) == (100, 133)
    assert rec["resolution"].view(np.uint32) == res.view(np.uint32) and rec["resolution"] == np.float32(0.03)
    assert rec["origin_x"] == ox and rec["origin_y"] == oy and rec["reserved"] == 0
    # georeferenced positions and a start index, which changes nothing
    g.start_row, g.start_col = 7, 99
    pos = np.array([[2.6e6 + 0.123, 1.2e6 - 0.377], [-512.25, 33.0], [0.1, 0.2]])
    recs = _info(te, g, pos)
    for r, p in zip(recs, pos):
        w, h, res, ox, oy = oo.occupancy_info(100, 133, 0.03, (g.length_x, g.length_y), p)
        assert (r["width"], r["height"], r["origin_x"], r["origin_y"]) == (w, h, ox, oy)
        assert np.float64(r["origin_x"]).view(np.uint64) == np.float64(ox).view(np.uint64)


def test_grid_info_errors_write_nothing(te):
    L = te.load_library()
    g = te.Geometry.make(8, 8, 0.1)
    out = np.zeros(3, dtype=te.capi.OCCUPANCY_INFO_DTYPE)
    out["width"] = 77
    pos = np.array([[0.0, 0.0], [1.0, np.nan], [2.0, 2.0]])
    bad_start = te.Geometry.make(8, 8, 0.1)
    bad_start.start_row = 8
    bad_pos = te.Geometry.make(8, 8, 0.1, (np.inf, 0.0))
    O = out.ctypes.data
    cases = [("null geometry", None, 1, None, O), ("zero rows", te.Geometry.make(0, 8, 0.1), 1, None, O),
             ("start index outside", bad_start, 1, None, O), ("negative n", g, -1, None, O),
             ("non-finite position", g, 3, pos.ctypes.data, O), ("non-finite geometry position", bad_pos, 2, None, O),
             ("null out", g, 1, None, None)]
    for what, gg, n, p, o in cases:
        rc = L.te_occupancy_grid_info(None if gg is None else C.byref(gg), n, p, o)
        assert rc == BAD_ARG, (what, rc)
        assert (out["width"] == 77).all(), what
    assert L.te_occupancy_grid_info(C.byref(g), 0, None, None) == 0
