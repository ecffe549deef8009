"""The CPU restatement of te_map_chain_windows' window rule and cut (tests/windows_oracle.cpp) on hand-worked cases.  The source
is 8 x 8 cells of 0.5 m centred on the origin, so row i's centre is 1.75 - 0.5 i (column j's likewise) and a position x lies in
row floor((2 - x) / 0.5); cell (i, j) holds 100 i + j."""
import numpy as np

import submap_oracle as sub
import windows_oracle as wo
from helpers import bits

N, RES = 8, 0.5
SRC = np.asfortranarray(100.0 * np.arange(N)[:, None] + np.arange(N)[None, :], dtype=np.float32)
NAN = 0x7fc00000


def _geo(oracle):
    return oracle.Geometry.make(N, N, RES)


def _expected(top, rows, cols):
    """The window by hand: SRC where the cell lies in the source, NaN 0x7fc00000 elsewhere."""
    out = np.full((rows, cols), np.nan, dtype=np.float32)
    for i in range(rows):
        for j in range(cols):
            a, b = top[0] + i, top[1] + j
            if 0 <= a < N and 0 <= b < N:
                out[i, j] = SRC[a, b]
    return out


def test_inside_window_is_getsubmaps(oracle):
    # getSubmap((0.1, -0.1), 1.75 m): corners (0.975, 0.775) and (-0.775, -0.975) fall in rows / columns 2 and 5: a 4 x 4 block
    g = _geo(oracle)
    s = sub.submap_geometry(g, [(0.1, -0.1)], [(1.75, 1.75)])
    assert s["success"][0] == 1 and (s["rows"][0], s["cols"][0], s["top_row"][0], s["top_col"][0]) == (4, 4, 2, 2)
    top, pos = wo.window_geometry(g, 4, 4, [(0.1, -0.1)], length=(1.75, 1.75))
    assert top[0].tolist() == [2, 2]
    # the window's position is the submap's: top-left corner 1.75 - 0.5 * 2 + 0.25 = 1.0, minus half of 4 cells
    assert pos[0].tolist() == [0.0, 0.0] == [s["position_x"][0], s["position_y"][0]]
    cut = wo.cut(SRC, (0, 0), top[0], 4, 4)
    assert np.array_equal(bits(cut), bits(SRC[2:6, 2:6]))


def test_top_left_one_cell_above_is_minus_one(oracle):
    # a 4 x 4 window of 2 m at x = 1.2: its top edge x = 2.2 lies 0.2 m above the map, -(2.2 - 2) / 0.5 = -0.4, which getIndex's
    # truncation would make row 0; the window takes row -1 (NaN) and rows 0..2
    top, pos = wo.window_geometry(_geo(oracle), 4, 4, [(1.2, -0.6)])
    assert top[0].tolist() == [-1, 3]
    assert pos[0, 0] == 1.5   # row -1's centre 2.25, its top edge 2.5, minus half of 2 m
    cut = wo.cut(SRC, (0, 0), top[0], 4, 4)
    assert (bits(cut[0]) == NAN).all()
    assert np.array_equal(bits(cut), bits(_expected((-1, 3), 4, 4)))
    assert np.array_equal(cut[1:], SRC[0:3, 3:7])


def test_half_and_fully_outside_windows(oracle):
    g = _geo(oracle)
    # x = -1.5: top edge -0.5 gives row 5, so rows 5..7 and one row past the bottom; y = 1.6: top edge 2.6 gives column -2
    top, _ = wo.window_geometry(g, 4, 4, [(-1.5, 1.6)])
    assert top[0].tolist() == [5, -2]
    cut = wo.cut(SRC, (0, 0), top[0], 4, 4)
    assert np.array_equal(bits(cut), bits(_expected((5, -2), 4, 4)))
    assert (bits(cut[3]) == NAN).all() and (bits(cut[:, :2]) == NAN).all() and np.array_equal(cut[:3, 2:], SRC[5:8, 0:2])
    # far away on both axes, and on one: every cell is unknown
    for p in [(10.0, 10.0), (0.0, -7.0), (-3.25, 0.0)]:
        top, _ = wo.window_geometry(g, 4, 4, [p])
        assert (bits(wo.cut(SRC, (0, 0), top[0], 4, 4)) == NAN).all(), p


def test_start_index_wraps_rows_and_columns(oracle):
    start = (3, 5)
    stored = np.asfortranarray(np.roll(SRC, start, axis=(0, 1)))   # cell (i, j) at ((i + 3) % 8, (j + 5) % 8)
    assert stored[3, 5] == SRC[0, 0] and stored[2, 4] == SRC[7, 7]
    # rows 3..6 are stored at 6, 7, 0, 1 and columns 1..5 at 6, 7, 0, 1, 2: both wrap inside the window
    for top in [(3, 1), (-2, 4), (6, -1), (0, 0)]:
        got = wo.cut(stored, start, top, 4, 5)
        assert np.array_equal(bits(got), bits(_expected(top, 4, 5))), top


def test_position_on_a_cell_edge(oracle):
    # x = 0.5 with 2 m: the top edge 1.5 is the boundary of rows 0 and 1; -(1.5 - 2) / 0.5 is exactly 1, so row 1, as getIndex
    # puts the edge in the lower row, and the window's position is the requested one
    g = _geo(oracle)
    top, pos = wo.window_geometry(g, 4, 4, [(0.5, -0.5)])
    assert top[0].tolist() == [1, 3] and pos[0].tolist() == [0.5, -0.5]
    s = sub.submap_geometry(g, [(0.5, -0.5)], [(2.0, 2.0)])
    assert (s["top_row"][0], s["top_col"][0]) == (1, 3)   # getSubmap's top-left, one cell more in size (5 x 5)
    assert (s["rows"][0], s["cols"][0]) == (5, 5)
