"""The untraversable polygon of the fresh circular and the polygonal path checks in the CPU oracles, against vertex lists derived by
hand.  Dyadic geometry (0.25 m cells, map centred on the origin) keeps every cell centre exact.  Cells are blocked through
checkForSlope: with max_gap_width 0.1 its critical count is floor(2 * 0.75 * (0.1 / 3) / 0.25^2) = 0, so a cell whose
traversability_slope is 0 fails isTraversableForFilters and no other cell does."""
import math

import numpy as np

import paths_oracle as po
from helpers import DYADIC_N as N, dyadic_cell as P, dyadic_map as _map, dyadic_x as X

Y = X


def _circle(g, fp, L, paths, radius=1.0, cup=1, robot_slope=None, capacity=64):
    """paths: lists of (x, y) poses; returns (is_safe, traversability, [vertex list per path])."""
    begin = np.cumsum([0] + [len(p) for p in paths]).astype(np.int32)
    poses = np.asarray([q for p in paths for q in p], np.float64).reshape(-1, 2)
    Ls = dict(L, robot_slope=robot_slope)
    safe, t, _, cnt, xy = po.check_request(g, fp, Ls, begin, poses, radius, cup=cup, capacity=capacity)
    ref_safe, ref_t = po.check_request(g, fp, Ls, begin, poses, radius, cup=cup, capacity=0)[:2]   # no polygon outputs
    assert np.array_equal(safe, ref_safe) and np.array_equal(t.view(np.uint64), ref_t.view(np.uint64))
    return safe, t, [[tuple(v) for v in xy[q, :min(cnt[q], capacity)]] for q in range(len(paths))]


def from_circle(cx, cy, r):
    """grid_map::Polygon::fromCircle(center, r), nVertices = 20 (recalled)."""
    out = []
    for j in range(20):
        th = j * 2 * math.pi / 19
        c, s = math.cos(th), math.sin(th)
        out.append((cx + (c * r + (-s) * 0.0), cy + (s * r + c * 0.0)))
    return out


def chain(points):
    """monotoneChainConvexHullOfPoints (recalled)."""
    if len(points) <= 3:
        return list(points)
    pts = sorted(points)
    cw = lambda o, a, b: (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0]) <= 0  # noqa: E731
    h = []
    for p in pts:
        while len(h) >= 2 and cw(h[-2], h[-1], p):
            h.pop()
        h.append(p)
    t = len(h) + 1
    for p in reversed(pts[:-1]):
        while len(h) >= t and cw(h[-2], h[-1], p):
            h.pop()
        h.append(p)
    return h[:-1]


def test_one_two_three_cells_in_visit_order(oracle):
    c = (32, 32)
    # one cell (the centre, ring 0); a later blocked cell of the annulus (5 cells = 1.25 m > radius 1.0) is not collected (:705)
    g, fp, L = _map(oracle, [c, (37, 32)])
    safe, _, poly = _circle(g, fp, L, [[P(*c)]])
    assert safe.tolist() == [0] and poly == [[P(32, 32)]]
    # two cells: ring 0, then ring 2
    g, fp, L = _map(oracle, [(34, 32), c])
    assert _circle(g, fp, L, [[P(*c)]])[2] == [[P(32, 32), P(34, 32)]]
    # three cells, visited ring 0, ring 1, ring 3: not the lexicographic order (X falls with the row index)
    g, fp, L = _map(oracle, [(32, 35), (33, 32), c])
    poly = _circle(g, fp, L, [[P(*c)]])[2][0]
    assert poly == [P(32, 32), P(33, 32), P(32, 35)] and poly != sorted(poly)
    # compute_untraversable_polygon off: no polygon
    assert _circle(g, fp, L, [[P(*c)]], cup=0)[2] == [[]]


def test_block_gives_square_from_lexicographic_minimum(oracle):
    g, fp, L = _map(oracle, [(a, b) for a in range(31, 34) for b in range(31, 34)])
    poly = _circle(g, fp, L, [[P(32, 32)]])[2][0]
    assert poly == [P(33, 33), P(31, 33), P(31, 31), P(33, 31)]


def test_four_cells_in_one_row(oracle):
    g, fp, L = _map(oracle, [(32, b) for b in (30, 31, 33, 34)])
    assert _circle(g, fp, L, [[P(32, 32)]])[2] == [[P(32, 34), P(32, 30)]]   # collinear: the two extremes


def test_first_blocker_in_the_annulus(oracle):
    g, fp, L = _map(oracle, [(37, 32), (32, 32 + 6)])
    safe, t, poly = _circle(g, fp, L, [[P(32, 32)]])
    assert safe.tolist() == [1] and poly == [[]]


def test_zero_radius_collects_every_blocked_cell(oracle):
    g, fp, L = _map(oracle, [(32, 34), (33, 32)])          # rmax = offset = 0.5 m: rings 0..2, both cells inside
    safe, _, poly = _circle(g, fp, L, [[P(32, 32)]], radius=0.0)
    assert safe.tolist() == [0] and poly == [[P(33, 32), P(32, 34)]]


def test_single_pose_outside_the_map(oracle):
    g, fp, L = _map(oracle)
    fp.traversability_default = 0.0
    pose = (X(0) + 3.0, 0.5)
    safe, _, poly = _circle(g, fp, L, [[pose]])
    assert safe.tolist() == [0] and poly == [from_circle(pose[0], pose[1], 1.5)] and len(poly[0]) == 20
    fp.traversability_default = 0.3
    assert _circle(g, fp, L, [[pose]])[2] == [[]]


def test_revisited_centre_cached_zero(oracle):
    trav = np.full((N, N), 0.5, np.float32)
    trav[:, 11:] = 0.0                 # the discs (3 cells) around columns 14 and 18 see only zero traversability
    g, fp, L = _map(oracle, trav=trav)
    A, M, B = (30, 10), (30, 14), (30, 18)
    # A -> B -> A: segment 2 checks A (cached > 0), then M, cached 0 on its first check: fromCircle(M), hulled for M and B
    safe, _, poly = _circle(g, fp, L, [[P(*A), P(*B), P(*A)]], radius=0.25)
    assert safe.tolist() == [0]
    want = chain(from_circle(X(M[0]), Y(M[1]), 0.75))
    assert poly == [want] and want[0] == min(want) and len(want) < 20
    assert _circle(g, fp, L, [[P(*A), P(*B)]], radius=0.25)[0].tolist() == [1]


def test_repeated_hull_of_a_failing_segment(oracle):
    # one blocked cell near B; the line from B to A is checked at cells 0, 4, 8 (9 cells) or 0, 4 (5 cells)
    g, fp, L = _map(oracle, [(30, 19)])
    A9, A5, B = (30, 10), (30, 14), (30, 18)
    _, _, poly = _circle(g, fp, L, [[P(*A9), P(*B)], [P(*A5), P(*B)]], radius=0.5)
    p = P(30, 19)
    assert poly == [[p, p, p], [p, p]]      # [p] hulled 3 times / 2 times: [p, p, p], [p, p]
    g, fp, L = _map(oracle, [(30, 19), (31, 18)])
    _, _, poly = _circle(g, fp, L, [[P(*A9), P(*B)]], radius=0.5)
    assert poly == [[P(31, 18), P(30, 19)]]  # two cells hulled again: their chain, from the lexicographic minimum
    _, _, poly = _circle(g, fp, L, [[P(*B)]], radius=0.5)
    assert poly == [[P(30, 19), P(31, 18)]]  # a single pose: once, in visit order


def test_inclination_failure_publishes_nothing(oracle):
    g, fp, L = _map(oracle, [(32, 32)])
    rs = np.ones((N, N), np.float32, order="F")
    rs[32, 32] = 0.0
    safe, _, poly = _circle(g, fp, L, [[P(32, 32)]], robot_slope=rs)
    assert safe.tolist() == [0] and poly == [[]]


def test_capacity_smaller_than_the_polygon(oracle):
    g, fp, L = _map(oracle, [(a, b) for a in range(31, 34) for b in range(31, 34)])
    begin, poses = np.array([0, 1], np.int32), np.array([P(32, 32)])
    _, _, _, cnt, xy = po.check_request(g, fp, L, begin, poses, [1.0], cup=[1], capacity=2)
    assert cnt.tolist() == [4] and [tuple(v) for v in xy[0]] == [P(33, 33), P(31, 33)]


SQUARE = np.array([[0.5, 0.5, 0.0], [-0.5, 0.5, 0.0], [-0.5, -0.5, 0.0], [0.5, -0.5, 0.0]], np.float32)


def _pose(x, y):
    return [x, y, 0.0, 0.0, 0.0, 0.0, 1.0]


def _polygonal(g, fp, L, paths, cup):
    begin = np.cumsum([0] + [len(p) for p in paths]).astype(np.int32)
    poses = np.asarray([_pose(*q) for p in paths for q in p], np.float64)
    out = po.check_request(g, fp, L, begin, poses, footprint_xyz=SQUARE, cup=cup)
    ref = po.check_request(g, fp, L, begin, poses, footprint_xyz=SQUARE, cup=1 - cup)   # is_safe, traversability, area: cup has no say
    for a, b in zip(out[:3], ref[:3]):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    return out[0], [[tuple(v) for v in out[4][q, :out[3][q]]] for q in range(len(paths))]


def test_polygonal_footprint_over_a_blocked_patch(oracle):
    patch = [(31, 31), (31, 32), (32, 31), (32, 32), (32, 33)]
    g, fp, L = _map(oracle, patch)
    pose = (X(32) - 0.125, Y(32) - 0.125)     # a cell corner: the footprint covers rows / columns 30 .. 33
    safe, poly = _polygonal(g, fp, L, [[pose]], 1)
    # lexicographic minimum (32, 33); (32, 32) lies on the edge to (32, 31) and is popped; counter-clockwise in (x, y)
    assert safe.tolist() == [0] and poly == [[P(32, 33), P(31, 32), P(31, 31), P(32, 31)]]
    safe, poly = _polygonal(g, fp, L, [[pose]], 0)
    assert safe.tolist() == [0] and poly == [[]]


def test_polygonal_path_reports_the_failing_segment(oracle):
    g, fp, L = _map(oracle, [(20, 32), (21, 32), (20, 33)])
    a, b, c, d = (X(40), Y(32)), (X(30), Y(32)), (X(20), Y(32)), (X(10), Y(32))
    safe, poly = _polygonal(g, fp, L, [[a, b, c, d], [a, b]], 1)
    assert safe.tolist() == [0, 1]
    assert poly == [[P(20, 32), P(20, 33), P(21, 32)], []]   # 3 cells in PolygonIterator order (rows, then columns)
