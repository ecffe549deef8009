"""The polygonal path check (checkPolygonalFootprintPath, TraversabilityMap.cpp:464-584 with isTraversable(polygon) :592-645) in
the CPU oracle, against values derived by hand.  Dyadic geometry throughout: 0.25 m cells on a 32 x 32 map centred on the origin
(cell centres x = 3.875 - 0.25 i, y = 3.875 - 0.25 j), dyadic vertices and poses, so no cell centre lies on a polygon edge and
every expected value below is exact."""
import numpy as np

import polygon_paths_oracle as ppo

RES, N = 0.25, 32
RECT = [(0.5, 0.25, 0.0), (-0.5, 0.25, 0.0), (-0.5, -0.25, 0.0), (0.5, -0.25, 0.0)]       # 1.0 x 0.5 m, centred
FWD = [(0.75, 0.25, 0.0), (-0.25, 0.25, 0.0), (-0.25, -0.25, 0.0), (0.75, -0.25, 0.0)]    # the same, shifted 0.25 m forward
IDENTITY = (0.0, 0.0, 0.0, 1.0)


def _row(i):
    return i / 64.0   # traversability of map row i (dyadic, exact in float32)


def _map(oracle, trav=None, rough_zero=(), default=0.3):
    g = oracle.Geometry.make(N, N, RES)
    one = np.ones((N, N), np.float32, order="F")
    t = np.asfortranarray(np.repeat(np.array([_row(i) for i in range(N)], np.float32)[:, None], N, axis=1)) if trav is None else trav
    rough = one.copy()
    for a, b in rough_zero:       # zero roughness traversability: a cell is blocked by checkForRoughness when 2+ such cells are near
        rough[a, b] = 0.0
    fp = oracle.FootprintParams.yaml_defaults()
    fp.verify_roughness = 1
    fp.traversability_default = default
    return g, fp, dict(traversability=t, slope=one, step=one, elevation=np.zeros((N, N), np.float32, order="F"), roughness=rough)


def _check(g, fp, L, footprint, paths, conservative=None, robot_slope=None):
    """paths: list of lists of poses (x, y) or (x, y, qx, qy, qz, qw)."""
    begin, poses = [0], []
    for path in paths:
        for p in path:
            x, y = p[0], p[1]
            q = p[2:] if len(p) > 2 else IDENTITY
            poses.append([x, y, 0.0, *q])
        begin.append(len(poses))
    return ppo.check_polygonal_paths(g, fp, L["traversability"], L["slope"], L["step"], L["elevation"], footprint, begin,
                                     np.asarray(poses, np.float64).reshape(-1, 7), robot_slope=robot_slope,
                                     roughness=L["roughness"], conservative=conservative)


def _mean_rows(rows):
    """Mean of the row traversabilities over x-cells `rows`, two y-cells each (the 0.5 m footprint depth)."""
    return sum(2 * _row(i) for i in rows) / (2 * len(rows))


def test_one_pose_uniform_traversability(oracle):
    trav = np.full((N, N), 0.625, np.float32, order="F")
    g, fp, L = _map(oracle, trav=trav)
    safe, t, area = _check(g, fp, L, RECT, [[(0.0, 0.0)]])
    assert safe.tolist() == [1] and t.tolist() == [0.625] and area.tolist() == [1.0 * 0.5]


def test_blocker_just_inside_and_just_outside(oracle):
    # cells (13, 15), (13, 16): x = 0.625, y = +-0.125; each sees the other's zero roughness -> both blocked (the sweep reduced to
    # the centre cell over a traversability of ones is 0 exactly at the blocked cells)
    g, fp, L = _map(oracle, rough_zero=[(13, 15), (13, 16)])
    f0 = oracle.FootprintParams.yaml_defaults()
    f0.radius, f0.offset, f0.verify_roughness = 0.0, 0.0, 1
    centre_only = oracle.footprint(g, f0, L["slope"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"])[0]
    assert sorted(zip(*np.nonzero(centre_only == 0.0))) == [(13, 15), (13, 16)]
    # front edge at x = 0.5625: the blocked centres at 0.625 lie 0.0625 outside; rows 14..17 inside
    safe, t, area = _check(g, fp, L, RECT, [[(0.0625, 0.0)]])
    assert safe.tolist() == [1] and t[0] == _mean_rows([14, 15, 16, 17]) and area[0] == 0.5
    # front edge at x = 0.6875: the blocked centres lie 0.0625 inside
    safe, t, area = _check(g, fp, L, RECT, [[(0.1875, 0.0)]])
    assert safe.tolist() == [0] and t.tolist() == [0.0] and area.tolist() == [0.0]


def test_yaw_180_on_an_asymmetric_footprint(oracle):
    g, fp, L = _map(oracle)
    safe, t, area = _check(g, fp, L, FWD, [[(0.0, 0.0)]])                                   # x in (-0.25, 0.75): rows 13..16
    assert safe.tolist() == [1] and t[0] == _mean_rows([13, 14, 15, 16]) == 14.5 / 64 and area[0] == 0.5
    safe, t, area = _check(g, fp, L, FWD, [[(0.0, 0.0, 0.0, 0.0, 1.0, 0.0)]])               # (qx, qy, qz, qw) = (0, 0, 1, 0)
    assert safe.tolist() == [1] and t[0] == _mean_rows([15, 16, 17, 18]) == 16.5 / 64 and area[0] == 0.5   # x in (-0.75, 0.25)


def test_non_unit_quaternion_and_vertex_z(oracle):
    """(qx, qy, qz, qw) = (0, 1, 0, 1) is used as given: row 0 of toRotationMatrix is (-1, 0, 2), so x = -v.x + 2 v.z + t.x."""
    g, fp, L = _map(oracle)
    fz = [(x, y, 0.5) for x, y, _ in FWD]                                                     # x = -v.x + 1.0: (0.25, 1.25)
    safe, t, area = _check(g, fp, L, fz, [[(0.0, 0.0, 0.0, 1.0, 0.0, 1.0)]])
    assert safe.tolist() == [1] and t[0] == _mean_rows([11, 12, 13, 14]) == 12.5 / 64 and area[0] == 0.5
    # the same vertices with z = 0 land on (-0.75, 0.25): the z column is live
    safe, t, _ = _check(g, fp, L, FWD, [[(0.0, 0.0, 0.0, 1.0, 0.0, 1.0)]])
    assert safe.tolist() == [1] and t[0] == _mean_rows([15, 16, 17, 18])


def test_two_and_three_poses_on_a_line(oracle):
    g, fp, L = _map(oracle)
    line = [(0.0, 0.0), (1.0, 0.0), (2.0, 0.0)]
    t1 = _mean_rows(range(10, 18))     # hull of poses 0, 1: x in (-0.5, 1.5), area 2.0 x 0.5
    t2 = _mean_rows(range(6, 14))      # hull of poses 1, 2: x in (0.5, 2.5)
    assert t1 == 13.5 / 64 and t2 == 9.5 / 64
    safe, t, area = _check(g, fp, L, RECT, [line[:2], line])
    assert safe.tolist() == [1, 1]
    assert area[0] == 1.0 and t[0] == t1
    a = 1.0 - 0.5                      # getArea(hull) - getArea(polygon1 = footprint at pose 1)
    assert area[1] == 1.0 + a and t[1] == (a * t2 + 1.0 * t1) / (1.0 + a)


def test_three_poses_conservative(oracle):
    """conservative: polygon1 of the second segment is the footprint at pose 1 listed three times (pose 1, pose 0 + d1, pose 2 - d2),
    and getArea of that concatenated list is 3 w h; the hulls are the same as without the flag."""
    g, fp, L = _map(oracle)
    line = [(0.0, 0.0), (1.0, 0.0), (2.0, 0.0)]
    t1, t2 = _mean_rows(range(10, 18)), _mean_rows(range(6, 14))
    safe, t, area = _check(g, fp, L, RECT, [line], conservative=[1])
    hull1 = hull2 = 1.0
    a = hull2 - 3 * 0.5
    assert safe.tolist() == [1] and area[0] == hull1 + hull2 - 3 * 0.5 == 0.5
    assert t[0] == (a * t2 + hull1 * t1) / (hull1 + a) == 17.5 / 64
    safe, t, area = _check(g, fp, L, RECT, [line[:2]], conservative=[1])   # one segment: hull of the doubled lists
    assert safe.tolist() == [1] and area[0] == 1.0 and t[0] == t1


def test_footprint_off_the_map(oracle):
    for default, want in ((0.3, ([1], [0.3], [0.5])), (0.0, ([0], [0.0], [0.0]))):
        g, fp, L = _map(oracle, default=default)
        safe, t, area = _check(g, fp, L, RECT, [[(10.0, 0.0)]])                              # the map spans -4 .. 4 m
        assert (safe.tolist(), t.tolist(), area.tolist()) == want
        safe, t, area = _check(g, fp, L, RECT, [[(10.0, 0.0), (10.0, 1.0)]])
        assert safe.tolist() == want[0] and t.tolist() == want[1]


def test_robot_slope_on_the_segment_line(oracle):
    g, fp, L = _map(oracle)
    path = [(0.0, 0.0), (1.0, 0.0)]                            # indices (16, 16) -> (12, 16)
    rs = np.ones((N, N), np.float32, order="F")
    rs[14, 16] = np.nan                                        # invalid cells are skipped
    safe, t, area = _check(g, fp, L, RECT, [path], robot_slope=rs)
    assert safe.tolist() == [1] and t[0] == _mean_rows(range(10, 18)) and area[0] == 1.0
    rs[14, 20] = 0.0                                           # off the line
    assert _check(g, fp, L, RECT, [path], robot_slope=rs)[0].tolist() == [1]
    rs[13, 16] = 0.0                                           # on the line
    safe, t, area = _check(g, fp, L, RECT, [path], robot_slope=rs)
    assert safe.tolist() == [0] and t.tolist() == [0.0] and area.tolist() == [0.0]
    # a single pose reads the layer at the pose; outside the map it is unsafe
    assert _check(g, fp, L, RECT, [[(0.75, 0.0)], [(0.5, 0.0)], [(10.0, 0.0)]], robot_slope=rs)[0].tolist() == [0, 1, 0]


def test_repeated_pose(oracle):
    g, fp, L = _map(oracle)
    single = _mean_rows([14, 15, 16, 17])
    safe, t, area = _check(g, fp, L, RECT, [[(0.0, 0.0)] * 2, [(0.0, 0.0)] * 3])
    assert safe.tolist() == [1, 1] and t.tolist() == [single, single] and area.tolist() == [0.5, 0.5]


def test_empty_path(oracle):
    g, fp, L = _map(oracle)
    safe, t, area = _check(g, fp, L, RECT, [[], [(0.0, 0.0)], []])
    assert safe.tolist() == [0, 1, 0] and t[0] == t[2] == 0.0 and area[0] == area[2] == 0.0 and area[1] == 0.5
