"""The fresh-cache circular path check (checkCircularFootprintPath on an empty traversability_footprint layer,
TraversabilityMap.cpp:345-462 with :679-736) in the CPU oracle, against answers derived by hand on constant maps: traversability
0.8 everywhere, cells blocked by patches of zero roughness traversability (verify_roughness, checkForRoughness :895-921)."""
import numpy as np

import paths_fresh_oracle as pfo

RES = 0.02


def _cell(g, i, j):
    """grid_map::getPosition of cell (i, j), in the library's operand order."""
    return ((g.position_x + (0.5 * g.length_x - 0.5 * RES)) + RES * (-float(i)),
            (g.position_y + (0.5 * g.length_y - 0.5 * RES)) + RES * (-float(j)))


def _map(oracle, rows, cols, patches):
    g = oracle.Geometry.make(rows, cols, RES)
    one = np.ones((rows, cols), np.float32, order="F")
    trav = np.full((rows, cols), 0.8, np.float32, order="F")
    rough = one.copy()
    for a, b in patches:                           # 7 x 7 patches of zero roughness traversability, top-left corner (a, b)
        rough[a:a + 7, b:b + 7] = 0.0
    fp = oracle.FootprintParams.yaml_defaults()
    fp.verify_roughness = 1
    z = np.zeros((rows, cols), np.float32, order="F")
    # which cells isTraversableForFilters blocks: the sweep degenerated to the centre cell (0 = blocked, else 0.8)
    f0 = oracle.FootprintParams.yaml_defaults()
    f0.radius, f0.offset, f0.verify_roughness = 0.0, 0.0, 1
    centre_only = oracle.footprint(g, f0, trav, one, one, z, roughness=rough)[0]
    blocked = centre_only == 0.0
    assert blocked.any() and set(np.unique(centre_only)) <= {np.float32(0.0), np.float32(0.8)}
    return g, fp, dict(traversability=trav, slope=one, step=one, elevation=z, roughness=rough), blocked


def _fresh(g, fp, L, poses, radius=0.3, cup=None, begin=None):
    poses = np.asarray(poses, dtype=np.float64).reshape(-1, 2)
    begin = [0, len(poses)] if begin is None else begin
    n = len(begin) - 1
    return pfo.check_circular_paths_fresh(g, fp, L["traversability"], L["slope"], L["step"], L["elevation"], begin, poses,
                                          [radius] * n, roughness=L["roughness"],
                                          compute_untraversable_polygon=None if cup is None else [cup] * n)


def _sweep_then_memo(oracle, g, fp, L, poses):
    """INTEGRATION.md route: the full sweep traversabilityFootprint(radius, offset), then the memoised path check."""
    fpl = oracle.footprint(g, fp, L["traversability"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"])[0]
    poses = np.asarray(poses, dtype=np.float64).reshape(-1, 2)
    return oracle.check_circular_paths(g, fpl, fp.traversability_default, [0, len(poses)], poses), fpl


def _first_blocked(oracle, blocked, ci, cj, rmax):
    """(n, di, dj): cells visited before the first blocked one of SpiralIterator(rmax) around (ci, cj), and its offset."""
    di, dj = oracle.spiral_offsets(rmax, RES)
    for k in range(len(di)):
        if blocked[ci + di[k], cj + dj[k]]:
            return k, int(di[k]), int(dj[k])
    raise AssertionError("no blocked cell in the disk")


def test_annulus_blocker_single_pose_at_cell_centre(oracle):
    g, fp, L, blocked = _map(oracle, 64, 64, [(51, 29)])   # the patch lies 19-25 rows below the centre cell (32, 32)
    pose = [_cell(g, 32, 32)]
    n, di, dj = _first_blocked(oracle, blocked, 32, 32, 0.45)
    uR = int(np.sqrt(di * di + dj * dj)) * RES            # getCurrentRadius with Eigen's integer norm
    assert 0.3 < uR <= 0.45 and n > 1000
    factor = ((uR - 0.3) / (0.45 - 0.3) + 1.0) / 2.0
    t = np.float64(n) * np.float64(np.float32(0.8))        # n terms of 0.8f added in double: exact
    # sweep + memo: the scaled value, stored as float32, makes the circle traversable (:673-675)
    (safe, val), fpl = _sweep_then_memo(oracle, g, fp, L, pose)
    assert safe.tolist() == [1] and val[0] == np.float64(np.float32(t * (factor / n)))
    assert fpl[32, 32] == np.float32(t * (factor / n))
    # fresh: the same value is stored, but isTraversable returns false (:705-716)
    safe, val = _fresh(g, fp, L, pose)
    assert safe.tolist() == [0] and val.tolist() == [0.0]
    # compute_untraversable_polygon: the loop ends traversable and divides by nCells a second time (:707, :733), in double
    safe, val = _fresh(g, fp, L, pose, cup=1)
    assert safe.tolist() == [1] and val[0] == (t * (factor / n)) / n


def test_blocker_within_inner_radius(oracle):
    g, fp, L, blocked = _map(oracle, 64, 64, [(41, 29)])   # nearest blocked cell 10 rows away: 0.2 m <= radius 0.3
    pose = [_cell(g, 32, 32)]
    _, di, dj = _first_blocked(oracle, blocked, 32, 32, 0.45)
    assert int(np.sqrt(di * di + dj * dj)) * RES <= 0.3
    (safe, _), fpl = _sweep_then_memo(oracle, g, fp, L, pose)
    assert safe.tolist() == [0] and fpl[32, 32] == 0.0
    for cup in (None, 1):
        safe, val = _fresh(g, fp, L, pose, cup=cup)
        assert safe.tolist() == [0] and val.tolist() == [0.0]


def test_pose_off_its_cell_centre(oracle):
    """SpiralIterator(map, pose, rMax) tests the last two rings against the pose, not against its cell centre."""
    g, fp, L, blocked = _map(oracle, 64, 64, [(52, 23)])
    cx, cy = _cell(g, 32, 20)
    px, py = cx - 0.45 * RES, cy                            # 0.45 cells toward the patch; still inside cell (32, 20)
    a, b = np.nonzero(blocked)
    X = np.array([_cell(g, i, 0)[0] for i in range(64)])
    Y = np.array([_cell(g, 0, j)[1] for j in range(64)])
    d_cell = np.sqrt((X[a] - cx) ** 2 + (Y[b] - cy) ** 2).min()
    d_pose = np.sqrt((X[a] - px) ** 2 + (Y[b] - py) ** 2).min()
    assert d_cell > 0.45 >= d_pose > 0.3                  # outside the circle around the cell centre, inside the one around the pose
    safe, val = _fresh(g, fp, L, [(cx, cy)])
    assert safe.tolist() == [1] and val[0] == np.float64(np.float32(0.8))
    safe, _ = _fresh(g, fp, L, [(px, py)])
    assert safe.tolist() == [0]                             # an annulus blocker the cell centre does not see
    safe, val = _fresh(g, fp, L, [(px, py)], cup=1)
    assert safe.tolist() == [1] and 0.0 < val[0] < 0.8
    (safe, val), _ = _sweep_then_memo(oracle, g, fp, L, [(px, py)])
    assert safe.tolist() == [1] and val[0] == np.float64(np.float32(0.8))   # the swept layer holds the cell centre's answer


def test_revisited_centres_read_the_float32_cache(oracle):
    """Within a path, a centre an earlier segment checked reads back the float32 value its first check stored (:673-675)."""
    rows = cols = 64
    g = oracle.Geometry.make(rows, cols, RES)
    rng = np.random.default_rng(5)
    trav = np.asfortranarray(rng.uniform(0.3, 1.0, (rows, cols)).astype(np.float32))
    trav[40:, 30:] = 0.0                                    # a region of zero traversability (not blocked: no filter fails)
    one = np.ones((rows, cols), np.float32, order="F")
    z = np.zeros((rows, cols), np.float32, order="F")
    L = dict(traversability=trav, slope=one, step=one, elevation=z, roughness=one)
    fp = oracle.FootprintParams.yaml_defaults()
    radius = 0.05                                           # radiusMax 0.2 m = 10 cells

    def single(i, j):
        s, t = _fresh(g, fp, L, [_cell(g, i, j)], radius=radius)
        assert s[0] == 1
        return t[0]

    def seg_len(p, q):
        (x0, y0), (x1, y1) = _cell(g, *p), _cell(g, *q)
        return np.sqrt((x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0))

    f32 = lambda v: np.float64(np.float32(v))  # noqa: E731
    A, M, B, N, C = (20, 12), (20, 16), (20, 20), (24, 20), (28, 20)   # both lines have 9 cells (= 1 mod 4): cells 0, 4, 8 checked
    fA, fM, fB, fN, fC = (single(*c) for c in (A, M, B, N, C))
    assert all(f32(v) != v for v in (fA, fM, fB))            # the float32 cache really differs from the double means

    def path(cells):
        poses = [_cell(g, *c) for c in cells]
        return _fresh(g, fp, L, poses, radius=radius)

    # A -> B -> A: the second segment (line from A to B) revisits A, M and B
    s, t = path([A, B, A])
    t1 = ((fB + fM) + fA) / 3.0
    t2 = ((f32(fA) + f32(fM)) + f32(fB)) / 3.0
    l1, l2 = seg_len(A, B), seg_len(B, A)
    assert s[0] == 1 and t[0] == (l2 * t2 + l1 * t1) / (l1 + l2)
    # A -> B -> C: the line from C to B ends on B, which the first segment checked first
    s, t = path([A, B, C])
    t2 = ((fC + fN) + f32(fB)) / 3.0
    l2 = seg_len(B, C)
    assert s[0] == 1 and t[0] == (l2 * t2 + l1 * t1) / (l1 + l2)
    # a revisited centre whose mean is exactly 0: traversable on its first check, untraversable when read back
    A3, M3, B3 = (52, 36), (52, 40), (52, 44)
    fA3, fM3, fB3 = (single(*c) for c in (A3, M3, B3))
    assert fM3 == 0.0 and fB3 == 0.0 and fA3 > 0.0
    s, t = path([A3, B3])
    assert s[0] == 1 and t[0] == ((fB3 + fM3) + fA3) / 3.0
    s, t = path([A3, B3, A3])
    assert s[0] == 0 and t[0] == 0.0
