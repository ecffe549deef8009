"""The footprint inputs of tests/far_geometry.py are adversarial: far from the origin the tables a sweep classifies on offsets
relative to the centre, with the tolerances sized for a map near the origin, disagree with the reference's decisions on absolute
cell centres, and near the origin they do not.  The coordinate-scaled tolerances disagree nowhere.  And the oracle, at those
positions and footprints, is the literal restatement."""
import numpy as np
import pytest

import at_poses_oracle as apo
import far_geometry as fg

ROWS = COLS = 160
CIRCLES = [(0.02, r, o) for r, o in fg.band_radii(0.02, (625,))] + \
          [(0.01, r, o) for r, o in fg.band_radii(0.01, (900, 845))]
POLYGONS = [(res, pts, yaw) for res in (0.02, 0.01) for pts, yaw in fg.band_polygons(res)]   # rectangle, slanted edge, rotated


def _coord_max(pos, res):
    return max(abs(pos[0]) + 0.5 * ROWS * res, abs(pos[1]) + 0.5 * COLS * res)


def test_circular_band_disagrees_far_from_the_origin_only():
    far = 0
    for res, r, o in CIRCLES:
        rmax = r + o
        assert int(np.ceil(rmax / res)) <= 31
        parent = fg.circle_classes(rmax, res)
        for name, pos in fg.POSITIONS.items():
            bad = fg.circle_disagreements(rmax, res, pos, parent, ROWS, COLS)
            if name == "origin":
                assert bad == 0, (res, rmax)
            far += bad
            assert fg.circle_disagreements(rmax, res, pos, fg.circle_classes(rmax, res, _coord_max(pos, res)), ROWS, COLS) == 0
    assert far > 1000, far


def test_polygonal_band_disagrees_far_from_the_origin_only():
    far = {}
    for n, (res, pts, yaw) in enumerate(POLYGONS):
        assert fg.polygon_reach(pts, res) <= 31
        parent = fg.polygon_classes(pts, yaw, res)
        for name, pos in fg.POSITIONS.items():
            bad = fg.polygon_disagreements(pts, yaw, res, pos, parent, ROWS, COLS)
            if name == "origin":
                assert bad == 0, (res, yaw)
            far[(n, name)] = bad
            scaled = fg.polygon_classes(pts, yaw, res, _coord_max(pos, res))
            assert fg.polygon_disagreements(pts, yaw, res, pos, scaled, ROWS, COLS) == 0, (res, yaw, name)
    assert far[(3, "utm")] > 100 and far[(4, "utm")] > 0, far   # 0.01 m: the vertex y comparisons and the slanted x threshold


def test_rotated_band_footprints_reach_the_band():
    """The yaw of the rotated footprint puts an x threshold within 1.5 times the parent's tolerance of a lattice point: the
    coordinate-scaled tables leave it uncertain far out."""
    for res in (0.02, 0.01):
        pts, yaw = fg.band_polygons(res)[2]
        assert abs(yaw - 0.7854) < 0.05
        assert "on" not in fg.polygon_classes(pts, yaw, res).values()
        assert "on" in fg.polygon_classes(pts, yaw, res, _coord_max(fg.UTM, res)).values()


def _layers(oracle, res, pos, seed):
    g = oracle.Geometry.make(ROWS, COLS, res, pos)
    one = np.ones((ROWS, COLS), np.float32, order="F")
    return g, fg.distinct_layer(ROWS, COLS, seed), one, one.copy(), np.zeros((ROWS, COLS), np.float32, order="F")


@pytest.mark.parametrize("pos", ["origin", "lv95", "utm"])
def test_oracle_circular_footprint_is_the_literal_restatement(oracle, pos):
    for k, (res, r, o) in enumerate(CIRCLES[::3]):
        g, t, s, st, e = _layers(oracle, res, fg.POSITIONS[pos], 5 + k)
        fp = oracle.FootprintParams.yaml_defaults()
        fp.radius, fp.offset = r, o
        out, _, _ = oracle.footprint(g, fp, t, s, st, e)
        X, Y = fg.cell_tables(ROWS, COLS, res, fg.POSITIONS[pos])
        ci, cj = fg.centres(ROWS, COLS, 40, 60, k)
        for i, j in zip(ci, cj):
            assert out[i, j] == fg.circle_mean(t, X, Y, i, j, r + o, res), (res, r + o, i, j)


@pytest.mark.parametrize("pos", ["origin", "lv95", "utm"])
def test_oracle_polygon_footprint_is_the_literal_restatement(oracle, pos):
    for k, (res, pts, yaw) in enumerate(POLYGONS):
        g, t, s, st, e = _layers(oracle, res, fg.POSITIONS[pos], 9 + k)
        fp = oracle.FootprintParams.yaml_defaults()
        ox, orot = oracle.footprint_polygon(g, fp, [list(v) for v in pts], yaw, t, s, st, e)
        X, Y = fg.cell_tables(ROWS, COLS, res, fg.POSITIONS[pos])
        ci, cj = fg.centres(ROWS, COLS, 40, 40, k)
        for i, j in zip(ci, cj):
            assert ox[i, j] == fg.polygon_mean(t, X, Y, i, j, pts, 0.0, res), (res, i, j)
            assert orot[i, j] == fg.polygon_mean(t, X, Y, i, j, pts, yaw, res), (res, yaw, i, j)


@pytest.mark.parametrize("res", [0.02, 0.01])
@pytest.mark.parametrize("pos", ["origin", "lv95", "utm"])
def test_oracle_at_poses_indexes_like_get_index(oracle, pos, res):
    """teo_at_poses at poses on and one nextafter either side of absolute cell edges (a centre plus or minus half a cell), identity
    orientation and a zero point: the cell is the one getIndexFromPosition finds."""
    p = fg.POSITIONS[pos]
    og = oracle.Geometry.make(ROWS, COLS, res, p)
    layer = np.asfortranarray(1000.0 * np.arange(ROWS)[:, None] + np.arange(COLS)[None, :], dtype=np.float32)
    X, Y = fg.cell_tables(ROWS, COLS, res, p)
    edges = lambda T: [v for c in T[::9] for e in (c + 0.5 * res, c - 0.5 * res)   # noqa: E731
                       for v in (np.nextafter(e, -np.inf), e, np.nextafter(e, np.inf))]
    xy = [(x, y) for x in edges(X) for y in edges(Y)[::5]] + [(x, Y[50]) for x in edges(X)]
    poses = [(x, y, 0.0, 0.0, 0.0, 0.0, 1.0) for x, y in xy]
    vals, ok = apo.at_poses(og, layer, poses, [(0.0, 0.0, 0.0)])
    for (x, y), v, k in zip(xy, vals[:, 0], ok[:, 0]):
        i, j, inside = fg.get_index(ROWS, COLS, res, p, x, y)
        assert k == int(inside), (x, y)
        if inside:
            assert v == layer[i, j], (x, y, i, j)
