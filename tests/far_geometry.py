"""A literal fp64 restatement of the reference's membership decisions, and generators of footprints that put lattice offsets in the
band where a table classified on offsets relative to the centre and the reference's arithmetic on absolute cell centres can
disagree once the map sits far from the origin.

Python floats and numpy float64 element-wise operations are IEEE doubles without contraction, so every expression below rounds
exactly as grid_map's does in its operand order:
  - cell_coord: getPositionFromIndex;
  - circle_inside: SpiralIterator::isInside and CircleIterator::isInside, (position - centre).squaredNorm() <= r^2;
  - place_polygon / polygon_inside: the footprint placed by toPosition * Quaternion * v, and Polygon::isInside;
  - get_index: getIndexFromPosition.
"""
import math

import numpy as np

ORIGIN = (0.0, 0.0)
LV95 = (2_600_000.25, 1_200_000.75)    # a Swiss LV95 easting / northing
UTM = (465_000.5, 5_247_000.5)         # a UTM easting / northing
POSITIONS = {"origin": ORIGIN, "lv95": LV95, "utm": UTM}

YAML_POLYGON = [(0.45, 0.30), (0.45, -0.30), (-0.45, -0.30), (-0.45, 0.30)]   # robot_footprint_parameter.yaml:3
SMALL_POLYGON = [(0.2, 0.15), (0.2, -0.15), (-0.2, -0.15), (-0.2, 0.15)]       # reach 0.25 m: 26 cells at 0.01 m


# ---- grid_map ---------------------------------------------------------------------------------------------------------------

def cell_coord(map_pos, length, res, idx):
    """getPositionFromIndex along one axis; idx may be a numpy integer array."""
    return (map_pos + (0.5 * length - 0.5 * res)) + res * (-np.asarray(idx, dtype=np.float64))


def cell_tables(rows, cols, res, pos):
    """Cell-centre coordinates X (rows) and Y (columns) of a map of rows x cols cells at `pos`."""
    return (cell_coord(pos[0], rows * res, res, np.arange(rows)), cell_coord(pos[1], cols * res, res, np.arange(cols)))


def get_index(rows, cols, res, pos, px, py):
    """getIndexFromPosition with isInside: (i, j, inside)."""
    lx, ly = rows * res, cols * res
    vx = ((px - 0.5 * lx) - pos[0]) / res
    vy = ((py - 0.5 * ly) - pos[1]) / res
    tx = -((px - pos[0]) - 0.5 * lx)
    ty = -((py - pos[1]) - 0.5 * ly)
    i, j = int(-vx), int(-vy)
    inside = tx >= 0.0 and ty >= 0.0 and tx < lx and ty < ly
    return i, j, inside and 0 <= i < rows and 0 <= j < cols


def circle_inside(xa, yb, cx, cy, r2):
    """SpiralIterator::isInside / CircleIterator::isInside of cell centre (xa, yb) for the circle of squared radius r2 at
    (cx, cy); numpy arrays broadcast."""
    dx, dy = xa - cx, yb - cy
    return dx * dx + dy * dy <= r2


def yaw_rotation(yaw):
    """Upper-left 2 x 2 of Eigen's toRotationMatrix of the quaternion (cos(yaw/2), 0, 0, sin(yaw/2)), in its operand order."""
    w, z = math.cos(0.5 * yaw), math.sin(0.5 * yaw)
    tz = 2.0 * z
    twz, tzz = tz * w, tz * z
    return (1.0 - (0.0 + tzz), 0.0 - twz, 0.0 + twz, 1.0 - (0.0 + tzz))


def rotate(pts, R):
    """The footprint's vertices rotated, relative to the centre: linear() * v (the z column is zero)."""
    return [((R[0] * px + R[1] * py) + 0.0, (R[2] * px + R[3] * py) + 0.0) for px, py in pts]


def place_polygon(rel, cx, cy):
    """Vertices at the centre (cx, cy): translation() + R v, with rel = rotate(pts, R).  cx, cy may be arrays."""
    return [(cx + rx, cy + ry) for rx, ry in rel]


def polygon_inside(poly, x, y):
    """grid_map::Polygon::isInside (crossing number), element-wise over numpy arrays."""
    cross = np.zeros(np.broadcast(x, y, *[c for v in poly for c in v]).shape, dtype=np.int64)
    n = len(poly)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(n):
            j = (i - 1) % n
            (xi, yi), (xj, yj) = poly[i], poly[j]
            straddle = (yi > y) != (yj > y)
            thr = (xj - xi) * (y - yi) / (yj - yi) + xi
            cross += straddle & (x < thr)
    return (cross % 2) != 0


# ---- the tables classified on relative offsets ------------------------------------------------------------------------------

def coord_ulp(m):
    """Spacing of the doubles at max(m, 1)."""
    return math.ldexp(1.0, math.frexp(max(m, 1.0))[1] - 53)


def circle_classes(rmax, res, coord_max=None):
    """{(k, l): 'in' | 'on' | 'out'} of every offset within nRings + 1, as the circular sweep's tables classify them: the
    parent's tolerance 1e-9 r^2 without coord_max, the coordinate-scaled one max(1e-9 r^2, 8 r ulp(M)) with it (M = coord_max +
    rmax).  'on' offsets are decided per centre on absolute positions."""
    r2 = rmax * rmax
    tol_far = 8.0 * rmax * coord_ulp(coord_max + rmax) if coord_max is not None else 0.0
    tol = max(1e-9 * r2, tol_far) + 1e-300
    L = int(math.floor(rmax / res + 1e-9))
    while float((L + 1) * (L + 1)) * res * res <= r2 + tol_far:
        L += 1
    n = int(math.ceil(rmax / res)) + 1
    out = {}
    for l in range(-n, n + 1):
        for k in range(-n, n + 1):
            d2 = float(k * k + l * l) * res * res
            if abs(k) <= L and abs(l) <= L and d2 < r2 - tol:
                out[(k, l)] = "in"
            elif abs(k) <= L and abs(l) <= L and abs(d2 - r2) <= tol:
                out[(k, l)] = "on"
            else:
                out[(k, l)] = "out"
    return out


def polygon_reach(pts, res):
    return int(math.ceil(max(math.hypot(x, y) for x, y in pts) / res)) + 1


def polygon_classes(pts, yaw, res, coord_max=None):
    """{(di, dj): 'in' | 'on' | 'out'} of classify_polygon: the parent's tolerance 1e-7 res without coord_max, the
    coordinate-scaled ones with it (4 ulp(M) for the y comparisons, 8 (1 + |slope|) ulp(M) for the x thresholds)."""
    Lp = polygon_reach(pts, res)
    rel = rotate(pts, yaw_rotation(yaw))
    vx = [v[0] for v in rel]
    vy = [v[1] for v in rel]
    cu = coord_ulp(coord_max + Lp * res) if coord_max is not None else 0.0
    tol = max(1e-7 * res, 4.0 * cu)
    n = len(rel)
    out = {}
    for dj in range(-Lp, Lp + 1):
        for di in range(-Lp, Lp + 1):
            ptx, pty = -res * di, -res * dj
            cross, fuzzy = 0, False
            for i in range(n):
                j = (i - 1) % n
                if vy[i] == vy[j]:
                    continue
                ui, uj = abs(vy[i] - pty) < tol, abs(vy[j] - pty) < tol
                fuzzy |= ui or uj
                ci, cj = vy[i] > pty, vy[j] > pty
                if ci != cj or ui or uj:
                    thr = (vx[j] - vx[i]) * (pty - vy[i]) / (vy[j] - vy[i]) + vx[i]
                    tol_x = max(tol, 8.0 * (1.0 + abs((vx[j] - vx[i]) / (vy[j] - vy[i]))) * cu)
                    if abs(ptx - thr) < tol_x or abs(vy[j] - vy[i]) < 1e3 * tol:
                        fuzzy = True
                    if ci != cj and ptx < thr:
                        cross += 1
            out[(di, dj)] = "on" if fuzzy else ("in" if cross & 1 else "out")
    return out


# ---- disagreements between the tables and the absolute decisions -------------------------------------------------------------

def centres(rows, cols, margin, count, seed):
    """`count` random centres (i, j) at least `margin` cells from the border."""
    rng = np.random.default_rng(seed)
    return rng.integers(margin, rows - margin, count), rng.integers(margin, cols - margin, count)


def circle_disagreements(rmax, res, pos, classes, rows=160, cols=160, ncentres=200, seed=0):
    """(centre, offset) pairs where `classes` says 'in' or 'out' and the reference's absolute test says otherwise."""
    X, Y = cell_tables(rows, cols, res, pos)
    ci, cj = centres(rows, cols, 40, ncentres, seed)
    cx, cy, r2 = X[ci], Y[cj], rmax * rmax
    bad = 0
    for (k, l), c in classes.items():
        if c == "on":
            continue
        inside = circle_inside(X[ci + k], Y[cj + l], cx, cy, r2)
        bad += int((inside != (c == "in")).sum())
    return bad


def polygon_disagreements(pts, yaw, res, pos, classes, rows=160, cols=160, ncentres=200, seed=0):
    X, Y = cell_tables(rows, cols, res, pos)
    ci, cj = centres(rows, cols, 40, ncentres, seed)
    poly = place_polygon(rotate(pts, yaw_rotation(yaw)), X[ci], Y[cj])
    bad = 0
    for (di, dj), c in classes.items():
        if c == "on":
            continue
        inside = polygon_inside(poly, X[ci + di], Y[cj + dj])
        bad += int((inside != (c == "in")).sum())
    return bad


# ---- generators --------------------------------------------------------------------------------------------------------------

def band_radii(res, norms, cs=(1.2, -1.2, 1.45, -1.45), offset=0.15):
    """(radius, offset) pairs whose rmax = radius + offset has rmax^2 = n res^2 + c * 1e-9 rmax^2 for the lattice norms n:
    the parent's tables call the offsets of norm n certainly inside (c > 1) or certainly outside (c < -1) while the reference's
    absolute test far from the origin moves them by more than that."""
    out = []
    for n in norms:
        for c in cs:
            rmax = math.sqrt(n * res * res * (1.0 + c * 1e-9))
            out.append((rmax - offset, offset))
    return out


def _edge_band_shift(rel_edge, res, target):
    """Horizontal shift of edge ((xi, yi), (xj, yj)) that puts its x threshold at a lattice row pt.x + target for the lattice
    column pt.y nearest the middle of the edge."""
    (xi, yi), (xj, yj) = rel_edge
    pty = -res * round(-0.5 * (yi + yj) / res)
    thr = (xj - xi) * (pty - yi) / (yj - yi) + xi
    ptx = -res * round(-thr / res)
    return (ptx + target) - thr


def band_polygons(res):
    """(points, yaw) footprints with comparisons 1.2 - 1.45 times the parent's tolerance (1e-7 res) from lattice offsets:
      - an axis-aligned rectangle whose half sizes are a lattice distance plus delta (the y comparison of a vertex, and the x
        threshold of a vertical edge);
      - a quadrilateral with a slanted edge whose x threshold passes delta from a lattice point;
      - the YAML rectangle (at 0.02 m; a smaller one at 0.01 m) at a yaw near 0.7854 chosen so that a rotated edge's x threshold
        passes delta from a lattice point."""
    tol = 1e-7 * res
    big = res >= 0.02
    # half sizes whose vertex comparisons the UTM position's rounding flips at 0.01 m (14 cells; none flips at 0.02 m)
    a, b = (0.44, 0.30) if big else (0.18, 0.14)
    out = [([(a + 1.05 * tol, b + 1.05 * tol), (a + 1.05 * tol, -b - 1.05 * tol), (-a - 1.05 * tol, -b - 1.05 * tol),
             (-a - 1.05 * tol, b + 1.05 * tol)], 0.0)]
    s = 2.0 if big else 1.0
    quad = [(0.1913 * s, -0.0437 * s), (-0.0929 * s, 0.0561 * s), (-0.1811 * s, -0.1633 * s), (0.1707 * s, -0.1519 * s)]
    for _ in range(3):   # the shift is linear in x up to rounding: a few rounds settle it
        d = _edge_band_shift((quad[1], quad[0]), res, 1.05 * tol)
        quad[0] = (quad[0][0] + d, quad[0][1])
        quad[1] = (quad[1][0] + d, quad[1][1])
    out.append((quad, 0.0))
    rect = YAML_POLYGON if big else SMALL_POLYGON
    out.append((rect, rotated_band_yaw(rect, res, 0.7854, 1.05 * tol)))
    return out


def _threshold_gap(rel, res, edge, di, dj):
    (xi, yi), (xj, yj) = rel[edge], rel[edge - 1]
    ptx, pty = -res * di, -res * dj
    return ptx - ((xj - xi) * (pty - yi) / (yj - yi) + xi)


def rotated_band_yaw(pts, res, yaw0, target):
    """A yaw near yaw0 at which edge 0 -> n-1 of the rotated polygon has its x threshold `target` from a lattice point: of the
    lattice points next to the edge at yaw0, the nearest one, then a secant solve in the yaw."""
    rel = rotate(pts, yaw_rotation(yaw0))
    (xi, yi), (xj, yj) = rel[0], rel[-1]
    best = None
    for dj in range(int(math.ceil(-max(yi, yj) / res)) + 1, int(math.floor(-min(yi, yj) / res))):
        thr = (xj - xi) * (-res * dj - yi) / (yj - yi) + xi
        di = round(-thr / res)
        gap = abs(_threshold_gap(rel, res, 0, di, dj))
        if best is None or gap < best[0]:
            best = (gap, di, dj)
    _, di, dj = best
    f = lambda y: _threshold_gap(rotate(pts, yaw_rotation(y)), res, 0, di, dj) - target   # noqa: E731
    y0, y1 = yaw0, yaw0 + 1e-4
    f0, f1 = f(y0), f(y1)
    for _ in range(100):
        if f1 == f0 or abs(f1) < 0.05 * target:
            break
        y0, y1, f0 = y1, y1 - f1 * (y1 - y0) / (f1 - f0), f1
        f1 = f(y1)
    return y1


# ---- isTraversable on a layer without blocked cells ------------------------------------------------------------------------

def distinct_layer(rows, cols, seed):
    """float32 traversability with a distinct value per cell in [0.25, 0.75): one cell more or less in a footprint moves its mean
    by about 1e-4, far beyond a float32 rounding, and double sums of these values are exact in any order."""
    rng = np.random.default_rng(seed)
    v = (0.25 + 0.5 * rng.permutation(rows * cols) / (rows * cols)).astype(np.float32)
    return np.asfortranarray(v.reshape(rows, cols))


def circle_mean(trav, X, Y, i, j, rmax, res):
    """isTraversable(centre of cell (i, j), rmax) with no blocked cell: the mean of the SpiralIterator's cells, the rings before
    nRings - 1 whole and the last two tested on absolute centres, as float32."""
    n_rings = int(math.ceil(rmax / res))
    r2 = rmax * rmax
    t, n = 0.0, 0
    for k in range(-n_rings - 1, n_rings + 2):
        for l in range(-n_rings - 1, n_rings + 2):
            ring = math.isqrt(k * k + l * l)
            if ring > n_rings:
                continue
            if ring >= max(n_rings - 1, 1) and not circle_inside(X[i + k], Y[j + l], X[i], Y[j], r2):
                continue
            t += float(trav[i + k, j + l])
            n += 1
    return np.float32(t / n)


def polygon_mean(trav, X, Y, i, j, pts, yaw, res):
    """isTraversable(footprint polygon at yaw placed at the centre of cell (i, j)) with no blocked cell, as float32."""
    Lp = polygon_reach(pts, res)
    poly = place_polygon(rotate(pts, yaw_rotation(yaw)), X[i], Y[j])
    a = np.arange(i - Lp, i + Lp + 1)[:, None]
    b = np.arange(j - Lp, j + Lp + 1)[None, :]
    inside = polygon_inside(poly, X[a], Y[b])
    vals = trav[i - Lp:i + Lp + 1, j - Lp:j + Lp + 1][inside].astype(np.float64)
    return np.float32(vals.sum() / len(vals)) if len(vals) else None
