"""The maps and requests of the path-check parameter tests (test_paths_params_gpu.py, test_paths_params_cpu.py).

A request is a dict: begin (npaths + 1), poses (nposes, 7), radius, kind (-1 circular, else an index into fps), cons, cup, fps.

The replay constructions put two or more circular single poses on one cell of a 40 x 40 map at 0.02 m (traversability 0.5,
max_gap_width 0.001 so that a zero-slope cell blocks alone).  Their first walk stores a NaN or an infinity at the cell, which the
reference does not treat as cached (isValid), so every later check there walks again with its own radius and flag:
  - nan_case: an invalid traversability cell next to the centre under a NaN or infinite default, and a blocker 12 cells out, beyond
    the inner radius of radius 0.2 (10 cells) and inside radiusMax 0.35.  cup = 1 walks on past the blocker and stores the
    non-finite mean; cup = 0 stops there, untraversable.
  - ring_case: offset 0 (radiusMax == radiusMin), the exact norm, a blocker at index offset (-10, -3) (norm 10.44 cells, beyond
    the inner radius) and the pose moved 0.45 cell toward it, so that the blocker is inside the circle: the ring factor
    (uR - rmin) / (rmax - rmin) is infinite.  With the integer norm the blocker lies on the inner radius and blocks."""
import math

import numpy as np

import far_geometry as fg

RES, N, CENTRE = 0.02, 40, 20
REPLAY_GAP = dict(max_gap_width=0.001)
IDENTITY = [0.0, 0.0, 0.0, 0.0, 1.0]   # z qx qy qz qw of a circular path's pose


def cells():
    return fg.cell_tables(N, N, RES, (0.0, 0.0))


def flat_map(invalid=(), blockers=()):
    """The replay map: traversability 0.5 with the `invalid` cells NaN, zero slope at the `blockers`."""
    t = np.full((N, N), 0.5, np.float32, order="F")
    for a, b in invalid:
        t[a, b] = np.nan
    slope = np.ones((N, N), np.float32, order="F")
    for a, b in blockers:
        slope[a, b] = 0.0
    one = np.ones((N, N), np.float32, order="F")
    return dict(traversability=t, slope=slope, step=one, roughness=one.copy(), elevation=np.zeros((N, N), np.float32, order="F"))


def request(paths, fps=()):
    """A request of `paths`: (poses (n, 2) or (n, 7), radius, footprint index or -1, cons, cup) each."""
    begin, poses, radius, kind, cons, cup = [0], [], [], [], [], []
    for p, r, k, c, u in paths:
        p = np.asarray(p, np.float64).reshape(len(p), -1)
        if p.shape[1] == 2:
            p = np.concatenate([p, np.tile(IDENTITY, (len(p), 1))], axis=1)
        poses.extend(p.tolist())
        begin.append(len(poses))
        radius.append(r)
        kind.append(k)
        cons.append(c)
        cup.append(u)
    return dict(begin=np.asarray(begin, np.int32), poses=np.asarray(poses, np.float64).reshape(-1, 7),
                radius=np.asarray(radius, np.float64), kind=np.asarray(kind), cons=np.asarray(cons, np.uint8),
                cup=np.asarray(cup, np.uint8), fps=list(fps))


def single(xy, radius, cup):
    return ([xy], radius, -1, 0, cup)


def centre_xy():
    X, Y = cells()
    return (float(X[CENTRE]), float(Y[CENTRE]))


def nan_case(default, cups=(1, 0), radii=(0.2, 0.2), fillers=0):
    """(map, parameters, request): single poses at the centre cell, one per entry of cups / radii, with `fillers` single poses on
    other cells between the first and the second (32 or more put them in different windows of the replay)."""
    m = flat_map(invalid=[(CENTRE + 1, CENTRE)], blockers=[(CENTRE + 12, CENTRE)])
    c = centre_xy()
    X, Y = cells()
    paths = [single(c, radii[0], cups[0])]
    for k in range(fillers):   # cells 4 to 7 rows up and across, away from the centre's cell
        paths.append(single((float(X[CENTRE - 4 - k % 4]), float(Y[4 + k % 32])), 0.1, k % 2))
    paths += [single(c, r, u) for r, u in zip(radii[1:], cups[1:])]
    return m, dict(traversability_default=default, **REPLAY_GAP), request(paths)


def ring_pose():
    """The pose of ring_case: the centre cell's centre moved 0.45 cell toward the blocker."""
    X, Y = cells()
    cx, cy = float(X[CENTRE]), float(Y[CENTRE])
    bx, by = float(X[CENTRE - 10]), float(Y[CENTRE - 3])
    d = math.hypot(bx - cx, by - cy)
    return (cx + 0.45 * RES * (bx - cx) / d, cy + 0.45 * RES * (by - cy) / d)


def ring_case(norm=0, cups=(1, 0), radii=(0.2, 0.2)):
    m = flat_map(blockers=[(CENTRE - 10, CENTRE - 3)])
    p = ring_pose()
    kw = dict(offset=0.0, traversability_default=0.3, radius_is_integer_norm=norm, **REPLAY_GAP)
    return m, kw, request([single(p, r, u) for r, u in zip(radii, cups)])


def mixed_case(default):
    """Lanes of one cell where a walk stores a finite value after non-finite ones: the invalid cell 8 cells out, beyond radiusMax
    0.15 of radius 0 and inside that of radius 0.2 (0.35); the blocker 12 cells out.  Radius 0.2 stores the non-finite mean,
    radius 0 a finite one that every later check reads, cup = 0 included."""
    m = flat_map(invalid=[(CENTRE + 8, CENTRE)], blockers=[(CENTRE + 12, CENTRE)])
    c = centre_xy()
    paths = [single(c, 0.2, 1), single(c, 0.2, 1), single(c, 0.0, 1), single(c, 0.2, 0), single(c, 0.2, 1)]
    return m, dict(traversability_default=default, **REPLAY_GAP), request(paths)
