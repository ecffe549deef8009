"""Helpers shared by the tests: layer comparison (SURVEY.md §8d tolerances), bit-for-bit comparison, and the maps, paths,
footprints and requests of the footprint path-check tests."""
import numpy as np

RTOL, ATOL = 1e-5, 1e-6  # |a-b| <= RTOL*|b| + ATOL ; NaN positions and exact 0.0/1.0 cells must match exactly


def compare_layer(got, ref, name=""):
    got = np.asarray(got)
    ref = np.asarray(ref)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    nan_mismatch = int((np.isnan(got) != np.isnan(ref)).sum())
    both = ~np.isnan(got) & ~np.isnan(ref)
    diff = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    tol = RTOL * np.abs(ref.astype(np.float64)) + ATOL
    out_of_tol = int((both & (diff > tol)).sum())
    rel_only = int((both & (diff > RTOL * np.abs(ref.astype(np.float64)))).sum())
    branch = both & ((ref == 0.0) | (ref == 1.0))
    branch_mismatch = int((branch & (got != ref)).sum())
    bit_exact = int((got.view(np.uint32) == ref.view(np.uint32)).sum()) + int((np.isnan(got) & np.isnan(ref)).sum()) \
        - int(((got.view(np.uint32) == ref.view(np.uint32)) & np.isnan(got)).sum())
    return {"name": name, "cells": got.size, "nan_mismatch": nan_mismatch, "out_of_tol": out_of_tol,
            "rel_only_violations": rel_only, "branch_mismatch": branch_mismatch, "bit_exact": bit_exact,
            "max_abs": float(diff[both].max()) if both.any() else 0.0}


def assert_parity(got: dict, ref: dict, keys=("slope", "step", "roughness", "traversability"), allow_out_of_tol=0):
    reports = [compare_layer(got[k], ref[k], k) for k in keys]
    for r in reports:
        assert r["nan_mismatch"] == 0, r
        assert r["out_of_tol"] <= allow_out_of_tol, r
        assert r["branch_mismatch"] <= allow_out_of_tol, r
    return reports


# ---- bit-for-bit comparison ------------------------------------------------------------------------------------------------

def same(a, b):
    """float64 equality bit for bit; a NaN (0/0 of a zero-area footprint, in the reference too) matches a NaN."""
    return bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def same_polygons(cnt, xy, ref_cnt, ref_xy, what):
    """Untraversable polygons: equal counts, and equal vertices bit for bit up to the count (or the capacity)."""
    assert np.array_equal(cnt, ref_cnt), (what, np.nonzero(cnt != ref_cnt)[0][:10])
    for q in np.nonzero(cnt > 0)[0]:
        k = min(int(cnt[q]), xy.shape[1])
        assert np.array_equal(xy[q, :k].view(np.uint64), ref_xy[q, :k].view(np.uint64)), (what, q)


# ---- maps, paths, footprints and requests of the path-check tests ----------------------------------------------------------

YAML = [(0.45, 0.30, 0.0), (0.45, -0.30, 0.0), (-0.45, -0.30, 0.0), (-0.45, 0.30, 0.0)]   # robot_footprint_parameter.yaml:3


def footprint_params(te, oracle, verify):
    """(library, oracle) FootprintParams: the YAML defaults with verify_roughness set."""
    ft, fo = te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults()
    ft.verify_roughness = fo.verify_roughness = verify
    return ft, fo


def chain_layers(oracle, og, z, seed):
    """The oracle chain's layers on elevation z, roughness with zero patches, and a robot_slope layer (zeros and NaNs)."""
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    rng = np.random.default_rng(seed)
    rough = ch["roughness"].copy()   # zero patches, so that checkForRoughness blocks cells the slope / step checks let through
    for _ in range(40):
        a, b = int(rng.integers(0, og.rows - 12)), int(rng.integers(0, og.cols - 12))
        rough[a:a + int(rng.integers(1, 12)), b:b + int(rng.integers(1, 12))] = 0.0
    rs = ch["slope"].copy()
    rs[rng.random(rs.shape) < 0.0005] = 0.0
    rs[rng.random(rs.shape) < 0.05] = np.nan
    f = lambda a: np.asfortranarray(a, dtype=np.float32)  # noqa: E731
    return dict(traversability=f(ch["traversability"]), slope=f(ch["slope"]), step=f(ch["step"]), elevation=f(z),
                roughness=f(rough)), f(rs)


def circular_paths(rng, og, npaths, radii=(0.0, 0.2, 0.3, 0.45), planner=False):
    """(path_begin, poses (n, 2), radius): random walks, planner-like (2-8 poses, radius 0.3) or not (0-6 poses, a few outside
    the map, mixed radii)."""
    lx, ly = og.rows * og.resolution, og.cols * og.resolution
    cx, cy = og.position_x, og.position_y
    begin, poses, radius = [0], [], []
    for q in range(npaths):
        if planner:
            n = int(rng.integers(2, 9))
        else:
            n = int(rng.integers(0, 7)) if q > 3 else (0, 1, 2, 5)[q]
        p = [rng.uniform([cx - 0.45 * lx, cy - 0.45 * ly], [cx + 0.45 * lx, cy + 0.45 * ly])]
        for _ in range(n - 1):   # 0.1 - 0.5 m steps, like a planner's poses; a few paths turn back on themselves
            ang, d = rng.uniform(0, 2 * np.pi), rng.uniform(0.1, 0.5)
            p.append(p[-1] + d * np.array([np.cos(ang), np.sin(ang)]) if rng.random() > 0.1 or len(p) < 2 else p[-2].copy())
        p = np.asarray(p[:n]).reshape(-1, 2)
        if not planner and q % 50 == 7 and n > 0:
            p[0] = [cx + 0.6 * lx, cy]                            # a pose outside the map
        poses.extend(p.tolist())
        begin.append(len(poses))
        radius.append(0.3 if planner else float(radii[int(rng.integers(0, len(radii)))]))
    return np.asarray(begin, np.int32), np.asarray(poses, np.float64).reshape(-1, 2), np.asarray(radius, np.float64)


def random_footprint(rng, nv):
    """A random footprint of nv vertices with z != 0: convex (sorted angles) or not (shuffled)."""
    ang = np.sort(rng.uniform(0, 2 * np.pi, nv))
    r = rng.uniform(0.1, 0.5, nv)
    v = np.stack([r * np.cos(ang), r * np.sin(ang), rng.uniform(-0.3, 0.3, nv)], axis=1)
    if rng.random() < 0.5:
        rng.shuffle(v)
    return v.astype(np.float32)


def quaternion(rng, kind):
    """qx qy qz qw: kind 0 a yaw, 1 a general unit quaternion, 2 one that is not normalised."""
    if kind == 0:
        a = rng.uniform(0, 2 * np.pi)
        return [0.0, 0.0, np.sin(a / 2), np.cos(a / 2)]
    q = rng.normal(size=4)
    if kind == 1:
        return (q / np.linalg.norm(q)).tolist()
    return (q * rng.uniform(0.5, 1.5)).tolist()


def polygonal_paths(rng, og, npaths, planner=False):
    """(path_begin, poses (n, 7)): the walks of circular_paths with a z and an orientation per pose."""
    lx, ly = og.rows * og.resolution, og.cols * og.resolution
    cx, cy = og.position_x, og.position_y
    begin, poses = [0], []
    for q in range(npaths):
        n = int(rng.integers(2, 9)) if planner else (int(rng.integers(0, 7)) if q > 3 else (0, 1, 2, 5)[q])
        p = [rng.uniform([cx - 0.45 * lx, cy - 0.45 * ly], [cx + 0.45 * lx, cy + 0.45 * ly])]
        for _ in range(n - 1):   # 0.1 - 0.5 m steps; a few paths turn back on themselves
            a, d = rng.uniform(0, 2 * np.pi), rng.uniform(0.1, 0.5)
            p.append(p[-1] + d * np.array([np.cos(a), np.sin(a)]) if rng.random() > 0.1 or len(p) < 2 else p[-2].copy())
        p = np.asarray(p[:n]).reshape(-1, 2)
        if not planner and q % 50 == 7 and n > 0:
            p[0] = [cx + 0.6 * lx, cy]                        # a pose outside the map
        kind = 0 if planner else int(rng.integers(0, 3))
        for x, y in p:
            poses.append([x, y, rng.uniform(-1, 1), *quaternion(rng, kind)])
        begin.append(len(poses))
    return np.asarray(begin, np.int32), np.asarray(poses, np.float64).reshape(-1, 7)


def request_footprints(rng):
    """The four footprints of a request: 1, 3, 4 (the YAML rectangle) and 16 vertices."""
    return [random_footprint(rng, 1), random_footprint(rng, 3), np.asarray(YAML, np.float32), random_footprint(rng, 16)]


def mixed_request(rng, og, npaths, fps, circular=0.4, planner=False, cap_path=True):
    """A mixed request: per path its poses (7 wide), radius, footprint index (-1: circular), conservative and cup.  Circular
    paths carry z / orientations the check must ignore (NaN in some); polygonal paths carry a NaN radius, which it ignores too."""
    lx, ly = og.rows * og.resolution, og.cols * og.resolution
    cx, cy = og.position_x, og.position_y
    begin, poses, radius, kind = [0], [], [], []
    for q in range(npaths):
        k = -1 if rng.random() < circular else int(rng.integers(0, len(fps)))
        if planner:
            n = int(rng.integers(2, 9))
        else:
            n = int(rng.integers(0, 9)) if q > 5 else (0, 1, 2, 1, 5, 8)[q]
        p = [rng.uniform([cx - 0.45 * lx, cy - 0.45 * ly], [cx + 0.45 * lx, cy + 0.45 * ly])]
        for _ in range(n - 1):   # 0.1 - 0.5 m steps; a few paths turn back on themselves
            a, d = rng.uniform(0, 2 * np.pi), rng.uniform(0.1, 0.5)
            p.append(p[-1] + d * np.array([np.cos(a), np.sin(a)]) if rng.random() > 0.1 or len(p) < 2 else p[-2].copy())
        p = np.asarray(p[:n]).reshape(-1, 2)
        if not planner and q % 40 == 9 and n > 0:
            p[0] = [cx + 0.6 * lx, cy]                        # a pose outside the map
        qkind = 0 if planner else int(rng.integers(0, 3))
        for x, y in p:
            rest = [rng.uniform(-1, 1), *quaternion(rng, qkind)]
            if k < 0 and rng.random() < 0.2:
                rest[-1] = np.nan
            poses.append([x, y, *rest])
        begin.append(len(poses))
        radius.append(float(rng.uniform(0.1, 0.5)) if k < 0 else np.nan)
        kind.append(k)
    if cap_path:   # a conservative YAML path of 256 poses: polygon2 reaches the 1024-vertex cap
        walk = np.cumsum(rng.uniform(-0.01, 0.01, (256, 2)), axis=0) + [cx + 0.1 * lx, cy - 0.1 * ly]
        poses.extend(np.concatenate([walk, np.tile([0.0, 0.0, 0.0, 0.0, 1.0], (256, 1))], axis=1).tolist())
        begin.append(len(poses))
        radius.append(np.nan)
        kind.append(2)
    m = len(kind)
    cons = (rng.random(m) < 0.3).astype(np.uint8)
    cup = (rng.random(m) < 0.5).astype(np.uint8)
    if cap_path:
        cons[-1] = cup[-1] = 1
    return dict(begin=np.asarray(begin, np.int32), poses=np.asarray(poses, np.float64).reshape(-1, 7),
                radius=np.asarray(radius, np.float64), kind=np.asarray(kind), cons=cons, cup=cup)


def footprint_arrays(R, fps):
    """footprint_begin / footprint_xyz of a request: path q's own copy of its footprint, none for circular paths."""
    fb, fx = [0], []
    for k in R["kind"]:
        if k >= 0:
            fx.extend(fps[k].tolist())
        fb.append(len(fx))
    return np.asarray(fb, np.int32), np.asarray(fx, np.float32).reshape(-1, 3)


# ---- the hand-derived maps of the untraversable-polygon tests --------------------------------------------------------------
# Dyadic geometry (0.25 m cells, 64 x 64, map centred on the origin) keeps every cell centre exact.  Cells are blocked through
# checkForSlope: with max_gap_width 0.1 its critical count is floor(2 * 0.75 * (0.1 / 3) / 0.25^2) = 0, so a cell whose
# traversability_slope is 0 fails isTraversableForFilters and no other cell does.

DYADIC_RES, DYADIC_N = 0.25, 64


def dyadic_x(i):
    """Cell centre coordinate of row (or column) i of the dyadic map."""
    return (0.0 + (0.5 * DYADIC_N * DYADIC_RES - 0.5 * DYADIC_RES)) + DYADIC_RES * (-float(i))


def dyadic_cell(i, j):
    return (dyadic_x(i), dyadic_x(j))


def dyadic_map(oracle, blocked=(), trav=0.5):
    """(geometry, FootprintParams, layers) of the dyadic map with the cells `blocked`; trav: a value or a layer."""
    N = DYADIC_N
    g = oracle.Geometry.make(N, N, DYADIC_RES)
    one = np.ones((N, N), np.float32, order="F")
    slope = one.copy()
    for a, b in blocked:
        slope[a, b] = 0.0
    t = trav if isinstance(trav, np.ndarray) else np.full((N, N), trav, np.float32, order="F")
    fp = oracle.FootprintParams.yaml_defaults()
    fp.max_gap_width, fp.offset, fp.traversability_default = 0.1, 0.5, 0.3
    return g, fp, dict(traversability=np.asfortranarray(t), slope=slope, step=one, elevation=one * 0)
