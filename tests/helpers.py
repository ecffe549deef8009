"""Helpers shared by the tests: layer comparison (SURVEY.md §8d tolerances), bit-for-bit comparison, and the maps, paths,
footprints, requests and parameters of the footprint path-check tests.  The te_map helpers are in map_helpers.py."""
import numpy as np

import synth

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


def assert_same_answers(got, want, what=""):
    """The outputs of two requests: is_safe equal, traversability and area bit for bit (NaN matches NaN), and the untraversable
    polygons, when the request returns them."""
    assert np.array_equal(got[0], want[0]), (what, np.nonzero(got[0] != want[0])[0][:10])
    assert same(got[1], want[1]) and same(got[2], want[2]), what
    if len(want) > 3:
        same_polygons(got[3], got[4], want[3], want[4], what)


def bits(a):
    """The uint32 bit patterns of `a` as float32."""
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_same_bits(a, b, what=""):
    """float32 bit for bit: every NaN payload too."""
    assert np.array_equal(bits(a), bits(b)), (what, int((bits(a) != bits(b)).sum()))


def same_bits_or_nan(a, b):
    """float32 bit for bit, except that a NaN matches any NaN (the GPU's NaN payloads differ from x86's)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))))


def same_bytes(a, b):
    """Equal shapes and equal bytes, of any dtype."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def same_values(a, b):
    """NaN at the same cells, and equal values at the others."""
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)])


def close_sweep(a, b):
    """The tolerance of the prefix-sum footprint sweeps against the oracle: they add the same float32 terms in another order (double
    accumulation), so a handful of cells whose disk holds default-valued (NaN) cells may differ in the last float32 bit.  NaN and
    zero (blocked) cells are the same."""
    if not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    m = ~np.isnan(a)
    if not np.array_equal(a[m] == 0, b[m] == 0):
        return False
    return float((a[m] == b[m]).mean()) > 0.999 and np.allclose(a[m], b[m], rtol=2e-7, atol=0)


# ---- maps, paths, footprints and requests of the path-check tests ----------------------------------------------------------

YAML = [(0.45, 0.30, 0.0), (0.45, -0.30, 0.0), (-0.45, -0.30, 0.0), (-0.45, 0.30, 0.0)]   # robot_footprint_parameter.yaml:3


def footprint_params(te, oracle, verify=0, **kw):
    """(library, oracle) FootprintParams: the YAML defaults with verify_roughness and the fields kw set."""
    return te_footprint_params(te, verify_roughness=verify, **kw), te_footprint_params(oracle, verify_roughness=verify, **kw)


def te_footprint_params(mod, **kw):
    """The FootprintParams of `mod` (the library or the oracle): the YAML defaults with the fields kw set."""
    p = mod.FootprintParams.yaml_defaults()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def chain_params(mod, **kw):
    """The ChainParams of `mod` (the library or the oracle): the YAML defaults with the fields kw set."""
    p = mod.ChainParams.yaml_defaults(0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


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


def batch_request(rng, og, npaths, nmaps, fps=None, exclude=None, offsets=None, permute=True, **kw):
    """A mixed_request (keywords kw) on a batch of nmaps maps of geometry og, with its footprints in R["fps"] (drawn first when
    fps is None) and a path_map R["map"] that interleaves the maps in no order, leaving map `exclude` out.  permute: the first
    paths visit every map.  offsets: per map, added to the x y of its paths' poses."""
    if fps is None:
        fps = request_footprints(rng)
    R = mixed_request(rng, og, npaths, fps, **kw)
    R["fps"] = fps
    maps = [m for m in range(nmaps) if m != exclude]
    R["map"] = np.asarray(maps, np.int32)[rng.integers(0, len(maps), len(R["kind"]))]
    if permute:
        R["map"][:len(maps)] = rng.permutation(maps)
    if offsets is not None:
        for q, m in enumerate(R["map"]):
            R["poses"][R["begin"][q]:R["begin"][q + 1], :2] += offsets[m]
    return R


def subset(R, idx):
    """The request of the paths `idx` of R, in that order: every per-path array R has, and its footprints."""
    b, idx = R["begin"], np.asarray(idx, dtype=np.int64)
    begin = np.concatenate([[0], np.cumsum(b[idx + 1] - b[idx])]).astype(np.int32)
    poses = np.concatenate([R["poses"][b[q]:b[q + 1]] for q in idx]) if len(idx) else np.zeros((0, 7))
    S = dict(begin=begin, poses=poses, **{k: R[k][idx] for k in ("radius", "kind", "cons", "cup", "map") if k in R})
    if "fps" in R:
        S["fps"] = R["fps"]
    return S


# ---- layers ------------------------------------------------------------------------------------------------------------------

def wrap(a, start):
    """A default-order (rows, cols) layer in the buffer order of start index `start`: cell (i, j) at ((i + sr) % rows, ...)."""
    return np.roll(a, (int(start[0]), int(start[1])), axis=(0, 1))


def unwrap(a, start):
    """The default order of a layer stored with start index `start`: the inverse of wrap."""
    return np.roll(a, (-int(start[0]), -int(start[1])), axis=(0, 1))


def noisy(rng, shape, nan, inf, ninf, zero):
    """A float32 layer with the fractions nan, inf, ninf and zero of NaN, +Inf, -Inf and exact zeros (a fraction of 0 draws
    nothing), and 1% NaN of other payloads, signalling ones included."""
    a = (rng.standard_normal(shape) * 3).astype(np.float32)
    for frac, v in ((nan, np.nan), (inf, np.inf), (ninf, -np.inf), (zero, 0.0)):
        if frac:
            a[rng.random(shape) < frac] = v
    odd = rng.random(shape) < 0.01
    a.view(np.uint32)[odd] = (rng.integers(0, 2, odd.sum()) << 31 | 0x7f800000 | rng.integers(1, 1 << 23, odd.sum())).astype(np.uint32)
    return a


def walled_terrain(rows, cols, res, kind, seed):
    """Neighbouring maps of a batch differ sharply: a flat map, a map walled along its first rows and columns, a terrain map, a map
    walled along its last rows and columns.  A value read across a map boundary would change the cells along that boundary."""
    if kind == 0:
        return np.zeros((rows, cols), dtype=np.float32)
    z = synth.terrain(rows, cols, res, seed, "mixed")
    if kind == 1:
        z[:5, :] += np.float32(1.0)
        z[:, :5] += np.float32(1.0)
    if kind == 3:
        z[-5:, :] += np.float32(1.0)
        z[:, -5:] += np.float32(1.0)
    return z


def walled_batch(oracle, rows, cols, res, n, seed, robot_slope=False):
    """Chain layers of n walled_terrain maps on the CPU oracle, stacked as (n, cols, rows): map k's layers are the column-major
    batch[k].T.  robot_slope: also a robot_slope layer per map (its slope with zeros and NaNs)."""
    og = oracle.Geometry.make(rows, cols, res)
    names = ("traversability", "slope", "step", "roughness", "elevation") + (("robot_slope",) if robot_slope else ())
    out = {k: [] for k in names}
    rng = np.random.default_rng(seed)
    for k in range(n):
        z = walled_terrain(rows, cols, res, k % 4, seed + k)
        ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
        slope, rough = np.array(ch["slope"], dtype=np.float32), np.array(ch["roughness"], dtype=np.float32)
        for _ in range(3 if k % 4 else 0):
            # zero patches: checkForRoughness blocks them when verify_roughness is set, checkForSlope with a small max_gap_width
            a, b = int(rng.integers(0, rows - 10)), int(rng.integers(0, cols - 10))
            rough[a:a + 9, b:b + 9] = 0.0
            a, b = int(rng.integers(0, rows - 10)), int(rng.integers(0, cols - 10))
            slope[a:a + 9, b:b + 9] = 0.0
        layers = [ch["traversability"], slope, ch["step"], rough, z]
        if robot_slope:
            rs = np.array(ch["slope"], dtype=np.float32)
            rs[rng.random(rs.shape) < 0.002] = 0.0
            rs[rng.random(rs.shape) < 0.05] = np.nan
            layers.append(rs)
        for name, layer in zip(names, layers):
            out[name].append(np.ascontiguousarray(np.asarray(layer, dtype=np.float32).T))
    return {k: np.stack(v) for k, v in out.items()}


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
