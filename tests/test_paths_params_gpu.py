"""The footprint path checks against the oracle away from the YAML parameters: te_check_footprint_paths_fresh2,
te_check_footprint_paths_polygon2, te_check_footprint_request(_batched) on a fresh map, and te_map_check_footprint_request in host
and in device memory on a cache that persists across requests.

Axes: traversability_default of every kind (invalid cells, poses outside the map, a polygon covering no cell centre), both radius
norms, offset 0 (radiusMax == radiusMin: an infinite ring factor), radius 0 and radius = offset = 0 (a spiral of the centre
only), a reach of exactly 127 rings (128 refused), max_gap_width / critical_step_height with and without roughness, and path
shapes random walks rarely make.  The replay cases put several checks on one cell whose first walk stores a NaN or an infinity:
the reference does not take such a cell as cached (isValid), so the next check there walks again with its own radius and flag
(paths_params_cases.py).  Every comparison is bit for bit (any NaN matches any NaN), the te_map's cache after every request
included, and every case asserts that it can fail."""
import math

import numpy as np
import pytest

import paths_oracle as po
import paths_params_cases as pc
from footprint_cases import BUILT_GAP, built_map, chain_map, unblocked
from helpers import (YAML, assert_same_answers, batch_request, footprint_arrays, mixed_request, request_footprints, same,
                     same_polygons, subset, te_footprint_params)
from map_helpers import CAP, ask, assert_batch_matches_singles, assert_same_cache, close_maps  # noqa: F401

pytestmark = pytest.mark.gpu

INF, NAN = float("inf"), float("nan")
DEFAULTS = [0.0, 1.0, -0.5, 0.3, NAN, INF, -INF]
FILTERS = [dict(max_gap_width=v) for v in (0.001, 0.05, 0.3, 1.0)] + [dict(critical_step_height=v) for v in (0.05, 0.12, 0.3)]
ERR_UNSUPPORTED = -4
MAPL = ("traversability", "slope", "step", "elevation")
EMPTY = [(0.004, 0.004, 0.0), (0.009, 0.004, 0.0), (0.004, 0.009, 0.0)]   # covers no cell centre at yaw 0
MAX_CHECKS = 1 << 20


def geoms(te, oracle, m, res):
    rows, cols = m["traversability"].shape
    return te.Geometry.make(rows, cols, res), oracle.Geometry.make(rows, cols, res)


def oracle_request(oracle, og, fo, m, R, cache=None):
    fb, fx = footprint_arrays(R, R["fps"])
    return po.check_request(og, fo, m, R["begin"], R["poses"], R["radius"], fb, fx, conservative=R["cons"], cup=R["cup"],
                            cache=cache, capacity=CAP)


def stateless(te, ctx, oracle, m, kw, R, res=0.02):
    """The fresh-map entries against the oracle: the whole request (te_check_footprint_request, and _batched on two copies of the
    map with the paths alternating between them), its circular paths (fresh2) and its polygonal paths per footprint (polygon2).
    Returns the oracle's answers."""
    g, og = geoms(te, oracle, m, res)
    ft, fo = te_footprint_params(te, **kw), te_footprint_params(oracle, **kw)
    ref = oracle_request(oracle, og, fo, m, R)
    fb, fx = footprint_arrays(R, R["fps"])
    lay, rough = [m[k] for k in MAPL], m["roughness"]
    pkw = dict(max_footprint_vertices=16, conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=CAP)
    got = ctx.check_footprint_request(g, ft, *lay, R["begin"], R["poses"], R["radius"], fb, fx, roughness=rough, **pkw)
    assert_same_answers(got, ref, (kw, "request"))
    n = len(R["begin"]) - 1
    two = lambda a: np.stack([np.ascontiguousarray(a.T)] * 2)  # noqa: E731
    got = ctx.check_footprint_request_batched(g, ft, 2, *(two(a) for a in lay), (np.arange(n) % 2).astype(np.int32), R["begin"],
                                              R["poses"], R["radius"], fb, fx, roughness=two(rough), **pkw)
    assert_same_answers(got, ref, (kw, "request_batched"))
    circ = np.nonzero(R["kind"] < 0)[0]
    if len(circ):
        S = subset(R, circ)
        got = ctx.check_footprint_paths_fresh(g, ft, *lay, S["begin"], S["poses"][:, :2], S["radius"], roughness=rough,
                                              compute_untraversable_polygon=S["cup"], untraversable_capacity=CAP)
        assert np.array_equal(got[0], ref[0][circ]) and same(got[1], ref[1][circ]), (kw, "fresh2")
        same_polygons(got[2], got[3], ref[3][circ], ref[4][circ], (kw, "fresh2"))
    for k in sorted(set(R["kind"][R["kind"] >= 0].tolist())):
        idx = np.nonzero(R["kind"] == k)[0]
        S = subset(R, idx)
        got = ctx.check_footprint_paths_polygon(g, ft, *lay, R["fps"][k], S["begin"], S["poses"], roughness=rough,
                                                conservative=S["cons"], compute_untraversable_polygon=S["cup"],
                                                untraversable_capacity=CAP)
        assert np.array_equal(got[0], ref[0][idx]) and same(got[1], ref[1][idx]) and same(got[2], ref[2][idx]), (kw, "polygon2", k)
        same_polygons(got[3], got[4], ref[3][idx], ref[4][idx], (kw, "polygon2", k))
    return ref


def device(m, ft, R):
    """te_map_check_footprint_request_device with every array in device memory; the outputs as numpy arrays."""
    import torch
    fb, fx = footprint_arrays(R, R["fps"])
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    n = len(R["begin"]) - 1
    out = dict(is_safe=torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
               area_out=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
               untraversable_count=torch.full((n,), 99, dtype=torch.int32, device="cuda"),
               untraversable_xy=torch.zeros((n, CAP, 2), dtype=torch.float64, device="cuda"))
    torch.cuda.synchronize()
    m.check_footprint_request_device(ft, dev(R["begin"], np.int32), dev(R["poses"], np.float64), dev(R["radius"], np.float64),
                                     dev(fb, np.int32), dev(fx, np.float32), max_checks=MAX_CHECKS, max_footprint_vertices=16,
                                     conservative=dev(R["cons"], np.uint8), compute_untraversable_polygon=dev(R["cup"], np.uint8),
                                     untraversable_capacity=CAP, **out)
    torch.cuda.synchronize()
    return tuple(out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out", "untraversable_count", "untraversable_xy"))


def on_map(te, ctx, oracle, m, kw, requests, res=0.02):
    """The requests in order on a te_map holding m, each asked twice, in host memory (one te_map) and in device memory (its twin),
    against the oracle on one persistent cache: answers, and the cache after every request.  Returns the oracle's answers."""
    g, og = geoms(te, oracle, m, res)
    ft, fo = te_footprint_params(te, **kw), te_footprint_params(oracle, **kw)
    H, D = ctx.map(), ctx.map()
    for x in (H, D):
        x.set_layers(g, *(m[k] for k in MAPL), roughness=m["roughness"])
    cache = po.empty_cache(og)
    refs = []
    for k, R in enumerate(requests):
        for rep in range(2):
            what = (kw, k, rep)
            want = oracle_request(oracle, og, fo, m, R, cache)
            assert_same_answers(ask(H, ft, R), want, ("te_map host",) + what)
            assert_same_cache(H.get_footprint(), cache, ("te_map host cache",) + what, nan_bits=False)
            assert_same_answers(device(D, ft, R), want, ("te_map device",) + what)
            assert_same_cache(D.get_footprint(), H.get_footprint(), ("te_map device cache",) + what)
            assert D.request_stats() == H.request_stats(), what
            if finite_stores(kw):
                cand, keys, stored = H.request_stats()
                assert stored <= keys <= cand, what
            refs.append(want)
    return refs


def finite_stores(kw):
    """Whether every walk stores a finite value: a finite default and a ring factor with radiusMax > radiusMin."""
    return math.isfinite(kw.get("traversability_default", 0.5)) and kw.get("offset", 0.15) > 0


def nonvacuous(ref, default=0.3):
    """Safe and unsafe paths; under a non-finite default, safe paths with a non-finite answer (a NaN under a NaN default)."""
    safe, trav = ref[0] == 1, ref[1]
    assert safe.any() and (~safe).any(), int(safe.sum())
    if math.isnan(default):
        assert np.isnan(trav[safe]).any()
    elif math.isinf(default):
        assert (~np.isfinite(trav[safe])).any()


# ---- traversability_default ----------------------------------------------------------------------------------------------------

def default_requests(og, m, seed):
    """Three mixed requests on the built map: random walks of both kinds, single poses outside the map, the polygon that covers
    no cell centre (a single pose and a segment), and single circles on and next to invalid cells."""
    rng = np.random.default_rng(seed)
    fps = request_footprints(rng) + [np.asarray(EMPTY, np.float32)]
    X, Y = pc.fg.cell_tables(*m["traversability"].shape, 0.02, (0.0, 0.0))
    inv = np.argwhere(~np.isfinite(m["traversability"]))[:6]
    extra = [([(0.0, 3.5)], 0.2, -1, 0, 1), ([(4.0, 0.1, 0.0, 0.0, 0.0, 0.0, 1.0)], NAN, 2, 0, 1),
             ([(0.011, 0.013)], NAN, 4, 0, 0), ([(0.011, 0.013), (0.011, 0.013)], NAN, 4, 0, 1)]
    extra += [([(float(X[a]), float(Y[b]))], r, -1, 0, u) for a, b in inv for r, u in ((0.0, 1), (0.1, 0))]
    E = pc.request(extra, fps)
    out = []
    for k in range(3):
        R = mixed_request(rng, og, 50, fps[:4], circular=0.6, cap_path=False)
        both = [dict(R, fps=fps), E] if k != 1 else [E, dict(R, fps=fps)]
        out.append(join(both))
    return out


def join(requests):
    """One request of the paths of `requests` in order (they share their footprint list)."""
    fps = requests[0]["fps"]
    begin, poses = [0], []
    for R in requests:
        poses.append(R["poses"])
        begin.extend((R["begin"][1:] + begin[-1]).tolist())
    cat = lambda k: np.concatenate([R[k] for R in requests])  # noqa: E731
    return dict(begin=np.asarray(begin, np.int32), poses=np.concatenate(poses), radius=cat("radius"), kind=cat("kind"),
                cons=cat("cons").astype(np.uint8), cup=cat("cup").astype(np.uint8), fps=fps)


@pytest.mark.parametrize("default", DEFAULTS, ids=[f"default={d}" for d in DEFAULTS])
def test_default(te, ctx, oracle, default):
    m = built_map()
    og = oracle.Geometry.make(*m["traversability"].shape, 0.02)
    kw = dict(traversability_default=default, **BUILT_GAP)
    seq = default_requests(og, m, 5)
    ref = stateless(te, ctx, oracle, m, kw, seq[0])
    nonvacuous(ref, default)
    # the polygon over no cell centre answers the default; single poses outside the map too
    empty = np.nonzero(seq[0]["kind"] == 4)[0]
    assert (ref[0][empty] == int(default != 0.0)).all()
    if default != 0.0:
        assert np.array_equal(ref[1][empty], np.full(len(empty), default), equal_nan=True)
    for r in on_map(te, ctx, oracle, m, kw, seq):
        nonvacuous(r, default)


# ---- radius_is_integer_norm, offset, radius 0 ----------------------------------------------------------------------------------

def cell_poses(m, radius, step=3, jitter=None, seed=0, cup=1):
    """Single circular poses of radius `radius` at every `step`-th cell centre away from the edges, moved by up to `jitter` of a
    cell (None: at the centre)."""
    rows, cols = m["traversability"].shape
    X, Y = pc.fg.cell_tables(rows, cols, 0.02, (0.0, 0.0))
    rng = np.random.default_rng(seed)
    paths = []
    for a in range(8, rows - 8, step):
        for b in range(8, cols - 8, step):
            x, y = float(X[a]), float(Y[b])
            if jitter is not None:
                x, y = x + jitter * 0.02 * rng.uniform(-1, 1), y + jitter * 0.02 * rng.uniform(-1, 1)
            paths.append(([(x, y)], radius, -1, 0, cup if cup is not None else int(rng.integers(0, 2))))
    return pc.request(paths)


def walks(og, seed, n=40, radius=None):
    rng = np.random.default_rng(seed)
    R = dict(mixed_request(rng, og, n, [], circular=1.0, cap_path=False), fps=[])
    if radius is not None:
        R["radius"][:] = radius
    return R


@pytest.mark.parametrize("norm", [0, 1])
def test_radius_norm(te, ctx, oracle, norm):
    """The first blocked cell of many circles falls on either side of the inner radius; the two norms answer differently."""
    m = built_map(spacing=24)
    og = oracle.Geometry.make(*m["traversability"].shape, 0.02)
    kw = dict(radius_is_integer_norm=norm, **BUILT_GAP)
    R = join([cell_poses(m, 0.2, cup=None), walks(og, 11, radius=0.2)])
    ref = stateless(te, ctx, oracle, m, kw, R)
    nonvacuous(ref)
    other = oracle_request(oracle, og, te_footprint_params(oracle, **dict(kw, radius_is_integer_norm=1 - norm)), m, R)
    assert (ref[0] != other[0]).any() and not same(ref[1], other[1])
    on_map(te, ctx, oracle, m, kw, [R])


OFFSETS = [(0.0, 0.0), (0.0, 0.2), (0.15, 0.0), (0.15, 0.2), (0.6, 0.0), (0.6, 0.2)]


@pytest.mark.parametrize("offset,radius", OFFSETS, ids=[f"offset={o}-radius={r}" for o, r in OFFSETS])
def test_offset_and_zero_radius(te, ctx, oracle, offset, radius):
    """offset 0 with single poses off their cell centre: the blocker beyond the inner radius gives an infinite ring factor (the
    exact norm).  radius 0: any blocked cell blocks; radius = offset = 0: the spiral is the centre alone (nr = 0)."""
    m = built_map(spacing=72 if radius == 0.0 and offset > 0.5 else 24)   # radius 0 with 30 rings: disks free of blockers
    og = oracle.Geometry.make(*m["traversability"].shape, 0.02)
    kw = dict(offset=offset, radius_is_integer_norm=0, **BUILT_GAP)
    poses = cell_poses(m, radius, step=2, jitter=0.49, seed=3, cup=None)
    R = join([poses, walks(og, 12, radius=radius)])
    ref = stateless(te, ctx, oracle, m, kw, R)
    nonvacuous(ref)
    safe = ref[0] == 1
    if offset == 0.0 and radius > 0:
        assert np.isposinf(ref[1][safe]).any()     # the infinite ring factor
    if offset == 0.0 and radius == 0.0:            # a single pose's circle is its cell alone: the cell's value or the default
        ns = len(poses["kind"])
        assert safe[:ns].sum() > 100 and np.isin(ref[1][:ns][safe[:ns]], np.append(m["traversability"], 0.3)).all()
    if offset > 0 and radius > 0:                  # the ring factor moves answers off the unblocked mean
        free = oracle_request(oracle, og, te_footprint_params(oracle, **kw), unblocked(m), R)
        assert (safe & (ref[1] != free[1])).any()
    on_map(te, ctx, oracle, m, kw, [R])


# ---- the ring limit ------------------------------------------------------------------------------------------------------------

def reach_127(offset):
    """(radius, offset) with ceil((radius + offset) / 0.02) == 127 exactly."""
    rmax = 127 * 0.02
    while math.ceil(rmax / 0.02) > 127:
        rmax = float(np.nextafter(rmax, 0.0))
    return rmax - offset, offset


def rim_map():
    """300 x 300 at 0.02 m: blockers 126 cells from cell (150, 150), on the rim of its 127-ring circle."""
    m = dict(built_map(0.02, 300, 300, 400, 9))
    slope = np.ones((300, 300), np.float32, order="F")
    for a, b in ((150 + 126, 150), (150 - 126, 150), (150, 150 + 126), (150, 150 - 126), (150 - 89, 150 - 89)):
        slope[a, b] = 0.0
    m["slope"] = slope
    return m


@pytest.mark.parametrize("inner", [False, True])
def test_ring_limit(te, ctx, oracle, inner):
    """A reach of exactly 127 rings with blockers near the rim and the polygon flag: the 255-row tables of the polygon kernels and
    the ±127 ring packing.  offset 0.15 puts the rim blockers beyond the inner radius (119.5 cells), offset 0.01 inside it
    (126.5 cells).  One ring more is refused in host memory and not checked in device memory."""
    radius, offset = reach_127(0.01 if inner else 0.15)
    m = rim_map()
    X, Y = pc.fg.cell_tables(300, 300, 0.02, (0.0, 0.0))
    c = (float(X[150]), float(Y[150]))
    paths = [([c], radius, -1, 0, 1), ([c], radius, -1, 0, 0), ([(c[0] + 0.05, c[1])], radius, -1, 0, 1),
             ([(float(X[150]), float(Y[100]))], radius, -1, 0, 1), ([(float(X[60]), float(Y[200]))], radius, -1, 0, 1),
             ([(float(X[140]), float(Y[150])), (float(X[160]), float(Y[170]))], radius, -1, 0, 1),
             ([(float(X[130]), float(Y[20])), (float(X[170]), float(Y[60]))], 0.3, -1, 0, 1)]
    R = pc.request(paths)
    kw = dict(offset=offset, **BUILT_GAP)
    ref = stateless(te, ctx, oracle, m, kw, R)
    assert (ref[0] == 0).any()
    if inner:   # the hull of the blocked cells of the centre's circle spans rows 24 .. 276
        span = ref[4][0, :ref[3][0], 0]
        assert ref[3][0] > 0 and span.max() - span.min() > 251 * 0.02
    else:       # the rim blockers lie beyond the inner radius: with the flag the centre's circle is traversable
        assert ref[0][0] == 1 and ref[0][1] == 0
    on_map(te, ctx, oracle, m, kw, [R])
    # 128 rings
    g, og = geoms(te, oracle, m, 0.02)
    big = float(np.nextafter(128 * 0.02 - offset, 1.0))
    assert math.ceil((big + offset) / 0.02) == 128
    B = pc.request([([c], big, -1, 0, 1), ([c], 0.3, -1, 0, 1)])
    ft = te_footprint_params(te, **kw)
    fb, fx = footprint_arrays(B, [])
    calls = [lambda: ctx.check_footprint_paths_fresh(g, ft, *(m[k] for k in MAPL), B["begin"], B["poses"][:, :2], B["radius"]),
             lambda: ctx.check_footprint_request(g, ft, *(m[k] for k in MAPL), B["begin"], B["poses"], B["radius"], fb, fx)]
    H, D = ctx.map(), ctx.map()
    for x in (H, D):
        x.set_layers(g, *(m[k] for k in MAPL))
    calls.append(lambda: ask(H, ft, dict(B, fps=[])))
    for call in calls:
        with pytest.raises(te.TEError) as err:
            call()
        assert err.value.code == ERR_UNSUPPORTED
    got = device(D, ft, dict(B, fps=[]))
    assert got[0][0] == 0 and np.isnan(got[1][0]) and np.isnan(got[2][0]) and got[3][0] == -1
    want = oracle_request(oracle, og, te_footprint_params(oracle, **kw), m, subset(dict(B, fps=[]), [1]), po.empty_cache(og))
    assert_same_answers(tuple(a[1:] for a in got), want, "the checked path")


# ---- filters -------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("verify", [0, 1])
@pytest.mark.parametrize("kw", FILTERS, ids=[f"{k}={v}" for d in FILTERS for k, v in d.items()])
def test_filters(te, ctx, oracle, kw, verify):
    """max_gap_width and critical_step_height change the cells blocked_memo_d blocks."""
    m = chain_map(oracle)
    og = oracle.Geometry.make(*m["traversability"].shape, 0.02)
    rng = np.random.default_rng(17)
    fps = request_footprints(rng)
    R = dict(mixed_request(rng, og, 60, fps, circular=0.6, cap_path=False), fps=fps)
    kw = dict(kw, verify_roughness=verify)
    nonvacuous(stateless(te, ctx, oracle, m, kw, R))
    on_map(te, ctx, oracle, m, kw, [R])


# ---- path shapes ---------------------------------------------------------------------------------------------------------------

def shape_request(og, m, res=0.02):
    rows, cols = m["traversability"].shape
    X, Y = pc.fg.cell_tables(rows, cols, res, (0.0, 0.0))
    P = lambda a, b: (float(X[a]), float(Y[b]))  # noqa: E731
    edge_x, edge_y = 0.5 * rows * res, 0.5 * cols * res
    shapes = [
        [P(60, 60), P(60, 60), P(70, 64)],                           # a repeated pose
        [P(50, 50)] * 3,                                             # every segment of length 0: lengthPath 0/0
        [P(40, 90), (float(X[40]) + 0.3 * res, float(Y[90]) - 0.2 * res)],   # both ends in one cell
        [P(30, 20), P(30, 70)],                                      # a row
        [P(20, 100), P(90, 100)],                                    # a column
        [P(100, 20), P(140, 60)],                                    # an exact diagonal
        [P(90, 70), P(100, 110)],                                    # steep
        [P(70, 30), P(75, 110)],
        [P(80, 80), (edge_x + 0.3, 0.0)],                            # one end outside the map
        [(float(X[60]) + 0.5 * res, float(Y[60]) + 0.5 * res), (float(X[66]) - 0.5 * res, float(Y[61]))],   # on cell boundaries
        [(edge_x - 1e-9, 0.0), (edge_x - 0.2, -edge_y + 1e-9)],      # on the map edge
        [(edge_x, 0.1)],
    ]
    # a path back and forth over one patch, more than 32 segments: its cells revisit earlier segments' checked and unchecked cells
    zig = []
    for k in range(44):
        zig.append(P(50 + (k % 3) * 3, 40 + (k % 4)) if k % 2 == 0 else P(63 + (k % 5), 47 + 2 * (k % 3)))
    zig2 = [P(110 + 2 * (k % 3), 60 + (k % 5)) if k % 2 == 0 else P(115 + (k % 2), 75 + 3 * (k % 4)) for k in range(40)]
    shapes += [zig, zig2]
    fps = [np.asarray([(0.1, 0.05, 0.0)], np.float32),                            # one vertex: hulls of <= 3 points
           np.asarray([(-0.2, -0.1, 0.0), (0.0, 0.0, 0.1), (0.2, 0.1, 0.0)], np.float32),   # collinear
           np.asarray(YAML, np.float32)]
    paths = []
    for s in shapes:
        for r, u in ((0.1, 1), (0.2, 0)):
            paths.append((s, r, -1, 0, u))
        for k, cons in ((0, 0), (1, 1), (2, 0), (2, 1)):
            if len(s) * (1 if not cons else len(fps[k])) <= 1024:
                paths.append(([(*p, 0.0, 0.0, 0.0, 0.0, 1.0) for p in s], NAN, k, cons, 1))
    R = pc.request(paths, fps)
    cap = mixed_request(np.random.default_rng(4), og, 0, [])   # only the conservative YAML path of 256 poses
    return join([R, dict(cap, fps=fps)])


@pytest.mark.parametrize("default", [0.3, NAN])
def test_path_shapes(te, ctx, oracle, default):
    """Zero-length segments, both ends in one cell, rows, columns, diagonals and steep lines, an end outside the map, poses on
    cell boundaries and on the map edge, paths that revisit their own cells across more than 32 segments, one-vertex and
    collinear footprints, and a conservative path at the 1024-vertex cap."""
    m = built_map(spacing=48)
    kw = dict(traversability_default=default, **BUILT_GAP)
    R = shape_request(oracle.Geometry.make(*m["traversability"].shape, 0.02), m)
    assert np.diff(R["begin"]).max() == 256 and R["cons"][-1] == 1
    ref = stateless(te, ctx, oracle, m, kw, R)
    nonvacuous(ref, default)
    on_map(te, ctx, oracle, m, kw, [R])


# ---- the replay of the service loop on a te_map --------------------------------------------------------------------------------

REPLAY = {
    # case: (map, parameters, request), the oracle's is_safe on the te_map (None: the first and the last path only)
    "nan": (lambda: pc.nan_case(NAN), [1, 0]),
    "inf": (lambda: pc.nan_case(INF), [1, 0]),
    "-inf": (lambda: pc.nan_case(-INF), [1, 0]),
    "offset0": (lambda: pc.ring_case(0), [1, 0]),
    "offset0-integer-norm": (lambda: pc.ring_case(1), [0, 0]),
    "radius-only": (lambda: pc.nan_case(NAN, cups=(1, 1), radii=(0.2, 0.26)), [1, 0]),
    "six-lanes": (lambda: pc.nan_case(INF, cups=(1, 1, 0, 1, 1, 0), radii=(0.2,) * 6), [1, 1, 0, 1, 1, 0]),
    "across-windows": (lambda: pc.nan_case(NAN, fillers=40), None),
    "finite-after-non-finite": (lambda: pc.mixed_case(NAN), [1] * 5),
}


@pytest.mark.parametrize("case", list(REPLAY))
def test_replay_non_finite_store(te, ctx, oracle, case):
    """Checks on one cell after a walk stored a NaN or an infinity there: each walks again (or reads the first finite float
    stored before it), in one window of the replay, across windows, and when asked again on the cache the request left."""
    build, want = REPLAY[case]
    m, kw, R = build()
    ref = stateless(te, ctx, oracle, m, kw, R, pc.RES)
    if case != "offset0-integer-norm":
        assert not math.isfinite(ref[1][0])
    first = on_map(te, ctx, oracle, m, kw, [R], pc.RES)[0]
    if want is not None:
        assert first[0].tolist() == want
    else:
        assert first[0][0] == 1 and first[0][-1] == 0


# ---- the batched entries -------------------------------------------------------------------------------------------------------

SUBSET = {
    "nan-default": dict(traversability_default=NAN),
    "offset0": dict(offset=0.0, radius_is_integer_norm=0),
    "inf-offset0.6": dict(traversability_default=-INF, offset=0.6),
}


@pytest.mark.parametrize("case", list(SUBSET))
def test_batched_entries_equal_the_single_map(te, ctx, oracle, case):
    """te_check_footprint_request_batched and a batched te_map equal the single-map entries bit for bit, answers and caches, and
    the oracle map by map."""
    kw = dict(SUBSET[case], **BUILT_GAP)
    maps = [built_map(spacing=24, seed=10 + k) for k in range(3)]
    g, og = geoms(te, oracle, maps[0], 0.02)
    ft, fo = te_footprint_params(te, **kw), te_footprint_params(oracle, **kw)
    rng = np.random.default_rng(31)
    R = batch_request(rng, og, 60, 3, circular=0.7, cap_path=False)
    fb, fx = footprint_arrays(R, R["fps"])
    pkw = dict(max_footprint_vertices=16, conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=CAP)
    stack = lambda k: np.stack([np.ascontiguousarray(mm[k].T) for mm in maps])  # noqa: E731
    got = ctx.check_footprint_request_batched(g, ft, 3, *(stack(k) for k in MAPL), R["map"], R["begin"], R["poses"], R["radius"],
                                              fb, fx, roughness=stack("roughness"), **pkw)
    for k, mm in enumerate(maps):
        idx = np.nonzero(R["map"] == k)[0]
        S = subset(R, idx)
        sb, sx = footprint_arrays(S, R["fps"])
        one = ctx.check_footprint_request(g, ft, *(mm[n] for n in MAPL), S["begin"], S["poses"], S["radius"], sb, sx,
                                          roughness=mm["roughness"], max_footprint_vertices=16, conservative=S["cons"],
                                          compute_untraversable_polygon=S["cup"], untraversable_capacity=CAP)
        assert_same_answers(tuple(a[idx] for a in got), one, (case, "request_batched", k))
        nonvacuous(one, kw.get("traversability_default", 0.3))
    B = ctx.map()
    B.set_layers_batched(g, 3, *(np.stack([mm[k] for mm in maps]) for k in MAPL), roughness=np.stack([mm["roughness"] for mm in maps]))
    singles = []
    for mm in maps:
        s = ctx.map()
        s.set_layers(g, *(mm[k] for k in MAPL), roughness=mm["roughness"])
        singles.append(s)
    caches = [po.empty_cache(og) for _ in maps]
    for R2 in (R, subset(R, rng.permutation(len(R["kind"])))):
        assert_batch_matches_singles(B, singles, ft, R2, (og, fo, maps, caches))
