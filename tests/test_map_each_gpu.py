"""Maps of a batched te_map with robots of their own: te_map_check_footprint_request_each, te_map_check_footprint_request_device_each
and te_map_footprint_each take one te_footprint_params per map.  For every map m, everything they return or store for m must be,
bit for bit, what the single-parameter entries return or store on a single-map te_map holding map m at its position, given
params[m]; with every params[m] the same they must be those entries, launches included."""
import ctypes as C

import numpy as np
import pytest

import paths_params_cases as pc
from helpers import (assert_same_answers, batch_request, footprint_arrays, subset, te_footprint_params, walled_batch, wrap)
from map_helpers import CAP, MISSING_LAYER, ask, assert_same_cache, close_maps, held  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, NMAPS = 150, 130, 0.02, 8
BAD_ARG = -1
UNSUPPORTED = -4
BIG = 1 << 22   # max_checks that no request here reaches
NAMES = ("traversability", "slope", "step", "elevation")
POS = np.array([(0.0, 0.0), (12.5, -3.25), (-40.31, 7.7), (0.37, 0.05), (101.125, 52.39), (-7.77, 0.05), (3.0, 3.0), (-0.5, 9.1)])
START = np.array([(0, 0)] * 3 + [(37, 53)] + [(0, 0)] * 4, np.int32)   # map 3 comes in its own circular-buffer order
# Per-map robots: the defaults the reference's YAML gives, and the parameters the path-check cases vary (paths_params_cases.py)
ROBOTS = [dict(),
          dict(traversability_default=0.0, max_gap_width=0.1, offset=0.0),
          dict(traversability_default=1.0, critical_step_height=0.05, verify_roughness=1),
          dict(traversability_default=float("nan"), radius_is_integer_norm=0, offset=0.05),
          dict(pc.REPLAY_GAP, traversability_default=0.3, verify_roughness=1, offset=0.3),
          dict(critical_step_height=0.25, max_gap_width=0.5, radius_is_integer_norm=0),
          dict(traversability_default=0.3, offset=0.0, radius_is_integer_norm=0, verify_roughness=1),
          dict(max_gap_width=0.2, critical_step_height=0.08)]


@pytest.fixture(scope="module")
def world(oracle):
    return walled_batch(oracle, ROWS, COLS, RES, NMAPS, 91, robot_slope=True)


def _layers(world, k=None, rough=True):
    """(n, rows, cols) layers of every map (k None, map 3 in its buffer order) or of map k alone, as set_layers_batched takes them."""
    names = NAMES + (("roughness",) if rough else ()) + ("robot_slope",)
    out = {}
    for n in names:
        a = world[n].transpose(0, 2, 1)
        out[n] = a[k:k + 1] if k is not None else np.stack([wrap(a[j], START[j]) for j in range(NMAPS)])
    return out


def _load(ctx, te, world, k=None, rough=True):
    """The batch (k None: every map at its position, map 3 with its start index) or a single-map te_map holding map k."""
    m = ctx.map()
    L = _layers(world, k, rough)
    g = te.Geometry.make(ROWS, COLS, RES)
    pos, start = (POS, START) if k is None else (POS[k:k + 1], None)
    m.set_layers_batched(g, len(L["traversability"]), *(L[n] for n in NAMES), roughness=L.get("roughness"),
                         robot_slope=L["robot_slope"], positions=pos, start_index=start)
    return m


def _params(te, robots=ROBOTS):
    return [te_footprint_params(te, **r) for r in robots]


def _cache(m, k):
    """Map k's cache in default order."""
    c = m.get_footprint()[k]
    return np.roll(c, (-int(START[k][0]), -int(START[k][1])), axis=(0, 1))


def _requests(oracle, n=3, npaths=90, seed=5):
    """n requests of circular and polygonal paths mixed, interleaved over the maps, each map's paths at its own position."""
    og = oracle.Geometry.make(ROWS, COLS, RES)
    rng = np.random.default_rng(seed)
    return [batch_request(rng, og, npaths, NMAPS, offsets=POS, cap_path=False, circular=0.6) for _ in range(n)]


def _each(m, params, R):
    fb, fx = footprint_arrays(R, R["fps"])
    return m.check_footprint_request_each(params, R["map"], R["begin"], R["poses"], R["radius"], fb, fx, max_footprint_vertices=16,
                                          conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=CAP)


def _device(m, params, R, fp=None):
    """The request through te_map_check_footprint_request_device_each (fp: te_map_check_footprint_request_device with fp);
    returns (run, fetch)."""
    import torch
    fb, fx = footprint_arrays(R, R["fps"])
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    n = len(R["kind"])
    out = dict(is_safe=torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
               area_out=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
               untraversable_count=torch.full((n,), 99, dtype=torch.int32, device="cuda"),
               untraversable_xy=torch.zeros((n, CAP, 2), dtype=torch.float64, device="cuda"))
    args = (dev(R["begin"], np.int32), dev(R["poses"], np.float64), dev(R["radius"], np.float64), dev(fb, np.int32), dev(fx, np.float32))
    kw = dict(max_checks=BIG, path_map=dev(R["map"], np.int32), max_footprint_vertices=16, conservative=dev(R["cons"], np.uint8),
              compute_untraversable_polygon=dev(R["cup"], np.uint8), untraversable_capacity=CAP, params=None if fp else params, **out)
    torch.cuda.synchronize()

    def run():
        m.check_footprint_request_device(fp, *args, **kw)

    def fetch():
        torch.cuda.synchronize()
        return tuple(out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out", "untraversable_count",
                                                     "untraversable_xy"))
    return run, fetch, out


def _on_singles(singles, params, R):
    """R's paths map by map on the single maps, each with its map's parameters: the answers in request order and the summed
    request_stats."""
    n = len(R["kind"])
    want = [np.zeros(n, np.uint8), np.zeros(n), np.zeros(n), np.zeros(n, np.int32), np.zeros((n, CAP, 2))]
    stats = np.zeros(3, np.int64)
    for k, s in enumerate(singles):
        idx = np.nonzero(R["map"] == k)[0]
        if not len(idx):
            continue
        for o, v in zip(want, ask(s, params[k], subset(R, idx))):
            o[idx] = v
        stats += s.request_stats()
    return want, tuple(int(v) for v in stats)


def test_mixed_parameters_match_single_maps(te, ctx, oracle, world):
    params = _params(te)
    b = _load(ctx, te, world)
    singles = [_load(ctx, te, world, k) for k in range(NMAPS)]
    for r, R in enumerate(_requests(oracle)):
        got = _each(b, params, R)
        want, stats = _on_singles(singles, params, R)
        assert_same_answers(got, want, ("request", r))
        assert b.request_stats() == stats, r
        for k, s in enumerate(singles):
            assert_same_cache(_cache(b, k), s.get_footprint(), ("cache", r, k))


def test_device_entry_equals_host_entry(te, ctx, oracle, world):
    params = _params(te)
    H, D = _load(ctx, te, world), _load(ctx, te, world)
    for r, R in enumerate(_requests(oracle, seed=8)):
        want = _each(H, params, R)
        run, fetch, _ = _device(D, params, R)
        run()
        assert_same_answers(fetch(), want, ("request", r))
        assert D.request_stats() == H.request_stats(), r
        assert_same_cache(D.get_footprint(), H.get_footprint(), ("cache", r))


def test_graph_capture_replays_the_device_entry(te, ctx, oracle, world):
    import torch
    params = _params(te)
    R = _requests(oracle, n=1, seed=13)[0]
    H, D = _load(ctx, te, world), _load(ctx, te, world)
    want = _each(H, params, R)
    run, fetch, out = _device(D, params, R)
    side = torch.cuda.Stream()
    ctx.set_stream(side.cuda_stream)
    try:
        with torch.cuda.stream(side):
            run()   # warm-up: workspace, ring table, memo and the per-map parameter table
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
            D.clear_footprint()
            run()
        for t in out.values():
            t.fill_(0)
        D.clear_footprint()
        side.synchronize()
        graph.replay()
        torch.cuda.synchronize()
    finally:
        ctx.set_stream(None)
    assert_same_answers(fetch(), want)
    assert_same_cache(D.get_footprint(), H.get_footprint())


def _launches(ctx, fn):
    a = ctx.stats()[0]
    fn()
    return ctx.stats()[0] - a


def test_uniform_parameters_are_the_existing_entries(te, ctx, oracle, world):
    p = te_footprint_params(te, verify_roughness=1, offset=0.1)
    params = [p] * NMAPS
    E, B = _load(ctx, te, world), _load(ctx, te, world)
    for r, R in enumerate(_requests(oracle, n=2, seed=21)):
        box = []
        n_each = _launches(ctx, lambda: box.append(_each(E, params, R)))
        n_batched = _launches(ctx, lambda: box.append(ask(B, p, R, R["map"])))
        assert_same_answers(box[0], box[1], ("host", r))
        assert n_each == n_batched, (r, n_each, n_batched)
        assert E.request_stats() == B.request_stats()
        assert_same_cache(E.get_footprint(), B.get_footprint(), ("host cache", r))
        run_e, fetch_e, _ = _device(E, params, R)
        run_b, fetch_b, _ = _device(B, None, R, fp=p)
        assert _launches(ctx, run_e) == _launches(ctx, run_b)
        assert_same_answers(fetch_e(), fetch_b(), ("device", r))
        assert E.request_stats() == B.request_stats()
        assert_same_cache(E.get_footprint(), B.get_footprint(), ("device cache", r))
    # the sweep: a whole batch is te_map_footprint, a selection te_map_footprint_maps
    E.clear_footprint()
    B.clear_footprint()
    box = []
    assert _launches(ctx, lambda: box.append(E.footprint_each(params))) == _launches(ctx, lambda: box.append(B.footprint(p)))
    assert_same_cache(box[0], box[1], "sweep")
    sel = [6, 1, 3]
    box = []
    assert _launches(ctx, lambda: box.append(E.footprint_each(params, sel))) == _launches(ctx, lambda: box.append(B.footprint_maps(p, sel)))
    assert_same_cache(box[0], box[1], "sweep selection")
    assert_same_cache(E.get_footprint(), B.get_footprint(), "caches after the sweeps")


def test_one_maps_memo_key_leaves_the_others_alone(te, ctx, oracle, world):
    """Map 2's max_gap_width changes between two requests: every other map answers and caches as in a run where nothing changed,
    and map 2 as a single map given its new parameters."""
    params = _params(te)
    changed = list(params)
    changed[2] = te_footprint_params(te, **dict(ROBOTS[2], max_gap_width=0.02))
    A, U = _load(ctx, te, world), _load(ctx, te, world)
    s2 = _load(ctx, te, world, 2)
    R1, R2 = _requests(oracle, n=2, seed=34)
    for m in (A, U):
        _each(m, params, R1)
    ask(s2, params[2], subset(R1, np.nonzero(R1["map"] == 2)[0]))
    got, same = _each(A, changed, R2), _each(U, params, R2)
    ask_2 = ask(s2, changed[2], subset(R2, np.nonzero(R2["map"] == 2)[0]))
    other = R2["map"] != 2
    assert_same_answers(tuple(a[other] for a in got), tuple(a[other] for a in same), "other maps")
    assert_same_answers(tuple(a[~other] for a in got), ask_2, "map 2")
    for k in range(NMAPS):
        if k != 2:
            assert_same_cache(_cache(A, k), _cache(U, k), ("cache", k))
    assert_same_cache(_cache(A, 2), s2.get_footprint(), "cache of map 2")


def test_memo_is_cleared_per_map(te, ctx, oracle, world):
    """te_map_get_memo after requests on map 0 alone: a changed memo key clears that map's memo bytes only, under the _each entry
    (map 2's max_gap_width) and under a single-parameter entry (every map whose key differs from p's)."""
    params = _params(te)
    changed = list(params)
    changed[2] = te_footprint_params(te, **dict(ROBOTS[2], max_gap_width=0.02))
    b = _load(ctx, te, world)
    R1, R2, R3 = _requests(oracle, n=3, seed=44)
    _each(b, params, R1)
    m1 = b.get_memo()
    assert all(m1[k].any() for k in range(NMAPS))   # every map has paths in R1 (batch_request's first paths visit every map)
    only0 = lambda R: subset(R, np.nonzero(R["map"] == 0)[0])  # noqa: E731
    _each(b, changed, only0(R2))
    m2 = b.get_memo()
    assert not m2[2].any()
    for k in range(1, NMAPS):
        if k != 2:
            assert np.array_equal(m2[k], m1[k]), k
    assert np.array_equal(m2[0][m1[0] != 0], m1[0][m1[0] != 0])   # map 0 keeps what it had and evaluates more
    # the single-parameter entry with map 0's parameters: maps 0 and 3 share its key (max_gap_width, critical_step_height,
    # verify_roughness), the others are cleared
    ask(b, params[0], only0(R3), np.zeros(int((R3["map"] == 0).sum()), np.int32))
    m3 = b.get_memo()
    assert np.array_equal(m3[3], m2[3])
    assert np.array_equal(m3[0][m2[0] != 0], m2[0][m2[0] != 0])
    for k in (1, 2, 4, 5, 6, 7):
        assert not m3[k].any(), k


def test_sweep_groups_parameter_sets(te, ctx, oracle, world):
    sets = [te_footprint_params(te, radius=0.3, offset=0.15),
            te_footprint_params(te, radius=0.2, offset=0.0, traversability_default=0.3, radius_is_integer_norm=0, verify_roughness=1),
            te_footprint_params(te, radius=0.45, offset=0.05, max_gap_width=0.1, critical_step_height=0.05)]
    params = [sets[k % 3] for k in range(NMAPS)]
    b = _load(ctx, te, world)
    singles = [_load(ctx, te, world, k) for k in range(NMAPS)]
    want = [s.footprint(params[k]) for k, s in enumerate(singles)]
    got = b.footprint_each(params)
    for k in range(NMAPS):
        assert_same_cache(np.roll(got[k], (-int(START[k][0]), -int(START[k][1])), axis=(0, 1)), want[k], ("whole", k))
        assert_same_cache(_cache(b, k), want[k], ("whole cache", k))
    # a selection, on emptied caches; the maps it leaves out keep theirs
    b.clear_footprint()
    sel = [5, 3, 0, 7, 1]
    got = b.footprint_each(params, sel)
    caches = b.get_footprint()
    for j, k in enumerate(sel):
        assert_same_cache(np.roll(got[j], (-int(START[k][0]), -int(START[k][1])), axis=(0, 1)), want[k], ("selection", k))
    for k in set(range(NMAPS)) - set(sel):
        assert np.isnan(caches[k]).all(), k
    # launches: those of one te_map_footprint_maps per distinct set, outputs aside
    idx = np.asarray([0, 3], np.int32)
    one = _launches(ctx, lambda: b._check(b._L.te_map_footprint_maps(b._h, C.byref(sets[0]), 2, idx.ctypes.data, None, 0)))
    arr = (te.FootprintParams * NMAPS)(*params)
    assert _launches(ctx, lambda: b._check(b._L.te_map_footprint_each(b._h, arr, 0, None, None, 0))) == 3 * one
    sel_idx = np.asarray(sel, np.int32)
    assert _launches(ctx, lambda: b._check(b._L.te_map_footprint_each(b._h, arr, len(sel), sel_idx.ctypes.data, None, 0))) == 3 * one


def test_errors_leave_the_map_unchanged(te, ctx, oracle, world):
    params = _params(te)
    b = _load(ctx, te, world)
    R1, R2 = _requests(oracle, n=2, seed=55)
    _each(b, params, R1)
    before, memo = held(te, b), b.get_memo()
    fb, fx = footprint_arrays(R2, R2["fps"])
    bad = list(params)
    bad[5] = te_footprint_params(te, **dict(ROBOTS[5], offset=-0.1))
    # the last of three parameter sets reaches 150 cells, beyond the sweep's 120: no set may be swept first
    far = [te_footprint_params(te, radius=0.3 if k < 4 else 0.2 if k < 7 else 3.0) for k in range(NMAPS)]

    def expect(code, fn):
        with pytest.raises(te.TEError) as e:
            fn()
        assert e.value.code == code
        after = held(te, b)
        for n in before:
            assert_same_cache(after[n], before[n], n)
        assert np.array_equal(b.get_memo(), memo)

    def host_null():
        n = len(R2["kind"])
        safe, trav, area = np.zeros(n, np.uint8), np.zeros(n), np.zeros(n)
        pm = np.ascontiguousarray(R2["map"], np.int32)
        b._check(b._L.te_map_check_footprint_request_each(b._h, None, pm.ctypes.data, n, len(R2["poses"]), R2["begin"].ctypes.data,
                                                           R2["poses"].ctypes.data, R2["radius"].ctypes.data, len(fx), fb.ctypes.data,
                                                           fx.ctypes.data, 16, None, None, safe.ctypes.data, trav.ctypes.data,
                                                           area.ctypes.data, 0, None, None))

    expect(BAD_ARG, host_null)
    expect(BAD_ARG, lambda: b._check(b._L.te_map_footprint_each(b._h, None, 0, None, None, 0)))
    expect(BAD_ARG, lambda: _each(b, bad, R2))
    expect(BAD_ARG, lambda: _device(b, bad, R2)[0]())
    expect(BAD_ARG, lambda: b.footprint_each(bad))
    expect(BAD_ARG, lambda: b.footprint_each(bad, [0, 5]))
    expect(UNSUPPORTED, lambda: b.footprint_each(far))
    expect(UNSUPPORTED, lambda: b.footprint_each(far, [0, 4, 7]))
    b.footprint_each(bad, [0, 4])   # map 5 is not swept: its parameters are not read
    # verify_roughness on a batch without roughness
    n = _load(ctx, te, world, rough=False)
    _each(n, [params[0]] * NMAPS, R1)
    before, memo = held(te, n), n.get_memo()
    b = n
    for fn in (lambda: _each(b, params, R2), lambda: _device(b, params, R2)[0](), lambda: b.footprint_each(params)):
        expect(MISSING_LAYER, fn)
