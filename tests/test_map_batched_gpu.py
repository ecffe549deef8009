"""A te_map holding a batch of maps (te_map_chain_batched, te_map_set_layers_batched and the _batched map entries).  For every map,
what a batched call returns or stores must equal, bit for bit, what a single-map te_map holding that map alone returns or stores
for the same calls restricted to it: request answers, untraversable polygons and the traversability_footprint cache afterwards."""
import numpy as np
import pytest

import paths_oracle as po
import synth
from helpers import batch_request, chain_layers, footprint_arrays, footprint_params, request_footprints, subset
from map_helpers import assert_batch_matches_singles, assert_same_cache, close_maps  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, NMAPS = 200, 180, 0.02, 5
EMPTY = 3    # the map without paths
BAD_ARG, UNSUPPORTED = -1, -4
FILTER = ("traversability", "slope", "step", "elevation")


@pytest.fixture(scope="module")
def maps(te, oracle):
    """NMAPS maps of one geometry, each its own terrain (different seeds): oracle chain layers, roughness with zero patches and a
    robot_slope layer with zeros and NaNs (helpers.chain_layers)."""
    og, g = oracle.Geometry.make(ROWS, COLS, RES), te.Geometry.make(ROWS, COLS, RES)
    per = []
    for k in range(NMAPS):
        z = synth.terrain(ROWS, COLS, RES, 81 + k, "mixed")
        L, rs = chain_layers(oracle, og, z, 81 + k)
        per.append(dict(L, robot_slope=rs))
    return og, g, per


def _stack(per, key):
    return np.stack([p[key] for p in per])


def _load(ctx, g, per, slope, rough=True):
    """The batch te_map, and one single-map te_map per map with the same layers."""
    opt = lambda p, k, on: p[k] if on else None  # noqa: E731
    b = ctx.map()
    b.set_layers_batched(g, len(per), *(_stack(per, k) for k in FILTER), roughness=_stack(per, "roughness") if rough else None,
                         robot_slope=_stack(per, "robot_slope") if slope else None)
    singles = []
    for p in per:
        s = ctx.map()
        s.set_layers(g, *(p[k] for k in FILTER), roughness=opt(p, "roughness", rough), robot_slope=opt(p, "robot_slope", slope))
        singles.append(s)
    return b, singles


def _request(rng, og, fps, npaths, planner=False):
    """A mixed request whose paths interleave the maps in no order and leave map EMPTY out."""
    return batch_request(rng, og, npaths, NMAPS, fps, exclude=EMPTY, circular=0.6, planner=planner, cap_path=False)


def _close(*ms):
    for m in ms:
        m.close()


def test_chain_batched_layers_equal_stateless_batch(te, ctx, maps):
    torch = pytest.importorskip("torch")
    og, g, per = maps
    p = te.ChainParams.yaml_defaults(0)
    elev = _stack(per, "elevation")
    b = ctx.map()
    got = b.chain_batched(g, p, NMAPS, elev, outputs=True)
    assert b.nmaps == NMAPS
    want = {k: np.empty((NMAPS, COLS, ROWS), np.float32) for k in ("slope", "step", "roughness", "traversability")}
    ctx.chain_batched(g, p, NMAPS, np.ascontiguousarray(elev.transpose(0, 2, 1)), want["slope"], want["step"], want["roughness"],
                      want["traversability"], te.MEM_HOST)
    names = {"traversability": "traversability", "traversability_slope": "slope", "traversability_step": "step",
             "traversability_roughness": "roughness"}
    host = b.get_layers(list(names) + ["elevation"])
    dev = torch.empty(len(names) * NMAPS * ROWS * COLS, dtype=torch.float32, device="cuda")
    dview = b.get_layers(list(names), out=dev, memory=te.MEM_DEVICE)
    ctx.synchronize()
    for name, k in names.items():
        w = want[k].transpose(0, 2, 1)
        assert np.array_equal(got[k].view(np.uint32), w.view(np.uint32)), k
        assert np.array_equal(host[name].view(np.uint32), w.view(np.uint32)), name
        assert np.array_equal(dview[name].cpu().numpy().view(np.uint32), w.view(np.uint32)), name
    assert np.array_equal(host["elevation"].view(np.uint32), elev.view(np.uint32))
    assert np.isnan(b.get_footprint()).all()
    with pytest.raises(te.TEError) as e:
        b.get_layers(["robot_slope"])
    assert e.value.code == -2   # te_map_chain_batched leaves the batch without robot_slope
    # a batch of one map is te_map_chain
    one, single = ctx.map(), ctx.map()
    one.chain_batched(g, p, 1, elev[2:3])
    single.chain(g, p, per[2]["elevation"])
    a, s = one.get_layers(list(names)), single.get_layers(list(names))
    for name in names:
        assert np.array_equal(a[name].view(np.uint32), s[name].view(np.uint32)), name
    _close(b, one, single)


@pytest.mark.parametrize("verify,slope,with_oracle", [(0, False, True), (1, True, False), (0, True, False)])
def test_request_sequences_equal_single_maps(te, ctx, oracle, maps, verify, slope, with_oracle):
    og, g, per = maps
    ft, fo = footprint_params(te, oracle, verify)
    b, singles = _load(ctx, g, per, slope)
    state = None
    if with_oracle:
        OL = [dict(p, robot_slope=p["robot_slope"] if slope else None) for p in per]
        state = (og, fo, OL, [po.empty_cache(og) for _ in per])
    rng = np.random.default_rng(31 + 2 * verify + slope)
    fps = request_footprints(rng)
    R1 = _request(rng, og, fps, 90)
    R2 = _request(rng, og, fps, 80, planner=True)
    again = subset(R1, rng.permutation(len(R1["kind"])))   # revisits: every cell R1 stored, in another order
    for R in (R1, again, R2):
        assert_batch_matches_singles(b, singles, ft, R, state)
    cand, keys, stored = b.request_stats()
    assert 0 < stored <= keys <= cand
    assert np.isnan(b.get_footprint()[EMPTY]).all()
    _close(b, *singles)


def test_same_cell_first_touched_on_two_maps(te, ctx, oracle, maps):
    """Single-pose circular paths at the same position on two maps whose circles differ: the keys must stay apart, so one map
    stores a traversable value and the other an untraversable one in the same request."""
    og, g, per = maps
    ft, _ = footprint_params(te, oracle)
    rng = np.random.default_rng(5)
    n = 400
    cells = rng.choice(ROWS * COLS, n, replace=False)   # one pose per cell, so every check is a first touch
    ci, cj = cells % ROWS, cells // ROWS
    poses = np.zeros((n, 7))
    poses[:, 0] = 0.5 * ROWS * RES - (ci + rng.uniform(0.1, 0.9, n)) * RES
    poses[:, 1] = 0.5 * COLS * RES - (cj + rng.uniform(0.1, 0.9, n)) * RES
    poses[:, 6] = 1.0
    one = dict(begin=np.arange(n + 1, dtype=np.int32), poses=poses, radius=np.full(n, 0.15), kind=np.full(n, -1),
               cons=np.zeros(n, np.uint8), cup=np.ones(n, np.uint8))
    fb, fx = footprint_arrays(one, [])
    safe = [ctx.check_footprint_request(g, ft, *(per[k][x] for x in FILTER), one["begin"], poses, one["radius"], fb, fx,
                                        compute_untraversable_polygon=one["cup"])[0] for k in (0, 1)]
    differ = np.nonzero(safe[0] != safe[1])[0][:20]
    assert len(differ) >= 4
    idx = np.repeat(differ, 2)
    R = subset(dict(one, map=np.zeros(n, np.int32)), idx)
    R["map"], R["fps"] = np.tile(np.array([0, 1], np.int32), len(differ)), []
    b, singles = _load(ctx, g, per, False)
    got = assert_batch_matches_singles(b, singles, ft, R)
    assert np.array_equal(got[0][0::2], safe[0][differ]) and np.array_equal(got[0][1::2], safe[1][differ])
    cache = b.get_footprint()
    stored = cache[:2, ci[differ], cj[differ]]
    assert np.isfinite(stored).all() and (stored[0].view(np.uint32) != stored[1].view(np.uint32)).any()
    _close(b, *singles)


def test_whole_map_entries_on_a_batch(te, ctx, oracle, maps):
    og, g, per = maps
    ft, _ = footprint_params(te, oracle, verify=1)
    b, singles = _load(ctx, g, per, True)
    rng = np.random.default_rng(41)
    fps = request_footprints(rng)
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 60))
    before = b.get_footprint()
    swept = b.footprint(ft)
    for k, s in enumerate(singles):   # te_map_footprint keeps each map's cached cells, as on a single map
        assert_same_cache(swept[k], s.footprint(ft), ("footprint", k))
    had = np.isfinite(before)
    assert had.any() and np.array_equal(swept[had].view(np.uint32), before[had].view(np.uint32))
    assert_same_cache(b.get_footprint(), swept, "cache after the sweep")
    # the polygon entries are the stateless batched ones on the resident layers
    pts = np.array([[0.3, 0.2], [-0.3, 0.2], [-0.3, -0.2], [0.3, -0.2]])
    yaws = [0.0, 0.4, 1.3, -2.0]
    lay = {k: np.ascontiguousarray(_stack(per, k).transpose(0, 2, 1)) for k in FILTER + ("roughness",)}
    want = np.empty((len(yaws), NMAPS, COLS, ROWS), np.float32)
    ctx.footprint_polygon_yaws(g, ft, NMAPS, pts, yaws, *(lay[k] for k in FILTER), want, te.MEM_HOST, roughness=lay["roughness"])
    got = b.footprint_polygon_yaws(ft, pts, yaws)
    assert got.shape == (len(yaws), NMAPS, ROWS, COLS)
    assert np.array_equal(got.view(np.uint32), want.transpose(0, 1, 3, 2).view(np.uint32))
    ww, wb = (np.empty((NMAPS, COLS, ROWS), np.float32) for _ in range(2))
    wy = np.empty((NMAPS, COLS, ROWS), np.int32)
    ctx.footprint_polygon_yaws_reduce(g, ft, NMAPS, pts, yaws, *(lay[k] for k in FILTER), ww, wb, wy, te.MEM_HOST,
                                      roughness=lay["roughness"])
    for a, w in zip(b.footprint_polygon_yaws_reduce(ft, pts, yaws), (ww, wb, wy)):
        assert np.array_equal(a.view(np.uint32), w.transpose(0, 2, 1).view(np.uint32))
    wx, wr = (np.empty((NMAPS, COLS, ROWS), np.float32) for _ in range(2))
    ctx.footprint_polygon_batched(g, ft, NMAPS, pts, 0.7, *(lay[k] for k in FILTER), wx, wr, te.MEM_HOST, roughness=lay["roughness"])
    for a, w in zip(b.footprint_polygon(ft, pts, 0.7), (wx, wr)):
        assert np.array_equal(a.view(np.uint32), w.transpose(0, 2, 1).view(np.uint32))
    assert_same_cache(b.get_footprint(), swept, "the polygon entries leave the cache alone")
    b.clear_footprint()
    assert np.isnan(b.get_footprint()).all()
    _close(b, *singles)


def test_read_side_on_a_batch(te, ctx, oracle, maps):
    torch = pytest.importorskip("torch")
    og, g, per = maps
    b, singles = _load(ctx, g, per, True)
    names = ["traversability", "elevation", "robot_slope"]
    rng = np.random.default_rng(51)
    nwin = 12
    pos = rng.uniform([-2.2, -2.0], [2.2, 2.0], (nwin, 2))
    pos[3] = [9.0, 0.0]   # outside every map: a failing window
    ln = rng.uniform(0.1, 1.5, (nwin, 2))
    wm = rng.integers(0, NMAPS, nwin).astype(np.int32)
    got = b.get_submaps_batched(wm, pos, ln, names)
    assert not got[3][0]["success"]
    for k in range(nwin):
        want = singles[wm[k]].get_submaps(pos[k:k + 1], ln[k:k + 1], names)[0]
        for f in ("success", "rows", "cols", "top_row", "top_col", "requested_row", "requested_col"):
            assert got[k][0][f] == want[0][f], (k, f)
        if want[1] is None:
            assert got[k][1] is None
            continue
        for n in names:
            assert np.array_equal(got[k][1][n].view(np.uint32), want[1][n].view(np.uint32)), (k, n)
    # valid_at: host and device memory, and a map outside the batch on the device
    n = 500
    xy = rng.uniform([-2.4, -2.2], [2.4, 2.2], (n, 2))
    pm = rng.integers(0, NMAPS, n).astype(np.int32)
    want = np.zeros(n, np.uint8)
    for k in range(NMAPS):
        idx = np.nonzero(pm == k)[0]
        want[idx] = singles[k].valid_at(xy[idx])
    assert 0 < want.sum() < n
    assert np.array_equal(b.valid_at_batched(pm, xy), want)
    pm_bad = pm.copy()
    pm_bad[::7] = NMAPS
    pm_bad[3::7] = -1
    out = torch.full((n,), 9, dtype=torch.uint8, device="cuda")
    b.valid_at_batched(torch.from_numpy(pm_bad).cuda(), torch.from_numpy(xy).cuda(), out=out, memory=te.MEM_DEVICE)
    ctx.synchronize()
    dv = out.cpu().numpy()
    bad = (pm_bad < 0) | (pm_bad >= NMAPS)
    assert (dv[bad] == 0).all() and np.array_equal(dv[~bad], want[~bad])
    _close(b, *singles)


def test_error_codes(te, ctx, oracle, maps):
    og, g, per = maps
    ft, _ = footprint_params(te, oracle)
    b = ctx.map()
    lay = [_stack(per, k) for k in FILTER]
    with pytest.raises(te.TEError) as e:
        b.set_layers_batched(g, 0, *(a[:0] for a in lay))
    assert e.value.code == BAD_ARG
    with pytest.raises(te.TEError) as e:
        b.chain_batched(g, te.ChainParams.yaml_defaults(0), 0, lay[3][:0])
    assert e.value.code == BAD_ARG
    gw = te.Geometry.make(ROWS, COLS, RES)
    gw.start_row, gw.start_col = 5, 7
    with pytest.raises(te.TEError) as e:
        b.set_layers_batched(gw, 2, *(a[:2] for a in lay))
    assert e.value.code == UNSUPPORTED
    with pytest.raises(te.TEError) as e:
        b.chain_batched(gw, te.ChainParams.yaml_defaults(0), 2, lay[3][:2])
    assert e.value.code == UNSUPPORTED
    b.set_layers_batched(g, NMAPS, *lay)
    assert b.nmaps == NMAPS
    rng = np.random.default_rng(61)
    fps = request_footprints(rng)
    R = _request(rng, og, fps, 8)
    fb, fx = footprint_arrays(R, fps)
    args = (R["begin"], R["poses"], R["radius"], fb, fx)
    for bad in (NMAPS, -1):
        with pytest.raises(te.TEError) as e:
            b.check_footprint_request_batched(ft, np.where(np.arange(8) == 5, bad, R["map"]).astype(np.int32), *args)
        assert e.value.code == BAD_ARG
        with pytest.raises(te.TEError) as e:
            b.get_submaps_batched([0, bad], [[0.0, 0.0], [0.1, 0.1]], [[0.5, 0.5], [0.5, 0.5]], ["traversability"])
        assert e.value.code == BAD_ARG
        with pytest.raises(te.TEError) as e:
            b.valid_at_batched([bad, 0], [[0.0, 0.0], [0.1, 0.1]])
        assert e.value.code == BAD_ARG
    # the entries that address one map fail on a batch and name their _batched entry
    for call, entry in ((lambda: b.check_footprint_request(ft, *args), "te_map_check_footprint_request_batched"),
                        (lambda: b.get_submaps([[0.0, 0.0]], [[0.5, 0.5]], ["traversability"]), "te_map_get_submaps_batched"),
                        (lambda: b.valid_at([[0.0, 0.0]]), "te_map_valid_at_batched")):
        with pytest.raises(te.TEError) as e:
            call()
        assert e.value.code == BAD_ARG and entry in str(e.value)
    # the same entries on a batch of one map work
    b.set_layers_batched(g, 1, *(a[:1] for a in lay))
    assert b.valid_at([[0.0, 0.0]])[0] in (0, 1)
    b.close()
