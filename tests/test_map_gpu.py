"""te_map on the GPU against the sequential CPU oracle (tests/map_oracle.cpp), bit for bit: is_safe, traversability, area,
untraversable polygons and the traversability_footprint cache after every call."""
import numpy as np
import pytest

import map_oracle as mo
import synth
from test_footprint_request_gpu import _footprint_arrays, _footprints, _request, _same, _same_polygons
from test_paths_fresh_gpu import _layers

pytestmark = pytest.mark.gpu

CAP = 64


def _setup(te, oracle, rows=200, cols=180, res=0.02, seed=61, position=(0.0, 0.0)):
    z = synth.terrain(rows, cols, res, seed, "mixed", position)
    og, g = oracle.Geometry.make(rows, cols, res, position), te.Geometry.make(rows, cols, res, position)
    L, rs = _layers(oracle, og, z, seed)
    return og, g, L, rs


def _params(te, oracle, verify=0, **kw):
    ft, fo = te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults()
    for p in (ft, fo):
        p.verify_roughness = verify
        for k, v in kw.items():
            setattr(p, k, v)
    return ft, fo


def _same_cache(a, b, what):
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) or _same(a.astype(np.float64), b.astype(np.float64)), \
        (what, int(np.sum(~((a == b) | (np.isnan(a) & np.isnan(b))))))


def _both(m, og, ft, fo, OL, cache, R, fps):
    """One request on the map and on the oracle; asserts every output and the cache are identical."""
    fb, fx = _footprint_arrays(R, fps)
    got = m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, max_footprint_vertices=16,
                                    conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=CAP)
    want = mo.check_request(og, fo, OL, cache, R["begin"], R["poses"], R["radius"], fb, fx, conservative=R["cons"],
                            compute_untraversable_polygon=R["cup"], capacity=CAP)
    assert np.array_equal(got[0], want[0]), np.nonzero(got[0] != want[0])[0][:10]
    assert _same(got[1], want[1]) and _same(got[2], want[2])
    _same_polygons(got[3], got[4], want[3], want[4], "polygons")
    _same_cache(m.get_footprint(), cache, "cache")
    return got


def _repeat(R, idx):
    """A request made of paths `idx` of R (planner batches overlap)."""
    b = R["begin"]
    begin = np.concatenate([[0], np.cumsum(b[idx + 1] - b[idx])]).astype(np.int32)
    poses = np.concatenate([R["poses"][b[q]:b[q + 1]] for q in idx])
    return dict(begin=begin, poses=poses, radius=R["radius"][idx], kind=R["kind"][idx], cons=R["cons"][idx], cup=R["cup"][idx])


@pytest.mark.parametrize("verify,slope", [(0, False), (1, True)])
def test_request_sequence_matches_oracle(te, ctx, oracle, verify, slope):
    og, g, L, rs = _setup(te, oracle)
    ft, fo = _params(te, oracle, verify)
    m = ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"],
                 robot_slope=rs if slope else None)
    OL = dict(L, robot_slope=rs if slope else None)
    cache = mo.empty_cache(og)
    rng = np.random.default_rng(7 + verify)
    fps = _footprints(rng)
    R1 = _request(rng, og, 60, fps, circular=0.6, cap_path=False)
    R2 = _request(rng, og, 80, fps, circular=0.7, planner=True, cap_path=False)
    for R in (R1, _repeat(R1, rng.permutation(len(R1["kind"]))), R2, _repeat(R2, np.arange(len(R2["kind"])) // 2)):
        _both(m, og, ft, fo, OL, cache, R, fps)
    cand, keys, stored = m.request_stats()
    assert keys <= cand and stored <= keys
    m.close()


def test_annulus_blocker_revisit_and_single_poses_in_one_cell(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, seed=62)
    ft, fo = _params(te, oracle)
    m = ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"])
    cache = mo.empty_cache(og)
    rng = np.random.default_rng(9)
    n = 300
    xy = rng.uniform([-1.8, -1.6], [1.8, 1.6], (n, 2))
    # every pose twice in the same request, the second one moved inside its cell; then the whole request again
    res = og.resolution
    xy2 = (np.floor(xy / res) + rng.uniform(0.05, 0.95, (n, 2))) * res
    poses = np.zeros((2 * n, 7))
    poses[:n, :2], poses[n:, :2], poses[:, 6] = xy, xy2, 1.0
    R = dict(begin=np.arange(2 * n + 1, dtype=np.int32), poses=poses, radius=np.full(2 * n, 0.1), kind=np.full(2 * n, -1),
             cons=np.zeros(2 * n, np.uint8), cup=(rng.random(2 * n) < 0.5).astype(np.uint8))
    first = _both(m, og, ft, fo, L, cache, R, [])
    second = _both(m, og, ft, fo, L, cache, R, [])
    assert np.sum((first[0][:n] == 0) & (second[0][:n] == 1)) > 0   # unsafe first, safe when asked again
    m.close()


def test_zero_mean_circle_then_fails(te, ctx, oracle):
    """Cells of traversability 0 that pass the predicates: the first check is traversable with mean 0 and stores 0.0, so a later
    check of that cell fails."""
    rows = cols = 64
    og, g = oracle.Geometry.make(rows, cols, 0.05), te.Geometry.make(rows, cols, 0.05)
    ones = np.ones((rows, cols), np.float32, order="F")
    L = dict(traversability=np.zeros((rows, cols), np.float32, order="F"), slope=ones, step=ones, elevation=0 * ones)
    ft, fo = _params(te, oracle)
    m = ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"])
    cache = mo.empty_cache(og)
    poses = np.array([[0.1, 0.2, 0, 0, 0, 0, 1.0]])
    R = dict(begin=np.array([0, 1], np.int32), poses=poses, radius=np.array([0.2]), kind=np.array([-1]), cons=np.zeros(1, np.uint8),
             cup=np.ones(1, np.uint8))
    a = _both(m, og, ft, fo, L, cache, R, [])
    b = _both(m, og, ft, fo, L, cache, R, [])
    assert a[0][0] == 1 and a[1][0] == 0.0 and b[0][0] == 0 and b[3][0] == 20   # fromCircle of the cached 0
    m.close()


def test_sweep_and_request_share_the_cache(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, rows=160, cols=150, seed=63)
    ft, fo = _params(te, oracle)
    m = ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"])
    cache = mo.empty_cache(og)
    rng = np.random.default_rng(11)
    fps = _footprints(rng)
    _both(m, og, ft, fo, L, cache, _request(rng, og, 40, fps, circular=0.8, cap_path=False), fps)
    before = m.get_footprint()
    after = m.footprint(ft)
    sweep = np.empty_like(after)
    ctx.footprint(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], sweep, te.MEM_HOST)
    had = np.isfinite(before)
    assert had.any() and np.array_equal(after[had].view(np.uint32), before[had].view(np.uint32))
    assert np.array_equal(after[~had].view(np.uint32), sweep[~had].view(np.uint32))
    assert np.array_equal(m.get_footprint().view(np.uint32), after.view(np.uint32))
    # a request after the sweep reads the swept cache: start the oracle from it
    cache = np.asfortranarray(after.copy())
    _both(m, og, ft, fo, L, cache, _request(rng, og, 40, fps, circular=0.8, cap_path=False), fps)
    m.close()


def test_new_layers_clear_cache_and_memo(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, rows=150, cols=140, seed=64)
    ft, fo = _params(te, oracle)
    m = ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"])
    rng = np.random.default_rng(13)
    R = _request(rng, og, 40, [], circular=1.0, cap_path=False)
    cache = mo.empty_cache(og)
    _both(m, og, ft, fo, L, cache, R, [])
    # a changed max_gap_width rebuilds the memo and keeps the cache
    ft2, fo2 = _params(te, oracle, max_gap_width=0.1)
    _both(m, og, ft2, fo2, L, cache, _request(rng, og, 40, [], circular=1.0, cap_path=False), [])
    # new layers: empty cache, fresh memo
    L2 = dict(L, traversability=np.asfortranarray(L["traversability"] * np.float32(0.5)))
    m.set_layers(g, L2["traversability"], L2["slope"], L2["step"], L2["elevation"])
    assert np.isnan(m.get_footprint()).all()
    cache = mo.empty_cache(og)
    _both(m, og, ft, fo, L2, cache, R, [])
    # te_map_chain: the chain's layers, an empty cache
    ch = m.chain(g, te.ChainParams.yaml_defaults(0), L["elevation"], outputs=True)
    want = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), L["elevation"])
    for k in ("slope", "step", "roughness", "traversability"):
        assert np.array_equal(ch[k].view(np.uint32), want[k].view(np.uint32)), k
    assert np.isnan(m.get_footprint()).all()
    L3 = dict(traversability=ch["traversability"], slope=ch["slope"], step=ch["step"], elevation=L["elevation"])
    cache = mo.empty_cache(og)
    _both(m, og, ft, fo, L3, cache, R, [])
    m.clear_footprint()
    assert np.isnan(m.get_footprint()).all()
    m.close()


def test_fresh_map_disjoint_cells_equal_stateless_request(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, seed=65)
    ft, _ = _params(te, oracle, verify=1)
    m = ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"], robot_slope=rs)
    rng = np.random.default_rng(15)
    fps = _footprints(rng)
    n = 150
    cells = rng.choice(og.rows * og.cols, n, replace=False)
    res = og.resolution
    poses = np.zeros((n, 7))
    poses[:, 0] = 0.5 * og.rows * res - (cells % og.rows + rng.uniform(0.1, 0.9, n)) * res
    poses[:, 1] = 0.5 * og.cols * res - (cells // og.rows + rng.uniform(0.1, 0.9, n)) * res
    poses[:, 6] = 1.0
    kind = np.where(rng.random(n) < 0.6, -1, rng.integers(0, len(fps), n))
    R = dict(begin=np.arange(n + 1, dtype=np.int32), poses=poses, radius=rng.choice([0.0, 0.1, 0.3], n), kind=kind,
             cons=np.zeros(n, np.uint8), cup=(rng.random(n) < 0.5).astype(np.uint8))
    fb, fx = _footprint_arrays(R, fps)
    got = m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, compute_untraversable_polygon=R["cup"],
                                    untraversable_capacity=CAP)
    want = ctx.check_footprint_request(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], R["begin"], R["poses"],
                                       R["radius"], fb, fx, robot_slope=rs, roughness=L["roughness"],
                                       compute_untraversable_polygon=R["cup"], untraversable_capacity=CAP)
    assert np.array_equal(got[0], want[0]) and _same(got[1], want[1]) and _same(got[2], want[2])
    _same_polygons(got[3], got[4], want[3], want[4], "polygons")
    # te_map_footprint_polygon is te_footprint_polygon on the map's layers
    pts = np.array([[0.2, 0.1], [-0.2, 0.1], [-0.2, -0.1], [0.2, -0.1]])
    gx, gr = m.footprint_polygon(ft, pts, 0.3)
    wx, wr = (np.empty((og.rows, og.cols), np.float32, order="F") for _ in range(2))
    ctx.footprint_polygon(g, ft, pts, 0.3, L["traversability"], L["slope"], L["step"], L["elevation"], wx, wr, te.MEM_HOST,
                          roughness=L["roughness"])
    assert np.array_equal(gx.view(np.uint32), wx.view(np.uint32)) and np.array_equal(gr.view(np.uint32), wr.view(np.uint32))
    m.close()


def test_start_index_layers(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, rows=120, cols=100, seed=66)
    ft, fo = _params(te, oracle)
    sr, sc = 37, 61
    wrap = lambda a: np.asfortranarray(np.roll(np.roll(a, sr, axis=0), sc, axis=1))  # noqa: E731  map cell (i, j) at (i+sr, j+sc)
    gw = te.Geometry.make(og.rows, og.cols, og.resolution)
    gw.start_row, gw.start_col = sr, sc
    m, mw = ctx.map(), ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"], robot_slope=rs)
    mw.set_layers(gw, *(wrap(L[k]) for k in ("traversability", "slope", "step", "elevation")), robot_slope=wrap(rs))
    rng = np.random.default_rng(17)
    R = _request(rng, og, 50, [], circular=1.0, cap_path=False)
    fb, fx = _footprint_arrays(R, [])
    a = m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, compute_untraversable_polygon=R["cup"],
                                  untraversable_capacity=CAP)
    b = mw.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, compute_untraversable_polygon=R["cup"],
                                   untraversable_capacity=CAP)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    assert np.array_equal(mw.get_footprint().view(np.uint32), wrap(m.get_footprint()).view(np.uint32))
    m.close()
    mw.close()


def test_error_codes(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, rows=64, cols=64, seed=67)
    ft, _ = _params(te, oracle)
    m = ctx.map()
    one = dict(path_begin=np.array([0, 1], np.int32), poses=np.array([[0.0, 0, 0, 0, 0, 0, 1]]), radius=np.array([0.2]),
               footprint_begin=np.zeros(2, np.int32), footprint_xyz=np.zeros((0, 3), np.float32))
    with pytest.raises(te.TEError) as e:
        m.check_footprint_request(ft, **one)
    assert e.value.code == -1   # no layers yet
    with pytest.raises(te.TEError) as e:
        m.get_footprint()
    assert e.value.code == -1
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"])
    ftr, _ = _params(te, oracle, verify=1)
    with pytest.raises(te.TEError) as e:
        m.check_footprint_request(ftr, **one)
    assert e.value.code == -2   # verify_roughness without a roughness layer
    with pytest.raises(te.TEError) as e:
        m.check_footprint_request(ft, **dict(one, radius=np.array([3.0])))
    assert e.value.code == -4   # more than 127 rings
    with pytest.raises(te.TEError) as e:
        m.check_footprint_request(ft, **dict(one, radius=np.array([-1.0])))
    assert e.value.code == -1
    with pytest.raises(te.TEError) as e:
        m.check_footprint_request(ft, max_footprint_vertices=17, **one)
    assert e.value.code == -1
    with pytest.raises(te.TEError) as e:
        m.set_layers(g, None, L["slope"], L["step"], L["elevation"])
    assert e.value.code == -2
    m.close()
