"""te_map_chain_submap and te_map_chain_windows on the GPU: a te_map computed from windows of a larger elevation map with a
circular-buffer start index, against the composition they replace (the windows cut by the CPU oracle, tests/windows_oracle.cpp,
then te_map_chain / te_map_chain_batched_at / te_map_chain_maps_at and te_map_carry_layers), bit for bit: every layer, the cache,
the positions, a circular sweep and a mixed request answered afterwards.  Also the agreement of the window rule with getSubmap,
the launch counts and the error table."""
import ctypes as C

import numpy as np
import pytest

import submap_oracle as so
import synth
import windows_oracle as wo
from helpers import assert_same_bits, batch_request, noisy, same_bytes
from map_helpers import ask, assert_same_held, close_maps, held  # noqa: F401

pytestmark = pytest.mark.gpu

RES = 0.02
SRC_ROWS, SRC_COLS, SRC_START, SRC_POS = 1536, 2048, (700, 333), (1.3, -2.7)
FUSED = ("elevation", "upper_bound", "lower_bound")
RAW = ("elevation", "variance", "horizontal_variance_x", "horizontal_variance_y", "horizontal_variance_xy", "time")
BAD_ARG, MISSING_LAYER, UNSUPPORTED = -1, -2, -4


@pytest.fixture(scope="module")
def source(te, oracle):
    """The elevation map: every layer unwrapped (cell (i, j) at [i, j]) and as its circular buffer stores it."""
    rng = np.random.default_rng(7)
    z = synth.terrain(SRC_ROWS, SRC_COLS, RES, 31, "mixed").astype(np.float32)
    lay = {"elevation": z}
    for n in FUSED[1:] + RAW[1:]:
        lay[n] = noisy(rng, (SRC_ROWS, SRC_COLS), nan=0.03, inf=0.01, ninf=0, zero=0.01)
    stored = {n: np.asfortranarray(np.roll(a, SRC_START, axis=(0, 1))) for n, a in lay.items()}
    g = te.Geometry.make(SRC_ROWS, SRC_COLS, RES, SRC_POS)
    g.start_row, g.start_col = SRC_START
    return dict(g=g, og=oracle.Geometry.make(SRC_ROWS, SRC_COLS, RES, SRC_POS), lay=lay, stored=stored,
                p=te.ChainParams.yaml_defaults(0))


def _layers(source, names, memory, torch=None):
    if memory == 0:
        return {n: source["stored"][n] for n in names}
    return {n: torch.from_numpy(np.ascontiguousarray(source["stored"][n].T).reshape(-1)).cuda() for n in names}


def _cut(source, name, top, rows, cols):
    return wo.cut(source["stored"][name], SRC_START, top, rows, cols)


def _held(te, m):
    return held(te, m, polygon=True, positions=True)


def _request(rng, g, positions, npaths, batched):
    """A mixed request whose paths visit the maps at `positions` in no order, each around its own map's position."""
    R = batch_request(rng, g, npaths, len(positions), offsets=np.asarray(positions) - (g.position_x, g.position_y), permute=False,
                      circular=0.6, cap_path=False)
    R["batched"] = batched
    return R


def _ask(m, te, R):
    return ask(m, te.FootprintParams.yaml_defaults(), R, R["map"] if R["batched"] else None)


def _same_answers(a, b, what=""):
    for k, (x, y) in enumerate(zip(a, b)):
        assert same_bytes(x, y), (what, k)


# ---- 1. a single map: the node's update ----------------------------------------------------------------------------------------

SUBMAP_CASES = [
    ("interior", (3.1, -1.7), (4.0, 4.0)),
    ("interior-odd", (-10.37, 12.64), (3.0, 5.55)),
    ("clipped-top-left", (SRC_POS[0] + 0.5 * SRC_ROWS * RES - 0.4, SRC_POS[1] + 0.5 * SRC_COLS * RES - 1.1), (4.0, 4.0)),
    ("clipped-bottom-right", (SRC_POS[0] - 0.5 * SRC_ROWS * RES + 0.7, SRC_POS[1] - 0.5 * SRC_COLS * RES + 0.03), (4.0, 6.0)),
]


@pytest.mark.parametrize("names", [FUSED, RAW], ids=["fused", "raw"])
@pytest.mark.parametrize("memory", [0, 1], ids=["host", "device"])
def test_chain_submap_equals_cut_chain_carry(te, ctx, source, names, memory):
    torch = pytest.importorskip("torch") if memory == 1 else None
    lay = _layers(source, names, memory, torch)
    rng = np.random.default_rng(11)
    m = ctx.map()
    for what, pos, length in SUBMAP_CASES:
        info = m.chain_submap(source["g"], lay, pos, length, source["p"], memory=memory)
        ref = so.submap_geometry(source["og"], [pos], [length])
        assert info.success == 1 and ref["success"][0] == 1, what
        for f in so.FIELDS[1:]:
            assert getattr(info, f) == ref[f][0], (what, f)
        if what == "clipped-top-left":   # getSubmap bounds the corner that leaves the map to its edge
            assert (info.top_row, info.top_col) == (0, 0)
        if what == "clipped-bottom-right":
            assert (info.top_row + info.rows, info.top_col + info.cols) == (SRC_ROWS, SRC_COLS)
        gs = te.Geometry(info.rows, info.cols, RES, info.length_x, info.length_y, info.position_x, info.position_y, 0, 0)
        top = (info.top_row, info.top_col)
        r = ctx.map()
        r.chain(gs, source["p"], _cut(source, "elevation", top, info.rows, info.cols))
        r.carry_layers(names[1:], [_cut(source, n, top, info.rows, info.cols) for n in names[1:]])
        assert_same_held(_held(te, m), _held(te, r), what)
        R = _request(rng, gs, np.array([[gs.position_x, gs.position_y]]), 40, False)
        _same_answers(_ask(m, te, R), _ask(r, te, R), what)
        assert_same_held(_held(te, m), _held(te, r), (what, "after the request"))
    # a failing getSubmap: info says so, the call refuses and the map is as it was
    before = _held(te, m)
    info = m.chain_submap(source["g"], lay, (500.0, 0.0), (4.0, 4.0), source["p"], memory=memory)
    assert info.success == 0 and info.rows == 0
    assert_same_held(_held(te, m), before, "failed getSubmap")


# ---- 2. a batch: a fleet cut out of one map --------------------------------------------------------------------------------------

NB, NB_ROWS, NB_COLS = 64, 256, 192


def _fleet_positions(rng):
    """NB positions: interior, across each of the four edges and each corner, and fully outside."""
    hx, hy = 0.5 * SRC_ROWS * RES, 0.5 * SRC_COLS * RES
    wx, wy = 0.5 * NB_ROWS * RES, 0.5 * NB_COLS * RES
    cx, cy = SRC_POS
    pos = []
    for _ in range(24):
        pos.append((cx + rng.uniform(-hx + wx + 1, hx - wx - 1), cy + rng.uniform(-hy + wy + 1, hy - wy - 1)))
    for sx in (-1, 0, 1):
        for sy in (-1, 0, 1):
            if sx == sy == 0:
                continue
            for _ in range(4):   # straddling the edge / corner by a random part of the window
                pos.append((cx + sx * (hx + rng.uniform(-wx, wx)) + (0 if sx else rng.uniform(-hx / 2, hx / 2)),
                            cy + sy * (hy + rng.uniform(-wy, wy)) + (0 if sy else rng.uniform(-hy / 2, hy / 2))))
    while len(pos) < NB:
        pos.append((cx + rng.choice([-1, 1]) * (hx + wx + rng.uniform(0.1, 50)), cy + rng.uniform(-3 * hy, 3 * hy)))
    return np.asarray(pos[:NB], np.float64)


def _oracle_windows(source, positions, rows, cols, names, length=None):
    top, at = wo.window_geometry(source["og"], rows, cols, positions, length=length)
    cuts = {n: np.stack([_cut(source, n, t, rows, cols) for t in top]) for n in names}
    return top, at, cuts


@pytest.fixture(params=["fused", "generic"])
def kernel(request, ctx, te):
    ctx.set_kernel(te.KERNEL_FUSED if request.param == "fused" else te.KERNEL_GENERIC)
    yield request.param
    ctx.set_kernel(te.KERNEL_AUTO)


@pytest.mark.parametrize("memory", [0, 1], ids=["host", "device"])
def test_chain_windows_batch(te, ctx, source, kernel, memory):
    torch = pytest.importorskip("torch") if memory == 1 else None
    rng = np.random.default_rng(23)
    pos = _fleet_positions(rng)
    g = te.Geometry.make(NB_ROWS, NB_COLS, RES)
    top, at, cuts = _oracle_windows(source, pos, NB_ROWS, NB_COLS, FUSED)
    inside = [(0 <= t[0] and t[0] + NB_ROWS <= SRC_ROWS and 0 <= t[1] and t[1] + NB_COLS <= SRC_COLS) for t in top]
    outside = [(t[0] >= SRC_ROWS or t[0] + NB_ROWS <= 0 or t[1] >= SRC_COLS or t[1] + NB_COLS <= 0) for t in top]
    assert sum(inside) >= 20 and sum(outside) >= 4 and NB - sum(inside) - sum(outside) >= 30
    m = ctx.map()
    m.chain_windows(g, source["g"], _layers(source, FUSED, memory, torch), pos, source["p"], memory=memory)
    r = ctx.map()
    r.chain_batched(g, source["p"], NB, cuts["elevation"], positions=at)
    r.carry_layers(FUSED[1:], [cuts[n] for n in FUSED[1:]])
    assert np.array_equal(m.positions(), at)
    assert_same_held(_held(te, m), _held(te, r), kernel)
    ft = te.FootprintParams.yaml_defaults()
    assert_same_bits(m.footprint(ft), r.footprint(ft), (kernel, "sweep"))
    R = _request(rng, g, at, 200, True)
    _same_answers(_ask(m, te, R), _ask(r, te, R), kernel)
    assert_same_held(_held(te, m), _held(te, r), (kernel, "after the request"))


def test_windows_agree_with_getsubmap(te, ctx, source):
    """Interior windows whose getSubmap (at g's length) has the batch's size: same top-left, position and cells."""
    rng = np.random.default_rng(5)
    n, mcols = 120, 90
    lx, ly = (n - 0.5) * RES, (mcols - 0.5) * RES   # getSubmap's size is n or n + 1 with the position's fraction of a cell
    g = te.Geometry(n, mcols, RES, lx, ly, 0.0, 0.0, 0, 0)
    hx, hy = 0.5 * SRC_ROWS * RES - lx, 0.5 * SRC_COLS * RES - ly
    pos = np.stack([SRC_POS[0] + rng.uniform(-hx, hx, 48), SRC_POS[1] + rng.uniform(-hy, hy, 48)], axis=1)
    top, at = wo.window_geometry(source["og"], n, mcols, pos, length=(lx, ly))
    ref = so.submap_geometry(source["og"], pos, np.tile([lx, ly], (len(pos), 1)))
    lib = te.capi.submap_geometry(source["g"], pos, np.tile([lx, ly], (len(pos), 1)))
    m = ctx.map()
    m.chain_windows(g, source["g"], _layers(source, ("elevation",), 0), pos, source["p"])
    got_pos = m.positions()
    elev = m.get_layers(["elevation"])["elevation"]
    matched = 0
    for k in range(len(pos)):
        assert ref["success"][k] == 1
        if (ref["rows"][k], ref["cols"][k]) != (n, mcols):
            continue
        matched += 1
        assert (lib["rows"][k], lib["cols"][k]) == (n, mcols)
        assert top[k].tolist() == [ref["top_row"][k], ref["top_col"][k]] == [lib["top_row"][k], lib["top_col"][k]], k
        assert at[k].tolist() == [ref["position_x"][k], ref["position_y"][k]] == got_pos[k].tolist(), k
        block = source["lay"]["elevation"][top[k][0]:top[k][0] + n, top[k][1]:top[k][1] + mcols]
        assert_same_bits(elev[k], block, k)
    assert matched >= 8, matched


# ---- 3. a selection --------------------------------------------------------------------------------------------------------------

NS = 16


def test_chain_windows_selection(te, ctx, source):
    rng = np.random.default_rng(41)
    g = te.Geometry.make(NB_ROWS, NB_COLS, RES)
    pos = _fleet_positions(rng)[rng.permutation(NB)[:NS]]
    held = ("elevation", "upper_bound", "lower_bound")
    top, at, cuts = _oracle_windows(source, pos, NB_ROWS, NB_COLS, held)
    m, r = ctx.map(), ctx.map()
    m.chain_windows(g, source["g"], _layers(source, held, 0), pos, source["p"])
    r.chain_batched(g, source["p"], NS, cuts["elevation"], positions=at)
    r.carry_layers(held[1:], [cuts[n] for n in held[1:]])
    ft = te.FootprintParams.yaml_defaults()
    assert_same_bits(m.footprint(ft), r.footprint(ft))   # fills the caches, which the unselected maps must keep
    R0 = _request(rng, g, at, 60, True)
    _same_answers(_ask(m, te, R0), _ask(r, te, R0))   # and the memo
    for rnd, given in enumerate([("elevation", "upper_bound", "lower_bound"), ("elevation", "lower_bound"), ("elevation",)]):
        idx = rng.permutation(NS)[:5 + rnd].astype(np.int32)
        new = _fleet_positions(rng)[rng.permutation(NB)[:len(idx)]]
        st, sat, sc = _oracle_windows(source, new, NB_ROWS, NB_COLS, given)
        m.chain_windows(g, source["g"], _layers(source, given, 0), new, source["p"], map_index=idx)
        r.chain_maps(g, source["p"], idx, sc["elevation"], positions=sat)
        if len(given) > 1:
            r.carry_layers(given[1:], [sc[n] for n in given[1:]], map_index=idx)
        hm, hr = _held(te, m), _held(te, r)
        assert_same_held(hm, hr, rnd)
        for n in set(held) - set(given):   # held but not given: NaN on the selected maps
            assert np.isnan(hm[n][idx]).all(), (rnd, n)
        R = _request(rng, g, hr["positions"], 60, True)
        _same_answers(_ask(m, te, R), _ask(r, te, R), rnd)
        assert_same_held(_held(te, m), _held(te, r), (rnd, "after the request"))
    # a carried layer the batch does not hold
    before = _held(te, m)
    with pytest.raises(te.TEError) as e:
        m.chain_windows(g, source["g"], _layers(source, ("elevation", "variance"), 0), pos[:2], source["p"], map_index=[0, 1])
    assert e.value.code == BAD_ARG
    assert_same_held(_held(te, m), before, "not held")


# ---- 4. launches -----------------------------------------------------------------------------------------------------------------

def _launches(ctx, fn):
    a = ctx.stats()[0]
    fn()
    return ctx.stats()[0] - a


@pytest.mark.parametrize("names", [("elevation",), FUSED, RAW], ids=["elevation", "fused", "raw"])
def test_one_launch_more(te, ctx, source, names):
    rng = np.random.default_rng(3)
    g = te.Geometry.make(NB_ROWS, NB_COLS, RES)
    pos = _fleet_positions(rng)[:NS]
    _, at, cuts = _oracle_windows(source, pos, NB_ROWS, NB_COLS, ("elevation",))
    lay = _layers(source, names, 0)
    p = source["p"]
    m, r = ctx.map(), ctx.map()
    for n in (1, NS):   # one map, all maps
        a = _launches(ctx, lambda: m.chain_windows(g, source["g"], lay, pos[:n], p))
        b = _launches(ctx, lambda: r.chain_batched(g, p, n, cuts["elevation"][:n], positions=at[:n]))
        assert a == b + 1, (n, a, b)
    if len(names) > 1:   # the batch holds the same carried layers as m's, so both selections fill the same layers
        r.carry_layers(names[1:], [np.zeros((NS, NB_ROWS, NB_COLS), np.float32)] * (len(names) - 1))
    idx = np.array([9, 2, 14, 5], np.int32)
    a = _launches(ctx, lambda: m.chain_windows(g, source["g"], lay, pos[:4], p, map_index=idx))
    b = _launches(ctx, lambda: r.chain_maps(g, p, idx, cuts["elevation"][:4], positions=at[:4]))
    assert a == b + 1, ("selection", a, b)
    a = _launches(ctx, lambda: m.chain_submap(source["g"], lay, (3.0, 1.0), (4.0, 4.0), p))
    info = te.capi.submap_geometry(source["g"], [(3.0, 1.0)], [(4.0, 4.0)])[0]
    gs = te.Geometry(int(info["rows"]), int(info["cols"]), RES, info["length_x"], info["length_y"], info["position_x"],
                     info["position_y"], 0, 0)
    b = _launches(ctx, lambda: r.chain(gs, p, np.zeros((gs.rows, gs.cols), np.float32)))
    assert a == b + 1, ("submap", a, b)


# ---- 5. errors ---------------------------------------------------------------------------------------------------------------------

def test_error_table(te, ctx, source):
    L = te.load_library()
    g = te.Geometry.make(NB_ROWS, NB_COLS, RES)
    pos = _fleet_positions(np.random.default_rng(2))[:NS]
    m = ctx.map()
    m.chain_windows(g, source["g"], _layers(source, FUSED, 0), pos, source["p"])
    st = source["stored"]
    ptrs = lambda *a: (C.c_void_p * len(a))(*(x if x is None else x.ctypes.data for x in a))  # noqa: E731
    good = ptrs(st["elevation"], st["upper_bound"], st["lower_bound"])
    mask = te.capi.layer_mask(FUSED)
    p = source["p"]

    def geo(**kw):
        s = te.Geometry.from_buffer_copy(source["g"])
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    xy = np.ascontiguousarray(pos[:2])
    idx = np.array([3, 7], np.int32)

    def win(gg=g, src=source["g"], mk=mask, lay=good, n=2, index=None, at=xy, memory=0):
        return L.te_map_chain_windows(m._h, C.byref(gg), C.byref(src), mk, lay, n, None if index is None else index.ctypes.data,
                                      None if at is None else at.ctypes.data, C.byref(p), memory)

    def sub(src=source["g"], mk=mask, lay=good, x=3.0, y=1.0, lx=4.0, ly=4.0, memory=0):
        info = te.capi.SubmapInfo()
        return L.te_map_chain_submap(m._h, C.byref(src), mk, lay, x, y, lx, ly, C.byref(p), C.byref(info), memory)

    nan, inf = float("nan"), float("inf")
    cases = [
        ("src rows", lambda: win(src=geo(rows=0)), BAD_ARG),
        ("src start index", lambda: win(src=geo(start_row=SRC_ROWS)), BAD_ARG),
        ("mask without elevation", lambda: win(mk=te.capi.layer_mask(["upper_bound"])), BAD_ARG),
        ("mask robot_slope", lambda: win(mk=mask | te.capi.layer_mask(["robot_slope"])), BAD_ARG),
        ("mask bit 7", lambda: win(mk=mask | 0x80), BAD_ARG),
        ("null layers", lambda: win(lay=None), BAD_ARG),
        ("null named layer", lambda: win(lay=ptrs(st["elevation"], None, st["lower_bound"])), MISSING_LAYER),
        ("memory", lambda: win(memory=7), BAD_ARG),
        ("resolution", lambda: win(gg=te.Geometry.make(NB_ROWS, NB_COLS, RES * (1 + 1e-15))), BAD_ARG),
        ("no positions", lambda: win(at=None), BAD_ARG),
        ("position nan", lambda: win(at=np.array([[0.0, 0.0], [nan, 0.0]])), BAD_ARG),
        ("position inf", lambda: win(at=np.array([[inf, 0.0], [0.0, 0.0]])), BAD_ARG),
        ("index past int32", lambda: win(at=np.array([[0.0, 0.0], [0.0, -2e8]])), BAD_ARG),
        ("nmaps", lambda: win(n=0), BAD_ARG),
        ("selection twice", lambda: win(index=np.array([3, 3], np.int32)), BAD_ARG),
        ("selection outside", lambda: win(index=np.array([3, NS], np.int32)), BAD_ARG),
        ("selection geometry", lambda: win(gg=te.Geometry.make(NB_ROWS + 1, NB_COLS, RES), index=idx), BAD_ARG),
        ("selection not held", lambda: win(mk=mask | te.capi.layer_mask(["time"]), lay=ptrs(st["elevation"], st["upper_bound"],
                                                                                          st["lower_bound"], st["time"]),
                                           index=idx), BAD_ARG),
        ("submap src", lambda: sub(src=geo(cols=-1)), BAD_ARG),
        ("submap null layer", lambda: sub(lay=ptrs(None, st["upper_bound"], st["lower_bound"])), MISSING_LAYER),
        ("submap mask", lambda: sub(mk=0), BAD_ARG),
        ("submap position", lambda: sub(x=nan), BAD_ARG),
        ("submap negative length", lambda: sub(ly=-1.0), BAD_ARG),
        ("submap length inf", lambda: sub(lx=inf), BAD_ARG),
        ("submap memory", lambda: sub(memory=-1), BAD_ARG),
        ("submap fails", lambda: sub(x=-900.0), BAD_ARG),
    ]
    before = _held(te, m)
    for what, call, code in cases:
        assert call() == code, (what, L.te_last_error())
        assert_same_held(_held(te, m), before, what)
    # the robot_slope refusal of the _maps entries
    m.carry_layers(["robot_slope"], [np.zeros((NS, NB_ROWS, NB_COLS), np.float32)])
    before = _held(te, m)
    assert win(index=idx) == UNSUPPORTED, L.te_last_error()
    assert_same_held(_held(te, m), before, "robot_slope")
