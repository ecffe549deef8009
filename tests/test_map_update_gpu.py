"""Updates of some maps of a batched te_map (te_map_chain_maps, te_map_set_layers_maps, te_map_footprint_maps).  A batch B of n
maps must behave as n single-map te_maps S_0..S_{n-1} under any interleaving of per-map updates, sweeps and requests: after every
step, B's answers, untraversable polygons, caches and layers equal, bit for bit, what the S_k return and hold, and a map outside
the selection keeps every bit of its layers, cache and memo."""
import ctypes as C

import numpy as np
import pytest

import paths_oracle as po
import synth
from helpers import batch_request, bits, chain_layers, mixed_request, request_footprints, same
from map_helpers import assert_batch_matches_singles, assert_same_held, close_maps, held  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, NMAPS = 200, 180, 0.02, 5
BAD_ARG, MISSING_LAYER, UNSUPPORTED = -1, -2, -4
FILTER = ("traversability", "slope", "step", "elevation")
NAMES = {"traversability": "traversability", "traversability_slope": "slope", "traversability_step": "step",
         "traversability_roughness": "roughness", "elevation": "elevation", "robot_slope": "robot_slope"}


@pytest.fixture(scope="module")
def maps(te, oracle):
    """Two terrains per map (old, new), each with the oracle chain's layers, roughness with zero patches and robot_slope."""
    og, g = oracle.Geometry.make(ROWS, COLS, RES), te.Geometry.make(ROWS, COLS, RES)
    old, new = [], []
    for k in range(NMAPS):
        for seed, dst in ((81 + k, old), (181 + k, new)):
            z = synth.terrain(ROWS, COLS, RES, seed, "mixed")
            L, rs = chain_layers(oracle, og, z, seed)
            dst.append(dict(L, robot_slope=rs))
    return og, g, old, new


def _stack(per, key, idx=None):
    return np.stack([per[k][key] for k in (range(len(per)) if idx is None else idx)])


def _same_state(te, b, singles, what):
    """B's layers and caches equal the single maps', map by map, bit for bit."""
    hb = {n: v[None] if b.nmaps == 1 else v for n, v in held(te, b).items()}
    for k, s in enumerate(singles):
        assert_same_held({n: v[k] for n, v in hb.items()}, held(te, s), (what, k))


def _request(rng, og, fps, npaths):
    """A mixed request whose paths visit every map in no order."""
    return batch_request(rng, og, npaths, NMAPS, fps, circular=0.6, cap_path=False)


def _load_chain(ctx, te, g, elev):
    """B from te_map_chain_batched and one te_map_chain per map."""
    p = te.ChainParams.yaml_defaults(0)
    b = ctx.map()
    b.chain_batched(g, p, len(elev), elev)
    singles = []
    for e in elev:
        s = ctx.map()
        s.chain(g, p, e)
        singles.append(s)
    return b, singles


def _load_set(ctx, g, per, slope=True):
    """B from te_map_set_layers_batched (roughness, and robot_slope when `slope`) and one te_map_set_layers per map."""
    rs = (lambda p: p["robot_slope"]) if slope else (lambda p: None)
    b = ctx.map()
    b.set_layers_batched(g, len(per), *(_stack(per, k) for k in FILTER), roughness=_stack(per, "roughness"),
                         robot_slope=_stack(per, "robot_slope") if slope else None)
    singles = []
    for p in per:
        s = ctx.map()
        s.set_layers(g, *(p[k] for k in FILTER), roughness=p["roughness"], robot_slope=rs(p))
        singles.append(s)
    return b, singles


def _chain_maps_device(te, b, g, p, idx, elev, outputs):
    """te_map_chain_maps in device memory: elevation and outputs torch tensors, map_index a host array."""
    torch = pytest.importorskip("torch")
    idx = np.ascontiguousarray(idx, dtype=np.int32)
    e = torch.from_numpy(np.ascontiguousarray(elev.transpose(0, 2, 1))).cuda()
    outs = {k: torch.empty_like(e) for k in ("slope", "step", "roughness", "traversability")} if outputs else {}
    torch.cuda.synchronize()
    rc = te.load_library().te_map_chain_maps(b._h, C.byref(g), C.byref(p), len(idx), idx.ctypes.data, e.data_ptr(),
                                             *(outs[k].data_ptr() if outputs else None for k in ("slope", "step", "roughness",
                                                                                              "traversability")), te.MEM_DEVICE)
    assert rc == 0, te.load_library().te_last_error()
    b._ctx.synchronize()
    return {k: v.cpu().numpy().transpose(0, 2, 1) for k, v in outs.items()} if outputs else None


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("outputs", [False, True])
def test_chain_maps_parity(te, ctx, oracle, maps, memory, outputs):
    og, g, old, new = maps
    p = te.ChainParams.yaml_defaults(0)
    ft = te.FootprintParams.yaml_defaults()
    b, singles = _load_chain(ctx, te, g, _stack(old, "elevation"))
    rng = np.random.default_rng(7)
    fps = request_footprints(rng)
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 60))   # caches and memos of every map in use
    before = held(te, b)
    sel = [3, 1]
    e = _stack(new, "elevation", sel)
    if memory == "host":
        got = b.chain_maps(g, p, sel, e, outputs=outputs)
    else:
        got = _chain_maps_device(te, b, g, p, sel, e, outputs)
    for k in sel:
        singles[k].chain(g, p, new[k]["elevation"])
    # the selected maps hold what te_chain_batched gives for E, and what te_map_chain gives each
    want = {k: np.empty((len(sel), COLS, ROWS), np.float32) for k in ("slope", "step", "roughness", "traversability")}
    ctx.chain_batched(g, p, len(sel), np.ascontiguousarray(e.transpose(0, 2, 1)), want["slope"], want["step"], want["roughness"],
                      want["traversability"], te.MEM_HOST)
    after = held(te, b)
    for j, k in enumerate(sel):
        for name, key in NAMES.items():
            if key in want:
                assert np.array_equal(bits(after[name][k]), bits(want[key][j].T)), (k, name)
                if outputs:
                    assert np.array_equal(bits(got[key][j]), bits(want[key][j].T)), (k, key)
        assert np.array_equal(bits(after["elevation"][k]), bits(e[j]))
        assert np.isnan(after["cache"][k]).all()
    assert got is None or set(got) == set(want)
    for k in set(range(NMAPS)) - set(sel):   # the other maps keep every bit
        for name in before:
            assert np.array_equal(bits(after[name][k]), bits(before[name][k])), (k, name)
    _same_state(te, b, singles, "after chain_maps")
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 60))   # the kept memos and caches answer as the single maps do


@pytest.mark.parametrize("kind", ["chain", "slope"])
def test_interleaved_updates_equal_single_maps(te, ctx, oracle, maps, kind):
    """request, update maps [3, 1] with new terrain, request, footprint_maps([0, 3]), request, set_layers_maps([2]), request:
    after every step the batch equals five single-map te_maps.  "chain": a batch from te_map_chain_batched, maps 3 and 1
    re-chained, replayed on the CPU oracle too; "slope": a batch with roughness and robot_slope, maps 3 and 1 reloaded."""
    og, g, old, new = maps
    p = te.ChainParams.yaml_defaults(0)
    ft, fo = te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults()
    slope = kind == "slope"
    if slope:
        b, singles = _load_set(ctx, g, old)
    else:
        b, singles = _load_chain(ctx, te, g, _stack(old, "elevation"))
    state = None
    if not slope:   # the oracle replays the requests on the layers the single maps hold
        OL = [{NAMES[n]: v for n, v in s.get_layers(["traversability", "traversability_slope", "traversability_step",
                                                      "traversability_roughness", "elevation"]).items()} for s in singles]
        state = (og, fo, OL, [po.empty_cache(og) for _ in singles])
    rng = np.random.default_rng(17 + slope)
    fps = request_footprints(rng)
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 70), state)

    sel = [3, 1]
    if slope:
        b.set_layers_maps(g, sel, *(_stack(new, k, sel) for k in FILTER), roughness=_stack(new, "roughness", sel),
                          robot_slope=_stack(new, "robot_slope", sel))
        for k in sel:
            singles[k].set_layers(g, *(new[k][x] for x in FILTER), roughness=new[k]["roughness"], robot_slope=new[k]["robot_slope"])
    else:
        b.chain_maps(g, p, sel, _stack(new, "elevation", sel))
        for k in sel:
            singles[k].chain(g, p, new[k]["elevation"])
            state[2][k] = {NAMES[n]: v for n, v in singles[k].get_layers(list(NAMES)[:5]).items()}
            state[3][k] = po.empty_cache(og)
    _same_state(te, b, singles, "after the update")
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 70), state)

    fsel = [0, 3]
    swept = b.footprint_maps(ft, fsel)
    for j, k in enumerate(fsel):
        assert np.array_equal(bits(swept[j]), bits(singles[k].footprint(ft))), ("footprint_maps", k)
        if state is not None:   # the oracle continues from the swept cache (the sweep's last bits are pinned in test_map_gpu)
            state[3][k] = np.asfortranarray(swept[j].copy())
    _same_state(te, b, singles, "after footprint_maps")
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 70), state)

    lay = {x: new[4][x] for x in FILTER + ("roughness", "robot_slope")}   # map 2 takes map 4's new terrain
    b.set_layers_maps(g, [2], *(lay[x][None] for x in FILTER), roughness=lay["roughness"][None],
                      robot_slope=lay["robot_slope"][None] if slope else None)
    singles[2].set_layers(g, *(lay[x] for x in FILTER), roughness=lay["roughness"], robot_slope=lay["robot_slope"] if slope else None)
    if state is not None:
        state[2][2] = {x: lay[x] for x in FILTER + ("roughness",)}
        state[3][2] = po.empty_cache(og)
    _same_state(te, b, singles, "after set_layers_maps")
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 70), state)
    # the read side too: submaps and valid_at of every map
    pos, ln = rng.uniform([-1.5, -1.5], [1.5, 1.5], (NMAPS, 2)), np.full((NMAPS, 2), 0.8)
    got = b.get_submaps_batched(np.arange(NMAPS, dtype=np.int32), pos, ln, ["traversability", "elevation"])
    for k, s in enumerate(singles):
        want = s.get_submaps(pos[k:k + 1], ln[k:k + 1], ["traversability", "elevation"])[0]
        for n in ("traversability", "elevation"):
            assert np.array_equal(bits(got[k][1][n]), bits(want[1][n])), (k, n)
    xy = rng.uniform([-2.4, -2.2], [2.4, 2.2], (300, 2))
    pm = rng.integers(0, NMAPS, 300).astype(np.int32)
    want = np.zeros(300, np.uint8)
    for k, s in enumerate(singles):
        idx = np.nonzero(pm == k)[0]
        want[idx] = s.valid_at(xy[idx])
    assert np.array_equal(b.valid_at_batched(pm, xy), want)


def test_stale_memo_would_show(te, ctx, oracle, maps):
    """Map 1's memo classifies cells of its old terrain.  Its new layers keep traversability and elevation but take slope, step
    and roughness (with other zero patches) from another terrain, so only isTraversableForFilters can change the answers: they
    must be the new layers', as the single map gives, and must differ from the old ones.  Map 0, not selected, keeps its cache."""
    og, g, old, new = maps
    ft = te.FootprintParams.yaml_defaults()
    ft.verify_roughness = 1
    per = old[:2]
    b, singles = _load_set(ctx, g, per, slope=False)
    rng = np.random.default_rng(23)
    R = mixed_request(rng, og, 120, [], circular=1.0, cap_path=False)
    R["map"], R["fps"] = np.tile(np.array([0, 1], np.int32), 60), []
    first = assert_batch_matches_singles(b, singles, ft, R)
    kept = b.get_footprint()[0]
    blocked = {x: (new if x in ("slope", "step", "roughness") else per)[1][x] for x in FILTER + ("roughness",)}
    b.set_layers_maps(g, [1], *(blocked[x][None] for x in FILTER), roughness=blocked["roughness"][None])
    singles[1].set_layers(g, *(blocked[x] for x in FILTER), roughness=blocked["roughness"])
    assert np.array_equal(bits(b.get_footprint()[0]), bits(kept)) and np.isnan(b.get_footprint()[1]).all()
    again = assert_batch_matches_singles(b, singles, ft, R)
    on1 = R["map"] == 1
    assert (again[0][on1] != first[0][on1]).any() or not same(again[1][on1], first[1][on1])


def test_whole_selection_and_one_map(te, ctx, oracle, maps):
    og, g, old, new = maps
    p = te.ChainParams.yaml_defaults(0)
    b, _ = _load_chain(ctx, te, g, _stack(old, "elevation"))
    perm = np.array([2, 4, 0, 3, 1], np.int32)
    out = b.chain_maps(g, p, perm, _stack(new, "elevation", perm), outputs=True)
    ref = ctx.map()
    ref.chain_batched(g, p, NMAPS, _stack(new, "elevation"))
    hb, hr = held(te, b), held(te, ref)
    for name in hr:
        assert np.array_equal(bits(hb[name]), bits(hr[name])), name
    for name, key in NAMES.items():
        if key in out:
            assert np.array_equal(bits(out[key]), bits(hr[name][perm])), key
    one, single = ctx.map(), ctx.map()
    one.chain(g, p, old[0]["elevation"])
    one.chain_maps(g, p, [0], new[0]["elevation"][None])
    single.chain(g, p, new[0]["elevation"])
    _same_state(te, one, [single], "one map")
    ft = te.FootprintParams.yaml_defaults()
    assert np.array_equal(bits(one.footprint_maps(ft, [0])[0]), bits(single.footprint(ft)))


def test_device_memory_entries(te, ctx, oracle, maps):
    """te_map_set_layers_maps and te_map_footprint_maps in device memory: a layer at an address that is not 16-byte aligned (the
    slot kernel's 4-byte accesses), and the sweep's output written map by map in map_index order."""
    torch = pytest.importorskip("torch")
    og, g, old, new = maps
    ft = te.FootprintParams.yaml_defaults()
    ft.verify_roughness = 1
    L = te.load_library()
    b, singles = _load_set(ctx, g, old)
    rng = np.random.default_rng(29)
    fps = request_footprints(rng)
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 40))
    sel = np.array([4, 0], np.int32)
    keys = ("traversability", "slope", "step", "roughness", "elevation", "robot_slope")
    dev = {k: torch.from_numpy(np.ascontiguousarray(_stack(new, k, sel).transpose(0, 2, 1))).cuda() for k in keys}
    shifted = torch.empty(dev["step"].numel() + 1, dtype=torch.float32, device="cuda")
    shifted[1:] = dev["step"].reshape(-1)   # 4 bytes past a 16-byte boundary
    ptr = {k: v.data_ptr() for k, v in dev.items()}
    ptr["step"] = shifted.data_ptr() + 4
    torch.cuda.synchronize()
    assert L.te_map_set_layers_maps(b._h, C.byref(g), len(sel), sel.ctypes.data, *(ptr[k] for k in keys), te.MEM_DEVICE) == 0
    for k in sel:
        singles[k].set_layers(g, *(new[k][x] for x in FILTER), roughness=new[k]["roughness"], robot_slope=new[k]["robot_slope"])
    ctx.synchronize()
    _same_state(te, b, singles, "set_layers_maps in device memory")
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 40))
    fsel = np.array([1, 4, 2], np.int32)
    out = torch.full((len(fsel), COLS, ROWS), 7.0, dtype=torch.float32, device="cuda")
    assert L.te_map_footprint_maps(b._h, C.byref(ft), len(fsel), fsel.ctypes.data, out.data_ptr(), te.MEM_DEVICE) == 0
    ctx.synchronize()
    got = out.cpu().numpy()
    for j, k in enumerate(fsel):
        assert np.array_equal(bits(got[j].T), bits(singles[k].footprint(ft))), k
    _same_state(te, b, singles, "footprint_maps in device memory")


def test_page_locked_map_index_reused_at_once(te, ctx, oracle, maps):
    """A device-memory call returns while the stream is still busy; a caller that refills its page-locked map_index right away
    must not redirect the update to other maps."""
    torch = pytest.importorskip("torch")
    og, g, old, new = maps
    p, ft = te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    L = te.load_library()
    b = ctx.map()
    b.chain_batched(g, p, NMAPS, _stack(old, "elevation"))
    before = held(te, b)
    idx = torch.empty(2, dtype=torch.int32, pin_memory=True).numpy()
    idx[:] = [3, 1]
    e = torch.from_numpy(np.ascontiguousarray(_stack(new, "elevation", [3, 1]).transpose(0, 2, 1))).cuda()
    torch.cuda.synchronize()
    for _ in range(4):   # keep the context stream busy, so a copy queued behind this work would read idx late
        assert L.te_map_footprint(b._h, C.byref(ft), None, te.MEM_DEVICE) == 0
    assert L.te_map_chain_maps(b._h, C.byref(g), C.byref(p), 2, idx.ctypes.data, e.data_ptr(), None, None, None, None,
                               te.MEM_DEVICE) == 0
    idx[:] = [0, 2]   # the next update's maps
    ctx.synchronize()
    after = held(te, b)
    for k in (0, 2, 4):
        for name in before:
            if name != "cache":   # the sweeps above filled every cache
                assert np.array_equal(bits(after[name][k]), bits(before[name][k])), (k, name)
        assert np.isfinite(after["cache"][k]).any(), k
    for k in (3, 1):
        assert np.array_equal(bits(after["elevation"][k]), bits(new[k]["elevation"])), k
        assert np.isnan(after["cache"][k]).all(), k


def test_odd_cell_count(te, ctx):
    """rows * cols not a multiple of 4: the slot kernel takes its 4-byte accesses.  Chain, reload and sweep of some maps equal the
    single maps'."""
    rows, cols = 61, 47
    g, p, ft = te.Geometry.make(rows, cols, RES), te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    z = [synth.terrain(rows, cols, RES, 300 + k, "mixed") for k in range(6)]
    b, singles = _load_chain(ctx, te, g, np.stack(z[:3]))
    b.chain_maps(g, p, [2, 0], np.stack([z[3], z[4]]))
    singles[2].chain(g, p, z[3])
    singles[0].chain(g, p, z[4])
    lay = singles[2].get_layers(["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"])
    b.set_layers_maps(g, [1], *(lay[n][None] for n in ("traversability", "traversability_slope", "traversability_step", "elevation")),
                      roughness=lay["traversability_roughness"][None])
    singles[1].set_layers(g, *(lay[n] for n in ("traversability", "traversability_slope", "traversability_step", "elevation")),
                          roughness=lay["traversability_roughness"])
    swept = b.footprint_maps(ft, [1, 2])
    for j, k in enumerate([1, 2]):
        assert np.array_equal(bits(swept[j]), bits(singles[k].footprint(ft))), k
    _same_state(te, b, singles, "odd cell count")


def test_launch_count_independent_of_nsel(te, ctx, oracle, maps):
    og, g, old, new = maps
    p, ft = te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    b, _ = _load_set(ctx, g, old, slope=False)
    b.chain_maps(g, p, [0], new[0]["elevation"][None])   # warm-up: scratch, geometry tables
    deltas = []
    for sel in ([4], [4, 0, 2, 1, 3]):
        row = []
        for call in (lambda: b.chain_maps(g, p, sel, _stack(new, "elevation", sel)),
                     lambda: b.set_layers_maps(g, sel, *(_stack(new, x, sel) for x in FILTER), roughness=_stack(new, "roughness", sel)),
                     lambda: b.footprint_maps(ft, sel)):
            n0 = ctx.stats()[0]
            call()
            row.append(ctx.stats()[0] - n0)
        deltas.append(row)
    assert deltas[0] == deltas[1], deltas
    assert deltas[0][1] == 1   # set_layers_maps: the one k_map_slots launch


def test_error_codes_leave_the_map_unchanged(te, ctx, oracle, maps):
    og, g, old, new = maps
    p, ft = te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    L = te.load_library()
    b, singles = _load_set(ctx, g, old, slope=False)
    rng = np.random.default_rng(3)
    fps = request_footprints(rng)
    assert_batch_matches_singles(b, singles, ft, _request(rng, og, fps, 20))   # caches and memos in use
    e1 = _stack(new, "elevation", [0])
    lay1 = {x: _stack(new, x, [0]) for x in FILTER + ("roughness", "robot_slope")}
    before = held(te, b)

    def expect(code, call):
        with pytest.raises(te.TEError) as e:
            call()
        assert e.value.code == code, (code, str(e.value))
        after = held(te, b)
        for name in before:
            assert np.array_equal(bits(after[name]), bits(before[name])), name

    for idx in ([1, 1], [-1], [NMAPS], [], [0, 1, 2, 3, 4, 0]):
        n = max(len(idx), 1)
        e = _stack(new, "elevation", [0] * n)
        expect(BAD_ARG, lambda: b.chain_maps(g, p, idx, e))
        expect(BAD_ARG, lambda: b.set_layers_maps(g, idx, *(_stack(new, x, [0] * n) for x in FILTER),
                                                  roughness=_stack(new, "roughness", [0] * n)))
        expect(BAD_ARG, lambda: b.footprint_maps(ft, idx))
    # a null map_index
    for rc in (L.te_map_chain_maps(b._h, C.byref(g), C.byref(p), 1, None, e1.ctypes.data, None, None, None, None, te.MEM_HOST),
               L.te_map_footprint_maps(b._h, C.byref(ft), 1, None, None, te.MEM_HOST)):
        assert rc == BAD_ARG
    assert np.array_equal(bits(held(te, b)["cache"]), bits(before["cache"]))
    # another geometry
    for gx in (te.Geometry.make(ROWS, COLS, RES, position=(0.5, 0.0)), te.Geometry.make(ROWS, COLS, 0.021)):
        expect(BAD_ARG, lambda: b.chain_maps(gx, p, [0], e1))
        expect(BAD_ARG, lambda: b.set_layers_maps(gx, [0], *(lay1[x] for x in FILTER), roughness=lay1["roughness"]))
    # the batch's optional layers: roughness missing, robot_slope extra, and chain_maps needs roughness and no robot_slope
    expect(MISSING_LAYER, lambda: b.set_layers_maps(g, [0], *(lay1[x] for x in FILTER)))
    expect(BAD_ARG, lambda: b.set_layers_maps(g, [0], *(lay1[x] for x in FILTER), roughness=lay1["roughness"],
                                              robot_slope=lay1["robot_slope"]))
    b = _load_set(ctx, g, old, slope=True)[0]
    before = held(te, b)
    expect(UNSUPPORTED, lambda: b.chain_maps(g, p, [0], e1))
    expect(MISSING_LAYER, lambda: b.set_layers_maps(g, [0], *(lay1[x] for x in FILTER), roughness=lay1["roughness"]))
    b = ctx.map()
    b.set_layers_batched(g, NMAPS, *(_stack(old, x) for x in FILTER))
    before = held(te, b)
    expect(UNSUPPORTED, lambda: b.chain_maps(g, p, [0], e1))
    # a te_map without layers
    empty = ctx.map()
    for call in (lambda: empty.chain_maps(g, p, [0], e1), lambda: empty.footprint_maps(ft, [0]),
                 lambda: empty.set_layers_maps(g, [0], *(lay1[x] for x in FILTER))):
        with pytest.raises(te.TEError) as e:
            call()
        assert e.value.code == BAD_ARG
    # a start index: in g, or on the te_map's layers
    gw = te.Geometry.make(ROWS, COLS, RES)
    gw.start_row, gw.start_col = 5, 7
    expect(UNSUPPORTED, lambda: b.chain_maps(gw, p, [0], e1))
    w = ctx.map()
    w.chain(gw, p, old[0]["elevation"])
    b, before = w, held(te, w)
    expect(UNSUPPORTED, lambda: w.chain_maps(gw, p, [0], e1))
    expect(UNSUPPORTED, lambda: w.footprint_maps(ft, [0]))
