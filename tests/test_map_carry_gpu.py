"""te_map_carry_layers and the layers it carries, on the GPU: the elevation map's upper_bound, lower_bound, variances and time,
and robot_slope, given to a te_map next to the chain's layers (mapOut = mapIn), read back bit for bit by te_map_get_layers and
te_map_get_submaps(_batched), uncertainty_range derived on the device, robot_slope gating the request exactly as when
te_map_set_layers gives it, the cache and the memo left alone, and the lifetime of the carried layers across map updates."""
import ctypes as C

import numpy as np
import pytest

import submap_oracle as so
import synth
from helpers import assert_same_answers, assert_same_bits, bits, mixed_request, noisy, request_footprints, unwrap
from map_helpers import ask, assert_same_held, check_submaps, close_maps, held, submap_windows  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, POS = 150, 130, 0.02, (0.37, -0.21)
BAD_ARG, MISSING_LAYER, UNSUPPORTED = -1, -2, -4
MAIN = ("traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation")
FILTER = ("traversability", "slope", "step", "elevation")
NOISE = (0.04, 0.02, 0.02, 0.02)   # fractions of NaN, +Inf, -Inf and zero cells of a noisy layer


def _geo(te, start=(0, 0), rows=ROWS, cols=COLS):
    g = te.Geometry.make(rows, cols, RES, POS)
    g.start_row, g.start_col = start
    return g


def _carried(te, seed, n=None):
    """The seven carried layers, (rows, cols) or (n, rows, cols)."""
    rng = np.random.default_rng(seed)
    shape = (ROWS, COLS) if n is None else (n, ROWS, COLS)
    return {k: noisy(rng, shape, *NOISE) for k in te.capi.CARRIED_LAYERS}


def _chain(te, ctx, g, seed=5, n=None):
    p = te.ChainParams.yaml_defaults(0)
    m = ctx.map()
    if n is None:
        m.chain(g, p, synth.terrain(g.rows, g.cols, RES, seed, "mixed"))
    else:
        m.chain_batched(g, p, n, np.stack([synth.terrain(g.rows, g.cols, RES, seed + k, "mixed") for k in range(n)]))
    return m


def _device(torch, a):
    """A host layer (rows, cols) or (n, rows, cols) as the device layout: every map column-major, back to back."""
    a = np.asarray(a, dtype=np.float32)
    a = a[None] if a.ndim == 2 else a
    return torch.from_numpy(np.ascontiguousarray(a.transpose(0, 2, 1)).reshape(-1)).cuda()


def _x86_sub(u, lo):
    """np.float32 subtraction, as the reference computes upper - lower."""
    with np.errstate(invalid="ignore", over="ignore"):
        return np.float32(u) - np.float32(lo)


# ---- 1. round trip ---------------------------------------------------------------------------------------------------------

def test_round_trip_single_map_with_start_index(te, ctx):
    torch = pytest.importorskip("torch")
    start = (37, 101)
    g = _geo(te, start)
    m = _chain(te, ctx, g)
    C7 = _carried(te, 1)
    names = list(te.capi.CARRIED_LAYERS)
    layers = [C7[n] for n in names]
    layers[names.index("lower_bound")] = None          # GridMap::add(layer, 0.0)
    m.carry_layers(names[::-1], layers[::-1])          # any order of names
    got = m.get_layers(names)
    for n in names:
        if n == "lower_bound":
            assert (bits(got[n]) == 0).all()
        else:
            assert_same_bits(got[n], C7[n], n)                    # re-wrapped: the buffer order the layers came in
    dev = torch.full((len(names) * ROWS * COLS,), 7.0, dtype=torch.float32, device="cuda")
    gd = m.get_layers(names, out=dev, memory=te.MEM_DEVICE)
    ctx.synchronize()
    for n in names:
        want = np.zeros((ROWS, COLS), np.float32) if n == "lower_bound" else unwrap(C7[n], start)
        assert_same_bits(gd[n].cpu().numpy(), want, n)            # device memory: default order
    # device layers are in default order; host reads re-wrap them
    D = _carried(te, 2)
    m.carry_layers(["upper_bound", "time"], [_device(torch, unwrap(D["upper_bound"], start)), None], memory=te.MEM_DEVICE)
    ctx.synchronize()
    got = m.get_layers(["upper_bound", "lower_bound", "time"])
    assert_same_bits(got["upper_bound"], D["upper_bound"])
    assert (bits(got["lower_bound"]) == 0).all() and (bits(got["time"]) == 0).all()


@pytest.mark.parametrize("memory", ["host", "device"])
def test_round_trip_batch(te, ctx, memory):
    torch = pytest.importorskip("torch")
    n = 3
    g = _geo(te)
    m = _chain(te, ctx, g, n=n)
    C7 = _carried(te, 3, n)
    names = ["robot_slope", "variance", "horizontal_variance_xy", "upper_bound"]
    C7["robot_slope"] = _carried(te, 4, n)["time"]
    layers = [C7[k] for k in names]
    if memory == "host":
        m.carry_layers(names, layers)
    else:
        m.carry_layers(names, [_device(torch, a) for a in layers], memory=te.MEM_DEVICE)
        ctx.synchronize()
    got = m.get_layers(names)
    for k in names:
        assert got[k].shape == (n, ROWS, COLS)
        assert_same_bits(got[k], C7[k], k)
    # a selection rewrites only its maps, in map_index order
    S = _carried(te, 5, 2)
    sel = [2, 0]
    if memory == "host":
        m.carry_layers(["variance", "upper_bound"], [S["variance"], None], map_index=sel)
    else:
        m.carry_layers(["variance", "upper_bound"], [_device(torch, S["variance"]), None], map_index=sel, memory=te.MEM_DEVICE)
        ctx.synchronize()
    got = m.get_layers(names)
    for j, k in enumerate(sel):
        assert_same_bits(got["variance"][k], S["variance"][j])
        assert (bits(got["upper_bound"][k]) == 0).all()
    assert_same_bits(got["variance"][1], C7["variance"][1])
    assert_same_bits(got["upper_bound"][1], C7["upper_bound"][1])
    for k in ("robot_slope", "horizontal_variance_xy"):
        assert_same_bits(got[k], C7[k], k)


# ---- 2. uncertainty_range --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("start", [(0, 0), (19, 62)])
def test_uncertainty_range_bits(te, ctx, start):
    torch = pytest.importorskip("torch")
    g = _geo(te, start)
    m = _chain(te, ctx, g)
    rng = np.random.default_rng(6)
    up, lo = noisy(rng, (ROWS, COLS), *NOISE), noisy(rng, (ROWS, COLS), *NOISE)
    up[:3, :] = np.inf                                  # Inf - Inf, -Inf - -Inf, Inf - -Inf
    lo[0, :], lo[1, :], lo[2, :] = np.inf, -np.inf, -np.inf
    up[3, :], lo[3, :] = -np.inf, -np.inf
    m.carry_layers(["upper_bound", "lower_bound"], [up, lo])
    want = _x86_sub(up, lo)
    assert np.isnan(want).sum() > 500 and np.isinf(want).any()
    got = m.get_layers(["traversability", "upper_bound", "lower_bound", "uncertainty_range"])
    assert list(got) == ["traversability", "upper_bound", "lower_bound", "uncertainty_range"]
    assert_same_bits(got["uncertainty_range"], want)
    assert_same_bits(got["upper_bound"], up)
    out = torch.full((2 * ROWS * COLS + 1,), 3.0, dtype=torch.float32, device="cuda")
    gd = m.get_layers(["uncertainty_range", "elevation"], out=out[1:], memory=te.MEM_DEVICE)   # 4 bytes off 16-byte alignment
    ctx.synchronize()
    assert_same_bits(gd["uncertainty_range"].cpu().numpy(), unwrap(want, start))
    # a batch, in both memory modes
    b = _chain(te, ctx, _geo(te), n=2)
    U, L = noisy(rng, (2, ROWS, COLS), *NOISE), noisy(rng, (2, ROWS, COLS), *NOISE)
    b.carry_layers(["lower_bound", "upper_bound"], [L, U])
    assert_same_bits(b.get_layers(["uncertainty_range"])["uncertainty_range"], _x86_sub(U, L))
    out = torch.empty(2 * ROWS * COLS, dtype=torch.float32, device="cuda")
    gd = b.get_layers(["uncertainty_range"], out=out, memory=te.MEM_DEVICE)
    ctx.synchronize()
    assert_same_bits(gd["uncertainty_range"].cpu().numpy(), _x86_sub(U, L))


def test_uncertainty_range_errors(te, ctx):
    m = _chain(te, ctx, _geo(te))
    rng = np.random.default_rng(7)
    m.carry_layers(["upper_bound"], [noisy(rng, (ROWS, COLS), *NOISE)])
    with pytest.raises(te.TEError) as e:
        m.get_layers(["uncertainty_range"])
    assert e.value.code == MISSING_LAYER
    m.carry_layers(["lower_bound"], [None])
    m.get_layers(["uncertainty_range"])
    for fn in (lambda: m.get_submaps([[0.3, -0.2]], [[0.5, 0.5]], ["uncertainty_range"]),
               lambda: m.get_submaps_batched([0], [[0.3, -0.2]], [[0.5, 0.5]], ["upper_bound", "uncertainty_range"])):
        with pytest.raises(te.TEError) as e:
            fn()
        assert e.value.code == BAD_ARG


# ---- 3. submaps ------------------------------------------------------------------------------------------------------------

def test_submaps_of_carried_layers(te, ctx, oracle):
    torch = pytest.importorskip("torch")
    start = (23, 7)
    m = _chain(te, ctx, _geo(te, start))
    C7 = _carried(te, 8)
    m.carry_layers(list(C7), list(C7.values()))
    names = ["traversability", "elevation", "lower_bound", "horizontal_variance_x", "time"]
    full = {k: unwrap(v, start) for k, v in m.get_layers(names).items()}   # bit order
    rng = np.random.default_rng(9)
    pos, length = submap_windows(rng, 150, _geo(te))
    want = so.submap_geometry(oracle.Geometry.make(ROWS, COLS, RES, POS), pos, length)
    assert 0 < want["success"].sum() < len(pos)
    check_submaps(m.get_submaps(pos, length, names), want, full, names)
    total = len(names) * int((want["rows"] * want["cols"]).sum())
    out = torch.full((total,), -3.0, dtype=torch.float32, device="cuda")
    res = m.get_submaps(pos, length, names, out=out, memory=te.MEM_DEVICE)
    ctx.synchronize()
    check_submaps([(i, None if d is None else {n: v.cpu().numpy() for n, v in d.items()}) for i, d in res], want, full, names)
    # a batch: window k on map win_map[k]
    n = 3
    b = _chain(te, ctx, _geo(te), n=n)
    B = _carried(te, 10, n)
    b.carry_layers(list(B), list(B.values()))
    bn = ["upper_bound", "variance", "horizontal_variance_y", "horizontal_variance_xy", "traversability_step"]
    fullb = b.get_layers(bn)
    wm = rng.integers(0, n, len(pos)).astype(np.int32)
    res = b.get_submaps_batched(wm, pos, length, bn)
    for k in range(n):
        idx = np.nonzero(wm == k)[0]
        wk = {f: v[idx] for f, v in want.items()}
        check_submaps([res[q] for q in idx], wk, {x: v[k] for x, v in fullb.items()}, bn)


# ---- 4. robot_slope through carry ------------------------------------------------------------------------------------------

def _robot_slope(rng, shape, base):
    """robot_slope with NaN cells and zero patches that the request's lines cross."""
    rs = np.array(base, dtype=np.float32)
    rs[rng.random(shape) < 0.05] = np.nan
    for _ in range(60):
        a, b = int(rng.integers(0, shape[-2] - 4)), int(rng.integers(0, shape[-1] - 4))
        rs[..., a:a + 3, b:b + 3] = 0.0
    return np.asfortranarray(rs) if rs.ndim == 2 else rs


@pytest.mark.parametrize("n", [None, 3])
def test_robot_slope_through_carry_equals_set_layers(te, ctx, oracle, n):
    g, og = te.Geometry.make(200, 180, RES), oracle.Geometry.make(200, 180, RES)
    p, ft = te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    rng = np.random.default_rng(11 if n is None else 12)
    k = 1 if n is None else n
    z = np.stack([synth.terrain(200, 180, RES, 40 + j, "mixed") for j in range(k)])
    a = ctx.map()
    outs = a.chain(g, p, z[0], outputs=True) if n is None else a.chain_batched(g, p, n, z, outputs=True)
    rs = _robot_slope(rng, (200, 180) if n is None else (n, 200, 180), outs["slope"])
    a.carry_layers(["robot_slope"], [rs])
    b, nr = ctx.map(), ctx.map()   # robot_slope through te_map_set_layers; and no robot_slope at all
    lay = [outs["traversability"], outs["slope"], outs["step"], z[0] if n is None else z]
    if n is None:
        b.set_layers(g, *lay, roughness=outs["roughness"], robot_slope=rs)
        nr.set_layers(g, *lay, roughness=outs["roughness"])
    else:
        b.set_layers_batched(g, n, *lay, roughness=outs["roughness"], robot_slope=rs)
        nr.set_layers_batched(g, n, *lay, roughness=outs["roughness"])
    assert_same_held(held(te, a), held(te, b), "layers")
    fps = request_footprints(rng)
    gated = False
    for step in range(3):
        R = dict(mixed_request(rng, og, 120, fps, circular=0.7, cap_path=False), fps=fps)
        pm = None if n is None else rng.integers(0, n, len(R["kind"])).astype(np.int32)
        ga, gb, gn = ask(a, ft, R, pm), ask(b, ft, R, pm), ask(nr, ft, R, pm)
        assert_same_answers(ga, gb, ("answers", step))
        assert_same_bits(a.get_footprint(), b.get_footprint(), ("cache", step))
        assert a.request_stats() == b.request_stats(), step
        gated = gated or not np.array_equal(ga[0], gn[0])
    assert gated   # the request crossed robot_slope zeros: without the layer some answers differ


# ---- 5. state untouched ----------------------------------------------------------------------------------------------------

def test_carry_leaves_cache_memo_and_answers(te, ctx, oracle):
    g, og = te.Geometry.make(200, 180, RES), oracle.Geometry.make(200, 180, RES)
    p, ft = te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    z = synth.terrain(200, 180, RES, 77, "mixed")
    a, b = ctx.map(), ctx.map()
    for m in (a, b):
        m.chain(g, p, z)
    rng = np.random.default_rng(13)
    fps = request_footprints(rng)
    R = dict(mixed_request(rng, og, 80, fps, circular=0.7, cap_path=False), fps=fps)
    assert_same_answers(ask(a, ft, R), ask(b, ft, R), "first")
    cache = a.get_footprint()
    assert np.isfinite(cache).any()
    a.carry_layers(list(te.capi.CARRIED_LAYERS), [None] * 4 + list(_carried(te, 14).values())[4:])
    assert_same_bits(a.get_footprint(), cache, "cache after carry")
    for step in range(2):
        R = dict(mixed_request(rng, og, 80, fps, circular=0.7, cap_path=False), fps=fps)
        assert_same_answers(ask(a, ft, R), ask(b, ft, R), step)
        assert_same_bits(a.get_footprint(), b.get_footprint(), step)
        assert a.request_stats() == b.request_stats(), step
    assert_same_bits(a.footprint(ft), b.footprint(ft), "sweep on the kept cache")
    # robot_slope only adds the inclination gates of later requests: the cache stays as it was
    cache = a.get_footprint()
    a.carry_layers(["robot_slope"], [np.ones((200, 180), np.float32)])
    assert_same_bits(a.get_footprint(), cache, "cache after carrying robot_slope")


# ---- 6. lifetime -----------------------------------------------------------------------------------------------------------

def test_whole_map_updates_drop_carried_layers(te, ctx):
    g = _geo(te)
    p = te.ChainParams.yaml_defaults(0)
    z = synth.terrain(ROWS, COLS, RES, 3, "mixed")
    gi = te.image_geometry(ROWS, COLS, RES)
    img = (np.arange(ROWS * COLS).reshape(ROWS, COLS) % 251).astype(np.uint8)
    m = ctx.map()
    m.chain(g, p, z)
    lay = m.get_layers(MAIN)
    updates = [lambda: m.chain(g, p, z), lambda: m.chain_batched(g, p, 2, np.stack([z, z])),
               lambda: m.set_layers(g, *(lay[k] for k in ("traversability", "traversability_slope", "traversability_step", "elevation"))),
               lambda: m.set_layers_batched(g, 2, *(np.stack([lay[k]] * 2) for k in ("traversability", "traversability_slope",
                                                                                     "traversability_step", "elevation"))),
               lambda: m.chain_image(gi, p, img, -1.0, 2.0), lambda: m.chain_image(gi, p, np.stack([img, img]), -1.0, 2.0)]
    for k, update in enumerate(updates):
        shape = (ROWS, COLS) if m.nmaps == 1 else (m.nmaps, ROWS, COLS)
        m.carry_layers(["upper_bound", "robot_slope", "time"], [np.ones(shape, np.float32), None, None])
        assert m.get_layers(["upper_bound"])["upper_bound"].shape == shape
        update()
        for name in ("upper_bound", "time", "robot_slope"):
            with pytest.raises(te.TEError) as e:
                m.get_layers([name])
            assert e.value.code == MISSING_LAYER, (k, name)


def test_maps_updates_fill_the_selected_maps_carried_layers_with_nan(te, ctx):
    n = 4
    g = te.image_geometry(ROWS, COLS, RES)
    p = te.ChainParams.yaml_defaults(0)
    b = ctx.map()
    b.chain_batched(g, p, n, np.stack([synth.terrain(ROWS, COLS, RES, 50 + k, "mixed") for k in range(n)]))
    C7 = _carried(te, 15, n)
    names = ["upper_bound", "lower_bound", "time"]
    b.carry_layers(names, [C7[k] for k in names])
    b.footprint(te.FootprintParams.yaml_defaults())   # every cache in use
    z = synth.terrain(ROWS, COLS, RES, 99, "mixed")
    img = (np.arange(ROWS * COLS).reshape(ROWS, COLS) % 241).astype(np.uint8)

    def set_maps(sel):
        lay = b.get_layers(MAIN)
        b.set_layers_maps(g, sel, *(lay[k][sel] for k in ("traversability", "traversability_slope", "traversability_step",
                                                          "elevation")), roughness=lay["traversability_roughness"][sel])

    for sel, update in (([2, 0], lambda s: b.chain_maps(g, p, s, np.stack([z] * len(s)))), ([1], set_maps),
                        ([3], lambda s: b.chain_image_maps(g, p, s, np.stack([img] * len(s)), 0.0, 1.5))):
        before = held(te, b)
        n0 = ctx.stats()[0]
        update(sel)
        after = held(te, b)
        assert set(after) == set(before)
        for k in range(n):
            for name in after:
                if k in sel and name in names:
                    assert np.isnan(after[name][k]).all(), (sel, k, name)
                elif k not in sel:
                    assert_same_bits(after[name][k], before[name][k], (sel, k, name))
        if update is set_maps:
            assert ctx.stats()[0] - n0 == 1   # the NaN fill rides the one k_map_slots launch
    # a selection may not add a layer the batch does not hold; the map is unchanged
    before = held(te, b)
    for name in ("variance", "robot_slope"):
        with pytest.raises(te.TEError) as e:
            b.carry_layers([name], [None], map_index=[0])
        assert e.value.code == BAD_ARG
        assert_same_held(held(te, b), before, name)
    b.carry_layers(["variance"], [None])   # every map: fine
    b.carry_layers(["variance"], [np.ones((1, ROWS, COLS), np.float32)], map_index=[2])
    got = b.get_layers(["variance"])["variance"]
    assert (got[2] == 1.0).all() and (bits(got[[0, 1, 3]]) == 0).all()


def test_launch_counts(te, ctx):
    b = _chain(te, ctx, _geo(te), n=3)
    one = np.ones((3, ROWS, COLS), np.float32)
    for names, layers, sel, want in ((["upper_bound", "time"], [one, one], None, 0), (["upper_bound", "time"], [one, None], None, 1),
                                     (["upper_bound", "time"], [None, None], None, 1), (["upper_bound", "time"], [one[:2], None], [2, 1], 1),
                                     (["upper_bound"], [one[:1]], [0], 1)):
        n0 = ctx.stats()[0]
        b.carry_layers(names, layers, map_index=sel)
        assert ctx.stats()[0] - n0 == want, (names, sel)


# ---- 7. error table --------------------------------------------------------------------------------------------------------

def test_error_table_leaves_the_map_unchanged(te, ctx):
    L = te.load_library()
    fn = L.te_map_carry_layers
    lay = np.ones((ROWS, COLS), np.float32, order="F")
    ptrs = lambda k: (C.c_void_p * k)(*([lay.ctypes.data] * k))  # noqa: E731  (lay outlives every call)
    empty = ctx.map()
    assert fn(empty._h, 0, None, 0x100, ptrs(1), te.MEM_HOST) == BAD_ARG   # no layers yet
    assert fn(None, 0, None, 0x100, ptrs(1), te.MEM_HOST) == BAD_ARG
    b = _chain(te, ctx, _geo(te), n=3)
    b.carry_layers(["upper_bound"], [np.zeros((3, ROWS, COLS), np.float32)])
    before = held(te, b)
    idx = lambda *v: np.asarray(v, np.int32)  # noqa: E731
    cases = [
        (BAD_ARG, 0, None, 0, 0),                        # empty mask
        (BAD_ARG, 0, None, 0x1, 1),                      # a chain layer
        (BAD_ARG, 0, None, 0x10, 1),                     # elevation
        (BAD_ARG, 0, None, 0x40, 1),                     # the cache
        (BAD_ARG, 0, None, 0x80, 1),                     # unassigned bit
        (BAD_ARG, 0, None, 0x8000, 1),                   # uncertainty_range is derived
        (BAD_ARG, 0, None, 0x10000, 1),                  # unknown bit
        (BAD_ARG, 0, None, 0x100 | 0x8, 2),              # a carried bit with roughness
        (BAD_ARG, 2, idx(1, 1), 0x100, 1),               # a map twice
        (BAD_ARG, 1, idx(3), 0x100, 1),                  # outside the batch
        (BAD_ARG, 1, idx(-1), 0x100, 1),
        (BAD_ARG, 4, idx(0, 1, 2, 0), 0x100, 1),         # more than nmaps
        (BAD_ARG, 1, None, 0x100, 1),                    # a null map_index with nsel > 0
        (BAD_ARG, 0, idx(0), 0x100, 1),                  # nsel 0 with a map_index
        (BAD_ARG, -1, idx(0), 0x100, 1),
        (BAD_ARG, 1, idx(0), 0x200, 1),                  # a layer the batch does not hold, to a selection
        (BAD_ARG, 1, idx(0), 0x20, 1),                   # robot_slope likewise
    ]
    for code, nsel, mi, mask, npt in cases:
        rc = fn(b._h, nsel, None if mi is None else mi.ctypes.data, mask, ptrs(max(npt, 1)), te.MEM_HOST)
        assert rc == code, (nsel, mi, hex(mask), rc, L.te_last_error())
        assert_same_held(held(te, b), before, (nsel, hex(mask)))
    assert fn(b._h, 0, None, 0x100, None, te.MEM_HOST) == BAD_ARG          # a null layers array
    assert fn(b._h, 0, None, 0x100, ptrs(1), 7) == BAD_ARG                 # an unknown memory mode
    assert_same_held(held(te, b), before, "null layers / memory")
    # a selection on a map whose layers came with a start index
    w = _chain(te, ctx, _geo(te, (5, 9)))
    w.carry_layers(["upper_bound"], [lay])
    before = held(te, w)
    sel0 = idx(0)
    assert fn(w._h, 1, sel0.ctypes.data, 0x100, ptrs(1), te.MEM_HOST) == UNSUPPORTED
    assert_same_held(held(te, w), before, "start index")
