"""A batched te_map whose maps come in their own circular-buffer order (te_map_chain_batched_wrapped,
te_map_set_layers_batched_wrapped, te_map_chain_maps_wrapped, te_map_set_layers_maps_wrapped, te_map_start_indices).  For every
map m, everything the batch returns or holds must equal, bit for bit (NaN payloads included), what a single-map te_map returns or
holds when it is loaded through te_map_chain in host memory with g at map m's position and g's start index set to map m's: host
outputs in that buffer order, device outputs in default order."""
import ctypes as C

import numpy as np
import pytest

import synth
from helpers import batch_request, bits, same_bytes, subset, unwrap, wrap
from map_helpers import ask, close_maps, held  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, NMAPS = 128, 112, 0.02, 6
BAD_ARG = -1
CHAIN = ("slope", "step", "roughness", "traversability")
HELD = ("traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation")
BOUNDS = ("upper_bound", "lower_bound")
PUBLISHED = HELD + BOUNDS + ("uncertainty_range",)
POLY = [(0.11, 0.07), (-0.1, 0.09), (-0.12, -0.08), (0.1, -0.1)]
YAWS = [0.0, 0.4, 1.3, 2.9]
START = np.array([(0, 0), (ROWS - 1, 0), (0, COLS - 1), (37, 53), (64, 1), (5, 100)], np.int32)
POS = np.array([(0.0, 0.0), (13.37, -3.21), (-101.23, 77.7), (0.31, 0.05), (250.125, 512.39), (-7.77, 0.05)])


def _geo(te, k, start=None):
    g = te.Geometry.make(ROWS, COLS, RES, position=tuple(POS[k]))
    g.start_row, g.start_col = (int(v) for v in (START[k] if start is None else start))
    return g


@pytest.fixture(scope="module")
def world(te):
    """Terrains in default order, their bounds (with NaN payloads the library must keep) and the same in each map's buffer order."""
    z = np.stack([synth.terrain(ROWS, COLS, RES, 700 + k, "mixed") for k in range(NMAPS)]).astype(np.float32)
    rng = np.random.default_rng(3)
    up = (z + rng.uniform(0.0, 0.2, z.shape)).astype(np.float32)
    lo = (z - rng.uniform(0.0, 0.2, z.shape)).astype(np.float32)
    payload = np.array([0x7fc12345, 0xffc00001, 0x7f800001], np.uint32).view(np.float32)
    for a, s in ((up, 0), (lo, 1)):
        cells = rng.integers(0, z.size, 200)
        a.reshape(-1)[cells] = payload[(np.arange(200) + s) % 3]
    buffered = lambda a: np.stack([wrap(a[k], START[k]) for k in range(NMAPS)])  # noqa: E731
    return dict(p=te.ChainParams.yaml_defaults(0), g=te.Geometry.make(ROWS, COLS, RES), z=z, up=up, lo=lo, zs=buffered(z),
                ups=buffered(up), los=buffered(lo))


def _single(ctx, te, world, k, z=None, start=None):
    """The oracle of map k: te_map_chain in host memory at map k's position with its start index in g, then its bounds carried."""
    st = START[k] if start is None else start
    s = ctx.map()
    out = s.chain(_geo(te, k, st), world["p"], wrap(world["z"][k], st) if z is None else wrap(z, st), outputs=True)
    s.carry_layers(BOUNDS, [wrap(world["up"][k], st), wrap(world["lo"][k], st)])
    return s, out


def _dev(torch, a):
    """(n, rows, cols) host layers as one device tensor, each map column-major."""
    return torch.as_tensor(np.ascontiguousarray(np.asarray(a, np.float32).transpose(0, 2, 1))).cuda()


def _load(b, te, ctx, world, memory, outputs=True):
    """The whole batch through te_map_chain_batched_wrapped and its bounds through te_map_carry_layers, inputs in `memory`.
    Returns the chain outputs: host arrays in buffer order, or (device memory) numpy copies of the default-order device outputs."""
    if memory == te.MEM_HOST:
        out = b.chain_batched(world["g"], world["p"], NMAPS, world["zs"], outputs=outputs, positions=POS, start_index=START)
        b.carry_layers(BOUNDS, [world["ups"], world["los"]])
        return out
    import torch
    e = _dev(torch, world["zs"])
    outs = [torch.empty(NMAPS * ROWS * COLS, dtype=torch.float32, device="cuda") for _ in CHAIN] if outputs else [None] * 4
    ctx._order_after_torch(te.MEM_DEVICE)
    xy, si = np.ascontiguousarray(POS), np.ascontiguousarray(START)
    b._check(b._L.te_map_chain_batched_wrapped(b._h, C.byref(world["g"]), C.byref(world["p"]), NMAPS, e.data_ptr(),
                                               *(o.data_ptr() if o is not None else None for o in outs), te.MEM_DEVICE,
                                               xy.ctypes.data, si.ctypes.data))
    b._g, b._n = world["g"], NMAPS
    b.carry_layers(BOUNDS, [_dev(torch, world["ups"]), _dev(torch, world["los"])], memory=te.MEM_DEVICE)
    ctx.synchronize()
    if not outputs:
        return None
    return {k: o.cpu().numpy().reshape(NMAPS, COLS, ROWS).transpose(0, 2, 1) for k, o in zip(CHAIN, outs)}


def _check_held(te, b, singles, idx=None, what=""):
    hb = held(te, b, PUBLISHED)
    for k, s in zip(range(NMAPS) if idx is None else idx, singles):
        hs = held(te, s, PUBLISHED)
        for name in hs:
            assert np.array_equal(bits(hb[name][k]), bits(hs[name])), (what, k, name)


def _request(rng, world, npaths):
    """A mixed request whose paths visit every map in no order, each around its own map's position."""
    return batch_request(rng, world["g"], npaths, NMAPS, offsets=POS, circular=0.6, cap_path=False)


def _check_request(b, singles, ft, R):
    got = ask(b, ft, R, R["map"])
    for m in range(NMAPS):
        idx = np.nonzero(R["map"] == m)[0]
        want = ask(singles[m], ft, subset(R, idx))
        for a, w, name in zip(got, want, ("is_safe", "traversability", "area", "count")):
            assert same_bytes(np.asarray(a)[idx], w), (m, name)
        for j, q in enumerate(idx):
            k = max(0, min(int(want[3][j]), 64))
            assert same_bytes(np.asarray(got[4])[q, :k], want[4][j, :k]), (m, q)


@pytest.mark.parametrize("memory", ["host", "device"])
def test_whole_batch_equals_single_maps(te, ctx, world, memory):
    torch = pytest.importorskip("torch")
    mem = te.MEM_HOST if memory == "host" else te.MEM_DEVICE
    ft = te.FootprintParams.yaml_defaults()
    b = ctx.map()
    got = _load(b, te, ctx, world, mem)
    assert np.array_equal(b.start_indices(), START) and np.array_equal(b.positions(), POS)
    singles, outs = zip(*(_single(ctx, te, world, k) for k in range(NMAPS)))
    for k in range(NMAPS):   # chain outputs: host ones in the map's buffer order, device ones in default order
        for name in CHAIN:
            want = outs[k][name] if mem == te.MEM_HOST else unwrap(outs[k][name], START[k])
            assert np.array_equal(bits(got[name][k]), bits(want)), (memory, k, name)
    _check_held(te, b, singles, what=memory)
    # device reads of the published layers are in default order
    dout = torch.empty(len(PUBLISHED) * NMAPS * ROWS * COLS, dtype=torch.float32, device="cuda")
    dl = b.get_layers(list(PUBLISHED), out=dout, memory=te.MEM_DEVICE)
    ctx.synchronize()
    for k, s in enumerate(singles):
        hs = s.get_layers(list(PUBLISHED))
        for name in PUBLISHED:
            assert np.array_equal(bits(dl[name][k].cpu().numpy()), bits(unwrap(hs[name], START[k]))), (memory, k, name)
    # the circular sweep, then the cache read back in both memories
    cache = b.footprint(ft)
    for k, s in enumerate(singles):
        assert np.array_equal(bits(cache[k]), bits(s.footprint(ft))), k
    dc = torch.empty(NMAPS * ROWS * COLS, dtype=torch.float32, device="cuda")
    b._check(b._L.te_map_get_footprint(b._h, dc.data_ptr(), te.MEM_DEVICE))
    ctx.synchronize()
    dc = dc.cpu().numpy().reshape(NMAPS, COLS, ROWS).transpose(0, 2, 1)
    for k, s in enumerate(singles):
        assert np.array_equal(bits(dc[k]), bits(unwrap(s.get_footprint(), START[k]))), k
    # the polygon sweeps, a list of yaws and its reduction (best_yaw included)
    bx, brot = b.footprint_polygon(ft, POLY, 0.7)
    stack = b.footprint_polygon_yaws(ft, POLY, YAWS)
    worst, best, best_yaw = b.footprint_polygon_yaws_reduce(ft, POLY, YAWS)
    for k, s in enumerate(singles):
        sx, srot = s.footprint_polygon(ft, POLY, 0.7)
        assert np.array_equal(bits(bx[k]), bits(sx)) and np.array_equal(bits(brot[k]), bits(srot)), k
        sstack = s.footprint_polygon_yaws(ft, POLY, YAWS)
        for y in range(len(YAWS)):
            assert np.array_equal(bits(stack[y, k]), bits(sstack[y])), (k, y)
        sw, sb, sy = s.footprint_polygon_yaws_reduce(ft, POLY, YAWS)
        assert np.array_equal(bits(worst[k]), bits(sw)) and np.array_equal(bits(best[k]), bits(sb)), k
        assert np.array_equal(best_yaw[k], sy), k
    # the kept polygon layers, each map at its own yaw
    yk = np.linspace(0.2, 2.7, NMAPS)
    kx, krot = b.footprint_polygon_keep(ft, POLY, yk, outputs=True)
    for k, s in enumerate(singles):
        sx, srot = s.footprint_polygon_keep(ft, POLY, [yk[k]], outputs=True)
        assert np.array_equal(bits(kx[k]), bits(sx)) and np.array_equal(bits(krot[k]), bits(srot)), k
    kept = b.get_layers(["traversability_x", "traversability_rot"])
    for k, s in enumerate(singles):
        sk = s.get_layers(["traversability_x", "traversability_rot"])
        for name in sk:
            assert np.array_equal(bits(kept[name][k]), bits(sk[name])), (k, name)
    # a mixed request with untraversable polygons, on caches the sweep filled
    _check_request(b, singles, ft, _request(np.random.default_rng(17), world, 40))
    _check_held(te, b, singles, what=f"{memory} after request")
    # submaps, valid_at and at_poses depend on positions only
    rng = np.random.default_rng(5)
    n = 36
    wmap = rng.integers(0, NMAPS, n).astype(np.int32)
    xy = POS[wmap] + rng.uniform(-1.5, 1.5, (n, 2)) * np.array([ROWS * RES, COLS * RES]) / 2
    ln = rng.uniform(0.0, 1.5, (n, 2))
    names = ["traversability", "elevation", "traversability_footprint", "upper_bound"]
    subs = b.get_submaps_batched(wmap, xy, ln, names)
    valid = b.valid_at_batched(wmap, xy)
    assert 0 < valid.sum() < n
    for q in range(n):
        s = singles[wmap[q]]
        (ri, rl), = s.get_submaps(xy[q:q + 1], ln[q:q + 1], names)
        gi, gl = subs[q]
        for f in ("success", "rows", "cols", "top_row", "top_col", "requested_row", "requested_col"):
            assert gi[f] == ri[f], (q, f)
        for f in ("length_x", "length_y", "position_x", "position_y"):
            assert np.float64(gi[f]).tobytes() == np.float64(ri[f]).tobytes(), (q, f)
        if rl is not None:
            for name in names:
                assert np.array_equal(bits(gl[name]), bits(rl[name])), (q, name)
        assert valid[q] == s.valid_at(xy[q:q + 1])[0], q
    poses = np.zeros((n, 7))
    poses[:, :2] = xy
    poses[:, 5], poses[:, 6] = np.sin(0.3), np.cos(0.3)
    points = rng.uniform(-0.4, 0.4, (9, 3)).astype(np.float32)
    lay, ok = b.at_poses(poses, points, ["traversability", "uncertainty_range"], pose_map=wmap)
    for q in range(n):
        sl, sok = singles[wmap[q]].at_poses(poses[q:q + 1], points, ["traversability", "uncertainty_range"])
        assert np.array_equal(ok[q], sok[0]), q
        for name in sl:
            assert np.array_equal(bits(lay[name][q]), bits(sl[name][0])), (q, name)


def _set_layers_args(out, world, wrapped):
    z = world["zs"] if wrapped else world["z"]
    return (out["traversability"], out["slope"], out["step"], z), dict(roughness=out["roughness"])


def test_null_or_zero_start_index_is_the_at_entry(te, world, ctx):
    """Every _wrapped entry with start_index NULL or all (0, 0) gives the bytes of its _at entry."""
    p, g = world["p"], world["g"]
    ft = te.FootprintParams.yaml_defaults()
    zero = np.zeros((NMAPS, 2), np.int32)
    snaps, outs = [], []
    for mode in ("at", "zero", "null"):
        m = ctx.map()
        if mode == "null":
            e = m._batch_layers(world["z"])
            o = {k: np.empty((NMAPS, COLS, ROWS), np.float32) for k in CHAIN}
            xy = np.ascontiguousarray(POS)
            m._check(m._L.te_map_chain_batched_wrapped(m._h, C.byref(g), C.byref(p), NMAPS, e.ctypes.data,
                                                       *(o[k].ctypes.data for k in CHAIN), te.MEM_HOST, xy.ctypes.data, None))
            m._g, m._n = g, NMAPS
            o = {k: v.transpose(0, 2, 1) for k, v in o.items()}
        else:
            o = m.chain_batched(g, p, NMAPS, world["z"], outputs=True, positions=POS, start_index=zero if mode == "zero" else None)
        m.footprint(ft)
        outs.append(o)
        snaps.append(_held_core(m))
    for h, o in zip(snaps[1:], outs[1:]):
        for name in h:
            assert np.array_equal(bits(h[name]), bits(snaps[0][name])), name
        for name in CHAIN:
            assert np.array_equal(bits(o[name]), bits(outs[0][name])), name
    # set_layers_batched and the two selection entries
    ref = outs[0]
    snaps = []
    for mode in ("at", "zero"):
        m = ctx.map()
        args, kw = _set_layers_args(ref, world, False)
        m.set_layers_batched(g, NMAPS, *args, positions=POS, start_index=zero if mode == "zero" else None, **kw)
        z2 = np.stack([synth.terrain(ROWS, COLS, RES, 950 + k, "rough") for k in range(2)]).astype(np.float32)
        m.chain_maps(g, p, [4, 1], z2, positions=POS[[0, 3]], start_index=zero[:2] if mode == "zero" else None)
        m.set_layers_maps(g, [2], *(a[:1] for a in args), roughness=kw["roughness"][:1], positions=POS[5:6],
                          start_index=zero[:1] if mode == "zero" else None)
        m.footprint(ft)
        snaps.append(_held_core(m))
    for name in snaps[1]:
        assert np.array_equal(bits(snaps[1][name]), bits(snaps[0][name])), name


def _held_core(m):
    return dict(m.get_layers(list(HELD)), cache=m.get_footprint())


def test_selections(te, world, ctx):
    p, g = world["p"], world["g"]
    ft = te.FootprintParams.yaml_defaults()
    b = ctx.map()
    _load(b, te, None, world, te.MEM_HOST, outputs=False)
    singles = [_single(ctx, te, world, k)[0] for k in range(NMAPS)]
    b.footprint(ft)
    for s in singles:
        s.footprint(ft)
    rng = np.random.default_rng(23)
    _check_request(b, singles, ft, _request(rng, world, 30))   # fills caches and memos
    before = held(te, b, PUBLISHED)
    # reload maps 4 and 1 in new buffer orders at new positions
    idx, new_st = [4, 1], np.array([(11, 97), (ROWS - 1, COLS - 1)], np.int32)
    z2 = np.stack([synth.terrain(ROWS, COLS, RES, 960 + k, "rough") for k in range(2)]).astype(np.float32)
    got = b.chain_maps(g, p, idx, np.stack([wrap(z2[j], new_st[j]) for j in range(2)]), outputs=True, positions=POS[[0, 3]],
                       start_index=new_st)
    want_st, want_pos = START.copy(), POS.copy()
    want_st[idx], want_pos[idx] = new_st, POS[[0, 3]]
    assert np.array_equal(b.start_indices(), want_st) and np.array_equal(b.positions(), want_pos)
    after = held(te, b, PUBLISHED)
    for k in set(range(NMAPS)) - set(idx):
        for name in after:
            assert np.array_equal(bits(after[name][k]), bits(before[name][k])), (k, name)
    for j, k in enumerate(idx):
        s = ctx.map()
        gk = te.Geometry.make(ROWS, COLS, RES, position=tuple(want_pos[k]))
        gk.start_row, gk.start_col = (int(v) for v in new_st[j])
        want = s.chain(gk, p, wrap(z2[j], new_st[j]), outputs=True)
        for name in CHAIN:
            assert np.array_equal(bits(got[name][j]), bits(want[name])), (k, name)
        singles[k] = s
    # the selection's bounds in their new buffer orders, then a selected sweep, a selected keep, and a request on every map:
    # the maps not reloaded answer from the caches and memos they kept
    b.carry_layers(BOUNDS, [np.stack([wrap(world[a][k], new_st[j]) for j, k in enumerate(idx)]) for a in ("up", "lo")], map_index=idx)
    for j, k in enumerate(idx):
        singles[k].carry_layers(BOUNDS, [wrap(world["up"][k], new_st[j]), wrap(world["lo"][k], new_st[j])])
    sel = b.footprint_maps(ft, [1, 3, 4])
    for j, k in enumerate([1, 3, 4]):
        assert np.array_equal(bits(sel[j]), bits(singles[k].footprint(ft))), k
    kx, krot = b.footprint_polygon_keep(ft, POLY, [0.3, 1.1], map_index=[4, 2], outputs=True)
    for j, (k, y) in enumerate(zip([4, 2], [0.3, 1.1])):
        sx, srot = singles[k].footprint_polygon_keep(ft, POLY, [y], outputs=True)
        assert np.array_equal(bits(kx[j]), bits(sx)) and np.array_equal(bits(krot[j]), bits(srot)), k
    _check_request(b, singles, ft, _request(rng, world, 30))
    _check_held(te, b, singles, what="after the selection")
    # set_layers_maps_wrapped: map 2 takes map 5's layers in map 5's buffer order, at map 5's position
    s5 = singles[5].get_layers(list(HELD))
    b.set_layers_maps(g, [2], s5["traversability"][None], s5["traversability_slope"][None], s5["traversability_step"][None],
                      s5["elevation"][None], roughness=s5["traversability_roughness"][None], positions=POS[5:6], start_index=START[5:6])
    assert tuple(b.start_indices()[2]) == tuple(START[5])
    b.carry_layers(BOUNDS, [world["ups"][5][None], world["los"][5][None]], map_index=[2])
    singles[5].clear_footprint()
    assert np.array_equal(bits(b.footprint_maps(ft, [2])[0]), bits(singles[5].footprint(ft)))
    _check_held(te, b, [singles[5]], [2], "set_layers_maps_wrapped")
    # an existing _maps entry gives the maps it loads (0, 0): their host outputs are in default order again
    b.chain_maps(g, p, [3], world["z"][3:4], positions=POS[3:4])
    assert tuple(b.start_indices()[3]) == (0, 0)
    s3, _ = _single(ctx, te, world, 3, start=(0, 0))
    b.carry_layers(BOUNDS, [world["up"][3][None], world["lo"][3][None]], map_index=[3])
    b.footprint_maps(ft, [3])
    s3.footprint(ft)
    _check_held(te, b, [s3], [3], "chain_maps after wrapped")


def test_one_map_from_device_memory(te, ctx, world):
    """nmaps = 1 from a device input with a start index equals te_map_chain in host memory with that start index."""
    torch = pytest.importorskip("torch")
    k = 3
    s, want = _single(ctx, te, world, k)
    b = ctx.map()
    e = _dev(torch, world["zs"][k:k + 1])
    outs = [torch.empty(ROWS * COLS, dtype=torch.float32, device="cuda") for _ in CHAIN]
    ctx._order_after_torch(te.MEM_DEVICE)
    xy, si = np.ascontiguousarray(POS[k:k + 1]), np.ascontiguousarray(START[k:k + 1])
    b._check(b._L.te_map_chain_batched_wrapped(b._h, C.byref(world["g"]), C.byref(world["p"]), 1, e.data_ptr(),
                                               *(o.data_ptr() for o in outs), te.MEM_DEVICE, xy.ctypes.data, si.ctypes.data))
    b._g, b._n = world["g"], 1
    b.carry_layers(BOUNDS, [_dev(torch, world["ups"][k:k + 1]), _dev(torch, world["los"][k:k + 1])], memory=te.MEM_DEVICE)
    ctx.synchronize()
    for name, o in zip(CHAIN, outs):
        assert np.array_equal(bits(o.cpu().numpy().reshape(COLS, ROWS).T), bits(unwrap(want[name], START[k]))), name
    hb, hs = held(te, b, PUBLISHED), held(te, s, PUBLISHED)
    for name in hs:
        assert np.array_equal(bits(hb[name]), bits(hs[name])), name


def test_launches(te, ctx, world):
    """A whole-batch _wrapped chain costs its _at entry's launches plus one, whatever nmaps; a host te_map_get_layers of up to
    eight layers costs one."""
    torch = pytest.importorskip("torch")
    p, g = world["p"], world["g"]

    def launches(fn):
        ctx.synchronize()
        before = ctx.stats()[0]
        fn()
        ctx.synchronize()
        return ctx.stats()[0] - before

    for n in (2, NMAPS):
        e = _dev(torch, world["zs"][:n])
        xy, si = np.ascontiguousarray(POS[:n]), np.ascontiguousarray(START[:n])
        m = ctx.map()
        at = lambda: m._check(m._L.te_map_chain_batched_at(m._h, C.byref(g), C.byref(p), n, e.data_ptr(), None, None, None, None,  # noqa: E731
                                                          te.MEM_DEVICE, xy.ctypes.data))
        wr = lambda: m._check(m._L.te_map_chain_batched_wrapped(m._h, C.byref(g), C.byref(p), n, e.data_ptr(), None, None, None,  # noqa: E731
                                                               None, te.MEM_DEVICE, xy.ctypes.data, si.ctypes.data))
        at()
        wr()   # warm: tables built, scratch grown
        assert launches(wr) == launches(at) + 1, n
        wr()   # the maps in their buffer orders again (the _at call gave them (0, 0))
        m._g, m._n = g, n
        m.carry_layers(BOUNDS, [_dev(torch, world["ups"][:n]), _dev(torch, world["los"][:n])], memory=te.MEM_DEVICE)
        names = list(HELD) + list(BOUNDS) + ["traversability_footprint"]
        assert len(names) == 8
        m.get_layers(names)
        assert launches(lambda: m.get_layers(names)) == 1, n


def test_errors_leave_the_map_unchanged(te, world, ctx):
    p, g = world["p"], world["g"]
    ft = te.FootprintParams.yaml_defaults()
    b = ctx.map()
    _load(b, te, None, world, te.MEM_HOST, outputs=False)
    b.footprint(ft)
    before, pos, st = held(te, b, PUBLISHED), b.positions(), b.start_indices()

    def expect(code, fn):
        with pytest.raises(te.TEError) as e:
            fn()
        assert e.value.code == code

    for bad in ((-1, 0), (0, -1), (ROWS, 0), (0, COLS)):
        s = START.copy()
        s[4] = bad
        expect(BAD_ARG, lambda: b.chain_batched(g, p, NMAPS, world["zs"], positions=POS, start_index=s))
        expect(BAD_ARG, lambda: b.chain_maps(g, p, [1, 2], world["zs"][:2], start_index=s[3:5]))
        out = b.get_layers(list(HELD))
        args = [out[n][:1] for n in ("traversability", "traversability_slope", "traversability_step", "elevation")]
        expect(BAD_ARG, lambda: b.set_layers_maps(g, [0], *args, roughness=out["traversability_roughness"][:1], start_index=s[4:5]))
        expect(BAD_ARG, lambda: b.set_layers_batched(g, NMAPS, *[out[n] for n in ("traversability", "traversability_slope",
                                                                                  "traversability_step", "elevation")],
                                                     roughness=out["traversability_roughness"], start_index=s))
    gs = te.Geometry.make(ROWS, COLS, RES)
    gs.start_row = 3
    expect(BAD_ARG, lambda: b.chain_batched(gs, p, NMAPS, world["zs"], positions=POS, start_index=START))
    expect(BAD_ARG, lambda: b.chain_maps(gs, p, [1], world["zs"][:1], start_index=START[:1]))
    expect(BAD_ARG, lambda: b.chain_maps(g, p, [1, 1], world["zs"][:2], start_index=START[:2]))
    expect(BAD_ARG, lambda: b.chain_maps(g, p, [NMAPS], world["zs"][:1], start_index=START[:1]))
    assert np.array_equal(b.positions(), pos) and np.array_equal(b.start_indices(), st)
    after = held(te, b, PUBLISHED)
    for name in after:
        assert np.array_equal(bits(after[name]), bits(before[name])), name
