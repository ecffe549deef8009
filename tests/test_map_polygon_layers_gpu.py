"""te_map_footprint_polygon_keep: traversability_x / traversability_rot kept on a te_map, swept for chosen maps of a batch at
their own footprint yaws and positions in one launch.  Every kept layer must equal, bit for bit, what te_map_footprint_polygon
returns on a single-map te_map holding that map at its position at that yaw; maps not swept, the cache and the other layers must
keep their bits; the layers must be served by te_map_get_layers and te_map_get_submaps(_batched) and follow the reference's
lifetime (a new map replaces the old one wholesale)."""
import ctypes as C

import numpy as np
import pytest

import synth
from helpers import assert_same_bits, bits, close_sweep
from map_helpers import assert_same_held, close_maps, held  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES = 128, 112, 0.02
POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]   # robot_footprint_parameter.yaml:3
XR = ["traversability_x", "traversability_rot"]
BAD_ARG, MISSING_LAYER, UNSUPPORTED = -1, -2, -4
SPREAD = np.array([(0.0, 0.0), (13.37, -3.21), (-101.23, 77.7), (1000.01, 0.05), (0.31, 512.39), (-7.77, -3.21)])


def _terrain(n, seed=0, rows=ROWS, cols=COLS):
    return np.stack([synth.terrain(rows, cols, RES, seed + k, "mixed") for k in range(n)]).astype(np.float32)


def _batch(te, ctx, z, positions=None):
    b = ctx.map()
    b.chain_batched(te.Geometry.make(z.shape[1], z.shape[2], RES), te.ChainParams.yaml_defaults(0), len(z), z, positions=positions)
    return b


def _single(te, ctx, z, pos=(0.0, 0.0)):
    s = ctx.map()
    s.chain(te.Geometry.make(z.shape[0], z.shape[1], RES, tuple(pos)), te.ChainParams.yaml_defaults(0), z)
    return s


# ---- 1. single map ---------------------------------------------------------------------------------------------------------

def test_single_map_with_start_index(te, ctx, oracle):
    ft = te.FootprintParams.yaml_defaults()
    start, pos, yaw = (37, 101), (1.25, -0.5), 0.7854
    g = te.Geometry.make(ROWS, COLS, RES, pos)
    g.start_row, g.start_col = start
    m = ctx.map()
    m.chain(g, te.ChainParams.yaml_defaults(0), _terrain(1, 3)[0])      # layers in buffer order
    want_x, want_rot = m.footprint_polygon(ft, POLY, yaw)
    got_x, got_rot = m.footprint_polygon_keep(ft, POLY, yaw, outputs=True)
    assert_same_bits(got_x, want_x, "x")
    assert_same_bits(got_rot, want_rot, "rot")
    kept = m.get_layers(XR)                                            # re-wrapped like the map's other outputs
    assert_same_bits(kept["traversability_x"], want_x)
    assert_same_bits(kept["traversability_rot"], want_rot)
    # the oracle on the unwrapped layers
    lay = m.get_layers(["traversability", "traversability_slope", "traversability_step", "elevation"])
    unwrap = lambda a: np.asfortranarray(np.roll(a, (-start[0], -start[1]), axis=(0, 1)))  # noqa: E731
    ox, orot = oracle.footprint_polygon(oracle.Geometry.make(ROWS, COLS, RES, pos), oracle.FootprintParams.yaml_defaults(), POLY, yaw,
                                        *(unwrap(lay[k]) for k in ("traversability", "traversability_slope", "traversability_step",
                                                                   "elevation")))
    assert close_sweep(unwrap(got_x), ox) and close_sweep(unwrap(got_rot), orot)
    assert (ox > 0).any()


# ---- 2. whole batch at one position, a yaw per map -------------------------------------------------------------------------

def test_whole_batch_a_yaw_per_map(te, ctx):
    ft = te.FootprintParams.yaml_defaults()
    z = _terrain(5, 10)
    yaws = [0.0, 0.7854, -1.3, 2.9, 0.7854]
    b = _batch(te, ctx, z)
    x, rot = b.footprint_polygon_keep(ft, POLY, yaws, outputs=True)
    kept = b.get_layers(XR)
    for k in range(len(z)):
        sx, srot = _single(te, ctx, z[k]).footprint_polygon(ft, POLY, yaws[k])
        for got in (x[k], kept["traversability_x"][k]):
            assert_same_bits(got, sx, k)
        for got in (rot[k], kept["traversability_rot"][k]):
            assert_same_bits(got, srot, k)
    # one yaw for every map
    b.footprint_polygon_keep(ft, POLY, -0.4)
    kept = b.get_layers(XR)
    for k in range(len(z)):
        sx, srot = _single(te, ctx, z[k]).footprint_polygon(ft, POLY, -0.4)
        assert_same_bits(kept["traversability_x"][k], sx, k)
        assert_same_bits(kept["traversability_rot"][k], srot, k)


# ---- 3. batch at several positions, scrambled selections -------------------------------------------------------------------

def test_selection_at_several_positions(te, ctx):
    ft = te.FootprintParams.yaml_defaults()
    n = len(SPREAD)
    z = _terrain(n, 20)
    b = _batch(te, ctx, z, SPREAD)
    b.carry_layers(["upper_bound", "time"], [np.full((n, ROWS, COLS), 0.5, np.float32), None])
    b.footprint(ft)                                                     # every cache in use
    stats = b.request_stats()
    singles = [_single(te, ctx, z[k], SPREAD[k]) for k in range(n)]

    def check(sel, yaws, before):
        after = held(te, b, polygon=True)
        assert set(after) == set(before) | set(XR), sorted(set(after) ^ set(before))
        for name in after:
            if name not in XR:
                assert_same_bits(after[name], before[name], name)                  # the cache and every other layer
        for j, k in enumerate(sel):
            sx, srot = singles[k].footprint_polygon(ft, POLY, yaws[j])
            assert_same_bits(after["traversability_x"][k], sx, (sel, k))
            assert_same_bits(after["traversability_rot"][k], srot, (sel, k))
        for k in set(range(n)) - set(sel):
            for name in XR:
                if name in before:
                    assert_same_bits(after[name][k], before[name][k], (sel, k, name))
                else:
                    assert (bits(after[name][k]) == 0xffffffff).all(), (sel, k, name)   # never swept
        assert b.request_stats() == stats

    before = held(te, b, polygon=True)
    sel, yaws = [4, 1], [0.5, -2.0]
    x, rot = b.footprint_polygon_keep(ft, POLY, yaws, map_index=sel, outputs=True)
    check(sel, yaws, before)
    after = held(te, b, polygon=True)
    for j, k in enumerate(sel):                                         # outputs: the swept maps in map_index order
        assert_same_bits(x[j], after["traversability_x"][k])
        assert_same_bits(rot[j], after["traversability_rot"][k])
    before = after
    sel, yaws = [3, 0, 5, 1], [1.1, 0.5, 1.1, 0.0]                      # repeated yaws, yaw 0, a map swept again
    b.footprint_polygon_keep(ft, POLY, yaws, map_index=sel)
    check(sel, yaws, before)


# ---- 4. launches -----------------------------------------------------------------------------------------------------------

def test_launch_counts(te, ctx):
    ft = te.FootprintParams.yaml_defaults()
    n = len(SPREAD)
    z = _terrain(n, 30)
    deltas = {}
    for where, positions in (("one position", None), ("many positions", SPREAD)):
        b = _batch(te, ctx, z, positions)
        for sel in (None, [2], [5, 0, 3, 1, 4, 2]):
            ns = n if sel is None else len(sel)
            for yaws in ([0.25], list(np.linspace(-3.0, 3.0, ns))):
                n0 = ctx.stats()[0]
                b.footprint_polygon_keep(ft, POLY, yaws, map_index=sel)
                deltas[(where, sel is None, ns, len(yaws))] = ctx.stats()[0] - n0
    for key, d in deltas.items():
        assert d == (3 if key[1] else 4), (key, d)                      # predicates + sweep, and the gather of a selection


# ---- 5. serving ------------------------------------------------------------------------------------------------------------

def test_get_layers_and_submaps(te, ctx):
    torch = pytest.importorskip("torch")
    ft = te.FootprintParams.yaml_defaults()
    n = 4
    z = _terrain(n, 40)
    b = _batch(te, ctx, z, SPREAD[:n])
    for names in (XR, ["traversability_x"]):
        with pytest.raises(te.TEError) as e:                            # not before the first keep-sweep
            b.get_layers(names)
        assert e.value.code == MISSING_LAYER
        with pytest.raises(te.TEError) as e:
            b.get_submaps_batched([0], [SPREAD[0]], [(0.5, 0.5)], names)
        assert e.value.code == MISSING_LAYER
    b.footprint_polygon_keep(ft, POLY, [0.3, -1.0, 2.2, 0.3])
    kept = b.get_layers(XR)
    names = ["traversability", "traversability_slope", "elevation"] + XR
    mixed = b.get_layers(["traversability_rot", "elevation", "traversability", "traversability_x", "traversability_slope"])
    assert list(mixed) == ["traversability", "traversability_slope", "elevation"] + XR   # bit order
    for name in XR:
        assert_same_bits(mixed[name], kept[name], name)
    out = torch.empty(len(names) * n * ROWS * COLS, dtype=torch.float32, device="cuda")
    dev = b.get_layers(names, out=out, memory=te.MEM_DEVICE)
    ctx.synchronize()
    for name in names:
        got = np.ascontiguousarray(dev[name].cpu().numpy())           # device layers: (n, rows, cols) views in default order
        assert_same_bits(got, mixed[name], name)
    # windows inside the map and at its edge, on every map
    half = np.array([0.5 * ROWS * RES, 0.5 * COLS * RES])
    win_map, centres, lengths = [], [], []
    for k in range(n):
        for off, ln in (((0.1, -0.2), (0.5, 0.3)), ((half[0] - 0.05, -half[1] + 0.03), (0.4, 0.4)), ((0.0, 0.0), (9.0, 9.0))):
            win_map.append(k)
            centres.append(SPREAD[k] + np.array(off))
            lengths.append(ln)
    res = b.get_submaps_batched(win_map, centres, lengths, XR)
    assert all(info["success"] for info, _ in res)
    for (info, lay), k in zip(res, win_map):
        r0, c0, nr, nc = int(info["top_row"]), int(info["top_col"]), int(info["rows"]), int(info["cols"])
        for name in XR:
            assert_same_bits(lay[name], kept[name][k][r0:r0 + nr, c0:c0 + nc], (k, name))
    s = _single(te, ctx, z[0])
    s.footprint_polygon_keep(ft, POLY, 0.3)
    (info, lay), = s.get_submaps([(0.1, 0.1)], [(0.6, 0.4)], XR + ["traversability"])
    assert_same_bits(lay["traversability_rot"], kept["traversability_rot"][0][int(info["top_row"]):int(info["top_row"]) + int(info["rows"]),
                                                                     int(info["top_col"]):int(info["top_col"]) + int(info["cols"])])


def test_device_memory_outputs(te, ctx):
    torch = pytest.importorskip("torch")
    ft = te.FootprintParams.yaml_defaults()
    n = 4
    z = _terrain(n, 45)
    h, d = _batch(te, ctx, z, SPREAD[:n]), _batch(te, ctx, z, SPREAD[:n])
    for sel, yaws in ((None, [0.3, -1.0, 2.2, 0.3]), ([3, 1], [0.9, 0.0])):
        ns = n if sel is None else len(sel)
        hx, hr = h.footprint_polygon_keep(ft, POLY, yaws, map_index=sel, outputs=True)
        dx, dr = (torch.empty(ns * ROWS * COLS, dtype=torch.float32, device="cuda") for _ in range(2))
        d.footprint_polygon_keep(ft, POLY, yaws, map_index=sel, outputs=(dx, None), memory=te.MEM_DEVICE)
        d.footprint_polygon_keep(ft, POLY, yaws, map_index=sel, outputs=(None, dr), memory=te.MEM_DEVICE)
        ctx.synchronize()
        as_host = lambda t: t.cpu().numpy().reshape(ns, COLS, ROWS).transpose(0, 2, 1)  # noqa: E731
        assert_same_bits(as_host(dx), hx, sel)
        assert_same_bits(as_host(dr), hr, sel)
        assert_same_held(held(te, d, polygon=True), held(te, h, polygon=True), sel)


# ---- 6. lifetime -----------------------------------------------------------------------------------------------------------

def _request(te, b, n):
    """A small circular request on every map (host memory) and the same request in device memory."""
    torch = pytest.importorskip("torch")
    ft = te.FootprintParams.yaml_defaults()
    pos = b.positions()
    begin = np.arange(0, 2 * n + 1, 2, dtype=np.int32)
    poses = np.zeros((2 * n, 7))
    poses[:, 6] = 1.0
    for k in range(n):
        poses[2 * k, :2], poses[2 * k + 1, :2] = pos[k] + (-0.3, 0.1), pos[k] + (0.4, -0.2)
    radius, fb, fx = np.full(n, 0.3), np.zeros(n + 1, np.int32), np.zeros((0, 3), np.float32)
    path_map = np.arange(n, dtype=np.int32)
    b.check_footprint_request_batched(ft, path_map, begin, poses, radius, fb, fx)
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    b.check_footprint_request_device(ft, dev(begin, np.int32), dev(poses, np.float64), dev(radius, np.float64), dev(fb, np.int32),
                                     dev(np.zeros(3, np.float32), np.float32), torch.zeros(n, dtype=torch.uint8, device="cuda"),
                                     torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda"),
                                     max_checks=4096, path_map=dev(path_map, np.int32))


def test_lifetime(te, ctx):
    ft = te.FootprintParams.yaml_defaults()
    n = 4
    g = te.Geometry.make(ROWS, COLS, RES)
    p = te.ChainParams.yaml_defaults(0)
    z = _terrain(n, 50)
    b = _batch(te, ctx, z)
    b.footprint_polygon_keep(ft, POLY, [0.1, 0.2, 0.3, 0.4])
    kept = b.get_layers(XR)
    # entries that leave both layers as they are
    for what, call in (("carry_layers", lambda: b.carry_layers(["upper_bound"], [None])),
                       ("footprint", lambda: b.footprint(ft)), ("footprint_maps", lambda: b.footprint_maps(ft, [2])),
                       ("requests", lambda: _request(te, b, n)), ("clear_footprint", b.clear_footprint),
                       ("footprint_polygon", lambda: b.footprint_polygon(ft, POLY, 1.0)),
                       ("footprint_polygon_yaws", lambda: b.footprint_polygon_yaws(ft, POLY, [1.0, 2.0])),
                       ("footprint_polygon_yaws_reduce", lambda: b.footprint_polygon_yaws_reduce(ft, POLY, [1.0, 2.0]))):
        call()
        ctx.synchronize()
        after = b.get_layers(XR)
        for name in XR:
            assert_same_bits(after[name], kept[name], (what, name))
    # the _maps updates fill the selected maps' layers with 0xffffffff and keep the others
    img = (np.arange(ROWS * COLS).reshape(ROWS, COLS) % 241).astype(np.uint8)
    lay = b.get_layers(["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"])

    def set_maps(sel, positions=None):
        b.set_layers_maps(g, sel, *(lay[k][sel] for k in ("traversability", "traversability_slope", "traversability_step",
                                                          "elevation")), roughness=lay["traversability_roughness"][sel],
                          positions=positions)

    for what, sel, update in (("chain_maps", [2, 0], lambda s: b.chain_maps(g, p, s, z[s])),
                              ("set_layers_maps", [1], set_maps),
                              ("chain_image_maps", [3], lambda s: b.chain_image_maps(g, p, s, np.stack([img] * len(s)), 0.0, 1.5)),
                              ("chain_maps_at", [0], lambda s: b.chain_maps(g, p, s, z[s], positions=[(3.5, -2.0)])),
                              ("set_layers_maps_at", [2, 1], lambda s: set_maps(s, positions=[(0.5, 0.5), (-1.0, 8.0)]))):
        b.footprint_polygon_keep(ft, POLY, 0.6)
        before = b.get_layers(XR)
        update(sel)
        after = b.get_layers(XR)
        for k in range(n):
            for name in XR:
                if k in sel:
                    assert (bits(after[name][k]) == 0xffffffff).all(), (what, k, name)
                else:
                    assert_same_bits(after[name][k], before[name][k], (what, k, name))
    # a _maps_at move, then a sweep of the moved map at its new position
    b.footprint_polygon_keep(ft, POLY, [0.6, 0.6], map_index=[2, 1])
    kept = b.get_layers(XR)
    for k, pos in ((2, (0.5, 0.5)), (1, (-1.0, 8.0))):
        s = ctx.map()
        s.set_layers(te.Geometry.make(ROWS, COLS, RES, pos), lay["traversability"][k], lay["traversability_slope"][k],
                     lay["traversability_step"][k], lay["elevation"][k], roughness=lay["traversability_roughness"][k])
        sx, srot = s.footprint_polygon(ft, POLY, 0.6)
        assert_same_bits(kept["traversability_x"][k], sx, k)
        assert_same_bits(kept["traversability_rot"][k], srot, k)
    # whole-map updates drop both layers
    one = _terrain(1, 60)[0]
    for what, update in (("chain_batched", lambda: b.chain_batched(g, p, n, z)),
                         ("chain_batched_at", lambda: b.chain_batched(g, p, n, z, positions=SPREAD[:n])),
                         ("set_layers_batched", lambda: b.set_layers_batched(g, n, lay["traversability"], lay["traversability_slope"],
                                                                             lay["traversability_step"], lay["elevation"])),
                         ("set_layers_batched_at", lambda: b.set_layers_batched(g, n, lay["traversability"], lay["traversability_slope"],
                                                                                lay["traversability_step"], lay["elevation"],
                                                                                positions=SPREAD[:n])),
                         ("chain_image", lambda: b.chain_image(g, p, np.stack([img] * n), 0.0, 1.5)),
                         ("chain", lambda: b.chain(g, p, one)),
                         ("set_layers", lambda: b.set_layers(g, *(np.zeros((ROWS, COLS), np.float32) for _ in range(4))))):
        b.footprint_polygon_keep(ft, POLY, 0.6)
        update()
        for name in XR:
            with pytest.raises(te.TEError) as e:
                b.get_layers([name])
            assert e.value.code == MISSING_LAYER, (what, name)


def test_maps_update_fills_every_held_layer(te, ctx):
    """A batch holding every carried layer and both polygon layers (nine to fill): a _maps update fills all of them for its maps,
    the ninth in a second k_map_slots launch."""
    ft = te.FootprintParams.yaml_defaults()
    n = 3
    g = te.Geometry.make(ROWS, COLS, RES)
    b = _batch(te, ctx, _terrain(n, 90))
    b.carry_layers(list(te.capi.CARRIED_LAYERS), [None] * len(te.capi.CARRIED_LAYERS))
    b.footprint_polygon_keep(ft, POLY, [0.2, 0.4, 0.6])
    before = held(te, b, polygon=True)
    lay = {k: before[k][[1]] for k in ("traversability", "traversability_slope", "traversability_step", "traversability_roughness",
                                       "elevation")}
    n0 = ctx.stats()[0]
    b.set_layers_maps(g, [1], lay["traversability"], lay["traversability_slope"], lay["traversability_step"], lay["elevation"],
                      roughness=lay["traversability_roughness"])
    assert ctx.stats()[0] - n0 == 2
    after = held(te, b, polygon=True)
    for name in te.capi.CARRIED_LAYERS + te.capi.POLYGON_LAYERS:
        assert (bits(after[name][1]) == 0xffffffff).all(), name
        for k in (0, 2):
            assert_same_bits(after[name][k], before[name][k], (k, name))


# ---- 7. errors -------------------------------------------------------------------------------------------------------------

def test_error_table_leaves_the_map_unchanged(te, ctx):
    L = te.load_library()
    fn = L.te_map_footprint_polygon_keep
    ft = te.FootprintParams.yaml_defaults()
    dbl = lambda v: np.ascontiguousarray(v, dtype=np.float64).reshape(-1)  # noqa: E731
    idx = lambda *v: np.asarray(v, np.int32)  # noqa: E731
    poly = dbl(POLY)
    out = np.zeros(3 * ROWS * COLS, np.float32)

    def call(m, nsel=0, mi=None, pts=poly, npts=None, yaws=dbl([0.5]), nyaws=None, p=ft, memory=te.MEM_HOST):
        return fn(m._h, C.byref(p), nsel, None if mi is None else mi.ctypes.data, len(pts) // 2 if npts is None else npts,
                  pts.ctypes.data, len(yaws) if nyaws is None else nyaws, None if yaws is None else yaws.ctypes.data,
                  out.ctypes.data, None, memory)

    empty = ctx.map()
    assert call(empty) == BAD_ARG                                        # no layers yet
    b = _batch(te, ctx, _terrain(3, 70))
    b.footprint_polygon_keep(ft, POLY, 0.5, map_index=[1])
    b.footprint(ft)
    before = held(te, b, polygon=True)
    rough = te.FootprintParams.yaml_defaults()
    rough.verify_roughness = 1
    nan_yaw = dbl([0.1, np.nan, 0.2])
    big = dbl([[1.2, 0.3], [1.2, -0.3], [-1.2, -0.3], [-1.2, 0.3]])      # reach beyond 31 cells
    cases = [
        (BAD_ARG, dict(nsel=2, mi=idx(1, 1))),                          # a map twice
        (BAD_ARG, dict(nsel=1, mi=idx(3))),                             # outside the batch
        (BAD_ARG, dict(nsel=1, mi=idx(-1))),
        (BAD_ARG, dict(nsel=4, mi=idx(0, 1, 2, 0))),                    # more than nmaps
        (BAD_ARG, dict(nsel=1)),                                        # a null map_index with nsel > 0
        (BAD_ARG, dict(nsel=0, mi=idx(0))),                             # nsel 0 with a map_index
        (BAD_ARG, dict(nsel=-1, mi=idx(0))),
        (BAD_ARG, dict(yaws=dbl([0.1, 0.2]))),                          # 2 yaws for 3 maps
        (BAD_ARG, dict(nsel=2, mi=idx(0, 2), yaws=dbl([0.1, 0.2, 0.3]))),
        (BAD_ARG, dict(yaws=dbl([0.1]), nyaws=0)),
        (BAD_ARG, dict(yaws=None, nyaws=1)),
        (BAD_ARG, dict(yaws=nan_yaw)),                                  # a non-finite yaw
        (BAD_ARG, dict(yaws=dbl([np.inf]))),
        (BAD_ARG, dict(pts=poly[:4])),                                  # two vertices
        (BAD_ARG, dict(pts=np.tile(poly, 5)[:34])),                     # 17 vertices
        (BAD_ARG, dict(pts=dbl([[0.45, np.nan], [0.45, -0.3], [-0.45, -0.3]]))),
        (UNSUPPORTED, dict(pts=big)),
        (BAD_ARG, dict(memory=7)),
    ]
    for code, kw in cases:
        rc = call(b, **kw)
        assert rc == code, (kw, rc, L.te_last_error())
        assert_same_held(held(te, b, polygon=True), before, kw)
    # verify_roughness without roughness
    nr = ctx.map()
    lay = b.get_layers(["traversability", "traversability_slope", "traversability_step", "elevation"])
    nr.set_layers_batched(te.Geometry.make(ROWS, COLS, RES), 3, *(lay[k] for k in ("traversability", "traversability_slope",
                                                                                     "traversability_step", "elevation")))
    nr_before = held(te, nr, polygon=True)
    assert call(nr, p=rough) == MISSING_LAYER
    assert_same_held(held(te, nr, polygon=True), nr_before, "verify_roughness")
    # a selection on a map whose layers came with a start index
    gw = te.Geometry.make(ROWS, COLS, RES)
    gw.start_row, gw.start_col = 5, 9
    w = ctx.map()
    w.chain(gw, te.ChainParams.yaml_defaults(0), _terrain(1, 80)[0])
    assert call(w, nsel=1, mi=idx(0)) == UNSUPPORTED
    assert "traversability_x" not in held(te, w, polygon=True)


def test_distinct_yaw_cap(te, ctx):
    """More than 1024 distinct yaws (by bits) is TE_ERR_UNSUPPORTED; 1024 distinct ones over more maps are fine."""
    ft = te.FootprintParams.yaml_defaults()
    rows = cols = 24
    n = 1026
    b = ctx.map()
    b.chain_batched(te.Geometry.make(rows, cols, RES), te.ChainParams.yaml_defaults(0), n, np.zeros((n, rows, cols), np.float32))
    yaws = np.linspace(-3.0, 3.0, n)
    with pytest.raises(te.TEError) as e:
        b.footprint_polygon_keep(ft, POLY, yaws)
    assert e.value.code == UNSUPPORTED
    for name in XR:                                                      # nothing was kept
        with pytest.raises(te.TEError):
            b.get_layers([name])
    yaws[1024:] = yaws[:2]                                               # 1024 distinct
    b.footprint_polygon_keep(ft, POLY, yaws)
    kept = b.get_layers(XR)
    for k in (0, 1, 1023, 1024, 1025):
        s = ctx.map()
        s.chain(te.Geometry.make(rows, cols, RES), te.ChainParams.yaml_defaults(0), np.zeros((rows, cols), np.float32))
        sx, srot = s.footprint_polygon(ft, POLY, yaws[k])
        assert_same_bits(kept["traversability_x"][k], sx, k)
        assert_same_bits(kept["traversability_rot"][k], srot, k)
