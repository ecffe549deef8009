"""A batched te_map whose maps sit at their own positions (te_map_chain_batched_at, te_map_set_layers_batched_at,
te_map_chain_maps_at, te_map_set_layers_maps_at, te_map_positions).  For every map m, everything the batch returns or holds must
equal, bit for bit (NaN masks included), what a single-map te_map holding map m at its position returns or holds.  The positions
are chosen so that the on-circle step tips of the fused kernel's mask tables differ between maps, which the test checks on the
host with the kernel's own test (d * d + 0.0 <= r^2 on cell-centre coordinate differences)."""
import ctypes as C

import numpy as np
import pytest

import synth
from helpers import batch_request, bits, footprint_arrays, same_bytes, subset
from map_helpers import ask, close_maps, held  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, NMAPS = 128, 112, 0.02, 4
BAD_ARG = -1
CHAIN = ("slope", "step", "roughness", "traversability")
HELD = ("traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation")


def _coords(px, length, n):
    """grid_map::getPositionFromIndex, in the library's operand order (te_grid.cuh cell_coord)."""
    off = 0.5 * length - 0.5 * RES
    return (px + off) + RES * (-np.arange(n, dtype=np.float64))


def _tip_masks(px, py, p):
    """The fused kernel's row and column mask bits (te_fused.cu fused_mask_bits) of a map at (px, py)."""
    out = []
    for P in (_coords(px, ROWS * RES, ROWS), _coords(py, COLS * RES, COLS)):
        n, b = len(P), np.zeros(len(P), np.uint8)
        r1, r2 = p.step_first_radius ** 2, p.step_second_radius ** 2
        d = P[:-2] - P[2:]                      # P[i - 2] - P[i] for i >= 2, and P[i + 2] - P[i] = -d for i < n - 2
        b[2:] |= np.where(d * d + 0.0 <= r1, 1, 0).astype(np.uint8) | np.where(d * d + 0.0 <= r2, 4, 0).astype(np.uint8)
        b[:n - 2] |= np.where(d * d + 0.0 <= r1, 2, 0).astype(np.uint8) | np.where(d * d + 0.0 <= r2, 8, 0).astype(np.uint8)
        out.append(b)
    return out


@pytest.fixture(scope="module")
def world(te):
    """Terrains, chain parameters and NMAPS positions whose tip masks are not all the same."""
    p = te.ChainParams.yaml_defaults(0)
    base = _tip_masks(0.0, 0.0, p)
    cands = [(0.0, 0.0)] + [(x, y) for x in (13.37, -101.23, 1000.01, 0.31, -7.77, 250.125) for y in (-3.21, 77.7, 0.05, 512.39)]
    pos = [cands[0]]
    for c in cands[1:]:
        if len(pos) == NMAPS:
            break
        m = _tip_masks(*c, p)
        if any(not np.array_equal(a, b) for a, b in zip(m, base)):
            pos.append(c)
    assert len(pos) == NMAPS, "no positions found whose on-circle tips differ"
    masks = [_tip_masks(*c, p) for c in pos]
    assert any(not np.array_equal(masks[0][0], mk[0]) for mk in masks[1:]), "row tips never flip"
    assert any(not np.array_equal(masks[0][1], mk[1]) for mk in masks[1:]), "column tips never flip"
    z = np.stack([synth.terrain(ROWS, COLS, RES, 400 + k, "mixed") for k in range(NMAPS)]).astype(np.float32)
    return dict(p=p, g=te.Geometry.make(ROWS, COLS, RES), pos=np.asarray(pos, np.float64), z=z,
                gs=[te.Geometry.make(ROWS, COLS, RES, position=tuple(c)) for c in pos])


@pytest.fixture(params=["fused", "generic"])
def kernel(request, ctx, te):
    """The fused kernel (no fall-back: its per-map mask tables must run) and the generic one."""
    ctx.set_kernel(te.KERNEL_FUSED if request.param == "fused" else te.KERNEL_GENERIC)
    yield request.param
    ctx.set_kernel(te.KERNEL_AUTO)


def _same_as_singles(te, b, singles, idx=None, what=""):
    hb = held(te, b, HELD)
    for k, s in zip(range(NMAPS) if idx is None else idx, singles):
        hs = held(te, s, HELD)
        for name in hs:
            assert np.array_equal(bits(hb[name][k]), bits(hs[name])), (what, k, name)


def _singles(ctx, world, z=None):
    out = []
    for k in range(NMAPS):
        s = ctx.map()
        s.chain(world["gs"][k], world["p"], world["z"][k] if z is None else z[k])
        out.append(s)
    return out


def test_chain_batched_at(world, kernel, te, ctx):
    b = ctx.map()
    got = b.chain_batched(world["g"], world["p"], NMAPS, world["z"], outputs=True, positions=world["pos"])
    assert np.array_equal(b.positions(), world["pos"])
    singles = []
    for k in range(NMAPS):
        s = ctx.map()
        want = s.chain(world["gs"][k], world["p"], world["z"][k], outputs=True)
        for name in CHAIN:
            assert np.array_equal(bits(got[name][k]), bits(want[name])), (kernel, k, name)
        singles.append(s)
    _same_as_singles(te, b, singles, what=kernel)
    # the positions reach the outputs: some map's elevation at map 0's position gives other step bits than at its own
    moved = 0
    for k in range(1, NMAPS):
        s0 = ctx.map()
        at0 = s0.chain(world["gs"][0], world["p"], world["z"][k], outputs=True)
        moved += not np.array_equal(bits(at0["step"]), bits(got["step"][k]))
    assert moved > 0, kernel


def test_footprint_submaps_valid_at(world, te, ctx):
    ft = te.FootprintParams.yaml_defaults()
    b = ctx.map()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=world["pos"])
    singles = _singles(ctx, world)
    # the circular sweep on every map, then on a selection in another order (after clearing)
    cache = b.footprint(ft)
    for k, s in enumerate(singles):
        assert np.array_equal(bits(cache[k]), bits(s.footprint(ft))), k
    b.clear_footprint()
    for s in singles:
        s.clear_footprint()
    idx = [2, 0]
    sel = b.footprint_maps(ft, idx)
    for j, k in enumerate(idx):
        assert np.array_equal(bits(sel[j]), bits(singles[k].footprint(ft))), k
    _same_as_singles(te, b, [singles[k] for k in idx], idx, "footprint_maps")
    # submaps and valid_at around each map's own centre, on interleaved maps
    rng = np.random.default_rng(5)
    n = 48
    wmap = rng.integers(0, NMAPS, n).astype(np.int32)
    xy = world["pos"][wmap] + rng.uniform(-1.5, 1.5, (n, 2)) * np.array([ROWS * RES, COLS * RES]) / 2
    ln = rng.uniform(0.0, 1.5, (n, 2))
    names = ["traversability", "elevation", "traversability_footprint"]
    got = b.get_submaps_batched(wmap, xy, ln, names)
    valid = b.valid_at_batched(wmap, xy)
    assert 0 < valid.sum() < n
    for q in range(n):
        s = singles[wmap[q]]
        (ri, rl), = s.get_submaps(xy[q:q + 1], ln[q:q + 1], names)
        gi, gl = got[q]
        for f in ("success", "rows", "cols", "top_row", "top_col", "requested_row", "requested_col"):
            assert gi[f] == ri[f], (q, f)
        for f in ("length_x", "length_y", "position_x", "position_y"):
            assert np.float64(gi[f]).tobytes() == np.float64(ri[f]).tobytes(), (q, f)
        if rl is not None:
            for name in names:
                assert np.array_equal(bits(gl[name]), bits(rl[name])), (q, name)
        assert valid[q] == s.valid_at(xy[q:q + 1])[0], q


def test_updates_at(world, te, kernel, ctx):
    """chain_maps_at and set_layers_maps_at move only the selected maps; the others keep every bit."""
    p, g = world["p"], world["g"]
    b = ctx.map()
    b.chain_batched(g, p, NMAPS, world["z"])            # every map at g's position
    assert np.array_equal(b.positions(), np.zeros((NMAPS, 2)))
    ft = te.FootprintParams.yaml_defaults()
    b.footprint(ft)
    before = held(te, b, HELD)
    idx = [3, 1]
    z2 = np.stack([synth.terrain(ROWS, COLS, RES, 900 + k, "rough") for k in idx]).astype(np.float32)
    got = b.chain_maps(g, p, idx, z2, outputs=True, positions=world["pos"][idx])
    want_pos = np.zeros((NMAPS, 2))
    want_pos[idx] = world["pos"][idx]
    assert np.array_equal(b.positions(), want_pos)
    after = held(te, b, HELD)
    for k in (0, 2):
        for name in after:
            assert np.array_equal(bits(after[name][k]), bits(before[name][k])), (k, name)
    singles = []
    for j, k in enumerate(idx):
        s = ctx.map()
        want = s.chain(world["gs"][k], p, z2[j], outputs=True)
        for name in CHAIN:
            assert np.array_equal(bits(got[name][j]), bits(want[name])), (k, name)
        singles.append(s)
    _same_as_singles(te, b, singles, idx, "chain_maps_at")
    # set_layers_maps_at: map 0 gets map 3's layers at map 2's position; NULL positions (positions=None) keep g's
    lay = b.get_layers(["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"])
    b.set_layers_maps(g, [0], lay["traversability"][3:4], lay["traversability_slope"][3:4], lay["traversability_step"][3:4],
                      lay["elevation"][3:4], roughness=lay["traversability_roughness"][3:4], positions=world["pos"][2:3])
    want_pos[0] = world["pos"][2]
    assert np.array_equal(b.positions(), want_pos)
    s = ctx.map()
    s.set_layers(world["gs"][2], lay["traversability"][3], lay["traversability_slope"][3], lay["traversability_step"][3],
                 lay["elevation"][3], roughness=lay["traversability_roughness"][3])
    assert np.array_equal(bits(b.footprint_maps(ft, [0])[0]), bits(s.footprint(ft)))
    _same_as_singles(te, b, [s], [0], "set_layers_maps_at")


def test_set_layers_batched_at(world, te, ctx):
    """set_layers_batched_at then the sweep equals single maps; robot_slope and the layers come back as given."""
    b = ctx.map()
    ref = ctx.map()
    out = ref.chain_batched(world["g"], world["p"], NMAPS, world["z"], outputs=True)
    rs = np.where(np.isnan(world["z"]), np.nan, 0.5).astype(np.float32)
    b.set_layers_batched(world["g"], NMAPS, out["traversability"], out["slope"], out["step"], world["z"], roughness=out["roughness"],
                         robot_slope=rs, positions=world["pos"])
    ft = te.FootprintParams.yaml_defaults()
    cache = b.footprint(ft)
    for k in range(NMAPS):
        s = ctx.map()
        s.set_layers(world["gs"][k], out["traversability"][k], out["slope"][k], out["step"][k], world["z"][k],
                     roughness=out["roughness"][k], robot_slope=rs[k])
        assert np.array_equal(bits(cache[k]), bits(s.footprint(ft))), k
    assert np.array_equal(bits(b.get_layers(["robot_slope"])["robot_slope"]), bits(rs))


def test_at_g_position_is_the_existing_entry(world, te, ctx):
    """Positions all equal to g's, and positions None, give the bytes of te_map_chain_batched."""
    ft = te.FootprintParams.yaml_defaults()
    snaps = []
    for mode in ("entry", "null", "g"):
        m = ctx.map()
        if mode == "entry":
            m.chain_batched(world["g"], world["p"], NMAPS, world["z"])
        elif mode == "g":
            m.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=np.zeros((NMAPS, 2)))
        else:   # te_map_chain_batched_at with position_xy NULL
            e = m._batch_layers(world["z"])
            m._check(m._L.te_map_chain_batched_at(m._h, C.byref(world["g"]), C.byref(world["p"]), NMAPS, e.ctypes.data, None, None,
                                                  None, None, te.MEM_HOST, None))
            m._g, m._n = world["g"], NMAPS
        m.footprint(ft)
        snaps.append(held(te, m, HELD))
    for h in snaps[1:]:
        for name in h:
            assert np.array_equal(bits(h[name]), bits(snaps[0][name])), name


def test_requests_at(world, te, ctx):
    """Host requests on interleaved maps (two in a row, so the second reads the first's cache), then a device request: answers,
    untraversable polygons, caches and te_map_request_stats equal those of single-map te_maps at the maps' positions."""
    torch = pytest.importorskip("torch")
    ft = te.FootprintParams.yaml_defaults()
    b = ctx.map()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=world["pos"])
    singles = _singles(ctx, world)
    rng = np.random.default_rng(17)
    for rnd in range(3):
        R = batch_request(rng, world["g"], 40, NMAPS, offsets=world["pos"], circular=0.6, cap_path=False)
        dev = rnd == 2
        if dev:
            fb, fx = footprint_arrays(R, R["fps"])
            n = len(R["kind"])
            t = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device="cuda")  # noqa: E731
            outs = (torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda"),
                    torch.zeros(n, dtype=torch.float64, device="cuda"))
            cnt, uxy = torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros((n, 64, 2), dtype=torch.float64, device="cuda")
            b.check_footprint_request_device(ft, t(R["begin"], torch.int32), t(R["poses"], torch.float64), t(R["radius"], torch.float64),
                                             t(fb, torch.int32), t(fx, torch.float32), *outs, 1 << 16, path_map=t(R["map"], torch.int32),
                                             max_footprint_vertices=16, conservative=t(R["cons"], torch.uint8),
                                             compute_untraversable_polygon=t(R["cup"], torch.uint8), untraversable_capacity=64,
                                             untraversable_count=cnt, untraversable_xy=uxy)
            ctx.synchronize()
            got = [o.cpu().numpy() for o in outs] + [cnt.cpu().numpy(), uxy.cpu().numpy()]
        else:
            got = ask(b, ft, R, R["map"])
        stats = np.zeros(3, np.int64)
        for m in range(NMAPS):
            idx = np.nonzero(R["map"] == m)[0]
            want = ask(singles[m], ft, subset(R, idx))
            stats += np.asarray(singles[m].request_stats())
            for a, w, name in zip(got, want, ("is_safe", "traversability", "area", "count")):
                assert same_bytes(np.asarray(a)[idx], w), (rnd, m, name)
            for j, q in enumerate(idx):
                k = max(0, min(int(want[3][j]), 64))
                assert same_bytes(np.asarray(got[4])[q, :k], want[4][j, :k]), (rnd, m, q)
        assert tuple(stats) == b.request_stats(), rnd
        _same_as_singles(te, b, singles, what=f"request {rnd}")


def test_polygon_sweeps_at(world, te, ctx):
    """The polygon sweep, a list of yaws and its reduction on maps at their own positions equal single maps at those positions."""
    ft = te.FootprintParams.yaml_defaults()
    b = ctx.map()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=world["pos"])
    singles = _singles(ctx, world)
    poly = [(0.11, 0.07), (-0.1, 0.09), (-0.12, -0.08), (0.1, -0.1)]
    yaws = [0.0, 0.4, 1.3, 2.9]
    bx, brot = b.footprint_polygon(ft, poly, 0.7)
    stack = b.footprint_polygon_yaws(ft, poly, yaws)
    worst, best, best_yaw = b.footprint_polygon_yaws_reduce(ft, poly, yaws)
    for m, s in enumerate(singles):
        sx, srot = s.footprint_polygon(ft, poly, 0.7)
        assert np.array_equal(bits(bx[m]), bits(sx)) and np.array_equal(bits(brot[m]), bits(srot)), m
        sstack = s.footprint_polygon_yaws(ft, poly, yaws)
        for k in range(len(yaws)):
            assert np.array_equal(bits(stack[k, m]), bits(sstack[k])), (m, k)
        sw, sb, sy = s.footprint_polygon_yaws_reduce(ft, poly, yaws)
        assert np.array_equal(bits(worst[m]), bits(sw)) and np.array_equal(bits(best[m]), bits(sb)), m
        assert np.array_equal(best_yaw[m], sy), m


def test_uniform_position_serves_every_entry(world, te, ctx):
    """A batch whose maps all sit at one position other than g's answers requests and polygon sweeps as single maps there."""
    ft = te.FootprintParams.yaml_defaults()
    P = world["pos"][1]
    b = ctx.map()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=np.tile(P, (NMAPS, 1)))
    s = ctx.map()
    s.chain(world["gs"][1], world["p"], world["z"][2])
    square = [(0.1, 0.1), (-0.1, 0.1), (-0.1, -0.1), (0.1, -0.1)]
    bx, brot = b.footprint_polygon(ft, square, 0.3)
    sx, srot = s.footprint_polygon(ft, square, 0.3)
    assert np.array_equal(bits(bx[2]), bits(sx)) and np.array_equal(bits(brot[2]), bits(srot))
    rng = np.random.default_rng(9)
    n = 12
    poses = np.zeros((2 * n, 7))
    poses[:, :2] = P + rng.uniform(-0.9, 0.9, (2 * n, 2))
    poses[:, 6] = 1.0
    begin = np.arange(0, 2 * n + 1, 2, dtype=np.int32)
    radius = np.full(n, 0.2)
    fb = np.zeros(n + 1, np.int32)
    got = b.check_footprint_request_batched(ft, np.full(n, 2, np.int32), begin, poses, radius, fb, np.zeros((0, 3), np.float32),
                                            max_footprint_vertices=0)
    want = s.check_footprint_request(ft, begin, poses, radius, fb, np.zeros((0, 3), np.float32), max_footprint_vertices=0)
    for a, w in zip(got, want):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(w).view(np.uint8))
    assert np.array_equal(bits(b.get_footprint()[2]), bits(s.get_footprint()))


def test_errors_leave_the_map_unchanged(world, te, ctx):
    ft = te.FootprintParams.yaml_defaults()
    p, g = world["p"], world["g"]
    b = ctx.map()
    b.chain_batched(g, p, NMAPS, world["z"], positions=world["pos"])
    b.footprint(ft)
    before, pos = held(te, b, HELD), b.positions()

    def expect(code, fn):
        with pytest.raises(te.TEError) as e:
            fn()
        assert e.value.code == code

    bad = world["pos"].copy()
    bad[1, 1] = np.nan
    z1 = world["z"][:1]
    expect(BAD_ARG, lambda: b.chain_batched(g, p, NMAPS, world["z"], positions=bad))
    bad[1] = (np.inf, 0.0)
    expect(BAD_ARG, lambda: b.chain_maps(g, p, [1], z1, positions=bad[1:2]))
    lay = b.get_layers(list(HELD))
    args = [lay[n][:1] for n in ("traversability", "traversability_slope", "traversability_step", "elevation")]
    expect(BAD_ARG, lambda: b.set_layers_maps(g, [1], *args, roughness=lay["traversability_roughness"][:1], positions=bad[1:2]))
    expect(BAD_ARG, lambda: b.chain_maps(te.Geometry.make(ROWS, COLS, 0.021), p, [1], z1, positions=world["pos"][:1]))
    expect(BAD_ARG, lambda: b.chain_maps(g, p, [1, 1], world["z"][:2], positions=world["pos"][:2]))
    assert np.array_equal(b.positions(), pos)
    after = held(te, b, HELD)
    for name in after:
        assert np.array_equal(bits(after[name]), bits(before[name])), name
