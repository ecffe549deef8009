"""A batched te_map whose maps sit at their own positions (te_map_chain_batched_at, te_map_set_layers_batched_at,
te_map_chain_maps_at, te_map_set_layers_maps_at, te_map_positions).  For every map m, everything the batch returns or holds must
equal, bit for bit (NaN masks included), what a single-map te_map holding map m at its position returns or holds.  The positions
are chosen so that the on-circle step tips of the fused kernel's mask tables differ between maps, which the test checks on the
host with the kernel's own test (d * d + 0.0 <= r^2 on cell-centre coordinate differences)."""
import ctypes as C

import numpy as np
import pytest

import synth
from helpers import footprint_arrays, mixed_request, request_footprints

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


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


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


@pytest.fixture
def maps(ctx):
    made = []

    def new():
        made.append(ctx.map())
        return made[-1]

    yield new
    for m in made:
        m.close()


def _held(m):
    return dict(m.get_layers(list(HELD)), cache=m.get_footprint())


def _same_as_singles(b, singles, idx=None, what=""):
    hb = _held(b)
    for k, s in zip(range(NMAPS) if idx is None else idx, singles):
        hs = _held(s)
        for name in hs:
            assert np.array_equal(_bits(hb[name][k]), _bits(hs[name])), (what, k, name)


def _singles(maps, world, z=None):
    out = []
    for k in range(NMAPS):
        s = maps()
        s.chain(world["gs"][k], world["p"], world["z"][k] if z is None else z[k])
        out.append(s)
    return out


def test_chain_batched_at(maps, world, kernel):
    b = maps()
    got = b.chain_batched(world["g"], world["p"], NMAPS, world["z"], outputs=True, positions=world["pos"])
    assert np.array_equal(b.positions(), world["pos"])
    singles = []
    for k in range(NMAPS):
        s = maps()
        want = s.chain(world["gs"][k], world["p"], world["z"][k], outputs=True)
        for name in CHAIN:
            assert np.array_equal(_bits(got[name][k]), _bits(want[name])), (kernel, k, name)
        singles.append(s)
    _same_as_singles(b, singles, what=kernel)
    # the positions reach the outputs: some map's elevation at map 0's position gives other step bits than at its own
    moved = 0
    for k in range(1, NMAPS):
        s0 = maps()
        at0 = s0.chain(world["gs"][0], world["p"], world["z"][k], outputs=True)
        moved += not np.array_equal(_bits(at0["step"]), _bits(got["step"][k]))
    assert moved > 0, kernel


def test_footprint_submaps_valid_at(maps, world, te):
    ft = te.FootprintParams.yaml_defaults()
    b = maps()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=world["pos"])
    singles = _singles(maps, world)
    # the circular sweep on every map, then on a selection in another order (after clearing)
    cache = b.footprint(ft)
    for k, s in enumerate(singles):
        assert np.array_equal(_bits(cache[k]), _bits(s.footprint(ft))), k
    b.clear_footprint()
    for s in singles:
        s.clear_footprint()
    idx = [2, 0]
    sel = b.footprint_maps(ft, idx)
    for j, k in enumerate(idx):
        assert np.array_equal(_bits(sel[j]), _bits(singles[k].footprint(ft))), k
    _same_as_singles(b, [singles[k] for k in idx], idx, "footprint_maps")
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
                assert np.array_equal(_bits(gl[name]), _bits(rl[name])), (q, name)
        assert valid[q] == s.valid_at(xy[q:q + 1])[0], q


def test_updates_at(maps, world, te, kernel):
    """chain_maps_at and set_layers_maps_at move only the selected maps; the others keep every bit."""
    p, g = world["p"], world["g"]
    b = maps()
    b.chain_batched(g, p, NMAPS, world["z"])            # every map at g's position
    assert np.array_equal(b.positions(), np.zeros((NMAPS, 2)))
    ft = te.FootprintParams.yaml_defaults()
    b.footprint(ft)
    before = _held(b)
    idx = [3, 1]
    z2 = np.stack([synth.terrain(ROWS, COLS, RES, 900 + k, "rough") for k in idx]).astype(np.float32)
    got = b.chain_maps(g, p, idx, z2, outputs=True, positions=world["pos"][idx])
    want_pos = np.zeros((NMAPS, 2))
    want_pos[idx] = world["pos"][idx]
    assert np.array_equal(b.positions(), want_pos)
    after = _held(b)
    for k in (0, 2):
        for name in after:
            assert np.array_equal(_bits(after[name][k]), _bits(before[name][k])), (k, name)
    singles = []
    for j, k in enumerate(idx):
        s = maps()
        want = s.chain(world["gs"][k], p, z2[j], outputs=True)
        for name in CHAIN:
            assert np.array_equal(_bits(got[name][j]), _bits(want[name])), (k, name)
        singles.append(s)
    _same_as_singles(b, singles, idx, "chain_maps_at")
    # set_layers_maps_at: map 0 gets map 3's layers at map 2's position; NULL positions (positions=None) keep g's
    lay = b.get_layers(["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"])
    b.set_layers_maps(g, [0], lay["traversability"][3:4], lay["traversability_slope"][3:4], lay["traversability_step"][3:4],
                      lay["elevation"][3:4], roughness=lay["traversability_roughness"][3:4], positions=world["pos"][2:3])
    want_pos[0] = world["pos"][2]
    assert np.array_equal(b.positions(), want_pos)
    s = maps()
    s.set_layers(world["gs"][2], lay["traversability"][3], lay["traversability_slope"][3], lay["traversability_step"][3],
                 lay["elevation"][3], roughness=lay["traversability_roughness"][3])
    assert np.array_equal(_bits(b.footprint_maps(ft, [0])[0]), _bits(s.footprint(ft)))
    _same_as_singles(b, [s], [0], "set_layers_maps_at")


def test_set_layers_batched_at(maps, world, te):
    """set_layers_batched_at then the sweep equals single maps; robot_slope and the layers come back as given."""
    b = maps()
    ref = maps()
    out = ref.chain_batched(world["g"], world["p"], NMAPS, world["z"], outputs=True)
    rs = np.where(np.isnan(world["z"]), np.nan, 0.5).astype(np.float32)
    b.set_layers_batched(world["g"], NMAPS, out["traversability"], out["slope"], out["step"], world["z"], roughness=out["roughness"],
                         robot_slope=rs, positions=world["pos"])
    ft = te.FootprintParams.yaml_defaults()
    cache = b.footprint(ft)
    for k in range(NMAPS):
        s = maps()
        s.set_layers(world["gs"][k], out["traversability"][k], out["slope"][k], out["step"][k], world["z"][k],
                     roughness=out["roughness"][k], robot_slope=rs[k])
        assert np.array_equal(_bits(cache[k]), _bits(s.footprint(ft))), k
    assert np.array_equal(_bits(b.get_layers(["robot_slope"])["robot_slope"]), _bits(rs))


def test_at_g_position_is_the_existing_entry(maps, world, te):
    """Positions all equal to g's, and positions None, give the bytes of te_map_chain_batched."""
    ft = te.FootprintParams.yaml_defaults()
    held = []
    for mode in ("entry", "null", "g"):
        m = maps()
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
        held.append(_held(m))
    for h in held[1:]:
        for name in h:
            assert np.array_equal(_bits(h[name]), _bits(held[0][name])), name


def _request(rng, world, te, npaths):
    """A mixed request whose paths visit every map in no order, each around its own map's position."""
    fps = request_footprints(rng)
    R = mixed_request(rng, world["g"], npaths, fps, circular=0.6, cap_path=False)
    R["fps"] = fps
    R["map"] = rng.integers(0, NMAPS, len(R["kind"])).astype(np.int32)
    R["map"][:NMAPS] = rng.permutation(NMAPS)
    for q, m in enumerate(R["map"]):
        R["poses"][R["begin"][q]:R["begin"][q + 1], :2] += world["pos"][m]
    return R


def _ask(m, ft, R, path_map=None):
    fb, fx = footprint_arrays(R, R["fps"])
    kw = dict(max_footprint_vertices=16, conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=64)
    if path_map is None:
        return m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, **kw)
    return m.check_footprint_request_batched(ft, path_map, R["begin"], R["poses"], R["radius"], fb, fx, **kw)


def _subset(R, idx):
    b = R["begin"]
    begin = np.concatenate([[0], np.cumsum(b[idx + 1] - b[idx])]).astype(np.int32)
    poses = np.concatenate([R["poses"][b[q]:b[q + 1]] for q in idx]) if len(idx) else np.zeros((0, 7))
    return dict(begin=begin, poses=poses, fps=R["fps"], **{k: R[k][idx] for k in ("radius", "kind", "cons", "cup", "map")})


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_requests_at(maps, world, te, ctx):
    """Host requests on interleaved maps (two in a row, so the second reads the first's cache), then a device request: answers,
    untraversable polygons, caches and te_map_request_stats equal those of single-map te_maps at the maps' positions."""
    torch = pytest.importorskip("torch")
    ft = te.FootprintParams.yaml_defaults()
    b = maps()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=world["pos"])
    singles = _singles(maps, world)
    rng = np.random.default_rng(17)
    for rnd in range(3):
        R = _request(rng, world, te, 40)
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
            got = _ask(b, ft, R, R["map"])
        stats = np.zeros(3, np.int64)
        for m in range(NMAPS):
            idx = np.nonzero(R["map"] == m)[0]
            want = _ask(singles[m], ft, _subset(R, idx))
            stats += np.asarray(singles[m].request_stats())
            for a, w, name in zip(got, want, ("is_safe", "traversability", "area", "count")):
                assert _same(np.asarray(a)[idx], w), (rnd, m, name)
            for j, q in enumerate(idx):
                k = max(0, min(int(want[3][j]), 64))
                assert _same(np.asarray(got[4])[q, :k], want[4][j, :k]), (rnd, m, q)
        assert tuple(stats) == b.request_stats(), rnd
        _same_as_singles(b, singles, what=f"request {rnd}")


def test_polygon_sweeps_at(maps, world, te):
    """The polygon sweep, a list of yaws and its reduction on maps at their own positions equal single maps at those positions."""
    ft = te.FootprintParams.yaml_defaults()
    b = maps()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=world["pos"])
    singles = _singles(maps, world)
    poly = [(0.11, 0.07), (-0.1, 0.09), (-0.12, -0.08), (0.1, -0.1)]
    yaws = [0.0, 0.4, 1.3, 2.9]
    bx, brot = b.footprint_polygon(ft, poly, 0.7)
    stack = b.footprint_polygon_yaws(ft, poly, yaws)
    worst, best, best_yaw = b.footprint_polygon_yaws_reduce(ft, poly, yaws)
    for m, s in enumerate(singles):
        sx, srot = s.footprint_polygon(ft, poly, 0.7)
        assert np.array_equal(_bits(bx[m]), _bits(sx)) and np.array_equal(_bits(brot[m]), _bits(srot)), m
        sstack = s.footprint_polygon_yaws(ft, poly, yaws)
        for k in range(len(yaws)):
            assert np.array_equal(_bits(stack[k, m]), _bits(sstack[k])), (m, k)
        sw, sb, sy = s.footprint_polygon_yaws_reduce(ft, poly, yaws)
        assert np.array_equal(_bits(worst[m]), _bits(sw)) and np.array_equal(_bits(best[m]), _bits(sb)), m
        assert np.array_equal(best_yaw[m], sy), m


def test_uniform_position_serves_every_entry(maps, world, te):
    """A batch whose maps all sit at one position other than g's answers requests and polygon sweeps as single maps there."""
    ft = te.FootprintParams.yaml_defaults()
    P = world["pos"][1]
    b = maps()
    b.chain_batched(world["g"], world["p"], NMAPS, world["z"], positions=np.tile(P, (NMAPS, 1)))
    s = maps()
    s.chain(world["gs"][1], world["p"], world["z"][2])
    square = [(0.1, 0.1), (-0.1, 0.1), (-0.1, -0.1), (0.1, -0.1)]
    bx, brot = b.footprint_polygon(ft, square, 0.3)
    sx, srot = s.footprint_polygon(ft, square, 0.3)
    assert np.array_equal(_bits(bx[2]), _bits(sx)) and np.array_equal(_bits(brot[2]), _bits(srot))
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
    assert np.array_equal(_bits(b.get_footprint()[2]), _bits(s.get_footprint()))


def test_errors_leave_the_map_unchanged(maps, world, te):
    ft = te.FootprintParams.yaml_defaults()
    p, g = world["p"], world["g"]
    b = maps()
    b.chain_batched(g, p, NMAPS, world["z"], positions=world["pos"])
    b.footprint(ft)
    before, pos = _held(b), b.positions()

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
    after = _held(b)
    for name in after:
        assert np.array_equal(_bits(after[name]), _bits(before[name])), name
