"""te_map_get_occupancy: GridMapRosConverter::toOccupancyGrid of a te_map's layers, a whole batch or a selection of its maps in one
launch.  Every grid must be, byte for byte, the CPU restatement (tests/occupancy_oracle.cpp) applied to te_map_get_layers' output;
host and device memory must agree; a start index, a batch at several positions, odd shapes and graph capture change nothing."""
import numpy as np
import pytest

import occupancy_oracle as oo
import synth
from helpers import footprint_arrays, mixed_request, request_footprints
from map_helpers import all_layer_names, close_maps  # noqa: F401

pytestmark = pytest.mark.gpu

RES = 0.04
YAML = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness"]  # traversability.yaml
POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]
BAD_ARG, MISSING_LAYER = -1, -2


def _same(got, want, what=""):
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    assert got.dtype == np.int8 and want.dtype == np.int8
    assert np.array_equal(got, want), (what, int((got != want).sum()))


def _dev_occupancy(torch, m, names, lo, hi, maps=None, offset=0):
    """get_occupancy in device memory into a canary-filled tensor, `offset` bytes into it (a misaligned output)."""
    rows, cols = m._shape()
    n = m.nmaps if maps is None else len(maps)
    buf = torch.full((len(names) * n * rows * cols + offset + 3,), 77, dtype=torch.int8, device="cuda")
    res = m.get_occupancy(names, lo, hi, maps=maps, out=buf[offset:offset + len(names) * n * rows * cols], memory=1)
    torch.cuda.synchronize()
    host = buf.cpu().numpy()
    assert (host[:offset] == 77).all() and (host[-3:] == 77).all()
    return {k: v.cpu().numpy() for k, v in res.items()}


def _noisy(rng, shape, nan=0.05):
    a = rng.uniform(-0.2, 1.2, shape).astype(np.float32)
    a[rng.random(shape) < nan] = np.nan
    return a


def _set(te, ctx, g, rng, n=None, positions=None, start_index=None):
    """A te_map of random layers (values around 0..1 with NaNs) at geometry g, or a batch of n maps."""
    m = ctx.map()
    shape = (g.rows, g.cols) if n is None else (n, g.rows, g.cols)
    t, s, st, e, r = (_noisy(rng, shape) for _ in range(5))
    if n is None:
        m.set_layers(g, t, s, st, e, roughness=r)
    else:
        m.set_layers_batched(g, n, t, s, st, e, roughness=r, positions=positions, start_index=start_index)
    return m


def _oracle_grids(m, names, ranges, start=(0, 0)):
    """The oracle on te_map_get_layers' host output (the maps in their buffer order), per name: (n, rows * cols) or (rows * cols)."""
    L = m.get_layers(names)
    out = {}
    for k, n in enumerate(names):
        lo, hi = ranges[k]
        a = L[n]
        if a.ndim == 2:
            out[n] = oo.occupancy_grid(a, lo, hi, start)
        else:
            si = start if np.ndim(start) == 1 else None
            out[n] = np.stack([oo.occupancy_grid(a[j], lo, hi, si if si is not None else start[j]) for j in range(len(a))])
    return out


# ---- 1. the golden fixture: the four grids of traversability.yaml ----------------------------------------------------------

def test_fixture_yaml_grids(te, ctx, fixture_map):
    md, d = fixture_map
    g = te.Geometry(md["rows"], md["cols"], md["resolution"], md["length_x"], md["length_y"], *md["position"], 0, 0)
    m = ctx.map()
    m.chain(g, te.ChainParams.yaml_defaults(0), d["elevation"])
    got = m.get_occupancy(YAML, 1.0, 0.0)
    want = _oracle_grids(m, YAML, [(1.0, 0.0)] * 4)
    L = m.get_layers(YAML)
    for n in YAML:
        assert got[n].shape == (md["cols"], md["rows"])                # (height, width)
        _same(got[n], want[n], n)
        _same(got[n], oo.occupancy_numpy(L[n], 1.0, 0.0), n)
        assert len(np.unique(got[n])) > 20, n
    # the chain's layers equal the fixture's, so these are the grids of the reference's published map
    _same(got["traversability"], oo.occupancy_grid(d["traversability"], 1.0, 0.0))
    info = te.capi.occupancy_grid_info(g)[0]
    assert (info["width"], info["height"]) == (100, 133) and info["resolution"] == np.float32(0.03)
    assert info["origin_x"] == 0.0 - 0.5 * md["length_x"] and info["origin_y"] == 0.0 - 0.5 * md["length_y"]


# ---- 2. the value sweep, every range --------------------------------------------------------------------------------------

def test_value_sweep(te, ctx):
    torch = pytest.importorskip("torch")
    v = oo.sweep_values()
    rows = 97
    cols = -(-len(v) // rows)
    base = np.zeros(rows * cols, np.float32)
    base[:len(v)] = v
    rng = np.random.default_rng(2)
    lay = [np.asfortranarray(base[rng.permutation(len(base)) if k else np.arange(len(base))].reshape(cols, rows).T) for k in range(5)]
    g = te.Geometry.make(rows, cols, RES)
    m = ctx.map()
    m.set_layers(g, lay[0], lay[1], lay[2], lay[4], roughness=lay[3])
    names = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"]  # lay[j]
    for k in range(0, len(oo.RANGES), 5):
        rg = (oo.RANGES[k:] + oo.RANGES)[:5]
        lo, hi = [r[0] for r in rg], [r[1] for r in rg]
        got = m.get_occupancy(names, lo, hi)
        dev = _dev_occupancy(torch, m, names, lo, hi)
        for j, n in enumerate(names):
            want = oo.occupancy_grid(lay[j], *rg[j])
            _same(got[n], want, (n, rg[j]))
            _same(dev[n], want, (n, rg[j]))
            _same(want, oo.occupancy_numpy(lay[j], *rg[j]), (n, rg[j]))
    assert len(np.unique(m.get_occupancy(["traversability"], 1.0, 0.0)["traversability"])) == 102


# ---- 3. every layer bit, each with its own range ---------------------------------------------------------------------------

def _full_map(te, ctx, rows, cols, start=(0, 0), seed=5, pos=(1.3, -0.7)):
    """A map holding every layer bit: the chain, robot_slope and the carried layers, a cache a request filled in part, and
    traversability_x / _rot.  start: the same map given with that circular-buffer start index."""
    g = te.Geometry.make(rows, cols, RES, pos)
    g.start_row, g.start_col = start
    wrap = lambda a: np.asfortranarray(np.roll(a, start, axis=(0, 1)))  # noqa: E731  unwrapped layer -> buffer order
    z = synth.terrain(rows, cols, RES, seed, "mixed", pos)
    rng = np.random.default_rng(seed)
    m = ctx.map()
    m.chain(g, te.ChainParams.yaml_defaults(0), wrap(z))
    names = ["robot_slope"] + list(te.capi.CARRIED_LAYERS)
    lay = {n: rng.normal(0.5, 0.5, (rows, cols)).astype(np.float32) for n in names}
    for a in lay.values():
        a[rng.random(a.shape) < 0.03] = np.nan
        a[rng.random(a.shape) < 0.01] = np.inf
    m.carry_layers(names, [wrap(a) for a in lay.values()])
    ft = te.FootprintParams.yaml_defaults()
    fps = request_footprints(rng)
    R = mixed_request(rng, te.Geometry.make(rows, cols, RES, pos), 60, fps, cap_path=False)
    fb, fx = footprint_arrays(R, fps)
    m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, max_footprint_vertices=16, conservative=R["cons"])
    m.footprint_polygon_keep(ft, POLY, 0.6)
    return m


def test_every_layer_bit(te, ctx):
    torch = pytest.importorskip("torch")
    m = _full_map(te, ctx, 320, 256)
    names = all_layer_names(te)
    rng = np.random.default_rng(3)
    lo = rng.uniform(-1, 1, len(names)).astype(np.float32)
    hi = (lo + rng.choice([-1.0, 1.0, 2.5], len(names))).astype(np.float32)
    got = m.get_occupancy(names, lo, hi)
    assert list(got) == names
    L = m.get_layers(names)
    cache = L["traversability_footprint"]
    assert np.isfinite(cache).any() and np.isnan(cache).any()
    for k, n in enumerate(names):
        _same(got[n], oo.occupancy_grid(L[n], lo[k], hi[k]), n)
    # ranges follow the names, not the bit order
    perm = rng.permutation(len(names))
    shuffled = m.get_occupancy([names[k] for k in perm], lo[perm], hi[perm])
    for n in names:
        _same(shuffled[n], got[n], n)
    dev = _dev_occupancy(torch, m, names, lo, hi)
    for n in names:
        _same(dev[n], got[n], n)


# ---- 4. batches: whole, selections, positions ------------------------------------------------------------------------------

def test_batch_and_selection_equal_single_maps(te, ctx):
    torch = pytest.importorskip("torch")
    n, rows, cols = 7, 64, 48
    rng = np.random.default_rng(4)
    positions = rng.uniform(-300, 300, (n, 2)).round(3)
    z = np.stack([synth.terrain(rows, cols, RES, 40 + k, "mixed") for k in range(n)]).astype(np.float32)
    g = te.Geometry.make(rows, cols, RES)
    b = ctx.map()
    b.chain_batched(g, te.ChainParams.yaml_defaults(0), n, z, positions=positions)
    lo, hi = [1.0, 1.0, 0.0, 0.2], [0.0, 0.0, 1.0, 0.7]
    whole = b.get_occupancy(YAML, lo, hi)
    assert whole["traversability"].shape == (n, cols, rows)
    sel = [5, 0, 3, 6]
    picked = b.get_occupancy(YAML, lo, hi, maps=sel)
    dwhole = _dev_occupancy(torch, b, YAML, lo, hi)
    dpicked = _dev_occupancy(torch, b, YAML, lo, hi, maps=sel)
    for k in range(n):
        s = ctx.map()
        s.chain(te.Geometry.make(rows, cols, RES, tuple(positions[k])), te.ChainParams.yaml_defaults(0), z[k])
        one = s.get_occupancy(YAML, lo, hi)
        for nm in YAML:
            _same(whole[nm][k], one[nm], (k, nm))
            _same(dwhole[nm][k], one[nm], (k, nm))
            if k in sel:
                _same(picked[nm][sel.index(k)], one[nm], (k, nm))
                _same(dpicked[nm][sel.index(k)], one[nm], (k, nm))
    # a selection of one map of a batch is (1, cols, rows)
    assert b.get_occupancy(["elevation"], 0.0, 1.0, maps=[2])["elevation"].shape == (1, cols, rows)
    # the grids' metadata at each map's own position
    xy = b.positions()
    assert np.array_equal(xy, positions)
    info = te.capi.occupancy_grid_info(g, xy)
    for k in range(n):
        w, h, res, ox, oy = oo.occupancy_info(rows, cols, RES, (g.length_x, g.length_y), xy[k])
        r = info[k]
        assert (r["width"], r["height"], r["origin_x"], r["origin_y"]) == (w, h, ox, oy)
        assert r["resolution"].view(np.uint32) == res.view(np.uint32)


# ---- 5. start indices ------------------------------------------------------------------------------------------------------

def test_start_indices_change_nothing(te, ctx):
    torch = pytest.importorskip("torch")
    n, rows, cols = 5, 45, 38
    rng = np.random.default_rng(5)
    starts = np.array([[0, 0], [rows - 1, 0], [0, cols - 1], [17, 9], [3, 30]], np.int32)
    g = te.Geometry.make(rows, cols, RES)
    lay = [_noisy(rng, (n, rows, cols)) for _ in range(5)]
    plain = ctx.map()
    plain.set_layers_batched(g, n, *lay[:4], roughness=lay[4])
    wrapped = ctx.map()
    buf = [np.stack([np.roll(a[k], tuple(starts[k]), axis=(0, 1)) for k in range(n)]) for a in lay]
    wrapped.set_layers_batched(g, n, *buf[:4], roughness=buf[4], start_index=starts)
    assert np.array_equal(wrapped.start_indices(), starts)
    lo, hi = 1.0, 0.0
    want = plain.get_occupancy(YAML, lo, hi)
    got = wrapped.get_occupancy(YAML, lo, hi)
    oracle = _oracle_grids(wrapped, YAML, [(lo, hi)] * 4, start=starts)   # on the buffer-order layers get_layers returns
    dev = _dev_occupancy(torch, wrapped, YAML, lo, hi)
    sel = [4, 1]
    dsel = _dev_occupancy(torch, wrapped, YAML, lo, hi, maps=sel)
    hsel = wrapped.get_occupancy(YAML, lo, hi, maps=sel)
    for nm in YAML:
        _same(got[nm], want[nm], nm)
        _same(got[nm], oracle[nm], nm)
        _same(dev[nm], want[nm], nm)
        _same(dsel[nm], want[nm][sel], nm)
        _same(hsel[nm], want[nm][sel], nm)
    # a single map whose start index came in g
    gs = te.Geometry.make(rows, cols, RES)
    gs.start_row, gs.start_col = 17, 9
    single = ctx.map()
    single.set_layers(gs, *(buf[j][3] for j in range(4)), roughness=buf[4][3])
    s_occ = single.get_occupancy(YAML, lo, hi)
    s_dev = _dev_occupancy(torch, single, YAML, lo, hi)
    s_sel = single.get_occupancy(YAML, lo, hi, maps=[0])
    s_oracle = _oracle_grids(single, YAML, [(lo, hi)] * 4, start=(17, 9))
    for nm in YAML:
        _same(s_occ[nm], want[nm][3], nm)
        _same(s_dev[nm], want[nm][3], nm)
        _same(s_sel[nm], want[nm][3], nm)
        _same(s_occ[nm], s_oracle[nm], nm)


# ---- 6. device memory and graph capture ------------------------------------------------------------------------------------

def test_graph_capture(te):
    torch = pytest.importorskip("torch")
    c = te.Context(0)
    m = None
    try:
        n, rows, cols = 3, 96, 80
        g = te.Geometry.make(rows, cols, RES, (0.5, -0.25))
        rng = np.random.default_rng(6)
        m = c.map()
        lay = [_noisy(rng, (n, rows, cols)) for _ in range(5)]
        m.set_layers_batched(g, n, *lay[:3], lay[4], roughness=lay[3])        # lay[k]: YAML[k]
        lo, hi = [1.0, 0.0, 0.2, -3.0], [0.0, 1.0, 0.7, 5.0]
        out = torch.empty(4 * n * rows * cols, dtype=torch.int8, device="cuda")
        stream = torch.cuda.Stream()
        c.set_stream(stream.cuda_stream)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            m.get_occupancy(YAML, lo, hi, out=out, memory=te.MEM_DEVICE)       # warm-up
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            m.get_occupancy(YAML, lo, hi, out=out, memory=te.MEM_DEVICE)
        stream.synchronize()
        c.set_stream(None)
        new = [_noisy(rng, (n, rows, cols)) for _ in range(5)]
        m.set_layers_batched(g, n, *new[:3], new[4], roughness=new[3])      # in place: the same geometry keeps the buffers
        out.fill_(55)
        c.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        replayed = out.cpu().numpy()
        fresh = m.get_occupancy(YAML, lo, hi)
        _same(replayed, np.concatenate([fresh[nm].reshape(-1) for nm in YAML]))
        for k, nm in enumerate(YAML):
            want = np.stack([oo.occupancy_grid(new[k][j], lo[k], hi[k]) for j in range(n)])
            _same(fresh[nm], want, nm)
    finally:
        if m is not None:
            m.close()                                                      # before its context
        c.close()


# ---- 7. odd shapes and misaligned blocks -----------------------------------------------------------------------------------

@pytest.mark.parametrize("rows,cols,n", [(1, 1, 1), (1, 37, 1), (37, 1, 1), (33, 35, 1), (33, 35, 5), (1, 1, 9), (3, 1, 6),
                                         (2, 3, 4), (65, 63, 3)])
def test_odd_shapes(te, ctx, rows, cols, n):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(rows * 1000 + cols * 10 + n)
    g = te.Geometry.make(rows, cols, RES)
    m = _set(te, ctx, g, rng, None if n == 1 else n)
    names = ["traversability", "elevation"]
    lo, hi = [1.0, 0.0], [0.0, 1.0]
    got = m.get_occupancy(names, lo, hi)
    want = _oracle_grids(m, names, list(zip(lo, hi)))
    for nm in names:
        _same(got[nm], want[nm], nm)
        for off in (0, 1, 2, 3):
            _same(_dev_occupancy(torch, m, names, lo, hi, offset=off)[nm], want[nm], (nm, off))
    if n > 1:
        sel = list(rng.permutation(n)[: max(1, n - 2)])
        got = m.get_occupancy(names, lo, hi, maps=sel)
        for nm in names:
            _same(got[nm], want[nm][sel], nm)
            _same(_dev_occupancy(torch, m, names, lo, hi, maps=sel, offset=1)[nm], want[nm][sel], nm)


# ---- 8. errors -------------------------------------------------------------------------------------------------------------

def test_errors_write_nothing(te, ctx):
    L = te.load_library()
    N = 16
    rng = np.random.default_rng(8)
    m = _set(te, ctx, te.Geometry.make(N, N, RES), rng)
    b = _set(te, ctx, te.Geometry.make(N, N, RES), rng, 3)
    empty = ctx.map()
    out = np.full(4 * 3 * N * N, 77, np.int8)
    lo = np.zeros(4, np.float32)
    hi = np.ones(4, np.float32)
    O, LO, HI = out.ctypes.data, lo.ctypes.data, hi.ctypes.data
    T = 1
    idx = lambda *v: np.array(v, np.int32)  # noqa: E731
    keep = [idx(0, 1), idx(0, 0), idx(0, 3), idx(-1), idx(0, 1, 2, 0)]
    cases = [
        ("no layers", empty, 0, None, T, LO, HI, O, 0, BAD_ARG),
        ("empty mask", m, 0, None, 0, LO, HI, O, 0, BAD_ARG),
        ("bit 7", m, 0, None, 1 << 7, LO, HI, O, 0, BAD_ARG),
        ("bit 18", m, 0, None, T | (1 << 18), LO, HI, O, 0, BAD_ARG),
        ("null data_min", m, 0, None, T, None, HI, O, 0, BAD_ARG),
        ("null data_max", m, 0, None, T, LO, None, O, 0, BAD_ARG),
        ("null out", m, 0, None, T, LO, HI, None, 0, BAD_ARG),
        ("memory 2", m, 0, None, T, LO, HI, O, 2, BAD_ARG),
        ("memory -1", b, 0, None, T, LO, HI, O, -1, BAD_ARG),
        ("nsel without map_index", b, 2, None, T, LO, HI, O, 0, BAD_ARG),
        ("map_index with nsel 0", b, 0, keep[0].ctypes.data, T, LO, HI, O, 0, BAD_ARG),
        ("negative nsel", b, -1, keep[0].ctypes.data, T, LO, HI, O, 0, BAD_ARG),
        ("nsel past the batch", b, 4, keep[4].ctypes.data, T, LO, HI, O, 0, BAD_ARG),
        ("duplicate", b, 2, keep[1].ctypes.data, T, LO, HI, O, 0, BAD_ARG),
        ("index past the batch", b, 2, keep[2].ctypes.data, T, LO, HI, O, 0, BAD_ARG),
        ("negative index", b, 1, keep[3].ctypes.data, T, LO, HI, O, 0, BAD_ARG),
        ("robot_slope missing", m, 0, None, T | (1 << 5), LO, HI, O, 0, MISSING_LAYER),
        ("carried layer missing", b, 0, None, 1 << 10, LO, HI, O, 0, MISSING_LAYER),
        ("uncertainty_range without bounds", m, 0, None, 1 << 15, LO, HI, O, 0, MISSING_LAYER),
        ("traversability_x missing", b, 2, keep[0].ctypes.data, 1 << 16, LO, HI, O, 0, MISSING_LAYER),
    ]
    for what, mp, *args, want in cases:
        rc = L.te_map_get_occupancy(mp._h, *args)
        assert rc == want, (what, rc, L.te_last_error().decode())
        assert (out == 77).all(), what
    assert L.te_map_get_occupancy(m._h, 0, None, 0xf, LO, HI, O, 0) == 0 and (out[:4 * N * N] != 77).any()
    with pytest.raises(te.TEError):
        m.get_occupancy(["robot_slope"], 0.0, 1.0)
    with pytest.raises(ValueError):
        m.get_occupancy(["traversability", "elevation"], [0.0, 1.0, 2.0], 1.0)


def test_one_launch_per_call(te, ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(9)
    b = _set(te, ctx, te.Geometry.make(40, 30, RES), rng, 4)
    calls = [lambda: b.get_occupancy(YAML, 1.0, 0.0), lambda: b.get_occupancy(["elevation"], 0.0, 1.0, maps=[3, 1]),
             lambda: _dev_occupancy(torch, b, YAML, 1.0, 0.0), lambda: _dev_occupancy(torch, b, YAML, 1.0, 0.0, maps=[2])]
    for f in calls:
        f()
        n0 = ctx.stats()[0]
        f()
        assert ctx.stats()[0] - n0 == 1


# ---- 9. one 8192^2 map, four layers ----------------------------------------------------------------------------------------

def test_8192_four_layers(te, ctx):
    N = 8192
    rng = np.random.default_rng(10)
    g = te.Geometry.make(N, N, 0.02)
    lay = []
    for _ in range(5):
        a = np.asfortranarray(rng.random((N, N), dtype=np.float32))
        a[rng.random((N, N), dtype=np.float32) < 0.01] = np.nan
        lay.append(a)
    m = ctx.map()
    m.set_layers(g, lay[0], lay[1], lay[2], lay[4], roughness=lay[3])
    got = m.get_occupancy(YAML, 1.0, 0.0)
    for k, nm in enumerate(YAML):
        assert got[nm].shape == (N, N)
        _same(got[nm], oo.occupancy_grid(lay[k], 1.0, 0.0), nm)
