"""te_map_get_point_cloud: GridMapRosConverter::toPointCloud of a te_map's layers, a whole batch or a selection of its maps.  Every
cloud must be, byte for byte, the CPU restatement (tests/point_cloud_oracle.cpp) applied to te_map_get_layers' host output, which
is in each map's buffer order; host and device memory must agree; start indices, positions, selections, odd shapes, the capacity
protocol and graph capture change nothing else."""
import numpy as np
import pytest

import point_cloud_oracle as pco
import synth
from helpers import footprint_arrays, mixed_request, request_footprints
from map_helpers import all_layer_names, close_maps  # noqa: F401

pytestmark = pytest.mark.gpu

RES = 0.04
POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]
BAD_ARG, MISSING_LAYER = -1, -2
CANARY = 0xA5


def _bits(te, names):
    return [0 if n not in te.capi.LAYER_BITS else 1 << te.capi.LAYER_BITS[n] for n in names]


def _want(m, fields, point="elevation", basic=(), nan_layers=(), maps=None):
    """The oracle per map of the call, on te_map_get_layers' host output (buffer order) with the map's start index and position."""
    g = m._g
    need = sorted({f for f in fields if f not in nan_layers} | {point} | set(basic))
    L = m.get_layers(need)
    starts, pos = m.start_indices(), m.positions()
    idx = range(m.nmaps) if maps is None else maps
    out = []
    for k in idx:
        lay = {n: (a if m.nmaps == 1 else a[k]) for n, a in L.items()}
        out.append(pco.point_cloud(lay, fields, point, g.resolution, (g.length_x, g.length_y), pos[k], basic=basic,
                                   nan_layers=nan_layers, start=starts[k])[0])
    return out


def _same(got, want, what=""):
    assert len(got) == len(want), what
    for k, (a, b) in enumerate(zip(got, want)):
        a = np.asarray(a).view(np.uint8).reshape(-1)
        assert len(a) == len(b) and np.array_equal(a, b), (what, k, len(a), len(b), int((a[:len(b)] != b[:len(a)]).sum()))


def _host(m, fields, point="elevation", **kw):
    layout, step, clouds = m.get_point_cloud(fields, point, **kw)
    assert step == 4 * len(layout)
    return [c.view(np.uint8).reshape(-1) for c in clouds]


def _dev(torch, m, fields, point="elevation", offset=0, **kw):
    """The clouds in device memory, `offset` bytes into a canary-filled buffer; the canary must stay."""
    _, step, host = m.get_point_cloud(fields, point, **kw)
    n = len(host)
    total = sum(len(c) for c in host)
    buf = torch.full((total * step + offset + 7,), CANARY, dtype=torch.uint8, device="cuda")
    offs = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda")
    m.get_point_cloud(fields, point, out=buf[offset:offset + total * step], offsets=offs, memory=1, **kw)
    torch.cuda.synchronize()
    b, o = buf.cpu().numpy(), offs.cpu().numpy()
    assert (b[:offset] == CANARY).all() and (b[offset + total * step:] == CANARY).all()
    assert o[0] == 0 and o[-1] == total and np.array_equal(np.diff(o), [len(c) for c in host])
    return [b[offset + o[k] * step:offset + o[k + 1] * step] for k in range(n)]


def _noisy(rng, shape, nan=0.05):
    a = rng.uniform(-0.2, 1.2, shape).astype(np.float32)
    a[rng.random(shape) < nan] = np.nan
    return a


def _set(te, ctx, g, rng, n=None, positions=None, start_index=None, nan=0.05):
    m = ctx.map()
    shape = (g.rows, g.cols) if n is None else (n, g.rows, g.cols)
    t, s, st, e, r = (_noisy(rng, shape, nan) for _ in range(5))
    if n is None:
        m.set_layers(g, t, s, st, e, roughness=r)
    else:
        m.set_layers_batched(g, n, t, s, st, e, roughness=r, positions=positions, start_index=start_index)
    return m


FIELDS = ["traversability", "step_footprint", "elevation", "traversability_slope"]  # elevation -> x y z; one NaN field
NAN = ("step_footprint",)


# ---- 1. the fixture as the reference publishes it --------------------------------------------------------------------------

def test_fixture_as_published(te, ctx, fixture_map, tmp_path):
    torch = pytest.importorskip("torch")
    md, d = fixture_map
    msg = pco.fixture_bag(tmp_path)
    g = te.Geometry(md["rows"], md["cols"], md["resolution"], md["length_x"], md["length_y"], *md["position"], 0, 0)
    m = ctx.map()
    m.set_layers(g, d["traversability"], d["traversability_slope"], d["traversability_step"], d["elevation"],
                 roughness=d["traversability_roughness"])
    m.carry_layers(["upper_bound", "lower_bound"], [msg.data["upper_bound"], msg.data["lower_bound"]])
    kw = dict(resolution=msg.resolution, length=(msg.length_x, msg.length_y), position=msg.pose[:2])
    want, n = pco.point_cloud(msg.data, msg.layers, "elevation", **kw)
    assert n == 13300 and len(want) == 13300 * 52
    # the memo layers and a fresh map's traversability_footprint are all NaN 0x7fc00000 in the published map
    nan = ("step_footprint", "slope_footprint", "traversability_footprint")
    layout, step, clouds = m.get_point_cloud(msg.layers, "elevation", nan_layers=nan)
    assert step == 52 and [o for _, o in layout] == list(range(0, 52, 4)) and len(clouds[0]) == 13300
    _same([clouds[0].view(np.uint8)], [want], "host")
    _same(_dev(torch, m, msg.layers, nan_layers=nan), [want], "device")
    assert clouds[0]["x"][0] == np.float32(1.485) and clouds[0]["z"][5] == d["elevation"][5, 0]
    # the cache as the field: the oracle on get_layers' cache (empty cells are NaN 0xffffffff there)
    _same(_host(m, msg.layers, nan_layers=nan[:2]), _want(m, msg.layers, nan_layers=nan[:2]), "cache field")


# ---- 2. every layer bit as a field and as the point layer, and basic layers -------------------------------------------------

def _full_map(te, ctx, rows, cols, seed=5, pos=(1.3, -0.7), specials=True):
    """A map holding every layer bit: the chain, robot_slope and the carried layers with NaN payloads, -0.0 and +-Inf, a cache a
    request filled in part, and traversability_x / _rot."""
    g = te.Geometry.make(rows, cols, RES, pos)
    z = synth.terrain(rows, cols, RES, seed, "mixed", pos)
    rng = np.random.default_rng(seed)
    m = ctx.map()
    m.chain(g, te.ChainParams.yaml_defaults(0), z)
    names = ["robot_slope"] + list(te.capi.CARRIED_LAYERS)
    lay = {n: rng.normal(0.5, 0.5, (rows, cols)).astype(np.float32) for n in names}
    if specials:
        for a in lay.values():
            r = rng.random(a.shape)
            a[r < 0.03] = np.nan
            a[(r >= 0.03) & (r < 0.04)] = np.inf
            a[(r >= 0.04) & (r < 0.05)] = -np.inf
            a[(r >= 0.05) & (r < 0.06)] = -0.0
            a.view(np.uint32)[(r >= 0.06) & (r < 0.07)] = 0x7fd00bad
            a.view(np.uint32)[(r >= 0.07) & (r < 0.08)] = 0xffc00001
    m.carry_layers(names, list(lay.values()))
    ft = te.FootprintParams.yaml_defaults()
    fps = request_footprints(rng)
    R = mixed_request(rng, te.Geometry.make(rows, cols, RES, pos), 60, fps, cap_path=False)
    fb, fx = footprint_arrays(R, fps)
    m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, max_footprint_vertices=16, conservative=R["cons"])
    m.footprint_polygon_keep(ft, POLY, 0.6)
    return m


def test_every_layer_bit_as_field(te, ctx):
    torch = pytest.importorskip("torch")
    m = _full_map(te, ctx, 96, 72)
    names = all_layer_names(te)
    rng = np.random.default_rng(1)
    fields = [names[k] for k in rng.permutation(len(names))] + ["memo_a", "memo_b"]
    for point in ("elevation", "upper_bound", "uncertainty_range", "traversability_footprint"):
        want = _want(m, fields, point, nan_layers=("memo_a", "memo_b"))
        got = _host(m, fields, point, nan_layers=("memo_a", "memo_b"))
        _same(got, want, point)
        _same(_dev(torch, m, fields, point, nan_layers=("memo_a", "memo_b")), want, point)
    # the stored bits survive: NaN payloads and -0.0 of a carried layer
    _, _, c = m.get_point_cloud(["elevation", "variance"], "elevation")
    v = c[0]["variance"].view(np.uint32)
    assert (v == 0x7fd00bad).any() and (v == 0xffc00001).any() and (v == 0x80000000).any()


def test_every_layer_bit_as_point_layer(te, ctx):
    torch = pytest.importorskip("torch")
    m = _full_map(te, ctx, 40, 35, seed=7)
    for point in all_layer_names(te):
        for fields in (list(dict.fromkeys(["traversability", point, "variance"])), ["time", "gap"]):
            want = _want(m, fields, point, nan_layers=("gap",))
            _same(_host(m, fields, point, nan_layers=("gap",)), want, (point, fields))
            _same(_dev(torch, m, fields, point, offset=2, nan_layers=("gap",)), want, (point, fields))


def test_basic_layers(te, ctx):
    torch = pytest.importorskip("torch")
    m = _full_map(te, ctx, 50, 44, seed=9)
    for basic in (["variance"], ["variance", "time", "robot_slope"], ["uncertainty_range", "elevation"], ["traversability_footprint"],
                  list(all_layer_names(te))):
        fields = ["elevation", "time", "traversability"]
        want = _want(m, fields, "elevation", basic=basic)
        _same(_host(m, fields, basic=basic), want, basic)
        _same(_dev(torch, m, fields, basic=basic), want, basic)
    n_all = len(_host(m, ["elevation"])[0]) // 12
    n_var = len(_host(m, ["elevation"], basic=["variance"])[0]) // 12
    assert 0 < n_var < n_all


def test_map_without_points(te, ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    b = _set(te, ctx, te.Geometry.make(30, 20, RES), rng, 3)
    e = b.get_layers(["elevation"])["elevation"]
    e[1] = np.nan                                                   # map 1 has no valid cell
    t, s, st, r = (b.get_layers([n])[n] for n in ("traversability", "traversability_slope", "traversability_step",
                                                  "traversability_roughness"))
    b.set_layers_batched(b._g, 3, t, s, st, e, roughness=r)
    got = _host(b, FIELDS, nan_layers=NAN)
    assert len(got[1]) == 0 and len(got[0]) > 0 and len(got[2]) > 0
    want = _want(b, FIELDS, nan_layers=NAN)
    _same(got, want)
    _same(_dev(torch, b, FIELDS, nan_layers=NAN, offset=1), want)


# ---- 3. start indices -----------------------------------------------------------------------------------------------------

def test_start_indices(te, ctx):
    torch = pytest.importorskip("torch")
    n, rows, cols = 5, 45, 38
    rng = np.random.default_rng(5)
    starts = np.array([[0, 0], [rows - 1, 0], [0, cols - 1], [17, 9], [3, 30]], np.int32)
    g = te.Geometry.make(rows, cols, RES, (2.0, -1.0))
    lay = [_noisy(rng, (n, rows, cols), 0.2) for _ in range(5)]
    buf = [np.stack([np.roll(a[k], tuple(starts[k]), axis=(0, 1)) for k in range(n)]) for a in lay]
    w = ctx.map()
    w.set_layers_batched(g, n, *buf[:4], roughness=buf[4], start_index=starts)
    assert np.array_equal(w.start_indices(), starts)
    want = _want(w, FIELDS, nan_layers=NAN)
    _same(_host(w, FIELDS, nan_layers=NAN), want)
    _same(_dev(torch, w, FIELDS, nan_layers=NAN), want)
    sel = [4, 1, 3]
    _same(_host(w, FIELDS, nan_layers=NAN, maps=sel), [want[k] for k in sel])
    _same(_dev(torch, w, FIELDS, nan_layers=NAN, maps=sel, offset=3), [want[k] for k in sel])
    # the order differs from the same map without a start index, the points do not
    plain = ctx.map()
    plain.set_layers_batched(g, n, *lay[:4], roughness=lay[4])
    p = _host(plain, FIELDS, nan_layers=NAN)
    assert p[3].tobytes() != want[3].tobytes()
    assert sorted(p[3].view(np.uint32).reshape(-1, 6).tolist()) == sorted(want[3].view(np.uint32).reshape(-1, 6).tolist())
    # a single map whose start index came in g
    gs = te.Geometry.make(rows, cols, RES, (2.0, -1.0))
    gs.start_row, gs.start_col = 17, 9
    single = ctx.map()
    single.set_layers(gs, *(buf[j][3] for j in range(4)), roughness=buf[4][3])
    _same(_host(single, FIELDS, nan_layers=NAN), [want[3]])
    _same(_dev(torch, single, FIELDS, nan_layers=NAN), [want[3]])
    _same(_host(single, FIELDS, nan_layers=NAN, maps=[0]), [want[3]])


# ---- 4. positions and selections ------------------------------------------------------------------------------------------

def test_positions_and_selections_equal_single_maps(te, ctx):
    torch = pytest.importorskip("torch")
    n, rows, cols = 7, 64, 48
    rng = np.random.default_rng(4)
    positions = rng.uniform(-300, 300, (n, 2)).round(3)
    positions[2] = (2.6e6 + 0.123, 1.2e6 - 0.377)                  # georeferenced
    z = np.stack([synth.terrain(rows, cols, RES, 40 + k, "mixed") for k in range(n)]).astype(np.float32)
    g = te.Geometry.make(rows, cols, RES)
    b = ctx.map()
    b.chain_batched(g, te.ChainParams.yaml_defaults(0), n, z, positions=positions)
    fields = ["traversability", "elevation", "traversability_step"]
    whole = _host(b, fields)
    dwhole = _dev(torch, b, fields)
    _same(whole, _want(b, fields))
    sel = [5, 0, 3, 6]
    picked = _host(b, fields, maps=sel)
    dpicked = _dev(torch, b, fields, maps=sel, offset=1)
    for k in range(n):
        s = ctx.map()
        s.chain(te.Geometry.make(rows, cols, RES, tuple(positions[k])), te.ChainParams.yaml_defaults(0), z[k])
        one = _host(s, fields)
        _same([whole[k], dwhole[k]], one * 2, k)
        if k in sel:
            _same([picked[sel.index(k)], dpicked[sel.index(k)]], one * 2, k)


# ---- 5 and 6. memory modes and capacity -------------------------------------------------------------------------------------

def test_capacity_host(te, ctx):
    L = te.load_library()
    rng = np.random.default_rng(6)
    b = _set(te, ctx, te.Geometry.make(33, 31, RES), rng, 3)
    want = _want(b, FIELDS, nan_layers=NAN)
    step = 24
    total = sum(len(w) for w in want) // step
    fa = np.array(_bits(te, FIELDS), np.uint32)
    E = 1 << 4
    offs = np.full(4, -3, np.int64)
    assert L.te_map_get_point_cloud(b._h, 0, None, 4, fa.ctypes.data, E, 0, None, 0, offs.ctypes.data, 0) == BAD_ARG  # sizing
    assert offs[0] == 0 and offs[-1] == total and np.array_equal(np.diff(offs), [len(w) // step for w in want])
    data = np.full(total * step + 8, CANARY, np.uint8)
    offs[:] = -3
    assert L.te_map_get_point_cloud(b._h, 0, None, 4, fa.ctypes.data, E, 0, data.ctypes.data, total - 1, offs.ctypes.data, 0) == BAD_ARG
    assert offs[-1] == total and (data == CANARY).all()
    assert L.te_map_get_point_cloud(b._h, 0, None, 4, fa.ctypes.data, E, 0, data.ctypes.data, total, offs.ctypes.data, 0) == 0
    assert np.array_equal(data[:total * step], np.concatenate(want)) and (data[total * step:] == CANARY).all()


def test_capacity_device(te, ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(7)
    b = _set(te, ctx, te.Geometry.make(40, 37, RES), rng, 3)
    want = np.concatenate(_want(b, FIELDS, nan_layers=NAN))
    step = 24
    total = len(want) // step
    for cap in (0, 1, total // 2, total - 1, total, total + 5):
        buf = torch.full(((total + 5) * step + 1,), CANARY, dtype=torch.uint8, device="cuda")
        offs = torch.full((4,), -3, dtype=torch.int64, device="cuda")
        b.get_point_cloud(FIELDS, nan_layers=NAN, out=buf[1:], offsets=offs, capacity=cap, memory=1)
        torch.cuda.synchronize()
        h, o = buf.cpu().numpy(), offs.cpu().numpy()
        assert o[0] == 0 and o[-1] == total, cap
        k = min(cap, total) * step
        assert np.array_equal(h[1:1 + k], want[:k]) and (h[1 + k:] == CANARY).all() and h[0] == CANARY, cap
    offs = torch.full((4,), -3, dtype=torch.int64, device="cuda")
    b.get_point_cloud(FIELDS, nan_layers=NAN, out=None, offsets=offs, capacity=0, memory=1)
    torch.cuda.synchronize()
    assert offs.cpu().numpy()[-1] == total


# ---- 7. odd shapes ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rows,cols,n", [(1, 1, 1), (1, 37, 1), (37, 1, 1), (33, 35, 1), (33, 35, 5), (1, 1, 9), (3, 1, 6),
                                         (2, 3, 4), (65, 63, 3), (32, 32, 2), (1025, 1, 2)])
def test_odd_shapes(te, ctx, rows, cols, n):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(rows * 1000 + cols * 10 + n)
    m = _set(te, ctx, te.Geometry.make(rows, cols, RES), rng, None if n == 1 else n, nan=0.2)
    want = _want(m, FIELDS, nan_layers=NAN)
    _same(_host(m, FIELDS, nan_layers=NAN), want)
    for off in (0, 1, 3):
        _same(_dev(torch, m, FIELDS, nan_layers=NAN, offset=off), want, off)
    if n > 1:
        sel = list(rng.permutation(n)[: max(1, n - 2)])
        _same(_host(m, FIELDS, nan_layers=NAN, maps=sel), [want[k] for k in sel])


# ---- 8. errors --------------------------------------------------------------------------------------------------------------

def test_errors_write_nothing(te, ctx):
    L = te.load_library()
    N = 16
    rng = np.random.default_rng(8)
    m = _set(te, ctx, te.Geometry.make(N, N, RES), rng)
    b = _set(te, ctx, te.Geometry.make(N, N, RES), rng, 3)
    empty = ctx.map()
    data = np.full(4 * 3 * N * N * 8, CANARY, np.uint8)
    offs = np.full(5, -3, np.int64)
    D, O, CAP = data.ctypes.data, offs.ctypes.data, 3 * N * N
    idx = lambda *v: np.array(v, np.int32)  # noqa: E731
    keep = [idx(0, 1), idx(0, 0), idx(0, 3), idx(-1)]
    f = lambda *v: np.array(v, np.uint32)   # noqa: E731
    keep_f = [f(1, 16, 0), f(1, 3, 16), f(1, 1 << 7), f(1, 1 << 18), f(1, 1, 16), f(*([1] + [0] * 32)), f(1, 1 << 5), f(1, 1 << 10),
              f(1 << 15), f(1 << 16)]
    F = keep_f[0].ctypes.data
    E = 16
    cases = [
        ("no layers", empty, 0, None, 3, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("nfields 0", m, 0, None, 0, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("nfields 33", m, 0, None, 33, keep_f[5].ctypes.data, E, 0, D, CAP, O, 0, BAD_ARG),
        ("null fields", m, 0, None, 3, None, E, 0, D, CAP, O, 0, BAD_ARG),
        ("null offsets", m, 0, None, 3, F, E, 0, D, CAP, None, 0, BAD_ARG),
        ("null data with room", m, 0, None, 3, F, E, 0, None, CAP, O, 0, BAD_ARG),
        ("negative capacity", m, 0, None, 3, F, E, 0, D, -1, O, 0, BAD_ARG),
        ("two bits in an entry", m, 0, None, 3, keep_f[1].ctypes.data, E, 0, D, CAP, O, 0, BAD_ARG),
        ("bit 7", m, 0, None, 2, keep_f[2].ctypes.data, E, 0, D, CAP, O, 0, BAD_ARG),
        ("bit 18", m, 0, None, 2, keep_f[3].ctypes.data, E, 0, D, CAP, O, 0, BAD_ARG),
        ("repeated bit", m, 0, None, 3, keep_f[4].ctypes.data, E, 0, D, CAP, O, 0, BAD_ARG),
        ("point layer 0", m, 0, None, 3, F, 0, 0, D, CAP, O, 0, BAD_ARG),
        ("point layer two bits", m, 0, None, 3, F, 3, 0, D, CAP, O, 0, BAD_ARG),
        ("point layer bit 7", m, 0, None, 3, F, 1 << 7, 0, D, CAP, O, 0, BAD_ARG),
        ("basic bit 7", m, 0, None, 3, F, E, 1 << 7, D, CAP, O, 0, BAD_ARG),
        ("basic bit 20", m, 0, None, 3, F, E, 1 | (1 << 20), D, CAP, O, 0, BAD_ARG),
        ("memory 2", m, 0, None, 3, F, E, 0, D, CAP, O, 2, BAD_ARG),
        ("memory -1", b, 0, None, 3, F, E, 0, D, CAP, O, -1, BAD_ARG),
        ("nsel without map_index", b, 2, None, 3, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("map_index with nsel 0", b, 0, keep[0].ctypes.data, 3, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("negative nsel", b, -1, keep[0].ctypes.data, 3, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("duplicate", b, 2, keep[1].ctypes.data, 3, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("index past the batch", b, 2, keep[2].ctypes.data, 3, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("negative index", b, 1, keep[3].ctypes.data, 3, F, E, 0, D, CAP, O, 0, BAD_ARG),
        ("robot_slope field missing", m, 0, None, 2, keep_f[6].ctypes.data, E, 0, D, CAP, O, 0, MISSING_LAYER),
        ("carried field missing", b, 0, None, 2, keep_f[7].ctypes.data, E, 0, D, CAP, O, 0, MISSING_LAYER),
        ("point layer missing", m, 0, None, 3, F, 1 << 5, 0, D, CAP, O, 0, MISSING_LAYER),
        ("point uncertainty_range without bounds", m, 0, None, 3, F, 1 << 15, 0, D, CAP, O, 0, MISSING_LAYER),
        ("field uncertainty_range without bounds", m, 0, None, 1, keep_f[8].ctypes.data, E, 0, D, CAP, O, 0, MISSING_LAYER),
        ("basic layer missing", b, 2, keep[0].ctypes.data, 3, F, E, 1 << 12, D, CAP, O, 0, MISSING_LAYER),
        ("traversability_x missing", b, 0, None, 1, keep_f[9].ctypes.data, E, 0, D, CAP, O, 0, MISSING_LAYER),
    ]
    for what, mp, *args, want in cases:
        rc = L.te_map_get_point_cloud(mp._h, *args)
        assert rc == want, (what, rc, L.te_last_error().decode())
        assert (data == CANARY).all() and (offs == -3).all(), what
    assert L.te_map_get_point_cloud(m._h, 0, None, 3, F, E, 0, D, CAP, O, 0) == 0 and (data != CANARY).any() and offs[0] == 0
    with pytest.raises(te.TEError):
        m.get_point_cloud(["robot_slope", "elevation"])
    with pytest.raises(ValueError):
        m.get_point_cloud(["elevation", "no_such_layer"])


# ---- 9. launches ------------------------------------------------------------------------------------------------------------

def test_fixed_launches(te, ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(9)
    b = _set(te, ctx, te.Geometry.make(40, 30, RES), rng, 4, positions=[[0, 0], [1, 1], [2, 2], [3, 3]],
             start_index=[[0, 0], [3, 4], [39, 29], [7, 0]])
    fresh = _set(te, ctx, te.Geometry.make(2000, 300, RES), rng)
    dout = torch.empty(24 * 10 ** 6, dtype=torch.uint8, device="cuda")
    doffs = torch.empty(5, dtype=torch.int64, device="cuda")
    calls = [lambda: b.get_point_cloud(FIELDS, nan_layers=NAN, capacity=10 ** 6),
             lambda: b.get_point_cloud(FIELDS, nan_layers=NAN, capacity=10 ** 6, maps=[3, 1]),
             lambda: fresh.get_point_cloud(FIELDS, nan_layers=NAN, capacity=10 ** 6),
             lambda: b.get_point_cloud(FIELDS, nan_layers=NAN, out=dout, offsets=doffs, memory=1),
             lambda: b.get_point_cloud(FIELDS, nan_layers=NAN, out=dout, offsets=doffs[:2], maps=[2], memory=1),
             lambda: fresh.get_point_cloud(FIELDS, nan_layers=NAN, out=dout, offsets=doffs[:2], memory=1)]
    for fn in calls:
        fn()
        torch.cuda.synchronize()
        n0 = ctx.stats()[0]
        fn()
        assert ctx.stats()[0] - n0 == 3   # the count kernel, the scan, the scatter kernel


# ---- 10. graph capture ------------------------------------------------------------------------------------------------------

def test_graph_capture(te):
    torch = pytest.importorskip("torch")
    c = te.Context(0)
    m = None
    try:
        n, rows, cols = 3, 96, 80
        g = te.Geometry.make(rows, cols, RES, (0.5, -0.25))
        rng = np.random.default_rng(10)
        pos, st = [[0.5, -0.25], [10.0, 3.0], [-4.0, 7.5]], [[0, 0], [5, 70], [95, 1]]
        m = c.map()
        lay = [_noisy(rng, (n, rows, cols), 0.1) for _ in range(5)]
        m.set_layers_batched(g, n, *lay[:4], roughness=lay[4], positions=pos, start_index=st)
        cap = n * rows * cols
        out = torch.full((cap * 24,), CANARY, dtype=torch.uint8, device="cuda")
        offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        stream = torch.cuda.Stream()
        c.set_stream(stream.cuda_stream)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            m.get_point_cloud(FIELDS, nan_layers=NAN, out=out, offsets=offs, memory=te.MEM_DEVICE)   # warm-up
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            m.get_point_cloud(FIELDS, nan_layers=NAN, out=out, offsets=offs, memory=te.MEM_DEVICE)
        stream.synchronize()
        c.set_stream(None)
        new = [_noisy(rng, (n, rows, cols), 0.3) for _ in range(5)]
        m.set_layers_batched(g, n, *new[:4], roughness=new[4], positions=pos, start_index=st)   # same buffers
        out.fill_(CANARY)
        offs.fill_(-1)
        c.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        o = offs.cpu().numpy()
        want = _want(m, FIELDS, nan_layers=NAN)
        assert np.array_equal(np.diff(o), [len(w) // 24 for w in want])
        got = out.cpu().numpy()
        _same([got[:o[-1] * 24]], [np.concatenate(want)])
        assert (got[o[-1] * 24:] == CANARY).all()
    finally:
        if m is not None:
            m.close()
        c.close()


# ---- 11. one 4096^2 map, the published field list --------------------------------------------------------------------------

def test_4096_published(te, ctx):
    N = 4096
    rng = np.random.default_rng(11)
    g = te.Geometry.make(N, N, 0.02, (3.0, -2.0))
    lay = {}
    for nm in ("traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation",
               "upper_bound", "lower_bound"):
        a = np.asfortranarray(rng.random((N, N), dtype=np.float32))
        lay[nm] = a
    lay["elevation"][rng.random((N, N), dtype=np.float32) < 0.01] = np.nan
    m = ctx.map()
    m.set_layers(g, lay["traversability"], lay["traversability_slope"], lay["traversability_step"], lay["elevation"],
                 roughness=lay["traversability_roughness"])
    m.carry_layers(["upper_bound", "lower_bound"], [lay["upper_bound"], lay["lower_bound"]])
    nan = ("step_footprint", "slope_footprint")
    layout, step, clouds = m.get_point_cloud(pco.PUBLISHED, nan_layers=nan)
    assert step == 52 and 0.98 * N * N < len(clouds[0]) < N * N
    _same([clouds[0].view(np.uint8)], _want(m, pco.PUBLISHED, nan_layers=nan))
