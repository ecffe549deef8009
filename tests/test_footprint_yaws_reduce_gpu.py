"""te_footprint_polygon_yaws_reduce and the te_map polygon entries for a list of yaws.  The reductions are defined on top of
te_footprint_polygon_yaws's stack: worst = stack[argmin], best = stack[argmax], best_yaw = argmax over the yaws (numpy's argmin /
argmax return the first index), compared bit for bit."""
import ctypes as C
import math

import numpy as np
import pytest

from test_footprint_yaws_gpu import (LAYERS, POLY, YAWS, _bits, _chain_batch, _fp, _groups, _sms, _tiles, _yaws_host,  # noqa: F401
                                     big)

pytestmark = pytest.mark.gpu
SENTINEL = 7.0


def _reduce(stack):
    """(worst, best, best_yaw) of a stack (nyaws, ...) over its first axis, first index on ties."""
    kmin, kmax = stack.argmin(0), stack.argmax(0)
    worst = np.take_along_axis(stack, kmin[None], 0)[0]
    best = np.take_along_axis(stack, kmax[None], 0)[0]
    return worst, best, kmax.astype(np.int32)


def _outputs(shape, want=(True, True, True)):
    w, b, k = want
    return (np.full(shape, SENTINEL, np.float32) if w else None, np.full(shape, SENTINEL, np.float32) if b else None,
            np.full(shape, -7, np.int32) if k else None)


def _reduce_host(te, ctx, g, p, B, nmaps, yaws, rough, want=(True, True, True), poly=POLY):
    o = _outputs((nmaps,) + B["traversability"].shape[1:], want)
    ctx.footprint_polygon_yaws_reduce(g, p, nmaps, poly, yaws, *(B[k][:nmaps] for k in LAYERS), *o, te.MEM_HOST,
                                      roughness=B["roughness"][:nmaps] if rough else None)
    return o


def _same(got, want):
    for a, b in zip(got, want):
        assert a.dtype == b.dtype
        assert np.array_equal(a.view(np.int32), b.view(np.int32)), int((a.view(np.int32) != b.view(np.int32)).sum())


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("rough", [False, True])
def test_reduce_equals_stack(te, ctx, big, memory, rough):
    """512 x 384 and the seven YAWS (split into yaw groups at this size), verify_roughness off and on, host and device memory."""
    import torch
    g, B = big
    p = _fp(te, 1 if rough else 0)
    assert _groups(_tiles(512, 384, 1), len(YAWS), _sms()) > 1
    want = _reduce(_yaws_host(te, ctx, g, p, B, 1, YAWS, rough))
    if memory == "host":
        got = _reduce_host(te, ctx, g, p, B, 1, YAWS, rough)
    else:
        D = {k: torch.from_numpy(v[:1]).cuda() for k, v in B.items()}
        shape = (1,) + B["traversability"].shape[1:]
        o = (torch.full(shape, SENTINEL, device="cuda"), torch.full(shape, SENTINEL, device="cuda"),
             torch.full(shape, -7, dtype=torch.int32, device="cuda"))
        ctx.set_stream(None)
        ctx.footprint_polygon_yaws_reduce(g, p, 1, POLY, YAWS, *(D[k] for k in LAYERS), *o, te.MEM_DEVICE,
                                          roughness=D["roughness"] if rough else None)
        ctx.synchronize()
        got = tuple(t.cpu().numpy() for t in o)
    _same(got, want)
    worst, best, k = got
    assert (worst == 0).any() and (best > worst).any() and len(np.unique(k)) > 2


def test_batch_of_maps(te, ctx):
    """nmaps = 5 neighbour-contrast maps: map m's reductions are those of its stack."""
    g, B = _chain_batch(te, ctx, 100, 90, 0.02, [0, 1, 2, 3, 0], 500)
    yaws = [0.7854, 0.0, -2.0, math.pi]
    p = _fp(te)
    _same(_reduce_host(te, ctx, g, p, B, 5, yaws, False), _reduce(_yaws_host(te, ctx, g, p, B, 5, yaws, False)))


@pytest.mark.parametrize("nmaps", [1, 5])
def test_yaw_groups(te, ctx, big, nmaps):
    """One 512 x 384 map splits 24 yaws into groups, whose partial results one more kernel folds; five such maps do not split."""
    g, B = big
    yaws = list(np.linspace(0.0, 2 * math.pi, 24, endpoint=False))
    ngroups = _groups(_tiles(512, 384, nmaps), len(yaws), _sms())
    assert (ngroups > 1) if nmaps == 1 else (ngroups == 1)
    p = _fp(te)
    l0 = ctx.stats()[0]
    stack = _yaws_host(te, ctx, g, p, B, nmaps, yaws, False)
    l1 = ctx.stats()[0]
    got = _reduce_host(te, ctx, g, p, B, nmaps, yaws, False)
    l2 = ctx.stats()[0]
    _same(got, _reduce(stack))
    assert l2 - l1 == (l1 - l0) + (1 if ngroups > 1 else 0)


def test_ties(te, ctx, big):
    """Repeated headings tie everywhere: best_yaw is the first of them, and a cell blocked at every heading has
    worst = best = 0 with best_yaw 0."""
    g, B = big
    yaws = [0.5, 0.0, 0.5, 0.0]
    p = _fp(te)
    stack = _yaws_host(te, ctx, g, p, B, 1, yaws, False)
    assert np.array_equal(_bits(stack[0]), _bits(stack[2])) and np.array_equal(_bits(stack[1]), _bits(stack[3]))
    got = _reduce_host(te, ctx, g, p, B, 1, yaws, False)
    _same(got, _reduce(stack))
    worst, best, k = got
    assert set(np.unique(k)) <= {0, 1}
    blocked = (stack == 0).all(0)
    assert blocked.any()
    assert (worst[blocked] == 0).all() and (best[blocked] == 0).all() and (k[blocked] == 0).all()


def test_one_yaw(te, ctx, big):
    g, B = big
    p = _fp(te)
    layer = _yaws_host(te, ctx, g, p, B, 1, [0.4], False)[0]
    worst, best, k = _reduce_host(te, ctx, g, p, B, 1, [0.4], False)
    assert np.array_equal(_bits(worst), _bits(layer)) and np.array_equal(_bits(best), _bits(layer)) and (k == 0).all()


@pytest.mark.parametrize("nmaps", [1, 5])
def test_optional_outputs(te, ctx, big, nmaps):
    """Every non-empty subset of the outputs equals the full call, with and without a yaw-group split."""
    g, B = big
    p = _fp(te)
    full = _reduce_host(te, ctx, g, p, B, nmaps, YAWS, False)
    for want in [(w, b, k) for w in (True, False) for b in (True, False) for k in (True, False) if w or b or k]:
        got = _reduce_host(te, ctx, g, p, B, nmaps, YAWS, False, want)
        for x, y, on in zip(got, full, want):
            assert (x is not None) == on
            if on:
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), (nmaps, want)


def test_1024_yaws(te, ctx):
    """The cap: 1024 yaws on a small map equal the reduction of the stack built in chunks of te_footprint_polygon_yaws calls."""
    g, B = _chain_batch(te, ctx, 100, 90, 0.02, [2], 900)
    yaws = list(np.linspace(-math.pi, math.pi, 1024, endpoint=False))
    p = _fp(te)
    stack = np.concatenate([_yaws_host(te, ctx, g, p, B, 1, yaws[a:a + 256], False) for a in range(0, 1024, 256)])
    worst, best, k = _reduce_host(te, ctx, g, p, B, 1, yaws, False)
    _same((worst, best, k), _reduce(stack))
    assert len(np.unique(k)) > 1


def test_launch_count(te, ctx):
    """Maps with enough tiles for the GPU need no yaw groups: the predicate launches plus one sweep, whatever nyaws and nmaps, as
    te_footprint_polygon_yaws takes.  (A split adds the fold: test_yaw_groups.)"""
    import torch
    rows, cols = 1024, 16 * -(-4 * _sms() // 16)
    assert _groups(_tiles(rows, cols, 1), 64, _sms()) == 1
    g, B = _chain_batch(te, ctx, rows, cols, 0.02, [1, 2, 3, 0, 2], 700)
    D = {k: torch.from_numpy(v).cuda() for k, v in B.items()}
    p = _fp(te)
    ctx.set_stream(None)
    counts, stacked = {}, set()
    for nmaps in (1, 5):
        for nyaws in (1, 7, 64):
            yaws = list(np.linspace(-math.pi, math.pi, nyaws, endpoint=False))
            o = [torch.empty((nmaps,) + B["traversability"].shape[1:], dtype=dt, device="cuda")
                 for dt in (torch.float32, torch.float32, torch.int32)]
            before = ctx.stats()[0]
            ctx.footprint_polygon_yaws_reduce(g, p, nmaps, POLY, yaws, *(D[k][:nmaps] for k in LAYERS), *o, te.MEM_DEVICE)
            counts[(nmaps, nyaws)] = ctx.stats()[0] - before
            out = torch.empty((nyaws, nmaps) + B["traversability"].shape[1:], dtype=torch.float32, device="cuda")
            before = ctx.stats()[0]
            ctx.footprint_polygon_yaws(g, p, nmaps, POLY, yaws, *(D[k][:nmaps] for k in LAYERS), out, te.MEM_DEVICE)
            stacked.add(ctx.stats()[0] - before)
            ctx.synchronize()
            del out
    assert len(stacked) == 1 and set(counts.values()) == stacked, (counts, stacked)


def test_argument_errors(te, ctx):
    rows, cols = 40, 30
    g = te.Geometry.make(rows, cols, 0.02)
    p = _fp(te)
    rng = np.random.default_rng(5)
    lay = [rng.random((1, cols, rows), dtype=np.float32), np.ones((1, cols, rows), np.float32), np.ones((1, cols, rows), np.float32),
           np.zeros((1, cols, rows), np.float32)]

    def call(yaws, want=(True, True, True), **kw):
        o = _outputs((1, cols, rows), want)
        with pytest.raises(te.TEError) as err:
            ctx.footprint_polygon_yaws_reduce(kw.get("g", g), kw.get("p", p), 1, kw.get("poly", POLY), yaws, *lay, *o, te.MEM_HOST)
        for x in o:
            assert x is None or (x.view(np.float32) == SENTINEL).all() or (x == -7).all()   # nothing written
        return err.value.code

    assert call([]) == -1                                           # nyaws < 1
    assert call(list(np.linspace(0.0, 1.0, 1025))) == -4            # nyaws > 1024
    assert call([0.0, float("nan")]) == -1                          # a non-finite yaw
    assert call([float("inf")]) == -1
    assert call([0.0, 1.0], poly=[[1.2, 0.3], [1.2, -0.3], [-1.2, -0.3], [-1.2, 0.3]]) == -4   # reach beyond 31 cells
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = 3, 4
    assert call([0.5], g=gw) == -4                                  # a circular-buffer start index
    assert call([0.5], p=_fp(te, 1)) == -2                          # verify_roughness without the roughness layer
    assert call([0.5], want=(False, False, False)) == -1            # no output
    for bad in (float("nan"), float("inf"), -float("inf")):         # a non-finite traversability_default
        pd = _fp(te)
        pd.traversability_default = bad
        assert call([0.5], p=pd) == -1
    L = ctx._L
    pts = np.ascontiguousarray(POLY, dtype=np.float64)
    ys = np.array([0.0, 1.0, 2.0])
    o = _outputs((1, cols, rows))
    args = lambda yaws_ptr: (ctx._h, C.byref(g), C.byref(p), 1, 4, pts.ctypes.data, 3, yaws_ptr,   # noqa: E731
                             *(a.ctypes.data for a in lay[:3]), None, lay[3].ctypes.data, *(x.ctypes.data for x in o), te.MEM_HOST)
    assert L.te_footprint_polygon_yaws_reduce(*args(None)) == -1    # null yaws
    assert (o[0] == SENTINEL).all() and (o[2] == -7).all()
    assert L.te_footprint_polygon_yaws_reduce(*args(ys.ctypes.data)) == 0
    assert not (o[0] == SENTINEL).any() and set(np.unique(o[2])) <= {0, 1, 2}


def test_map_entries(te, ctx):
    """te_map_footprint_polygon_yaws(_reduce) on the map's layers equal the stateless entries on the same layers.  Host layers
    with a start index give every output, each stacked layer and best_yaw included, re-wrapped to it; device outputs of the same
    map are in default order.  Neither call touches the traversability_footprint cache."""
    import torch
    rows, cols = 200, 150
    g, B = _chain_batch(te, ctx, rows, cols, 0.02, [2], 1100)
    L = {k: np.asfortranarray(v[0].T) for k, v in B.items()}   # (rows, cols) unwrapped
    yaws = [0.3, math.pi / 2, -1.0, 0.0, 2.5]
    p = _fp(te, 1)
    stack = _yaws_host(te, ctx, g, p, B, 1, yaws, True)[:, 0]  # (nyaws, cols, rows)
    want = _reduce(stack)
    sr, sc = 3, 4
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = sr, sc
    wrap = lambda a: np.asfortranarray(np.roll(a, (sr, sc), axis=(0, 1)))   # noqa: E731  stored[(i + sr) % rows, (j + sc) % cols]
    m, mw = ctx.map(), ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"])
    mw.set_layers(gw, *(wrap(L[k]) for k in ("traversability", "slope", "step", "elevation")), roughness=wrap(L["roughness"]))
    fp0 = mw.footprint(p)                                     # fills the cache
    # unwrapped map
    s = m.footprint_polygon_yaws(p, POLY, yaws)
    assert s.shape == (len(yaws), rows, cols)
    assert np.array_equal(_bits(s), _bits(stack.transpose(0, 2, 1)))
    _same(m.footprint_polygon_yaws_reduce(p, POLY, yaws), tuple(w.T for w in want))
    # start index (3, 4), host memory: every layer re-wrapped
    sw = mw.footprint_polygon_yaws(p, POLY, yaws)
    for k in range(len(yaws)):
        assert np.array_equal(_bits(sw[k]), _bits(wrap(stack[k].T))), k
    _same(mw.footprint_polygon_yaws_reduce(p, POLY, yaws), tuple(wrap(w.T) for w in want))
    # the same map in device memory: default order
    ctx.set_stream(None)
    ys = np.ascontiguousarray(yaws, dtype=np.float64)
    pts = np.ascontiguousarray(POLY, dtype=np.float64)
    od = torch.full((len(yaws), cols, rows), SENTINEL, device="cuda")
    rd = (torch.full((cols, rows), SENTINEL, device="cuda"), torch.full((cols, rows), SENTINEL, device="cuda"),
          torch.full((cols, rows), -7, dtype=torch.int32, device="cuda"))
    Lb = ctx._L
    Lb.te_map_footprint_polygon_yaws.argtypes = [C.c_void_p, C.POINTER(te.FootprintParams), C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                                 C.c_void_p, C.c_int]
    Lb.te_map_footprint_polygon_yaws_reduce.argtypes = [C.c_void_p, C.POINTER(te.FootprintParams), C.c_int32, C.c_void_p, C.c_int32,
                                                        C.c_void_p] + [C.c_void_p] * 3 + [C.c_int]
    assert Lb.te_map_footprint_polygon_yaws(mw._h, C.byref(p), len(pts), pts.ctypes.data, len(ys), ys.ctypes.data, od.data_ptr(),
                                            te.MEM_DEVICE) == 0
    assert Lb.te_map_footprint_polygon_yaws_reduce(mw._h, C.byref(p), len(pts), pts.ctypes.data, len(ys), ys.ctypes.data,
                                                   *(t.data_ptr() for t in rd), te.MEM_DEVICE) == 0
    ctx.synchronize()
    assert np.array_equal(_bits(od.cpu().numpy()), _bits(stack))
    _same(tuple(t.cpu().numpy() for t in rd), want)
    # the cache is unchanged by all of them
    assert np.array_equal(mw.get_footprint().view(np.uint32), fp0.view(np.uint32))
    assert np.isnan(m.get_footprint()).all()
    m.close()
    mw.close()
