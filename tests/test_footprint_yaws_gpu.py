"""te_footprint_polygon_yaws: the polygonal footprint sweep at a whole list of yaws in one call.  Every layer equals, bit for bit,
the traversability_rot of te_footprint_polygon at that yaw on that map alone, and against the oracle it keeps that entry's
tolerance."""
import math

import numpy as np
import pytest

import synth
from helpers import bits, close_sweep, te_footprint_params, walled_terrain

pytestmark = pytest.mark.gpu

POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]                 # robot_footprint_parameter.yaml:3
PENTAGON = [[0.5, 0.2], [0.1, -0.3], [-0.5, -0.2], [-0.4, 0.26], [0.0, 0.1]]
# pi/2 and pi make the rectangle's edges axis-parallel again: long lists of uncertain offsets
YAWS = [0.0, 0.7854, math.pi / 2, -0.3, math.pi, 5.0, 2 * math.pi + 0.1]
LAYERS = ("traversability", "slope", "step", "elevation")


def _groups(tiles, nyaws, sms):
    """The launcher's yaw-group rule (polygon_groups in te_footprint_polygon.cu): as many groups as bring the launch to 4 * sms blocks."""
    return min(nyaws, max(1, -(-4 * sms // tiles)))


def _tiles(rows, cols, nmaps):
    return -(-rows // 64) * -(-cols // 16) * nmaps


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _chain_batch(te, ctx, rows, cols, res, kinds, seed):
    """Chain layers (te_chain_batched) of len(kinds) maps as host arrays (n, cols, rows), with zero patches in slope and roughness
    (checkForSlope and, with verify_roughness, checkForRoughness block them) on every map but the flat ones."""
    import torch
    n = len(kinds)
    g = te.Geometry.make(rows, cols, res)
    z = torch.from_numpy(np.stack([np.ascontiguousarray(walled_terrain(rows, cols, res, k, seed + i).T) for i, k in enumerate(kinds)])).cuda()
    slope, step, rough, trav = (torch.empty_like(z) for _ in range(4))
    ctx.set_stream(None)
    ctx.chain_batched(g, te.ChainParams.yaml_defaults(0), n, z, slope, step, rough, trav, te.MEM_DEVICE)
    ctx.synchronize()
    B = {"traversability": trav.cpu().numpy(), "slope": slope.cpu().numpy(), "step": step.cpu().numpy(),
         "roughness": rough.cpu().numpy(), "elevation": z.cpu().numpy()}
    rng = np.random.default_rng(seed)
    for m, k in enumerate(kinds):
        for _ in range(4 if k else 0):
            a, b = int(rng.integers(0, cols - 10)), int(rng.integers(0, rows - 10))
            B["roughness"][m, a:a + 9, b:b + 9] = 0.0
            a, b = int(rng.integers(0, cols - 10)), int(rng.integers(0, rows - 10))
            B["slope"][m, a:a + 9, b:b + 9] = 0.0
    return g, B


def _single(te, ctx, g, p, B, m, yaw, rough, poly=POLY):
    """te_footprint_polygon on map m alone (host memory): (traversability_x, traversability_rot) as (cols, rows)."""
    x, r = np.empty(B["traversability"].shape[1:], np.float32), np.empty(B["traversability"].shape[1:], np.float32)
    ctx.footprint_polygon(g, p, poly, yaw, *(B[k][m] for k in LAYERS), x, r, te.MEM_HOST,
                          roughness=B["roughness"][m] if rough else None)
    return x, r


def _yaws_host(te, ctx, g, p, B, nmaps, yaws, rough, poly=POLY):
    out = np.full((len(yaws), nmaps) + B["traversability"].shape[1:], 7.0, np.float32)
    ctx.footprint_polygon_yaws(g, p, nmaps, poly, yaws, *(B[k][:nmaps] for k in LAYERS), out, te.MEM_HOST,
                               roughness=B["roughness"][:nmaps] if rough else None)
    return out


@pytest.mark.parametrize("case", [
    dict(rows=160, cols=140, seed=61, res=0.02, poly=POLY),                                     # YAML footprint, 0.30 m = 15 cells
    dict(rows=150, cols=133, seed=62, res=0.03, poly=PENTAGON, position=(57.25, -31.5)),
])
def test_yaws_match_oracle(te, ctx, oracle, case):
    """Every layer against oracle.footprint_polygon(..., yaw)[1]: the zero masks exactly, the values under the sweep's tolerance."""
    res, pos, poly = case["res"], case.get("position", (0.0, 0.0)), case["poly"]
    rows, cols = case["rows"], case["cols"]
    z = synth.terrain(rows, cols, res, case["seed"], "mixed", pos)
    og, g = oracle.Geometry.make(rows, cols, res, pos), te.Geometry.make(rows, cols, res, pos)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    lay = [np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], z)]
    out = np.full((len(YAWS), 1, cols, rows), 7.0, np.float32)
    ctx.footprint_polygon_yaws(g, te.FootprintParams.yaml_defaults(), 1, poly, YAWS, *lay, out, te.MEM_HOST)
    fo = oracle.FootprintParams.yaml_defaults()
    for k, yaw in enumerate(YAWS):
        _, ref = oracle.footprint_polygon(og, fo, poly, yaw, *lay)
        got = out[k, 0].T
        assert not np.isnan(got).any(), yaw
        assert np.array_equal(got == 0, ref == 0), (yaw, int(((got == 0) != (ref == 0)).sum()))
        assert close_sweep(got, ref), (yaw, int((got != ref).sum()), float(np.abs(got - ref).max()))
    assert (out == 0).any() and (out > 0).any()
    assert not np.array_equal(out[0], out[1])


@pytest.fixture(scope="module")
def big(te, ctx):
    """One 512 x 384 terrain map and five of the batch kinds, 512 x 384 each."""
    return _chain_batch(te, ctx, 512, 384, 0.02, [2, 0, 1, 2, 3], 300)


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("rough", [False, True])
def test_yaws_equal_single_entry(te, ctx, big, memory, rough):
    """512 x 384, verify_roughness off and on: every layer is te_footprint_polygon's traversability_rot at that yaw, and the yaw 0
    layer also its traversability_x.  At this size the launcher splits the seven yaws into groups."""
    import torch
    g, B = big
    p = te_footprint_params(te, verify_roughness=1 if rough else 0)
    assert _groups(_tiles(512, 384, 1), len(YAWS), _sms()) > 1
    if memory == "host":
        out = _yaws_host(te, ctx, g, p, B, 1, YAWS, rough)
    else:
        D = {k: torch.from_numpy(v[:1]).cuda() for k, v in B.items()}
        od = torch.full((len(YAWS), 1) + B["traversability"].shape[1:], 7.0, dtype=torch.float32, device="cuda")
        ctx.set_stream(None)
        ctx.footprint_polygon_yaws(g, p, 1, POLY, YAWS, *(D[k] for k in LAYERS), od, te.MEM_DEVICE,
                                   roughness=D["roughness"] if rough else None)
        ctx.synchronize()
        out = od.cpu().numpy()
    for k, yaw in enumerate(YAWS):
        x, r = _single(te, ctx, g, p, B, 0, yaw, rough)
        assert np.array_equal(bits(out[k, 0]), bits(r)), (memory, rough, yaw)
        if yaw == 0.0:
            assert np.array_equal(bits(out[k, 0]), bits(x))
    assert (out == 0).any() and (out > 0).any()
    if rough:   # the zero-roughness patches block cells that are open without the check
        plain = _yaws_host(te, ctx, g, te_footprint_params(te), B, 1, YAWS[:1], False)
        assert (out[0] == 0).sum() > (plain[0] == 0).sum()


def test_batch_of_maps(te, ctx):
    """nmaps = 5 neighbour-contrast maps, four yaws: layer (k, m) is te_footprint_polygon on map m alone."""
    g, B = _chain_batch(te, ctx, 100, 90, 0.02, [0, 1, 2, 3, 0], 500)
    yaws = [0.7854, 0.0, -2.0, math.pi]
    p = te_footprint_params(te)
    out = _yaws_host(te, ctx, g, p, B, 5, yaws, False)
    for m in range(5):
        for k, yaw in enumerate(yaws):
            x, r = _single(te, ctx, g, p, B, m, yaw, False)
            assert np.array_equal(bits(out[k, m]), bits(r)), (m, yaw)
            if yaw == 0.0:
                assert np.array_equal(bits(out[k, m]), bits(x)), m
    assert (out[:, 0] > 0).all() and (out[:, 1] == 0).any() and (out[:, 3] == 0).any()


@pytest.mark.parametrize("nmaps", [1, 5])
def test_yaw_groups(te, ctx, big, nmaps):
    """Both sides of the yaw-group rule give the per-yaw entry's bits: one 512 x 384 map has too few tiles for the GPU and splits
    the 24 yaws into groups; five such maps have enough, and every block sweeps all 24."""
    g, B = big
    yaws = list(np.linspace(0.0, 2 * math.pi, 24, endpoint=False))
    ngroups = _groups(_tiles(512, 384, nmaps), len(yaws), _sms())
    assert (ngroups > 1) if nmaps == 1 else (ngroups == 1)
    p = te_footprint_params(te)
    out = _yaws_host(te, ctx, g, p, B, nmaps, yaws, False)
    for m in range(nmaps):
        for k in (0, 1, 7, 11, 23) if nmaps == 1 else (0, 5, 23):
            _, r = _single(te, ctx, g, p, B, m, yaws[k], False)
            assert np.array_equal(bits(out[k, m]), bits(r)), (nmaps, m, k)


def test_launch_count(te, ctx):
    """The predicate launches plus one sweep, whatever nyaws and nmaps; the two-layer entry takes as many."""
    import torch
    g, B = _chain_batch(te, ctx, 100, 90, 0.02, [1, 2, 3, 0, 2], 700)
    D = {k: torch.from_numpy(v).cuda() for k, v in B.items()}
    p = te_footprint_params(te)
    ctx.set_stream(None)
    counts = {}
    for nmaps in (1, 5):
        for nyaws in (1, 7, 64):
            out = torch.empty((nyaws, nmaps) + B["traversability"].shape[1:], dtype=torch.float32, device="cuda")
            yaws = list(np.linspace(-math.pi, math.pi, nyaws, endpoint=False))
            before = ctx.stats()[0]
            ctx.footprint_polygon_yaws(g, p, nmaps, POLY, yaws, *(D[k][:nmaps] for k in LAYERS), out, te.MEM_DEVICE)
            counts[(nmaps, nyaws)] = ctx.stats()[0] - before
    ctx.synchronize()
    x, r = (torch.empty(B["traversability"].shape[1:], dtype=torch.float32, device="cuda") for _ in range(2))
    before = ctx.stats()[0]
    ctx.footprint_polygon(g, p, POLY, 0.7854, *(D[k][0] for k in LAYERS), x, r, te.MEM_DEVICE)
    single = ctx.stats()[0] - before
    ctx.synchronize()
    assert set(counts.values()) == {single}, (counts, single)


def test_argument_errors(te, ctx):
    import ctypes as C
    rows, cols = 40, 30
    g = te.Geometry.make(rows, cols, 0.02)
    p = te_footprint_params(te)
    rng = np.random.default_rng(5)
    lay = [rng.random((1, cols, rows), dtype=np.float32), np.ones((1, cols, rows), np.float32), np.ones((1, cols, rows), np.float32),
           np.zeros((1, cols, rows), np.float32)]

    def call(yaws, out=None, **kw):
        o = np.full((max(len(yaws), 1), 1, cols, rows), 7.0, np.float32) if out is None else out
        with pytest.raises(te.TEError) as err:
            ctx.footprint_polygon_yaws(kw.get("g", g), kw.get("p", p), 1, kw.get("poly", POLY), yaws, *lay, o, te.MEM_HOST)
        return err.value.code, o

    code, o = call([])                                              # nyaws < 1
    assert code == -1 and (o == 7.0).all()
    code, o = call(list(np.linspace(0.0, 1.0, 1025)))               # nyaws > 1024: unsupported, nothing written
    assert code == -4 and (o == 7.0).all()
    assert call([0.0, float("nan")])[0] == -1                       # a non-finite yaw
    assert call([float("inf")])[0] == -1
    assert call([0.0, 1.0], **{"poly": [[1.2, 0.3], [1.2, -0.3], [-1.2, -0.3], [-1.2, 0.3]]})[0] == -4   # reach beyond 31 cells
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = 3, 4
    assert call([0.5], g=gw)[0] == -4                               # a circular-buffer start index, even for one map and one yaw
    pr = te_footprint_params(te, verify_roughness=1)
    assert call([0.5], p=pr)[0] == -2                               # verify_roughness without the roughness layer
    L = ctx._L
    pts = np.ascontiguousarray(POLY, dtype=np.float64)
    out = np.full((3, 1, cols, rows), 7.0, np.float32)
    ys = np.array([0.0, 1.0, 2.0])
    args = lambda yaws_ptr, out_ptr: (ctx._h, C.byref(g), C.byref(p), 1, 4, pts.ctypes.data, 3, yaws_ptr,   # noqa: E731
                                      *(a.ctypes.data for a in lay[:3]), None, lay[3].ctypes.data, out_ptr, te.MEM_HOST)
    assert L.te_footprint_polygon_yaws(*args(None, out.ctypes.data)) == -1      # null yaws
    assert L.te_footprint_polygon_yaws(*args(ys.ctypes.data, None)) == -1       # null output
    assert (out == 7.0).all()
    assert L.te_footprint_polygon_yaws(*args(ys.ctypes.data, out.ctypes.data)) == 0
    assert not (out == 7.0).any()
