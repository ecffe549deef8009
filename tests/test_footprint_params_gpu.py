"""The footprint sweeps against the oracle away from the YAML parameters: the circular sweep (k_sweep_fast on prefix sums, k_sweep
in visit order) and the polygonal sweep (k_poly_tile) at both radius norms, a zero inner radius, the largest reaches each kernel
takes, polygons of every shape they accept, and traversability_default, max_gap_width and critical_step_height away from the YAML.

Chain layers block nearly every disk at large radii, so most cases also run on built layers where one cell more or less in a
footprint shows: a traversability with a distinct value per cell (far_geometry.distinct_layer), about one invalid cell in 400, and
isolated zero-slope blockers that block alone with max_gap_width 0.001 (checkForSlope's critical count floor(2 gap / res) is then
0), spaced so that the first blocked cell of many disks falls on either side of the inner radius.  Every case asserts that it can
fail: the oracle's layer holds zeros and finite non-zero values, non-finite values under a non-finite default, and, where the case
is about the ring factor, values that differ from the unblocked mean."""
import functools
import math
import os

import numpy as np
import pytest

import far_geometry as fg
from footprint_cases import BUILT_GAP, LAYERS, built_map, chain_map, unblocked
from helpers import YAML, close_sweep, same_bits_or_nan, same_values, te_footprint_params

pytestmark = pytest.mark.gpu

INF, NAN = float("inf"), float("nan")
DEFAULTS = [0.0, 1.0, -0.5, 0.3, NAN, INF, -INF]
ERR_BAD_ARG, ERR_UNSUPPORTED = -1, -4


def geoms(te, oracle, m, res):
    rows, cols = m["traversability"].shape
    return te.Geometry.make(rows, cols, res), oracle.Geometry.make(rows, cols, res)


# ---- the circular sweep --------------------------------------------------------------------------------------------------------

def sweep(te, ctx, g, ft, m, brute):
    """te_footprint2 in host memory: (traversability_footprint, slope_footprint, step_footprint, roughness_footprint)."""
    if brute:
        os.environ["TE_FOOTPRINT_BRUTE"] = "1"
    try:
        out = [np.full(m["traversability"].shape, 7.0, np.float32, order="F") for _ in range(4)]
        ctx.footprint(g, ft, *(m[k] for k in LAYERS), out[0], te.MEM_HOST, slope_fp=out[1], step_fp=out[2],
                      roughness=m["roughness"], roughness_fp=out[3])
    finally:
        os.environ.pop("TE_FOOTPRINT_BRUTE", None)
    return out


def same_inf(a, b):
    return np.array_equal(np.isposinf(a), np.isposinf(b)) and np.array_equal(np.isneginf(a), np.isneginf(b))


def close(a, b):
    """close_sweep, and the same infinities; a layer that is NaN everywhere matches one that is NaN everywhere."""
    if np.isnan(b).all():
        return bool(np.isnan(a).all())
    return close_sweep(a, b) and same_inf(a, b)


def check_circle(te, ctx, oracle, m, res, kw, fast=True):
    """Brute (bit for bit) and fast (close_sweep) te_footprint2 against oracle.footprint with parameters kw; the memo layers bit
    for bit.  Returns the oracle's layer."""
    g, og = geoms(te, oracle, m, res)
    ft, fo = te_footprint_params(te, **kw), te_footprint_params(oracle, **kw)
    ref = oracle.footprint(og, fo, *(m[k] for k in LAYERS), roughness=m["roughness"])
    for brute in (True, False) if fast else (True,):
        got = sweep(te, ctx, g, ft, m, brute)
        what = (kw, "brute" if brute else "fast")
        assert (same_values if brute else close)(got[0], ref[0]) and same_inf(got[0], ref[0]), (what, int((got[0] != ref[0]).sum()))
        for k, name in ((1, "slope"), (2, "step"), (3, "roughness"))[:3 if kw.get("verify_roughness") else 2]:
            assert same_bits_or_nan(got[k], ref[k]), (what, name)
    return ref[0]


def nonvacuous(ref, default=0.3, differs_from=None):
    """The layer can fail: zeros, finite non-zero values, non-finite values of the default's kind when it is not finite, and
    finite non-zero values other than `differs_from` (the unblocked result) when given."""
    f = np.isfinite(ref)
    assert (ref[f] == 0).sum() > 0 and (ref[f] != 0).sum() > 0, (int((ref[f] == 0).sum()), int((ref[f] != 0).sum()))
    if math.isnan(default):
        assert np.isnan(ref).sum() > 0
    elif math.isinf(default):
        assert (ref == default).sum() > 0
    if differs_from is not None:
        assert (f & (ref != 0) & (ref != differs_from)).sum() > 0


def oracle_circle(oracle, m, res, kw):
    og = oracle.Geometry.make(*m["traversability"].shape, res)
    return oracle.footprint(og, te_footprint_params(oracle, **kw), *(m[k] for k in LAYERS))[0]


def lattice_reach(rmax, res):
    """The largest |offset| of the circular sweep's tables: offsets inside the circle or on it within the tables' tolerance."""
    return max(max(abs(k), abs(l)) for (k, l), c in fg.circle_classes(rmax, res).items() if c != "out")


@pytest.mark.parametrize("offset", [0.15, 0.0])
@pytest.mark.parametrize("norm", [1, 0])
@pytest.mark.parametrize("res", [0.02, 0.03])
def test_radius_norm(te, ctx, oracle, res, norm, offset):
    """radius_is_integer_norm decides the ring of the first blocked cell (k_sweep_fast's early out and its ring walk)."""
    kw = dict(radius=0.30, offset=offset, radius_is_integer_norm=norm)
    m = built_map(res, spacing=40)
    ref = check_circle(te, ctx, oracle, m, res, dict(kw, **BUILT_GAP))
    nonvacuous(ref, differs_from=oracle_circle(oracle, unblocked(m), res, dict(kw, **BUILT_GAP)) if offset else None)
    if offset:   # the norms give different layers here
        other = oracle_circle(oracle, m, res, dict(kw, radius_is_integer_norm=1 - norm, **BUILT_GAP))
        assert (np.nan_to_num(other, nan=-1) != np.nan_to_num(ref, nan=-1)).sum() > 0
    nonvacuous(check_circle(te, ctx, oracle, chain_map(oracle, res), res, kw))


@pytest.mark.parametrize("radius,offset", [(0.0, 0.3), (0.0, 0.0)])
def test_zero_radius(te, ctx, oracle, radius, offset):
    """radius 0: any blocked cell in the disk gives 0 (rmin == 0); radius = offset = 0: the disk is the cell itself."""
    kw = dict(radius=radius, offset=offset)
    m = built_map()
    ref = check_circle(te, ctx, oracle, m, 0.02, dict(kw, **BUILT_GAP))
    nonvacuous(ref)
    if offset == 0.0:
        t = m["traversability"]
        want = np.where(m["slope"] == 0, np.float32(0), np.where(np.isfinite(t), t, np.float32(0.3)))
        assert np.array_equal(ref, want)
    nonvacuous(check_circle(te, ctx, oracle, chain_map(oracle), 0.02, kw))


def reach_radii(cells, res=0.02):
    """(radius, offset) with radius + offset = `cells` cells exactly, and ceil(rmax / res) == ceil(cells)."""
    rmax = cells * res
    while math.ceil(rmax / res) > math.ceil(cells):
        rmax = float(np.nextafter(rmax, 0.0))
    return rmax - 0.5 * rmax, 0.5 * rmax


# cells, map size, blocker spacing, table reach (None: above 31, brute only)
REACH = [(30, 160, 48, 30), (31, 160, 48, 31), (32.5, 160, 52, 32), (60, 128, 96, None), (120, 128, 192, None)]


@pytest.mark.parametrize("cells,n,spacing,L", REACH, ids=[f"{c}cells" for c, *_ in REACH])
def test_reach(te, ctx, oracle, cells, n, spacing, L):
    """The fast sweep at its largest reach (L = 31 fills k_fp_nearest's 63-row window and the 64-entry tables) and the brute
    sweep to its 120-cell limit; half the reach is the inner radius."""
    radius, offset = reach_radii(cells)
    if L is not None:
        assert lattice_reach(radius + offset, 0.02) == L
    kw = dict(radius=radius, offset=offset, **BUILT_GAP)
    m = built_map(0.02, n, n, spacing, 5)
    ref = check_circle(te, ctx, oracle, m, 0.02, kw, fast=L is not None and L <= 31)
    nonvacuous(ref, differs_from=oracle_circle(oracle, unblocked(m), 0.02, kw))


def test_reach_beyond_120_cells_is_refused(te, ctx, oracle):
    m = built_map(0.02, 128, 128, 192, 5)
    g, _ = geoms(te, oracle, m, 0.02)
    radius, offset = reach_radii(121)
    with pytest.raises(te.TEError) as err:
        sweep(te, ctx, g, te_footprint_params(te, radius=radius, offset=offset), m, False)
    assert err.value.code == ERR_UNSUPPORTED


@pytest.mark.parametrize("default", DEFAULTS, ids=[f"default={d}" for d in DEFAULTS])
def test_circle_default(te, ctx, oracle, default):
    """traversability_default of the invalid cells a disk visits; a NaN or infinite one reaches only those disks."""
    kw = dict(traversability_default=default)
    nonvacuous(check_circle(te, ctx, oracle, built_map(), 0.02, dict(kw, **BUILT_GAP)), default)
    nonvacuous(check_circle(te, ctx, oracle, chain_map(oracle), 0.02, kw), default)


FILTERS = [dict(max_gap_width=v) for v in (0.001, 0.05, 0.3, 1.0)] + [dict(critical_step_height=v) for v in (0.05, 0.12, 0.3)]


@pytest.mark.parametrize("verify", [0, 1])
@pytest.mark.parametrize("kw", FILTERS, ids=[f"{k}={v}" for d in FILTERS for k, v in d.items()])
def test_circle_filters(te, ctx, oracle, kw, verify):
    """max_gap_width and critical_step_height change the predicate pass (k_pred_heavy) and so the blocked cells."""
    nonvacuous(check_circle(te, ctx, oracle, chain_map(oracle), 0.02, dict(kw, verify_roughness=verify)))


# ---- the polygonal sweep -------------------------------------------------------------------------------------------------------

def regular(nv, r, phase):
    return [(r * math.cos(phase + 2 * math.pi * k / nv), r * math.sin(phase + 2 * math.pi * k / nv)) for k in range(nv)]


SHAPES = {
    "triangle": [(0.35, 0.0), (-0.2, 0.25), (-0.15, -0.3)],
    "16-gon": regular(16, 0.33, 0.1),
    # a notch from +y: the columns it crosses hold two runs
    "notch": [(0.4, 0.3), (0.4, -0.3), (-0.4, -0.3), (-0.4, 0.3), (-0.1, 0.3), (-0.1, -0.05), (0.1, -0.05), (0.1, 0.3)],
    "yaml-cw": [v[:2] for v in YAML],
    "yaml-ccw": [v[:2] for v in YAML[::-1]],
    "reach31": [(0.5, 0.3), (0.5, -0.3), (-0.5, -0.3), (-0.5, 0.3)],     # largest vertex norm 29.15 cells at 0.02 m
}
EMPTY = [(0.004, 0.004), (0.009, 0.004), (0.004, 0.009)]                # covers no cell centre at any yaw of YAWS
REACH32 = [(0.5, 0.35), (0.5, -0.35), (-0.5, -0.35), (-0.5, 0.35)]     # 30.5 cells
YAWS = [0.0, math.pi / 2, math.pi, 3 * math.pi / 2, -math.pi / 2]
YAML_YAWS = [0.0, 0.7854]


def polygon(te, ctx, g, ft, pts, yaw, m):
    ox, orot = (np.full(m["traversability"].shape, 7.0, np.float32, order="F") for _ in range(2))
    ctx.footprint_polygon(g, ft, pts, yaw, *(m[k] for k in LAYERS), ox, orot, te.MEM_HOST, roughness=m["roughness"])
    return ox, orot


def check_polygon(te, ctx, oracle, m, pts, yaws, kw, res=0.02):
    """te_footprint_polygon against oracle.footprint_polygon at every yaw: blocked cells and NaN exactly, the others within
    close_sweep.  Returns the oracle's traversability_rot layers."""
    g, og = geoms(te, oracle, m, res)
    ft, fo = te_footprint_params(te, **kw), te_footprint_params(oracle, **kw)
    refs = []
    for yaw in yaws:
        rx, rrot = oracle.footprint_polygon(og, fo, pts, yaw, *(m[k] for k in LAYERS), roughness=m["roughness"])
        ox, orot = polygon(te, ctx, g, ft, pts, yaw, m)
        for a, b, name in ((ox, rx, "x"), (orot, rrot, "rot")):
            what = (kw, yaw, name)
            assert np.array_equal(a == 0, b == 0) and close(a, b), (what, int((a != b).sum()))
        refs.append(rrot)
    return refs


def shape_yaws(name):
    return YAML_YAWS if name.startswith("yaml") else YAWS


@pytest.mark.parametrize("name", list(SHAPES))
def test_polygon_shapes(te, ctx, oracle, name):
    pts = SHAPES[name]
    if name == "reach31":
        assert fg.polygon_reach(pts, 0.02) == 31
    if name == "notch":   # a column offset with two runs of certain cells
        cls = fg.polygon_classes(pts, 0.0, 0.02)
        runs = {}
        for dj in {dj for _, dj in cls}:
            col = [cls[(di, dj)] == "in" for di in sorted({di for di, _ in cls})]
            runs[dj] = sum(1 for k in range(len(col)) if col[k] and (k == 0 or not col[k - 1]))
        assert max(runs.values()) == 2
    m = built_map(spacing=56)
    for ref in check_polygon(te, ctx, oracle, m, pts, shape_yaws(name), BUILT_GAP):
        nonvacuous(ref)
    for ref in check_polygon(te, ctx, oracle, chain_map(oracle), pts, shape_yaws(name)[:2], {}):
        nonvacuous(ref)


@pytest.mark.parametrize("default", [0.3, NAN])
def test_polygon_covering_no_cell_centre(te, ctx, oracle, default):
    """n == 0: the layer is the default everywhere."""
    m = built_map()
    for ref in check_polygon(te, ctx, oracle, m, EMPTY, YAWS, dict(BUILT_GAP, traversability_default=default)):
        assert same_values(ref, np.full(ref.shape, default, np.float32))


def test_polygon_reach_32_is_refused(te, ctx, oracle):
    assert fg.polygon_reach(REACH32, 0.02) == 32
    m = built_map()
    g, _ = geoms(te, oracle, m, 0.02)
    with pytest.raises(te.TEError) as err:
        polygon(te, ctx, g, te_footprint_params(te), REACH32, 0.0, m)
    assert err.value.code == ERR_UNSUPPORTED


@pytest.mark.parametrize("default", DEFAULTS, ids=[f"default={d}" for d in DEFAULTS])
def test_polygon_default(te, ctx, oracle, default):
    kw = dict(traversability_default=default)
    for name in ("yaml-cw", "notch"):
        for ref in check_polygon(te, ctx, oracle, built_map(spacing=56), SHAPES[name], shape_yaws(name)[:2], dict(kw, **BUILT_GAP)):
            nonvacuous(ref, default)
    for ref in check_polygon(te, ctx, oracle, chain_map(oracle), SHAPES["yaml-cw"], YAML_YAWS, kw):
        nonvacuous(ref, default)


@pytest.mark.parametrize("verify", [0, 1])
@pytest.mark.parametrize("kw", FILTERS, ids=[f"{k}={v}" for d in FILTERS for k, v in d.items()])
def test_polygon_filters(te, ctx, oracle, kw, verify):
    for ref in check_polygon(te, ctx, oracle, chain_map(oracle), SHAPES["yaml-cw"], YAML_YAWS, dict(kw, verify_roughness=verify)):
        nonvacuous(ref)


# ---- the other entries, on a subset of the cases -------------------------------------------------------------------------------

R31 = reach_radii(31)
SUBSET = {   # circle parameters, polygon, polygon parameters
    "nan-default": (dict(traversability_default=NAN, **BUILT_GAP), SHAPES["yaml-cw"], dict(traversability_default=NAN, **BUILT_GAP)),
    "L31": (dict(radius=R31[0], offset=R31[1], **BUILT_GAP), SHAPES["triangle"], dict(BUILT_GAP)),
    "Lp31": (dict(BUILT_GAP), SHAPES["reach31"], dict(BUILT_GAP)),
    "norm0": (dict(radius_is_integer_norm=0, **BUILT_GAP), SHAPES["notch"], dict(traversability_default=-INF, **BUILT_GAP)),
}
NMAPS = 3


def batch_maps():
    return [built_map(spacing=48, seed=10 + k) for k in range(NMAPS)]


def stacked(maps, name):
    """(nmaps, cols, rows): map k's layer column-major at k * rows * cols."""
    return np.stack([np.ascontiguousarray(mm[name].T) for mm in maps])


def assert_bits(a, b, what):
    assert same_bits_or_nan(a, b), (what, int((a != b).sum()))


@pytest.mark.parametrize("case", list(SUBSET))
def test_batched_and_map_entries_equal_the_single_map(te, ctx, oracle, case):
    """te_footprint_batched, te_map_footprint, te_footprint_polygon_batched, te_footprint_polygon_yaws and
    te_map_footprint_polygon_keep give the single-map entries' layers bit for bit."""
    ckw, pts, pkw = SUBSET[case]
    maps = batch_maps()
    g, _ = geoms(te, oracle, maps[0], 0.02)
    rows, cols = maps[0]["traversability"].shape
    fc, fpp = te_footprint_params(te, **ckw), te_footprint_params(te, **pkw)
    one = [sweep(te, ctx, g, fc, mm, False)[0] for mm in maps]
    B = {k: stacked(maps, k) for k in LAYERS + ("roughness",)}
    out = np.full((NMAPS, cols, rows), 7.0, np.float32)
    ctx.footprint_batched(g, fc, NMAPS, *(B[k] for k in LAYERS), out, te.MEM_HOST, roughness=B["roughness"])
    for k in range(NMAPS):
        assert_bits(out[k].T, one[k], (case, "te_footprint_batched", k))
    yaw = 0.7854
    singles = [polygon(te, ctx, g, fpp, pts, yaw, mm) for mm in maps]
    ox, orot = (np.full((NMAPS, cols, rows), 7.0, np.float32) for _ in range(2))
    ctx.footprint_polygon_batched(g, fpp, NMAPS, pts, yaw, *(B[k] for k in LAYERS), ox, orot, te.MEM_HOST, roughness=B["roughness"])
    for k in range(NMAPS):
        assert_bits(ox[k].T, singles[k][0], (case, "polygon_batched x", k))
        assert_bits(orot[k].T, singles[k][1], (case, "polygon_batched rot", k))
    yaws = [0.0, yaw, -math.pi / 2]
    stack = np.full((len(yaws), NMAPS, cols, rows), 7.0, np.float32)
    ctx.footprint_polygon_yaws(g, fpp, NMAPS, pts, yaws, *(B[k] for k in LAYERS), stack, te.MEM_HOST, roughness=B["roughness"])
    for q, y in enumerate(yaws):
        for k in range(NMAPS):
            assert_bits(stack[q, k].T, polygon(te, ctx, g, fpp, pts, y, maps[k])[1], (case, "polygon_yaws", y, k))
    m = ctx.map()
    try:
        m.set_layers_batched(g, NMAPS, *(np.stack([mm[k] for mm in maps]) for k in LAYERS),
                             roughness=np.stack([mm["roughness"] for mm in maps]))
        got = m.footprint(fc)
        for k in range(NMAPS):
            assert_bits(got[k], one[k], (case, "te_map_footprint", k))
        kx, krot = m.footprint_polygon_keep(fpp, pts, yaw, outputs=True)
        for k in range(NMAPS):
            assert_bits(kx[k], singles[k][0], (case, "te_map_footprint_polygon_keep x", k))
            assert_bits(krot[k], singles[k][1], (case, "te_map_footprint_polygon_keep rot", k))
    finally:
        m.close()


def circle_halo(kw, res=0.02):
    p = {"radius": 0.30, "offset": 0.15, "max_gap_width": 0.3, **kw}
    return math.ceil((p["radius"] + p["offset"]) / res) + max(4, 3 + 1 + math.ceil(p["max_gap_width"] / res) + 1)


def polygon_halo(kw, pts, res=0.02):
    p = {"max_gap_width": 0.3, **kw}
    return fg.polygon_reach(pts, res) + max(4, 3 + 1 + math.ceil(p["max_gap_width"] / res) + 1)


@pytest.mark.parametrize("case", list(SUBSET))
def test_two_slabs_at_the_exact_halo(te, ctx, oracle, case):
    """max_gap_width 1.0: the gap walk sets the halo.  Two slabs with exactly the halo the entry demands equal the whole map bit
    for bit; one halo column fewer is refused."""
    ckw, pts, pkw = SUBSET[case]
    ckw, pkw = dict(ckw, max_gap_width=1.0), dict(pkw, max_gap_width=1.0)
    m = built_map(0.02, 128, 2 * 96, 48, 7)
    g, _ = geoms(te, oracle, m, 0.02)
    rows, cols = m["traversability"].shape
    fc, fpp = te_footprint_params(te, **ckw), te_footprint_params(te, **pkw)
    whole_c = sweep(te, ctx, g, fc, m, False)[0]
    whole_p = polygon(te, ctx, g, fpp, pts, 0.7854, m)
    b = cols // 2
    for halo, run in ((circle_halo(ckw), "circle"), (polygon_halo(pkw, pts), "polygon")):
        assert halo < b
        for lo, hi, hl, hr in ((0, b, 0, halo), (b, cols, halo, 0)):
            for short in (False, True):
                s = te.Slab(lo, hi - lo, hl - (short and hl > 0), hr - (short and hr > 0))
                a, e = lo - s.halo_left, hi + s.halo_right
                lay = {k: np.asfortranarray(m[k][:, a:e]) for k in LAYERS + ("roughness",)}
                outs = [np.full((rows, hi - lo), 7.0, np.float32, order="F") for _ in range(2)]
                if run == "circle":
                    call = lambda: ctx.footprint(g, fc, *(lay[k] for k in LAYERS), outs[0], te.MEM_HOST, slab=s,  # noqa: E731
                                                 roughness=lay["roughness"])
                else:
                    call = lambda: ctx.footprint_polygon(g, fpp, pts, 0.7854, *(lay[k] for k in LAYERS), outs[0], outs[1],  # noqa: E731
                                                         te.MEM_HOST, slab=s, roughness=lay["roughness"])
                if short:
                    with pytest.raises(te.TEError) as err:
                        call()
                    assert err.value.code == ERR_BAD_ARG, (case, run, lo)
                    continue
                call()
                if run == "circle":
                    assert_bits(outs[0], whole_c[:, lo:hi], (case, run, lo))
                else:
                    assert_bits(outs[0], whole_p[0][:, lo:hi], (case, "x", lo))
                    assert_bits(outs[1], whole_p[1][:, lo:hi], (case, "rot", lo))


def test_parameter_switches_on_one_context_and_map(te, ctx, oracle):
    """The spiral and the tables are cached under the geometry and parameters: A, B, A on one context and on one te_map give what
    a fresh context gives, bit for bit.  The te_map's layers are set again before each circular sweep: its traversability_footprint
    cache keeps a cached cell's value whatever the parameters (te_map_footprint), as the reference's does; new layers empty the
    cache and leave the spiral and the tables as they were."""
    m = built_map()
    g, _ = geoms(te, oracle, m, 0.02)
    seq = ["nan-default", "L31", "nan-default", "norm0", "Lp31", "norm0", "nan-default"]
    fresh = {}
    for case in dict.fromkeys(seq):
        ckw, pts, pkw = SUBSET[case]
        c = te.Context(0)
        try:
            fresh[case] = (sweep(te, c, g, te_footprint_params(te, **ckw), m, False)[0],
                           polygon(te, c, g, te_footprint_params(te, **pkw), pts, 0.7854, m))
        finally:
            c.close()
    mp = ctx.map()
    try:
        mp.set_layers(g, *(m[k] for k in LAYERS), roughness=m["roughness"])
        for case in seq:
            ckw, pts, pkw = SUBSET[case]
            fc, fpp = te_footprint_params(te, **ckw), te_footprint_params(te, **pkw)
            wc, (wx, wrot) = fresh[case]
            assert_bits(sweep(te, ctx, g, fc, m, False)[0], wc, (case, "context circle"))
            ox, orot = polygon(te, ctx, g, fpp, pts, 0.7854, m)
            assert_bits(ox, wx, (case, "context x"))
            assert_bits(orot, wrot, (case, "context rot"))
            mp.set_layers(g, *(m[k] for k in LAYERS), roughness=m["roughness"])
            assert_bits(mp.footprint(fc), wc, (case, "map circle"))
            kx, krot = mp.footprint_polygon_keep(fpp, pts, 0.7854, outputs=True)
            assert_bits(kx, wx, (case, "map x"))
            assert_bits(krot, wrot, (case, "map rot"))
    finally:
        mp.close()
