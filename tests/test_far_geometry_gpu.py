"""The footprint sweeps and the chain's windows at georeferenced map positions (LV95, UTM) and at the origin, with the YAML
footprints and the band footprints of tests/far_geometry.py, against the oracle.  On a traversability layer with a distinct value
per cell and no blocked cell every footprint mean is an exact double sum, so one cell more or less in a footprint shows as a
wrong value: the sweeps must give the oracle's bits there."""
import os

import numpy as np
import pytest

import far_geometry as fg
import paths_oracle as po
import synth
from helpers import assert_parity, chain_layers, close_sweep, same_values

pytestmark = pytest.mark.gpu

ROWS, COLS = 160, 144
POS = ["origin", "lv95", "utm"]


def _geoms(te, oracle, res, pos):
    return te.Geometry.make(ROWS, COLS, res, pos), oracle.Geometry.make(ROWS, COLS, res, pos)


def _distinct(seed):
    one = np.ones((ROWS, COLS), np.float32, order="F")
    return [fg.distinct_layer(ROWS, COLS, seed), one, one.copy(), np.zeros((ROWS, COLS), np.float32, order="F")]


def _chain_layers(oracle, og, res, pos, seed):
    z = synth.terrain(ROWS, COLS, res, seed, "mixed", pos)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    return [np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], z)]


def _circles(res):
    yaml = [(0.30, 0.15)] if res == 0.02 else [(0.15, 0.15)]   # reach 0.45 m is 45 cells at 0.01 m: the fast sweep stops at 31
    return yaml + fg.band_radii(res, (625,) if res == 0.02 else (900, 845))


def _footprint(te, ctx, g, ft, lay, brute):
    if brute:
        os.environ["TE_FOOTPRINT_BRUTE"] = "1"
    try:
        out = np.empty_like(lay[0])
        ctx.footprint(g, ft, *lay, out, te.MEM_HOST)
    finally:
        os.environ.pop("TE_FOOTPRINT_BRUTE", None)
    return out


@pytest.mark.parametrize("res", [0.02, 0.01])
@pytest.mark.parametrize("pos", POS)
def test_circular_sweep_membership(te, ctx, oracle, pos, res):
    g, og = _geoms(te, oracle, res, fg.POSITIONS[pos])
    lay = _distinct(3)
    wrong = {}
    for r, o in _circles(res):
        fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
        fo.radius = ft.radius = r
        fo.offset = ft.offset = o
        ref, _, _ = oracle.footprint(og, fo, *lay)
        for brute in (True, False):
            got = _footprint(te, ctx, g, ft, lay, brute)
            n = int((got != ref).sum())
            if n:
                wrong[(r + o, "brute" if brute else "fast")] = n
        # te_footprint2: the same sweep with checkForRoughness on a roughness layer that blocks nothing
        fo.verify_roughness = ft.verify_roughness = 1
        ref2, _, _, _ = oracle.footprint(og, fo, *lay, roughness=lay[1])
        out = np.empty_like(lay[0])
        ctx.footprint(g, ft, *lay, out, te.MEM_HOST, roughness=lay[1])
        if not same_values(out, ref2):
            wrong[(r + o, "roughness")] = int((out != ref2).sum())
    assert not wrong, wrong


@pytest.mark.parametrize("res", [0.02, 0.01])
@pytest.mark.parametrize("pos", POS)
def test_circular_sweep_on_chain_layers(te, ctx, oracle, pos, res):
    g, og = _geoms(te, oracle, res, fg.POSITIONS[pos])
    lay = _chain_layers(oracle, og, res, fg.POSITIONS[pos], 31)
    for r, o in _circles(res)[::2]:
        fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
        fo.radius = ft.radius = r
        fo.offset = ft.offset = o
        ref, _, _ = oracle.footprint(og, fo, *lay)
        assert same_values(_footprint(te, ctx, g, ft, lay, True), ref), (r + o, "brute")
        assert close_sweep(_footprint(te, ctx, g, ft, lay, False), ref), (r + o, "fast")


def _polygons(res):
    yaml = [(fg.YAML_POLYGON, 0.7854)] if res == 0.02 else [(fg.SMALL_POLYGON, 0.7854)]
    return yaml + fg.band_polygons(res)


@pytest.mark.parametrize("res", [0.02, 0.01])
@pytest.mark.parametrize("pos", POS)
def test_polygon_sweep_membership(te, ctx, oracle, pos, res):
    g, og = _geoms(te, oracle, res, fg.POSITIONS[pos])
    lay = _distinct(4)
    fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
    wrong = {}
    for k, (pts, yaw) in enumerate(_polygons(res)):
        poly = [list(v) for v in pts]
        rx, rrot = oracle.footprint_polygon(og, fo, poly, yaw, *lay)
        ox, orot = np.empty_like(lay[0]), np.empty_like(lay[0])
        ctx.footprint_polygon(g, ft, poly, yaw, *lay, ox, orot, te.MEM_HOST)
        for a, b, name in ((ox, rx, "x"), (orot, rrot, "rot")):
            if not same_values(a, b):
                wrong[(k, name)] = int((a != b).sum())
    assert not wrong, wrong


@pytest.mark.parametrize("res", [0.02, 0.01])
@pytest.mark.parametrize("pos", POS)
def test_polygon_sweep_on_chain_layers(te, ctx, oracle, pos, res):
    g, og = _geoms(te, oracle, res, fg.POSITIONS[pos])
    lay = _chain_layers(oracle, og, res, fg.POSITIONS[pos], 37)
    fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
    for pts, yaw in _polygons(res):
        poly = [list(v) for v in pts]
        rx, rrot = oracle.footprint_polygon(og, fo, poly, yaw, *lay)
        ox, orot = np.empty_like(lay[0]), np.empty_like(lay[0])
        ctx.footprint_polygon(g, ft, poly, yaw, *lay, ox, orot, te.MEM_HOST)
        for a, b in ((ox, rx), (orot, rrot)):
            assert np.array_equal(a == 0, b == 0) and close_sweep(a, b), yaw


@pytest.mark.parametrize("pos", POS)
def test_chain_window_in_the_band(te, ctx, oracle, pos):
    """Normals and roughness radius with r^2 = 8 res^2 (1 - 1.45e-9): the offsets (+-2, +-2) lie just outside the circle, by
    less than the reference's rounding at LV95 / UTM.  Near the origin the fused kernel takes the window; far out it leaves it
    to the generic kernel.  Either way the layers are the oracle's."""
    res, n = 0.02, 256
    p = fg.POSITIONS[pos]
    rn = float(np.sqrt(8 * res * res * (1.0 - 1.45e-9)))
    z = synth.terrain(n, n, res, 77, "mixed", p)
    g, og = te.Geometry.make(n, n, res, p), oracle.Geometry.make(n, n, res, p)
    pt, po = te.ChainParams.yaml_defaults(0), oracle.ChainParams.yaml_defaults(0)
    pt.normals_radius = pt.roughness_radius = po.normals_radius = po.roughness_radius = rn
    ref = oracle.chain(og, po, z)
    assert_parity(ctx.chain_host(g, pt, z), ref)
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        if pos == "origin":
            assert_parity(ctx.chain_host(g, pt, z), ref)
        else:
            with pytest.raises(te.TEError):
                ctx.chain_host(g, pt, z)
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)


# ---- a te_map whose maps sit at their own positions, moved between the origin and far out ------------------------------------

def _oracle_maps(oracle, res, positions, lay, fo):
    return [oracle.footprint(oracle.Geometry.make(ROWS, COLS, res, p), fo, *lay)[0] for p in positions]


@pytest.mark.parametrize("res", [0.02, 0.01])
def test_map_footprint_at_positions(te, ctx, oracle, res):
    """te_map_footprint / te_map_footprint_maps on a batch whose maps start at the origin and then move to LV95 and UTM
    (te_map_set_layers_maps_at): the sweep's tables were built for coordinates near the origin and must be rebuilt for the far
    maps.  Then the polygon sweeps over a list of yaws and their reduction on the far batch."""
    g = te.Geometry.make(ROWS, COLS, res)
    lay = _distinct(6)
    stack = lambda a: np.stack([a] * 3)   # noqa: E731
    m = ctx.map()
    try:
        for r, o in _circles(res)[1:3]:
            fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
            fo.radius = ft.radius = r
            fo.offset = ft.offset = o
            near = [fg.ORIGIN] * 3
            m.set_layers_batched(g, 3, *(stack(a) for a in lay), positions=np.asarray(near))
            got = m.footprint(ft)
            for k, ref in enumerate(_oracle_maps(oracle, res, near, lay, fo)):
                assert same_values(got[k], ref), (r + o, "origin", k)
            far = [fg.LV95, fg.UTM]
            m.set_layers_maps(g, [1, 2], *(np.stack([a] * 2) for a in lay), positions=np.asarray(far))
            got = m.footprint_maps(ft, [1, 2])
            for k, ref in enumerate(_oracle_maps(oracle, res, far, lay, fo)):
                assert same_values(got[k], ref), (r + o, far[k], int((got[k] != ref).sum()))
        positions = [fg.ORIGIN, fg.LV95, fg.UTM]
        m.set_layers_batched(g, 3, *(stack(a) for a in lay), positions=np.asarray(positions))
        fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
        for pts, yaw in fg.band_polygons(res)[:2] + [fg.band_polygons(res)[2]]:
            yaws = [0.0, yaw, 0.3]
            layers = m.footprint_polygon_yaws(ft, pts, yaws)
            worst, best, best_yaw = m.footprint_polygon_yaws_reduce(ft, pts, yaws)
            for k, p in enumerate(positions):
                og = oracle.Geometry.make(ROWS, COLS, res, p)
                refs = np.stack([oracle.footprint_polygon(og, fo, [list(v) for v in pts], y, *lay)[1] for y in yaws])
                for q in range(len(yaws)):
                    assert same_values(layers[q, k], refs[q]), (p, yaws[q], int((layers[q, k] != refs[q]).sum()))
                assert same_values(worst[k], refs.min(axis=0)) and same_values(best[k], refs.max(axis=0)), p
                assert np.array_equal(best_yaw[k], np.argmax(refs, axis=0)), p
    finally:
        m.close()


# ---- fresh path checks with band radii, poses on cell centres -----------------------------------------------------------------

@pytest.mark.parametrize("res", [0.02, 0.01])
@pytest.mark.parametrize("pos", POS)
def test_fresh_paths_with_band_radii(te, ctx, oracle, pos, res):
    """te_check_footprint_paths_fresh with per-path radii from the band, every pose on a cell centre: bit for bit the oracle's
    check_request, whose circles are the reference's SpiralIterator on absolute positions."""
    p = fg.POSITIONS[pos]
    og, g = oracle.Geometry.make(ROWS, COLS, res, p), te.Geometry.make(ROWS, COLS, res, p)
    z = synth.terrain(ROWS, COLS, res, 91, "mixed", p)
    L, _ = chain_layers(oracle, og, z, 91)
    X, Y = fg.cell_tables(ROWS, COLS, res, p)
    rng = np.random.default_rng(5)
    radii = [r for r, _ in _circles(res)]
    begin, poses, radius = [0], [], []
    for q in range(120):
        n = int(rng.integers(1, 5))
        i, j = rng.integers(35, ROWS - 35, n), rng.integers(35, COLS - 35, n)
        poses.extend(zip(X[i], Y[j]))
        begin.append(len(poses))
        radius.append(radii[q % len(radii)])
    begin, poses, radius = np.asarray(begin, np.int32), np.asarray(poses, np.float64), np.asarray(radius, np.float64)
    ft, fo = te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults()
    ref_safe, ref_t = po.check_request(og, fo, dict(L, robot_slope=None), begin, poses, radius)[:2]
    safe, t = ctx.check_footprint_paths_fresh(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], begin, poses,
                                              radius)
    assert np.array_equal(safe, ref_safe) and np.array_equal(t.view(np.uint64), ref_t.view(np.uint64))


# ---- the chain's slab halo at a radius just below a whole number of cells --------------------------------------------------

@pytest.mark.parametrize("pos", POS)
def test_chain_halo_far_from_the_origin(te, ctx, oracle, pos):
    """Step radii of 2 cells less 2e-10 m: near the origin the step window reaches 1 cell, at LV95 / UTM the reference's circle
    test on absolute centres admits offset 2 for some centres, so a slab needs 2 + 2 halo columns instead of 1 + 1.  A slab with
    the smaller halo is refused far out; with the larger one it equals the whole map, which equals the oracle."""
    import torch
    res, rows, cols = 0.02, 128, 200
    p = fg.POSITIONS[pos]
    r = 2 * res - 2e-10
    z = synth.terrain(rows, cols, res, 17, "mixed", p)
    g, og = te.Geometry.make(rows, cols, res, p), oracle.Geometry.make(rows, cols, res, p)
    pt, pr = te.ChainParams.yaml_defaults(0), oracle.ChainParams.yaml_defaults(0)
    pt.step_first_radius = pt.step_second_radius = pr.step_first_radius = pr.step_second_radius = r
    assert_parity(ctx.chain_host(g, pt, z), oracle.chain(og, pr, z))
    zd = torch.from_numpy(np.ascontiguousarray(z.T)).cuda()
    ctx.set_stream(None)
    whole = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
    ctx.chain(g, pt, zd, *whole, te.MEM_DEVICE)
    b, e = 80, 140
    need = 2 if pos == "origin" else 4   # the normals window (2 cells) alone near the origin
    for h in (need - 1, need):
        s = te.Slab(b, e - b, h, h)
        outs = [torch.empty((e - b, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
        if h < need:
            with pytest.raises(te.TEError):
                ctx.chain(g, pt, zd[b - h:e + h].contiguous(), *outs, te.MEM_DEVICE, slab=s)
            continue
        ctx.chain(g, pt, zd[b - h:e + h].contiguous(), *outs, te.MEM_DEVICE, slab=s)
        ctx.synchronize()
        for w, o in zip(whole, outs):
            assert torch.equal(w[b:e].view(torch.int32), o.view(torch.int32))


# ---- reads at positions one ulp either side of absolute cell edges --------------------------------------------------------

@pytest.mark.parametrize("res", [0.02, 0.01])
@pytest.mark.parametrize("pos", POS)
def test_reads_at_cell_edges(te, ctx, oracle, pos, res):
    """te_map_valid_at and te_map_at_poses at positions on and one nextafter either side of cell edges computed in absolute
    coordinates (a cell centre plus or minus half a cell): the cell getIndexFromPosition finds, as far_geometry restates it."""
    p = fg.POSITIONS[pos]
    g = te.Geometry.make(ROWS, COLS, res, p)
    t = np.asfortranarray(100.0 * np.arange(ROWS)[:, None] + np.arange(COLS)[None, :], dtype=np.float32)
    t[::3, ::2] = np.nan                                             # valid_at reads finiteness: holes make an index error show
    one = np.ones((ROWS, COLS), np.float32, order="F")
    X, Y = fg.cell_tables(ROWS, COLS, res, p)
    xs, ys = [], []
    for i in range(0, ROWS, 7):
        for e in (X[i] + 0.5 * res, X[i] - 0.5 * res):
            xs += [np.nextafter(e, -np.inf), e, np.nextafter(e, np.inf)]
    for j in range(0, COLS, 7):
        for e in (Y[j] + 0.5 * res, Y[j] - 0.5 * res):
            ys += [np.nextafter(e, -np.inf), e, np.nextafter(e, np.inf)]
    xy = np.array([(x, y) for x in xs[::2] for y in ys[::2]] + [(x, Y[40]) for x in xs] + [(X[40], y) for y in ys], np.float64)
    want_v, want_t = [], []
    for x, y in xy:
        i, j, inside = fg.get_index(ROWS, COLS, res, p, x, y)
        want_t.append(t[i, j] if inside else np.nan)
        want_v.append(int(inside and np.isfinite(t[i, j])))
    m = ctx.map()
    try:
        m.set_layers(g, t, one, one, one * 0)
        assert np.array_equal(m.valid_at(xy), np.asarray(want_v, np.uint8))
        poses = np.concatenate([xy, np.zeros((len(xy), 1)), np.tile([0.0, 0.0, 0.0, 1.0], (len(xy), 1))], axis=1)
        vals, ok = m.at_poses(poses, np.zeros((1, 3), np.float32), ["traversability"])
        got = vals["traversability"][:, 0]
        want = np.asarray(want_t, np.float32)
        assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])
    finally:
        m.close()
