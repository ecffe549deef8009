"""GPU parity of the circular footprint sweep (TraversabilityMap::traversabilityFootprint) against the oracle."""
import numpy as np
import pytest

import synth
from helpers import close_sweep, same_values

pytestmark = pytest.mark.gpu


def _run(te, ctx, oracle, g, og, layers, fp_t, fp_o):
    import os
    t, s, st, e = (np.asfortranarray(x, dtype=np.float32) for x in layers)
    ref, rs, rt = oracle.footprint(og, fp_o, t, s, st, e)
    res = []
    for brute in (True, False):
        if brute:
            os.environ["TE_FOOTPRINT_BRUTE"] = "1"   # the visit-by-visit kernel: bit-exact by construction
        else:
            os.environ.pop("TE_FOOTPRINT_BRUTE", None)
        out = np.empty_like(t)
        sfp = np.empty_like(t)
        tfp = np.empty_like(t)
        ctx.footprint(g, fp_t, t, s, st, e, out, te.MEM_HOST, slope_fp=sfp, step_fp=tfp)
        res.append((out, sfp, tfp))
    assert same_values(res[0][0], ref), "visit-by-visit sweep differs from the oracle"
    assert close_sweep(res[1][0], ref), ("prefix-sum sweep differs from the oracle", int((res[1][0] != ref).sum()),
                                    float(np.nanmax(np.abs(res[1][0] - ref))))
    return (ref, res[1][1], res[1][2]), (ref, rs, rt)


def test_footprint_on_fixture_layers(te, ctx, oracle, fixture_map):
    m, d = fixture_map
    g = te.Geometry(m["rows"], m["cols"], m["resolution"], m["length_x"], m["length_y"], *m["position"], 0, 0)
    og = oracle.Geometry(m["rows"], m["cols"], m["resolution"], m["length_x"], m["length_y"], *m["position"])
    layers = (d["traversability"], d["traversability_slope"], d["traversability_step"], d["elevation"])
    got, ref = _run(te, ctx, oracle, g, og, layers, te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults())
    for a, b, name in zip(got, ref, ("traversability_footprint", "slope_footprint", "step_footprint")):
        assert same_values(a, b), name
    assert (ref[0] == 0).sum() > 100 and (ref[0] > 0).sum() > 100


@pytest.mark.parametrize("case", [
    dict(rows=160, cols=140, seed=21, res=0.02, offset=0.15),
    dict(rows=160, cols=140, seed=22, res=0.02, offset=0.0),      # rMax = rMin = 0.3: 12 on-circle offsets
    dict(rows=120, cols=133, seed=23, res=0.03, offset=0.15),
    dict(rows=140, cols=120, seed=24, res=0.02, offset=0.15, position=(123.456, -78.9)),
])
def test_footprint_matches_oracle_on_chain_outputs(te, ctx, oracle, case):
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og = oracle.Geometry.make(case["rows"], case["cols"], res, pos)
    g = te.Geometry.make(case["rows"], case["cols"], res, pos)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
    fo.offset = ft.offset = case["offset"]
    got, ref = _run(te, ctx, oracle, g, og, (ch["traversability"], ch["slope"], ch["step"], z), ft, fo)
    for a, b, name in zip(got, ref, ("traversability_footprint", "slope_footprint", "step_footprint")):
        assert same_values(a, b), (name, int((np.isnan(a) != np.isnan(b)).sum()), float(np.nanmax(np.abs(a - b))))
    assert (ref[0] == 0).any() and (ref[0] > 0).any()
    assert np.isfinite(ref[2]).sum() > 0  # step == 0 cells exist, so the gap walk was exercised


def test_footprint_slabs_equal_whole_map(te, ctx, oracle):
    """Multi-GPU tiling of the sweep: a column slab with a 43-column halo gives exactly the whole-map result."""
    import torch
    rows, cols = 128, 300
    z = synth.terrain(rows, cols, 0.02, 41, "mixed")
    og = oracle.Geometry.make(rows, cols, 0.02)
    g = te.Geometry.make(rows, cols, 0.02)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    fp = te.FootprintParams.yaml_defaults()
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32).T)).cuda()  # noqa: E731
    lay = [dev(ch["traversability"]), dev(ch["slope"]), dev(ch["step"]), dev(z)]
    ctx.set_stream(None)
    whole = torch.empty((cols, rows), dtype=torch.float32, device="cuda")
    ctx.footprint(g, fp, *lay, whole, te.MEM_DEVICE)
    ctx.synchronize()
    H = 43
    for b, e in ((0, 140), (140, 300)):
        hl, hr = min(H, b), min(H, cols - e)
        part = [x[b - hl:e + hr].contiguous() for x in lay]
        out = torch.empty((e - b, rows), dtype=torch.float32, device="cuda")
        ctx.footprint(g, fp, *part, out, te.MEM_DEVICE, slab=te.Slab(b, e - b, hl, hr))
        ctx.synchronize()
        a, c = whole[b:e], out
        assert torch.equal(torch.isnan(a), torch.isnan(c))
        assert torch.equal(a[~torch.isnan(a)], c[~torch.isnan(c)]), (b, e)
    with pytest.raises(te.TEError):
        ctx.footprint(g, fp, *[x[130:300].contiguous() for x in lay], torch.empty((160, rows), dtype=torch.float32, device="cuda"),
                      te.MEM_DEVICE, slab=te.Slab(140, 160, 10, 0))


@pytest.mark.parametrize("offset", [0.15, 0.0])
def test_footprint_1024_matches_oracle(te, ctx, oracle, offset):
    """VERDICT r1 item 3: the sweep at 1024 x 1024 on chain outputs, both offsets of BASELINE config 5."""
    n = 1024
    z = synth.terrain(n, n, 0.02, 1024, "mixed")
    og, g = oracle.Geometry.make(n, n, 0.02), te.Geometry.make(n, n, 0.02)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
    fo.offset = ft.offset = offset
    t, s, st, e = (np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], z))
    ref, rs, rt = oracle.footprint(og, fo, t, s, st, e)
    out, sfp, tfp = np.empty_like(t), np.empty_like(t), np.empty_like(t)
    ctx.footprint(g, ft, t, s, st, e, out, te.MEM_HOST, slope_fp=sfp, step_fp=tfp)
    assert close_sweep(out, ref), (int((out != ref).sum()), float(np.nanmax(np.abs(out - ref))))
    assert same_values(sfp, rs) and same_values(tfp, rt)
    assert (ref == 0).any() and (ref > 0).any()


def test_footprint_with_roughness_verification(te, ctx, oracle):
    """verify_roughness_footprint (robot_footprint_parameter.yaml:9): isTraversableForFilters also runs checkForRoughness
    (TraversabilityMap.cpp:779-783, 895-921).  A rough terrain makes zero-roughness-traversability patches that block cells the
    slope/step checks let through."""
    rows, cols = 200, 180
    z = synth.terrain(rows, cols, 0.02, 61, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    # a terrain whose roughness layer hits 0 is blocked by its step layer long before (3 cm of noise already saturates the step
    # filter), so the roughness layer of this test is synthetic: the chain's own layer with patches of zeros of several sizes
    rng = np.random.default_rng(61)
    rough = ch["roughness"].copy()
    for _ in range(60):
        a, b, h, w = int(rng.integers(0, rows - 12)), int(rng.integers(0, cols - 12)), int(rng.integers(1, 12)), int(rng.integers(1, 12))
        rough[a:a + h, b:b + w] = 0.0
    ch["roughness"] = rough
    assert (ch["roughness"] == 0).sum() > 500
    fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
    t, s, st, r, e = (np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], ch["roughness"], z))
    base, _, _ = oracle.footprint(og, fo, t, s, st, e)
    fo.verify_roughness = ft.verify_roughness = 1
    ref, rs, rt, rr = oracle.footprint(og, fo, t, s, st, e, roughness=r)
    assert (np.nan_to_num(ref) != np.nan_to_num(base)).sum() > 100       # the extra check changes the layer
    assert np.isfinite(rr).sum() > 0 and (rr == 0).sum() > 0
    import os
    for brute in (True, False):
        if brute:
            os.environ["TE_FOOTPRINT_BRUTE"] = "1"
        else:
            os.environ.pop("TE_FOOTPRINT_BRUTE", None)
        out, sfp, tfp, rfp = (np.empty_like(t) for _ in range(4))
        ctx.footprint(g, ft, t, s, st, e, out, te.MEM_HOST, slope_fp=sfp, step_fp=tfp, roughness=r, roughness_fp=rfp)
        assert (same_values if brute else close_sweep)(out, ref)
        assert same_values(sfp, rs) and same_values(tfp, rt) and same_values(rfp, rr)
    with pytest.raises(te.TEError) as err:   # the flag without the layer: TE_ERR_MISSING_LAYER, like GridMap::at on a missing layer
        ctx.footprint(g, ft, t, s, st, e, out, te.MEM_HOST)
    assert err.value.code == -2


def test_batched_circular_footprint_paths(te, ctx, oracle):
    """§8(f)-2: checkCircularFootprintPath (TraversabilityMap.cpp:345-462) for a batch of paths on the footprint layer."""
    rows, cols = 256, 240
    z = synth.terrain(rows, cols, 0.02, 91, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    fo = oracle.FootprintParams.yaml_defaults()
    fpl, _, _ = oracle.footprint(og, fo, ch["traversability"], ch["slope"], ch["step"], z)
    rng = np.random.default_rng(7)
    lx, ly = rows * 0.02, cols * 0.02
    begin, poses = [0], []
    for q in range(400):
        n = int(rng.integers(0, 7)) if q > 3 else (0, 1, 2, 5)[q]      # empty, single-pose and multi-pose paths
        p = rng.uniform([-0.48 * lx, -0.48 * ly], [0.48 * lx, 0.48 * ly], size=(n, 2))
        if q % 50 == 7 and n > 0:
            p[0] = [0.6 * lx, 0.0]                                       # a pose outside the map
        poses.extend(p.tolist())
        begin.append(len(poses))
    poses = np.asarray(poses, dtype=np.float64).reshape(-1, 2)
    ref_safe, ref_t = oracle.check_circular_paths(og, fpl, fo.traversability_default, begin, poses)
    safe, t = ctx.check_footprint_paths(g, fpl, fo.traversability_default, begin, poses)
    assert np.array_equal(safe, ref_safe)
    assert np.array_equal(t, ref_t)                                     # same double arithmetic, bit for bit
    assert 10 < int(safe.sum()) < 390 and safe[0] == 0                   # safe and unsafe paths both occur; the empty path is unsafe
    # checkRobotInclination_ (TraversabilityMap.cpp:359-363, 386-390 -> checkInclination :748-762) on a robot_slope layer with
    # zero patches and holes: fewer safe paths, same arithmetic for the survivors
    rs = np.asfortranarray(ch["slope"].copy())
    rs[rng.random(rs.shape) < 0.002] = 0.0
    rs[rng.random(rs.shape) < 0.05] = np.nan
    ref_safe2, ref_t2 = oracle.check_circular_paths(og, fpl, fo.traversability_default, begin, poses, robot_slope=rs)
    safe2, t2 = ctx.check_footprint_paths(g, fpl, fo.traversability_default, begin, poses, robot_slope=rs)
    assert np.array_equal(safe2, ref_safe2) and np.array_equal(t2, ref_t2)
    assert int(safe2.sum()) < int(safe.sum()) and not (safe2 & ~safe).any()


@pytest.mark.parametrize("case", [
    dict(rows=160, cols=140, seed=61, res=0.02, yaw=0.7854),          # YAML footprint + robot.yaml yaw: 92 on-edge offsets at 0.02 m
    dict(rows=150, cols=133, seed=62, res=0.03, yaw=0.3, position=(57.25, -31.5)),
    dict(rows=96, cols=200, seed=63, res=0.02, yaw=1.5707963267948966, poly=[[0.5, 0.2], [0.1, -0.3], [-0.5, -0.2], [-0.4, 0.26], [0.0, 0.1]]),
    dict(rows=640, cols=512, seed=64, res=0.02, yaw=0.7854),          # many tiles in both directions, ~1 s of oracle on the GPU box's cores
])
def test_polygon_footprint_sweep_matches_oracle(te, ctx, oracle, case):
    """§8(f)-3: traversabilityFootprint(yaw) (TraversabilityMap.cpp:239-305, :592-645): traversability_x / traversability_rot."""
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    poly = case.get("poly", [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]])   # robot_footprint_parameter.yaml:3
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og = oracle.Geometry.make(case["rows"], case["cols"], res, pos)
    g = te.Geometry.make(case["rows"], case["cols"], res, pos)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
    layers = [np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], z)]
    rx, rrot = oracle.footprint_polygon(og, fo, poly, case["yaw"], *layers)
    ox, orot = np.empty_like(layers[0]), np.empty_like(layers[0])
    ctx.footprint_polygon(g, ft, poly, case["yaw"], *layers, ox, orot, te.MEM_HOST)
    for a, b, name in ((ox, rx, "traversability_x"), (orot, rrot, "traversability_rot")):
        assert not np.isnan(a).any() and not np.isnan(b).any(), name
        assert np.array_equal(a == 0, b == 0), (name, int(((a == 0) != (b == 0)).sum()))   # same cells blocked: same polygon membership
        assert close_sweep(a, b), (name, int((a != b).sum()), float(np.abs(a - b).max()))
    assert (rx == 0).any() and (rx > 0).any() and (rrot > 0).any()
    if case["yaw"] != 0.0:
        assert not np.array_equal(rx, rrot)


def test_polygon_footprint_slabs_equal_whole_map(te, ctx, oracle):
    """Multi-GPU tiling of the polygon sweep: a column slab with its halo gives exactly the whole-map layers."""
    import torch
    rows, cols = 128, 300
    z = synth.terrain(rows, cols, 0.02, 43, "mixed")
    og = oracle.Geometry.make(rows, cols, 0.02)
    g = te.Geometry.make(rows, cols, 0.02)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    fp = te.FootprintParams.yaml_defaults()
    poly = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32).T)).cuda()  # noqa: E731
    lay = [dev(ch["traversability"]), dev(ch["slope"]), dev(ch["step"]), dev(z)]
    ctx.set_stream(None)
    wx, wr = (torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(2))
    ctx.footprint_polygon(g, fp, poly, 0.7854, *lay, wx, wr, te.MEM_DEVICE)
    ctx.synchronize()
    H = 29 + 20   # reach of the polygon (0.541 m -> 28 + 1 cells) + the predicates' halo
    for b, e in ((0, 150), (150, 300)):
        hl, hr = min(H, b), min(H, cols - e)
        part = [x[b - hl:e + hr].contiguous() for x in lay]
        ox, orr = (torch.empty((e - b, rows), dtype=torch.float32, device="cuda") for _ in range(2))
        ctx.footprint_polygon(g, fp, poly, 0.7854, *part, ox, orr, te.MEM_DEVICE, slab=te.Slab(b, e - b, hl, hr))
        ctx.synchronize()
        assert torch.equal(wx[b:e], ox) and torch.equal(wr[b:e], orr), (b, e)


def test_polygon_footprint_with_roughness_check_and_argument_errors(te, ctx, oracle):
    """verify_roughness_footprint in the polygon sweep (isTraversableForFilters :779-783) and the argument checks of the entry."""
    rows, cols, res = 128, 120, 0.03
    z = synth.terrain(rows, cols, res, 71, "mixed")
    og, g = oracle.Geometry.make(rows, cols, res), te.Geometry.make(rows, cols, res)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    fo, ft = oracle.FootprintParams.yaml_defaults(), te.FootprintParams.yaml_defaults()
    fo.verify_roughness = ft.verify_roughness = 1
    poly = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]
    lay = [np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], z)]
    rough = np.asfortranarray(ch["roughness"], dtype=np.float32)
    rx, rrot = oracle.footprint_polygon(og, fo, poly, 0.5, *lay, roughness=rough)
    ox, orot = np.empty_like(lay[0]), np.empty_like(lay[0])
    ctx.footprint_polygon(g, ft, poly, 0.5, *lay, ox, orot, te.MEM_HOST, roughness=rough)
    assert np.array_equal(ox == 0, rx == 0) and np.array_equal(orot == 0, rrot == 0)
    assert close_sweep(ox, rx) and close_sweep(orot, rrot)
    fo.verify_roughness = 0
    nx, _ = oracle.footprint_polygon(og, fo, poly, 0.5, *lay)
    assert (rx == 0).sum() >= (nx == 0).sum()                           # the extra predicate can only block more
    with pytest.raises(te.TEError) as err:                               # the flag without the layer
        ctx.footprint_polygon(g, ft, poly, 0.5, *lay, ox, orot, te.MEM_HOST)
    assert err.value.code == -2
    ft.verify_roughness = 0
    with pytest.raises(te.TEError) as err:                               # a polygon needs three vertices
        ctx.footprint_polygon(g, ft, poly[:2], 0.5, *lay, ox, orot, te.MEM_HOST)
    assert err.value.code == -1
    with pytest.raises(te.TEError) as err:                               # reach beyond 31 cells: not supported, said so
        ctx.footprint_polygon(g, ft, [[1.2, 0.3], [1.2, -0.3], [-1.2, -0.3], [-1.2, 0.3]], 0.5, *lay, ox, orot, te.MEM_HOST)
    assert err.value.code == -4


def test_footprint_entries_take_circular_buffer_maps(te, ctx, oracle):
    """te_footprint / te_footprint_polygon (TE_MEM_HOST, whole map) with a non-zero grid_map start index: layers in buffer order in,
    layers in buffer order out, equal to the unwrapped map's result bitwise."""
    rows, cols, sr, sc = 144, 120, 55, 97
    z = synth.terrain(rows, cols, 0.02, 47, "mixed")
    og = oracle.Geometry.make(rows, cols, 0.02)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    g0 = te.Geometry.make(rows, cols, 0.02)
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = sr, sc
    fp = te.FootprintParams.yaml_defaults()
    poly = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]
    lay = [np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], z)]
    wl = [np.asfortranarray(np.roll(x, (sr, sc), axis=(0, 1))) for x in lay]
    ctx.set_stream(None)
    ref, refw = np.empty_like(lay[0]), np.empty_like(lay[0])
    ctx.footprint(g0, fp, *lay, ref, te.MEM_HOST)
    ctx.footprint(gw, fp, *wl, refw, te.MEM_HOST)
    assert same_values(ref, np.roll(refw, (-sr, -sc), axis=(0, 1)))
    px, pr, pxw, prw = (np.empty_like(lay[0]) for _ in range(4))
    ctx.footprint_polygon(g0, fp, poly, 0.7854, *lay, px, pr, te.MEM_HOST)
    ctx.footprint_polygon(gw, fp, poly, 0.7854, *wl, pxw, prw, te.MEM_HOST)
    assert np.array_equal(px, np.roll(pxw, (-sr, -sc), axis=(0, 1))) and np.array_equal(pr, np.roll(prw, (-sr, -sc), axis=(0, 1)))
