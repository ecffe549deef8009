"""The untraversable polygons of te_check_footprint_paths_fresh2 / _polygon2 on the GPU against the CPU oracles, bit for bit in
count and vertices; is_safe, traversability and area against the entries without polygons."""
import numpy as np
import pytest

import paths_oracle as po
import synth
from helpers import (DYADIC_N, DYADIC_RES, YAML, chain_layers, circular_paths, dyadic_cell, dyadic_map, footprint_params,
                     polygonal_paths, same, same_polygons)

pytestmark = pytest.mark.gpu

CAP = 64


def _circle(ctx, g, ft, L, begin, poses, radius, rs, cup, cap=CAP):
    return ctx.check_footprint_paths_fresh(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], begin, poses, radius,
                                           robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                           compute_untraversable_polygon=cup, untraversable_capacity=cap)


def _check_circle(ctx, g, og, ft, fo, L, begin, poses, radius, rs, cup, what, cap=CAP):
    got = _circle(ctx, g, ft, L, begin, poses, radius, rs, cup, cap)
    want = po.check_request(og, fo, dict(L, robot_slope=rs), begin, poses, radius, cup=cup, capacity=cap)
    assert np.array_equal(got[0], want[0]) and same(got[1], want[1]), what
    same_polygons(got[2], got[3], want[3], want[4], what)
    old = ctx.check_footprint_paths_fresh(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], begin, poses, radius,
                                          robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                          compute_untraversable_polygon=cup)
    assert np.array_equal(got[0], old[0]) and same(got[1], old[1]), what
    return got


def _poly(ctx, g, ft, L, fxyz, begin, poses, rs, cons, cup, cap=CAP):
    return ctx.check_footprint_paths_polygon(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], fxyz, begin, poses,
                                             robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                             conservative=cons, compute_untraversable_polygon=cup, untraversable_capacity=cap)


def _check_poly(ctx, g, og, ft, fo, L, fxyz, begin, poses, rs, cons, cup, what, cap=CAP):
    got = _poly(ctx, g, ft, L, fxyz, begin, poses, rs, cons, cup, cap)
    want = po.check_request(og, fo, dict(L, robot_slope=rs), begin, poses, footprint_xyz=fxyz, conservative=cons, cup=cup,
                            capacity=cap)
    for k in range(3):
        assert same(got[k].astype(np.float64) if k == 0 else got[k], want[k].astype(np.float64) if k == 0 else want[k]), (what, k)
    same_polygons(got[3], got[4], want[3], want[4], what)
    old = ctx.check_footprint_paths_polygon(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], fxyz, begin, poses,
                                            robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                            conservative=cons)
    assert np.array_equal(got[0], old[0]) and same(got[1], old[1]) and same(got[2], old[2]), what
    return got


CASES = [
    dict(rows=200, cols=180, res=0.02, seed=31),
    dict(rows=160, cols=150, res=0.03, seed=32),
    dict(rows=190, cols=170, res=0.02, seed=33, position=(123.456, -78.9)),
]


@pytest.mark.parametrize("case", CASES)
def test_circular_polygons_match_oracle(te, ctx, oracle, case):
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og, g = oracle.Geometry.make(case["rows"], case["cols"], res, pos), te.Geometry.make(case["rows"], case["cols"], res, pos)
    L, rs = chain_layers(oracle, og, z, case["seed"])
    rng = np.random.default_rng(case["seed"])
    begin, poses, radius = circular_paths(rng, og, 400, radii=(0.0, 0.2, 0.3, 0.45, 1.0))
    cup = (rng.random(len(radius)) < 0.6).astype(np.uint8)
    for verify in (0, 1):
        ft, fo = footprint_params(te, oracle, verify)
        for slope_layer in (None, rs):
            got = _check_circle(ctx, g, og, ft, fo, L, begin, poses, radius, slope_layer, cup, (verify, slope_layer is None))
            assert (got[2] > 3).sum() > 10 and (got[2][cup == 0] == 0).all()
    # traversability_default 0: single poses outside the map give fromCircle
    ft, fo = footprint_params(te, oracle, 0)
    ft.traversability_default = fo.traversability_default = 0.0
    got = _check_circle(ctx, g, og, ft, fo, L, begin, poses, radius, None, cup, "default 0")
    assert (got[2] == 20).any() or (got[2] > 0).any()


def test_circular_radii_up_to_the_ring_cap(te, ctx, oracle):
    rows = cols = 320
    z = synth.terrain(rows, cols, 0.02, 91, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, _ = chain_layers(oracle, og, z, 91)
    rng = np.random.default_rng(91)
    begin, poses, radius = circular_paths(rng, og, 120, radii=(1.2, 2.0, 2.38))   # 2.38 + 0.15 m at 0.02 m: 127 rings
    ft, fo = footprint_params(te, oracle, 1)
    got = _check_circle(ctx, g, og, ft, fo, L, begin, poses, radius, None, np.ones(len(radius), np.uint8), "big radii", cap=512)
    assert got[2].max() > 8


def test_hand_derived_cases_on_the_gpu(te, ctx, oracle):
    """The geometry of test_untraversable_cpu.py: single cells, 2 / 3 cells in visit order, collinear rows, repeated hulls."""
    blocked = [[(32, 32)], [(34, 32), (32, 32)], [(32, 35), (33, 32), (32, 32)], [(a, b) for a in range(31, 34) for b in range(31, 34)],
               [(32, b) for b in (30, 31, 33, 34)], [(37, 32)], [(30, 19)], [(30, 19), (31, 18)]]
    for cells in blocked:
        og, fo, L = dyadic_map(oracle, cells)
        g, ft = te.Geometry.make(DYADIC_N, DYADIC_N, DYADIC_RES), te.FootprintParams.yaml_defaults()
        ft.max_gap_width, ft.offset, ft.traversability_default = fo.max_gap_width, fo.offset, fo.traversability_default
        L["roughness"] = None
        P = dyadic_cell
        paths = [[P(32, 32)], [P(30, 10), P(30, 18)], [P(30, 14), P(30, 18)], [P(30, 18)]]
        begin = np.cumsum([0] + [len(p) for p in paths]).astype(np.int32)
        poses = np.asarray([q for p in paths for q in p], np.float64)
        for radius in (0.0, 0.5, 1.0):
            _check_circle(ctx, g, og, ft, fo, L, begin, poses, np.full(len(paths), radius), None, np.ones(len(paths), np.uint8), cells)


@pytest.mark.parametrize("case", CASES)
def test_polygonal_polygons_match_oracle(te, ctx, oracle, case):
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og, g = oracle.Geometry.make(case["rows"], case["cols"], res, pos), te.Geometry.make(case["rows"], case["cols"], res, pos)
    L, rs = chain_layers(oracle, og, z, case["seed"])
    rng = np.random.default_rng(case["seed"] + 10)
    begin, poses = polygonal_paths(rng, og, 300)
    cons = (rng.random(len(begin) - 1) < 0.3).astype(np.uint8)
    cup = (rng.random(len(begin) - 1) < 0.6).astype(np.uint8)
    fxyz = np.asarray(YAML, np.float32)
    for verify in (0, 1):
        ft, fo = footprint_params(te, oracle, verify)
        for slope_layer in (None, rs):
            got = _check_poly(ctx, g, og, ft, fo, L, fxyz, begin, poses, slope_layer, cons, cup, (verify, slope_layer is None))
            assert (got[3] > 3).sum() > 10 and (got[3][cup == 0] == 0).all()
    # compute_untraversable_polygon NULL: no polygons
    ft, fo = footprint_params(te, oracle, 0)
    got = _check_poly(ctx, g, og, ft, fo, L, fxyz, begin, poses, None, cons, None, "no cup")
    assert (got[3] == 0).all()


def test_conservative_paths_at_the_vertex_cap(te, ctx, oracle):
    rows = cols = 240
    z = synth.terrain(rows, cols, 0.02, 93, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, _ = chain_layers(oracle, og, z, 93)
    rng = np.random.default_rng(93)
    begin, poses = polygonal_paths(rng, og, 40, planner=True)
    # one path of 256 poses with the 4-vertex footprint: polygon2 reaches the 1024-vertex cap
    walk = np.cumsum(rng.uniform(-0.01, 0.01, (256, 2)), axis=0) + [0.5, -0.3]
    long = np.concatenate([walk, np.tile([0.0, 0.0, 0.0, 0.0, 1.0], (256, 1))], axis=1)
    begin = np.append(begin, begin[-1] + 256).astype(np.int32)
    poses = np.concatenate([poses, long])
    cons = np.ones(len(begin) - 1, np.uint8)
    ft, fo = footprint_params(te, oracle, 1)
    got = _check_poly(ctx, g, og, ft, fo, L, np.asarray(YAML, np.float32), begin, poses, None, cons,
                      np.ones(len(begin) - 1, np.uint8), "conservative")
    assert (got[3] > 0).any()


def test_planner_paths_2048(te, ctx, oracle):
    n = 2048
    z = synth.terrain(n, n, 0.02, 2048, "mixed")
    og, g = oracle.Geometry.make(n, n, 0.02), te.Geometry.make(n, n, 0.02)
    L, _ = chain_layers(oracle, og, z, 2048)
    rng = np.random.default_rng(2050)
    ft, fo = footprint_params(te, oracle, 0)
    begin, poses, radius = circular_paths(rng, og, 1000, planner=True)
    cup = (rng.random(len(radius)) < 0.5).astype(np.uint8)
    got = _check_circle(ctx, g, og, ft, fo, L, begin, poses, radius, None, cup, "2048 circular")
    assert (got[2] > 0).any()
    pb, pp = polygonal_paths(rng, og, 1000, planner=True)
    pcup = (rng.random(len(pb) - 1) < 0.5).astype(np.uint8)
    got = _check_poly(ctx, g, og, ft, fo, L, np.asarray(YAML, np.float32), pb, pp, None, None, pcup, "2048 polygonal")
    assert (got[3] > 0).any()


def test_capacity_smaller_than_the_hull(te, ctx, oracle):
    rows, cols = 200, 180
    z = synth.terrain(rows, cols, 0.02, 31, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, _ = chain_layers(oracle, og, z, 31)
    rng = np.random.default_rng(31)
    begin, poses, radius = circular_paths(rng, og, 400, radii=(0.45, 1.0))
    ft, fo = footprint_params(te, oracle, 1)
    cup = np.ones(len(radius), np.uint8)
    full = _circle(ctx, g, ft, L, begin, poses, radius, None, cup, cap=512)
    got = _check_circle(ctx, g, og, ft, fo, L, begin, poses, radius, None, cup, "cap 3", cap=3)
    assert np.array_equal(got[2], full[2]) and (full[2] > 3).any()
    same_polygons(got[2], got[3], full[2], full[3][:, :3], "prefix of 3")
    zero = _circle(ctx, g, ft, L, begin, poses, radius, None, cup, cap=0)   # counts only
    assert np.array_equal(zero[2], full[2])
    pb, pp = polygonal_paths(rng, og, 300)
    pcup = np.ones(len(pb) - 1, np.uint8)
    fxyz = np.asarray(YAML, np.float32)
    full = _poly(ctx, g, ft, L, fxyz, pb, pp, None, None, pcup, cap=512)
    got = _check_poly(ctx, g, og, ft, fo, L, fxyz, pb, pp, None, None, pcup, "cap 2", cap=2)
    assert np.array_equal(got[3], full[3]) and (full[3] > 2).any()
    same_polygons(got[3], got[4], full[3], full[4][:, :2], "prefix of 2")


def test_device_mode_on_a_torch_stream(te, oracle):
    import torch
    rows, cols = 160, 150
    z = synth.terrain(rows, cols, 0.02, 71, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, rs = chain_layers(oracle, og, z, 71)
    rng = np.random.default_rng(71)
    begin, poses, radius = circular_paths(rng, og, 300)
    radius[5] = 3.0                                   # past the ring table: -1 with cup, 0 without
    radius[6] = 3.0
    cup = (rng.random(len(radius)) < 0.5).astype(np.uint8)
    cup[5], cup[6] = 1, 0
    pb, pp = polygonal_paths(rng, og, 200)
    bad = next(q for q in range(4, len(pb) - 1) if pb[q + 1] - pb[q] >= 2)
    pp[int(pb[bad]), 0] = np.nan                      # a path the check cannot read: -1 with cup
    pcup = (rng.random(len(pb) - 1) < 0.5).astype(np.uint8)
    pcup[bad] = 1
    ft, _ = footprint_params(te, oracle, 1)
    fxyz = np.asarray(YAML, np.float32)
    ctx = te.Context(0)
    try:
        host_radius = radius.copy()
        host_radius[5] = host_radius[6] = 0.3
        want = _circle(ctx, g, ft, L, begin, poses, host_radius, rs, cup)
        host_pp = pp.copy()
        host_pp[int(pb[bad]), 0] = 0.0
        want_p = _poly(ctx, g, ft, L, fxyz, pb, host_pp, rs, None, pcup)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
        lay = lambda a: torch.from_numpy(np.ascontiguousarray(a.T)).cuda()  # noqa: E731
        Ld = {k: lay(v) for k, v in L.items()}
        n, m = len(radius), len(pb) - 1
        out = dict(is_safe=torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
                   traversability_out=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
                   untraversable_count=torch.full((n,), 99, dtype=torch.int32, device="cuda"),
                   untraversable_xy=torch.zeros((n, CAP, 2), dtype=torch.float64, device="cuda"))
        pout = dict(is_safe=torch.full((m,), 7, dtype=torch.uint8, device="cuda"),
                    traversability_out=torch.full((m,), -1.0, dtype=torch.float64, device="cuda"),
                    area_out=torch.full((m,), -1.0, dtype=torch.float64, device="cuda"),
                    untraversable_count=torch.full((m,), 99, dtype=torch.int32, device="cuda"),
                    untraversable_xy=torch.zeros((m, CAP, 2), dtype=torch.float64, device="cuda"))
        args = (dev(begin), dev(poses), dev(radius))
        pargs = (dev(pb), dev(pp))
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            ctx.check_footprint_paths_fresh(g, ft, Ld["traversability"], Ld["slope"], Ld["step"], Ld["elevation"], *args,
                                            robot_slope=lay(rs), roughness=Ld["roughness"], compute_untraversable_polygon=dev(cup),
                                            memory=te.MEM_DEVICE, untraversable_capacity=CAP, **out)
            ctx.check_footprint_paths_polygon(g, ft, Ld["traversability"], Ld["slope"], Ld["step"], Ld["elevation"], fxyz, *pargs,
                                              robot_slope=lay(rs), roughness=Ld["roughness"], compute_untraversable_polygon=dev(pcup),
                                              memory=te.MEM_DEVICE, untraversable_capacity=CAP, **pout)
        stream.synchronize()
        got = [out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "untraversable_count", "untraversable_xy")]
        ok = np.ones(n, bool)
        ok[[5, 6]] = False
        assert np.array_equal(got[0][ok], want[0][ok]) and same(got[1][ok], want[1][ok])
        same_polygons(got[2][ok], got[3][ok], want[2][ok], want[3][ok], "device circular")
        assert got[2][5] == -1 and got[2][6] == 0 and got[0][5] == 0 and np.isnan(got[1][5])
        pgot = [pout[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out", "untraversable_count", "untraversable_xy")]
        ok = np.ones(m, bool)
        ok[bad] = False
        assert np.array_equal(pgot[0][ok], want_p[0][ok]) and same(pgot[1][ok], want_p[1][ok]) and same(pgot[2][ok], want_p[2][ok])
        same_polygons(pgot[3][ok], pgot[4][ok], want_p[3][ok], want_p[4][ok], "device polygonal")
        assert pgot[3][bad] == -1 and pgot[0][bad] == 0 and np.isnan(pgot[1][bad])
        ctx.set_stream(None)
    finally:
        ctx.close()


def test_host_mode_with_start_index(te, ctx, oracle):
    rows, cols = 150, 140
    z = synth.terrain(rows, cols, 0.02, 81, "mixed")
    og = oracle.Geometry.make(rows, cols, 0.02)
    L, rs = chain_layers(oracle, og, z, 81)
    rng = np.random.default_rng(81)
    begin, poses, radius = circular_paths(rng, og, 200)
    pb, pp = polygonal_paths(rng, og, 200)
    cup, pcup = np.ones(len(radius), np.uint8), np.ones(len(pb) - 1, np.uint8)
    ft, _ = footprint_params(te, oracle, 1)
    fxyz = np.asarray(YAML, np.float32)
    g = te.Geometry.make(rows, cols, 0.02)
    want = _circle(ctx, g, ft, L, begin, poses, radius, rs, cup)
    want_p = _poly(ctx, g, ft, L, fxyz, pb, pp, rs, None, pcup)
    sr, sc = 37, 101
    wrap = lambda a: np.asfortranarray(np.roll(np.roll(a, sr, axis=0), sc, axis=1))  # noqa: E731
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = sr, sc
    Lw = {k: wrap(v) for k, v in L.items()}
    got = _circle(ctx, gw, ft, Lw, begin, poses, radius, wrap(rs), cup)
    got_p = _poly(ctx, gw, ft, Lw, fxyz, pb, pp, wrap(rs), None, pcup)
    for a, b in zip(got[:2] + got_p[:3], want[:2] + want_p[:3]):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    same_polygons(got[2], got[3], want[2], want[3], "start index circular")
    same_polygons(got_p[3], got_p[4], want_p[3], want_p[4], "start index polygonal")
    assert (want[2] > 3).any() and (want_p[3] > 3).any()


def test_error_codes(te, ctx, oracle):
    rows, cols = 64, 64
    g = te.Geometry.make(rows, cols, 0.02)
    one = np.ones((rows, cols), np.float32, order="F")
    begin, poses, radius = np.array([0, 1], np.int32), np.zeros((1, 2)), np.array([0.3])
    ft, _ = footprint_params(te, oracle, 0)
    lib = te.load_library()
    fresh = lib.te_check_footprint_paths_fresh2
    s8, d1, c1, xy = np.zeros(1, np.uint8), np.zeros(1), np.zeros(1, np.int32), np.zeros(8)
    L = [one.ctypes.data, one.ctypes.data, one.ctypes.data, None, one.ctypes.data, None]

    def f(maxv, cnt, uxy):
        return fresh(ctx._h, g, ft, *L, 1, begin.ctypes.data, poses.ctypes.data, radius.ctypes.data, None, s8.ctypes.data,
                     d1.ctypes.data, maxv, cnt, uxy, te.MEM_HOST)
    assert f(-1, c1.ctypes.data, xy.ctypes.data) == -1          # negative max_vertices
    assert f(4, c1.ctypes.data, None) == -1                     # counts without room for vertices
    assert f(4, None, xy.ctypes.data) == -1                     # vertices without counts
    assert f(0, c1.ctypes.data, None) == 0 and c1[0] == 0       # counts only
    assert f(0, None, None) == 0                                # exactly te_check_footprint_paths_fresh
    fxyz = np.asarray(YAML, np.float32)
    poly = lib.te_check_footprint_paths_polygon2
    pose = np.array([[0.0, 0, 0, 0, 0, 0, 1]])
    cup = np.ones(1, np.uint8)

    def p(maxv, cnt, uxy, poses=pose, fxyz=fxyz):
        return poly(ctx._h, g, ft, *L, len(fxyz), fxyz.ctypes.data, 1, len(poses), begin.ctypes.data, poses.ctypes.data, None,
                    s8.ctypes.data, d1.ctypes.data, d1.ctypes.data, cup.ctypes.data, maxv, cnt, uxy, te.MEM_HOST)
    assert p(-2, c1.ctypes.data, xy.ctypes.data) == -1
    assert p(4, c1.ctypes.data, None) == -1
    assert p(4, None, xy.ctypes.data) == -1
    assert p(4, c1.ctypes.data, xy.ctypes.data) == 0
    # a polygon whose bounding box spans more than 1024 map rows: unsupported in host memory (a 2048-row map, a 25 m footprint)
    ft.max_gap_width = 0.001                                         # checkForSlope's critical count 0: a zero slope blocks its cell
    gb = te.Geometry.make(2048, 8, 0.02)
    big = np.zeros((2048, 8), np.float32, order="F")               # slope 0 everywhere: every cell blocked
    ob = np.ones((2048, 8), np.float32, order="F")
    Lb = [ob.ctypes.data, big.ctypes.data, ob.ctypes.data, None, ob.ctypes.data, None]
    wide = np.array([[12.5, 0.05, 0], [-12.5, 0.05, 0], [-12.5, -0.05, 0], [12.5, -0.05, 0]], np.float32)
    rc = poly(ctx._h, gb, ft, *Lb, 4, wide.ctypes.data, 1, 1, begin.ctypes.data, pose.ctypes.data, None, s8.ctypes.data,
              d1.ctypes.data, d1.ctypes.data, cup.ctypes.data, 4, c1.ctypes.data, xy.ctypes.data, te.MEM_HOST)
    assert rc == -4
    rc = poly(ctx._h, gb, ft, *Lb, 4, wide.ctypes.data, 1, 1, begin.ctypes.data, pose.ctypes.data, None, s8.ctypes.data,
              d1.ctypes.data, d1.ctypes.data, None, 4, c1.ctypes.data, xy.ctypes.data, te.MEM_HOST)
    assert rc == 0 and c1[0] == 0 and s8[0] == 0                  # no polygon requested: no bound
