"""te_check_footprint_paths_fresh on the GPU against the CPU oracle of the fresh-cache path check, bit for bit."""
import numpy as np
import pytest

import paths_oracle as po
import synth
from helpers import chain_layers, circular_paths, footprint_params

pytestmark = pytest.mark.gpu


def _gpu(ctx, g, ft, L, begin, poses, radius, rs, cup, **kw):
    return ctx.check_footprint_paths_fresh(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], begin, poses, radius,
                                           robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                           compute_untraversable_polygon=cup, **kw)


def _cpu(og, fo, L, begin, poses, radius, rs, cup):
    return po.check_request(og, fo, dict(L, robot_slope=rs), begin, poses, radius, cup=cup)[:2]


@pytest.mark.parametrize("case", [
    dict(rows=200, cols=180, res=0.02, seed=31),
    dict(rows=160, cols=150, res=0.03, seed=32),
    dict(rows=190, cols=170, res=0.02, seed=33, position=(123.456, -78.9)),
])
def test_fresh_paths_match_oracle(te, ctx, oracle, case):
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og, g = oracle.Geometry.make(case["rows"], case["cols"], res, pos), te.Geometry.make(case["rows"], case["cols"], res, pos)
    L, rs = chain_layers(oracle, og, z, case["seed"])
    rng = np.random.default_rng(case["seed"])
    begin, poses, radius = circular_paths(rng, og, 400)
    cup = (rng.random(len(radius)) < 0.3).astype(np.uint8)
    for verify in (0, 1):
        ft, fo = footprint_params(te, oracle, verify)
        for slope_layer in (None, rs):
            ref_safe, ref_t = _cpu(og, fo, L, begin, poses, radius, slope_layer, cup)
            safe, t = _gpu(ctx, g, ft, L, begin, poses, radius, slope_layer, cup)
            assert np.array_equal(safe, ref_safe), (verify, slope_layer is None, np.nonzero(safe != ref_safe)[0][:10])
            assert np.array_equal(t.view(np.uint64), ref_t.view(np.uint64)), (verify, np.nonzero(t != ref_t)[0][:10])
            assert 10 < int(safe.sum()) < 390 and safe[0] == 0
    # the route of INTEGRATION.md (sweep at 0.3 m, then the memoised check) answers a different question for some paths
    ft, fo = footprint_params(te, oracle, 1)
    sel = np.nonzero(radius == 0.3)[0]
    sb = np.concatenate([[0], np.cumsum(np.diff(begin)[sel])]).astype(np.int32)
    sp = np.concatenate([poses[begin[q]:begin[q + 1]] for q in sel]).reshape(-1, 2)
    out = np.empty_like(L["traversability"])
    ctx.footprint(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], out, te.MEM_HOST, roughness=L["roughness"])
    swept_safe, _ = ctx.check_footprint_paths(g, out, ft.traversability_default, sb, sp)
    fresh_safe, _ = _gpu(ctx, g, ft, L, sb, sp, radius[sel], None, None)
    assert (swept_safe != fresh_safe).any()


def test_fresh_planner_paths_2048(te, ctx, oracle):
    n = 2048
    z = synth.terrain(n, n, 0.02, 2048, "mixed")
    og, g = oracle.Geometry.make(n, n, 0.02), te.Geometry.make(n, n, 0.02)
    L, _ = chain_layers(oracle, og, z, 2048)
    begin, poses, radius = circular_paths(np.random.default_rng(2048), og, 2000, planner=True)
    ft, fo = footprint_params(te, oracle, 0)
    ref_safe, ref_t = _cpu(og, fo, L, begin, poses, radius, None, None)
    safe, t = _gpu(ctx, g, ft, L, begin, poses, radius, None, None)
    assert np.array_equal(safe, ref_safe) and np.array_equal(t.view(np.uint64), ref_t.view(np.uint64))
    assert safe.any() and not safe.all()


def test_fresh_device_mode_on_a_torch_stream(te, oracle):
    import torch
    rows, cols = 160, 150
    z = synth.terrain(rows, cols, 0.02, 71, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, rs = chain_layers(oracle, og, z, 71)
    rng = np.random.default_rng(71)
    begin, poses, radius = circular_paths(rng, og, 300)
    radius[5] = 3.0                                          # 0.3 + 3.0 m at 0.02 m: 158 rings, more than the ring table holds
    radius[6] = -1.0
    cup = (rng.random(len(radius)) < 0.3).astype(np.uint8)
    ft, _ = footprint_params(te, oracle, 1)
    ctx = te.Context(0)
    try:
        host_radius = radius.copy()
        host_radius[5] = host_radius[6] = 0.3
        want_safe, want_t = _gpu(ctx, g, ft, L, begin, poses, host_radius, rs, cup)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
        lay = lambda a: torch.from_numpy(np.ascontiguousarray(a.T)).cuda()  # noqa: E731  column-major layer -> (cols, rows) tensor
        Ld = {k: lay(v) for k, v in L.items()}
        safe = torch.full((len(radius),), 7, dtype=torch.uint8, device="cuda")
        trav = torch.full((len(radius),), -1.0, dtype=torch.float64, device="cuda")
        args = [dev(begin), dev(poses), dev(radius)]
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            _gpu(ctx, g, ft, Ld, *args, lay(rs), dev(cup), memory=te.MEM_DEVICE, is_safe=safe, traversability_out=trav)
        stream.synchronize()
        s, t = safe.cpu().numpy(), trav.cpu().numpy()
        ok = np.ones(len(radius), bool)
        ok[[5, 6]] = False
        assert np.array_equal(s[ok], want_safe[ok]) and np.array_equal(t[ok].view(np.uint64), want_t[ok].view(np.uint64))
        assert s[5] == 0 and s[6] == 0 and np.isnan(t[5]) and np.isnan(t[6])
        assert not np.isnan(want_t).any()
        ctx.set_stream(None)
    finally:
        ctx.close()


def test_fresh_host_mode_with_start_index(te, ctx, oracle):
    rows, cols = 150, 140
    z = synth.terrain(rows, cols, 0.02, 81, "mixed")
    og = oracle.Geometry.make(rows, cols, 0.02)
    L, rs = chain_layers(oracle, og, z, 81)
    begin, poses, radius = circular_paths(np.random.default_rng(81), og, 200)
    ft, _ = footprint_params(te, oracle, 1)
    g = te.Geometry.make(rows, cols, 0.02)
    want = _gpu(ctx, g, ft, L, begin, poses, radius, rs, None)
    sr, sc = 37, 101
    wrap = lambda a: np.asfortranarray(np.roll(np.roll(a, sr, axis=0), sc, axis=1))  # noqa: E731  stored[(i + sr) % rows, (j + sc) % cols]
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = sr, sc
    got = _gpu(ctx, gw, ft, {k: wrap(v) for k, v in L.items()}, begin, poses, radius, wrap(rs), None)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint64), want[1].view(np.uint64))
    assert 10 < int(want[0].sum()) < 190


def test_fresh_error_codes(te, ctx, oracle):
    import torch
    rows, cols = 64, 64
    g = te.Geometry.make(rows, cols, 0.02)
    one = np.ones((rows, cols), np.float32, order="F")
    L = dict(traversability=one, slope=one, step=one, elevation=one * 0, roughness=one)
    begin, poses, radius = np.array([0, 1], np.int32), np.zeros((1, 2)), np.array([0.3])
    ft, _ = footprint_params(te, oracle, 0)
    assert _gpu(ctx, g, ft, L, begin, poses, radius, None, None)[0].tolist() == [1]

    def code(fn):
        with pytest.raises(te.TEError) as e:
            fn()
        return e.value.code

    fv, _ = footprint_params(te, oracle, 1)
    assert code(lambda: ctx.check_footprint_paths_fresh(g, fv, one, one, one, one * 0, begin, poses, radius)) == -2   # no roughness
    assert code(lambda: ctx.check_footprint_paths_fresh(g, ft, None, one, one, one * 0, begin, poses, radius)) == -2
    assert code(lambda: _gpu(ctx, g, ft, L, begin, poses, np.array([np.nan]), None, None)) == -1
    assert code(lambda: _gpu(ctx, g, ft, L, begin, poses, np.array([-0.1]), None, None)) == -1
    assert code(lambda: _gpu(ctx, g, ft, L, begin, poses, np.array([2.4]), None, None)) == -4    # ceil(2.55 / 0.02) = 128 rings
    assert _gpu(ctx, g, ft, L, begin, poses, np.array([2.38]), None, None)[0].tolist() == [1]   # 127 rings
    fneg, _ = footprint_params(te, oracle, 0)
    fneg.offset = -0.1
    assert code(lambda: _gpu(ctx, g, fneg, L, begin, poses, radius, None, None)) == -1
    lib = te.load_library()
    fn = lib.te_check_footprint_paths_fresh
    assert fn(ctx._h, g, ft, one.ctypes.data, one.ctypes.data, one.ctypes.data, None, one.ctypes.data, None, -1, begin.ctypes.data,
              poses.ctypes.data, radius.ctypes.data, None, None, None, te.MEM_HOST) == -1                          # negative count
    out8, outd = np.zeros(1, np.uint8), np.zeros(1)
    assert fn(ctx._h, g, ft, one.ctypes.data, one.ctypes.data, one.ctypes.data, None, one.ctypes.data, None, 1, begin.ctypes.data,
              poses.ctypes.data, None, None, out8.ctypes.data, outd.ctypes.data, te.MEM_HOST) == -1             # radius missing
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row = 3
    dev = torch.ones((cols, rows), dtype=torch.float32, device="cuda")
    assert code(lambda: ctx.check_footprint_paths_fresh(gw, ft, dev, dev, dev, dev, torch.tensor([0, 1], dtype=torch.int32, device="cuda"),
                                                        torch.zeros((1, 2), dtype=torch.float64, device="cuda"),
                                                        torch.tensor([0.3], dtype=torch.float64, device="cuda"), memory=te.MEM_DEVICE,
                                                        is_safe=torch.zeros(1, dtype=torch.uint8, device="cuda"),
                                                        traversability_out=torch.zeros(1, dtype=torch.float64, device="cuda"))) == -4
