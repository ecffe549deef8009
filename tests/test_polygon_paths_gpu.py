"""te_check_footprint_paths_polygon on the GPU against the CPU oracle of checkPolygonalFootprintPath, bit for bit."""
import numpy as np
import pytest

import paths_oracle as po
import synth
from helpers import YAML, chain_layers, footprint_params, polygonal_paths, random_footprint, same

pytestmark = pytest.mark.gpu

def _gpu(ctx, g, ft, L, fxyz, begin, poses, rs, cons, **kw):
    return ctx.check_footprint_paths_polygon(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], fxyz, begin, poses,
                                             robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                             conservative=cons, **kw)


def _cpu(og, fo, L, fxyz, begin, poses, rs, cons):
    return po.check_request(og, fo, dict(L, robot_slope=rs), begin, poses, footprint_xyz=fxyz, conservative=cons)[:3]


def _assert_match(got, want, what):
    assert np.array_equal(got[0], want[0]), (what, np.nonzero(got[0] != want[0])[0][:10])
    assert same(got[1], want[1]), (what, np.nonzero(got[1] != want[1])[0][:10])
    assert same(got[2], want[2]), (what, np.nonzero(got[2] != want[2])[0][:10])


@pytest.mark.parametrize("case", [
    dict(rows=200, cols=180, res=0.02, seed=41),
    dict(rows=160, cols=150, res=0.03, seed=42),
    dict(rows=190, cols=170, res=0.02, seed=43, position=(123.456, -78.9)),
])
def test_polygon_paths_match_oracle(te, ctx, oracle, case):
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og, g = oracle.Geometry.make(case["rows"], case["cols"], res, pos), te.Geometry.make(case["rows"], case["cols"], res, pos)
    L, rs = chain_layers(oracle, og, z, case["seed"])
    rng = np.random.default_rng(case["seed"])
    begin, poses = polygonal_paths(rng, og, 300)
    cons = (rng.random(len(begin) - 1) < 0.3).astype(np.uint8)
    feet = [np.asarray(YAML, np.float32)] + [random_footprint(rng, nv) for nv in (1, 2, 3, 7, 16)]
    for fi, fxyz in enumerate(feet):
        for verify in (0, 1):
            ft, fo = footprint_params(te, oracle, verify)
            for slope_layer in ((None, rs) if fi < 2 else (rs if verify else None,)):
                want = _cpu(og, fo, L, fxyz, begin, poses, slope_layer, cons)
                got = _gpu(ctx, g, ft, L, fxyz, begin, poses, slope_layer, cons)
                _assert_match(got, want, (fi, verify, slope_layer is None))
                if fi == 0:
                    assert 10 < int(want[0].sum()) < 290 and want[0][0] == 0


def test_polygon_planner_paths_2048(te, ctx, oracle):
    n = 2048
    z = synth.terrain(n, n, 0.02, 2049, "mixed")
    og, g = oracle.Geometry.make(n, n, 0.02), te.Geometry.make(n, n, 0.02)
    L, _ = chain_layers(oracle, og, z, 2049)
    rng = np.random.default_rng(2049)
    begin, poses = polygonal_paths(rng, og, 1000, planner=True)
    cons = (rng.random(len(begin) - 1) < 0.5).astype(np.uint8)
    ft, fo = footprint_params(te, oracle, 0)
    fxyz = np.asarray(YAML, np.float32)
    want = _cpu(og, fo, L, fxyz, begin, poses, None, cons)
    _assert_match(_gpu(ctx, g, ft, L, fxyz, begin, poses, None, cons), want, "2048")
    assert want[0].any() and not want[0].all()
    # two identical calls give identical bytes
    a, b = _gpu(ctx, g, ft, L, fxyz, begin, poses, None, cons), _gpu(ctx, g, ft, L, fxyz, begin, poses, None, cons)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _small(oracle, te, seed, rows=150, cols=140):
    z = synth.terrain(rows, cols, 0.02, seed, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, rs = chain_layers(oracle, og, z, seed)
    return og, g, L, rs


def test_conservative_vertex_cap(te, ctx, oracle):
    og, g, L, _ = _small(oracle, te, 91)
    rng = np.random.default_rng(91)
    fxyz = random_footprint(rng, 16)
    ft, fo = footprint_params(te, oracle, 0)

    def line(n, y):
        return [[-1.2 + 0.03 * k, y, 0.0, 0.0, 0.0, 0.0, 1.0] for k in range(n)]
    begin = np.array([0, 64, 128], np.int32)                       # 16 x 64 = 1024 vertices: checkable
    poses = np.asarray(line(64, 0.3) + line(64, -0.3), np.float64)
    cons = np.array([1, 0], np.uint8)
    want = _cpu(og, fo, L, fxyz, begin, poses, None, cons)
    _assert_match(_gpu(ctx, g, ft, L, fxyz, begin, poses, None, cons), want, "cap")
    begin65 = np.array([0, 65, 130], np.int32)                     # one pose past the cap
    poses65 = np.asarray(line(65, 0.3) + line(65, -0.3), np.float64)
    with pytest.raises(te.TEError) as e:
        _gpu(ctx, g, ft, L, fxyz, begin65, poses65, None, cons)
    assert e.value.code == -4
    want65 = _cpu(og, fo, L, fxyz, begin65, poses65, None, cons)
    import torch
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    lay = lambda a: torch.from_numpy(np.ascontiguousarray(a.T)).cuda()  # noqa: E731
    safe = torch.full((2,), 7, dtype=torch.uint8, device="cuda")
    trav = torch.full((2,), -1.0, dtype=torch.float64, device="cuda")
    area = torch.full((2,), -1.0, dtype=torch.float64, device="cuda")
    _gpu(ctx, g, ft, {k: lay(v) for k, v in L.items()}, fxyz, dev(begin65), dev(poses65), None, dev(cons), memory=te.MEM_DEVICE,
         is_safe=safe, traversability_out=trav, area_out=area)
    ctx.synchronize()
    s, t, a = safe.cpu().numpy(), trav.cpu().numpy(), area.cpu().numpy()
    assert s[0] == 0 and np.isnan(t[0]) and np.isnan(a[0])
    assert s[1] == want65[0][1] and same(t[1:], want65[1][1:]) and same(a[1:], want65[2][1:])


def test_polygon_device_mode_on_a_torch_stream(te, oracle):
    import torch
    og, g, L, rs = _small(oracle, te, 71, 160, 150)
    rng = np.random.default_rng(71)
    begin, poses = polygonal_paths(rng, og, 300)
    cons = (rng.random(len(begin) - 1) < 0.3).astype(np.uint8)
    bad = poses.copy()
    q5 = int(np.nonzero(np.diff(begin) > 1)[0][5])
    bad[begin[q5] + 1, 4] = np.nan                               # a non-finite pose: not checkable
    fxyz = np.asarray(YAML, np.float32)
    ft, _ = footprint_params(te, oracle, 1)
    ctx = te.Context(0)
    try:
        want = _gpu(ctx, g, ft, L, fxyz, begin, poses, rs, cons)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
        lay = lambda a: torch.from_numpy(np.ascontiguousarray(a.T)).cuda()  # noqa: E731  column-major layer -> (cols, rows) tensor
        Ld = {k: lay(v) for k, v in L.items()}
        n = len(begin) - 1
        safe = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
        trav = torch.full((n,), -1.0, dtype=torch.float64, device="cuda")
        area = torch.full((n,), -1.0, dtype=torch.float64, device="cuda")
        args = [dev(begin), dev(bad)]
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            _gpu(ctx, g, ft, Ld, fxyz, *args, lay(rs), dev(cons), memory=te.MEM_DEVICE, is_safe=safe, traversability_out=trav,
                 area_out=area)
        stream.synchronize()
        s, t, a = safe.cpu().numpy(), trav.cpu().numpy(), area.cpu().numpy()
        ok = np.ones(n, bool)
        ok[q5] = False
        _assert_match((s[ok], t[ok], a[ok]), (want[0][ok], want[1][ok], want[2][ok]), "device")
        assert s[q5] == 0 and np.isnan(t[q5]) and np.isnan(a[q5])
        assert not np.isnan(want[1]).any() and not np.isnan(want[2]).any()
        ctx.set_stream(None)
    finally:
        ctx.close()


def test_polygon_host_mode_with_start_index(te, ctx, oracle):
    og, g, L, rs = _small(oracle, te, 81)
    begin, poses = polygonal_paths(np.random.default_rng(81), og, 200)
    fxyz = np.asarray(YAML, np.float32)
    ft, _ = footprint_params(te, oracle, 1)
    want = _gpu(ctx, g, ft, L, fxyz, begin, poses, rs, None)
    sr, sc = 37, 101
    wrap = lambda a: np.asfortranarray(np.roll(np.roll(a, sr, axis=0), sc, axis=1))  # noqa: E731  stored[(i + sr) % rows, (j + sc) % cols]
    gw = te.Geometry.make(g.rows, g.cols, 0.02)
    gw.start_row, gw.start_col = sr, sc
    got = _gpu(ctx, gw, ft, {k: wrap(v) for k, v in L.items()}, fxyz, begin, poses, wrap(rs), None)
    _assert_match(got, want, "start index")
    assert 10 < int(want[0].sum()) < 190


def test_polygon_error_codes(te, ctx, oracle):
    import torch
    rows, cols = 64, 64
    g = te.Geometry.make(rows, cols, 0.02)
    one = np.ones((rows, cols), np.float32, order="F")
    L = dict(traversability=one, slope=one, step=one, elevation=one * 0, roughness=one)
    begin, poses = np.array([0, 1], np.int32), np.array([[0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]])
    fxyz = np.asarray(YAML, np.float32)
    ft, _ = footprint_params(te, oracle, 0)
    s, t, a = _gpu(ctx, g, ft, L, fxyz, begin, poses, None, None)
    assert s.tolist() == [1] and t.tolist() == [1.0] and abs(a[0] - 0.9 * 0.6) < 1e-6

    def code(fn):
        with pytest.raises(te.TEError) as e:
            fn()
        return e.value.code

    fv, _ = footprint_params(te, oracle, 1)
    assert code(lambda: ctx.check_footprint_paths_polygon(g, fv, one, one, one, one * 0, fxyz, begin, poses)) == -2   # no roughness
    assert code(lambda: ctx.check_footprint_paths_polygon(g, ft, None, one, one, one * 0, fxyz, begin, poses)) == -2
    assert code(lambda: ctx.check_footprint_paths_polygon(g, ft, one, one, one, None, fxyz, begin, poses)) == -2
    assert code(lambda: _gpu(ctx, g, ft, L, np.zeros((17, 3), np.float32), begin, poses, None, None)) == -1   # 17 vertices
    assert code(lambda: _gpu(ctx, g, ft, L, np.zeros((0, 3), np.float32), begin, poses, None, None)) == -1    # none
    nanfp = fxyz.copy()
    nanfp[2, 2] = np.inf
    assert code(lambda: _gpu(ctx, g, ft, L, nanfp, begin, poses, None, None)) == -1
    nanpose = poses.copy()
    nanpose[0, 5] = np.nan
    assert code(lambda: _gpu(ctx, g, ft, L, fxyz, begin, nanpose, None, None)) == -1
    assert code(lambda: _gpu(ctx, g, ft, L, fxyz, np.array([0, 2, 1], np.int32), poses, None, None)) == -1      # decreasing
    lib = te.load_library()
    fn = lib.te_check_footprint_paths_polygon
    o8, od, oa = np.zeros(1, np.uint8), np.zeros(1), np.zeros(1)
    args = lambda nfp, npaths, nposes, pb, area: (ctx._h, g, ft, one.ctypes.data, one.ctypes.data, one.ctypes.data, None,  # noqa: E731
                                                  one.ctypes.data, None, nfp, fxyz.ctypes.data, npaths, nposes, pb, poses.ctypes.data,
                                                  None, o8.ctypes.data, od.ctypes.data, area, te.MEM_HOST)
    assert fn(*args(4, -1, 1, begin.ctypes.data, oa.ctypes.data)) == -1                        # negative path count
    assert fn(*args(4, 1, -1, begin.ctypes.data, oa.ctypes.data)) == -1                        # negative pose count
    assert fn(*args(4, 1, 2, begin.ctypes.data, oa.ctypes.data)) == -1                         # nposes != path_begin[npaths]
    assert fn(*args(4, 1, 1, None, oa.ctypes.data)) == -1                                      # path_begin missing
    assert fn(*args(4, 1, 1, begin.ctypes.data, None)) == -1                                   # area missing
    assert fn(*args(4, 1, 1, begin.ctypes.data, oa.ctypes.data)) == 0 and o8[0] == 1
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row = 3
    dev = torch.ones((cols, rows), dtype=torch.float32, device="cuda")
    out = lambda dt: torch.zeros(1, dtype=dt, device="cuda")  # noqa: E731
    assert code(lambda: ctx.check_footprint_paths_polygon(gw, ft, dev, dev, dev, dev, fxyz, torch.tensor([0, 1], dtype=torch.int32, device="cuda"),
                                                          torch.from_numpy(poses).cuda(), memory=te.MEM_DEVICE, is_safe=out(torch.uint8),
                                                          traversability_out=out(torch.float64), area_out=out(torch.float64))) == -4
