"""te_check_footprint_paths_polygon on the GPU against the CPU oracle of checkPolygonalFootprintPath, bit for bit."""
import numpy as np
import pytest

import polygon_paths_oracle as ppo
import synth

pytestmark = pytest.mark.gpu

YAML = [(0.45, 0.30, 0.0), (0.45, -0.30, 0.0), (-0.45, -0.30, 0.0), (-0.45, 0.30, 0.0)]   # robot_footprint_parameter.yaml:3


def _layers(oracle, og, z, seed):
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    rng = np.random.default_rng(seed)
    rough = ch["roughness"].copy()   # zero patches, so that checkForRoughness blocks cells the slope / step checks let through
    for _ in range(40):
        a, b = int(rng.integers(0, og.rows - 12)), int(rng.integers(0, og.cols - 12))
        rough[a:a + int(rng.integers(1, 12)), b:b + int(rng.integers(1, 12))] = 0.0
    rs = ch["slope"].copy()
    rs[rng.random(rs.shape) < 0.0005] = 0.0
    rs[rng.random(rs.shape) < 0.05] = np.nan
    f = lambda a: np.asfortranarray(a, dtype=np.float32)  # noqa: E731
    return dict(traversability=f(ch["traversability"]), slope=f(ch["slope"]), step=f(ch["step"]), elevation=f(z),
                roughness=f(rough)), f(rs)


def _footprint(rng, nv):
    """A random footprint of nv vertices with z != 0: convex (sorted angles) or not (shuffled)."""
    ang = np.sort(rng.uniform(0, 2 * np.pi, nv))
    r = rng.uniform(0.1, 0.5, nv)
    v = np.stack([r * np.cos(ang), r * np.sin(ang), rng.uniform(-0.3, 0.3, nv)], axis=1)
    if rng.random() < 0.5:
        rng.shuffle(v)
    return v.astype(np.float32)


def _quat(rng, kind):
    if kind == 0:    # yaw only
        a = rng.uniform(0, 2 * np.pi)
        return [0.0, 0.0, np.sin(a / 2), np.cos(a / 2)]
    q = rng.normal(size=4)
    if kind == 1:    # general unit quaternion
        return (q / np.linalg.norm(q)).tolist()
    return (q * rng.uniform(0.5, 1.5)).tolist()   # not normalised


def _paths(rng, og, npaths, planner=False):
    lx, ly = og.rows * og.resolution, og.cols * og.resolution
    cx, cy = og.position_x, og.position_y
    begin, poses = [0], []
    for q in range(npaths):
        n = int(rng.integers(2, 9)) if planner else (int(rng.integers(0, 7)) if q > 3 else (0, 1, 2, 5)[q])
        p = [rng.uniform([cx - 0.45 * lx, cy - 0.45 * ly], [cx + 0.45 * lx, cy + 0.45 * ly])]
        for _ in range(n - 1):   # 0.1 - 0.5 m steps; a few paths turn back on themselves
            a, d = rng.uniform(0, 2 * np.pi), rng.uniform(0.1, 0.5)
            p.append(p[-1] + d * np.array([np.cos(a), np.sin(a)]) if rng.random() > 0.1 or len(p) < 2 else p[-2].copy())
        p = np.asarray(p[:n]).reshape(-1, 2)
        if not planner and q % 50 == 7 and n > 0:
            p[0] = [cx + 0.6 * lx, cy]                        # a pose outside the map
        kind = 0 if planner else int(rng.integers(0, 3))
        for x, y in p:
            poses.append([x, y, rng.uniform(-1, 1), *_quat(rng, kind)])
        begin.append(len(poses))
    return np.asarray(begin, np.int32), np.asarray(poses, np.float64).reshape(-1, 7)


def _fps(te, oracle, verify):
    ft, fo = te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults()
    ft.verify_roughness = fo.verify_roughness = verify
    return ft, fo


def _gpu(ctx, g, ft, L, fxyz, begin, poses, rs, cons, **kw):
    return ctx.check_footprint_paths_polygon(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], fxyz, begin, poses,
                                             robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                             conservative=cons, **kw)


def _cpu(og, fo, L, fxyz, begin, poses, rs, cons):
    return ppo.check_polygonal_paths(og, fo, L["traversability"], L["slope"], L["step"], L["elevation"], fxyz, begin, poses,
                                     robot_slope=rs, roughness=L["roughness"] if fo.verify_roughness else None, conservative=cons)


def _same(a, b):
    """float64 equality bit for bit; a NaN (0/0 of a zero-area footprint, in the reference too) matches a NaN."""
    return bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def _assert_match(got, want, what):
    assert np.array_equal(got[0], want[0]), (what, np.nonzero(got[0] != want[0])[0][:10])
    assert _same(got[1], want[1]), (what, np.nonzero(got[1] != want[1])[0][:10])
    assert _same(got[2], want[2]), (what, np.nonzero(got[2] != want[2])[0][:10])


@pytest.mark.parametrize("case", [
    dict(rows=200, cols=180, res=0.02, seed=41),
    dict(rows=160, cols=150, res=0.03, seed=42),
    dict(rows=190, cols=170, res=0.02, seed=43, position=(123.456, -78.9)),
])
def test_polygon_paths_match_oracle(te, ctx, oracle, case):
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og, g = oracle.Geometry.make(case["rows"], case["cols"], res, pos), te.Geometry.make(case["rows"], case["cols"], res, pos)
    L, rs = _layers(oracle, og, z, case["seed"])
    rng = np.random.default_rng(case["seed"])
    begin, poses = _paths(rng, og, 300)
    cons = (rng.random(len(begin) - 1) < 0.3).astype(np.uint8)
    feet = [np.asarray(YAML, np.float32)] + [_footprint(rng, nv) for nv in (1, 2, 3, 7, 16)]
    for fi, fxyz in enumerate(feet):
        for verify in (0, 1):
            ft, fo = _fps(te, oracle, verify)
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
    L, _ = _layers(oracle, og, z, 2049)
    rng = np.random.default_rng(2049)
    begin, poses = _paths(rng, og, 1000, planner=True)
    cons = (rng.random(len(begin) - 1) < 0.5).astype(np.uint8)
    ft, fo = _fps(te, oracle, 0)
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
    L, rs = _layers(oracle, og, z, seed)
    return og, g, L, rs


def test_conservative_vertex_cap(te, ctx, oracle):
    og, g, L, _ = _small(oracle, te, 91)
    rng = np.random.default_rng(91)
    fxyz = _footprint(rng, 16)
    ft, fo = _fps(te, oracle, 0)

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
    assert s[1] == want65[0][1] and _same(t[1:], want65[1][1:]) and _same(a[1:], want65[2][1:])


def test_polygon_device_mode_on_a_torch_stream(te, oracle):
    import torch
    og, g, L, rs = _small(oracle, te, 71, 160, 150)
    rng = np.random.default_rng(71)
    begin, poses = _paths(rng, og, 300)
    cons = (rng.random(len(begin) - 1) < 0.3).astype(np.uint8)
    bad = poses.copy()
    q5 = int(np.nonzero(np.diff(begin) > 1)[0][5])
    bad[begin[q5] + 1, 4] = np.nan                               # a non-finite pose: not checkable
    fxyz = np.asarray(YAML, np.float32)
    ft, _ = _fps(te, oracle, 1)
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
    begin, poses = _paths(np.random.default_rng(81), og, 200)
    fxyz = np.asarray(YAML, np.float32)
    ft, _ = _fps(te, oracle, 1)
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
    ft, _ = _fps(te, oracle, 0)
    s, t, a = _gpu(ctx, g, ft, L, fxyz, begin, poses, None, None)
    assert s.tolist() == [1] and t.tolist() == [1.0] and abs(a[0] - 0.9 * 0.6) < 1e-6

    def code(fn):
        with pytest.raises(te.TEError) as e:
            fn()
        return e.value.code

    fv, _ = _fps(te, oracle, 1)
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
