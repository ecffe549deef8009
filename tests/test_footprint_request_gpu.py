"""te_check_footprint_request on the GPU: a whole check_footprint_path request, circular and polygonal paths mixed, each with its own
footprint.  Every path must get, bit for bit, what te_check_footprint_paths_fresh2 (circular) or te_check_footprint_paths_polygon2
(polygonal, once per footprint group) give for it."""
import numpy as np
import pytest

import synth
import untraversable_oracle as uo
from test_paths_fresh_gpu import _layers
from test_polygon_paths_gpu import YAML, _footprint, _quat

pytestmark = pytest.mark.gpu

CAP = 64
CASES = [
    dict(rows=200, cols=180, res=0.02, seed=41),
    dict(rows=160, cols=150, res=0.03, seed=42),
    dict(rows=190, cols=170, res=0.02, seed=43, position=(123.456, -78.9)),
    dict(rows=2048, cols=2048, res=0.02, seed=44),
]


def _fps(te, oracle, verify):
    ft, fo = te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults()
    ft.verify_roughness = fo.verify_roughness = verify
    return ft, fo


def _same(a, b):
    return bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def _same_polygons(cnt, xy, ref_cnt, ref_xy, what):
    assert np.array_equal(cnt, ref_cnt), (what, np.nonzero(cnt != ref_cnt)[0][:10])
    for q in np.nonzero(cnt > 0)[0]:
        k = min(int(cnt[q]), xy.shape[1])
        assert np.array_equal(xy[q, :k].view(np.uint64), ref_xy[q, :k].view(np.uint64)), (what, q)


def _footprints(rng):
    """The four footprints of a request: 1, 3, 4 (the YAML rectangle) and 16 vertices."""
    return [_footprint(rng, 1), _footprint(rng, 3), np.asarray(YAML, np.float32), _footprint(rng, 16)]


def _request(rng, og, npaths, fps, circular=0.4, planner=False, cap_path=True):
    """A mixed request: per path its poses (7 wide), radius, footprint index (-1: circular), conservative and cup.  Circular
    paths carry z / orientations the check must ignore (NaN in some); polygonal paths carry a NaN radius, which it ignores too."""
    lx, ly = og.rows * og.resolution, og.cols * og.resolution
    cx, cy = og.position_x, og.position_y
    begin, poses, radius, kind = [0], [], [], []
    for q in range(npaths):
        k = -1 if rng.random() < circular else int(rng.integers(0, len(fps)))
        if planner:
            n = int(rng.integers(2, 9))
        else:
            n = int(rng.integers(0, 9)) if q > 5 else (0, 1, 2, 1, 5, 8)[q]
        p = [rng.uniform([cx - 0.45 * lx, cy - 0.45 * ly], [cx + 0.45 * lx, cy + 0.45 * ly])]
        for _ in range(n - 1):   # 0.1 - 0.5 m steps; a few paths turn back on themselves
            a, d = rng.uniform(0, 2 * np.pi), rng.uniform(0.1, 0.5)
            p.append(p[-1] + d * np.array([np.cos(a), np.sin(a)]) if rng.random() > 0.1 or len(p) < 2 else p[-2].copy())
        p = np.asarray(p[:n]).reshape(-1, 2)
        if not planner and q % 40 == 9 and n > 0:
            p[0] = [cx + 0.6 * lx, cy]                        # a pose outside the map
        qkind = 0 if planner else int(rng.integers(0, 3))
        for x, y in p:
            rest = [rng.uniform(-1, 1), *_quat(rng, qkind)]
            if k < 0 and rng.random() < 0.2:
                rest[-1] = np.nan
            poses.append([x, y, *rest])
        begin.append(len(poses))
        radius.append(float(rng.uniform(0.1, 0.5)) if k < 0 else np.nan)
        kind.append(k)
    if cap_path:   # a conservative YAML path of 256 poses: polygon2 reaches the 1024-vertex cap
        walk = np.cumsum(rng.uniform(-0.01, 0.01, (256, 2)), axis=0) + [cx + 0.1 * lx, cy - 0.1 * ly]
        poses.extend(np.concatenate([walk, np.tile([0.0, 0.0, 0.0, 0.0, 1.0], (256, 1))], axis=1).tolist())
        begin.append(len(poses))
        radius.append(np.nan)
        kind.append(2)
    m = len(kind)
    cons = (rng.random(m) < 0.3).astype(np.uint8)
    cup = (rng.random(m) < 0.5).astype(np.uint8)
    if cap_path:
        cons[-1] = cup[-1] = 1
    return dict(begin=np.asarray(begin, np.int32), poses=np.asarray(poses, np.float64).reshape(-1, 7),
                radius=np.asarray(radius, np.float64), kind=np.asarray(kind), cons=cons, cup=cup)


def _footprint_arrays(R, fps):
    """footprint_begin / footprint_xyz of a request: path q's own copy of its footprint, none for circular paths."""
    fb, fx = [0], []
    for k in R["kind"]:
        if k >= 0:
            fx.extend(fps[k].tolist())
        fb.append(len(fx))
    return np.asarray(fb, np.int32), np.asarray(fx, np.float32).reshape(-1, 3)


def _subset(R, idx):
    """path_begin and poses of the paths `idx` of a request, in that order."""
    b = R["begin"]
    begin = np.concatenate([[0], np.cumsum(b[idx + 1] - b[idx])]).astype(np.int32)
    poses = np.concatenate([R["poses"][b[q]:b[q + 1]] for q in idx]) if len(idx) else np.zeros((0, 7))
    return begin, poses


def _run(ctx, g, ft, L, R, fps, rs, cap, memory=0, **kw):
    fb, fx = _footprint_arrays(R, fps)
    args = (g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], R["begin"], R["poses"], R["radius"], fb, fx)
    return ctx.check_footprint_request(*args, robot_slope=rs, roughness=L["roughness"] if ft.verify_roughness else None,
                                       conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=cap,
                                       memory=memory, **kw)


def _split(ctx, g, ft, L, R, fps, rs, cap):
    """What a node computes today: te_check_footprint_paths_fresh2 on the circular paths, te_check_footprint_paths_polygon2 once
    per footprint, results scattered back into request order (area 0 for circular paths)."""
    m = len(R["kind"])
    safe, trav, area = np.zeros(m, np.uint8), np.zeros(m), np.zeros(m)
    counts, xy = np.zeros(m, np.int32), np.zeros((m, cap or 0, 2))
    rough = L["roughness"] if ft.verify_roughness else None
    idx = np.nonzero(R["kind"] < 0)[0]
    if len(idx):
        b, p = _subset(R, idx)
        got = ctx.check_footprint_paths_fresh(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], b, p[:, :2].copy(),
                                              R["radius"][idx], robot_slope=rs, roughness=rough,
                                              compute_untraversable_polygon=R["cup"][idx], untraversable_capacity=cap)
        safe[idx], trav[idx] = got[0], got[1]
        if cap is not None:
            counts[idx], xy[idx] = got[2], got[3]
    for k, fxyz in enumerate(fps):
        idx = np.nonzero(R["kind"] == k)[0]
        if not len(idx):
            continue
        b, p = _subset(R, idx)
        got = ctx.check_footprint_paths_polygon(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], fxyz, b, p,
                                                robot_slope=rs, roughness=rough, conservative=R["cons"][idx],
                                                compute_untraversable_polygon=R["cup"][idx], untraversable_capacity=cap)
        safe[idx], trav[idx], area[idx] = got[0], got[1], got[2]
        if cap is not None:
            counts[idx], xy[idx] = got[3], got[4]
    return (safe, trav, area) if cap is None else (safe, trav, area, counts, xy)


def _assert_equal(got, want, what):
    assert np.array_equal(got[0], want[0]), (what, np.nonzero(got[0] != want[0])[0][:10])
    assert _same(got[1], want[1]) and _same(got[2], want[2]), what
    if len(want) > 3:
        _same_polygons(got[3], got[4], want[3], want[4], what)


def _to_device(R, fps, L, rs):
    import torch
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    lay = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a.T)).cuda()  # noqa: E731
    fb, fx = _footprint_arrays(R, fps)
    D = {k: dev(R[k]) for k in ("begin", "poses", "radius", "cons", "cup")}
    D["fb"], D["fx"] = dev(fb), dev(fx)
    return D, {k: lay(v) for k, v in L.items()}, lay(rs)


def _run_device(ctx, g, ft, Ld, rsd, D, cap, mfv=16):
    import torch
    m = int(D["begin"].numel()) - 1
    out = dict(is_safe=torch.full((m,), 7, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.full((m,), -1.0, dtype=torch.float64, device="cuda"),
               area_out=torch.full((m,), -1.0, dtype=torch.float64, device="cuda"))
    if cap is not None:
        out.update(untraversable_count=torch.full((m,), 99, dtype=torch.int32, device="cuda"),
                   untraversable_xy=torch.zeros((m, cap, 2), dtype=torch.float64, device="cuda"))
    ctx.check_footprint_request(g, ft, Ld["traversability"], Ld["slope"], Ld["step"], Ld["elevation"], D["begin"], D["poses"],
                                D["radius"], D["fb"], D["fx"], max_footprint_vertices=mfv, robot_slope=rsd,
                                roughness=Ld["roughness"] if ft.verify_roughness else None, conservative=D["cons"],
                                compute_untraversable_polygon=D["cup"], memory=1, untraversable_capacity=cap, **out)
    torch.cuda.synchronize()
    keys = ("is_safe", "traversability_out", "area_out") + (() if cap is None else ("untraversable_count", "untraversable_xy"))
    return tuple(out[k].cpu().numpy() for k in keys)


def _case_id(c):
    return f"{c['rows']}x{c['cols']}@{c['res']}" + ("+off" if "position" in c else "")


@pytest.fixture(scope="module", params=CASES, ids=_case_id)
def mixed_case(request, te, oracle):
    return _mixed(te, oracle, request.param)


def _mixed(te, oracle, case):
    """A map case with its chain layers, a robot_slope layer and a mixed request of about 200 paths over four footprints (the
    last one the conservative 256-pose path whose polygon2 reaches the vertex cap)."""
    res, pos = case["res"], case.get("position", (0.0, 0.0))
    z = synth.terrain(case["rows"], case["cols"], res, case["seed"], "mixed", pos)
    og, g = oracle.Geometry.make(case["rows"], case["cols"], res, pos), te.Geometry.make(case["rows"], case["cols"], res, pos)
    L, rs = _layers(oracle, og, z, case["seed"])
    rng = np.random.default_rng(case["seed"])
    fps = _footprints(rng)
    R = _request(rng, og, 200, fps, planner=case["rows"] >= 2048)
    return dict(og=og, g=g, L=L, rs=rs, fps=fps, R=R)


def test_mixed_requests_equal_the_split_calls(te, ctx, oracle, mixed_case):
    g, L, rs, fps, R = (mixed_case[k] for k in ("g", "L", "rs", "fps", "R"))
    kinds = R["kind"]
    assert (kinds < 0).sum() > 40 and all((kinds == k).sum() > 10 for k in range(4))
    D, Ld, rsd = _to_device(R, fps, L, rs)
    for verify in (0, 1):
        ft, _ = _fps(te, oracle, verify)
        for slope_layer, slope_dev in ((None, None), (rs, rsd)):
            for cap in (None, CAP):
                what = (verify, slope_layer is None, cap)
                want = _split(ctx, g, ft, L, R, fps, slope_layer, cap)
                got = _run(ctx, g, ft, L, R, fps, slope_layer, cap)
                _assert_equal(got, want, ("host",) + what)
                assert (got[2][kinds < 0] == 0).all()
                _assert_equal(_run_device(ctx, g, ft, Ld, slope_dev, D, cap), want, ("device",) + what)
                if cap is not None:
                    assert (got[3] > 0).any() and (got[3][R["cup"] == 0] == 0).all()
    assert want[0].any() and not want[0].all()


def _oracle(og, fo, L, R, fps, rs):
    """The CPU oracles' answer to a request, path by path in request order: check_circular_paths_fresh2 for its circular paths
    (area 0), check_polygonal_paths2 once per footprint for its polygonal paths."""
    m = len(R["kind"])
    out = (np.zeros(m, np.uint8), np.zeros(m), np.zeros(m), np.zeros(m, np.int32), np.zeros((m, CAP, 2)))
    rough = L["roughness"] if fo.verify_roughness else None
    for k in range(-1, len(fps)):
        idx = np.nonzero(R["kind"] == k)[0]
        if not len(idx):
            continue
        b, p = _subset(R, idx)
        if k < 0:
            w = uo.check_circular_paths_fresh2(og, fo, L["traversability"], L["slope"], L["step"], L["elevation"], b, p[:, :2].copy(),
                                               R["radius"][idx], robot_slope=rs, roughness=rough,
                                               compute_untraversable_polygon=R["cup"][idx], capacity=CAP)
            w = (w[0], w[1], np.zeros(len(idx)), w[2], w[3])
        else:
            w = uo.check_polygonal_paths2(og, fo, L["traversability"], L["slope"], L["step"], L["elevation"], fps[k], b, p,
                                          robot_slope=rs, roughness=rough, conservative=R["cons"][idx],
                                          compute_untraversable_polygon=R["cup"][idx], capacity=CAP)
        for a, v in zip(out, w):
            a[idx] = v
    return out


def test_request_matches_the_cpu_oracles(te, ctx, oracle):
    """Every output of a mixed request against the CPU oracles, bit for bit, on the three small maps: with and without
    verify_roughness, robot_slope and polygon outputs."""
    for case in CASES[:3]:
        M = _mixed(te, oracle, case)
        og, g, L, fps, R = (M[k] for k in ("og", "g", "L", "fps", "R"))
        assert R["cons"][-1] and R["cup"][-1] and R["begin"][-1] - R["begin"][-2] == 256
        for verify in (0, 1):
            ft, fo = _fps(te, oracle, verify)
            for rs in (None, M["rs"]):
                want = _oracle(og, fo, L, R, fps, rs)
                for cap in (None, CAP):
                    got = _run(ctx, g, ft, L, R, fps, rs, cap)
                    _assert_equal(got, want if cap else want[:3], ("oracle", _case_id(case), verify, rs is None, cap))
                assert want[0].any() and not want[0].all() and (want[3] > 0).any()


def test_degenerate_requests(te, ctx, oracle):
    rows, cols = 160, 150
    z = synth.terrain(rows, cols, 0.02, 52, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, rs = _layers(oracle, og, z, 52)
    rng = np.random.default_rng(52)
    fps = _footprints(rng)
    ft, _ = _fps(te, oracle, 1)
    for circular in (1.0, 0.0):   # all circular; all polygonal over one footprint
        R = _request(rng, og, 150, fps[2:3], circular=circular, cap_path=False)
        for cap in (None, CAP):
            _assert_equal(_run(ctx, g, ft, L, R, fps[2:3], rs, cap), _split(ctx, g, ft, L, R, fps[2:3], rs, cap), (circular, cap))
    empty = _request(rng, og, 0, fps, cap_path=False)
    got = _run(ctx, g, ft, L, empty, fps, None, CAP)
    assert all(len(a) == 0 for a in got)


def test_device_mode_on_a_torch_stream(te, oracle):
    import torch
    rows, cols = 160, 150
    z = synth.terrain(rows, cols, 0.02, 53, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, rs = _layers(oracle, og, z, 53)
    rng = np.random.default_rng(53)
    fps = _footprints(rng)
    R = _request(rng, og, 200, fps, cap_path=False)
    R["cup"][:] = 1
    ft, _ = _fps(te, oracle, 1)
    ctx = te.Context(0)
    try:
        want = _run(ctx, g, ft, L, R, fps, rs, CAP)
        circ = np.nonzero(R["kind"] < 0)[0]
        bad_radius = circ[3]
        R["radius"][bad_radius] = 3.0                 # past the ring table: not checkable in device memory
        D, Ld, rsd = _to_device(R, fps, L, rs)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            got = _run_device(ctx, g, ft, Ld, rsd, D, CAP, mfv=4)   # the 16-vertex footprint is over the bound
        ctx.set_stream(None)
        marked = (R["kind"] == 3) | (np.arange(len(R["kind"])) == bad_radius)
        assert (R["kind"] == 3).sum() > 10
        assert (got[0][marked] == 0).all() and np.isnan(got[1][marked]).all() and np.isnan(got[2][marked]).all()
        assert (got[3][marked] == -1).all()
        ok = ~marked
        _assert_equal(tuple(a[ok] for a in got), tuple(a[ok] for a in want), "neighbours")
    finally:
        ctx.close()


def test_host_mode_with_start_index(te, ctx, oracle):
    rows, cols = 150, 140
    z = synth.terrain(rows, cols, 0.02, 54, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, rs = _layers(oracle, og, z, 54)
    rng = np.random.default_rng(54)
    fps = _footprints(rng)
    R = _request(rng, og, 200, fps, cap_path=False)
    ft, _ = _fps(te, oracle, 1)
    want = _run(ctx, g, ft, L, R, fps, rs, CAP)
    sr, sc = 37, 101
    wrap = lambda a: np.asfortranarray(np.roll(np.roll(a, sr, axis=0), sc, axis=1))  # noqa: E731
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = sr, sc
    got = _run(ctx, gw, ft, {k: wrap(v) for k, v in L.items()}, R, fps, wrap(rs), CAP)
    for a, b in zip(got[:3], want[:3]):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    _same_polygons(got[3], got[4], want[3], want[4], "start index")
    assert (want[3] > 3).any()


def test_launch_count_does_not_depend_on_the_footprints(te, ctx, oracle):
    rows, cols = 120, 120
    z = synth.terrain(rows, cols, 0.02, 55, "mixed")
    og, g = oracle.Geometry.make(rows, cols, 0.02), te.Geometry.make(rows, cols, 0.02)
    L, rs = _layers(oracle, og, z, 55)
    rng = np.random.default_rng(55)
    fps = _footprints(rng)
    R = _request(rng, og, 100, fps, cap_path=False)
    ft, _ = _fps(te, oracle, 0)
    counts = []
    for footprints in (fps[2:3] * 4, fps):   # the same request over 1 and over 4 distinct footprints
        for cap in (None, CAP):
            before = ctx.stats()[0]
            _run(ctx, g, ft, L, R, footprints, rs, cap)
            counts.append(ctx.stats()[0] - before)
    assert counts[0] == counts[2] and counts[1] == counts[3] and counts[0] == 3, counts


def test_error_codes(te, ctx, oracle):
    rows, cols = 64, 64
    g = te.Geometry.make(rows, cols, 0.02)
    one = np.ones((rows, cols), np.float32, order="F")
    ft, _ = _fps(te, oracle, 0)
    lib = te.load_library()
    fn = lib.te_check_footprint_request
    pose = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]
    yaml = np.asarray(YAML, np.float32)

    def call(kinds, poses_per_path=1, radius=0.3, fxyz=None, fb=None, mfv=16, nvertices=None, layers=None, geo=g, fp=ft,
             cons=None, cup=None, maxv=4, memory=te.MEM_HOST, poses=None, nposes=None):
        m = len(kinds)
        pb = np.arange(m + 1, dtype=np.int32) * poses_per_path
        ps = np.tile(pose, (m * poses_per_path, 1)) if poses is None else poses
        fx = np.concatenate([yaml[:k] for k in kinds] + [np.zeros((0, 3), np.float32)]) if fxyz is None else fxyz
        fbeg = np.concatenate([[0], np.cumsum(kinds)]).astype(np.int32) if fb is None else fb
        rad = np.full(m, radius)
        out = [np.zeros(m, np.uint8), np.zeros(m), np.zeros(m), np.zeros(m, np.int32), np.zeros(2 * max(m * maxv, 1))]
        lay = [one.ctypes.data, one.ctypes.data, one.ctypes.data, None, one.ctypes.data, None] if layers is None else layers
        ad = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        return fn(ctx._h, geo, fp, *lay, m, len(ps) if nposes is None else nposes, pb.ctypes.data, ps.ctypes.data, rad.ctypes.data,
                  len(fx) if nvertices is None else nvertices, fbeg.ctypes.data, fx.ctypes.data, mfv, ad(cons), ad(cup),
                  *(a.ctypes.data for a in out[:3]), maxv, out[3].ctypes.data, out[4].ctypes.data, memory)

    # sets argtypes
    ctx.check_footprint_request(g, ft, one, one, one, one * 0, [0, 1], [pose], [0.3], [0, 0], np.zeros((0, 3), np.float32))
    assert call([0, 4, 3]) == 0
    assert call([]) == 0                                            # npaths = 0
    # new: max_footprint_vertices, footprint_begin, vertex bound, non-finite vertex
    assert call([0, 4], mfv=-1) == -1 and call([0, 4], mfv=17) == -1
    assert call([0, 4], mfv=3) == -1                                # a footprint longer than max_footprint_vertices
    assert call([0, 4], mfv=0) == -1 and call([0, 0], mfv=0) == 0
    assert call([0, 4], fb=np.array([1, 1, 5], np.int32)) == -1    # does not start at 0
    assert call([0, 4], fb=np.array([0, 3, 2], np.int32), nvertices=2) == -1   # decreases
    assert call([0, 4], fb=np.array([0, 0, 4], np.int32), nvertices=3) == -1   # does not end at nvertices
    nanv = yaml.copy()
    nanv[2, 2] = np.nan
    assert call([4], fxyz=nanv) == -1
    # the predecessors' codes, per kind of path
    assert call([0, 4], radius=np.nan) == -1                        # a circular radius
    assert call([4, 3], radius=np.nan) == 0                         # ignored by polygonal paths
    assert call([0], radius=3.0) == -4                              # past the 127-ring table
    assert call([4], radius=3.0) == 0
    bad = np.tile(pose, (2, 1))
    bad[1, 6] = np.nan
    assert call([0, 4], poses=bad) == -1                            # a non-finite polygonal pose
    assert call([4, 0], poses=bad) == 0                             # a circular path reads x and y only
    assert call([4, 0], nposes=3) == -1                             # path_begin[npaths] != nposes
    assert call([4], poses_per_path=257, cons=np.ones(1, np.uint8)) == -4   # past the conservative cap
    assert call([4], poses_per_path=256, cons=np.ones(1, np.uint8)) == 0
    assert call([0, 4], maxv=-1) == -1
    assert call([0, 4], layers=[one.ctypes.data, None, one.ctypes.data, None, one.ctypes.data, None]) == -2
    neg = te.FootprintParams.yaml_defaults()
    neg.offset = -0.1
    assert call([0, 4], fp=neg) == -1
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row = 3
    assert call([0, 4], geo=gw, memory=te.MEM_DEVICE) == -4
    # a polygon whose bounding box spans more than 1024 map rows: unsupported in host memory
    fpb = te.FootprintParams.yaml_defaults()
    fpb.max_gap_width = 0.001                                       # checkForSlope's critical count 0: a zero slope blocks its cell
    gb = te.Geometry.make(2048, 8, 0.02)
    big = np.zeros((2048, 8), np.float32, order="F")
    ob = np.ones((2048, 8), np.float32, order="F")
    Lb = [ob.ctypes.data, big.ctypes.data, ob.ctypes.data, None, ob.ctypes.data, None]
    wide = np.array([[12.5, 0.05, 0], [-12.5, 0.05, 0], [-12.5, -0.05, 0], [12.5, -0.05, 0]], np.float32)
    assert call([0, 4], fxyz=wide, geo=gb, fp=fpb, layers=Lb, cup=np.ones(2, np.uint8)) == -4
    assert call([0, 4], fxyz=wide, geo=gb, fp=fpb, layers=Lb) == 0
