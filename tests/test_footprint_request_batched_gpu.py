"""te_check_footprint_request_batched: the footprint path checks of a whole batch of maps in one call.  Every path must get, bit
for bit, what te_check_footprint_request returns for it on its own map alone, and a path must never see the cells or the
isTraversableForFilters memo of another map."""
import numpy as np
import pytest

import paths_oracle as po
from helpers import (YAML, assert_same_answers, batch_request, footprint_arrays, request_footprints, subset, te_footprint_params, walled_batch,
                     walled_terrain)

pytestmark = pytest.mark.gpu

ROWS, COLS, NMAPS, RES = 100, 90, 12, 0.02   # rows not a multiple of 32, columns not of 16
EMPTY = 7                                     # the map without paths
CAP = 64
LAYERS = ("traversability", "slope", "step", "roughness", "elevation", "robot_slope")


def _one(B, k):
    """Map k's layers, column-major (rows, cols)."""
    return {x: np.asfortranarray(B[x][k].T) for x in LAYERS}


def _request(rng, og, fps, npaths):
    """A mixed request on maps of geometry og, with a path_map that interleaves the maps in no order and leaves map EMPTY out.
    Every sixth path starts at a map corner or edge midpoint, one cell inside: its spirals and hulls reach past the map."""
    R = batch_request(rng, og, npaths, NMAPS, fps, exclude=EMPTY)   # every other map has paths
    lx, ly = og.rows * og.resolution, og.cols * og.resolution
    edges = [(sx * 0.49 * lx, sy * 0.49 * ly) for sx, sy in ((1, 1), (1, -1), (-1, 1), (-1, -1), (1, 0), (-1, 0), (0, 1), (0, -1))]
    for j, q in enumerate(range(2, npaths, 6)):
        if R["begin"][q + 1] > R["begin"][q]:
            R["poses"][R["begin"][q], :2] = edges[j % len(edges)]
    return R


def _batched(ctx, g, ft, B, R, fps, slope, cap, nmaps=NMAPS, memory=0, path_map=None, **kw):
    fb, fx = footprint_arrays(R, fps)
    return ctx.check_footprint_request_batched(
        g, ft, nmaps, B["traversability"], B["slope"], B["step"], B["elevation"], R["map"] if path_map is None else path_map,
        R["begin"], R["poses"], R["radius"], fb, fx, robot_slope=B["robot_slope"] if slope else None,
        roughness=B["roughness"] if ft.verify_roughness else None, conservative=R["cons"], compute_untraversable_polygon=R["cup"],
        untraversable_capacity=cap, memory=memory, **kw)


def _single(ctx, g, ft, L, R, fps, slope, cap):
    fb, fx = footprint_arrays(R, fps)
    return ctx.check_footprint_request(g, ft, L["traversability"], L["slope"], L["step"], L["elevation"], R["begin"], R["poses"],
                                       R["radius"], fb, fx, robot_slope=L["robot_slope"] if slope else None,
                                       roughness=L["roughness"] if ft.verify_roughness else None, conservative=R["cons"],
                                       compute_untraversable_polygon=R["cup"], untraversable_capacity=cap)


def _map_by_map(ctx, g, ft, B, R, fps, slope, cap):
    """te_check_footprint_request on each map with its paths, scattered back into request order."""
    m = len(R["kind"])
    out = [np.zeros(m, np.uint8), np.zeros(m), np.zeros(m), np.zeros(m, np.int32), np.zeros((m, cap, 2))]
    for k in range(NMAPS):
        idx = np.nonzero(R["map"] == k)[0]
        if len(idx):
            got = _single(ctx, g, ft, _one(B, k), subset(R, idx), fps, slope, cap)
            for o, v in zip(out, got):
                o[idx] = v
    return tuple(out)


@pytest.fixture(scope="module")
def batch(oracle):
    return walled_batch(oracle, ROWS, COLS, RES, NMAPS, 500, robot_slope=True)


@pytest.fixture(scope="module")
def request_(oracle):
    rng = np.random.default_rng(77)
    fps = request_footprints(rng)
    return _request(rng, oracle.Geometry.make(ROWS, COLS, RES), fps, 300), fps


@pytest.mark.parametrize("verify", [0, 1])
@pytest.mark.parametrize("slope", [False, True], ids=["no_robot_slope", "robot_slope"])
def test_batch_equals_map_by_map(te, ctx, batch, request_, verify, slope):
    R, fps = request_
    g, ft = te.Geometry.make(ROWS, COLS, RES), te_footprint_params(te, verify_roughness=verify)
    got = _batched(ctx, g, ft, batch, R, fps, slope, CAP)
    want = _map_by_map(ctx, g, ft, batch, R, fps, slope, CAP)
    assert_same_answers(got, want, (verify, slope))
    assert (R["kind"] < 0).sum() > 60 and (R["kind"] >= 0).sum() > 60
    assert not (R["map"] == EMPTY).any() and len(set(R["map"].tolist())) == NMAPS - 1
    assert want[0].any() and not want[0].all() and (want[3] > 0).any()
    walled = np.isin(R["map"], [1, 3, 5, 9, 11])
    assert not want[0][walled].all() and want[0][R["map"] % 4 == 0].any()


def test_batch_matches_the_cpu_oracle(te, ctx, oracle, batch, request_):
    R, fps = request_
    g, og = te.Geometry.make(ROWS, COLS, RES), oracle.Geometry.make(ROWS, COLS, RES)
    for verify in (0, 1):
        ft = te_footprint_params(te, verify_roughness=verify)
        fo = oracle.FootprintParams.yaml_defaults()
        fo.verify_roughness = verify
        got = _batched(ctx, g, ft, batch, R, fps, True, CAP)
        for k in (1, 2):
            idx = np.nonzero(R["map"] == k)[0]
            S = subset(R, idx)
            fb, fx = footprint_arrays(S, fps)
            want = po.check_request(og, fo, _one(batch, k), S["begin"], S["poses"], S["radius"], footprint_begin=fb, footprint_xyz=fx,
                                    conservative=S["cons"], cup=S["cup"], capacity=CAP)
            assert_same_answers(tuple(a[idx] for a in got), want, ("oracle", verify, k))
            assert want[0].any() and not want[0].all()


def test_each_map_has_its_own_memo(te, ctx):
    """The same paths on two maps, one cell blocked on map 0 only: each copy gets its own map's answer.  With one memo for the
    batch, whichever copy ran second would read the other map's memo byte for that cell."""
    n, res = 64, 0.25       # dyadic: cell centres are exact
    g = te.Geometry.make(n, n, res)
    ft = te.FootprintParams.yaml_defaults()
    ft.max_gap_width, ft.offset, ft.traversability_default = 0.1, 0.5, 0.3   # one zero-slope cell blocks (checkForSlope)
    one = np.ones((2, n, n), np.float32)
    B = dict(traversability=one * 0.5, slope=one.copy(), step=one.copy(), elevation=one * 0, roughness=one.copy(),
             robot_slope=one.copy())
    B["slope"][0, 32, 32] = 0.0   # (column 32, row 32) of map 0
    x = (0.5 * n * res - 0.5 * res) - res * 32
    pose = [x, x, 0.0, 0.0, 0.0, 0.0, 1.0]
    seg = [[x + 0.6, x, 0.0, 0.0, 0.0, 0.0, 1.0], [x - 0.6, x, 0.0, 0.0, 0.0, 0.0, 1.0]]
    # per map: a circular pose, a circular segment, a polygonal pose and a polygonal segment across the cell
    paths = [[pose], seg, [pose], seg] * 2
    R = dict(begin=np.cumsum([0] + [len(p) for p in paths]).astype(np.int32),
             poses=np.asarray([p for path in paths for p in path], np.float64), radius=np.full(8, 0.3),
             kind=np.asarray([-1, -1, 0, 0] * 2), cons=np.zeros(8, np.uint8), cup=np.zeros(8, np.uint8))
    fps = [np.asarray(YAML, np.float32)]
    for order in ([0, 0, 0, 0, 1, 1, 1, 1], [1, 1, 1, 1, 0, 0, 0, 0]):
        R["map"] = np.asarray(order, np.int32)
        got = _batched(ctx, g, ft, B, R, fps, False, CAP, nmaps=2)
        for k in (0, 1):
            idx = np.nonzero(R["map"] == k)[0]
            want = _single(ctx, g, ft, _one(B, k), subset(R, idx), fps, False, CAP)
            assert_same_answers(tuple(a[idx] for a in got), want, (order, k))
            assert (want[0] == (1 if k == 1 else 0)).all(), (order, k, want[0])


def _device(B):
    import torch
    return {k: torch.from_numpy(v).cuda() for k, v in B.items()}


def _request_device(R, fps):
    import torch
    fb, fx = footprint_arrays(R, fps)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    D = {k: dev(R[k]) for k in ("begin", "poses", "radius", "cons", "cup", "map")}
    D["fb"], D["fx"] = dev(fb), dev(fx)
    return D


def _run_device(ctx, g, ft, Bd, D, nmaps, slope, cap=CAP):
    import torch
    m = int(D["begin"].numel()) - 1
    out = dict(is_safe=torch.full((m,), 7, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.full((m,), -1.0, dtype=torch.float64, device="cuda"),
               area_out=torch.full((m,), -1.0, dtype=torch.float64, device="cuda"),
               untraversable_count=torch.full((m,), 99, dtype=torch.int32, device="cuda"),
               untraversable_xy=torch.zeros((m, cap, 2), dtype=torch.float64, device="cuda"))
    ctx.check_footprint_request_batched(g, ft, nmaps, Bd["traversability"], Bd["slope"], Bd["step"], Bd["elevation"], D["map"],
                                        D["begin"], D["poses"], D["radius"], D["fb"], D["fx"], max_footprint_vertices=16,
                                        robot_slope=Bd["robot_slope"] if slope else None,
                                        roughness=Bd["roughness"] if ft.verify_roughness else None, conservative=D["cons"],
                                        compute_untraversable_polygon=D["cup"], memory=1, untraversable_capacity=cap, **out)
    torch.cuda.synchronize()
    return tuple(out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out", "untraversable_count", "untraversable_xy"))


def test_device_memory_on_a_torch_stream(te, batch, request_):
    """TE_MEM_DEVICE equals TE_MEM_HOST; a path on a map outside the batch gets 0 / NaN / NaN / -1 and changes no other path."""
    import torch
    R, fps = request_
    g, ft = te.Geometry.make(ROWS, COLS, RES), te_footprint_params(te, verify_roughness=1)
    ctx = te.Context(0)
    try:
        want = _batched(ctx, g, ft, batch, R, fps, True, CAP)
        Bd = _device(batch)
        bad = np.concatenate([np.nonzero(R["kind"] < 0)[0][:2], np.nonzero(R["kind"] >= 0)[0][:2]])   # circular and polygonal
        Rb = dict(R, map=R["map"].copy(), cup=R["cup"].copy())
        Rb["map"][bad] = [NMAPS, -1, NMAPS + 100, -7]
        Rb["cup"][bad] = 1
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            got = _run_device(ctx, g, ft, Bd, _request_device(R, fps), NMAPS, True)
            marked = _run_device(ctx, g, ft, Bd, _request_device(Rb, fps), NMAPS, True)
        ctx.set_stream(None)
        assert_same_answers(got, want, "device")
        assert (marked[0][bad] == 0).all() and np.isnan(marked[1][bad]).all() and np.isnan(marked[2][bad]).all()
        assert (marked[3][bad] == -1).all()
        ok = np.ones(len(R["kind"]), bool)
        ok[bad] = False
        assert_same_answers(tuple(a[ok] for a in marked), tuple(a[ok] for a in want), "neighbours")
    finally:
        ctx.close()


def test_a_batch_of_one(te, ctx, batch, request_):
    R, fps = request_
    g, ft = te.Geometry.make(ROWS, COLS, RES), te_footprint_params(te, verify_roughness=1)
    R1 = dict(R, map=np.zeros(len(R["kind"]), np.int32))
    got = _batched(ctx, g, ft, {k: v[3:4] for k, v in batch.items()}, R1, fps, True, CAP, nmaps=1)
    want = _single(ctx, g, ft, _one(batch, 3), R, fps, True, CAP)
    assert_same_answers(got, want, "nmaps = 1")


def test_batched_chain_then_batched_request(te, ctx, request_):
    """te_chain_batched -> te_check_footprint_request_batched in device memory equals te_chain + te_check_footprint_request map by
    map."""
    import torch
    R, fps = request_
    n = NMAPS
    g, cp, ft = te.Geometry.make(ROWS, COLS, RES), te.ChainParams.yaml_defaults(0), te_footprint_params(te)
    z = torch.from_numpy(np.stack([np.ascontiguousarray(walled_terrain(ROWS, COLS, RES, k % 4, 900 + k).T) for k in range(n)])).cuda()
    ctx.set_stream(None)
    slope, step, rough, trav = (torch.empty((n, COLS, ROWS), dtype=torch.float32, device="cuda") for _ in range(4))
    ctx.chain_batched(g, cp, n, z, slope, step, rough, trav, te.MEM_DEVICE)
    Bd = dict(traversability=trav, slope=slope, step=step, elevation=z, roughness=rough, robot_slope=None)
    got = _run_device(ctx, g, ft, Bd, _request_device(R, fps), n, False)
    want = [np.zeros(len(R["kind"]), np.uint8), np.zeros(len(R["kind"])), np.zeros(len(R["kind"])),
            np.zeros(len(R["kind"]), np.int32), np.zeros((len(R["kind"]), CAP, 2))]
    for k in range(n):
        idx = np.nonzero(R["map"] == k)[0]
        if not len(idx):
            continue
        one = [torch.empty((COLS, ROWS), dtype=torch.float32, device="cuda") for _ in range(4)]
        ctx.chain(g, cp, z[k], *one, te.MEM_DEVICE)
        S = subset(R, idx)
        Ld = dict(traversability=one[3], slope=one[0], step=one[1], elevation=z[k], roughness=one[2], robot_slope=None)
        Dk = _request_device(dict(S, map=np.zeros(len(idx), np.int32)), fps)
        m = len(idx)
        out = dict(is_safe=torch.zeros(m, dtype=torch.uint8, device="cuda"),
                   traversability_out=torch.zeros(m, dtype=torch.float64, device="cuda"),
                   area_out=torch.zeros(m, dtype=torch.float64, device="cuda"),
                   untraversable_count=torch.zeros(m, dtype=torch.int32, device="cuda"),
                   untraversable_xy=torch.zeros((m, CAP, 2), dtype=torch.float64, device="cuda"))
        ctx.check_footprint_request(g, ft, Ld["traversability"], Ld["slope"], Ld["step"], Ld["elevation"], Dk["begin"], Dk["poses"],
                                    Dk["radius"], Dk["fb"], Dk["fx"], max_footprint_vertices=16, conservative=Dk["cons"],
                                    compute_untraversable_polygon=Dk["cup"], memory=te.MEM_DEVICE, untraversable_capacity=CAP, **out)
        torch.cuda.synchronize()
        for o, key in zip(want, ("is_safe", "traversability_out", "area_out", "untraversable_count", "untraversable_xy")):
            o[idx] = out[key].cpu().numpy()
    assert_same_answers(got, tuple(want), "pipeline")
    assert want[0].any() and not want[0].all()


def test_launch_count_does_not_depend_on_the_batch(te, ctx, batch, request_):
    R, fps = request_
    g, ft = te.Geometry.make(ROWS, COLS, RES), te_footprint_params(te)
    counts = []
    for nmaps in (1, NMAPS):
        Rn = dict(R, map=R["map"] % nmaps)
        for cap in (None, CAP):
            before = ctx.stats()[0]
            _batched(ctx, g, ft, {k: v[:nmaps] for k, v in batch.items()}, Rn, fps, True, cap, nmaps=nmaps)
            counts.append(ctx.stats()[0] - before)
    assert counts == [3, 3, 3, 3], counts


def test_error_codes(te, ctx, batch, request_):
    R, fps = request_
    g, ft = te.Geometry.make(ROWS, COLS, RES), te_footprint_params(te)

    def code(path_map=None, **kw):
        fb, fx = footprint_arrays(R, fps)
        B = kw.pop("B", batch)
        try:
            ctx.check_footprint_request_batched(kw.pop("g", g), ft, kw.pop("nmaps", NMAPS), B["traversability"], B["slope"], B["step"],
                                                B["elevation"], path_map, R["begin"], R["poses"], R["radius"], fb, fx, **kw)
        except te.TEError as err:
            return err.code
        return 0

    assert code(R["map"]) == 0
    assert code(R["map"], nmaps=0) == -1 and code(R["map"], nmaps=-1) == -1
    assert code(None) == -1                                  # a null path_map
    bad = R["map"].copy()
    bad[10] = NMAPS
    assert code(bad) == -1                                   # host memory: a map outside the batch
    bad[10] = -1
    assert code(bad) == -1
    assert (R["map"] == NMAPS - 1).any() and code(R["map"], nmaps=NMAPS - 1) == -1   # map 11 is outside a batch of 11
    assert code(R["map"], B=dict(batch, slope=None)) == -2   # a layer missing
    gw = te.Geometry.make(ROWS, COLS, RES)
    gw.start_row, gw.start_col = 3, 4
    assert code(R["map"], g=gw) == -4                        # a batch takes maps in default order only
