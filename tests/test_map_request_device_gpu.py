"""te_map_check_footprint_request_device: a request on a te_map with every array in device memory.  Unless a case says otherwise,
every output, the traversability_footprint cache after each request and request_stats must be bit-identical to what the host
entry (te_map_check_footprint_request(_batched)) returns and leaves on a twin te_map holding the same layers."""
import ctypes as C

import numpy as np
import pytest

import paths_oracle as po
import synth
from helpers import chain_layers, footprint_arrays, mixed_request, request_footprints, same, same_polygons

pytestmark = pytest.mark.gpu

CAP = 64
BIG = 1 << 22   # max_checks that no request here reaches
BAD_ARG = -1
FILTER = ("traversability", "slope", "step", "elevation")


@pytest.fixture(autouse=True)
def _close_maps(ctx, monkeypatch):
    """Every te_map a test opens is destroyed when it ends, failed or not, while the context still exists."""
    made, real = [], ctx.map
    monkeypatch.setattr(ctx, "map", lambda: made.append(real()) or made[-1])
    yield
    for m in made:
        m.close()


def _setup(te, oracle, rows=200, cols=180, res=0.02, seed=61):
    z = synth.terrain(rows, cols, res, seed, "mixed")
    og, g = oracle.Geometry.make(rows, cols, res), te.Geometry.make(rows, cols, res)
    L, rs = chain_layers(oracle, og, z, seed)
    return og, g, L, rs


def _params(te, oracle, verify=0):
    ft, fo = te.FootprintParams.yaml_defaults(), oracle.FootprintParams.yaml_defaults()
    ft.verify_roughness = fo.verify_roughness = verify
    return ft, fo


def _twins(ctx, g, L, rough=None, robot_slope=None):
    """A te_map for the host entry and one for the device entry, holding the same layers."""
    out = []
    for _ in range(2):
        m = ctx.map()
        m.set_layers(g, *(L[k] for k in FILTER), roughness=rough, robot_slope=robot_slope)
        out.append(m)
    return out


def _subset(R, idx):
    b = R["begin"]
    idx = np.asarray(idx, dtype=np.int64)
    begin = np.concatenate([[0], np.cumsum(b[idx + 1] - b[idx])]).astype(np.int32)
    poses = np.concatenate([R["poses"][b[q]:b[q + 1]] for q in idx]) if len(idx) else np.zeros((0, 7))
    S = dict(begin=begin, poses=poses)
    for k in ("radius", "kind", "cons", "cup", "map"):
        if k in R:
            S[k] = R[k][idx]
    return S


def _host(m, ft, R, fps, batched=False):
    fb, fx = footprint_arrays(R, fps)
    kw = dict(max_footprint_vertices=16, conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=CAP)
    if batched:
        return m.check_footprint_request_batched(ft, R["map"], R["begin"], R["poses"], R["radius"], fb, fx, **kw)
    return m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, **kw)


def _prepare(m, ft, R, fps, max_checks=BIG, batched=False, path_map=None, poses=None):
    """The request's device arrays; returns (run, fetch): the call alone, and the outputs as numpy arrays.  `poses` (default
    R["poses"]) may hold poses outside every path."""
    import torch
    fb, fx = footprint_arrays(R, fps)
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    n = len(R["begin"]) - 1
    out = dict(is_safe=torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
               area_out=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
               untraversable_count=torch.full((n,), 99, dtype=torch.int32, device="cuda"),
               untraversable_xy=torch.zeros((n, CAP, 2), dtype=torch.float64, device="cuda"))
    pm = path_map if path_map is not None else (dev(R["map"], np.int32) if batched else None)
    args = (dev(R["begin"], np.int32), dev(R["poses"] if poses is None else poses, np.float64), dev(R["radius"], np.float64),
            dev(fb, np.int32), dev(fx, np.float32))
    kw = dict(max_checks=max_checks, path_map=pm, max_footprint_vertices=16, conservative=dev(R["cons"], np.uint8),
              compute_untraversable_polygon=dev(R["cup"], np.uint8), untraversable_capacity=CAP, **out)
    torch.cuda.synchronize()

    def run():
        m.check_footprint_request_device(ft, *args, **kw)

    def fetch():
        torch.cuda.synchronize()
        return tuple(out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out", "untraversable_count",
                                                     "untraversable_xy"))
    return run, fetch


def _device(m, ft, R, fps, max_checks=BIG, batched=False, path_map=None, poses=None):
    """The request in device memory; returns the outputs as numpy arrays."""
    run, fetch = _prepare(m, ft, R, fps, max_checks, batched, path_map, poses)
    run()
    return fetch()


def _same_out(got, want, what=""):
    assert np.array_equal(got[0], want[0]), (what, np.nonzero(got[0] != want[0])[0][:10])
    assert same(got[1], want[1]) and same(got[2], want[2]), what
    same_polygons(got[3], got[4], want[3], want[4], what)


def _same_cache(a, b, what="cache"):
    equal = a.view(np.uint32) == b.view(np.uint32)
    assert equal.all(), (what, int(np.sum(~equal)))


def _both(H, D, ft, R, fps, batched=False, max_checks=BIG):
    """One request on the host twin and the device twin; asserts outputs, caches and request_stats are identical."""
    want = _host(H, ft, R, fps, batched)
    got = _device(D, ft, R, fps, max_checks, batched)
    _same_out(got, want)
    _same_cache(D.get_footprint(), H.get_footprint())
    assert D.request_stats() == H.request_stats()
    return got


def _repeat(R, idx):
    return _subset(R, idx)


@pytest.mark.parametrize("verify,slope", [(0, False), (1, True), (1, False), (0, True)])
def test_request_sequence_equals_host(te, ctx, oracle, verify, slope):
    og, g, L, rs = _setup(te, oracle)
    ft, fo = _params(te, oracle, verify)
    H, D = _twins(ctx, g, L, rough=L["roughness"], robot_slope=rs if slope else None)
    rng = np.random.default_rng(7 + verify)
    fps = request_footprints(rng)
    R1 = mixed_request(rng, og, 60, fps, circular=0.6, cap_path=False)
    R2 = mixed_request(rng, og, 80, fps, circular=0.7, planner=True, cap_path=False)
    seq = (R1, _repeat(R1, rng.permutation(len(R1["kind"]))), R2, _repeat(R2, np.arange(len(R2["kind"])) // 2))
    cache = po.empty_cache(og)
    OL = dict(L, robot_slope=rs if slope else None)
    for k, R in enumerate(seq):
        got = _both(H, D, ft, R, fps)
        if k == 0:   # the device entry against the sequential CPU oracle directly
            fb, fx = footprint_arrays(R, fps)
            want = po.check_request(og, fo, OL, R["begin"], R["poses"], R["radius"], fb, fx, conservative=R["cons"], cup=R["cup"],
                                    cache=cache, capacity=CAP)
            _same_out(got, want, "oracle")
            assert np.array_equal(D.get_footprint().view(np.uint32), cache.view(np.uint32)) or \
                same(D.get_footprint().astype(np.float64), cache.astype(np.float64))
    cand, keys, stored = D.request_stats()
    assert 0 < keys <= cand and stored <= keys


def test_annulus_blocker_revisit_and_single_poses_in_one_cell(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, seed=62)
    ft, _ = _params(te, oracle)
    H, D = _twins(ctx, g, L)
    rng = np.random.default_rng(9)
    n = 600
    xy = rng.uniform([-1.8, -1.6], [1.8, 1.6], (n, 2))
    res = og.resolution
    xy2 = (np.floor(xy / res) + rng.uniform(0.05, 0.95, (n, 2))) * res
    poses = np.zeros((2 * n, 7))
    poses[:n, :2], poses[n:, :2], poses[:, 6] = xy, xy2, 1.0
    order = rng.permutation(2 * n)   # same-cell poses close together, so that windows hold several
    poses = poses[np.argsort(np.floor(poses[:, 0] / (4 * res)) * 1e6 + order)]
    R = dict(begin=np.arange(2 * n + 1, dtype=np.int32), poses=poses, radius=np.full(2 * n, 0.1), kind=np.full(2 * n, -1),
             cons=np.zeros(2 * n, np.uint8), cup=(rng.random(2 * n) < 0.5).astype(np.uint8))
    first = _both(H, D, ft, R, [])
    second = _both(H, D, ft, R, [])
    assert np.sum((first[0] == 0) & (second[0] == 1)) > 0   # unsafe first, safe when asked again


def test_zero_mean_circle_then_fails(te, ctx, oracle):
    rows = cols = 64
    g = te.Geometry.make(rows, cols, 0.05)
    ones = np.ones((rows, cols), np.float32, order="F")
    L = dict(traversability=np.zeros((rows, cols), np.float32, order="F"), slope=ones, step=ones, elevation=0 * ones)
    ft, _ = _params(te, oracle)
    H, D = _twins(ctx, g, L)
    poses = np.array([[0.1, 0.2, 0, 0, 0, 0, 1.0]] * 3)
    R = dict(begin=np.arange(4, dtype=np.int32), poses=poses, radius=np.full(3, 0.2), kind=np.full(3, -1), cons=np.zeros(3, np.uint8),
             cup=np.ones(3, np.uint8))
    a = _both(H, D, ft, R, [])
    assert a[0][0] == 1 and a[1][0] == 0.0 and a[0][1] == 0 and a[3][1] == 20   # the second reads the stored 0 in one window


def _line_path(og, x0, y0, x1, y1, n):
    t = np.linspace(0.0, 1.0, n)
    p = np.zeros((n, 7))
    p[:, 0], p[:, 1], p[:, 6] = x0 + t * (x1 - x0), y0 + t * (y1 - y0), 1.0
    return p


def test_back_and_forth_and_failures_across_windows(te, ctx, oracle):
    """A path that goes back and forth along one line (its own centres repeat inside a window), and many straight paths of every
    length through obstacles: failures land on every lane of a window, followed by paths over the failed paths' dropped cells."""
    og, g, L, rs = _setup(te, oracle, seed=64)
    ft, _ = _params(te, oracle)
    H, D = _twins(ctx, g, L)
    rng = np.random.default_rng(21)
    paths = [np.concatenate([_line_path(og, -1.2, -0.3, 1.2, -0.3, 2), _line_path(og, 1.2, -0.3, -1.2, -0.3, 2),
                             _line_path(og, -1.2, -0.3, 0.4, -0.3, 2)])]
    for k in range(160):
        x0, y0 = rng.uniform(-1.8, 1.8), rng.uniform(-1.6, 1.6)
        ln = 0.08 * (1 + k % 40) * 4 * og.resolution / 0.08   # 1 .. 40 checked cells
        a = rng.uniform(0, 2 * np.pi)
        paths.append(_line_path(og, x0, y0, x0 + ln * np.cos(a), y0 + ln * np.sin(a), int(rng.integers(2, 4))))
    begin = np.concatenate([[0], np.cumsum([len(p) for p in paths])]).astype(np.int32)
    n = len(paths)
    R = dict(begin=begin, poses=np.concatenate(paths), radius=rng.choice([0.05, 0.1, 0.2], n), kind=np.full(n, -1),
             cons=np.zeros(n, np.uint8), cup=(rng.random(n) < 0.5).astype(np.uint8))
    first = _both(H, D, ft, R, [])
    assert (first[0] == 0).sum() > 10 and (first[0] == 1).sum() > 10
    _both(H, D, ft, _subset(R, rng.permutation(n)), [])
    _both(H, D, ft, _subset(R, np.arange(n)[::-1]), [])


def test_batch_equals_host_batched(te, ctx, oracle):
    rows, cols, res, nmaps = 160, 150, 0.02, 8
    g = te.Geometry.make(rows, cols, res)
    z = np.stack([synth.terrain(rows, cols, res, 90 + k, "mixed") for k in range(nmaps)])
    cp = te.ChainParams.yaml_defaults(0)
    H, D = ctx.map(), ctx.map()
    for m in (H, D):
        m.chain_batched(g, cp, nmaps, z)
    ft, _ = _params(te, oracle)
    og = oracle.Geometry.make(rows, cols, res)
    rng = np.random.default_rng(23)
    fps = request_footprints(rng)
    used = [0, 1, 3, 4, 6, 7]   # maps 2 and 5 have no paths
    for planner in (False, True, False):
        R = mixed_request(rng, og, 90, fps, circular=0.7, planner=planner, cap_path=False)
        R["map"] = np.asarray(rng.choice(used, len(R["kind"])), np.int32)
        R["map"][:len(used)] = used
        if not planner:   # a cell first touched on two maps: paths 1 and 3 are the same single pose, on maps 0 and 1
            R["kind"][[1, 3]], R["radius"][[1, 3]], R["map"][[1, 3]] = -1, 0.2, [0, 1]
            R["poses"][R["begin"][3]] = R["poses"][R["begin"][1]]
        _both(H, D, ft, R, fps, batched=True)


def test_unchecked_paths_in_device_memory(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, seed=65)
    ft, _ = _params(te, oracle)
    rng = np.random.default_rng(25)
    fps = request_footprints(rng)
    R = mixed_request(rng, og, 60, fps, circular=0.8, cap_path=False)
    n = len(R["kind"])
    bad_at = [3, 10, 17, 30, 44]
    parts = []
    for q in range(n):
        if q in bad_at:
            parts.append(("bad", bad_at.index(q)))
        parts.append(("ok", q))
    # the whole request: every good path, and a bad circular path at each of bad_at
    idx = [q for kind, q in parts if kind == "ok"]
    good = _subset(R, idx)
    B = dict(begin=[0], poses=[], radius=[], kind=[], cons=[], cup=[], map=[])
    bads = []
    for kind, q in parts:
        if kind == "ok":
            b0, b1 = R["begin"][q], R["begin"][q + 1]
            B["poses"].extend(R["poses"][b0:b1]); B["radius"].append(R["radius"][q]); B["kind"].append(R["kind"][q])
            B["cons"].append(R["cons"][q]); B["cup"].append(R["cup"][q]); B["map"].append(0)
        else:
            j = q
            p = np.array([[0.1 * j, -0.2, 0, 0, 0, 0, 1.0], [0.1 * j + 0.3, 0.1, 0, 0, 0, 0, 1.0]])
            r = [np.nan, -0.1, 128.5 * og.resolution, 0.1, 0.1][j]
            if j == 3:
                p[1, 1] = np.nan
            B["poses"].extend(p); B["radius"].append(r); B["kind"].append(-1)
            B["cons"].append(0); B["cup"].append(1); B["map"].append(5 if j == 4 else 0)
            bads.append(len(B["kind"]) - 1)
        B["begin"].append(len(B["poses"]))
    B = {k: np.asarray(v) for k, v in B.items()}
    B["begin"] = B["begin"].astype(np.int32)
    B["cons"], B["cup"] = B["cons"].astype(np.uint8), B["cup"].astype(np.uint8)
    H, D = _twins(ctx, g, L)
    import torch
    pm = torch.from_numpy(B["map"].astype(np.int32)).cuda()   # one map: a path on map 5 is outside it
    got = _device(D, ft, B, fps, path_map=pm)
    want = _host(H, ft, good, fps)
    keep = np.setdiff1d(np.arange(len(B["kind"])), bads)
    _same_out(tuple(a[keep] for a in got), want)
    assert (got[0][bads] == 0).all() and np.isnan(got[1][bads]).all() and np.isnan(got[2][bads]).all()
    assert (got[3][bads] == -1).all()
    _same_cache(D.get_footprint(), H.get_footprint())
    assert D.request_stats() == H.request_stats()


def test_capacity_prefix(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, seed=66)
    ft, _ = _params(te, oracle)
    rng = np.random.default_rng(27)
    fps = request_footprints(rng)
    R = mixed_request(rng, og, 80, fps, circular=0.7, planner=True, cap_path=False)
    circ = np.nonzero(R["kind"] < 0)[0]
    poly = np.nonzero(R["kind"] >= 0)[0]
    H, D = _twins(ctx, g, L)
    seen_cut = False
    for max_checks in (0, 40, 300, 1500, BIG):
        H.clear_footprint()
        D.clear_footprint()
        got = _device(D, ft, R, fps, max_checks)
        answered = ~np.isnan(got[1][circ])
        k = int(answered.sum())
        assert answered[:k].all() and not answered[k:].any(), "the answered circular paths are a prefix"
        if max_checks == 0:
            assert k == 0
        seen_cut |= 0 < k < len(circ)
        cut = circ[k:]
        assert (got[0][cut] == 0).all() and np.isnan(got[2][cut]).all() and (got[3][cut][R["cup"][cut] == 1] == -1).all()
        kept = np.sort(np.concatenate([poly, circ[:k]]))
        want = _host(H, ft, _subset(R, kept), fps)
        _same_out(tuple(a[kept] for a in got), want)
        _same_cache(D.get_footprint(), H.get_footprint())
        assert D.request_stats() == H.request_stats()
    assert seen_cut


def _kernels(ctx, m, ft, R, fps, batched=False):
    """The CUDA kernels one device request runs (torch.profiler, memsets and copies left out) and its te_get_stats delta."""
    import torch
    run, fetch = _prepare(m, ft, R, fps, batched=batched)
    run()   # warm-up: workspace and ring table
    fetch()
    a = ctx.stats()[0]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    counted = ctx.stats()[0] - a
    names = sorted(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and not e.name.startswith(("Memset", "Memcpy", "[memory]")))
    return names, counted


def test_launches_fixed(te, ctx, oracle):
    """The same kernels, each launched once, for 1 and 1 000 paths and for 1 and 8 maps: none of the grids' counts depends on the
    request (a grid's size may)."""
    og, g, L, rs = _setup(te, oracle, seed=67)
    ft, _ = _params(te, oracle)
    rng = np.random.default_rng(29)
    fps = request_footprints(rng)
    _, D = _twins(ctx, g, L)
    R = mixed_request(rng, og, 1000, [], circular=1.0, planner=True, cap_path=False)
    k1, c1 = _kernels(ctx, D, ft, _subset(R, np.arange(1)), [])
    k1000, c1000 = _kernels(ctx, D, ft, R, [])
    assert k1 == k1000 and c1 == c1000, (k1, k1000)
    assert any("k_req_replay" in k for k in k1) and any("k_map_eval_circles_dev" in k for k in k1)
    Rm = mixed_request(rng, og, 200, fps, circular=0.5, planner=True, cap_path=False)
    Rm["kind"][0], Rm["kind"][1] = -1, 0
    assert _kernels(ctx, D, ft, _subset(Rm, np.arange(2)), fps) == _kernels(ctx, D, ft, Rm, fps)
    B = ctx.map()
    z = np.stack([synth.terrain(64, 64, 0.02, 95 + k, "mixed") for k in range(8)])
    B.chain_batched(te.Geometry.make(64, 64, 0.02), te.ChainParams.yaml_defaults(0), 8, z)
    S = ctx.map()
    S.chain(te.Geometry.make(64, 64, 0.02), te.ChainParams.yaml_defaults(0), z[0])
    og64 = oracle.Geometry.make(64, 64, 0.02)
    R8 = mixed_request(rng, og64, 50, [], circular=1.0, planner=True, cap_path=False)
    R8["map"] = np.asarray(rng.integers(0, 8, 50), np.int32)
    R1 = dict(R8, map=np.zeros(50, np.int32))
    assert _kernels(ctx, B, ft, R8, [], batched=True) == _kernels(ctx, S, ft, R1, [], batched=True)


def test_poses_outside_every_path(te, ctx, oracle):
    """Poses before path_begin[0] (the host entry accepts them) and after path_begin[npaths] (a preallocated pose buffer) belong
    to no path: the request equals the host entry's on the same path_begin."""
    og, g, L, rs = _setup(te, oracle, seed=70)
    ft, _ = _params(te, oracle)
    rng = np.random.default_rng(33)
    fps = request_footprints(rng)
    H, D = _twins(ctx, g, L, robot_slope=rs)
    for planner in (False, True):
        R = mixed_request(rng, og, 50, fps, circular=0.7, planner=planner, cap_path=False)
        R["kind"][0], R["radius"][0] = -1, 0.2   # path 0 circular: leading poses would fall to it
        lead, trail = R["poses"][-9:].copy(), R["poses"][:11].copy()
        S = dict(R, begin=(R["begin"] + len(lead)).astype(np.int32), poses=np.concatenate([lead, R["poses"]]))
        want = _host(H, ft, S, fps)   # host memory: nposes = path_begin[npaths], the leading poses included
        got = _device(D, ft, S, fps, poses=np.concatenate([S["poses"], trail]))
        _same_out(got, want)
        _same_cache(D.get_footprint(), H.get_footprint())
        assert D.request_stats() == H.request_stats()


def _cell(n, res, i):
    """grid_map's cell-centre coordinate of index i on an n-cell axis of a map centred at 0 (getPositionFromIndex)."""
    return (0.0 + (0.5 * (n * res) - 0.5 * res)) + res * (-float(i))


@pytest.mark.parametrize("lane", [0, 1, 30, 31])
def test_failure_at_window_lane_then_dropped_cells(te, ctx, oracle, lane):
    """A gate (a segment leaving the map) as entry 64 + lane of the map's list: lane `lane` of the third window fails.  The failed
    path's later segments are dropped, and the paths after it check those dropped cells, first in the same window."""
    n, res = 128, 0.05
    g = te.Geometry.make(n, n, res)
    ones = np.ones((n, n), np.float32, order="F")
    L = dict(traversability=np.full((n, n), 0.5, np.float32, order="F"), slope=ones, step=ones, elevation=0 * ones)
    ft, _ = _params(te, oracle)
    H, D = _twins(ctx, g, L)
    pose = lambda i, j: [_cell(n, res, i), _cell(n, res, j), 0, 0, 0, 0, 1.0]  # noqa: E731
    out = [0.5 * n * res + 1.0, 0.0, 0, 0, 0, 0, 1.0]
    rng = np.random.default_rng(35 + lane)
    paths = []
    nab = 5                                   # rows 20 -> 36: 17 cells, every fourth checked
    for _ in range(64 + lane - nab):          # single poses: one entry each, all traversable
        paths.append([pose(*rng.integers(10, 118, 2))])
    paths.append([pose(20, 30), pose(36, 30), out, pose(40, 50), pose(72, 50), pose(72, 80)])   # fails at its gate
    paths.append([pose(40, 50), pose(72, 50)])                  # the dropped cells, in the same window as the failure
    paths += [[pose(72, 50), pose(72, 80)], [pose(56, 50)], [pose(72, 60), pose(72, 70)]]
    paths += [[pose(*rng.integers(10, 118, 2))] for _ in range(40)]
    begin = np.concatenate([[0], np.cumsum([len(p) for p in paths])]).astype(np.int32)
    k = len(paths)
    R = dict(begin=begin, poses=np.asarray([x for p in paths for x in p], np.float64), radius=np.full(k, 0.1),
             kind=np.full(k, -1), cons=np.zeros(k, np.uint8), cup=np.ones(k, np.uint8))
    first = _both(H, D, ft, R, [])
    failed = 64 + lane - nab
    assert first[0][failed] == 0 and first[3][failed] == 0 and first[0][:failed].all() and first[0][failed + 1:].all()
    _both(H, D, ft, R, [])   # again, on the cache the first request left


def test_graph_capture_replays_the_request(te, ctx, oracle):
    import torch
    og, g, L, rs = _setup(te, oracle, seed=68)
    ft, _ = _params(te, oracle)
    rng = np.random.default_rng(31)
    fps = request_footprints(rng)
    R = mixed_request(rng, og, 60, fps, circular=0.7, cap_path=False)
    H, D = _twins(ctx, g, L)
    want = _host(H, ft, R, fps)
    fb, fx = footprint_arrays(R, fps)
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    n = len(R["kind"])
    args = (dev(R["begin"], np.int32), dev(R["poses"], np.float64), dev(R["radius"], np.float64), dev(fb, np.int32),
            dev(fx, np.float32))
    out = dict(is_safe=torch.zeros(n, dtype=torch.uint8, device="cuda"), traversability_out=torch.zeros(n, dtype=torch.float64, device="cuda"),
               area_out=torch.zeros(n, dtype=torch.float64, device="cuda"), untraversable_count=torch.zeros(n, dtype=torch.int32, device="cuda"),
               untraversable_xy=torch.zeros((n, CAP, 2), dtype=torch.float64, device="cuda"))
    kw = dict(max_checks=BIG, max_footprint_vertices=16, conservative=dev(R["cons"], np.uint8),
              compute_untraversable_polygon=dev(R["cup"], np.uint8), untraversable_capacity=CAP, **out)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    ctx.set_stream(side.cuda_stream)
    try:
        with torch.cuda.stream(side):
            D.check_footprint_request_device(ft, *args, **kw)   # warm-up: workspace, ring table, memo
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
            D.clear_footprint()
            D.check_footprint_request_device(ft, *args, **kw)
        for t in out.values():
            t.fill_(0)
        D.clear_footprint()
        side.synchronize()
        graph.replay()
        torch.cuda.synchronize()
    finally:
        ctx.set_stream(None)
    got = tuple(out[k].cpu().numpy() for k in ("is_safe", "traversability_out", "area_out", "untraversable_count", "untraversable_xy"))
    _same_out(got, want)
    _same_cache(D.get_footprint(), H.get_footprint())


def test_synchronous_errors(te, ctx, oracle):
    import torch
    og, g, L, rs = _setup(te, oracle, rows=64, cols=64, seed=69)
    ft, _ = _params(te, oracle)
    L1 = ctx._L
    m = ctx.map()
    dv = lambda a, dt: torch.from_numpy(np.asarray(a, dtype=dt)).cuda()  # noqa: E731
    pb, ps, rad = dv([0, 1], np.int32), dv([[0.0, 0, 0, 0, 0, 0, 1]], np.float64), dv([0.2], np.float64)
    fb, fx = dv([0, 0], np.int32), dv(np.zeros((0, 3)), np.float32)
    safe, tr, ar = dv([0], np.uint8), dv([0.0], np.float64), dv([0.0], np.float64)

    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731

    def call(mh=None, npaths=1, nposes=1, path_map=None, pb_=pb, safe_=safe, max_checks=100):
        return L1.te_map_check_footprint_request_device(
            mh if mh is not None else m._h, C.byref(ft), path_map, npaths, nposes, ptr(pb_), ps.data_ptr(), rad.data_ptr(), 0,
            fb.data_ptr(), fx.data_ptr(), 16, None, None, ptr(safe_), tr.data_ptr(), ar.data_ptr(), 0, None, None, max_checks)
    assert call() == BAD_ARG   # a map without layers
    m.set_layers(g, *(L[k] for k in FILTER))
    assert call() == 0
    torch.cuda.synchronize()
    assert call(npaths=-1) == BAD_ARG
    assert call(nposes=-1) == BAD_ARG
    assert call(pb_=None) == BAD_ARG
    assert call(safe_=None) == BAD_ARG
    assert call(max_checks=-1) == BAD_ARG
    B = ctx.map()
    B.set_layers_batched(g, 2, *(np.stack([L[k]] * 2) for k in FILTER))
    assert call(mh=B._h) == BAD_ARG and "path_map" in L1.te_last_error().decode()
    torch.cuda.synchronize()
