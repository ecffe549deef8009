"""te_map_at_poses: GridMap::atPosition for every layer a te_map holds, at robot-frame points around poses, in one launch.  Every
value must be, bit for bit, the CPU restatement (tests/at_poses_oracle.cpp, teo_at_poses) applied to te_map_get_layers' output; host
and device memory must agree; a start index, a batch at several positions and graph capture must change nothing."""
import numpy as np
import pytest

import at_poses_oracle as so
import synth
from helpers import assert_same_bits, bits, footprint_arrays, mixed_request, quaternion, request_footprints
from map_helpers import all_layer_names, close_maps  # noqa: F401

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, POS = 640, 512, 0.04, (1.3, -0.7)
POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]   # robot_footprint_parameter.yaml:3
BAD_ARG, MISSING_LAYER, UNSUPPORTED = -1, -2, -4
NAN_BITS = 0x7fc00000


def _carried(rng, rows, cols):
    """robot_slope and the seven carried layers, with NaNs of several payloads, infinities and -0.0 among them."""
    lay = {n: rng.normal(size=(rows, cols)).astype(np.float32) for n in ("robot_slope", "upper_bound", "lower_bound", "variance",
                                                                         "horizontal_variance_x", "horizontal_variance_y",
                                                                         "horizontal_variance_xy", "time")}
    for n, a in lay.items():
        u = a.view(np.uint32)
        r = rng.random(a.shape)
        u[r < 0.02] = 0x7fc00000 | rng.integers(0, 1 << 22, size=int((r < 0.02).sum())).astype(np.uint32)
        u[(r >= 0.02) & (r < 0.03)] = 0xffc12345
        a[(r >= 0.03) & (r < 0.035)] = np.inf
        a[(r >= 0.035) & (r < 0.04)] = -np.inf
        a[(r >= 0.04) & (r < 0.045)] = -0.0
    return lay


def _full_map(te, ctx, start=(0, 0), seed=5):
    """A ROWS x COLS map holding every layer bit: the chain, robot_slope and the carried layers, a cache a request filled in part,
    and traversability_x / _rot.  start: the same map given with that circular-buffer start index."""
    g = te.Geometry.make(ROWS, COLS, RES, POS)
    g.start_row, g.start_col = start
    wrap = lambda a: np.asfortranarray(np.roll(a, start, axis=(0, 1)))  # noqa: E731  unwrapped layer -> buffer order
    z = synth.terrain(ROWS, COLS, RES, seed, "mixed", POS)
    rng = np.random.default_rng(seed)
    m = ctx.map()
    m.chain(g, te.ChainParams.yaml_defaults(0), wrap(z))
    lay = _carried(rng, ROWS, COLS)
    m.carry_layers(list(lay), [wrap(a) for a in lay.values()])
    ft = te.FootprintParams.yaml_defaults()
    fps = request_footprints(rng)
    R = mixed_request(rng, g, 80, fps, cap_path=False)
    fb, fx = footprint_arrays(R, fps)
    m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, max_footprint_vertices=16, conservative=R["cons"])
    m.footprint_polygon_keep(ft, POLY, 0.6)
    return m


def _poses(rng, n, center, half):
    """n poses around `center` within 1.1 * half (so some lie off the map): yawed, tilted and non-normalised quaternions, a few
    non-finite entries."""
    xy = rng.uniform(np.asarray(center) - 1.1 * np.asarray(half), np.asarray(center) + 1.1 * np.asarray(half), (n, 2))
    q = np.array([quaternion(rng, k % 3) for k in range(n)])
    p = np.concatenate([xy, rng.uniform(-1, 1, (n, 1)), q], axis=1)
    p[3, 0] = np.nan
    p[7, 1] = np.inf
    p[11, 5] = np.nan
    p[13, 6] = -np.inf
    return p


def _edge_poses(g):
    """Identity poses on cell edges and on the map's edges."""
    x0, y0 = g.position_x + 0.5 * g.length_x, g.position_y + 0.5 * g.length_y
    xs = [x0, x0 - g.length_x, x0 - RES, x0 - 17 * RES, x0 - (g.rows - 1) * RES, np.nextafter(x0 - g.length_x, np.inf)]
    ys = [y0, y0 - g.length_y, y0 - RES, y0 - 33 * RES, y0 - (g.cols - 1) * RES, np.nextafter(y0, -np.inf)]
    return np.array([[x, y, 0.0, 0.0, 0.0, 0.0, 1.0] for x in xs for y in ys])


def _pattern():
    """40 robot-frame points: a 6 x 6 grid on multiples of the resolution (cell edges for a pose on one), the origin and three
    points with z."""
    k = np.arange(-3, 3) * RES
    grid = [(a, b, 0.0) for a in k for b in k]
    return np.array(grid + [(0, 0, 0), (0.5 * RES, 0.5 * RES, 0.3), (0.3, -0.2, -0.5), (-1.0, 0.7, 0.9)], np.float32)


def _oracle_geo(oracle, g, pos=None):
    return oracle.Geometry.make(g.rows, g.cols, g.resolution, tuple(pos) if pos is not None else (g.position_x, g.position_y))


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _at_device(torch, m, names, poses, pts, pose_map=None, nl=None):
    nl = len(names) if nl is None else nl
    n, t = len(poses), len(pts)
    out = torch.full((nl * n * t,), 12345.0, dtype=torch.float32, device="cuda")
    valid = torch.full((n * t,), 7, dtype=torch.uint8, device="cuda")
    lay, v = m.at_poses(_dev(torch, poses), _dev(torch, pts), names, None if pose_map is None else _dev(torch, pose_map), out=out,
                        valid=valid, memory=1)
    torch.cuda.synchronize()
    return {k: a.cpu().numpy() for k, a in lay.items()}, v.cpu().numpy()


# ---- 1. every layer against the oracle, host and device --------------------------------------------------------------------

def test_every_layer_against_the_oracle(te, ctx, oracle):
    torch = pytest.importorskip("torch")
    m = _full_map(te, ctx)
    g = te.Geometry.make(ROWS, COLS, RES, POS)
    names = all_layer_names(te)
    L = m.get_layers(names)
    cache = L["traversability_footprint"]
    assert np.isfinite(cache).any() and np.isnan(cache).any()          # a cache the request filled in part
    rng = np.random.default_rng(1)
    poses = np.concatenate([_poses(rng, 1964, POS, (0.5 * ROWS * RES, 0.5 * COLS * RES)), _edge_poses(g)])
    pts = _pattern()
    got, valid = m.at_poses(poses, pts, names)
    assert list(got) == names                                          # bit order
    og = _oracle_geo(oracle, g)
    for n in names:
        want, wv = so.at_poses(og, L[n], poses, pts)
        assert_same_bits(got[n], want, n)
        assert np.array_equal(valid, wv), n
    assert 0.5 < valid.mean() < 0.99
    assert (bits(got["traversability"])[valid == 0] == NAN_BITS).all()
    dev, dvalid = _at_device(torch, m, names, poses, pts)
    for n in names:
        assert_same_bits(dev[n], got[n], n)
    assert np.array_equal(dvalid, valid)


# ---- 2. a start index changes nothing --------------------------------------------------------------------------------------

def test_start_index_gives_identical_outputs(te, ctx):
    names = all_layer_names(te)
    rng = np.random.default_rng(2)
    poses = _poses(rng, 600, POS, (0.5 * ROWS * RES, 0.5 * COLS * RES))
    pts = _pattern()
    a, va = _full_map(te, ctx).at_poses(poses, pts, names)
    b, vb = _full_map(te, ctx, start=(211, 97)).at_poses(poses, pts, names)
    for n in names:
        assert_same_bits(b[n], a[n], n)
    assert np.array_equal(va, vb)


# ---- 3. one point (0, 0, 0): atPosition at the poses' positions ------------------------------------------------------------

def test_single_point_is_at_position(te, ctx, oracle):
    m = _full_map(te, ctx)
    g = te.Geometry.make(ROWS, COLS, RES, POS)
    rng = np.random.default_rng(3)
    poses = _poses(rng, 3000, POS, (0.5 * ROWS * RES, 0.5 * COLS * RES))
    ok = np.isfinite(poses).all(axis=1)
    poses, xy = poses[ok], poses[ok, :2]
    got, valid = m.at_poses(poses, [(0.0, 0.0, 0.0)], ["traversability", "elevation"])
    assert np.array_equal(valid[:, 0] & np.isfinite(got["traversability"][:, 0]), m.valid_at(xy))
    # the oracle's index, read through a layer that holds it
    index = np.asfortranarray(np.arange(ROWS * COLS, dtype=np.float32).reshape(COLS, ROWS).T)
    idx, iv = so.at_poses(_oracle_geo(oracle, g), index, poses, [(0.0, 0.0, 0.0)])
    assert np.array_equal(iv, valid)
    L = m.get_layers(["traversability", "elevation"])
    k = valid[:, 0] == 1
    i, j = idx[k, 0].astype(np.int64) % ROWS, idx[k, 0].astype(np.int64) // ROWS
    assert_same_bits(got["traversability"][k, 0], L["traversability"][i, j])
    assert_same_bits(got["elevation"][k, 0], L["elevation"][i, j])


# ---- 4. a batch at several positions ---------------------------------------------------------------------------------------

def test_batch_at_positions(te, ctx):
    torch = pytest.importorskip("torch")
    n, N = 16, 256
    rng = np.random.default_rng(4)
    positions = rng.uniform(-300, 300, (n, 2)).round(3)
    z = np.stack([synth.terrain(N, N, RES, 40 + k, "mixed") for k in range(n)]).astype(np.float32)
    lay = np.stack([_carried(rng, N, N)["upper_bound"] for _ in range(n)])
    g = te.Geometry.make(N, N, RES)
    b = ctx.map()
    b.chain_batched(g, te.ChainParams.yaml_defaults(0), n, z, positions=positions)
    b.carry_layers(["upper_bound"], [lay])
    names = ["traversability", "traversability_slope", "elevation", "upper_bound"]
    per = 120
    pose_map = rng.permutation(np.repeat(np.arange(n), per)).astype(np.int32)
    half = 0.5 * N * RES
    poses = _poses(rng, len(pose_map), (0.0, 0.0), (half, half))
    poses[:, :2] += positions[pose_map]                                # each pose around its own map
    pts = _pattern()
    got, valid = b.at_poses(poses, pts, names, pose_map=pose_map)
    dev, dvalid = _at_device(torch, b, names, poses, pts, pose_map)
    assert np.array_equal(dvalid, valid)
    for k in range(n):
        s = ctx.map()
        s.chain(te.Geometry.make(N, N, RES, tuple(positions[k])), te.ChainParams.yaml_defaults(0), z[k])
        s.carry_layers(["upper_bound"], [lay[k]])
        sel = pose_map == k
        want, wv = s.at_poses(poses[sel], pts, names)
        assert np.array_equal(valid[sel], wv), k
        assert wv.any() and not wv.all()
        for nm in names:
            assert_same_bits(got[nm][sel], want[nm], (k, nm))
            assert_same_bits(dev[nm][sel], want[nm], (k, nm))


# ---- 5. uncertainty_range --------------------------------------------------------------------------------------------------

def test_uncertainty_range_is_numpy_subtraction(te, ctx):
    m = _full_map(te, ctx)
    rng = np.random.default_rng(6)
    poses = _poses(rng, 2000, POS, (0.5 * ROWS * RES, 0.5 * COLS * RES))
    got, valid = m.at_poses(poses, _pattern(), ["upper_bound", "lower_bound", "uncertainty_range"])
    k = valid == 1
    with np.errstate(invalid="ignore"):                                # Inf - Inf
        want = np.subtract(got["upper_bound"][k], got["lower_bound"][k])
    assert_same_bits(got["uncertainty_range"][k], want)
    assert np.isnan(want).sum() > 100 and len(set(bits(want)[np.isnan(want)].tolist())) > 3   # NaN payloads of both kinds
    assert (bits(got["uncertainty_range"])[~k] == NAN_BITS).all()


# ---- 6. invalid points -----------------------------------------------------------------------------------------------------

def test_invalid_points(te, ctx):
    torch = pytest.importorskip("torch")
    N = 64
    z = np.stack([synth.terrain(N, N, RES, 70 + k, "mixed") for k in range(2)]).astype(np.float32)
    b = ctx.map()
    b.chain_batched(te.Geometry.make(N, N, RES), te.ChainParams.yaml_defaults(0), 2, z, positions=[(0.0, 0.0), (10.0, 0.0)])
    poses = np.array([[0.0, 0.0, 0, 0, 0, 0, 1]] * 3 + [[5.0, 0.0, 0, 0, 0, 0, 1], [np.nan, 0, 0, 0, 0, 0, 1],
                                                        [0, 0, 0, 0, 0, np.inf, 1], [0, 0, 0, 0, 0, 0, 1], [10, 0, 0, 0, 0, 0, 1]])
    pose_map = np.array([-1, 2, 1000, 0, 0, 0, 0, 1], np.int32)
    pts = np.array([(0, 0, 0), (0.1, 0.1, 0.0)], np.float32)
    dev, dvalid = _at_device(torch, b, ["traversability", "elevation"], poses, pts, pose_map)
    assert dvalid[:7].sum() == 2 and dvalid[6].all() and dvalid[7].all()    # maps outside the batch, off-map, non-finite
    for n in dev:
        assert (bits(dev[n])[dvalid == 0] == NAN_BITS).all() and np.isfinite(dev[n][6]).all()
    # host memory: the same points on the maps inside the batch
    got, valid = b.at_poses(poses[3:], pts, ["traversability", "elevation"], pose_map=pose_map[3:])
    assert np.array_equal(valid, dvalid[3:])
    for n in got:
        assert_same_bits(got[n], dev[n][3:])


# ---- 7. errors -------------------------------------------------------------------------------------------------------------

def test_errors_write_nothing(te, ctx):
    L = te.load_library()
    N = 64
    z = synth.terrain(N, N, RES, 80, "mixed").astype(np.float32)
    m = ctx.map()
    m.chain(te.Geometry.make(N, N, RES), te.ChainParams.yaml_defaults(0), z)
    b = ctx.map()
    b.chain_batched(te.Geometry.make(N, N, RES), te.ChainParams.yaml_defaults(0), 2, np.stack([z, z]))
    empty = ctx.map()
    poses = np.array([[0, 0, 0, 0, 0, 0, 1]] * 4, np.float64)
    pts = np.zeros((3, 3), np.float32)
    out = np.full(64, 12345.0, np.float32)
    valid = np.full(12, 7, np.uint8)
    pm_bad = np.array([0, 1, 2, 0], np.int32)
    T = 1
    P, Q, O, V = poses.ctypes.data, pts.ctypes.data, out.ctypes.data, valid.ctypes.data
    cases = [
        ("no layers", empty, None, 4, P, 3, Q, T, O, V, 0, BAD_ARG),
        ("empty mask", m, None, 4, P, 3, Q, 0, O, V, 0, BAD_ARG),
        ("bit 7", m, None, 4, P, 3, Q, 1 << 7, O, V, 0, BAD_ARG),
        ("bit 18", m, None, 4, P, 3, Q, T | (1 << 18), O, V, 0, BAD_ARG),
        ("null poses", m, None, 4, None, 3, Q, T, O, V, 0, BAD_ARG),
        ("null points", m, None, 4, P, 3, None, T, O, V, 0, BAD_ARG),
        ("null out", m, None, 4, P, 3, Q, T, None, V, 0, BAD_ARG),
        ("nposes < 0", m, None, -1, P, 3, Q, T, O, V, 0, BAD_ARG),
        ("npoints 0", m, None, 4, P, 0, Q, T, O, V, 0, BAD_ARG),
        ("memory 2", m, None, 4, P, 3, Q, T, O, V, 2, BAD_ARG),
        ("null pose_map on a batch", b, None, 4, P, 3, Q, T, O, V, 0, BAD_ARG),
        ("host pose_map outside", b, pm_bad.ctypes.data, 4, P, 3, Q, T, O, V, 0, BAD_ARG),
        ("robot_slope missing", m, None, 4, P, 3, Q, T | (1 << 5), O, V, 0, MISSING_LAYER),
        ("carried layer missing", m, None, 4, P, 3, Q, 1 << 10, O, V, 0, MISSING_LAYER),
        ("uncertainty_range without bounds", m, None, 4, P, 3, Q, 1 << 15, O, V, 0, MISSING_LAYER),
        ("traversability_x missing", m, None, 4, P, 3, Q, 1 << 16, O, V, 0, MISSING_LAYER),
        ("2^31 samples", m, None, 1 << 16, P, 1 << 15, Q, T, O, V, 0, UNSUPPORTED),
    ]
    for what, mp, *args, want in cases:
        rc = L.te_map_at_poses(mp._h, *args)
        assert rc == want, (what, rc, L.te_last_error().decode())
        assert (out == 12345.0).all() and (valid == 7).all(), what
    # one below the limit is accepted up to the layer check
    assert L.te_map_at_poses(m._h, None, (1 << 16), P, (1 << 15) - 1, Q, 1 << 5, O, V, 0) == MISSING_LAYER
    with pytest.raises(te.TEError):
        m.at_poses(poses, pts, ["robot_slope"])


# ---- 8. launches -----------------------------------------------------------------------------------------------------------

def test_one_launch_per_call(te, ctx):
    torch = pytest.importorskip("torch")
    m = _full_map(te, ctx)
    rng = np.random.default_rng(8)
    poses, pts = _poses(rng, 500, POS, (0.5 * ROWS * RES, 0.5 * COLS * RES)), _pattern()
    names = all_layer_names(te)
    N = 64
    z = np.stack([synth.terrain(N, N, RES, 90 + k, "mixed") for k in range(3)]).astype(np.float32)
    b = ctx.map()
    b.chain_batched(te.Geometry.make(N, N, RES), te.ChainParams.yaml_defaults(0), 3, z, positions=[(0, 0), (5, 5), (-9, 2)])
    pm = rng.integers(0, 3, len(poses)).astype(np.int32)
    calls = [lambda: m.at_poses(poses, pts, names), lambda: m.at_poses(poses, pts, ["traversability"]),
             lambda: b.at_poses(poses, pts, ["traversability", "elevation"], pose_map=pm),
             lambda: _at_device(torch, m, names, poses, pts), lambda: _at_device(torch, b, ["elevation"], poses, pts, pm)]
    for f in calls:
        f()                                                            # per-map tables built
        n0 = ctx.stats()[0]
        f()
        assert ctx.stats()[0] - n0 == 1
    n0 = ctx.stats()[0]
    lay, valid = m.at_poses(np.zeros((0, 7)), pts, names)
    assert ctx.stats()[0] == n0 and valid.shape == (0, len(pts)) and all(a.shape == (0, len(pts)) for a in lay.values())


# ---- 9. graph capture ------------------------------------------------------------------------------------------------------

def test_graph_capture(te, oracle):
    torch = pytest.importorskip("torch")
    c = te.Context(0)
    try:
        m = c.map()
        N = 128
        z = synth.terrain(N, N, RES, 95, "mixed").astype(np.float32)
        g = te.Geometry.make(N, N, RES, (0.5, -0.25))
        m.chain(g, te.ChainParams.yaml_defaults(0), z)
        rng = np.random.default_rng(9)
        names = ["traversability", "elevation"]
        pts = _pattern()
        poses = _dev(torch, _poses(rng, 300, (0.5, -0.25), (0.5 * N * RES,) * 2))
        dpts = _dev(torch, pts)
        out = torch.empty(len(names) * 300 * len(pts), dtype=torch.float32, device="cuda")
        valid = torch.empty(300 * len(pts), dtype=torch.uint8, device="cuda")
        stream = torch.cuda.Stream()
        c.set_stream(stream.cuda_stream)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            m.at_poses(poses, dpts, names, out=out, valid=valid, memory=te.MEM_DEVICE)       # warm-up
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            m.at_poses(poses, dpts, names, out=out, valid=valid, memory=te.MEM_DEVICE)
        new = _poses(np.random.default_rng(10), 300, (0.5, -0.25), (0.5 * N * RES,) * 2)
        poses.copy_(torch.from_numpy(new))
        out.fill_(0.0)
        graph.replay()
        torch.cuda.synchronize()
        replayed, rvalid = out.cpu().numpy().copy(), valid.cpu().numpy().copy()
        c.set_stream(None)
        fresh, fvalid = m.at_poses(new, pts, names)
        assert_same_bits(replayed, np.concatenate([fresh[n].reshape(-1) for n in names]))
        assert np.array_equal(rvalid, fvalid.reshape(-1))
        want, _ = so.at_poses(_oracle_geo(oracle, g), m.get_layers(["traversability"])["traversability"], new, pts)
        assert_same_bits(fresh["traversability"], want)
        m.close()
    finally:
        c.close()
