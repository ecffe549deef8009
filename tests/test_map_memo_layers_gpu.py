"""The slope_footprint / step_footprint / roughness_footprint layers a te_map records, bit for bit against the CPU oracle
(tests/memo_layers_oracle.cpp) after sequences of requests, sweeps, clears and reloads, on every entry that reads them; and
recording changes nothing that was observable before."""
import json
import os
import zlib

import numpy as np
import pytest

import memo_layers_oracle as mo
import occupancy_oracle as oo
import synth
from helpers import (assert_same_answers, batch_request, chain_layers, footprint_arrays, footprint_params, mixed_request, request_footprints,
                     subset)
from map_helpers import CAP, ask
from helpers import wrap

pytestmark = pytest.mark.gpu

NAMES = mo.NAMES


def _setup(te, oracle, rows=160, cols=140, res=0.02, seed=81):
    z = synth.terrain(rows, cols, res, seed, "mixed", (0.0, 0.0))
    og, g = oracle.Geometry.make(rows, cols, res, (0.0, 0.0)), te.Geometry.make(rows, cols, res, (0.0, 0.0))
    L, rs = chain_layers(oracle, og, z, seed)
    return og, g, L, rs


def _map(ctx, g, L, rs=None):
    m = ctx.map()
    m.set_layers(g, L["traversability"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"], robot_slope=rs)
    return m


def _assert_layers(m, states, what=""):
    """The map's three layers (every map of a batch) equal the oracle states', bit for bit."""
    got = m.get_layers(list(NAMES))
    for name in NAMES:
        a = got[name] if len(states) > 1 else got[name][None]
        for k, s in enumerate(states):
            x, y = np.ascontiguousarray(a[k]).view(np.uint32), np.ascontiguousarray(s.memo[name]).view(np.uint32)
            assert np.array_equal(x, y), (what, name, k, int(np.sum(x != y)))


def _observable(m):
    """What a te_map showed before it recorded these layers: the memo, the cache and the request counters."""
    return m.get_memo().copy(), m.get_footprint().copy(), m.request_stats()


def _assert_same_observable(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)) and a[2] == b[2]


def _assert_cloud(m, full, elev):
    """te_map_get_point_cloud's memo-layer fields equal `full` (get_layers' host output) point by point: a point per cell of finite
    elevation (`elev`, per map in the same order as `full`), cells in column-major order."""
    layout, step, clouds = m.get_point_cloud(["elevation", *NAMES])
    for k, cloud in enumerate(clouds):
        point = np.isfinite(np.asarray(elev[k])).reshape(-1, order="F")
        for name in NAMES:
            want = np.asarray(full[name][k], np.float32).reshape(-1, order="F")[point]
            assert np.array_equal(np.asarray(cloud[name], np.float32).view(np.uint32), want.view(np.uint32)), (name, k)


@pytest.mark.parametrize("verify,slope", [(0, False), (1, True)])
def test_requests_sweeps_and_clears_match_oracle(te, ctx, oracle, verify, slope):
    og, g, L, rs = _setup(te, oracle)
    ft, fo = footprint_params(te, oracle, verify)
    OL = dict(L, robot_slope=rs if slope else None)
    m, twin = _map(ctx, g, L, rs if slope else None), _map(ctx, g, L, rs if slope else None)
    s = mo.State(og, OL)
    _assert_layers(m, [s], "fresh")
    rng = np.random.default_rng(11 + verify)
    fps = request_footprints(rng)
    for k in range(3):   # cup on and off, radius_min > 0, polygonal and circular items mixed
        R = mixed_request(rng, og, 50, fps, circular=0.6, planner=k == 2, cap_path=False)
        got = ask(m, ft, dict(R, fps=fps))
        assert_same_answers(got, ask(twin, ft, dict(R, fps=fps)))
        s.request(fo, R, fps)
        _assert_layers(m, [s], ("request", k))
        _assert_same_observable(_observable(m), _observable(twin))
    # a sweep on a partly cached map: only the prefixes of the empty centres
    assert np.array_equal(m.footprint(ft).view(np.uint32), twin.footprint(ft).view(np.uint32))
    s.sweep(fo)
    _assert_layers(m, [s], "sweep on a partly cached map")
    m.clear_footprint()
    twin.clear_footprint()
    s.clear()
    _assert_layers(m, [s], "clear keeps roughness_footprint")
    m.footprint(ft)
    s.sweep(fo)
    _assert_layers(m, [s], "sweep on an empty cache")
    R = mixed_request(rng, og, 40, fps, circular=0.8, cap_path=False)
    ask(m, ft, dict(R, fps=fps))
    s.request(fo, R, fps)
    _assert_layers(m, [s], "request after the sweep")
    m.close()
    twin.close()


def test_empty_cache_sweep_is_the_predicate_layers(te, ctx, oracle):
    og, g, L, _ = _setup(te, oracle, seed=82)
    ft, fo = footprint_params(te, oracle, 1)
    m = _map(ctx, g, L)
    m.footprint(ft)
    ref = oracle.footprint(og, fo, L["traversability"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"])
    got = m.get_layers(list(NAMES))
    for name, want in zip(NAMES, ref[1:]):
        a, b = got[name], want
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)]), name
    m.close()


def test_fixture_publishes_the_bags_nan_layers(te, ctx):
    here = os.path.dirname(os.path.abspath(__file__))
    d = np.load(os.path.join(here, "golden", "fixture_gridmap.npz"))
    meta = json.load(open(os.path.join(here, "golden", "fixture_gridmap.json")))
    g = te.Geometry.make(meta["rows"], meta["cols"], meta["resolution"])
    m = ctx.map()
    m.chain(g, te.ChainParams.yaml_defaults(0), np.asfortranarray(d["elevation"]))
    got = m.get_layers(["slope_footprint", "step_footprint"])
    for name in ("slope_footprint", "step_footprint"):
        assert "%08x" % zlib.crc32(np.asfortranarray(got[name]).tobytes(order="F")) == meta["crc32"][name]
    m.close()


def test_batch_each_key_change_reload_and_readers(te, ctx, oracle):
    og, g, L, rs = _setup(te, oracle, rows=96, cols=88, seed=83)
    n = 3
    Ls = [L]
    for k in range(1, n):
        Ls.append(_setup(te, oracle, rows=96, cols=88, seed=83 + k)[2])
    stack = lambda key: np.stack([x[key] for x in Ls])  # noqa: E731
    m = ctx.map()
    m.set_layers_batched(g, n, stack("traversability"), stack("slope"), stack("step"), stack("elevation"), roughness=stack("roughness"))
    states = [mo.State(og, x) for x in Ls]
    ft, fo = footprint_params(te, oracle, 1)
    rng = np.random.default_rng(5)
    R = batch_request(rng, og, 60, n, circular=0.6, cap_path=False)
    ask(m, ft, R, R["map"])
    for k, s in enumerate(states):
        idx = np.nonzero(R["map"] == k)[0]
        s.request(fo, subset(R, idx), R["fps"])
    _assert_layers(m, states, "batched request")
    # _each: map 1 with another max_gap_width (a new memo key: its layers reset, its cache stays), the others as before
    ft2, fo2 = footprint_params(te, oracle, 1, max_gap_width=0.25)
    m.footprint_each([ft, ft2, ft])
    for k, s in enumerate(states):
        if k == 1:
            s.reset_memo()
        s.sweep(fo2 if k == 1 else fo)
    _assert_layers(m, states, "footprint_each with a key change")
    # a reload of map 2: its layers NaN again
    m.set_layers_maps(g, [2], Ls[2]["traversability"][None], Ls[2]["slope"][None], Ls[2]["step"][None], Ls[2]["elevation"][None],
                      roughness=Ls[2]["roughness"][None])
    states[2] = mo.State(og, Ls[2])
    _assert_layers(m, states, "reload")
    # the readers: submaps, occupancy and point cloud fields serve the same layers
    full = m.get_layers(list(NAMES))
    res = m.get_submaps_batched([1], [[0.0, 0.0]], [[1.0, 0.8]], list(NAMES))
    info, sub = res[0]
    r0, c0 = int(info["top_row"]), int(info["top_col"])
    for name in NAMES:
        a = sub[name]
        assert np.array_equal(a.view(np.uint32), full[name][1][r0:r0 + a.shape[0], c0:c0 + a.shape[1]].view(np.uint32)), name
    occ = m.get_occupancy(list(NAMES), 0.0, 1.0)
    for name in NAMES:
        want = np.stack([oo.occupancy_grid(full[name][k], 0.0, 1.0, (0, 0)) for k in range(n)])
        assert np.array_equal(np.asarray(occ[name]).reshape(-1), want.reshape(-1)), name
    # at_poses: a pose at the centre of cell (i, j) of each map reads that cell
    i, j = 10, 20
    x = 0.5 * og.rows * og.resolution - (i + 0.5) * og.resolution
    y = 0.5 * og.cols * og.resolution - (j + 0.5) * og.resolution
    layers, valid = m.at_poses(np.array([[x, y, 0, 0, 0, 0, 1.0]] * n), np.zeros((1, 3), np.float32), list(NAMES), pose_map=np.arange(n))
    assert (valid == 1).all()
    for name in NAMES:
        for k in range(n):
            assert np.float32(layers[name][k, 0]).view(np.uint32) == np.float32(full[name][k][i, j]).view(np.uint32), (name, k)
    # point cloud fields: a point per cell with a finite elevation, in the map's column-major cell order
    _assert_cloud(m, full, [x["elevation"] for x in Ls])
    m.close()


def test_device_request_and_graph_capture(te, ctx, oracle):
    import torch
    og, g, L, rs = _setup(te, oracle, seed=84)
    ft, fo = footprint_params(te, oracle)
    rng = np.random.default_rng(17)
    fps = request_footprints(rng)
    R = mixed_request(rng, og, 60, fps, circular=0.7, cap_path=False)
    D = _map(ctx, g, L)
    fb, fx = footprint_arrays(R, fps)
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    n = len(R["kind"])
    args = (dev(R["begin"], np.int32), dev(R["poses"], np.float64), dev(R["radius"], np.float64), dev(fb, np.int32), dev(fx, np.float32))
    out = dict(is_safe=torch.zeros(n, dtype=torch.uint8, device="cuda"), traversability_out=torch.zeros(n, dtype=torch.float64, device="cuda"),
               area_out=torch.zeros(n, dtype=torch.float64, device="cuda"), untraversable_count=torch.zeros(n, dtype=torch.int32, device="cuda"),
               untraversable_xy=torch.zeros((n, CAP, 2), dtype=torch.float64, device="cuda"))
    kw = dict(max_checks=1 << 22, max_footprint_vertices=16, conservative=dev(R["cons"], np.uint8),
              compute_untraversable_polygon=dev(R["cup"], np.uint8), untraversable_capacity=CAP, **out)
    torch.cuda.synchronize()
    D.check_footprint_request_device(ft, *args, **kw)
    torch.cuda.synchronize()
    s = mo.State(og, L)
    s.request(fo, R, fps)
    _assert_layers(D, [s], "device request")
    side = torch.cuda.Stream()
    ctx.set_stream(side.cuda_stream)
    try:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
            D.clear_footprint()
            D.check_footprint_request_device(ft, *args, **kw)
        side.synchronize()
        graph.replay()
        torch.cuda.synchronize()
    finally:
        ctx.set_stream(None)
    s.clear()
    s.request(fo, R, fps)
    _assert_layers(D, [s], "graph replay")
    D.close()


# ---- maps at their own positions and start indices; robots of their own -----------------------------------------------------

POS = np.array([(0.0, 0.0), (13.37, -3.21), (0.31, 0.05)])
START = np.array([(0, 0), (37, 53), (95, 1)], np.int32)


def _spread(te, oracle, rows=96, cols=88, res=0.02, n=3, seed=91):
    """n maps of their own terrain, each with its oracle geometry at POS[k]."""
    ogs, Ls = [], []
    for k in range(n):
        z = synth.terrain(rows, cols, res, seed + k, "mixed", tuple(POS[k]))
        og = oracle.Geometry.make(rows, cols, res, tuple(POS[k]))
        ogs.append(og)
        Ls.append(chain_layers(oracle, og, z, seed + k)[0])
    return ogs, Ls, te.Geometry.make(rows, cols, res)


def _per_map(R, k):
    return subset(R, np.nonzero(R["map"] == k)[0])


def test_positions_and_start_indices(te, ctx, oracle):
    """A batch at its own positions, each map in its own buffer order: requests and sweeps recorded per map, every reader in the
    map's buffer order."""
    ogs, Ls, g = _spread(te, oracle)
    n = len(ogs)
    buf = lambda key: np.stack([wrap(Ls[k][key], START[k]) for k in range(n)])  # noqa: E731
    m = ctx.map()
    m.set_layers_batched(g, n, buf("traversability"), buf("slope"), buf("step"), buf("elevation"), roughness=buf("roughness"),
                         positions=POS, start_index=START)
    states = [mo.State(og, L) for og, L in zip(ogs, Ls)]
    ft, fo = footprint_params(te, oracle, 1)
    rng = np.random.default_rng(41)

    def check(what):
        got = m.get_layers(list(NAMES))   # host memory: each map in its buffer order
        for name in NAMES:
            for k, st in enumerate(states):
                want = wrap(st.memo[name], START[k])
                assert np.array_equal(got[name][k].view(np.uint32), want.view(np.uint32)), (what, name, k)
        return got

    R = batch_request(rng, ogs[0], 60, n, circular=0.6, cap_path=False, offsets=POS)
    ask(m, ft, R, R["map"])
    for k, st in enumerate(states):
        st.request(fo, _per_map(R, k), R["fps"])
    check("request")
    m.footprint(ft)   # partly cached maps whose records cover their caches
    for st in states:
        st.sweep(fo)
    full = check("sweep")
    # the readers, each in the map's buffer order
    elev = m.get_layers(["elevation"])["elevation"]
    _assert_cloud(m, full, elev)
    occ = m.get_occupancy(list(NAMES), 0.0, 1.0)
    for name in NAMES:
        want = np.stack([oo.occupancy_grid(full[name][k], 0.0, 1.0, START[k]) for k in range(n)])
        assert np.array_equal(np.asarray(occ[name]).reshape(-1), want.reshape(-1)), name
    i, j = 30, 41   # the default-order cell (i, j) of every map, at its own position
    xy = [(POS[k][0] + 0.5 * g.rows * g.resolution - (i + 0.5) * g.resolution,
           POS[k][1] + 0.5 * g.cols * g.resolution - (j + 0.5) * g.resolution) for k in range(n)]
    layers, valid = m.at_poses(np.array([[x, y, 0, 0, 0, 0, 1.0] for x, y in xy]), np.zeros((1, 3), np.float32), list(NAMES),
                               pose_map=np.arange(n))
    assert (valid == 1).all()
    for name in NAMES:
        for k in range(n):
            assert np.float32(layers[name][k, 0]).view(np.uint32) == states[k].memo[name][i, j].view(np.uint32), (name, k)
    m.close()


def test_request_each_and_device_each_with_key_changes(te, ctx, oracle):
    """Robots of their own on maps at their own positions: te_map_check_footprint_request_each, then _device_each with new memo
    keys on maps 1 and 2 (their layers reset, their caches kept), then te_map_footprint_each, which walks those two maps."""
    import torch
    ogs, Ls, g = _spread(te, oracle, seed=95)
    n = len(ogs)
    stack = lambda key: np.stack([x[key] for x in Ls])  # noqa: E731
    m = ctx.map()
    m.set_layers_batched(g, n, stack("traversability"), stack("slope"), stack("step"), stack("elevation"), roughness=stack("roughness"),
                         positions=POS)
    states = [mo.State(og, L) for og, L in zip(ogs, Ls)]
    kw = [dict(verify=0, offset=0.1), dict(verify=1, offset=0.0), dict(verify=0, offset=0.2, traversability_default=0.3)]
    first = [footprint_params(te, oracle, k.get("verify", 0), **{a: b for a, b in k.items() if a != "verify"}) for k in kw]
    rng = np.random.default_rng(43)
    R = batch_request(rng, ogs[0], 60, n, circular=0.6, cap_path=False, offsets=POS)
    fb, fx = footprint_arrays(R, R["fps"])
    m.check_footprint_request_each([p[0] for p in first], R["map"], R["begin"], R["poses"], R["radius"], fb, fx,
                                   max_footprint_vertices=16, conservative=R["cons"], compute_untraversable_polygon=R["cup"],
                                   untraversable_capacity=CAP)
    for k, st in enumerate(states):
        st.request(first[k][1], _per_map(R, k), R["fps"])
    _assert_layers(m, states, "request_each")
    # new memo keys on maps 1 and 2
    second = [first[0], footprint_params(te, oracle, 0, offset=0.0), footprint_params(te, oracle, 0, offset=0.2, max_gap_width=0.25)]
    R2 = batch_request(rng, ogs[0], 60, n, fps=R["fps"], circular=0.6, cap_path=False, offsets=POS)
    fb, fx = footprint_arrays(R2, R2["fps"])
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()  # noqa: E731
    npaths = len(R2["kind"])
    out = dict(is_safe=torch.zeros(npaths, dtype=torch.uint8, device="cuda"),
               traversability_out=torch.zeros(npaths, dtype=torch.float64, device="cuda"),
               area_out=torch.zeros(npaths, dtype=torch.float64, device="cuda"))
    m.check_footprint_request_device(None, dev(R2["begin"], np.int32), dev(R2["poses"], np.float64), dev(R2["radius"], np.float64),
                                     dev(fb, np.int32), dev(fx, np.float32), max_checks=1 << 20, path_map=dev(R2["map"], np.int32),
                                     max_footprint_vertices=16, conservative=dev(R2["cons"], np.uint8),
                                     compute_untraversable_polygon=dev(R2["cup"], np.uint8), params=[p[0] for p in second], **out)
    torch.cuda.synchronize()
    for k, st in enumerate(states):
        if k > 0:
            st.reset_memo()
        st.request(second[k][1], _per_map(R2, k), R2["fps"])
    _assert_layers(m, states, "device_each with new keys")
    # the sweep: maps 1 and 2 hold cached cells their bytes no longer record, so their empty centres walk
    m.footprint_each([p[0] for p in second])
    for k, st in enumerate(states):
        st.sweep(second[k][1])
    _assert_layers(m, states, "footprint_each after the key changes")
    m.close()
