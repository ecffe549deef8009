"""The read side of a te_map on the GPU, bit for bit: te_map_get_layers against the layers that went in or came out of the chain,
te_map_get_submaps against numpy slices at the CPU oracle's getSubmap geometry (tests/submap_oracle.cpp), and te_map_valid_at
against the oracle's getIndex + isfinite."""
import ctypes as C

import numpy as np
import pytest

import submap_oracle as so
import synth

pytestmark = pytest.mark.gpu

ROWS, COLS, RES, POS = 150, 130, 0.02, (0.37, -0.21)


def _bits(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    return a.view(np.uint32)


def _same(a, b, what=""):
    assert np.array_equal(_bits(a), _bits(b)), what


def _layers(seed, rows=ROWS, cols=COLS):
    """Random layers with NaN and +-Inf cells: traversability, slope, step, roughness, elevation, robot_slope."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(6):
        a = rng.standard_normal((rows, cols)).astype(np.float32)
        a[rng.random(a.shape) < 0.05] = np.nan
        a[rng.random(a.shape) < 0.01] = np.inf
        a[rng.random(a.shape) < 0.01] = -np.inf
        out.append(np.asfortranarray(a))
    return out


def _geo(te, start=(0, 0), rows=ROWS, cols=COLS):
    g = te.Geometry.make(rows, cols, RES, POS)
    g.start_row, g.start_col = start
    return g


def _unwrap(a, start):
    """Default order of a layer stored with a circular-buffer start index: cell (i, j) is stored at ((i + sr) % rows, ...)."""
    return np.roll(a, (-start[0], -start[1]), axis=(0, 1))


def _set(te, ctx, seed=1, start=(0, 0), rough=True, rslope=True):
    t, s, st, r, e, rs = _layers(seed)
    m = ctx.map()
    m.set_layers(_geo(te, start), t, s, st, e, roughness=r if rough else None, robot_slope=rs if rslope else None)
    return m, dict(traversability=t, traversability_slope=s, traversability_step=st, traversability_roughness=r, elevation=e,
                   robot_slope=rs)


def _torch():
    return pytest.importorskip("torch")


def test_get_layers_after_set_layers_host_with_start_index(te, ctx):
    start = (37, 101)
    m, L = _set(te, ctx, start=start)
    got = m.get_layers(te.capi.LAYERS)
    for k in L:
        _same(got[k], L[k], k)                   # re-wrapped: the buffer order the layers came in
    assert np.isnan(got["traversability_footprint"]).all() and _bits(got["traversability_footprint"]).min() == 0xffffffff
    sub = m.get_layers(["elevation", "traversability_step"])
    assert list(sub) == ["traversability_step", "elevation"]          # bit order, whatever the order asked for
    _same(sub["elevation"], L["elevation"])
    m.close()


def test_get_layers_device_memory_is_unwrapped(te, ctx):
    torch = _torch()
    start = (5, 77)
    m, L = _set(te, ctx, start=start)
    names = ["traversability", "traversability_roughness", "elevation", "robot_slope"]
    out = torch.full((len(names) * ROWS * COLS,), 7.0, dtype=torch.float32, device="cuda")
    got = m.get_layers(names, out=out, memory=te.MEM_DEVICE)
    ctx.synchronize()
    for k in names:
        _same(got[k].cpu().numpy(), _unwrap(L[k], start), k)
    m.close()


def test_get_layers_after_chain_equals_the_chain_outputs(te, ctx):
    z = synth.terrain(ROWS, COLS, RES, seed=3, preset="mixed")
    g = _geo(te, (11, 4))
    m = ctx.map()
    outs = m.chain(g, te.ChainParams.yaml_defaults(0), z, outputs=True)
    got = m.get_layers(["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"])
    for k, o in (("traversability", "traversability"), ("traversability_slope", "slope"), ("traversability_step", "step"),
                 ("traversability_roughness", "roughness")):
        _same(got[k], outs[o], k)
    _same(got["elevation"], np.asarray(z, dtype=np.float32))
    # the cache after a footprint request is what te_map_get_footprint returns
    fp = m.footprint(te.FootprintParams.yaml_defaults())
    _same(m.get_layers(["traversability_footprint"])["traversability_footprint"], m.get_footprint())
    _same(fp, m.get_footprint())
    with pytest.raises(te.TEError) as e:            # computeTraversability leaves robot_slope to setTraversabilityMap
        m.get_layers(["robot_slope"])
    assert e.value.code == -2
    m.close()


def test_layer_errors(te, ctx):
    m = ctx.map()
    with pytest.raises(te.TEError) as e:
        m.get_layers(["traversability"])            # no layers yet
    assert e.value.code == -1
    with pytest.raises(te.TEError) as e:
        m.valid_at(np.zeros((1, 2)))
    assert e.value.code == -1
    m.close()
    m, _ = _set(te, ctx, rough=False, rslope=False)
    for name in ("traversability_roughness", "robot_slope"):
        with pytest.raises(te.TEError) as e:
            m.get_layers(["traversability", name])
        assert e.value.code == -2
        with pytest.raises(te.TEError) as e:
            m.get_submaps([[0.3, -0.2]], [[0.5, 0.5]], [name])
        assert e.value.code == -2
    L = te.load_library()
    L.te_map_get_layers.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int]
    buf = np.zeros(ROWS * COLS, dtype=np.float32)
    assert L.te_map_get_layers(m._h, 0, buf.ctypes.data, 0) == -1          # empty mask
    assert L.te_map_get_layers(m._h, 0x80, buf.ctypes.data, 0) == -1       # unknown bit
    assert L.te_map_get_layers(m._h, 1, None, 0) == -1
    m.close()


def _windows(rng, n, g):
    """Windows of 0 to 1.5 m around centres inside, near the edges (straddling them) and outside the map."""
    P, Lm = np.array(POS), np.array([g.length_x, g.length_y])
    kind = rng.integers(0, 3, n)
    pos = P + rng.uniform(-0.45, 0.45, (n, 2)) * Lm
    edge = kind == 1
    pos[edge] = P + rng.choice([-0.5, 0.5], (edge.sum(), 2)) * Lm + rng.uniform(-0.1, 0.1, (edge.sum(), 2))
    pos[kind == 2] = P + rng.uniform(-1.2, 1.2, ((kind == 2).sum(), 2)) * Lm
    length = rng.uniform(0.0, 1.5, (n, 2))
    length[rng.random(n) < 0.1] = 0.0
    length[rng.random(n) < 0.1] = 2.5 * RES
    return pos, length


def _oracle_geometry(oracle, pos, length):
    return so.submap_geometry(oracle.Geometry.make(ROWS, COLS, RES, POS), pos, length)


def _check_windows(res, want, full, names):
    """Every window: geometry as the oracle's, layers equal to the block of the default-order layers `full`."""
    assert len(res) == len(want["success"])
    for k, (info, lay) in enumerate(res):
        for f in so.FIELDS:
            assert info[f] == want[f][k] or (np.isnan(info[f]) and np.isnan(want[f][k])), (k, f)
        if not info["success"]:
            assert lay is None
            continue
        r0, c0, nr, nc = (int(info[f]) for f in ("top_row", "top_col", "rows", "cols"))
        assert list(lay) == [n for n in full if n in names]
        for n in lay:
            _same(np.asarray(lay[n]), full[n][r0:r0 + nr, c0:c0 + nc], (k, n))


@pytest.mark.parametrize("names", [None, ["traversability"], ["traversability_step", "elevation", "traversability_footprint"]])
def test_submaps_host_memory_are_slices_of_the_layers(te, ctx, oracle, names):
    start = (0, 0) if names else (19, 62)
    m, L = _set(te, ctx, seed=4, start=start)
    names = names or list(te.capi.LAYERS)
    full = {k: _unwrap(v, start) for k, v in m.get_layers(te.capi.LAYERS).items()}
    rng = np.random.default_rng(8)
    pos, length = _windows(rng, 120, _geo(te))
    res = m.get_submaps(pos, length, names)
    want = _oracle_geometry(oracle, pos, length)
    assert 0 < want["success"].sum() < len(pos)
    _check_windows(res, want, {k: v for k, v in full.items() if k in names}, names)
    m.close()


def test_submaps_device_memory_and_one_call_equals_single_calls(te, ctx, oracle):
    torch = _torch()
    start = (3, 9)
    m, L = _set(te, ctx, seed=6, start=start)
    names = ["traversability", "traversability_roughness", "robot_slope"]
    full = {k: _unwrap(v, start) for k, v in m.get_layers(names).items()}
    rng = np.random.default_rng(12)
    pos, length = _windows(rng, 300, _geo(te))
    want = _oracle_geometry(oracle, pos, length)
    total = len(names) * int((want["rows"] * want["cols"]).sum())
    out = torch.full((total + 5,), -3.0, dtype=torch.float32, device="cuda")
    res = m.get_submaps(pos, length, names, out=out, memory=te.MEM_DEVICE)
    ctx.synchronize()
    host = out.cpu().numpy()
    assert (host[total:] == -3.0).all()                        # nothing written beyond the windows
    res_np = [(i, None if d is None else {n: v.cpu().numpy() for n, v in d.items()}) for i, d in res]
    _check_windows(res_np, want, full, names)
    # 300 windows in one call equal 300 calls of one window each, in host memory
    hres = m.get_submaps(pos, length, names)
    for k in range(len(pos)):
        (i1, d1), = m.get_submaps(pos[k:k + 1], length[k:k + 1], names)
        i0, d0 = hres[k]
        assert bool(i1["success"]) == bool(i0["success"])
        if d0 is not None:
            for n in names:
                _same(d1[n], d0[n], (k, n))
                _same(d0[n], res_np[k][1][n], (k, n))
    m.close()


def test_capacity_retry_failed_windows_and_launch_count(te, ctx):
    m, L = _set(te, ctx, seed=9)
    Lib = te.load_library()
    fn = Lib.te_map_get_submaps
    fn.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int]
    pos = np.array([[0.37, -0.21], [50.0, 50.0], [0.2, -0.1], [-50.0, 0.0]])      # windows 1 and 3 lie outside the map
    length = np.array([[0.5, 0.4], [1.0, 1.0], [0.1, 0.3], [1.0, 1.0]])
    mask = 0x11
    info = np.zeros(4, dtype=te.capi.SUBMAP_INFO_DTYPE)
    out = np.full(8, 5.0, dtype=np.float32)
    rc = fn(m._h, 4, pos.ctypes.data, length.ctypes.data, mask, info.ctypes.data, out.ctypes.data, len(out), te.MEM_HOST)
    assert rc == -1 and (out == 5.0).all()                     # too small: info filled, nothing written
    assert list(info["success"]) == [1, 0, 1, 0]
    size = 2 * info["rows"].astype(np.int64) * info["cols"]
    assert list(info["offset"]) == [0, size[0], size[0], size[0] + size[2]]         # failed windows take no space
    total = int(info["offset"][-1] + size[-1])
    assert info["rows"][1] == 0 and info["cols"][1] == 0
    out = np.full(total, 5.0, dtype=np.float32)
    rc = fn(m._h, 4, pos.ctypes.data, length.ctypes.data, mask, info.ctypes.data, out.ctypes.data, total, te.MEM_HOST)
    assert rc == 0 and not (out == 5.0).any()
    # one gather launch whatever the window count; none when no window has cells
    rng = np.random.default_rng(2)
    for n in (1, 16, 300):
        p, ln = _windows(rng, n, _geo(te))
        p[0], ln[0] = POS, (0.3, 0.3)
        before = ctx.stats()[0]
        m.get_submaps(p, ln, ["traversability", "elevation"])
        assert ctx.stats()[0] - before == 1, n
    before = ctx.stats()[0]
    assert all(d is None for _, d in m.get_submaps(pos[[1, 3]], length[[1, 3]], ["traversability"]))
    assert ctx.stats()[0] == before
    with pytest.raises(te.TEError) as e:
        m.get_submaps([[0.0, 0.0]], [[-1.0, 1.0]], ["traversability"])
    assert e.value.code == -1
    m.close()


@pytest.mark.parametrize("start", [(0, 0), (71, 12)])
def test_valid_at_matches_oracle(te, ctx, oracle, start):
    m, L = _set(te, ctx, seed=13, start=start)
    trav = _unwrap(L["traversability"], start)
    rng = np.random.default_rng(21)
    g = _geo(te)
    n = 5000
    xy = np.array(POS) + rng.uniform(-0.6, 0.6, (n, 2)) * np.array([g.length_x, g.length_y])
    # cell centres and edges exactly, and non-finite positions
    i, j = rng.integers(0, ROWS, 500), rng.integers(0, COLS, 500)
    cx = (g.position_x + (0.5 * g.length_x - 0.5 * RES)) + RES * (-i.astype(np.float64))
    cy = (g.position_y + (0.5 * g.length_y - 0.5 * RES)) + RES * (-j.astype(np.float64))
    xy = np.concatenate([xy, np.stack([cx, cy], 1), np.stack([cx + 0.5 * RES, cy - 0.5 * RES], 1), [[np.nan, 0.3], [np.inf, 0.0]]])
    want = so.valid_at(oracle.Geometry.make(ROWS, COLS, RES, POS), trav, xy)
    assert 0 < want.sum() < len(xy)
    assert np.array_equal(m.valid_at(xy), want)
    torch = _torch()
    dxy = torch.from_numpy(xy).cuda()
    dv = torch.full((len(xy),), 9, dtype=torch.uint8, device="cuda")
    m.valid_at(dxy, out=dv, memory=te.MEM_DEVICE)
    ctx.synchronize()
    assert np.array_equal(dv.cpu().numpy(), want)
    m.close()
