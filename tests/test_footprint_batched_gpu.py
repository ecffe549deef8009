"""te_footprint_batched / te_footprint_polygon_batched: the footprint sweeps of a batch of maps in one call equal, bit for bit,
the single-map entries run map by map, and a map never sees the cells of its neighbours."""
import numpy as np
import pytest

from helpers import close_sweep, same_values, te_footprint_params, walled_batch, walled_terrain

pytestmark = pytest.mark.gpu

POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]   # robot_footprint_parameter.yaml:3
YAW = 0.7854


def _circular_batched(te, ctx, g, p, B, n, memory, rough_outputs):
    shape = B["traversability"].shape
    out, sfp, tfp, rfp = (np.full(shape, 7.0, dtype=np.float32) for _ in range(4))
    ctx.footprint_batched(g, p, n, B["traversability"], B["slope"], B["step"], B["elevation"], out, memory, slope_fp=sfp, step_fp=tfp,
                          roughness=B["roughness"] if rough_outputs else None, roughness_fp=rfp if rough_outputs else None)
    return out, sfp, tfp, rfp


def _circular_one(te, ctx, g, p, B, k, rough_outputs):
    lay = [np.asfortranarray(B[x][k].T) for x in ("traversability", "slope", "step", "elevation")]
    out, sfp, tfp, rfp = (np.full(lay[0].shape, 7.0, dtype=np.float32, order="F") for _ in range(4))   # column-major layers
    ctx.footprint(g, p, *lay, out, te.MEM_HOST, slope_fp=sfp, step_fp=tfp,
                  roughness=np.asfortranarray(B["roughness"][k].T) if rough_outputs else None, roughness_fp=rfp if rough_outputs else None)
    return out, sfp, tfp, rfp


@pytest.fixture(scope="module")
def batch(oracle):
    rows, cols, n = 100, 90, 12   # rows not a multiple of 32 or 64, columns not a multiple of 16
    return rows, cols, n, walled_batch(oracle, rows, cols, 0.02, n, 500)


@pytest.fixture(scope="module")
def batch_fine(oracle):
    rows, cols, n = 100, 90, 6    # 0.01 m: radius + offset is 45 cells, beyond the prefix-sum sweep's 31
    return rows, cols, n, walled_batch(oracle, rows, cols, 0.01, n, 700)


@pytest.mark.parametrize("case", ["offset0.15", "offset0", "roughness", "brute"])
def test_circular_batch_equals_map_by_map(te, ctx, oracle, batch, case, monkeypatch):
    rows, cols, n, B = batch
    g = te.Geometry.make(rows, cols, 0.02)
    p = te_footprint_params(te, offset=0.0 if case == "offset0" else 0.15, verify_roughness=1 if case == "roughness" else 0)
    if case == "brute":
        monkeypatch.setenv("TE_FOOTPRINT_BRUTE", "1")   # the visit-by-visit k_sweep
    rough = case == "roughness"
    got = _circular_batched(te, ctx, g, p, B, n, te.MEM_HOST, rough)
    for k in range(n):
        one = _circular_one(te, ctx, g, p, B, k, rough)
        for a, b, name in zip(got, one, ("traversability_footprint", "slope_footprint", "step_footprint", "roughness_footprint")):
            assert same_values(a[k].T, b), (case, k, name)
    fpl = got[0]
    for k in range(n):   # every kind of map has blocked and open cells, and the walls block the edges they stand on
        assert (fpl[k] > 0).any(), k
        if k % 4 == 1:
            assert (fpl[k][:, :8] == 0).any() and (fpl[k][:8, :] == 0).any(), k
        if k % 4 == 3:
            assert (fpl[k][:, -8:] == 0).any() and (fpl[k][-8:, :] == 0).any(), k
    assert (fpl[0] > 0).all()   # the flat map is open everywhere, next to the walled map 1
    # two maps of the batch against the oracle: exact for the visit-by-visit sweep and the memo layers
    og = oracle.Geometry.make(rows, cols, 0.02)
    fo = oracle.FootprintParams.yaml_defaults()
    fo.offset, fo.verify_roughness = p.offset, p.verify_roughness
    for k in (1, 3):
        lay = [np.asfortranarray(B[x][k].T) for x in ("traversability", "slope", "step", "elevation")]
        ref = oracle.footprint(og, fo, *lay, roughness=np.asfortranarray(B["roughness"][k].T) if rough else None)
        assert (same_values if case == "brute" else close_sweep)(got[0][k].T, ref[0]), (case, k)
        assert same_values(got[1][k].T, ref[1]) and same_values(got[2][k].T, ref[2]), (case, k)
        if rough:
            assert same_values(got[3][k].T, ref[3]), (case, k)


def test_circular_batch_beyond_31_cells(te, ctx, oracle, batch_fine):
    """Radius + offset of 45 cells selects k_sweep for every map of the batch."""
    rows, cols, n, B = batch_fine
    g = te.Geometry.make(rows, cols, 0.01)
    p = te_footprint_params(te)
    p.max_gap_width = 0.1   # at 0.01 m checkForSlope then blocks the zero-slope patches
    got = _circular_batched(te, ctx, g, p, B, n, te.MEM_HOST, False)
    for k in range(n):
        one = _circular_one(te, ctx, g, p, B, k, False)
        for a, b in zip(got[:3], one[:3]):
            assert same_values(a[k].T, b), k
    og = oracle.Geometry.make(rows, cols, 0.01)
    lay = [np.asfortranarray(B[x][3].T) for x in ("traversability", "slope", "step", "elevation")]
    fo = oracle.FootprintParams.yaml_defaults()
    fo.max_gap_width = p.max_gap_width
    ref = oracle.footprint(og, fo, *lay)
    assert same_values(got[0][3].T, ref[0]) and same_values(got[1][3].T, ref[1]) and same_values(got[2][3].T, ref[2])
    assert (ref[0] == 0).any() and (ref[0] > 0).any()


@pytest.mark.parametrize("case", ["plain", "roughness"])
def test_polygon_batch_equals_map_by_map(te, ctx, oracle, batch, case):
    rows, cols, n, B = batch
    g = te.Geometry.make(rows, cols, 0.02)
    rough = case == "roughness"
    p = te_footprint_params(te, verify_roughness=1 if rough else 0)
    shape = B["traversability"].shape
    ox, orot = np.full(shape, 7.0, dtype=np.float32), np.full(shape, 7.0, dtype=np.float32)
    ctx.footprint_polygon_batched(g, p, n, POLY, YAW, B["traversability"], B["slope"], B["step"], B["elevation"], ox, orot, te.MEM_HOST,
                                  roughness=B["roughness"] if rough else None)
    for k in range(n):
        lay = [np.asfortranarray(B[x][k].T) for x in ("traversability", "slope", "step", "elevation")]
        x1, r1 = np.empty_like(lay[0]), np.empty_like(lay[0])
        ctx.footprint_polygon(g, p, POLY, YAW, *lay, x1, r1, te.MEM_HOST, roughness=np.asfortranarray(B["roughness"][k].T) if rough else None)
        assert np.array_equal(ox[k].T, x1) and np.array_equal(orot[k].T, r1), (case, k)
    assert (ox[0] > 0).all() and (ox[1] == 0).any() and (ox[3] == 0).any()
    og = oracle.Geometry.make(rows, cols, 0.02)
    fo = oracle.FootprintParams.yaml_defaults()
    fo.verify_roughness = p.verify_roughness
    for k in (1, 2):
        lay = [np.asfortranarray(B[x][k].T) for x in ("traversability", "slope", "step", "elevation")]
        rx, rrot = oracle.footprint_polygon(og, fo, POLY, YAW, *lay, roughness=np.asfortranarray(B["roughness"][k].T) if rough else None)
        assert close_sweep(ox[k].T, rx) and close_sweep(orot[k].T, rrot), (case, k)


def test_device_memory_and_a_batch_of_one(te, ctx, batch):
    """TE_MEM_DEVICE gives what TE_MEM_HOST gives, and nmaps = 1 gives what the single-map entries give."""
    import torch
    rows, cols, n, B = batch
    g = te.Geometry.make(rows, cols, 0.02)
    p = te_footprint_params(te)
    ctx.set_stream(None)
    D = {k: torch.from_numpy(v).cuda() for k, v in B.items()}
    host = _circular_batched(te, ctx, g, p, B, n, te.MEM_HOST, False)
    dev = [torch.full(B["traversability"].shape, 7.0, dtype=torch.float32, device="cuda") for _ in range(3)]
    ctx.footprint_batched(g, p, n, D["traversability"], D["slope"], D["step"], D["elevation"], dev[0], te.MEM_DEVICE, slope_fp=dev[1],
                          step_fp=dev[2])
    ctx.synchronize()
    for a, b in zip(host[:3], dev):
        assert same_values(a, b.cpu().numpy())
    shape = B["traversability"].shape
    hx, hr = np.empty(shape, dtype=np.float32), np.empty(shape, dtype=np.float32)
    ctx.footprint_polygon_batched(g, p, n, POLY, YAW, B["traversability"], B["slope"], B["step"], B["elevation"], hx, hr, te.MEM_HOST)
    dx, dr = (torch.empty(shape, dtype=torch.float32, device="cuda") for _ in range(2))
    ctx.footprint_polygon_batched(g, p, n, POLY, YAW, D["traversability"], D["slope"], D["step"], D["elevation"], dx, dr, te.MEM_DEVICE)
    ctx.synchronize()
    assert np.array_equal(hx, dx.cpu().numpy()) and np.array_equal(hr, dr.cpu().numpy())
    # nmaps = 1 on map 5
    one_b = _circular_batched(te, ctx, g, p, {k: v[5:6] for k, v in B.items()}, 1, te.MEM_HOST, False)
    one = _circular_one(te, ctx, g, p, B, 5, False)
    for a, b in zip(one_b[:3], one[:3]):
        assert same_values(a[0].T, b)
    bx, br = np.empty((1,) + shape[1:], dtype=np.float32), np.empty((1,) + shape[1:], dtype=np.float32)
    ctx.footprint_polygon_batched(g, p, 1, POLY, YAW, *(B[x][5:6] for x in ("traversability", "slope", "step", "elevation")), bx, br,
                                  te.MEM_HOST)
    lay = [np.asfortranarray(B[x][5].T) for x in ("traversability", "slope", "step", "elevation")]
    x1, r1 = np.empty_like(lay[0]), np.empty_like(lay[0])
    ctx.footprint_polygon(g, p, POLY, YAW, *lay, x1, r1, te.MEM_HOST)
    assert np.array_equal(bx[0].T, x1) and np.array_equal(br[0].T, r1)


def test_batched_chain_then_batched_footprint(te, ctx):
    """te_chain_batched -> te_footprint_batched in device memory equals te_chain + te_footprint map by map."""
    import torch
    rows, cols, n, res = 100, 90, 8, 0.02
    g = te.Geometry.make(rows, cols, res)
    cp, p = te.ChainParams.yaml_defaults(0), te_footprint_params(te)
    z = torch.from_numpy(np.stack([np.ascontiguousarray(walled_terrain(rows, cols, res, k % 4, 900 + k).T) for k in range(n)])).cuda()
    ctx.set_stream(None)
    lay = [torch.empty((n, cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]   # slope step roughness traversability
    ctx.chain_batched(g, cp, n, z, *lay, te.MEM_DEVICE)
    out = torch.empty((n, cols, rows), dtype=torch.float32, device="cuda")
    ctx.footprint_batched(g, p, n, lay[3], lay[0], lay[1], z, out, te.MEM_DEVICE)
    ctx.synchronize()
    for k in range(n):
        one = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
        ctx.chain(g, cp, z[k], *one, te.MEM_DEVICE)
        o1 = torch.empty((cols, rows), dtype=torch.float32, device="cuda")
        ctx.footprint(g, p, one[3], one[0], one[1], z[k], o1, te.MEM_DEVICE)
        ctx.synchronize()
        a, b = out[k].cpu().numpy(), o1.cpu().numpy()
        assert same_values(a, b), k
    assert (out == 0).any() and (out > 0).any()


def test_argument_errors(te, ctx, batch):
    rows, cols, n, B = batch
    g = te.Geometry.make(rows, cols, 0.02)
    p = te_footprint_params(te)
    lay = [B[x] for x in ("traversability", "slope", "step", "elevation")]
    out = np.empty_like(B["traversability"])
    for bad in (0, -3):
        with pytest.raises(te.TEError) as err:
            ctx.footprint_batched(g, p, bad, *lay, out, te.MEM_HOST)
        assert err.value.code == -1
        with pytest.raises(te.TEError) as err:
            ctx.footprint_polygon_batched(g, p, bad, POLY, YAW, *lay, out, out.copy(), te.MEM_HOST)
        assert err.value.code == -1
    with pytest.raises(te.TEError) as err:   # a layer missing
        ctx.footprint_batched(g, p, n, lay[0], None, lay[2], lay[3], out, te.MEM_HOST)
    assert err.value.code == -2
    with pytest.raises(te.TEError) as err:
        ctx.footprint_polygon_batched(g, p, n, POLY, YAW, lay[0], lay[1], None, lay[3], out, out.copy(), te.MEM_HOST)
    assert err.value.code == -2
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = 3, 4
    with pytest.raises(te.TEError) as err:   # a batch takes maps in default order only
        ctx.footprint_batched(gw, p, n, *lay, out, te.MEM_HOST)
    assert err.value.code == -4
    with pytest.raises(te.TEError) as err:
        ctx.footprint_polygon_batched(gw, p, n, POLY, YAW, *lay, out, out.copy(), te.MEM_HOST)
    assert err.value.code == -4
    # 65535 maps (a grid dimension) is the largest batch; 1 x 1 maps keep every buffer correctly sized
    g1 = te.Geometry.make(1, 1, 0.02)
    rng = np.random.default_rng(3)
    one = {"traversability": rng.random((65536, 1, 1), dtype=np.float32), "slope": np.ones((65536, 1, 1), dtype=np.float32),
           "step": np.ones((65536, 1, 1), dtype=np.float32), "elevation": np.zeros((65536, 1, 1), dtype=np.float32)}
    one_lay = [one[x] for x in ("traversability", "slope", "step", "elevation")]
    o1 = np.empty((65536, 1, 1), dtype=np.float32)
    with pytest.raises(te.TEError) as err:
        ctx.footprint_batched(g1, p, 65536, *one_lay, o1, te.MEM_HOST)
    assert err.value.code == -4
    with pytest.raises(te.TEError) as err:
        ctx.footprint_polygon_batched(g1, p, 65536, POLY, YAW, *one_lay, o1, o1.copy(), te.MEM_HOST)
    assert err.value.code == -4
    ctx.footprint_batched(g1, p, 65535, *one_lay, o1, te.MEM_HOST)
    assert np.array_equal(o1[:65535], one["traversability"][:65535])   # a 1 x 1 map's disk holds its own cell only
