"""The chain against the oracle on every validity pattern of its normals windows (the probe maps of window_masks.py).

A window with a hole or a map border in it takes tier 2's validity-mask path: offset moments from popcounts of hand-written
bit patterns, Halley's method on the characteristic polynomial, a rank and a conditioning threshold, and tier 3's replay of the
reference's rank test behind them; holes and infinite elevations take the step filter's minNum / maxNum path and step_t2.  A
wrong bit or threshold there changes the result only for the masks that touch it, and random terrain reaches a few hundred of
the 2^20 masks of the YAML disk.  Every comparison covers every cell of the map, not only the block centres."""
import time

import numpy as np
import pytest

import window_masks as wm
from helpers import assert_parity, chain_params, compare_layer

pytestmark = pytest.mark.gpu

LAYERS = ("slope", "step", "roughness", "traversability")
SEED = 7
FAR = (2_600_000.0, 1_200_000.0)


@pytest.fixture(scope="module", autouse=True)
def _clock():
    t = time.time()
    yield
    print(f"\ntest_window_masks_gpu: {time.time() - t:.1f} s")


def _params(mod, shape, **kw):
    return chain_params(mod, **{**wm.chain_kwargs(shape), **kw})


def _parity(got, ref):
    """assert_parity for slope, step and roughness; the traversability's exact cells are those where each of its three terms is
    a branch value (0 or 1) in the reference and in the result (as test_chain_params_gpu._parity)."""
    assert_parity(got, ref, keys=("slope", "step", "roughness"))
    tr = compare_layer(got["traversability"], ref["traversability"], "traversability")
    assert tr["nan_mismatch"] == 0 and tr["out_of_tol"] == 0, tr
    exact = np.ones(ref["traversability"].shape, bool)
    for k in ("slope", "step", "roughness"):
        exact &= ((ref[k] == 0.0) | (ref[k] == 1.0)) & (got[k] == ref[k])
    a, b = got["traversability"][exact], ref["traversability"][exact]
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), int((a != b).sum())


def _literal_off(got, ref):
    """Cells of the four layers that are not bit-exact; asserts an exact NaN mask.  Elsewhere the literal kernel may differ from
    the oracle where the device's libm acos / sqrt rounds differently from the host's; on these maps it never does (measured on
    an H100: 0 cells in every case), so none is allowed."""
    off = 0
    for k in LAYERS:
        a, b = got[k], ref[k]
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        ok = ~np.isnan(b)
        off += int((a[ok].view(np.uint32) != b[ok].view(np.uint32)).sum())
    return off


def _run(te, ctx, kernel, g, p, z):
    """The chain on z in device memory: one launch over the whole map, so that the flag counters and the escalation histogram
    count every cell (the host path pipelines large maps in column chunks, one launch each)."""
    import torch
    rows, cols = z.shape
    zd = torch.from_numpy(np.ascontiguousarray(z.T)).cuda()   # (cols, rows) tensor == column-major layer
    outs = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in LAYERS]
    ctx.set_stream(None)
    ctx.set_kernel(kernel)
    try:
        ctx.chain(g, p, zd, *outs, te.MEM_DEVICE)
        ctx.synchronize()
        got = {k: np.asfortranarray(o.cpu().numpy().T) for k, o in zip(LAYERS, outs)}
        return got, ctx.flag_counters(), ctx.escalation_stats()
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)


def _masks(shape, sample):
    return wm.sample_masks(shape, sample, SEED) if sample else wm.all_masks(shape)


# (shape, family, slope_critical, position, masks: 0 = all, else a sample of that many)
CASES = [(s, f, c, (0.0, 0.0), 0 if s != "tips" else 1 << 16)
         for s in ("A", "B", "tips") for f, c in (("tilt", 1.0), ("planar", 1.0), ("nearflat", 1.0), ("nearflat", 0.1),
                                                   ("inf", 1.0))] + \
        [("A", f, c, FAR, 1 << 16) for f, c in (("planar", 1.0), ("nearflat", 1.0), ("nearflat", 0.1))]
IDS = [f"{s}-{f}-crit{c}" + ("-far" if pos != (0.0, 0.0) else "") for s, f, c, pos, _ in CASES]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_fused_and_literal_against_the_oracle(te, ctx, oracle, case):
    shape, family, crit, pos, sample = case
    cid = IDS[CASES.index(case)]
    t = time.time()
    z = wm.probe(shape, _masks(shape, sample), family, SEED)
    rows, cols = z.shape
    res = wm.SHAPES[shape][0]
    g, og = te.Geometry.make(rows, cols, res, pos), oracle.Geometry.make(rows, cols, res, pos)
    ref = oracle.chain(og, _params(oracle, shape, slope_critical=crit), z, with_normals=True)
    t_oracle = time.time() - t
    p = _params(te, shape, slope_critical=crit)

    fused, cnt, (why, nvalid) = _run(te, ctx, te.KERNEL_FUSED, g, p, z)   # KERNEL_FUSED raises rather than fall back
    partial = int(wm.partial_windows(np.isfinite(z), shape).sum())
    print(f"\n{cid} {rows}x{cols}: tier 2 {cnt[0]} cells ({partial} valid cells with a partial window), tier 3 {cnt[4]}; "
          f"escalations by reason {why}; by valid window cells {nvalid}")
    assert cnt[2] == 0, cnt
    assert cnt[0] >= partial, (cnt, partial)
    _parity(fused, ref)

    literal, _, _ = _run(te, ctx, te.KERNEL_GENERIC, g, p, z)
    off = _literal_off(literal, ref)
    print(f"{cid}: literal kernel {off} cells not bit-exact; oracle {t_oracle:.1f} s, case {time.time() - t:.1f} s")
    assert off == 0, off

    if family == "planar":
        # exactly planar windows sit on the reference's rank threshold: tier 2 passes them on and tier 3 decides
        ci, cj = wm.centres(rows, cols)
        fallback = ref["nz"] == 1.0
        fs, ls, rs = (a[ci, cj].view(np.uint32) for a in (fused["slope"], literal["slope"], ref["slope"]))
        decided = ls == rs
        print(f"{cid}: {int(fallback.sum())} cells with the rank fallback, {int(fallback[ci, cj].sum())} of {len(ci)} centres; "
              f"literal slope bit-exact at {int(decided.sum())} centres")
        assert cnt[4] >= len(ci) // 2, cnt
        assert why[5] > 0, why                                    # rank of a partial window
        assert fallback[ci, cj].any()
        assert (fused["slope"][fallback] == 1.0).all(), int((fused["slope"][fallback] != 1.0).sum())
        assert np.array_equal(fs[decided], ls[decided]), int((fs[decided] != ls[decided]).sum())
    if family == "nearflat" and pos == FAR:
        assert why[9] > 0, why                                    # n_z within nz_guard of a float32 rounding boundary


@pytest.mark.parametrize("shape", ["A", "tips"])
def test_batch_at_different_positions(te, ctx, oracle, shape):
    """Infinite and NaN holes in four maps of one te_map at their own positions: each map's step tips are decided by its own
    masks, which step_t2 reads through the per-map rowmask_stride / colmask_stride."""
    positions = [(0.0, 0.0), FAR, (1234.5678, -987.6543), (-3.3, 7.7)]
    zs = [wm.probe(shape, wm.sample_masks(shape, 1 << 16, SEED + m), "inf", SEED + m) for m in range(len(positions))]
    rows, cols = zs[0].shape
    res = wm.SHAPES[shape][0]
    g = te.Geometry.make(rows, cols, res)
    ctx.set_kernel(te.KERNEL_FUSED)
    m = te.Map(ctx)
    try:
        got = m.chain_batched(g, _params(te, shape), len(zs), np.stack(zs), outputs=True, positions=positions)
    finally:
        m.close()
        ctx.set_kernel(te.KERNEL_AUTO)
    for k, (z, pos) in enumerate(zip(zs, positions)):
        ref = oracle.chain(oracle.Geometry.make(rows, cols, res, pos), _params(oracle, shape), z)
        _parity({name: np.asarray(got[name][k]) for name in LAYERS}, ref)


def test_slabs_equal_the_whole_map(te, ctx):
    """The ShapeA probe map as 8 column slabs with 4-column halos, bit-identical to the whole map: windows that straddle a seam
    see the slab's edge, and tier 2 must read the halo rather than take it for the map's border."""
    import torch
    z = wm.probe("A", wm.all_masks("A"), "tilt", SEED)
    rows, cols = z.shape
    g, p = te.Geometry.make(rows, cols, wm.SHAPES["A"][0]), _params(te, "A")
    zd = torch.from_numpy(np.ascontiguousarray(z.T)).cuda()   # (cols, rows) tensor == column-major layer
    ctx.set_stream(None)
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        whole = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
        ctx.chain(g, p, zd, *whole, te.MEM_DEVICE)
        ctx.synchronize()
        w = cols // 8
        for b in range(0, cols, w):
            e = b + w
            hl, hr = min(4, b), min(4, cols - e)
            outs = [torch.empty((e - b, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
            ctx.chain(g, p, zd[b - hl:e + hr].contiguous(), *outs, te.MEM_DEVICE, slab=te.Slab(b, e - b, hl, hr))
            ctx.synchronize()
            for name, a, o in zip(LAYERS, whole, outs):
                assert torch.equal(a[b:e].view(torch.int32), o.view(torch.int32)), (b, name)
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)
