"""Every cell the fused chain's fix-up tiers recompute, held to what each tier claims (tier_exact.py states the exact values and
the rounding rule).

The chain runs KERNEL_FUSED in device memory, one launch, and te_get_fixup_cells reads the tier-2 and tier-3 work lists of that
launch.  On every listed cell:

  tier 2, do_n, not escalated  n_x, n_y, n_z and roughness are the correctly rounded exact values of the window on tier 2's
                               nominal grid (tier_exact.correctly_rounded; the roughness from the kernel's own normal); the slope
                               is within acos_t2's bound of the exact 1 - acos(n_z) / crit, and 0 from theta >= crit (1 + 2e-7)
  tier 2, do_s                 the step is the oracle's bit for bit (step_t2 is the reference's double arithmetic)
  tier 3                       slope, roughness and the normals are the oracle's bit for bit, the slope but where
                               literal_cases.slope_explained puts the difference on libm's acos
and on every cell, listed or not, the traversability is fmul_rn(w, fadd_rn(fadd_rn(s, t), r)) of the kernel's own layers, and
the fused n_z is the oracle's bit for bit wherever the oracle's lies in the certification band s = 1 - n_z < nz_check_limit
(DESIGN.md §4.1: such a cell is rounded exactly like the reference or flagged).  The tier-2 list holds every partial window and
every cell within the step reach of an infinite elevation.

Tolerance-based tests cannot see a tier 2 that lost precision (one moment in float, an early Halley stop, a wrong 1/n): within
1e-5 |b| + 1e-6 all of those pass.  These rules fail on one ulp."""
import time

import numpy as np
import pytest

import literal_cases as lc
import tier_exact as tx
import window_masks as wm
from helpers import chain_params

pytestmark = pytest.mark.gpu

SEED = 7
ORIGIN, MID, LV95 = (0.0, 0.0), (1234.5678, -987.6543), (2_600_000.0, 1_200_000.0)
LAYERS = ("slope", "step", "roughness", "traversability")
NORMALS = ("nx", "ny", "nz")
# Explained cells (tier 2 passes with the neighbour of the nearest float, the exact value within delta of a midpoint) per layer:
# at most 1e-4 of the tier-2 cells checked, plus one.  A correct tier 2 sits within ~1e-14 (1 + kappa) of the exact value, so a
# cell is explained only when its exact value falls within delta of a midpoint: a share of about 2 delta / ulp, below 1e-5 for
# every layer of these maps.
BUDGET = 1e-4
CHUNK = 200_000


@pytest.fixture(scope="module", autouse=True)
def _clock():
    t = time.time()
    yield
    print(f"\ntest_fused_tiers_gpu: {time.time() - t:.1f} s")


def _run(te, ctx, g, p, z, nmaps=1, normals=True):
    """KERNEL_FUSED on z ((nmaps,) rows, cols column-major float32) in device memory: one launch.  Returns the layers as
    (nmaps, rows, cols) arrays and the two work lists."""
    import torch
    zs = z if z.ndim == 3 else z[None]
    nm, rows, cols = zs.shape
    zd = torch.from_numpy(np.ascontiguousarray(zs.transpose(0, 2, 1))).cuda()   # (nmaps, cols, rows) == column-major layers
    names = LAYERS + (NORMALS if normals else ())
    outs = {k: torch.empty((nm, cols, rows), dtype=torch.float32, device="cuda") for k in names}
    ctx.set_stream(None)
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        if nm == 1:
            ctx.chain(g, p, zd, *(outs[k] for k in LAYERS), te.MEM_DEVICE,
                      **({k: outs[k] for k in NORMALS} if normals else {}))
        else:
            ctx.chain_batched(g, p, nm, zd, *(outs[k] for k in LAYERS), te.MEM_DEVICE)
        ctx.synchronize()
        got = {k: o.cpu().numpy().transpose(0, 2, 1) for k, o in outs.items()}
        return got, ctx.fixup_cells(2), ctx.fixup_cells(3), ctx.flag_counters()
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _fuse(w, s, t, r):
    f = np.float32
    with np.errstate(invalid="ignore", over="ignore"):
        return (f(w) * ((s.astype(f) + t.astype(f)).astype(f) + r.astype(f)).astype(f)).astype(f)


def _disk(res, r):
    """(k, l) offsets strictly inside a step window of radius r (on-circle tips left out: their membership is decided by the
    absolute coordinates)."""
    q = (r / res) ** 2
    return [(k, l) for k in range(-3, 4) for l in range(-3, 4) if k * k + l * l < q - 1e-6]


def _dilate(mask, offsets):
    rows, cols = mask.shape
    out = np.zeros_like(mask)
    ii, jj = np.nonzero(mask)
    for k, l in offsets:
        a, b = ii + k, jj + l
        ok = (a >= 0) & (a < rows) & (b >= 0) & (b < cols)
        out[a[ok], b[ok]] = True
    return out


def check_map(label, z, res, shape, crit, pos, got, l2, l3, ref, w, rough_crit=0.05, step_r=(0.04, 0.04), normals=True, stats=None):
    """Every rule of the module docstring on one map; got / ref hold that map's layers, l2 / l3 its work-list entries (cell index
    within the map)."""
    rows, cols = z.shape
    valid = np.isfinite(z)
    c2, c3 = l2 & 0x3FFFFFFF, l3 & 0x3FFFFFFF
    do_n, do_s = (l2 >> 30) & 1 == 1, (l2 >> 31) & 1 == 1
    assert len(np.unique(c2)) == len(c2) and len(np.unique(c3)) == len(c3), "a cell listed twice"
    assert np.isin(c3, c2[do_n]).all(), "tier 3 holds a cell tier 2 did not recompute"
    esc = np.zeros(rows * cols, bool)
    esc[c3] = True
    flat = lambda a: np.asarray(a).reshape(-1, order="F")   # noqa: E731  cell index = column * rows + row
    s = stats if stats is not None else {}
    s.update(listed2=len(c2), listed3=len(c3))

    # every cell: the traversability of the kernel's own layers, NaN exactly where a term is NaN
    fz = _fuse(w, got["slope"], got["step"], got["roughness"])
    assert _bits_equal(got["traversability"], fz).all(), int((~_bits_equal(got["traversability"], fz)).sum())

    # list contents
    partial = flat(wm.partial_windows(valid, shape))
    listed_n = np.zeros(rows * cols, bool)
    listed_n[c2[do_n]] = True
    assert listed_n[partial].all(), int((partial & ~listed_n).sum())
    inf = ~np.isnan(z) & ~np.isfinite(z)
    if inf.any():
        # cells whose step window holds a valid cell whose first window holds an infinite elevation (a step height of an invalid
        # centre is NaN and carries nothing)
        near = _dilate(_dilate(inf, _disk(res, step_r[0])) & valid, _disk(res, step_r[1]))
        listed_s = np.zeros(rows * cols, bool)
        listed_s[c2[do_s]] = True
        assert listed_s[flat(near)].all(), int((flat(near) & ~listed_s).sum())
        s["inf_reach"] = int(near.sum())

    # tier 2, do_s: step_t2 is the reference's arithmetic
    st = c2[do_s]
    assert _bits_equal(flat(got["step"])[st], flat(ref["step"])[st]).all(), int((~_bits_equal(flat(got["step"])[st], flat(ref["step"])[st])).sum())

    # tier 3: the literal kernel
    keys = ("slope", "roughness") + (NORMALS if normals else ())
    for k in keys:
        a, b = flat(got[k])[c3], flat(ref[k])[c3]
        off = np.nonzero(~_bits_equal(a, b))[0]
        if k == "slope" and len(off):
            x = flat(ref["nz"])[c3] if "nz" in ref else None
            assert x is not None, "tier-3 slope differs and no n_z to explain it"
            off = [q for q in off if not lc.slope_explained(float(x[q]), crit, a[q], b[q])[0]]
        assert len(off) == 0, (k, len(off))

    if not normals:
        return s
    # every cell in the certification band of n_z: the oracle's n_z bit for bit
    nzr = flat(ref["nz"])
    with np.errstate(invalid="ignore"):
        band = np.nonzero(np.isfinite(nzr) & (1.0 - nzr.astype(np.float64) < tx.nz_check_limit(crit)))[0]
    assert _bits_equal(flat(got["nz"])[band], nzr[band]).all(), int((~_bits_equal(flat(got["nz"])[band], nzr[band])).sum())
    s["band"] = len(band)

    # tier 2, do_n, not escalated: the exact values
    cells = c2[do_n]
    cells = cells[~esc[cells]]
    ci, cj = cells % rows, cells // rows
    hole = ~valid[ci, cj]
    for k in ("slope", "roughness") + NORMALS:
        assert np.isnan(got[k][ci[hole], cj[hole]]).all(), k
    ci, cj = ci[~hole], cj[~hole]
    s.update(checked=len(ci), expl_n=np.zeros(3, np.int64), expl_r=0, mp=0, slope_ratio=0.0)
    for q in range(0, len(ci), CHUNK):
        i, j = ci[q:q + CHUNK], cj[q:q + CHUNK]
        win = tx.Windows(z, shape, i, j, res)          # the nominal grid tier 2 computes on
        gn = np.stack([got[k][i, j] for k in NORMALS], -1)
        bad, expl, mp = tx.check_normals(win, gn)
        assert len(bad) == 0, (label, "normals", len(bad), [(int(i[b]), int(j[b]), gn[b].tolist()) for b in bad[:5]])
        bad_r, expl_r, mp_r = tx.check_roughness(win, gn, got["roughness"][i, j], rough_crit)
        assert len(bad_r) == 0, (label, "roughness", len(bad_r), [(int(i[b]), int(j[b])) for b in bad_r[:5]])
        ok, ratio = tx.slope_bound_ok(got["slope"][i, j], gn[:, 2], crit)
        assert ok.all(), (label, "slope", int((~ok).sum()), float(ratio.max()))
        s["expl_n"] += expl
        s["expl_r"] += expl_r
        s["mp"] += mp + mp_r
        s["slope_ratio"] = max(s["slope_ratio"], float(ratio.max()) if len(ratio) else 0.0)
    lim = BUDGET * s["checked"] + 1
    assert s["expl_n"].max() <= lim and s["expl_r"] <= lim, (label, s["expl_n"].tolist(), s["expl_r"], lim)
    return s


def _report(label, s, t):
    print(f"\n{label}: tier 2 {s['listed2']} listed, tier 3 {s['listed3']} escalated; "
          + (f"{s['checked']} checked, explained n {s['expl_n'].tolist()} roughness {s['expl_r']} (mpmath {s['mp']}), "
             f"worst slope error {s['slope_ratio']:.3f} of its bound; n_z band {s['band']} cells; " if "checked" in s else "")
          + (f"inf reach {s['inf_reach']}; " if "inf_reach" in s else "") + f"{time.time() - t:.1f} s")


def _masks(shape):
    return wm.sample_masks(shape, 1 << 16, SEED) if len(wm.DISKS[shape]) > 16 else wm.all_masks(shape)


PROBES = [(s, f, c, ORIGIN) for s in ("A", "B", "tips") for f in ("tilt", "nearflat", "inf") for c in (1.0, 0.1)] + \
         [("A", f, 1.0, pos) for pos in (MID, LV95) for f in ("tilt", "nearflat")]
PROBE_IDS = [f"{s}-{f}-crit{c}" + {ORIGIN: "", MID: "-mid", LV95: "-lv95"}[pos] for s, f, c, pos in PROBES]


@pytest.mark.parametrize("case", PROBES, ids=PROBE_IDS)
def test_window_mask_probes(te, ctx, oracle, case):
    shape, family, crit, pos = case
    label = PROBE_IDS[PROBES.index(case)]
    t = time.time()
    z = wm.probe(shape, _masks(shape), family, SEED)
    rows, cols = z.shape
    res = wm.SHAPES[shape][0]
    kw = {**wm.chain_kwargs(shape), "slope_critical": crit}
    ref = oracle.chain(oracle.Geometry.make(rows, cols, res, pos), chain_params(oracle, **kw), z, with_normals=True)
    got, l2, l3, cnt = _run(te, ctx, te.Geometry.make(rows, cols, res, pos), chain_params(te, **kw), z)
    assert cnt[2] == 0 and cnt[0] == len(l2) and cnt[4] == len(l3), (cnt, len(l2), len(l3))
    got = {k: v[0] for k, v in got.items()}
    # at LV95 the oracle's roughness carries its absolute-coordinate rounding: tier 2's is held to the exact value only (as
    # everywhere), tier 3's replays the oracle's arithmetic and must match it there too
    s = check_map(label, z, res, shape, crit, pos, got, l2, l3, ref, lc.YAML_W, step_r=(wm.SHAPES[shape][2],) * 2)
    _report(label, s, t)


def test_every_cell_on_the_slow_path(te, ctx, oracle):
    """An exactly planar map riddled with holes: the fp32 stencil certifies nothing, every valid cell is listed for tier 2 and
    most go on to tier 3 (the reference's rank test)."""
    t = time.time()
    rows, cols = 512, 384
    i, j = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    z = (0.25 * i + 0.125 * j).astype(np.float32) * np.float32(0.02)
    z[(i % 7 == 3) & (j % 5 == 1)] = np.nan
    z = np.asfortranarray(z)
    ref = oracle.chain(oracle.Geometry.make(rows, cols, 0.02), oracle.ChainParams.yaml_defaults(0), z, with_normals=True)
    got, l2, l3, _ = _run(te, ctx, te.Geometry.make(rows, cols, 0.02), te.ChainParams.yaml_defaults(0), z)
    got = {k: v[0] for k, v in got.items()}
    assert np.isin(np.nonzero(np.isfinite(z).reshape(-1, order="F"))[0], l2 & 0x3FFFFFFF).all()
    assert len(l3) > 0.5 * np.isfinite(z).sum(), len(l3)
    s = check_map("slow-path", z, 0.02, "A", 1.0, ORIGIN, got, l2, l3, ref, lc.YAML_W)
    _report("slow-path", s, t)


@pytest.mark.parametrize("res,shape", [(0.02, "A"), (0.03, "B")], ids=["0.02m", "0.03m"])
def test_bench_terrain(te, ctx, oracle, res, shape):
    """The benchmark's terrain at 2048^2: full windows reach tier 2 through the lambda_0, eigen-gap and n_z-band flags, the
    closed-form branch of k_fixup_t2 that the probes' partial windows do not take."""
    import torch
    import bench
    t = time.time()
    n = 2048
    z = np.asfortranarray(bench.terrain_torch(torch, n, 0, n, n, 3, True, "cpu").numpy().T)
    ref = oracle.chain(oracle.Geometry.make(n, n, res), oracle.ChainParams.yaml_defaults(0), z, with_normals=True)
    got, l2, l3, _ = _run(te, ctx, te.Geometry.make(n, n, res), te.ChainParams.yaml_defaults(0), z)
    got = {k: v[0] for k, v in got.items()}
    full = ~np.isin(l2 & 0x3FFFFFFF, np.nonzero(wm.partial_windows(np.isfinite(z), shape).reshape(-1, order="F"))[0])
    assert full.sum() > 100, int(full.sum())   # full windows on the list: the closed form is exercised
    label = f"bench-{res}m"
    s = check_map(label, z, res, shape, 1.0, ORIGIN, got, l2, l3, ref, lc.YAML_W)
    print(f"\n{label}: {int(full.sum())} listed cells with a full window")
    _report(label, s, t)


def test_batch_of_256_maps(te, ctx, oracle):
    """256 maps of 512^2 in one launch: the work lists index cells across maps (map * rows * cols + cell).  Eight terrains, each
    repeated over 32 maps; maps 0, 32, .., 224 are checked against the oracle.  The batched entry has no normals outputs, so the
    rules that need the kernel's normal are left to the single-map cases."""
    import torch
    import bench
    t = time.time()
    nm, n = 256, 512
    base = [np.asfortranarray(bench.terrain_torch(torch, n, 0, n, n, 100 + k, True, "cpu").numpy().T) for k in range(8)]
    zs = np.stack([base[m // 32] for m in range(nm)])
    got, l2, l3, _ = _run(te, ctx, te.Geometry.make(n, n, 0.02), te.ChainParams.yaml_defaults(0), zs, normals=False)
    cells = n * n
    for m in range(0, nm, 32):
        ref = oracle.chain(oracle.Geometry.make(n, n, 0.02), oracle.ChainParams.yaml_defaults(0), zs[m], with_normals=True)
        a2, a3 = l2[(l2 & 0x3FFFFFFF) // cells == m], l3[(l3 & 0x3FFFFFFF) // cells == m]
        a2 = (a2 & 0xC0000000) | ((a2 & 0x3FFFFFFF) - m * cells)
        a3 = (a3 & 0xC0000000) | ((a3 & 0x3FFFFFFF) - m * cells)
        s = check_map(f"batch map {m}", zs[m], 0.02, "A", 1.0, ORIGIN, {k: v[m] for k, v in got.items()}, a2.astype(np.uint32),
                      a3.astype(np.uint32), ref, lc.YAML_W, normals=False)
        _report(f"batch map {m}", s, t)


def test_batch_at_own_positions(te, ctx, oracle):
    """Probe maps with infinite holes, one te_map at four positions: step_t2 reads each map's own tip masks."""
    positions = [ORIGIN, LV95, MID, (-3.3, 7.7)]
    shape = "A"
    zs = [wm.probe(shape, wm.sample_masks(shape, 1 << 14, SEED + m), "inf", SEED + m) for m in range(len(positions))]
    rows, cols = zs[0].shape
    res = wm.SHAPES[shape][0]
    t = time.time()
    ctx.set_kernel(te.KERNEL_FUSED)
    m = te.Map(ctx)
    try:
        got = m.chain_batched(te.Geometry.make(rows, cols, res), chain_params(te, **wm.chain_kwargs(shape)), len(zs), np.stack(zs),
                              outputs=True, positions=positions)
        l2, l3 = ctx.fixup_cells(2), ctx.fixup_cells(3)
    finally:
        m.close()
        ctx.set_kernel(te.KERNEL_AUTO)
    cells = rows * cols
    for k, (z, pos) in enumerate(zip(zs, positions)):
        ref = oracle.chain(oracle.Geometry.make(rows, cols, res, pos), chain_params(oracle, **wm.chain_kwargs(shape)), z,
                           with_normals=True)
        a2, a3 = l2[(l2 & 0x3FFFFFFF) // cells == k], l3[(l3 & 0x3FFFFFFF) // cells == k]
        a2 = (a2 & 0xC0000000) | ((a2 & 0x3FFFFFFF) - k * cells)
        a3 = (a3 & 0xC0000000) | ((a3 & 0x3FFFFFFF) - k * cells)
        s = check_map(f"positions map {k}", z, res, shape, 1.0, pos, {name: np.asarray(got[name][k]) for name in LAYERS},
                      a2.astype(np.uint32), a3.astype(np.uint32), ref, lc.YAML_W, step_r=(wm.SHAPES[shape][2],) * 2, normals=False)
        _report(f"positions map {k}", s, t)
