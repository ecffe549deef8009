"""The fused chain against the oracle away from the YAML parameters.  fused_eligible accepts any slope_critical,
step_critical, roughness_critical above 0, any step_critical_cells and fuse_weight, and any radii and resolution whose windows
fall into its two instantiated shapes; the plugin shells pass a robot's YAML straight through.  Every case runs KERNEL_FUSED,
which raises TE_ERR_UNSUPPORTED rather than fall back to the generic kernel, and compares with oracle.chain: tolerance, exact
NaN mask and exact 0/1 branch cells (for the traversability: where its three terms are branch values).  Besides random terrain there are maps built to put many cells where the layers are
sensitive: an inclination ramp (theta in [0.012, 0.05] rad, where one float32 ulp of n_z moves the slope layer by more than its
tolerance when slope_critical is small, and theta around every critical value), a roughness ramp, and step terraces whose
nCells / step_critical_cells * stepMax lands within a float32 ulp of step_critical."""
import functools

import numpy as np
import pytest

import synth
from helpers import assert_parity, chain_params, compare_layer

pytestmark = pytest.mark.gpu

LAYERS = ("slope", "step", "roughness", "traversability")
N = 1024


# Open case: with a power-of-two step_critical_cells, CNT * (1/ncrit) * stepMax rounds once in fp32 and may land just below
# step_critical where the reference's double step is >= it, so the step layer comes out ~1e-7 instead of exactly 0 (the YAML's
# 0.12 m and 4 cells too, in a 1e-9 m wide window of stepMax that the terraces there happen to miss).  Rounding 1/crit up would
# change the YAML outputs; deciding the branch exactly costs march-step instructions.  Allowed: these step branch cells, and
# nothing else on those maps.
STEP_BRANCH_OPEN = {(0.04, 4): 64, (0.01, 4): 64}


def _parity(got, ref, step_branch=0):
    """assert_parity for slope and roughness; the step layer may have `step_branch` branch cells off (and nothing else); the
    traversability's exact cells are those where each of its three terms is a branch value (0 or 1) in the reference and in
    the result: w * (s + t + r) equals 1.0 also where s + t + r = 1/w from terms inside their tolerance, which is no branch."""
    assert_parity(got, ref, keys=("slope", "roughness"))
    st = compare_layer(got["step"], ref["step"], "step")
    assert st["nan_mismatch"] == 0 and st["out_of_tol"] == 0 and st["branch_mismatch"] <= step_branch, st
    tr = compare_layer(got["traversability"], ref["traversability"], "traversability")
    assert tr["nan_mismatch"] == 0 and tr["out_of_tol"] == 0, tr
    exact = np.ones(ref["traversability"].shape, bool)
    for k in ("slope", "step", "roughness"):
        exact &= ((ref[k] == 0.0) | (ref[k] == 1.0)) & (got[k] == ref[k])
    a, b = got["traversability"][exact], ref["traversability"][exact]
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), int((a != b).sum())


def _fused(te, ctx, oracle, z, res=0.02, pos=(0.0, 0.0), what="", step_branch=0, **kw):
    """KERNEL_FUSED and oracle.chain on z with the parameters kw; parity asserted; returns (layers, oracle layers, counters)."""
    rows, cols = z.shape
    g, og = te.Geometry.make(rows, cols, res, pos), oracle.Geometry.make(rows, cols, res, pos)
    ref = oracle.chain(og, chain_params(oracle, **kw), z)
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        got = ctx.chain_host(g, chain_params(te, **kw), z)
        cnt = ctx.flag_counters()
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)
    print(f"{what} {kw}: tier 2 {cnt[0]} cells, tier 3 {cnt[4]} cells")
    assert cnt[2] == 0, cnt
    _parity(got, ref, step_branch)
    return got, ref, cnt


@functools.lru_cache(maxsize=None)
def _terrain(preset, n=N, seed=21):
    return synth.terrain(n, n, 0.02, seed, preset)


# ---- one parameter at a time around the YAML values, then a few combinations -------------------------------------------

AXES = [("slope_critical", v) for v in (1.0, np.pi / 4, 0.5, 0.436332, 0.3, 0.2, 0.1, 0.05)] + \
       [("roughness_critical", v) for v in (0.05, 0.3, 0.1, 0.02, 0.01, 0.005)] + \
       [("step_critical", v) for v in (0.12, 0.3, 0.04, 0.01)] + \
       [("step_critical_cells", v) for v in (1, 2, 3, 4, 5, 9)] + \
       [("fuse_weight", v) for v in (float(np.float32(1.0) / np.float32(3.0)), 1.0, 0.5, float(np.float32(0.1)))]
COMBOS = [dict(slope_critical=0.3, roughness_critical=0.02, step_critical_cells=3),
          dict(slope_critical=0.1, roughness_critical=0.01, step_critical=0.04, step_critical_cells=5, fuse_weight=0.5),
          dict(slope_critical=0.436332, roughness_critical=0.3, step_critical=0.3, step_critical_cells=9, fuse_weight=1.0),
          dict(slope_critical=0.05, roughness_critical=0.005, step_critical=0.01, step_critical_cells=2)]


@pytest.mark.parametrize("preset", ["gentle", "mixed", "rough"])
@pytest.mark.parametrize("name,value", AXES, ids=[f"{k}={v:.6g}" for k, v in AXES])
def test_one_parameter_at_a_time(te, ctx, oracle, preset, name, value):
    _fused(te, ctx, oracle, _terrain(preset), what=preset, **{name: value})


@pytest.mark.parametrize("preset", ["gentle", "mixed", "rough"])
@pytest.mark.parametrize("combo", range(len(COMBOS)))
def test_combinations(te, ctx, oracle, preset, combo):
    _fused(te, ctx, oracle, _terrain(preset), what=preset, **COMBOS[combo])


def test_2048_at_a_low_slope_critical(te, ctx, oracle):
    _fused(te, ctx, oracle, _terrain("mixed", 2048, 5), what="2048", slope_critical=0.3)


# ---- terrain aimed at the sensitive bands -----------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _inclination_ramp():
    """Inclination rising smoothly along the columns from 0 to 1.3 rad (a quadratic in the column so that a fifth of the map has
    theta < 0.1), plus fbm and 1 mm of white noise: curved, rough enough that fp32 certifies the cells rather than tier 3
    handling exact planes."""
    rows = cols = N
    t = 1.3 * (np.arange(cols) / (cols - 1.0)) ** 2
    z = np.cumsum(np.tan(t)) * 0.02                                           # dz/dy = tan(theta(y))
    rng = np.random.default_rng(3)
    zz = z[None, :] + synth.fbm(rows, cols, 0.02, 4, 0.01) + 1e-3 * rng.standard_normal((rows, cols))
    return np.asfortranarray(zz.astype(np.float32))


@functools.lru_cache(maxsize=None)
def _roughness_ramp(crit):
    """White noise whose amplitude rises along the rows, so that the roughness spans 0 to about 3 * crit, on gentle fbm."""
    rows = cols = N
    rng = np.random.default_rng(int(crit * 1e4))
    amp = 3.0 * crit * np.arange(rows) / (rows - 1.0)
    z = synth.fbm(rows, cols, 0.02, 8, 0.15) + amp[:, None] * rng.standard_normal((rows, cols))
    return np.asfortranarray(z.astype(np.float32))


@pytest.mark.parametrize("crit", [1.0, np.pi / 4, 0.5, 0.436332, 0.3, 0.2, 0.1, 0.05])
def test_inclination_ramp(te, ctx, oracle, crit):
    z = _inclination_ramp()
    _, ref, _ = _fused(te, ctx, oracle, z, what="inclination ramp", slope_critical=crit)
    s = ref["slope"][np.isfinite(ref["slope"])]
    assert (s == 0.0).any() and ((s > 0.0) & (s < 1e-3)).any()               # the ramp crosses theta = crit


@pytest.mark.parametrize("crit", [0.05, 0.3, 0.1, 0.02, 0.01, 0.005])
def test_roughness_ramp(te, ctx, oracle, crit):
    z = _roughness_ramp(crit)
    _fused(te, ctx, oracle, z, what="roughness ramp", roughness_critical=crit)


def _terraces(crit, ncrit, rows=512, cols=512):
    """Single raised cells on flat ground, 12 cells apart.  A pillar of height H gives step_height H to the cells of its first
    step window, and the cells around see n of those in their second window, n = 1 .. 13: their step is min(H, n / ncrit * H).
    The heights are the float32 values within 3 ulps of crit * ncrit / n for every n (and of crit), so that the step lands within
    an ulp of step_critical on either side, where the kernel's CNT * (1/ncrit) * stepMax in fp32 and the reference's double
    expression must take the same branch."""
    targets = sorted({crit * ncrit / n for n in range(1, 14)} | {crit})
    heights = []
    for t in targets:
        h = np.float32(t)
        below, above = [h], [h]
        for _ in range(3):
            below.append(np.nextafter(below[-1], np.float32(-np.inf)))
            above.append(np.nextafter(above[-1], np.float32(np.inf)))
        heights += below[:0:-1] + above
    z = np.zeros((rows, cols), np.float32)
    slots = [(i, j) for i in range(6, rows - 6, 12) for j in range(6, cols - 6, 12)]
    assert len(slots) >= len(heights)
    for q, (i, j) in enumerate(slots):
        z[i, j] = heights[q % len(heights)]
    return np.asfortranarray(z)


TERRACES = [(0.12, c) for c in (1, 2, 3, 4, 5, 9)] + [(s, c) for s in (0.3, 0.04, 0.01) for c in (3, 4)]


@pytest.mark.parametrize("step_crit,ncrit", TERRACES)
def test_step_terraces(te, ctx, oracle, step_crit, ncrit):
    z = _terraces(step_crit, ncrit)
    _, ref, _ = _fused(te, ctx, oracle, z, what="terraces", step_critical=step_crit, step_critical_cells=ncrit,
                       step_branch=STEP_BRANCH_OPEN.get((step_crit, ncrit), 0))
    near = (ref["step"] == 0.0) | ((ref["step"] > 0.0) & (ref["step"] < 1e-6))
    assert near.sum() > 100, int(near.sum())                                  # many cells sit on the branch point


# ---- radii and resolutions inside the two instantiated shapes ----------------------------------------------------------------

SHAPES = [  # (resolution, normals = roughness radius, step first, step second)
    (0.02, 0.046, 0.04, 0.04),    # ShapeA, r/res = 2.3 in (sqrt 5, sqrt 8)
    (0.02, 0.055, 0.04, 0.04),    # ShapeA, r/res = 2.75
    (0.021, 0.05, 0.042, 0.042),  # ShapeA, step tips exactly on the circle: decided by the double-precision masks
    (0.025, 0.045, 0.03, 0.03),   # ShapeB
]


@pytest.mark.parametrize("shape", range(len(SHAPES)))
@pytest.mark.parametrize("nondefault", [False, True])
def test_radii_inside_the_fused_shapes(te, ctx, oracle, shape, nondefault):
    res, rn, r1, r2 = SHAPES[shape]
    z = synth.terrain(512, 512, res, 40 + shape, "mixed")
    kw = dict(normals_radius=rn, roughness_radius=rn, step_first_radius=r1, step_second_radius=r2)
    if nondefault:
        kw.update(slope_critical=0.3, roughness_critical=0.02, step_critical_cells=3)
    _fused(te, ctx, oracle, z, res=res, what=f"shape {SHAPES[shape]}", **kw)   # KERNEL_FUSED raises if it refuses them


# ---- map positions far from the origin ------------------------------------------------------------------------------------

@pytest.mark.parametrize("pos", [(2_600_000.0, 1_200_000.0), (1234.5678, -987.6543)])
@pytest.mark.parametrize("kw", [dict(), dict(slope_critical=0.3, roughness_critical=0.02, step_critical_cells=3),
                                dict(slope_critical=0.1)], ids=["yaml", "set", "slope0.1"])
def test_far_from_the_origin(te, ctx, oracle, pos, kw):
    """The reference forms window offsets from absolute coordinates: its rounding there moves its n_z, and nz_guard (tier 2's
    band around a float32 rounding boundary) grows with the coordinates."""
    z = synth.terrain(N, N, 0.02, 61, "mixed", pos)
    _fused(te, ctx, oracle, z, pos=pos, what=f"at {pos}", **kw)


# ---- the other entries at one non-default set --------------------------------------------------------------------------------

SET = dict(slope_critical=0.3, roughness_critical=0.02, step_critical_cells=3)


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).T)).cuda()   # (cols, rows) tensor == column-major layer


def _bits_equal(torch, a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_batched_equals_single_maps(te, ctx):
    import torch
    rows, cols, n = 512, 384, 8
    g, p = te.Geometry.make(rows, cols, 0.02), chain_params(te, **SET)
    maps = np.stack([np.ascontiguousarray(synth.terrain(rows, cols, 0.02, 500 + k, ("gentle", "mixed", "rough")[k % 3]).T)
                     for k in range(n)])
    zd = torch.from_numpy(maps).cuda()
    outs = [torch.empty((n, cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
    ctx.set_stream(None)
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        ctx.chain_batched(g, p, n, zd, *outs, te.MEM_DEVICE)
        ctx.synchronize()
        for k in range(n):
            one = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
            ctx.chain(g, p, zd[k], *one, te.MEM_DEVICE)
            ctx.synchronize()
            for name, a, b in zip(LAYERS, outs, one):
                assert _bits_equal(torch, a[k], b), (k, name)
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)


def test_slabs_equal_the_whole_map(te, ctx):
    import torch
    rows = cols = 2048
    z = _terrain("mixed", 2048, 5)
    g, p = te.Geometry.make(rows, cols, 0.02), chain_params(te, **SET)
    zd = _dev(torch, z)
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
                assert _bits_equal(torch, a[b:e], o), (b, name)
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)


def test_map_chain_equals_context_chain(te, ctx):
    z = _terrain("rough", 512, 9)
    g, p = te.Geometry.make(512, 512, 0.02), chain_params(te, **SET)
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        want = ctx.chain_host(g, p, z)
        m = te.Map(ctx)
        try:
            got = m.chain(g, p, z, outputs=True)
        finally:
            m.close()
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)
    for k in LAYERS:
        assert np.array_equal(np.asarray(got[k]).view(np.uint32), want[k].view(np.uint32)), k


# ---- parameter switches on one context ----------------------------------------------------------------------------------------

def test_parameter_switches_on_one_context(te, ctx):
    """FusedState caches its tables under a memcmp of (geometry, parameters), and the counters are double-buffered: alternating
    parameter sets on one context must give what a fresh context gives, bit for bit, every time."""
    z = _terrain("mixed", 512, 13)
    g = te.Geometry.make(512, 512, 0.02)
    sets = [dict(), SET, dict(slope_critical=0.1, step_critical=0.04, step_critical_cells=5, fuse_weight=0.5), SET, dict(),
            dict(normals_radius=0.055, roughness_radius=0.055), dict()]
    fresh = {}
    for kw in sets:
        key = tuple(sorted(kw.items()))
        if key not in fresh:
            c = te.Context(0)
            try:
                c.set_kernel(te.KERNEL_FUSED)
                fresh[key] = (c.chain_host(g, chain_params(te, **kw), z), c.flag_counters())
            finally:
                c.close()
    ctx.set_kernel(te.KERNEL_FUSED)
    try:
        for kw in sets:
            got = ctx.chain_host(g, chain_params(te, **kw), z)
            want, cnt = fresh[tuple(sorted(kw.items()))]
            for k in LAYERS:
                assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), (kw, k)
            c = ctx.flag_counters()   # cells flagged, overflow, tier 3 (entry 1 counts chunks, which depend on the warps' order)
            assert (c[0], c[2], c[4]) == (cnt[0], cnt[2], cnt[4]), (kw, c, cnt)
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)
