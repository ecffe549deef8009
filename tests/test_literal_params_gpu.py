"""The literal kernels against the oracle across the parameters they accept.

KERNEL_GENERIC runs every parameter set, and TE_KERNEL_AUTO sends it every set fused_eligible refuses (raw-moment normals, a positive
axis other than z, rows % 4 != 0, a critical of 0, any radius outside the two fused shapes); te_normals, te_step, te_roughness and
te_slope run the same code.  They restate the oracle's double arithmetic operation for operation, so the rule is bit for bit, NaN
matching NaN: nx, ny, nz, step and roughness always, the traversability as numpy's float32 w * ((s + t) + r) of the kernel's own
layers, and the slope except at cells literal_cases.slope_explained puts within the double acos's error of a decision (CUDA's and
glibc's acos may round theta differently there).  A one-step float32 change anywhere else fails.

te_slope streams (k_slope_stream, a certified polynomial acos) when its pointers are 16-byte aligned and hands the rest to k_slope;
the stream must equal k_slope on every one of the 2^32 float32 inputs."""
import functools
import math

import numpy as np
import pytest

import literal_cases as lc
from helpers import same_bits_or_nan

pytestmark = pytest.mark.gpu

LAYERS = ("slope", "step", "roughness", "traversability")
EXACT = ("nx", "ny", "nz", "step", "roughness")
CRITS = (5e-324, 1e-300, 1e-12, 0.05, 0.436332, math.pi / 4, 1.0, float(np.nextafter(math.pi / 2, 0.0)), math.pi / 2)


@functools.lru_cache(maxsize=None)
def _ref(oracle, name):
    c = next(c for c in lc.CASES if c["name"] == name)
    return c, lc.terrain(c), oracle.chain(lc.geometry(oracle, c), lc.params(oracle, c), lc.terrain(c), with_normals=True)


def _explain_slope(nz, crit, got, ref, what):
    """The slope rule: (explained cells, largest distance to a decision in double ulps)."""
    ok, no = lc.slope_mismatches(nz, crit, got, ref)
    assert not no, (what, [(float(np.asarray(nz).reshape(-1)[c]), float(np.asarray(got).reshape(-1)[c]),
                            float(np.asarray(ref).reshape(-1)[c])) for c in no[:5]], len(no))
    return len(ok), max((k for _, k in ok), default=0)


def _assert_chain(got, ref, crit, w, what):
    for k in EXACT:
        assert same_bits_or_nan(got[k], ref[k]), (what, k, int((np.asarray(got[k]) != ref[k]).sum()))
    n, k = _explain_slope(got["nz"], crit, got["slope"], ref["slope"], what)
    fused = np.float32(w) * ((got["slope"] + got["step"]) + got["roughness"])
    assert same_bits_or_nan(got["traversability"], fused), what
    return n, k


@pytest.mark.parametrize("case", lc.IDS)
def test_generic_chain_against_the_oracle(te, ctx, oracle, case):
    c, z, ref = _ref(oracle, case)
    ctx.set_kernel(te.KERNEL_GENERIC)
    try:
        got = ctx.chain_host(lc.geometry(te, c), lc.params(te, c), z, with_normals=True)
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)
    p = lc.params(te, c)
    n, k = _assert_chain(got, ref, p.slope_critical, p.fuse_weight, case)
    axis = p.normals_positive_axis
    flipped = int((np.asarray(got[("nx", "ny", "nz")[axis]]) > 0).sum()) if axis != 2 else 0
    print(f"{case}: {c['fails']}; cells {z.size}, n[{axis}] > 0 on {flipped}, slope cells explained by acos {n} (<= {k} ulps)")


@pytest.mark.parametrize("case", lc.IDS)
def test_auto_takes_the_literal_kernels_where_fused_refuses(te, ctx, oracle, case):
    c, z, _ = _ref(oracle, case)
    g, p = lc.geometry(te, c), lc.params(te, c)
    out = {}
    try:
        for name, kernel in (("generic", te.KERNEL_GENERIC), ("auto", te.KERNEL_AUTO)):
            ctx.set_kernel(kernel)
            out[name] = ctx.chain_host(g, p, z, with_normals=True)
        ctx.set_kernel(te.KERNEL_FUSED)
        with pytest.raises(te.TEError) as e:
            ctx.chain_host(g, p, z)
        assert e.value.code == -4, (case, lc.refusal(c))
    finally:
        ctx.set_kernel(te.KERNEL_AUTO)
    for k in out["generic"]:
        assert same_bits_or_nan(out["auto"][k], out["generic"][k]), (case, k)
    print(f"{case}: refused for {lc.refusal(c)}")


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32).T)).cuda()   # (cols, rows) == column-major layer


@pytest.mark.parametrize("memory", ["host", "device"])
@pytest.mark.parametrize("case", lc.IDS)
def test_standalone_filters_against_the_oracle(te, ctx, oracle, case, memory):
    import torch
    c, z, ref = _ref(oracle, case)
    g, og, p, po = lc.geometry(te, c), lc.geometry(oracle, c), lc.params(te, c), lc.params(oracle, c)
    rows, cols = z.shape
    nx, ny, nz = ref["nx"], ref["ny"], ref["nz"]
    want = dict(nx=nx, ny=ny, nz=nz, step=oracle.step(og, po, z), roughness=oracle.roughness(og, po, z, nx, ny, nz),
                slope=oracle.slope(og, po.slope_critical, nz))
    if memory == "host":
        M, new, inp, back = te.MEM_HOST, (lambda: np.empty((rows, cols), np.float32, order="F")), (lambda a: a), (lambda a: a)
    else:
        ctx.set_stream(None)
        M = te.MEM_DEVICE
        new = lambda: torch.empty((cols, rows), dtype=torch.float32, device="cuda")  # noqa: E731
        inp, back = (lambda a: _dev(torch, a)), (lambda t: (ctx.synchronize(), t.cpu().numpy().T)[1])
    got = {k: new() for k in want}
    dz, dnx, dny, dnz = (inp(a) for a in (z, nx, ny, nz))   # alive until the kernels that read them have finished
    ctx.normals(g, p, dz, got["nx"], got["ny"], got["nz"], M)
    ctx.step(g, p, dz, got["step"], M)
    ctx.roughness(g, p, dz, dnx, dny, dnz, got["roughness"], M)
    ctx.slope(g, p.slope_critical, dnz, got["slope"], M)
    got = {k: back(v) for k, v in got.items()}
    for k in EXACT:
        assert same_bits_or_nan(got[k], want[k]), (case, memory, k)
    n, k = _explain_slope(nz, p.slope_critical, got["slope"], want["slope"], case)
    print(f"{case} {memory}: slope cells explained by acos {n} (<= {k} ulps)")


# ---- te_slope: its edge entries, the stream against k_slope on every float32, the literal slope against the oracle ----------------

def _slope_dev(te, ctx, crit, x, out):
    n = x.numel()
    ctx.slope(te.Geometry.make(n, 1, 0.02), crit, x, out, te.MEM_DEVICE)


def test_slope_edge_entries(te, ctx, oracle):
    import torch
    ctx.set_stream(None)
    rng = np.random.default_rng(3)
    for n in (1, 2, 3, 5, 6, 7, 4096 + 3):                   # total % 4 != 0: the tail cells run k_slope after the stream
        x = rng.uniform(-1.2, 1.2, n).astype(np.float32)
        x[::5] = np.nan
        for crit in (0.0, 0.3, 1.0):
            want = oracle.slope(oracle.Geometry.make(n, 1, 0.02), crit, x.reshape(n, 1)).reshape(-1)
            for misalign in (0, 1):                          # the output 4 bytes off 16-byte alignment: k_slope for the whole layer
                buf = torch.full((n + 4,), 7.0, dtype=torch.float32, device="cuda")
                out = buf[misalign:misalign + n]
                _slope_dev(te, ctx, crit, torch.from_numpy(x).cuda(), out)
                ctx.synchronize()
                _explain_slope(x, crit, out.cpu().numpy(), want, (n, crit, misalign))
                b = buf.cpu().numpy()
                assert (np.delete(b, np.arange(misalign, misalign + n)) == 7.0).all()     # nothing written outside the layer
            if crit == 0.0:
                assert (want[np.isfinite(x)] == 0.0).all()   # theta < 0 never holds
    x = torch.from_numpy(rng.uniform(-1, 1, 64).astype(np.float32)).cuda()
    out = torch.full((64,), 7.0, dtype=torch.float32, device="cuda")
    for crit in (float("nan"), -1e-300, -0.5, math.pi / 2 * (1 + 1e-15), 2.0, float("inf")):
        with pytest.raises(te.TEError) as e:
            _slope_dev(te, ctx, crit, x, out)
        assert e.value.code == -1, crit
        ctx.synchronize()
        assert (out.cpu().numpy() == 7.0).all(), crit
        h = np.full(64, 7.0, np.float32)
        with pytest.raises(te.TEError):
            ctx.slope(te.Geometry.make(64, 1, 0.02), crit, x.cpu().numpy(), h, te.MEM_HOST)
        assert (h == 7.0).all()


CHUNK = 1 << 28


@pytest.mark.parametrize("crit", CRITS, ids=[f"{c!r}" for c in CRITS])
def test_slope_stream_equals_k_slope_on_every_float32(te, ctx, crit):
    """Every float32 bit pattern through te_slope twice: 16-byte aligned (k_slope_stream) and with the output one float off
    (k_slope).  Equal bit for bit, NaNs included."""
    import time
    import torch
    ctx.set_stream(None)
    base = torch.arange(CHUNK, dtype=torch.int32, device="cuda")
    x = torch.empty(CHUNK, dtype=torch.int32, device="cuda")
    a = torch.empty(CHUNK, dtype=torch.float32, device="cuda")
    b = torch.empty(CHUNK + 4, dtype=torch.float32, device="cuda")
    t0 = time.perf_counter()
    bad = 0
    try:
        for k in range(1 << 4):
            lo = -(1 << 31) + k * CHUNK
            torch.add(base, lo, out=x)
            f = x.view(torch.float32)
            _slope_dev(te, ctx, crit, f, a)
            _slope_dev(te, ctx, crit, f, b[1:CHUNK + 1])
            ctx.synchronize()
            bad += int((a.view(torch.int32) != b[1:CHUNK + 1].view(torch.int32)).sum())
    finally:
        del base, x, a, b
        torch.cuda.empty_cache()
    print(f"crit {crit!r}: 2^32 inputs in {time.perf_counter() - t0:.2f} s, {bad} differ")
    assert bad == 0


def _decision_criticals():
    """(crit, x) pairs whose slope 1 - acos(x) / crit lies on a decision of k_slope_stream: a float32 rounding midpoint just below a
    power of two (where the float32 spacing halves), a midpoint elsewhere, and the branch point acos(x) == crit.  The polynomial
    acos and the literal one then round to different sides unless the stream hands the cell to the literal expression."""
    rng = np.random.default_rng(17)
    out = []
    for x in np.sort(rng.uniform(0.2, 0.99, 48).astype(np.float32)):
        t = math.acos(float(x))
        for e in (-1, -2, -3):
            m = 2.0 ** e - 2.0 ** (e - 25)                                         # midpoint of 2^e and the float32 below it
            out.append((t / (1.0 - m), x))
        v = np.float32(rng.uniform(0.1, 0.9))
        m = (float(v) + float(np.nextafter(v, np.float32(1)))) / 2                 # a midpoint elsewhere
        out.append((t / (1.0 - m), x))
        out.append((t, x))                                                         # the branch point
    return [(c, x) for c, x in out if 0.0 < c <= math.pi / 2]


def test_slope_stream_on_its_decisions(te, ctx, oracle):
    """At criticals built to put an input's slope on each decision of the stream, stream and k_slope agree bit for bit, and the
    oracle agrees under the acos rule.  The inputs around x (64 float32 on either side) sit next to the same decisions."""
    import torch
    ctx.set_stream(None)
    cases = _decision_criticals()
    assert len(cases) > 120
    near = far = 0
    for crit, x in cases:
        xs = (x.view(np.int32) + np.arange(-64, 64, dtype=np.int32)).view(np.float32)
        xd = torch.from_numpy(xs).cuda()
        out = torch.empty(len(xs) + 4, dtype=torch.float32, device="cuda")
        _slope_dev(te, ctx, crit, xd, out[:len(xs)])
        ctx.synchronize()
        a = out[:len(xs)].cpu().numpy()
        _slope_dev(te, ctx, crit, xd, out[1:len(xs) + 1])
        ctx.synchronize()
        b = out[1:len(xs) + 1].cpu().numpy()
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (crit, float(x))
        want = oracle.slope(oracle.Geometry.make(len(xs), 1, 0.02), crit, xs.reshape(-1, 1)).reshape(-1)
        n, k = _explain_slope(xs, crit, b, want, crit)
        near, far = near + n, max(far, k)
    print(f"{len(cases)} criticals, {near} cells explained by acos (<= {far} ulps)")


def _dense_inputs():
    """Every float32 in [0.5, 1], every 64th in [0, 0.5), and the specials."""
    half, one = np.float32(0.5).view(np.uint32), np.float32(1.0).view(np.uint32)
    specials = np.array([0.0, -0.0, 1.0, -1.0, 1.5, -1.5, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, 1.1754942e-38, np.nan],
                        np.float32)
    payloads = np.array([0x7f800001, 0xff800001, 0x7fc00001, 0xffffffff, 0x7fbfffff], np.uint32).view(np.float32)
    return np.concatenate([np.arange(half, one + 1, dtype=np.uint32).view(np.float32),
                           np.arange(0, half, 64, dtype=np.uint32).view(np.float32), specials, payloads])


@pytest.mark.parametrize("crit", CRITS, ids=[f"{c!r}" for c in CRITS])
def test_literal_slope_against_the_oracle_on_dense_inputs(te, ctx, oracle, crit):
    import torch
    x = _dense_inputs()
    x = np.concatenate([x, np.zeros((-len(x)) % 4, np.float32)])
    want = oracle.slope(oracle.Geometry.make(len(x), 1, 0.02), crit, x.reshape(-1, 1)).reshape(-1)
    ctx.set_stream(None)
    xd = torch.from_numpy(x).cuda()
    out = torch.empty(len(x) + 4, dtype=torch.float32, device="cuda")
    for name, o in (("stream", out[:len(x)]), ("k_slope", out[1:len(x) + 1])):
        _slope_dev(te, ctx, crit, xd, o)
        ctx.synchronize()
        n, k = _explain_slope(x, crit, o.cpu().numpy(), want, (crit, name))
        print(f"crit {crit!r} {name}: {len(x)} inputs, explained by acos {n} (<= {k} ulps)")


# ---- the other chain entries at two refused parameter sets ---------------------------------------------------------------------

def _lattice_reach(r, res, cu):
    n = math.floor(r / res + 1e-9)
    while float((n + 1) * (n + 1)) * res * res <= r * r + 8.0 * r * cu:
        n += 1
    return n


def _chain_halo(g, p):
    """The dependency radius in columns that a slab must carry (te_capi.cu chain_halo, restated)."""
    rmax = max(p.normals_radius, p.roughness_radius, p.step_first_radius + p.step_second_radius)
    m = max(abs(g.position_x) + 0.5 * g.length_x, abs(g.position_y) + 0.5 * g.length_y) + rmax
    cu = math.ldexp(1.0, math.frexp(max(m, 1.0))[1] - 1 - 52)
    lr = lambda r: _lattice_reach(r, g.resolution, cu)  # noqa: E731
    return max(lr(p.normals_radius), lr(p.roughness_radius), lr(p.step_first_radius) + lr(p.step_second_radius))


def _maps(n, rows, cols, seed):
    import synth
    return [np.asfortranarray(synth.terrain(rows, cols, 0.02, seed + k, ("gentle", "mixed", "rough")[k % 3])) for k in range(n)]


def _bits_equal(torch, a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("which", list(lc.OTHER_SETS))
def test_batched_equals_single_maps(te, ctx, which):
    import torch
    rows, cols, n = 256, 192, 8
    g, p = te.Geometry.make(rows, cols, 0.02), lc.params(te, dict(params=lc.OTHER_SETS[which]))
    zd = torch.stack([_dev(torch, z) for z in _maps(n, rows, cols, 300)])
    outs = [torch.empty((n, cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
    ctx.set_stream(None)
    ctx.chain_batched(g, p, n, zd, *outs, te.MEM_DEVICE)
    ctx.synchronize()
    for k in range(n):
        one = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
        ctx.chain(g, p, zd[k].contiguous(), *one, te.MEM_DEVICE)
        ctx.synchronize()
        for name, a, b in zip(LAYERS, outs, one):
            assert _bits_equal(torch, a[k], b), (which, k, name)


@pytest.mark.parametrize("which", list(lc.OTHER_SETS))
def test_slabs_at_the_halo_equal_the_whole_map(te, ctx, which):
    import torch
    rows, cols = 128, 160
    for pos in ((0.0, 0.0), lc.LV95):
        g, p = te.Geometry.make(rows, cols, 0.02, pos), lc.params(te, dict(params=lc.OTHER_SETS[which]))
        h = _chain_halo(g, p)
        assert h >= 1
        zd = _dev(torch, _maps(1, rows, cols, 310)[0])
        ctx.set_stream(None)
        whole = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
        ctx.chain(g, p, zd, *whole, te.MEM_DEVICE)
        ctx.synchronize()
        for b, e in ((0, 40), (40, 100), (100, cols)):
            hl, hr = min(h, b), min(h, cols - e)
            outs = [torch.empty((e - b, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
            ctx.chain(g, p, zd[b - hl:e + hr].contiguous(), *outs, te.MEM_DEVICE, slab=te.Slab(b, e - b, hl, hr))
            ctx.synchronize()
            for name, a, o in zip(LAYERS, whole, outs):
                assert _bits_equal(torch, a[b:e], o), (which, pos, b, name)
        with pytest.raises(te.TEError) as err:                # one halo column fewer is refused
            outs = [torch.empty((60, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
            ctx.chain(g, p, zd[40 - h:100 + h - 1].contiguous(), *outs, te.MEM_DEVICE, slab=te.Slab(40, 60, h, h - 1))
        assert err.value.code == -1
        print(f"{which} at {pos}: halo {h}")


@pytest.mark.parametrize("which", list(lc.OTHER_SETS))
def test_map_chain_batched_at_lv95_equals_single_chains(te, ctx, which):
    rows, cols, n = 128, 96, 4
    p = lc.params(te, dict(params=lc.OTHER_SETS[which]))
    zs = _maps(n, rows, cols, 320)
    pos = np.array([[lc.LV95[0] + 3.0 * k, lc.LV95[1] - 1.5 * k] for k in range(n)])
    m = ctx.map()
    try:
        got = m.chain_batched(te.Geometry.make(rows, cols, 0.02), p, n, np.stack(zs), outputs=True, positions=pos)
    finally:
        m.close()
    for k in range(n):
        want = ctx.chain_host(te.Geometry.make(rows, cols, 0.02, tuple(pos[k])), p, zs[k])
        for name in LAYERS:
            assert same_bits_or_nan(got[name][k], want[name]), (which, k, name)
