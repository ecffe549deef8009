"""Edge cases of the chain on the GPU: the certification ladder must hand every hard cell to a tier that gets it right."""
import numpy as np
import pytest

import literal_cases
import synth
from helpers import assert_parity, compare_layer

pytestmark = pytest.mark.gpu


def _pair(te, ob, rows, cols, res=0.02, pos=(0.0, 0.0)):
    return te.Geometry.make(rows, cols, res, pos), ob.Geometry.make(rows, cols, res, pos)


def test_exact_planes_go_to_the_literal_tier(te, ctx, oracle):
    """Exactly planar windows are rank-deficient for the reference's QR test (normal (0,0,1) even when tilted): fp32 cannot
    decide that, tier 2 passes it on, tier 3 replays the reference arithmetic."""
    rows, cols = 128, 96
    g, og = _pair(te, oracle, rows, cols)
    i, j = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    z = (0.125 * i + 0.0625 * j).astype(np.float32) * np.float32(0.02)   # dyadic slopes: exactly representable plane
    z[40:60, 30:50] = np.float32(0.5)                                      # an exactly flat plateau with cliffs around it
    ref = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z, with_normals=True)
    ctx.set_kernel(te.KERNEL_FUSED)
    got = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z, with_normals=True)
    cnt = ctx.flag_counters()
    assert cnt[4] > 1000, cnt                  # the planar interior reached tier 3
    assert_parity(got, ref)
    # the reference's own quirk: on an exactly planar tilted window the rank test sits on rounding noise of the absolute
    # positions, so the layer is 1.0 (normal (0,0,1)) at some cells and the true inclination at others — tier 3 reproduces both
    interior = ref["slope"][5:30, 5:25]
    assert (interior == 1.0).any() and (interior < 0.9).any()
    assert np.array_equal(got["slope"][5:30, 5:25].view(np.uint32), interior.view(np.uint32))


def test_infinite_and_huge_elevations(te, ctx, oracle):
    rows, cols = 128, 120
    g, og = _pair(te, oracle, rows, cols)
    z = synth.terrain(rows, cols, 0.02, 77, "mixed")
    z[20, 20] = np.inf
    z[50, 70] = -np.inf
    z[90, 30] = np.float32(3e30)      # finite but overflows the fp32 moments
    z[91, 31] = np.float32(-3e30)
    z[100:104, 100:104] = np.float32(1e-30)
    ref = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    for kernel in (te.KERNEL_FUSED, te.KERNEL_GENERIC):
        ctx.set_kernel(kernel)
        got = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z)
        assert_parity(got, ref)
    assert np.isnan(ref["slope"][20, 20]) and np.isfinite(ref["step"][20, 20])


@pytest.mark.parametrize("rows,cols", [(4, 4), (8, 3), (60, 64), (124, 17), (130, 50), (7, 9)])
def test_small_and_odd_sizes(te, ctx, oracle, rows, cols):
    g, og = _pair(te, oracle, rows, cols)
    z = synth.fbm(rows, cols, 0.02, rows * 100 + cols, 0.15)
    if rows * cols > 40:
        z[rows // 2, cols // 2] = np.nan
    ref = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    ctx.set_kernel(te.KERNEL_AUTO)   # rows % 4 != 0 silently uses the generic kernel
    got = ctx.chain_host(g, te.ChainParams.yaml_defaults(0), z)
    assert_parity(got, ref)


def test_other_radii_and_raw_moment_algorithm_use_the_generic_kernel(te, ctx, oracle):
    rows, cols = 96, 88
    g, og = _pair(te, oracle, rows, cols, 0.025)
    z = synth.terrain(rows, cols, 0.025, 5, "mixed")
    for alg, rn, r1, r2, rr in ((0, 0.08, 0.06, 0.03, 0.07), (1, 0.05, 0.04, 0.04, 0.05)):
        pt, po = te.ChainParams.yaml_defaults(alg), oracle.ChainParams.yaml_defaults(alg)
        for p in (pt, po):
            p.normals_radius, p.step_first_radius, p.step_second_radius, p.roughness_radius = rn, r1, r2, rr
            p.step_critical_cells = 3
            p.slope_critical = 0.7
        ref = oracle.chain(og, po, z, with_normals=True)
        ctx.set_kernel(te.KERNEL_AUTO)
        got = ctx.chain_host(g, pt, z, with_normals=True)
        reports = assert_parity(got, ref)
        assert all(r["bit_exact"] >= r["cells"] - 3 for r in reports), reports   # literal kernels replay the oracle
        with pytest.raises(te.TEError):
            ctx.set_kernel(te.KERNEL_FUSED)
            ctx.chain_host(g, pt, z)
    ctx.set_kernel(te.KERNEL_AUTO)


def test_standalone_filters_match_oracle(te, ctx, oracle):
    rows, cols = 100, 92
    g, og = _pair(te, oracle, rows, cols, 0.02, (12.5, -3.25))
    z = np.asfortranarray(synth.terrain(rows, cols, 0.02, 9, "mixed", (12.5, -3.25)))  # raw pointers: column-major like grid_map
    pt, po = te.ChainParams.yaml_defaults(0), oracle.ChainParams.yaml_defaults(0)
    nx, ny, nz = oracle.normals(og, po, z)
    new = lambda: np.empty((rows, cols), np.float32, order="F")  # noqa: E731
    a, b, c = new(), new(), new()
    ctx.normals(g, pt, z, a, b, c, te.MEM_HOST)
    for x, y in ((a, nx), (b, ny), (c, nz)):
        assert compare_layer(x, y)["bit_exact"] >= rows * cols - 2
    s = new(); ctx.slope(g, 1.0, nz, s, te.MEM_HOST)
    assert np.array_equal(np.isnan(s), np.isnan(nz))
    assert compare_layer(s, oracle.slope(og, 1.0, nz))["max_abs"] < 1e-7
    t = new(); ctx.step(g, pt, z, t, te.MEM_HOST)
    assert np.array_equal(t.view(np.uint32), oracle.step(og, po, z).view(np.uint32))
    r = new(); ctx.roughness(g, pt, z, nx, ny, nz, r, te.MEM_HOST)
    assert compare_layer(r, oracle.roughness(og, po, z, nx, ny, nz))["max_abs"] < 1e-7
    with pytest.raises(te.TEError) as e:   # missing layer -> TE_ERR_MISSING_LAYER
        ctx.roughness(g, pt, z, None, ny, nz, r, te.MEM_HOST)
    assert e.value.code == -2


def test_fused_against_literal_kernel_at_scale(te, ctx):
    """16.7 M cells: the fused stencil (fp32 + certification ladder) against the literal double-precision kernel, which is
    bit-exact against the oracle at every size the oracle can check.  No cell may leave the tolerance."""
    import torch
    import bench
    rows = cols = 4096
    z = bench.terrain_torch(torch, rows, 0, cols, cols, 11, 0.01, torch.device("cuda"))
    torch.cuda.synchronize()   # the context runs on its own stream: the input must be complete
    g = te.Geometry.make(rows, cols, 0.02)
    p = te.ChainParams.yaml_defaults(0)
    ctx.set_stream(None)
    res = {}
    for name, kernel in (("fused", te.KERNEL_FUSED), ("literal", te.KERNEL_GENERIC)):
        ctx.set_kernel(kernel)
        outs = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
        ctx.chain(g, p, z, *outs, te.MEM_DEVICE)
        ctx.synchronize()
        res[name] = outs
    ctx.set_kernel(te.KERNEL_AUTO)
    worst = {}
    for k, a, b in zip(("slope", "step", "roughness", "traversability"), res["fused"], res["literal"]):
        assert torch.equal(torch.isnan(a), torch.isnan(b)), k
        ok = ~torch.isnan(b)
        d = (a[ok].double() - b[ok].double()).abs()
        tol = 1e-5 * b[ok].double().abs() + 1e-6
        bad = int((d > tol).sum())
        worst[k] = (bad, float((d / tol).max()))
        assert bad == 0, (k, bad, float(d.max()))
    print(worst)


def test_streaming_slope_filter_is_bit_identical_to_the_literal_expression(te, ctx):
    """te_slope streams (certified polynomial acos, fp64 fallback on rounding boundaries): every float32 of the layer must equal
    float32(acos(double(nz)) < crit ? 1 - acos/crit : 0), the reference's expression (SlopeFilter.cpp:74-81), including exact 0/1,
    NaN, negative and out-of-range normals, and the neighbourhood of the branch point."""
    import torch
    n = 1 << 22
    gen = torch.Generator().manual_seed(5)
    nz = torch.rand(n, generator=gen, dtype=torch.float64)
    nz[: n // 4] = 1.0 - nz[: n // 4] ** 4 * 1e-3                 # near-flat normals, where acos is ill-conditioned
    nz = nz.to(torch.float32)
    nz[0:8] = torch.tensor([1.0, 0.0, -1.0, -0.25, float("nan"), 1.5, float("inf"), 0.5403023], dtype=torch.float32)  # cos(1.0) ~ branch point
    g = te.Geometry.make(2048, n // 2048, 0.02)
    for crit in (1.0, 0.7853981633974483, 0.3):
        ref = torch.acos(nz.double())
        ref = torch.where(ref < crit, 1.0 - ref / crit, torch.zeros_like(ref)).to(torch.float32)
        ref[~torch.isfinite(nz)] = float("nan")
        d_in, d_out = nz.cuda(), torch.empty(n, dtype=torch.float32, device="cuda")
        ctx.slope(g, crit, d_in, d_out, te.MEM_DEVICE)
        ctx.synchronize()
        got = d_out.cpu()
        # torch's acos on the CPU and CUDA's libdevice acos may differ in the last bits of the double: a cell may differ only
        # where the exact acos lies within their error of a decision of the expression
        ok, no = literal_cases.slope_mismatches(nz.numpy(), crit, got.numpy(), ref.numpy())
        assert not no, (crit, len(no), got[no[:5]], ref[no[:5]])
        print(f"crit {crit}: {len(ok)} cells explained by acos")


@pytest.mark.parametrize("rows,cols,sr,sc", [(192, 160, 37, 101), (128, 96, 0, 5), (128, 96, 127, 0), (2048, 2048, 1000, 77)])
def test_circular_buffer_start_index_through_the_host_path(te, ctx, rows, cols, sr, sc):
    """SURVEY §8(f)-1: te_chain(TE_MEM_HOST) takes the layers of a moving (robot-centric) grid_map as stored — cell (i, j) at buffer
    index ((i + start_row) % rows, (j + start_col) % cols) — and returns its layers in the same order; the copies to and from the
    device unwrap and re-wrap (2048^2 goes through the pipelined chunked path).  Must equal the unwrapped map's result bitwise."""
    z = synth.terrain(rows, cols, 0.02, 91, "mixed")
    g0 = te.Geometry.make(rows, cols, 0.02)
    p = te.ChainParams.yaml_defaults(0)
    ctx.set_kernel(te.KERNEL_AUTO)
    ctx.set_stream(None)
    ref = ctx.chain_host(g0, p, z, with_normals=True)
    gw = te.Geometry.make(rows, cols, 0.02)
    gw.start_row, gw.start_col = sr, sc
    stored = np.asfortranarray(np.roll(z, (sr, sc), axis=(0, 1)))        # stored[(i + sr) % rows, (j + sc) % cols] = z[i, j]
    got = ctx.chain_host(gw, p, stored, with_normals=True)
    for k, a in ref.items():
        b = np.roll(got[k], (-sr, -sc), axis=(0, 1))
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        assert np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)]), k
    import torch
    with pytest.raises(te.TEError) as err:                                # device memory has no circular-buffer form here
        zd = torch.zeros((cols, rows), dtype=torch.float32, device="cuda")
        outs = [torch.empty((cols, rows), dtype=torch.float32, device="cuda") for _ in range(4)]
        ctx.chain(gw, p, zd, *outs, te.MEM_DEVICE)
    assert err.value.code == -4
