"""The chain, the footprint sweeps and a batched te_map at the top of the index range their entries accept.

Every other parity test launches at most 2^26 cells.  The entries take far more — te_chain_batched's fused kernel below 2^30 cells
(TE_KERNEL_AUTO hands bigger launches to the generic kernel), te_footprint_batched below 2^32 cells — and they stay right only
because 32-bit cell arithmetic holds inside those limits: the fix-up work lists pack a cell index into bits 0-29 under two tier
flags, k_chain_fused runs an unsigned output offset across the maps of a launch, the predicate list and k_sweep_fast index the
batch's cells in unsigned.  A narrowing anywhere there corrupts only the last maps of a large batch.

Method: a batch is built on the device from a few distinct 512 x 512 tiles at 0.02 m (the YAML windows, fused shape A).  The bulk
of the batch repeats cheap terrain tiles; the hard tiles — window-mask probe maps with NaN and +-inf holes, an exactly planar
tilted map riddled with holes, random terrain — sit in the LAST maps, at the top of the index range.  Every cell of every map of
the batch must equal, bit for bit (NaN payloads included), its tile's result from a launch of that tile alone: it is the same
kernel on the same inputs.  Each tile's single launch is checked against the oracle by the rules the other suites use, which ties
the large launches back to the reference.  Each case asserts that it reaches the boundary it claims to reach.

The cases need up to about 61 GB of device memory (the prefix-sum footprint sweep).  Each checks what its shapes need against the free memory before it allocates and
skips, naming the shortfall, when the GPU does not have it; each runs on a fresh context that it closes, so the context's scratch
(work lists, prefix sums) does not pile up from case to case."""
import contextlib
import gc
import time

import numpy as np
import pytest

import literal_cases as lc
import synth
import window_masks as wm
from helpers import assert_parity, chain_params, close_sweep, compare_layer, same_bits_or_nan, same_values, te_footprint_params, walled_terrain

pytestmark = pytest.mark.gpu

ROWS = COLS = 512
CELLS = ROWS * COLS                      # 2^18 cells per map
MB = CELLS * 4                           # bytes of one float32 layer of one map
GB = 1 << 30
RES = wm.SHAPES["A"][0]
LAYERS = ("slope", "step", "roughness", "traversability")
SENTINEL = 0x7FC0BEEF                    # a NaN payload no kernel writes
POLY = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]   # robot_footprint_parameter.yaml:3
YAW = 0.7854
MARGIN = 2 * GB                          # CUDA context, cuBLAS-free torch workspace, comparison temporaries


def _pad(z):
    """A probe map cut or padded with NaN to the tile shape, column-major."""
    out = np.full((ROWS, COLS), np.nan, np.float32)
    r, c = min(ROWS, z.shape[0]), min(COLS, z.shape[1])
    out[:r, :c] = z[:r, :c]
    return np.asfortranarray(out)


def _planar_holes(seed):
    """An exactly planar tilted map (dyadic slopes: every z exact) with 5 % NaN holes: every valid cell is rank-deficient for the
    reference's QR test, so the fused kernel sends it down the fix-up tiers."""
    i, j = np.meshgrid(np.arange(ROWS), np.arange(COLS), indexing="ij")
    z = (0.125 * i + 0.0625 * j).astype(np.float32) * np.float32(RES)
    z[np.random.default_rng(seed).random((ROWS, COLS)) < 0.05] = np.nan
    return np.asfortranarray(z)


def _chain_tiles():
    """(names, tiles, number of easy tiles): the easy tiles fill the bulk of a batch, the hard ones its last maps."""
    masks = wm.sample_masks("A", 102 * 102, 7)                 # 510 x 510 probe maps
    easy = [("terrain-%d" % s, np.asfortranarray(synth.terrain(ROWS, COLS, RES, s, "mixed"))) for s in (1, 2, 3)]
    hard = [("probe-inf", _pad(wm.probe("A", masks, "inf", 7))), ("probe-planar", _pad(wm.probe("A", masks, "planar", 8))),
            ("probe-nearflat", _pad(wm.probe("A", masks, "nearflat", 9))), ("planar-holes", _planar_holes(10)),
            ("terrain-rough", np.asfortranarray(synth.terrain(ROWS, COLS, RES, 11, "rough", holes=0.05)))]
    names, tiles = zip(*(easy + hard))
    return list(names), list(tiles), len(easy)


def _layout(n, n_tiles, n_easy):
    """Tile of each map of an n-map batch: the easy tiles in turn, then every hard tile once in the last maps."""
    n_hard = n_tiles - n_easy
    idx = np.arange(n) % n_easy
    idx[n - n_hard:] = np.arange(n_easy, n_tiles)
    return idx


@contextlib.contextmanager
def _case(te, name, need):
    """A fresh context for one case, after checking that `need` bytes are free; prints the case's wall time and peak memory."""
    import torch
    gc.collect()   # an earlier case's tensors may sit in a reference cycle (an exception's traceback holds its frame)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < need + MARGIN:
        pytest.skip(f"{name}: needs {(need + MARGIN) / GB:.1f} GB free, the GPU has {free / GB:.1f} GB of {total / GB:.1f} GB: "
                    f"{(need + MARGIN - free) / GB:.1f} GB short")
    torch.cuda.reset_peak_memory_stats()
    ctx = te.Context(0)
    ctx.set_stream(None)
    stats = {"peak_other": 0}
    t = time.time()

    def sample():   # device memory held outside torch's allocator (the library's scratch), at its largest so far
        torch.cuda.synchronize()
        f, tot = torch.cuda.mem_get_info()
        stats["peak_other"] = max(stats["peak_other"], tot - f - torch.cuda.memory_reserved())

    try:
        yield ctx, sample
    finally:
        ctx.close()
        torch.cuda.synchronize()
        wall = time.time() - t
        gc.collect()
        print(f"\n{name}: {wall:.1f} s; peak torch allocation {torch.cuda.max_memory_allocated() / GB:.2f} GB, library and CUDA "
              f"context outside torch {stats['peak_other'] / GB:.2f} GB; budget {need / GB:.1f} GB")
        torch.cuda.empty_cache()


def _assert_maps_equal(out, single, idx, what, chunk=512):
    """Every map m of out (L, n, cols, rows) equals single[:, idx[m]] bit for bit, every cell, NaN payloads included."""
    import torch
    n = out.shape[1]
    didx = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    for k in range(out.shape[0]):
        ref_k = single[k].view(torch.int32)
        bad = torch.cat([(out[k, a:min(n, a + chunk)].view(torch.int32) != ref_k[didx[a:min(n, a + chunk)]]).flatten(1).sum(1)
                         for a in range(0, n, chunk)])
        if bool(bad.any()):
            maps = torch.nonzero(bad).flatten().tolist()
            shown = maps[:4] + maps[-4:] if len(maps) > 8 else maps
            pytest.fail(f"{what}: layer {k}: {len(maps)} maps differ from their tile's single launch, the first and last of them "
                        f"{shown} ({[int(bad[m]) for m in shown]} cells)")


def _device(tiles):
    """(T, cols, rows) device tensor of column-major tiles."""
    import torch
    return torch.from_numpy(np.stack([np.ascontiguousarray(t.T) for t in tiles])).cuda()


def _single_chain(te, ctx, g, p, tiles_d):
    """Each tile's chain in a launch of its own: (4, T, cols, rows)."""
    import torch
    out = torch.empty((4, tiles_d.shape[0], COLS, ROWS), dtype=torch.float32, device="cuda")
    for t in range(tiles_d.shape[0]):
        ctx.chain_batched(g, p, 1, tiles_d[t], *(out[k, t] for k in range(4)), te.MEM_DEVICE)
    ctx.synchronize()
    return out


def _host(single, t):
    return {k: np.asfortranarray(single[i, t].cpu().numpy().T) for i, k in enumerate(LAYERS)}


def _fused_parity(got, ref):
    """The fused rule of test_window_masks_gpu: assert_parity on slope, step and roughness; the traversability within tolerance
    everywhere and bit for bit where each of its three terms is a branch value (0 or 1) in both."""
    assert_parity(got, ref, keys=("slope", "step", "roughness"))
    tr = compare_layer(got["traversability"], ref["traversability"], "traversability")
    assert tr["nan_mismatch"] == 0 and tr["out_of_tol"] == 0, tr
    exact = np.ones(ref["traversability"].shape, bool)
    for k in ("slope", "step", "roughness"):
        exact &= ((ref[k] == 0.0) | (ref[k] == 1.0)) & (got[k] == ref[k])
    a, b = got["traversability"][exact], ref["traversability"][exact]
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), int((a != b).sum())


def _literal_parity(got, ref, crit, w):
    """The literal rule of test_literal_params_gpu: step and roughness bit for bit (NaN matches NaN), the slope except where the
    double acos lies within its error of a decision, the traversability as float32 w * ((s + t) + r) of the kernel's own layers."""
    for k in ("step", "roughness"):
        assert same_bits_or_nan(got[k], ref[k]), (k, int((got[k] != ref[k]).sum()))
    _, no = lc.slope_mismatches(ref["nz"], crit, got["slope"], ref["slope"])
    assert not no, len(no)
    s, t, r = (np.asarray(got[k], np.float32) for k in ("slope", "step", "roughness"))
    assert same_bits_or_nan(got["traversability"], np.float32(w) * ((s + t) + r))
    assert np.array_equal(np.isnan(got["traversability"]), np.isnan(ref["traversability"]))


@pytest.fixture(scope="module")
def chain_tiles(oracle):
    """(names, tiles, easy tile count, the oracle's chain of each tile with normals)."""
    names, tiles, n_easy = _chain_tiles()
    og = oracle.Geometry.make(ROWS, COLS, RES)
    refs = [oracle.chain(og, chain_params(oracle, **wm.chain_kwargs("A")), z, with_normals=True) for z in tiles]
    return names, tiles, n_easy, refs


def _big_batch(tiles_d, idx, sentinel=False):
    """The elevation of the batch whose map m is tile idx[m], built on the device, and room for its four chain layers:
    (elevation (n, cols, rows), outputs (4, n, cols, rows)); sentinel: the outputs filled with the SENTINEL bit pattern."""
    import torch
    z = torch.index_select(tiles_d, 0, torch.from_numpy(idx).cuda())
    out = torch.empty((4, len(idx), COLS, ROWS), dtype=torch.float32, device="cuda")
    if sentinel:
        out.view(torch.int32).fill_(SENTINEL)
    torch.cuda.synchronize()
    return z, out


def _chain_budget(n, fused):
    """Bytes of an n-map chain: input and four outputs, the fused kernel's two work lists (every cell plus chunk padding)."""
    return n * MB * (5 + (2.1 if fused else 0)) + 3 * 8 * MB * 4


def test_fused_chain_at_its_largest_launch(te, chain_tiles):
    """4095 maps: 2^30 - 2^18 cells, the largest launch k_chain_fused takes.  Tier-2 and tier-3 list entries reach cell indices
    >= 2^29 from the hard tiles in the top maps, and every map equals its tile's single launch."""
    _, tiles, n_easy, refs = chain_tiles
    n = (1 << 30) // CELLS - 1
    idx = _layout(n, len(tiles), n_easy)
    g, p = te.Geometry.make(ROWS, COLS, RES), chain_params(te, **wm.chain_kwargs("A"))
    with _case(te, "fused chain, 4095 maps", _chain_budget(n, True)) as (ctx, sample):
        ctx.set_kernel(te.KERNEL_FUSED)
        tiles_d = _device(tiles)
        z, out = _big_batch(tiles_d, idx)
        ctx.chain_batched(g, p, n, z, *(out[k] for k in range(4)), te.MEM_DEVICE)
        ctx.synchronize()
        sample()
        cnt = ctx.flag_counters()
        lists = {tier: ctx.fixup_cells(tier) & np.uint32(0x3FFFFFFF) for tier in (2, 3)}
        del z
        single = _single_chain(te, ctx, g, p, tiles_d)
        _assert_maps_equal(out, single, idx, "fused, 4095 maps")
        assert cnt[2] == 0, cnt
        top = (n - (len(tiles) - n_easy)) * CELLS            # first cell of the hard tiles
        for tier, cells in lists.items():
            high = int((cells >= (1 << 29)).sum())
            largest = int(cells.max()) if len(cells) else -1
            print(f"tier {tier}: {len(cells)} entries, {high} at cell index >= 2^29, largest {largest} (2^30 = {1 << 30}); "
                  f"{int((cells >= top).sum())} in the hard tiles from cell {top}")
            assert high > 0 and largest >= top, (tier, len(cells), high, largest)
        for t in range(len(tiles)):
            _fused_parity(_host(single, t), refs[t])
        del out, single, tiles_d


def test_fused_refuses_2_30_cells_and_auto_hands_them_to_the_generic_kernel(te, chain_tiles):
    """4096 maps: exactly 2^30 cells.  KERNEL_FUSED is TE_ERR_UNSUPPORTED and writes nothing; KERNEL_AUTO runs the generic kernel,
    and every map equals the generic kernel's launch of its tile alone."""
    import torch
    _, tiles, n_easy, refs = chain_tiles
    n = (1 << 30) // CELLS
    idx = _layout(n, len(tiles), n_easy)
    g, p = te.Geometry.make(ROWS, COLS, RES), chain_params(te, **wm.chain_kwargs("A"))
    with _case(te, "fused refusal and generic hand-over, 4096 maps", _chain_budget(n, False)) as (ctx, sample):
        tiles_d = _device(tiles)
        z, out = _big_batch(tiles_d, idx, sentinel=True)
        ctx.set_kernel(te.KERNEL_FUSED)
        with pytest.raises(te.TEError) as e:
            ctx.chain_batched(g, p, n, z, *(out[k] for k in range(4)), te.MEM_DEVICE)
        assert e.value.code == -4, e.value
        ctx.synchronize()
        assert bool((out.view(torch.int32) == SENTINEL).all()), "the refused launch wrote to its outputs"
        ctx.set_kernel(te.KERNEL_AUTO)
        before, _ = ctx.stats()
        ctx.chain_batched(g, p, n, z, *(out[k] for k in range(4)), te.MEM_DEVICE)
        ctx.synchronize()
        sample()
        launches = ctx.stats()[0] - before
        print(f"KERNEL_AUTO on {n * CELLS} cells: {launches} launches (the generic kernel runs map by map)")
        assert n * CELLS == 1 << 30 and launches >= n, launches
        del z
        ctx.set_kernel(te.KERNEL_GENERIC)
        single = _single_chain(te, ctx, g, p, tiles_d)
        _assert_maps_equal(out, single, idx, "generic, 4096 maps")
        pr = chain_params(te, **wm.chain_kwargs("A"))
        for t in range(len(tiles)):
            _literal_parity(_host(single, t), refs[t], pr.slope_critical, pr.fuse_weight)
        del out, single, tiles_d


def test_generic_chain_past_2_31_cells(te, chain_tiles):
    """8193 maps: 2^31 + 2^18 cells, past the signed 32-bit cell index, on the generic kernel (four outputs, no normals)."""
    _, tiles, n_easy, _ = chain_tiles
    n = (1 << 31) // CELLS + 1
    idx = _layout(n, len(tiles), n_easy)
    g, p = te.Geometry.make(ROWS, COLS, RES), chain_params(te, **wm.chain_kwargs("A"))
    with _case(te, "generic chain, 8193 maps", _chain_budget(n, False)) as (ctx, sample):
        ctx.set_kernel(te.KERNEL_AUTO)
        tiles_d = _device(tiles)
        z, out = _big_batch(tiles_d, idx)
        t0 = time.time()
        ctx.chain_batched(g, p, n, z, *(out[k] for k in range(4)), te.MEM_DEVICE)
        ctx.synchronize()
        print(f"generic chain on {n * CELLS} cells: {time.time() - t0:.1f} s")
        sample()
        assert (n - 1) * CELLS >= 1 << 31   # the last map lies past 2^31 cells
        del z
        ctx.set_kernel(te.KERNEL_GENERIC)
        single = _single_chain(te, ctx, g, p, tiles_d)
        _assert_maps_equal(out, single, idx, "generic, 8193 maps")
        del out, single, tiles_d


def test_fused_normals_past_2_31_bytes_per_layer(te, chain_tiles):
    """te_chain with the nx / ny / nz outputs on one map of 512 rows x 2049 tiles of columns: 2^29 + 2^18 cells, so every layer
    passes 2^31 bytes and the work-list entries of the last tiles hold cell indices >= 2^29.  The whole map must equal column slabs
    of it launched on their own (slabs of 64 tiles with 4-column halos, the chain's reach at these windows)."""
    import torch
    _, tiles, n_easy, _ = chain_tiles
    n = (1 << 29) // CELLS + 1
    idx = _layout(n, len(tiles), n_easy)
    cols = n * COLS
    g, p = te.Geometry.make(ROWS, cols, RES), chain_params(te, **wm.chain_kwargs("A"))
    need = n * MB * (8 + 2.1) + 2 * 64 * MB * 8
    with _case(te, "fused chain with normals, 2049 tiles", need) as (ctx, sample):
        ctx.set_kernel(te.KERNEL_FUSED)
        tiles_d = _device(tiles)
        z = torch.index_select(tiles_d, 0, torch.from_numpy(idx).cuda()).reshape(cols, ROWS)
        out = torch.empty((7, cols, ROWS), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        ctx.chain(g, p, z, *(out[k] for k in range(4)), te.MEM_DEVICE, nx=out[4], ny=out[5], nz=out[6])
        ctx.synchronize()
        sample()
        top = (n - (len(tiles) - n_easy)) * CELLS
        for tier in (2, 3):
            cells = ctx.fixup_cells(tier) & np.uint32(0x3FFFFFFF)
            largest = int(cells.max()) if len(cells) else -1
            print(f"tier {tier}: {len(cells)} entries, {int((cells >= (1 << 29)).sum())} at cell index >= 2^29, largest "
                  f"{largest}; layer bytes {cols * ROWS * 4} (2^31 = {1 << 31})")
            assert largest >= max(top, 1 << 29), (tier, len(cells), largest)
        assert cols * ROWS * 4 > 1 << 31
        w = 64 * COLS
        for b in range(0, cols, w):
            e = min(cols, b + w)
            hl, hr = min(4, b), min(4, cols - e)
            part = torch.empty((7, e - b, ROWS), dtype=torch.float32, device="cuda")
            ctx.chain(g, p, z[b - hl:e + hr].contiguous(), *(part[k] for k in range(4)), te.MEM_DEVICE,
                      slab=te.Slab(b, e - b, hl, hr), nx=part[4], ny=part[5], nz=part[6])
            ctx.synchronize()
            bad = (out[:, b:e].view(torch.int32) != part.view(torch.int32)).flatten(1).sum(1)
            assert not bool(bad.any()), (b, bad.tolist())
        del z, out, part, tiles_d


def _footprint_tiles(oracle):
    """(tiles of (traversability, slope = step, elevation), easy tile count).  The layers are the oracle chain's on walled_terrain
    maps.  The easy tile is the flat map, on which no filter check runs; the hard ones are walled or terrain maps with zero patches
    in their step layer (blocked cells, the predicate list's entries) and NaN and +-inf traversability cells."""
    rng = np.random.default_rng(21)
    og = oracle.Geometry.make(ROWS, COLS, RES)
    out = []
    for kind in range(4):
        z = walled_terrain(ROWS, COLS, RES, kind, 21 + kind)
        ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
        t, s = np.array(ch["traversability"], np.float32), np.array(ch["step"], np.float32)
        if kind:
            t[rng.random((ROWS, COLS)) < 0.03] = np.nan
            t[rng.random((ROWS, COLS)) < 0.005] = np.inf
            t[rng.random((ROWS, COLS)) < 0.005] = -np.inf
            for a, b in rng.integers(0, ROWS - 10, (6, 2)):
                s[a:a + 9, b:b + 9] = 0.0
        out.append(tuple(np.asfortranarray(x) for x in (t, s, z)))
    return out, 1


@pytest.fixture(scope="module")
def footprint_tiles(oracle):
    return _footprint_tiles(oracle)


@pytest.mark.parametrize("sweep", ["prefix", "brute", "polygon"])
def test_footprint_sweeps_past_2_31_cells(te, oracle, footprint_tiles, sweep, monkeypatch):
    """te_footprint_batched (prefix-sum and visit-by-visit sweeps) and te_footprint_polygon_batched on 8193 maps, 2^31 + 2^18 input
    cells: their cell arithmetic is unsigned up to 2^32.  slope and step are one shared read-only tensor (the single-map launches
    and the oracle read the same aliasing).  The maps past 2^31 cells hold blocked, open and non-finite cells."""
    import torch
    tiles, n_easy = footprint_tiles
    n = (1 << 31) // CELLS + 1
    idx = _layout(n, len(tiles), n_easy)
    g = te.Geometry.make(ROWS, COLS, RES)
    p = te_footprint_params(te)
    nout = 2 if sweep == "polygon" else 1
    # inputs (3 layers), outputs, predicate bytes and list; the prefix sums ((rows + 1) doubles, bit words and a byte per cell)
    need = n * MB * (3 + nout + 0.25 + 1) + (n * (ROWS + 1) * COLS * 8 + n * MB // 4 if sweep == "prefix" else 0)
    if sweep == "brute":
        monkeypatch.setenv("TE_FOOTPRINT_BRUTE", "1")
    with _case(te, f"footprint {sweep}, 8193 maps", need) as (ctx, sample):
        lay_d = [_device([tile[k] for tile in tiles]) for k in range(3)]   # traversability, slope = step, elevation
        didx = torch.from_numpy(idx).cuda()
        big = [torch.index_select(x, 0, didx) for x in lay_d]
        out = torch.empty((nout, n, COLS, ROWS), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

        def run(k, lay, o):
            trav, s, elev = lay
            if sweep == "polygon":
                ctx.footprint_polygon_batched(g, p, k, POLY, YAW, trav, s, s, elev, o[0], o[1], te.MEM_DEVICE)
            else:
                ctx.footprint_batched(g, p, k, trav, s, s, elev, o[0], te.MEM_DEVICE)

        before = ctx.stats()[0]
        run(n, big, out)
        ctx.synchronize()
        sample()
        # the prefix-sum sweep is five launches (predicates 2, prefix sums, nearest blocked cells, k_sweep_fast), the visit-by-visit
        # and the polygonal sweeps three: a prefix case that fell back to k_sweep would test the brute sweep twice
        launches = ctx.stats()[0] - before
        print(f"{sweep}: {launches} launches")
        assert launches == (5 if sweep == "prefix" else 3), launches
        first = (1 << 31) // CELLS
        inf_cells = int(torch.isinf(big[0][first:]).sum())
        del big
        single = torch.empty((nout, len(tiles), COLS, ROWS), dtype=torch.float32, device="cuda")
        for t in range(len(tiles)):
            run(1, [x[t] for x in lay_d], [single[k, t] for k in range(nout)])
        ctx.synchronize()
        last = out[:, first:]
        blocked, open_ = int((last == 0).sum()), int((last > 0).sum())
        print(f"{sweep}: maps {first}..{n - 1} start at cell >= 2^31; {blocked} blocked, {open_} open and {inf_cells} infinite "
              f"traversability cells there")
        assert first * CELLS >= 1 << 31 and blocked > 0 and open_ > 0 and inf_cells > 0
        _assert_maps_equal(out, single, idx, f"footprint {sweep}, 8193 maps")
        og = oracle.Geometry.make(ROWS, COLS, RES)
        fo = oracle.FootprintParams.yaml_defaults()
        for t in range(len(tiles)):
            tr, s, e = tiles[t]
            got = [single[k, t].cpu().numpy().T for k in range(nout)]
            if sweep == "polygon":
                rx, rrot = oracle.footprint_polygon(og, fo, POLY, YAW, tr, s, s, e)
                assert close_sweep(got[0], rx) and close_sweep(got[1], rrot), t
            else:
                ref = oracle.footprint(og, fo, tr, s, s, e)[0]
                assert (same_values if sweep == "brute" else close_sweep)(got[0], ref), t
        del out, single, lay_d


def _same(a, b):
    """Equal shapes and equal bytes, NaN payloads included, of two host arrays (or device tensors) of any dtype."""
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    b = b.cpu().numpy() if hasattr(b, "cpu") else np.asarray(b)
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


MAP_NAMES = ["traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation"]
# Layers a te_map of these calls holds: te_map_chain's five chain layers and the footprint cache (map_reset reserves those
# six), traversability_x / traversability_rot (footprint_polygon_keep), slope / step / roughness_footprint (the sweep's memo).
MAP_HELD = 6 + 2 + 3


def _map_layers(te, ctx, m, n):
    """MAP_NAMES of the n maps of te_map m, read into device memory: (5, n, cols, rows)."""
    import torch
    out = torch.empty((len(MAP_NAMES), n, COLS, ROWS), dtype=torch.float32, device="cuda")
    m.get_layers(MAP_NAMES, out=out, memory=te.MEM_DEVICE)
    ctx.synchronize()
    return out


def test_map_batch_past_2_31_bytes_per_layer(te, chain_tiles):
    """A te_map holding 2049 maps, 2^29 + 2^18 cells: every layer passes 2^31 bytes and the last map starts at cell 2^29.  Every
    te_map entry that offsets the batch's layers, memo or cache per map runs on the last maps (map 2048 always among them) and
    must equal, bit for bit, a single-map te_map holding that map's tile: the chain from device memory and the layers read back,
    submaps, valid_at, at_poses, occupancy grids, point clouds, the circular sweep and its cache, the polygonal sweep kept on the
    map, footprint path requests on the cache (twice: the second request answers from what the first stored), and the re-chaining
    of the last map from an elevation map, a mono16 image and a window of a source map of more than 2^29 cells, each of which
    must leave every bit of every other map as it was."""
    import torch
    from helpers import footprint_arrays, mixed_request, request_footprints, subset
    _, tiles, n_easy, _ = chain_tiles
    n = (1 << 29) // CELLS + 1
    idx = _layout(n, len(tiles), n_easy)
    last = list(range(n - (len(tiles) - n_easy), n))          # the hard tiles; the last map starts at cell 2^29
    assert last[-1] == n - 1 and (n - 1) * CELLS == 1 << 29
    g, p = te.Geometry.make(ROWS, COLS, RES), chain_params(te, **wm.chain_kwargs("A"))
    fp = te_footprint_params(te)
    # the map's layers, its chain work lists, the footprint sweep's prefix sums (2 layers), predicate bytes, list and values (2.5)
    # and its memo and codes (0.5); the input, which is also the source map of the windows; two reads of five layers, the cache
    need = n * MB * (MAP_HELD + 2.1 + 5 + 1 + 2 * len(MAP_NAMES) + 1)
    with _case(te, "te_map, 2049 maps", need) as (ctx, sample):
        ctx.set_kernel(te.KERNEL_AUTO)
        tiles_d = _device(tiles)
        singles = []
        for z in tiles:
            one = te.Map(ctx)
            one.chain(g, p, z)
            singles.append(one)
        single = torch.stack([_map_layers(te, ctx, one, 1)[:, 0] for one in singles], 1)
        m = te.Map(ctx)
        try:
            z = torch.index_select(tiles_d, 0, torch.from_numpy(idx).cuda())
            m.chain_batched(g, p, n, z, memory=te.MEM_DEVICE)
            out = _map_layers(te, ctx, m, n)
            sample()
            _assert_maps_equal(out, single, idx, "te_map_chain_batched + te_map_get_layers, 2049 maps")
            del out
            one_of = {k: singles[idx[k]] for k in last}
            rng = np.random.default_rng(3)
            half = 0.5 * ROWS * RES

            # ---- readers of the chain layers ------------------------------------------------------------------------------------
            pos = rng.uniform(-half, half, (len(last), 2))
            length = rng.uniform(0.5, 2 * half, (len(last), 2))
            got = m.get_submaps_batched(np.asarray(last, np.int32), pos, length, MAP_NAMES)
            for k, (info, lay) in zip(last, got):
                ref_info, ref = one_of[k].get_submaps(pos[[last.index(k)]], length[[last.index(k)]], MAP_NAMES)[0]
                assert info["success"] and ref_info["success"], k
                assert (info["rows"], info["cols"]) == (ref_info["rows"], ref_info["cols"]), k
                assert all(_same(lay[x], ref[x]) for x in MAP_NAMES), ("submap", k)

            xy = rng.uniform(-1.1 * half, 1.1 * half, (len(last) * 200, 2))
            pos_map = np.repeat(np.asarray(last, np.int32), 200)
            valid = m.valid_at_batched(pos_map, xy)
            for j, k in enumerate(last):
                ref = one_of[k].valid_at(xy[j * 200:(j + 1) * 200])
                assert _same(valid[j * 200:(j + 1) * 200], ref), ("valid_at", k)
                assert 0 < int(ref.sum()) < 200, k

            poses = np.zeros((len(last) * 8, 7))
            poses[:, :2] = rng.uniform(-half, half, (len(poses), 2))
            yaw = rng.uniform(-np.pi, np.pi, len(poses))
            poses[:, 5], poses[:, 6] = np.sin(yaw / 2), np.cos(yaw / 2)
            points = rng.uniform(-1.0, 1.0, (64, 3)).astype(np.float32)
            pose_map = np.repeat(np.asarray(last, np.int32), 8)
            lay, ok = m.at_poses(poses, points, MAP_NAMES, pose_map=pose_map)
            for j, k in enumerate(last):
                rl, rok = one_of[k].at_poses(poses[j * 8:(j + 1) * 8], points, MAP_NAMES)
                assert _same(ok[j * 8:(j + 1) * 8], rok), ("at_poses valid", k)
                assert all(_same(lay[x][j * 8:(j + 1) * 8], rl[x]) for x in MAP_NAMES), ("at_poses", k)

            occ = m.get_occupancy(MAP_NAMES, 0.0, 1.0, maps=last)
            for j, k in enumerate(last):
                ref = one_of[k].get_occupancy(MAP_NAMES, 0.0, 1.0)
                assert all(_same(occ[x][j], ref[x]) for x in MAP_NAMES), ("occupancy", k)

            fields = ["traversability", "elevation", "traversability_slope", "traversability_step"]
            _, _, clouds = m.get_point_cloud(fields, maps=last)
            for j, k in enumerate(last):
                _, _, ref = one_of[k].get_point_cloud(fields)
                assert len(ref[0]) > 0 and _same(clouds[j], ref[0]), ("point cloud", k)
            print(f"te_map readers: maps {last[0]}..{last[-1]}, the last from cell {(n - 1) * CELLS} (2^29 = {1 << 29})")

            # ---- the circular sweep and its cache, path requests on it, the polygonal sweep kept on the map ---------------------
            cache = torch.empty((n, COLS, ROWS), dtype=torch.float32, device="cuda")
            m.footprint(fp, out=cache, memory=te.MEM_DEVICE)
            ctx.synchronize()
            sample()
            for k in last:
                ref = one_of[k].footprint(fp)
                assert _same(cache[k].cpu().numpy().T, ref), ("footprint", k)
            del cache
            fps = request_footprints(rng)
            R = mixed_request(rng, g, 60, fps, cap_path=False)
            R["map"] = np.asarray(last, np.int32)[rng.integers(0, len(last), len(R["kind"]))]
            for rnd in range(2):   # the second request answers circular paths from what the first stored in the caches
                fb, fx = footprint_arrays(R, fps)
                got = m.check_footprint_request_batched(fp, R["map"], R["begin"], R["poses"], R["radius"], fb, fx,
                                                         conservative=R["cons"])
                for k in last:
                    q = np.nonzero(R["map"] == k)[0]
                    S = subset(R, q)
                    sfb, sfx = footprint_arrays(S, fps)
                    ref = one_of[k].check_footprint_request(fp, S["begin"], S["poses"], S["radius"], sfb, sfx, conservative=S["cons"])
                    for a, b in zip(got, ref):
                        assert _same(a[q], b), ("request", rnd, k)
                R = subset(R, rng.permutation(len(R["kind"])))
            cache = torch.empty((n, COLS, ROWS), dtype=torch.float32, device="cuda")
            m.get_layers(["traversability_footprint"], out=cache, memory=te.MEM_DEVICE)
            ctx.synchronize()
            for k in last:
                assert _same(cache[k].cpu().numpy().T, one_of[k].get_footprint()), ("cache after the requests", k)
            del cache
            gx, grot = m.footprint_polygon_keep(fp, POLY, [YAW] * len(last), map_index=last, outputs=True)
            for j, k in enumerate(last):
                rx, rrot = one_of[k].footprint_polygon_keep(fp, POLY, [YAW], outputs=True)
                assert _same(gx[j], rx) and _same(grot[j], rrot), ("polygon keep", k)
            print(f"te_map sweeps and requests: maps {last[0]}..{last[-1]}")

            # ---- re-chaining the last map: an elevation map, a mono16 image, a window of a source map past 2^29 cells -----------
            def rechained(one, what):
                """The last map now holds what te_map `one` holds; every other map keeps its bits."""
                nonlocal single, idx
                single = torch.cat([single, _map_layers(te, ctx, one, 1)], 1)
                idx = idx.copy()
                idx[-1] = single.shape[1] - 1
                _assert_maps_equal(_map_layers(te, ctx, m, n), single, idx, what)

            m.chain_maps(g, p, [n - 1], tiles[0][None])
            rechained(singles[0], "te_map_chain_maps on the last of 2049 maps")
            image = (np.nan_to_num(tiles[3], nan=0.0, posinf=0.0, neginf=0.0) * 4000 + 30000).clip(0, 65535).astype(np.uint16)
            m.chain_image_maps(g, p, [n - 1], image[None], -1.0, 2.0)
            img = te.Map(ctx)
            img.chain_image(g, p, image, -1.0, 2.0)
            singles.append(img)
            rechained(img, "te_map_chain_image_maps (mono16) on the last of 2049 maps")
            src_g = te.Geometry.make(ROWS, n * COLS, RES)            # the batch's elevation as one wide map: 2^29 + 2^18 cells
            src = {"elevation": z.reshape(-1)}
            far = (0.0, 0.5 * src_g.length_y - RES * (n * COLS - COLS // 2))   # centre of the last tile: the far corner
            j0 = int(round((0.5 * src_g.length_y - far[1]) / RES))
            assert j0 * ROWS >= 1 << 29 and n * COLS * ROWS > 1 << 29
            m.chain_windows(g, src_g, src, [far], p, map_index=[n - 1], memory=te.MEM_DEVICE)
            win = te.Map(ctx)
            win.chain_windows(g, src_g, src, [far], p, memory=te.MEM_DEVICE)
            singles.append(win)
            rechained(win, "te_map_chain_windows on the last of 2049 maps")
            print(f"te_map re-chained map {n - 1}; window of the source map at column {j0} (cell {j0 * ROWS}, 2^29 = {1 << 29})")
            del z
        finally:
            m.close()
            for one in singles:
                one.close()
        del single, tiles_d
