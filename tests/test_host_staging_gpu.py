"""Host staging of the TE_MEM_HOST entries on circular-buffer (start-index) maps, and the start-index rejections of the entries
that do not honour one."""
import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

ROWS, COLS, SR, SC = 144, 120, 55, 97


def _unroll(a):
    return np.roll(a, (-SR, -SC), axis=(0, 1))


def _wrapped_geometry(te):
    g = te.Geometry.make(ROWS, COLS, 0.02)
    g.start_row, g.start_col = SR, SC
    return g


def test_footprint_with_roughness_on_circular_buffer_map(te, ctx, oracle):
    """te_footprint2 with verify_roughness (five input and four output layers staged) on a start-index map: every output equals the
    unwrapped map's bitwise."""
    z = synth.terrain(ROWS, COLS, 0.02, 53, "mixed")
    og = oracle.Geometry.make(ROWS, COLS, 0.02)
    ch = oracle.chain(og, oracle.ChainParams.yaml_defaults(0), z)
    rough = ch["roughness"].copy()
    rng = np.random.default_rng(53)
    for _ in range(40):   # zero-roughness patches, so that the roughness predicate blocks cells the others let through
        a, b = int(rng.integers(0, ROWS - 10)), int(rng.integers(0, COLS - 10))
        rough[a:a + int(rng.integers(1, 10)), b:b + int(rng.integers(1, 10))] = 0.0
    lay = [np.asfortranarray(x, dtype=np.float32) for x in (ch["traversability"], ch["slope"], ch["step"], rough, z)]
    wl = [np.asfortranarray(np.roll(x, (SR, SC), axis=(0, 1))) for x in lay]
    fp = te.FootprintParams.yaml_defaults()
    fp.verify_roughness = 1
    g0 = te.Geometry.make(ROWS, COLS, 0.02)
    ctx.set_stream(None)
    ref = [np.empty_like(lay[0]) for _ in range(4)]
    got = [np.empty_like(lay[0]) for _ in range(4)]
    for g, (t, s, st, r, e), (out, sfp, tfp, rfp) in ((g0, lay, ref), (_wrapped_geometry(te), wl, got)):
        ctx.footprint(g, fp, t, s, st, e, out, te.MEM_HOST, slope_fp=sfp, step_fp=tfp, roughness=r, roughness_fp=rfp)
    for name, a, b in zip(("traversability_footprint", "slope_footprint", "step_footprint", "roughness_footprint"), ref, got):
        assert np.array_equal(a, _unroll(b), equal_nan=True), name
    assert (ref[0] == 0).any() and (ref[0] > 0).any() and (ref[3] == 0).any()


def test_start_index_rejections(te, ctx):
    """A start index where an entry cannot honour it is TE_ERR_UNSUPPORTED (-4): the footprint sweeps with a slab or in device
    memory, and the single-filter entries always."""
    g = _wrapped_geometry(te)
    p = te.ChainParams.yaml_defaults(0)
    fp = te.FootprintParams.yaml_defaults()
    fp.verify_roughness = 1
    poly = [[0.45, 0.30], [0.45, -0.30], [-0.45, -0.30], [-0.45, 0.30]]
    lay = [np.zeros((ROWS, COLS), np.float32, order="F") for _ in range(5)]
    o1, o2, o3, o4 = (np.empty((ROWS, COLS), np.float32, order="F") for _ in range(4))
    slab = te.Slab(0, COLS // 2, 0, COLS - COLS // 2)
    calls = {
        "te_footprint2 slab": lambda: ctx.footprint(g, fp, *lay[:3], lay[4], o1, te.MEM_HOST, slab=slab, roughness=lay[3], roughness_fp=o2),
        "te_footprint2 device": lambda: ctx.footprint(g, fp, *lay[:3], lay[4], o1, te.MEM_DEVICE, roughness=lay[3], roughness_fp=o2),
        "te_footprint_polygon slab": lambda: ctx.footprint_polygon(g, fp, poly, 0.5, *lay[:3], lay[4], o1, o2, te.MEM_HOST, slab=slab,
                                                                    roughness=lay[3]),
        "te_footprint_polygon device": lambda: ctx.footprint_polygon(g, fp, poly, 0.5, *lay[:3], lay[4], o1, o2, te.MEM_DEVICE,
                                                                      roughness=lay[3]),
        "te_slope": lambda: ctx.slope(g, 0.5, lay[0], o1, te.MEM_HOST),
        "te_normals": lambda: ctx.normals(g, p, lay[0], o1, o2, o3, te.MEM_HOST),
        "te_step": lambda: ctx.step(g, p, lay[0], o1, te.MEM_HOST),
        "te_roughness": lambda: ctx.roughness(g, p, lay[0], lay[1], lay[2], lay[3], o4, te.MEM_HOST),
    }
    for name, call in calls.items():
        with pytest.raises(te.TEError) as err:
            call()
        assert err.value.code == -4, name
