"""te_map_chain_image / te_map_chain_image_maps (the reference node's image topic: addLayerFromImage, then computeTraversability).
The elevation they give equals the CPU oracle's addLayerFromImage (tests/image_oracle.cpp) bit for bit, for mono8 and mono16,
every pixel value, awkward shapes, padded and misaligned strides, host and device memory; everything after the elevation equals
te_map_chain(_batched/_maps) on that elevation bit for bit; errors leave the te_map unchanged; one launch is added."""
import ctypes as C

import numpy as np
import pytest

import image_oracle as io
from helpers import bits, mixed_request, request_footprints, same_bits_or_nan, same_bytes
from map_helpers import ask, close_maps  # noqa: F401

pytestmark = pytest.mark.gpu

BAD_ARG, MISSING_LAYER, UNSUPPORTED = -1, -2, -4
MONO8, MONO16 = 0, 1
CHAIN = ("traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation")
# inverted, equal, negative, a difference that rounds in float32, and one that overflows to inf (pixel 0 then gives NaN)
PAIRS = [(0.0, 1.0), (2.0, -1.5), (0.25, 0.25), (-7.5, -0.3), (-1e7, 0.1), (1.0, 1e-8), (-3e38, 3e38)]
SHAPES = [(1, 1), (1, 300), (300, 1), (37, 1000), (1000, 37), (513, 511)]


class Images:
    """n images of rows x cols pixels in one byte buffer: row stride rs, image stride ims, starting `offset` bytes in."""

    def __init__(self, pix, rs=None, ims=None, offset=0):
        self.pix = pix  # (n, rows, cols) uint8 / uint16
        n, rows, cols = pix.shape
        b = pix.itemsize
        self.rs = rs or cols * b
        self.ims = ims or rows * self.rs
        self.offset = offset
        self.buf = np.zeros(offset + (n - 1) * self.ims + (rows - 1) * self.rs + cols * b + 16, np.uint8)
        for k in range(n):
            for i in range(rows):
                o = offset + k * self.ims + i * self.rs
                self.buf[o:o + cols * b] = pix[k, i].view(np.uint8)
        self.encoding = MONO8 if b == 1 else MONO16

    def host(self):
        return self.buf.ctypes.data + self.offset

    def device(self):
        import torch
        packed = self.offset == 0 and self.rs == self.pix.shape[2] * self.pix.itemsize and self.ims == self.pix.shape[1] * self.rs
        if packed:  # the images as a torch tensor of their own type (int16: torch has no uint16 arithmetic to need)
            self.dev = torch.from_numpy(self.pix if self.pix.itemsize == 1 else self.pix.view(np.int16)).cuda()
            torch.cuda.synchronize()
            return self.dev.data_ptr()
        self.dev = torch.from_numpy(self.buf).cuda()
        torch.cuda.synchronize()
        return self.dev.data_ptr() + self.offset


def _chain_image(te, m, g, p, im, lo, hi, memory, nmaps=None, outs=None, sel=None):
    """The raw entry (te_map_chain_image, or _maps with sel); returns its code.  outs: four float32 arrays or tensors."""
    L = te.load_library()
    ptr = im.host() if memory == te.MEM_HOST else im.device()
    o = [None] * 4 if outs is None else [a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr() for a in outs]
    n = im.pix.shape[0] if nmaps is None else nmaps
    if sel is None:
        rc = L.te_map_chain_image(m._h, C.byref(g), C.byref(p), n, im.encoding, ptr, im.rs, im.ims, lo, hi, *o, memory)
        if rc == 0:
            m._g, m._n = g, n
    else:
        idx = np.ascontiguousarray(sel, np.int32)
        rc = L.te_map_chain_image_maps(m._h, C.byref(g), C.byref(p), len(idx), idx.ctypes.data, im.encoding, ptr, im.rs, im.ims, lo, hi,
                                       *o, memory)
    if memory == te.MEM_DEVICE:
        m._ctx.synchronize()
    return rc


def _elevation(m):
    e = m.get_layers(["elevation"])["elevation"]
    return e if m.nmaps > 1 else e[None]


def _layouts(pix):
    """Packed; rows padded by 3 pixels (a stride that is no multiple of 4 or 16), images padded by 2 pixels and the base moved by
    one pixel (no wide loads); rows padded to a multiple of 16 bytes."""
    n, rows, cols = pix.shape
    b = pix.itemsize
    yield Images(pix)
    yield Images(pix, rs=(cols + 3) * b, ims=rows * (cols + 3) * b + 2 * b, offset=b)
    yield Images(pix, rs=(cols * b + 15) // 16 * 16 + 16)


@pytest.mark.parametrize("memory", [0, 1], ids=["host", "device"])
@pytest.mark.parametrize("nmaps", [1, 5])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{r}x{c}" for r, c in SHAPES])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_elevation_bits(te, ctx, dtype, shape, nmaps, memory):
    rng = np.random.default_rng(shape[0] * 7 + shape[1] + nmaps)
    pix = rng.integers(0, np.iinfo(dtype).max + 1, (nmaps,) + shape, dtype=dtype)
    flat = pix.reshape(-1)
    flat[:2] = [0, np.iinfo(dtype).max][:flat.size]  # both ends of the pixel range
    g = te.image_geometry(shape[0], shape[1], 0.05, (1.5, -2.0))
    p = te.ChainParams.yaml_defaults(0)
    m = ctx.map()
    for k, im in enumerate(_layouts(pix)):
        for lo, hi in PAIRS[k::2] + [PAIRS[-1]]:
            assert _chain_image(te, m, g, p, im, lo, hi, memory) == 0, te.load_library().te_last_error()
            assert same_bits_or_nan(_elevation(m), io.elevation(pix, lo, hi)), (k, lo, hi)


@pytest.mark.parametrize("memory", [0, 1], ids=["host", "device"])
def test_every_pixel_value(te, ctx, memory):
    """A 256 x 256 mono16 image holding every value once and a 16 x 16 mono8 one, at every (min, max) pair."""
    p = te.ChainParams.yaml_defaults(0)
    rng = np.random.default_rng(5)
    for pix in (rng.permutation(65536).astype(np.uint16).reshape(1, 256, 256), rng.permutation(256).astype(np.uint8).reshape(1, 16, 16)):
        g = te.image_geometry(pix.shape[1], pix.shape[2], 0.02)
        m = ctx.map()
        for lo, hi in PAIRS:
            assert _chain_image(te, m, g, p, Images(pix), lo, hi, memory) == 0
            assert same_bits_or_nan(_elevation(m), io.elevation(pix, lo, hi)), (pix.dtype, lo, hi)


def _held(m):
    h = dict(m.get_layers(CHAIN), cache=m.get_footprint())
    return h if m.nmaps > 1 else {k: v[None] for k, v in h.items()}


@pytest.mark.parametrize("memory", [0, 1], ids=["host", "device"])
@pytest.mark.parametrize("nmaps", [1, 5])
def test_chain_layers_equal_float_chain(te, ctx, oracle, nmaps, memory):
    """Every chain layer, the outputs and the empty cache equal te_map_chain(_batched) on the oracle's elevation; one mixed request
    then answers identically on both."""
    rows, cols, res = 200, 180, 0.02
    rng = np.random.default_rng(17 + nmaps)
    yy, xx = np.mgrid[0:rows, 0:cols]
    base = (np.sin(xx / 9.0) * np.cos(yy / 13.0) * 20000 + 30000 + (xx > 90) * 8000).astype(np.int64)
    pix = np.stack([np.clip(base + rng.integers(-600, 600, base.shape), 0, 65535) for _ in range(nmaps)]).astype(np.uint16)
    lo, hi = -0.4, 0.35
    g = te.image_geometry(rows, cols, res)
    p = te.ChainParams.yaml_defaults(0)
    elev = io.elevation(pix, lo, hi)
    a, b = ctx.map(), ctx.map()
    outs = [np.empty(nmaps * rows * cols, np.float32) for _ in range(4)] if memory == te.MEM_HOST else None
    if memory == te.MEM_DEVICE:
        import torch
        outs = [torch.empty(nmaps * rows * cols, dtype=torch.float32, device="cuda") for _ in range(4)]
    assert _chain_image(te, a, g, p, Images(pix), lo, hi, memory, outs=outs) == 0
    if nmaps == 1:
        ref = b.chain(g, p, elev[0], outputs=True)
    else:
        ref = b.chain_batched(g, p, nmaps, elev, outputs=True)
    for o, k in zip(outs, ("slope", "step", "roughness", "traversability")):
        got = o if isinstance(o, np.ndarray) else o.cpu().numpy()
        want = np.asarray(ref[k]).reshape(nmaps, rows, cols).transpose(0, 2, 1).reshape(-1)  # per map column-major
        assert same_bits_or_nan(got, want), k
    ha, hb = _held(a), _held(b)
    for k in hb:
        assert same_bits_or_nan(ha[k], hb[k]), k
    assert np.isnan(ha["cache"]).all()
    with pytest.raises(te.TEError):  # no robot_slope afterwards
        a.get_layers(["robot_slope"])
    if nmaps == 1:
        fps = request_footprints(rng)
        R = dict(mixed_request(rng, oracle.Geometry.make(rows, cols, res), 60, fps), fps=fps)
        ft = te.FootprintParams.yaml_defaults()
        ga, gb = ask(a, ft, R), ask(b, ft, R)
        for x, y in zip(ga, gb):
            assert same_bytes(x, y)
        assert same_bits_or_nan(a.get_footprint(), b.get_footprint())


@pytest.mark.parametrize("memory", [0, 1], ids=["host", "device"])
def test_selected_maps_only(te, ctx, memory):
    """te_map_chain_image_maps equals te_map_chain_maps on the oracle's elevation, and every other map keeps its layers and cache."""
    n, rows, cols, res = 5, 96, 80, 0.02
    rng = np.random.default_rng(23)
    g = te.image_geometry(rows, cols, res)
    p, ft = te.ChainParams.yaml_defaults(0), te.FootprintParams.yaml_defaults()
    first = rng.integers(0, 256, (n, rows, cols)).astype(np.uint8)
    a, b = ctx.map(), ctx.map()
    for m in (a, b):
        m.chain_image(g, p, first, -0.2, 0.3)
        m.footprint(ft)  # fill the caches
    before = _held(a)
    sel = [3, 0]
    pix = rng.integers(0, 256, (2, rows, cols)).astype(np.uint8)
    padded = Images(pix, rs=cols + 5, ims=(cols + 5) * rows + 3, offset=1)
    outs = [np.empty(2 * rows * cols, np.float32) for _ in range(4)] if memory == te.MEM_HOST else None
    assert _chain_image(te, a, g, p, padded, -0.1, 0.5, memory, sel=sel, outs=outs) == 0
    ref = b.chain_maps(g, p, sel, io.elevation(pix, -0.1, 0.5), outputs=True)
    ha, hb = _held(a), _held(b)
    for k in hb:
        assert same_bits_or_nan(ha[k], hb[k]), k
        for j in range(n):
            if j not in sel:
                assert same_bits_or_nan(ha[k][j], before[k][j]), (k, j)
    assert np.isnan(ha["cache"][sel]).all()
    if outs is not None:
        for o, k in zip(outs, ("slope", "step", "roughness", "traversability")):
            assert same_bits_or_nan(o, ref[k].transpose(0, 2, 1).reshape(-1)), k


def test_python_views(te, ctx):
    """Map.chain_image takes sliced, padded, batched and byte-swapped views without the caller copying them."""
    rng = np.random.default_rng(29)
    big = rng.integers(0, 65536, (3, 70, 90)).astype(np.uint16)
    view = big[:, 3:67, 5:81]  # padded rows and images
    g = te.image_geometry(64, 76, 0.05)
    p = te.ChainParams.yaml_defaults(0)
    m = ctx.map()
    out = m.chain_image(g, p, view, 0.1, 2.0, outputs=True)
    assert m.nmaps == 3 and out["slope"].shape == (3, 64, 76)
    assert same_bits_or_nan(m.get_layers(["elevation"])["elevation"], io.elevation(np.ascontiguousarray(view), 0.1, 2.0))
    m.chain_image(g, p, view[1].astype(">u2"), 0.1, 2.0)
    assert m.nmaps == 1 and same_bits_or_nan(m.get_layers(["elevation"])["elevation"], io.elevation(np.ascontiguousarray(view[1]), 0.1, 2.0))
    m2 = ctx.map()
    m2.chain_image(g, p, np.zeros((3, 64, 76), np.uint16), 0.0, 1.0)
    m2.chain_image_maps(g, p, [2], view[1:2], 0.1, 2.0)
    assert same_bits_or_nan(m2.get_layers(["elevation"])["elevation"][2], io.elevation(np.ascontiguousarray(view[1]), 0.1, 2.0))


def test_errors_leave_the_map_unchanged(te, ctx):
    rows, cols, n = 40, 30, 3
    rng = np.random.default_rng(31)
    g = te.image_geometry(rows, cols, 0.05)
    p = te.ChainParams.yaml_defaults(0)
    pix16 = rng.integers(0, 65536, (n, rows, cols)).astype(np.uint16)
    m = ctx.map()
    m.chain_image(g, p, pix16, 0.0, 1.0)
    m.footprint(te.FootprintParams.yaml_defaults())
    before = _held(m)
    g_start = te.image_geometry(rows, cols, 0.05)
    g_start.start_row = 1
    good = Images(pix16)
    odd = Images(pix16, offset=1)
    L = te.load_library()

    class Raw:
        def __init__(self, **kw):
            self.__dict__.update(dict(encoding=good.encoding, ptr=good.host(), rs=good.rs, ims=good.ims, g=g), **kw)

    cases = [
        (UNSUPPORTED, Raw(g=g_start)),
        (UNSUPPORTED, Raw(encoding=2)),  # rgb8
        (UNSUPPORTED, Raw(encoding=9)),  # bgra16
        (BAD_ARG, Raw(encoding=10)),
        (BAD_ARG, Raw(encoding=-1)),
        (MISSING_LAYER, Raw(ptr=None)),
        (BAD_ARG, Raw(rs=cols * 2 - 2)),
        (BAD_ARG, Raw(ims=rows * cols * 2 - 2)),
        (BAD_ARG, Raw(ptr=odd.host(), rs=odd.rs, ims=odd.ims)),  # odd base
        (BAD_ARG, Raw(rs=cols * 2 + 1, ims=(cols * 2 + 1) * rows + 1)),  # odd strides
        (BAD_ARG, Raw(ims=rows * cols * 2 + 1)),
    ]
    for memory in (te.MEM_HOST, te.MEM_DEVICE):
        for want, c in cases:
            for sel in (None, [1, 0, 2]):
                ns = n if sel is None else len(sel)
                if sel is None:
                    rc = L.te_map_chain_image(m._h, C.byref(c.g), C.byref(p), ns, c.encoding, c.ptr, c.rs, c.ims, 0.0, 1.0, None, None, None,
                                              None, memory)
                else:
                    idx = np.asarray(sel, np.int32)
                    rc = L.te_map_chain_image_maps(m._h, C.byref(c.g), C.byref(p), ns, idx.ctypes.data, c.encoding, c.ptr, c.rs, c.ims, 0.0,
                                                   1.0, None, None, None, None, memory)
                assert rc == want, (memory, sel, vars(c), rc, L.te_last_error())
    # the _maps rules: a selection error, a geometry that is not the batch's
    idx = np.asarray([0, 0], np.int32)
    assert L.te_map_chain_image_maps(m._h, C.byref(g), C.byref(p), 2, idx.ctypes.data, good.encoding, good.host(), good.rs, good.ims,
                                     0.0, 1.0, None, None, None, None, te.MEM_HOST) == BAD_ARG
    g2 = te.image_geometry(rows, cols, 0.04)
    idx = np.asarray([0], np.int32)
    assert L.te_map_chain_image_maps(m._h, C.byref(g2), C.byref(p), 1, idx.ctypes.data, good.encoding, good.host(), good.rs, good.ims,
                                     0.0, 1.0, None, None, None, None, te.MEM_HOST) == BAD_ARG
    after = _held(m)
    for k in before:
        assert np.array_equal(bits(after[k]), bits(before[k])), k


def test_launches(te, ctx):
    """A call adds one launch (the conversion) to te_map_chain(_batched/_maps)'s, whatever nmaps."""
    rows, cols = 120, 100
    g = te.image_geometry(rows, cols, 0.02)
    p = te.ChainParams.yaml_defaults(0)
    rng = np.random.default_rng(37)
    pix = rng.integers(0, 256, (4, rows, cols)).astype(np.uint8)
    elev = io.elevation(pix, 0.0, 0.5)
    m = ctx.map()

    def delta(call):
        n0 = ctx.stats()[0]
        call()
        return ctx.stats()[0] - n0

    for _ in range(2):  # the second round is warm
        d = [delta(lambda: m.chain_image(g, p, pix[0], 0.0, 0.5)), delta(lambda: m.chain(g, p, elev[0])),
             delta(lambda: m.chain_image(g, p, pix, 0.0, 0.5)), delta(lambda: m.chain_batched(g, p, 4, elev)),
             delta(lambda: m.chain_image_maps(g, p, [2], pix[:1], 0.0, 0.5)), delta(lambda: m.chain_maps(g, p, [2], elev[:1])),
             delta(lambda: m.chain_image_maps(g, p, [3, 1, 0], pix[:3], 0.0, 0.5)), delta(lambda: m.chain_maps(g, p, [3, 1, 0], elev[:3]))]
    assert d[0] == d[1] + 1 and d[2] == d[3] + 1 and d[4] == d[5] + 1 and d[6] == d[7] + 1, d
