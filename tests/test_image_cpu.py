"""te_image_geometry without a GPU: initializeFromImage's geometry, bit for bit against the CPU oracle (tests/image_oracle.cpp), and
its argument errors; and the oracle's own addLayerFromImage arithmetic at the ends of the pixel range."""
import ctypes as C

import numpy as np
import pytest

import image_oracle as io

BAD_ARG = -1
SIZES = [(1, 1), (1, 7), (9, 1), (480, 640), (37, 1000), (8192, 8192), (65535, 3)]
# 0.1, 0.03, 0.07 and 0.3 are not binary fractions: resolution * size / resolution is then not always exactly size
RESOLUTIONS = [0.02, 0.05, 0.1, 0.03, 0.07, 0.3, 1.0 / 3.0, 0.25, 1e-3, 7.5, 5e-300]
POSITIONS = [(0.0, 0.0), (1.2345, -7.891), (2.6e6, 1.2e6)]


def _fields(g):
    return np.array([g.length_x, g.length_y, g.position_x, g.position_y, g.resolution]).view(np.uint64), (g.rows, g.cols,
                                                                                                          g.start_row, g.start_col)


@pytest.mark.parametrize("pos", POSITIONS)
def test_geometry_equals_oracle(te, pos):
    inexact = 0
    for h, w in SIZES:
        for res in RESOLUTIONS:
            g = te.image_geometry(h, w, res, pos)
            o = io.image_geometry(h, w, res, pos)
            want = np.array([o["length_x"], o["length_y"], o["position_x"], o["position_y"], res]).view(np.uint64)
            got, ints = _fields(g)
            assert np.array_equal(got, want), (h, w, res)
            assert ints == (o["rows"], o["cols"], 0, 0), (h, w, res)
            inexact += (res * h / res != h) + (res * w / res != w)
    assert inexact > 0  # the sizes above do exercise the rounding in setGeometry


@pytest.mark.parametrize("args", [
    (0, 5, 0.1, 0.0, 0.0), (5, 0, 0.1, 0.0, 0.0), (-3, 5, 0.1, 0.0, 0.0),
    (5, 5, 0.0, 0.0, 0.0), (5, 5, -0.1, 0.0, 0.0), (5, 5, float("nan"), 0.0, 0.0), (5, 5, float("inf"), 0.0, 0.0),
    (5, 5, 0.1, float("nan"), 0.0), (5, 5, 0.1, 0.0, float("inf")), (5, 5, 0.1, float("-inf"), 0.0),
    (2 ** 31 - 1, 5, 1e300, 0.0, 0.0),
])
def test_geometry_errors_leave_out_untouched(te, args):
    L = te.load_library()
    g = te.Geometry(11, 12, 0.5, 5.5, 6.0, 1.0, 2.0, 3, 4)
    before = bytes(g)
    assert L.te_image_geometry(*args, C.byref(g)) == BAD_ARG
    assert bytes(g) == before
    assert L.te_image_geometry(5, 5, 0.1, 0.0, 0.0, None) == BAD_ARG


def test_python_view_raises(te):
    with pytest.raises(te.TEError):
        te.image_geometry(0, 4, 0.1)


@pytest.mark.parametrize("dtype,top", [(np.uint8, 255), (np.uint16, 65535)])
@pytest.mark.parametrize("lo,hi", [(0.0, 1.0), (-2.5, 7.25), (3.0, -1.0), (0.4, 0.4), (1.0, 1e-8), (-1e7, 0.1), (0.1, 0.3)])
def test_oracle_pixel_range(dtype, top, lo, hi):
    """Pixel 0 gives (float)min_height; the top pixel gives lower + (upper - lower) * 1.0f in float32, which need not be
    (float)max_height: the oracle computes it and does not shortcut either end."""
    img = np.array([[0, top]], dtype=dtype)
    e = io.elevation(img, lo, hi)
    lower, upper = np.float32(lo), np.float32(hi)
    assert e[0, 0].view(np.uint32) == lower.view(np.uint32)
    with np.errstate(over="ignore"):
        want_top = lower + (upper - lower) * np.float32(1.0)
    assert e[0, 1].view(np.uint32) == np.float32(want_top).view(np.uint32)
    if (lo, hi) == (1.0, 1e-8):  # upper - lower rounds to -1: the top pixel gives 0, not 1e-8
        assert e[0, 1] == 0.0 and upper != 0.0


def test_oracle_every_value():
    """Every mono16 value against numpy's float32 evaluation of the same formula, and the transposed layout."""
    v = np.arange(65536, dtype=np.uint16).reshape(256, 256)
    lo, hi = np.float32(-3.7), np.float32(12.9)
    e = io.elevation(v, -3.7, 12.9)
    want = lo + (hi - lo) * (v.astype(np.float32) / np.float32(65535.0))
    assert np.array_equal(e.view(np.uint32), want.astype(np.float32).view(np.uint32))
    strided = np.zeros((5, 300), dtype=np.uint8)
    strided[:, :7] = np.arange(35).reshape(5, 7)
    assert np.array_equal(io.elevation(strided[:, :7], 0.0, 2.0), io.elevation(np.ascontiguousarray(strided[:, :7]), 0.0, 2.0))
