"""ctypes view of occupancy_oracle.cpp (test infrastructure): GridMapRosConverter::toOccupancyGrid on the CPU.  Compiled on first
use into a temporary directory (the source tree may be read-only), with the footprint oracle's floating-point flags."""
from __future__ import annotations

import ctypes as C

import numpy as np

import cpp_oracle

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cpp_oracle.load("occupancy_oracle")
        L.teo_occupancy_grid.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_void_p]
        L.teo_occupancy_info.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p,
                                         C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def occupancy_grid(layer, data_min, data_max, start=(0, 0)):
    """OccupancyGrid.data (int8, rows * cols) of `layer` (rows, cols), given in the buffer order of start index `start`."""
    lay = np.asfortranarray(layer, dtype=np.float32)
    rows, cols = lay.shape
    out = np.empty(rows * cols, dtype=np.int8)
    assert lib().teo_occupancy_grid(rows, cols, int(start[0]), int(start[1]), lay.ctypes.data, float(np.float32(data_min)),
                                    float(np.float32(data_max)), out.ctypes.data) == 0
    return out


def _around(x, n=4):
    """float32 x and its n neighbours on either side."""
    out, lo, hi = [np.float32(x)], np.float32(x), np.float32(x)
    for _ in range(n):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        out += [lo, hi]
    return out


# data_min / data_max pairs of the value sweep: the visualization config's (1, 0), its reverse, inner and wide ranges, equal bounds
# and non-finite bounds
RANGES = [(1.0, 0.0), (0.0, 1.0), (0.2, 0.7), (-3.0, 5.0), (0.5, 0.5), (0.0, 0.0), (np.nan, 1.0), (0.0, np.inf), (-np.inf, 1.0)]

_NAN_PAYLOADS = [0x7fc00000, 0x7fc12345, 0xffc00000, 0xffc00001, 0x7f800001, 0xff812345, 0x7fffffff]


def sweep_values():
    """float32 values where toOccupancyGrid's rounding and special cases matter: every float within 4 ulp of k/100 and 1 - k/100
    (k = 0..100) and of the points k/100 of each range of RANGES, +-0, denormals, 1 +- ulp, +-Inf, NaNs of several payloads and
    large magnitudes."""
    v = []
    for k in range(101):
        v += _around(np.float32(k) / np.float32(100)) + _around(np.float32(1) - np.float32(k) / np.float32(100))
        for lo, hi in RANGES:
            if np.isfinite(lo) and np.isfinite(hi) and lo != hi:
                v += _around(np.float32(lo) + (np.float32(hi) - np.float32(lo)) * (np.float32(k) / np.float32(100)))
    tiny = np.array([1, 2, 0x7fffff, 0x800000], dtype=np.uint32).view(np.float32)  # denormals and the smallest normal
    v += [np.float32(0.0), np.float32(-0.0), *tiny, *(-tiny), *_around(1.0, 2), np.float32(np.inf), np.float32(-np.inf)]
    v += list(np.array(_NAN_PAYLOADS, dtype=np.uint32).view(np.float32))
    big = np.array([3.4028235e38, 1e30, 1e10, 16777217.0, 65504.0, 1e4, 101.0, 2.0], dtype=np.float32)
    v += [*big, *(-big)]
    return np.array(v, dtype=np.float32)


def occupancy_numpy(layer, data_min, data_max):
    """An independent numpy float32 restatement of toOccupancyGrid on a default-order layer (rows, cols): int8 rows * cols."""
    f = np.float32
    v = np.asarray(layer, dtype=np.float32)
    with np.errstate(all="ignore"):
        q = (v - f(data_min)) / (f(data_max) - f(data_min))
        nan = np.isnan(q)
        r = f(0) + np.minimum(np.maximum(f(0), np.where(nan, f(0), q)), f(1)) * f(100)
        assert r.dtype == np.float32
        g = np.where(nan, np.int8(-1), np.trunc(r).astype(np.int8))
    return np.ascontiguousarray(g.reshape(-1, order="F")[::-1])


def occupancy_info(rows, cols, resolution, length, position):
    """(width, height, resolution float32, origin_x, origin_y) of toOccupancyGrid's MapMetaData."""
    size = np.zeros(2, dtype=np.int32)
    res = np.zeros(1, dtype=np.float32)
    origin = np.zeros(2, dtype=np.float64)
    assert lib().teo_occupancy_info(int(rows), int(cols), float(resolution), float(length[0]), float(length[1]), float(position[0]),
                                    float(position[1]), size.ctypes.data, res.ctypes.data, origin.ctypes.data) == 0
    return int(size[0]), int(size[1]), res[0], float(origin[0]), float(origin[1])
