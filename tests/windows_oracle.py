"""ctypes view of windows_oracle.cpp (test infrastructure): the window rule of te_map_chain_windows and the cut of a window out of
a circular-buffer elevation map, on the CPU.  Compiled on first use into a temporary directory (the source tree may be read-only),
with the footprint oracle's flags."""
from __future__ import annotations

import ctypes as C

import numpy as np

import cpp_oracle

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cpp_oracle.load("windows_oracle", cpp_oracle.FOOTPRINT_ORACLE, ["-fopenmp"])
        L.teo_window_geometry.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_void_p,
                                          C.c_void_p]
        L.teo_cut.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p]
        _lib = L
    return _lib


def window_geometry(og, rows, cols, positions, length=None):
    """(top int64 (n, 2), position float64 (n, 2)) of windows of rows x cols cells at `positions` (n, 2) on the map of
    oracle.binding Geometry `og`; length: the windows' (length_x, length_y), rows * res and cols * res when None."""
    xy = np.ascontiguousarray(positions, dtype=np.float64).reshape(-1, 2)
    lx, ly = (rows * og.resolution, cols * og.resolution) if length is None else length
    top = np.zeros((len(xy), 2), dtype=np.int64)
    pos = np.zeros((len(xy), 2), dtype=np.float64)
    assert lib().teo_window_geometry(C.byref(og), len(xy), rows, cols, lx, ly, xy.ctypes.data, top.ctypes.data, pos.ctypes.data) == 0
    return top, pos


def cut(layer, start, top, rows, cols):
    """The rows x cols window from map cell `top` of `layer`, a (src_rows, src_cols) array as the circular buffer stores it with
    start index `start`: float32 (rows, cols), NaN outside the map."""
    lay = np.asfortranarray(layer, dtype=np.float32)
    out = np.empty((rows, cols), dtype=np.float32, order="F")
    assert lib().teo_cut(lay.shape[0], lay.shape[1], int(start[0]), int(start[1]), lay.ctypes.data, int(top[0]), int(top[1]), rows,
                         cols, out.ctypes.data) == 0
    return out
