"""ctypes view of submap_oracle.cpp (test infrastructure): GridMap::getSubmap's geometry and mapHasValidTraversabilityAt on the
CPU.  Compiled on first use into a temporary directory (the source tree may be read-only), with the footprint oracle's flags."""
from __future__ import annotations

import ctypes as C

import numpy as np

import cpp_oracle

FIELDS = ("success", "rows", "cols", "top_row", "top_col", "requested_row", "requested_col", "length_x", "length_y", "position_x",
          "position_y")
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cpp_oracle.load("submap_oracle", cpp_oracle.FOOTPRINT_ORACLE, ["-fopenmp"])
        L.teo_submap_geometry.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.teo_valid_at.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def submap_geometry(og, positions, lengths):
    """dict of FIELDS -> array[n] (ints as int64, lengths and positions as float64) for oracle.binding Geometry `og`."""
    p = np.ascontiguousarray(positions, dtype=np.float64).reshape(-1, 2)
    ln = np.ascontiguousarray(lengths, dtype=np.float64).reshape(-1, 2)
    out = np.zeros((len(p), len(FIELDS)), dtype=np.float64)
    assert lib().teo_submap_geometry(C.byref(og), len(p), p.ctypes.data, ln.ctypes.data, out.ctypes.data) == 0
    return {f: (out[:, k] if k >= 7 else out[:, k].astype(np.int64)) for k, f in enumerate(FIELDS)}


def valid_at(og, traversability, xy):
    t = np.asfortranarray(traversability, dtype=np.float32)
    p = np.ascontiguousarray(xy, dtype=np.float64).reshape(-1, 2)
    v = np.zeros(len(p), dtype=np.uint8)
    assert lib().teo_valid_at(C.byref(og), t.ctypes.data, len(p), p.ctypes.data, v.ctypes.data) == 0
    return v
