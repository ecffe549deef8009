"""ctypes view of at_poses_oracle.cpp (test infrastructure): GridMap::atPosition at robot-frame points around poses on the CPU.
Compiled on first use into a temporary directory (the source tree may be read-only), with the footprint oracle's flags."""
from __future__ import annotations

import ctypes as C

import numpy as np

import cpp_oracle

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cpp_oracle.load("at_poses_oracle", cpp_oracle.FOOTPRINT_ORACLE, ["-fopenmp"])
        L.teo_at_poses.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def at_poses(og, layer, poses, points):
    """(values float32 (nposes, npoints), valid uint8 (nposes, npoints)): `layer` (rows, cols) at points (npoints, 3) placed at
    poses (nposes, 7) x y z qx qy qz qw, as te_map_at_poses reads one layer, for oracle.binding Geometry `og`."""
    lay = np.asfortranarray(layer, dtype=np.float32)
    q = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
    pts = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    out = np.empty((len(q), len(pts)), dtype=np.float32)
    v = np.empty((len(q), len(pts)), dtype=np.uint8)
    assert lib().teo_at_poses(C.byref(og), lay.ctypes.data, len(q), q.ctypes.data, len(pts), pts.ctypes.data, out.ctypes.data,
                              v.ctypes.data) == 0
    return out, v
