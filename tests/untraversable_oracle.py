"""ctypes view of untraversable_oracle.cpp (test infrastructure): the CPU restatement of the untraversable polygons of
te_check_footprint_paths_fresh2 / te_check_footprint_paths_polygon2.

The library is compiled on first use into a temporary directory (the source tree may be read-only), with the flags of the
footprint oracle (oracle/Makefile: literal double arithmetic, no contraction).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "untraversable_oracle.cpp")
_DEPS = [_SRC, os.path.join(_HERE, "polygon_paths_oracle.cpp"), os.path.join(_HERE, "..", "oracle", "te_oracle_footprint.cpp"),
         os.path.join(_HERE, "..", "oracle", "te_oracle.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _DEPS)).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"te_untraversable_oracle_{os.getuid()}_{h}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}"
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                                   "-shared", "-o", tmp, _SRC])
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.teo_check_circular_paths_fresh2.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 6 + \
            [C.c_int, C.c_void_p, C.c_void_p]
        L.teo_check_polygonal_paths2.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_int] + \
            [C.c_void_p] * 6 + [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def check_circular_paths_fresh2(g, fp, traversability, slope, step, elevation, path_begin, poses_xy, radius, robot_slope=None,
                                roughness=None, compute_untraversable_polygon=None, capacity=64):
    """(is_safe, traversability, counts int32[npaths], xy float64[npaths, capacity, 2]): check_circular_paths_fresh plus the
    untraversable polygon the service publishes per path (its first min(count, capacity) vertices)."""
    lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
    t, s, st, e, rs, r = (lay(a) for a in (traversability, slope, step, elevation, robot_slope, roughness))
    for a in (t, s, st, e, rs, r):
        assert a is None or a.shape == (g.rows, g.cols), a.shape
    pb = np.ascontiguousarray(path_begin, dtype=np.int32)
    xy = np.ascontiguousarray(poses_xy, dtype=np.float64).reshape(-1, 2)
    rad = np.ascontiguousarray(radius, dtype=np.float64)
    cup = None if compute_untraversable_polygon is None else np.ascontiguousarray(compute_untraversable_polygon, dtype=np.uint8)
    n = len(pb) - 1
    assert len(rad) == n and (cup is None or len(cup) == n)
    safe = np.zeros(n, dtype=np.uint8)
    trav = np.zeros(n, dtype=np.float64)
    counts = np.zeros(n, dtype=np.int32)
    uxy = np.zeros((n, capacity, 2), dtype=np.float64)
    ad = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    rc = lib().teo_check_circular_paths_fresh2(C.byref(g), C.byref(fp), ad(t), ad(s), ad(st), ad(r), ad(e), ad(rs), n, pb.ctypes.data,
                                               xy.ctypes.data, rad.ctypes.data, ad(cup), safe.ctypes.data, trav.ctypes.data, capacity,
                                               counts.ctypes.data, uxy.ctypes.data)
    assert rc == 0, rc
    return safe, trav, counts, uxy


def check_polygonal_paths2(g, fp, traversability, slope, step, elevation, footprint_xyz, path_begin, poses, robot_slope=None,
                           roughness=None, conservative=None, compute_untraversable_polygon=None, capacity=64):
    """(is_safe, traversability, area, counts int32[npaths], xy float64[npaths, capacity, 2]): check_polygonal_paths plus the
    untraversable polygon the service publishes per path (its first min(count, capacity) vertices)."""
    lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
    t, s, st, e, rs, r = (lay(a) for a in (traversability, slope, step, elevation, robot_slope, roughness))
    for a in (t, s, st, e, rs, r):
        assert a is None or a.shape == (g.rows, g.cols), a.shape
    fxyz = np.ascontiguousarray(footprint_xyz, dtype=np.float32).reshape(-1, 3)
    pb = np.ascontiguousarray(path_begin, dtype=np.int32)
    ps = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
    n = len(pb) - 1
    cons = None if conservative is None else np.ascontiguousarray(conservative, dtype=np.uint8)
    cup = None if compute_untraversable_polygon is None else np.ascontiguousarray(compute_untraversable_polygon, dtype=np.uint8)
    assert (cons is None or len(cons) == n) and (cup is None or len(cup) == n)
    safe = np.zeros(n, dtype=np.uint8)
    trav = np.zeros(n, dtype=np.float64)
    area = np.zeros(n, dtype=np.float64)
    counts = np.zeros(n, dtype=np.int32)
    uxy = np.zeros((n, capacity, 2), dtype=np.float64)
    ad = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    rc = lib().teo_check_polygonal_paths2(C.byref(g), C.byref(fp), ad(t), ad(s), ad(st), ad(r), ad(e), ad(rs), len(fxyz), fxyz.ctypes.data,
                                          n, pb.ctypes.data, ps.ctypes.data, ad(cons), safe.ctypes.data, trav.ctypes.data,
                                          area.ctypes.data, ad(cup), capacity, counts.ctypes.data, uxy.ctypes.data)
    assert rc == 0, rc
    return safe, trav, area, counts, uxy
