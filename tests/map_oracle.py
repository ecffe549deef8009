"""ctypes view of map_oracle.cpp (test infrastructure): the sequential CPU restatement of te_map — the check_footprint_path
service loop and traversabilityFootprint(radius, offset) on a persistent traversability_footprint layer.

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
_SRC = os.path.join(_HERE, "map_oracle.cpp")
_DEPS = [_SRC, os.path.join(_HERE, "untraversable_oracle.cpp"), os.path.join(_HERE, "polygon_paths_oracle.cpp"),
         os.path.join(_HERE, "..", "oracle", "te_oracle_footprint.cpp"), os.path.join(_HERE, "..", "oracle", "te_oracle.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _DEPS)).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"te_map_oracle_{os.getuid()}_{h}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}"
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                                   "-shared", "-o", tmp, _SRC])
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.teo_map_check_request.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 11 + \
            [C.c_int, C.c_void_p, C.c_void_p]
        L.teo_map_footprint.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6
        _lib = L
    return _lib


def empty_cache(g):
    return np.full((g.rows, g.cols), np.nan, dtype=np.float32, order="F")


def check_request(g, fp, layers, cache, path_begin, poses, radius, footprint_begin, footprint_xyz, conservative=None,
                  compute_untraversable_polygon=None, capacity=64):
    """One request on `cache` (float32 rows x cols, Fortran order, NaN = empty; updated in place).  layers: dict with
    traversability, slope, step, elevation and optionally roughness, robot_slope.  Returns (is_safe, traversability, area, counts,
    xy[npaths, capacity, 2])."""
    assert cache.dtype == np.float32 and cache.flags.f_contiguous and cache.shape == (g.rows, g.cols)
    lay = lambda k: None if layers.get(k) is None else np.asfortranarray(layers[k], dtype=np.float32)  # noqa: E731
    t, s, st, r, e, rs = (lay(k) for k in ("traversability", "slope", "step", "roughness", "elevation", "robot_slope"))
    pb = np.ascontiguousarray(path_begin, dtype=np.int32)
    ps = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
    rad = np.ascontiguousarray(radius, dtype=np.float64)
    fb = np.ascontiguousarray(footprint_begin, dtype=np.int32)
    fxyz = np.ascontiguousarray(footprint_xyz, dtype=np.float32).reshape(-1, 3)
    n = len(pb) - 1
    per_path = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint8)  # noqa: E731
    cons, cup = per_path(conservative), per_path(compute_untraversable_polygon)
    safe, trav, area = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.float64), np.zeros(n, dtype=np.float64)
    counts = np.zeros(n, dtype=np.int32)
    uxy = np.zeros((n, capacity, 2), dtype=np.float64)
    ad = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    rc = lib().teo_map_check_request(C.byref(g), C.byref(fp), ad(t), ad(s), ad(st), ad(r), ad(e), ad(rs), n, pb.ctypes.data,
                                     ps.ctypes.data, rad.ctypes.data, fb.ctypes.data, ad(fxyz) if len(fxyz) else None, ad(cons), ad(cup),
                                     cache.ctypes.data, safe.ctypes.data, trav.ctypes.data, area.ctypes.data, capacity,
                                     counts.ctypes.data, uxy.ctypes.data)
    assert rc == 0, rc
    return safe, trav, area, counts, uxy


def footprint(g, fp, layers, cache):
    """traversabilityFootprint(radius, offset) on `cache` (updated in place)."""
    lay = lambda k: None if layers.get(k) is None else np.asfortranarray(layers[k], dtype=np.float32)  # noqa: E731
    t, s, st, r, e = (lay(k) for k in ("traversability", "slope", "step", "roughness", "elevation"))
    ad = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    assert lib().teo_map_footprint(C.byref(g), C.byref(fp), ad(t), ad(s), ad(st), ad(r), ad(e), cache.ctypes.data) == 0
