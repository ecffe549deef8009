"""ctypes view of polygon_paths_oracle.cpp (test infrastructure): the CPU restatement of te_check_footprint_paths_polygon.

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
_SRC = os.path.join(_HERE, "polygon_paths_oracle.cpp")
_DEPS = [_SRC, os.path.join(_HERE, "..", "oracle", "te_oracle_footprint.cpp"), os.path.join(_HERE, "..", "oracle", "te_oracle.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(b"".join(open(p, "rb").read() for p in _DEPS)).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"te_polygon_paths_oracle_{os.getuid()}_{h}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}"
            subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
                                   "-shared", "-o", tmp, _SRC])
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.teo_check_polygonal_paths.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_int] + \
            [C.c_void_p] * 6
        _lib = L
    return _lib


def check_polygonal_paths(g, fp, traversability, slope, step, elevation, footprint_xyz, path_begin, poses, robot_slope=None,
                          roughness=None, conservative=None):
    """(is_safe uint8[npaths], traversability float64[npaths], area float64[npaths]); g / fp are oracle.binding Geometry /
    FootprintParams; footprint_xyz: (n, 3) vertices (float32); poses: (nposes, 7) x y z qx qy qz qw."""
    lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
    t, s, st, e, rs, r = (lay(a) for a in (traversability, slope, step, elevation, robot_slope, roughness))
    for a in (t, s, st, e, rs, r):
        assert a is None or a.shape == (g.rows, g.cols), a.shape
    fxyz = np.ascontiguousarray(footprint_xyz, dtype=np.float32).reshape(-1, 3)
    pb = np.ascontiguousarray(path_begin, dtype=np.int32)
    ps = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
    n = len(pb) - 1
    cons = None if conservative is None else np.ascontiguousarray(conservative, dtype=np.uint8)
    assert cons is None or len(cons) == n
    safe = np.zeros(n, dtype=np.uint8)
    trav = np.zeros(n, dtype=np.float64)
    area = np.zeros(n, dtype=np.float64)
    ad = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    rc = lib().teo_check_polygonal_paths(C.byref(g), C.byref(fp), ad(t), ad(s), ad(st), ad(r), ad(e), ad(rs), len(fxyz), fxyz.ctypes.data,
                                         n, pb.ctypes.data, ps.ctypes.data, ad(cons), safe.ctypes.data, trav.ctypes.data,
                                         area.ctypes.data)
    assert rc == 0, rc
    return safe, trav, area
