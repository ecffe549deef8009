"""ctypes view of paths_oracle.cpp (test infrastructure): the CPU restatement of the footprint path checks — a whole
check_footprint_path request on a fresh map or on a persistent traversability_footprint layer, and traversabilityFootprint on
that layer.

The library is compiled on first use into a temporary directory (the source tree may be read-only), with the flags of the
footprint oracle (oracle/Makefile: literal double arithmetic, no contraction).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import cpp_oracle

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cpp_oracle.load("paths_oracle", cpp_oracle.FOOTPRINT_ORACLE, ["-fopenmp"])
        L.teo_check_request.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 11 + \
            [C.c_int, C.c_void_p, C.c_void_p]
        L.teo_map_footprint.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6
        _lib = L
    return _lib


def empty_cache(g):
    """A traversability_footprint layer with nothing stored (NaN everywhere)."""
    return np.full((g.rows, g.cols), np.nan, dtype=np.float32, order="F")


def _layers(g, layers, keys):
    out = [None if layers.get(k) is None else np.asfortranarray(layers[k], dtype=np.float32) for k in keys]
    assert all(a is None or a.shape == (g.rows, g.cols) for a in out)
    return out


def _ad(a):
    return None if a is None else a.ctypes.data


def check_request(g, fp, layers, path_begin, poses, radius=None, footprint_begin=None, footprint_xyz=None, conservative=None,
                  cup=None, cache=None, capacity=64):
    """One check_footprint_path request; g / fp are oracle.binding Geometry / FootprintParams, layers a dict with traversability,
    slope, step, elevation and optionally roughness and robot_slope.

    poses: (nposes, 7) x y z qx qy qz qw, or (nposes, 2) x y when every path is circular.  radius: per path or one for all
    (circular paths only).  footprint_xyz: (n, 3) vertices; with footprint_begin (npaths + 1) path q's footprint is rows
    footprint_begin[q] .. footprint_begin[q+1]-1 (none: circular), without it every path shares footprint_xyz.  conservative /
    cup (compute_untraversable_polygon): per path, one for all or None.  cache: None checks every path on a fresh map; a layer
    from empty_cache is read and updated in place, paths in request order.

    Returns (is_safe, traversability, area, count int32[npaths], xy float64[npaths, capacity, 2]): the published untraversable
    polygon's vertex count and its first min(count, capacity) vertices."""
    pb = np.ascontiguousarray(path_begin, dtype=np.int32)
    n = len(pb) - 1
    ps = np.asarray(poses, dtype=np.float64)
    ps = ps.reshape(-1, ps.shape[-1] if ps.ndim == 2 else 7)
    if ps.shape[1] == 2:   # circular paths read x and y only: the rest is NaN, so that a read of it would show
        assert footprint_xyz is None
        ps = np.concatenate([ps, np.full((len(ps), 5), np.nan)], axis=1)
    ps = np.ascontiguousarray(ps)
    assert ps.shape[1] == 7
    fxyz = np.ascontiguousarray(np.zeros((0, 3)) if footprint_xyz is None else footprint_xyz, dtype=np.float32).reshape(-1, 3)
    if footprint_begin is None:   # one footprint for every path: each gets its own copy
        footprint_begin = np.arange(n + 1) * len(fxyz)
        fxyz = np.ascontiguousarray(np.tile(fxyz, (n, 1)))
    fb = np.ascontiguousarray(footprint_begin, dtype=np.int32)
    rad = np.ascontiguousarray(np.broadcast_to(np.nan if radius is None else radius, (n,)), dtype=np.float64)
    per_path = lambda a: None if a is None else np.ascontiguousarray(np.broadcast_to(a, (n,)), dtype=np.uint8)  # noqa: E731
    cons, cu = per_path(conservative), per_path(cup)
    assert len(fb) == n + 1 and fb[-1] == len(fxyz)
    if cache is not None:
        assert cache.dtype == np.float32 and cache.flags.f_contiguous and cache.shape == (g.rows, g.cols)
    t, s, st, r, e, rs = _layers(g, layers, ("traversability", "slope", "step", "roughness", "elevation", "robot_slope"))
    safe, trav, area = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.float64), np.zeros(n, dtype=np.float64)
    counts = np.zeros(n, dtype=np.int32)
    uxy = np.zeros((n, capacity, 2), dtype=np.float64)
    rc = lib().teo_check_request(C.byref(g), C.byref(fp), _ad(t), _ad(s), _ad(st), _ad(r), _ad(e), _ad(rs), n, pb.ctypes.data,
                                 ps.ctypes.data, rad.ctypes.data, fb.ctypes.data, _ad(fxyz) if len(fxyz) else None, _ad(cons), _ad(cu),
                                 _ad(cache), safe.ctypes.data, trav.ctypes.data, area.ctypes.data, capacity, counts.ctypes.data,
                                 uxy.ctypes.data)
    assert rc == 0, rc
    return safe, trav, area, counts, uxy


def footprint(g, fp, layers, cache):
    """traversabilityFootprint(radius, offset) on `cache` (updated in place)."""
    t, s, st, r, e = _layers(g, layers, ("traversability", "slope", "step", "roughness", "elevation"))
    assert lib().teo_map_footprint(C.byref(g), C.byref(fp), _ad(t), _ad(s), _ad(st), _ad(r), _ad(e), cache.ctypes.data) == 0
