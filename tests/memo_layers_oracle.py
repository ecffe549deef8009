"""ctypes view of memo_layers_oracle.cpp (test infrastructure): the slope_footprint / step_footprint / roughness_footprint layers
the reference leaves after a sequence of requests, sweeps and clears on one map.

State keeps one map's traversability_footprint cache and the three layers, as the reference node's traversabilityMap_ holds them,
and replays calls on them in order."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import cpp_oracle
import paths_oracle as po

_lib = None
NAMES = ("slope_footprint", "step_footprint", "roughness_footprint")


def lib():
    global _lib
    if _lib is None:
        deps = (*cpp_oracle.FOOTPRINT_ORACLE, os.path.join(cpp_oracle.HERE, "paths_oracle.cpp"))
        L = cpp_oracle.load("memo_layers_oracle", deps, ["-fopenmp"])
        L.teo_memo_request.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 11
        L.teo_memo_sweep.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 9
        _lib = L
    return _lib


def _ad(a):
    return None if a is None else a.ctypes.data


class State:
    """One map of geometry g (oracle.binding Geometry) with `layers` (po.check_request's dict): its cache and the three layers
    (NaN 0x7fc00000 where nothing wrote them, as computeTraversability adds them)."""

    def __init__(self, g, layers):
        self.g, self.layers = g, layers
        self.cache = po.empty_cache(g)
        self.memo = {n: np.full((g.rows, g.cols), np.nan, np.float32, order="F") for n in NAMES}

    def _in(self, keys):
        return po._layers(self.g, self.layers, keys)

    def request(self, fp, R, fps):
        """Request R (helpers.mixed_request, footprints fps) with FootprintParams fp, on the cache and the layers."""
        from helpers import footprint_arrays
        fb, fx = footprint_arrays(R, fps)
        n = len(R["kind"])
        t, s, st, r, e, rs = self._in(("traversability", "slope", "step", "roughness", "elevation", "robot_slope"))
        u8 = lambda a: np.ascontiguousarray(np.broadcast_to(a, (n,)), dtype=np.uint8)  # noqa: E731
        cons, cup = u8(R["cons"]), u8(R["cup"])
        pb = np.ascontiguousarray(R["begin"], np.int32)
        ps = np.ascontiguousarray(R["poses"], np.float64).reshape(-1, 7)
        rad = np.ascontiguousarray(R["radius"], np.float64)
        fb = np.ascontiguousarray(fb, np.int32)
        fx = np.ascontiguousarray(fx, np.float32).reshape(-1, 3)
        m = self.memo
        rc = lib().teo_memo_request(C.byref(self.g), C.byref(fp), _ad(t), _ad(s), _ad(st), _ad(r), _ad(e), _ad(rs), n, _ad(pb),
                                    _ad(ps), _ad(rad), _ad(fb), _ad(fx) if len(fx) else None, _ad(cons), _ad(cup), _ad(self.cache),
                                    _ad(m[NAMES[0]]), _ad(m[NAMES[1]]), _ad(m[NAMES[2]]))
        assert rc == 0, rc

    def sweep(self, fp):
        """traversabilityFootprint(radius, offset) with FootprintParams fp."""
        t, s, st, r, e = self._in(("traversability", "slope", "step", "roughness", "elevation"))
        m = self.memo
        assert lib().teo_memo_sweep(C.byref(self.g), C.byref(fp), _ad(t), _ad(s), _ad(st), _ad(r), _ad(e), _ad(self.cache),
                                    _ad(m[NAMES[0]]), _ad(m[NAMES[1]]), _ad(m[NAMES[2]])) == 0

    def clear(self):
        """resetTraversabilityFootprintLayers: the cache, slope_footprint and step_footprint; roughness_footprint stays."""
        self.cache[...] = np.nan
        self.memo[NAMES[0]][...] = np.nan
        self.memo[NAMES[1]][...] = np.nan

    def reset_memo(self):
        """A new memo key: the three layers NaN, the cache kept."""
        for a in self.memo.values():
            a[...] = np.nan
