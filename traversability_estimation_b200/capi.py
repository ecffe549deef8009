"""ctypes view of include/te_b200.h."""
from __future__ import annotations

import ctypes as C
import os
import sys
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# TE_B200_LIBRARY: development only — load a variant built with `make -C csrc variant NAME=... EXTRA=...` (several builds
# of the kernels can then be timed in one GPU session); the product library is the one next to this file.
_LIB = os.environ.get("TE_B200_LIBRARY") or os.path.join(_HERE, "libte_b200.so")

MEM_HOST, MEM_DEVICE = 0, 1
KERNEL_AUTO, KERNEL_GENERIC, KERNEL_FUSED = 0, 1, 2

IPC_HANDLE_BYTES = 80  # TE_IPC_HANDLE_BYTES

# te_layer: bit k of a layer mask is LAYERS[k]; outputs that hold several layers have them in this order.
LAYERS = ("traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation", "robot_slope",
          "traversability_footprint")


def layer_mask(names) -> int:
    """The te_layer mask of layer names (any order; each once)."""
    names = list(names)
    unknown = [n for n in names if n not in LAYERS]
    if unknown or len(set(names)) != len(names):
        raise ValueError(f"layer names {names}: each once, from {LAYERS}")
    return sum(1 << LAYERS.index(n) for n in names)


class SubmapInfo(C.Structure):
    """te_submap_info."""
    _fields_ = [("success", C.c_int32), ("rows", C.c_int32), ("cols", C.c_int32), ("top_row", C.c_int32), ("top_col", C.c_int32),
                ("requested_row", C.c_int32), ("requested_col", C.c_int32), ("reserved", C.c_int32),
                ("length_x", C.c_double), ("length_y", C.c_double), ("position_x", C.c_double), ("position_y", C.c_double),
                ("offset", C.c_int64)]


# te_submap_info as a numpy record, for arrays of them
SUBMAP_INFO_DTYPE = np.dtype([(n, np.dtype(t._type_)) for n, t in SubmapInfo._fields_])
assert SUBMAP_INFO_DTYPE.itemsize == C.sizeof(SubmapInfo)


def _windows(positions, lengths):
    p = np.ascontiguousarray(positions, dtype=np.float64).reshape(-1, 2)
    ln = np.ascontiguousarray(lengths, dtype=np.float64).reshape(-1, 2)
    if len(p) != len(ln):
        raise ValueError(f"{len(p)} positions but {len(ln)} lengths")
    return p, ln


class TEError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"te_b200 error {code}: {msg}")
        self.code = code


class Geometry(C.Structure):
    _fields_ = [("rows", C.c_int32), ("cols", C.c_int32), ("resolution", C.c_double),
                ("length_x", C.c_double), ("length_y", C.c_double),
                ("position_x", C.c_double), ("position_y", C.c_double),
                ("start_row", C.c_int32), ("start_col", C.c_int32)]

    @classmethod
    def make(cls, rows, cols, resolution, position=(0.0, 0.0)):
        # GridMap::setGeometry: length = size * resolution
        return cls(rows, cols, resolution, rows * resolution, cols * resolution, position[0], position[1], 0, 0)


class Slab(C.Structure):
    _fields_ = [("col_begin", C.c_int32), ("col_count", C.c_int32), ("halo_left", C.c_int32), ("halo_right", C.c_int32)]


class HaloPeer(C.Structure):
    """te_halo_peer: a neighbour's slab buffer as mapped into this process."""
    _fields_ = [("layer", C.c_void_p), ("slab", Slab), ("ready_event", C.c_void_p)]


class ChainParams(C.Structure):
    _fields_ = [("normals_radius", C.c_double), ("normals_algorithm", C.c_int32),
                ("normals_positive_axis", C.c_int32), ("slope_critical", C.c_double),
                ("step_critical", C.c_double), ("step_first_radius", C.c_double),
                ("step_second_radius", C.c_double), ("step_critical_cells", C.c_int32),
                ("reserved0", C.c_int32), ("roughness_critical", C.c_double),
                ("roughness_radius", C.c_double), ("fuse_weight", C.c_float), ("reserved1", C.c_int32)]

    @classmethod
    def yaml_defaults(cls, algorithm=0):
        """traversability_estimation/config/robot_filter_parameter.yaml:2-37"""
        return cls(0.05, algorithm, 2, 1.0, 0.12, 0.04, 0.04, 4, 0, 0.05, 0.05,
                   np.float32(1.0) / np.float32(3.0), 0)


class FootprintParams(C.Structure):
    _fields_ = [("radius", C.c_double), ("offset", C.c_double), ("traversability_default", C.c_double),
                ("max_gap_width", C.c_double), ("critical_step_height", C.c_double),
                ("radius_is_integer_norm", C.c_int32), ("verify_roughness", C.c_int32)]

    @classmethod
    def yaml_defaults(cls):
        """robot_footprint_parameter.yaml:5-8, robot.yaml:10, robot_filter_parameter.yaml:18"""
        return cls(0.30, 0.15, 0.3, 0.3, 0.12, 1, 0)


# Every entry point of include/te_b200.h in header order: name -> (restype, argtypes), applied once by load_library().  Without
# argtypes ctypes passes a Python int as a C int, so an undeclared entry would get truncated addresses.  Kinds: handles (te_ctx*,
# te_map*), void* and every data pointer or array, host or device, are c_void_p; a parameter struct is a POINTER to its Structure
# (pass byref(s) or s); int and int32_t are c_int32.  tests/test_capi_signatures_cpu.py checks the table against the header.
_P, _I, _U, _L, _Z, _D = C.c_void_p, C.c_int32, C.c_uint32, C.c_int64, C.c_size_t, C.c_double
_G, _S, _CP, _FP, _HP = (C.POINTER(s) for s in (Geometry, Slab, ChainParams, FootprintParams, HaloPeer))
_R = C.c_int
SIGNATURES = {
    "te_create": (_R, [_P, _I]),
    "te_destroy": (_R, [_P]),
    "te_last_error": (C.c_char_p, []),
    "te_abi_version": (_R, []),
    "te_host_alloc": (_R, [_P, _Z]),
    "te_host_free": (_R, [_P]),
    "te_set_stream": (_R, [_P, _P]),
    "te_synchronize": (_R, [_P]),
    "te_set_kernel": (_R, [_P, _I]),
    "te_get_stats": (_R, [_P, _P, _P]),
    "te_enable_timing": (_R, [_P, _I]),
    "te_get_timing": (_R, [_P, _P, _P, _P]),
    "te_get_flag_counters": (_R, [_P, _P]),
    "te_get_escalation_stats": (_R, [_P, _P, _P]),
    "te_fused_plan": (_R, [_I, _I, _I, _I, _P]),
    "te_slope": (_R, [_P, _G, _D, _P, _P, _I]),
    "te_normals": (_R, [_P, _G, _CP, _P, _P, _P, _P, _I]),
    "te_step": (_R, [_P, _G, _CP, _P, _P, _I]),
    "te_roughness": (_R, [_P, _G, _CP, _P, _P, _P, _P, _P, _I]),
    "te_chain": (_R, [_P, _G, _S, _CP, _P, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_chain_batched": (_R, [_P, _G, _CP, _I, _P, _P, _P, _P, _P, _I]),
    "te_footprint": (_R, [_P, _G, _S, _FP, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_footprint2": (_R, [_P, _G, _S, _FP, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_footprint_polygon": (_R, [_P, _G, _S, _FP, _I, _P, _D, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_footprint_batched": (_R, [_P, _G, _FP, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_footprint_polygon_batched": (_R, [_P, _G, _FP, _I, _I, _P, _D, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_footprint_polygon_yaws": (_R, [_P, _G, _FP, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_footprint_polygon_yaws_reduce": (_R, [_P, _G, _FP, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_check_footprint_paths": (_R, [_P, _G, _P, _D, _I, _P, _P, _P, _P, _I]),
    "te_check_footprint_paths2": (_R, [_P, _G, _P, _P, _D, _I, _P, _P, _P, _P, _I]),
    "te_check_footprint_paths_fresh": (_R, [_P, _G, _FP, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I]),
    "te_check_footprint_paths_polygon": (_R, [_P, _G, _FP, _P, _P, _P, _P, _P, _P, _I, _P, _I, _I, _P, _P, _P, _P, _P, _P, _I]),
    "te_check_footprint_paths_fresh2": (_R, [_P, _G, _FP, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _P, _P, _I]),
    "te_check_footprint_paths_polygon2": (_R, [_P, _G, _FP, _P, _P, _P, _P, _P, _P, _I, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _I]),
    "te_check_footprint_request": (_R, [_P, _G, _FP, _P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P, _I]),
    "te_check_footprint_request_batched": (_R, [_P, _G, _FP, _I, _P, _P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P, _I]),
    "te_map_create": (_R, [_P, _P]),
    "te_map_destroy": (_R, [_P]),
    "te_map_chain": (_R, [_P, _G, _CP, _P, _P, _P, _P, _P, _I]),
    "te_map_set_layers": (_R, [_P, _G, _P, _P, _P, _P, _P, _P, _I]),
    "te_map_chain_batched": (_R, [_P, _G, _CP, _I, _P, _P, _P, _P, _P, _I]),
    "te_map_set_layers_batched": (_R, [_P, _G, _I, _P, _P, _P, _P, _P, _P, _I]),
    "te_map_footprint": (_R, [_P, _FP, _P, _I]),
    "te_map_footprint_polygon": (_R, [_P, _FP, _I, _P, _D, _P, _P, _I]),
    "te_map_footprint_polygon_yaws": (_R, [_P, _FP, _I, _P, _I, _P, _P, _I]),
    "te_map_footprint_polygon_yaws_reduce": (_R, [_P, _FP, _I, _P, _I, _P, _P, _P, _P, _I]),
    "te_map_check_footprint_request": (_R, [_P, _FP, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_check_footprint_request_batched": (_R, [_P, _FP, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_check_footprint_request_device": (_R, [_P, _FP, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P, _L]),
    "te_map_get_footprint": (_R, [_P, _P, _I]),
    "te_map_clear_footprint": (_R, [_P]),
    "te_map_request_stats": (_R, [_P, _P]),
    "te_submap_geometry": (_R, [_G, _I, _P, _P, _P]),
    "te_map_get_layers": (_R, [_P, _U, _P, _I]),
    "te_map_get_submaps": (_R, [_P, _I, _P, _P, _U, _P, _P, _L, _I]),
    "te_map_get_submaps_batched": (_R, [_P, _I, _P, _P, _P, _U, _P, _P, _L, _I]),
    "te_map_valid_at": (_R, [_P, _I, _P, _P, _I]),
    "te_map_valid_at_batched": (_R, [_P, _I, _P, _P, _P, _I]),
    "te_ipc_export": (_R, [_P, _P]),
    "te_ipc_open": (_R, [_P, _P]),
    "te_ipc_close": (_R, [_P]),
    "te_event_create_ipc": (_R, [_P, _P, _P]),
    "te_event_open_ipc": (_R, [_P, _P]),
    "te_event_record": (_R, [_P, _P]),
    "te_event_destroy": (_R, [_P]),
    "te_halo_pull": (_R, [_P, _G, _S, _P, _HP, _HP]),
}
EXPORTS = list(SIGNATURES)


def library_path() -> str:
    return _LIB


def build_library(force: bool = False) -> str:
    """nvcc-compile csrc/ for sm_90a into libte_b200.so, next to this file."""
    args = ["make", "-C", os.path.join(_HERE, "csrc"), "-s"]
    if force:
        args.append("-B")
    subprocess.check_call(args)
    return _LIB


_lib = None


def load_library():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB):
            raise ImportError(f"{_LIB} is missing: run traversability_estimation_b200.build_library() "
                              "(there is no CPU fallback)")
        L = C.CDLL(_LIB)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = L
    return _lib


def fused_plan(rows: int, out_ncols: int, nmaps: int = 1, sms: int = 132) -> dict:
    """te_fused_plan: the (level, map, segment, strip) work units of the fused launch; host arithmetic, no GPU needed."""
    L = load_library()
    out = (C.c_int32 * 19)()
    rc = L.te_fused_plan(rows, out_ncols, nmaps, sms, out)
    if rc != 0:
        raise TEError(rc, "te_fused_plan: invalid argument")
    nl = out[1]
    levels = [dict(unit0=out[2 + 4 * i], col0=out[3 + 4 * i], seg_len=out[4 + 4 * i], nseg=out[5 + 4 * i]) for i in range(nl)]
    return {"strips": out[0], "levels": levels, "units": out[2 + 4 * nl]}


def submap_geometry(g, positions, lengths):
    """te_submap_geometry: GridMap::getSubmap's geometry of each window ((x, y) position and length per row) on the map `g`, as
    an array of SUBMAP_INFO_DTYPE records; offsets count one layer per window.  Host arithmetic, no GPU needed."""
    L = load_library()
    p, ln = _windows(positions, lengths)
    info = np.zeros(len(p), dtype=SUBMAP_INFO_DTYPE)
    rc = L.te_submap_geometry(C.byref(g), len(p), p.ctypes.data, ln.ctypes.data, info.ctypes.data)
    if rc != 0:
        raise TEError(rc, L.te_last_error().decode())
    return info


def _addr(a):
    """Address of a numpy array (host) / torch tensor (device) / int / None."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError(type(a))


def _untraversable_outputs(npaths, capacity):
    """Host outputs of the untraversable polygons: counts int32[npaths], xy float64[npaths, capacity, 2]."""
    if int(capacity) < 0:
        raise ValueError("untraversable_capacity must be >= 0")
    return np.zeros(npaths, dtype=np.int32), np.zeros((npaths, int(capacity), 2), dtype=np.float64)


class Context:
    """One te_ctx (one per rank / plugin instance)."""

    def __init__(self, device: int = 0):
        self._L = load_library()
        h = C.c_void_p()
        self._check(self._L.te_create(C.byref(h), device))
        self._h = h
        self._own_stream = True   # device-memory calls run on the context's own (non-blocking) stream until set_stream(ptr)

    def _order_after_torch(self, memory):
        """This ctypes view is used with torch tensors as device memory.  While the context runs on its own stream nothing orders
        its kernels after the torch kernels that produce their inputs: drain torch's current stream first (callers that pass
        their stream with set_stream need no such thing, nor does the C ABI itself — ordering is the caller's there)."""
        if memory == MEM_DEVICE and self._own_stream and "torch" in sys.modules:
            torch = sys.modules["torch"]
            if torch.cuda.is_available():
                torch.cuda.current_stream().synchronize()

    def _check(self, rc):
        if rc != 0:
            raise TEError(rc, self._L.te_last_error().decode())

    def close(self):
        if getattr(self, "_h", None):
            self._L.te_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, stream_ptr):
        self._check(self._L.te_set_stream(self._h, stream_ptr))
        self._own_stream = not stream_ptr

    def synchronize(self):
        self._check(self._L.te_synchronize(self._h))

    def set_kernel(self, choice):
        self._check(self._L.te_set_kernel(self._h, choice))

    def stats(self):
        a, b = C.c_int64(), C.c_int64()
        self._check(self._L.te_get_stats(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def enable_timing(self, on=True):
        self._check(self._L.te_enable_timing(self._h, 1 if on else 0))

    def timing(self):
        """(main kernel ms, fix-up kernel ms, timed launches) since the last call."""
        a, b, n = C.c_double(), C.c_double(), C.c_int64()
        self._check(self._L.te_get_timing(self._h, C.byref(a), C.byref(b), C.byref(n)))
        return a.value, b.value, n.value

    def flag_counters(self):
        a = (C.c_uint32 * 5)()
        self._check(self._L.te_get_flag_counters(self._h, a))
        return list(a)

    def escalation_stats(self):
        """(cells by escalation reason [16], cells by number of valid window cells [26]) of the last fused launch."""
        a, b = (C.c_uint32 * 16)(), (C.c_uint32 * 26)()
        self._check(self._L.te_get_escalation_stats(self._h, a, b))
        return list(a), list(b)

    def slope(self, g, critical, nz, out, memory):
        self._order_after_torch(memory)
        self._check(self._L.te_slope(self._h, C.byref(g), critical, _addr(nz), _addr(out), memory))

    def normals(self, g, p, elevation, nx, ny, nz, memory):
        self._order_after_torch(memory)
        self._check(self._L.te_normals(self._h, C.byref(g), C.byref(p), _addr(elevation), _addr(nx), _addr(ny), _addr(nz), memory))

    def step(self, g, p, elevation, out, memory):
        self._order_after_torch(memory)
        self._check(self._L.te_step(self._h, C.byref(g), C.byref(p), _addr(elevation), _addr(out), memory))

    def roughness(self, g, p, elevation, nx, ny, nz, out, memory):
        self._order_after_torch(memory)
        self._check(self._L.te_roughness(self._h, C.byref(g), C.byref(p), _addr(elevation), _addr(nx), _addr(ny), _addr(nz),
                                         _addr(out), memory))

    def chain(self, g, p, elevation, slope, step, roughness, traversability, memory, slab=None, nx=None, ny=None, nz=None):
        self._order_after_torch(memory)
        self._check(self._L.te_chain(self._h, C.byref(g), C.byref(slab) if slab is not None else None, C.byref(p),
                                     _addr(elevation), _addr(slope), _addr(step), _addr(roughness), _addr(traversability),
                                     _addr(nx), _addr(ny), _addr(nz), memory))

    def chain_batched(self, g, p, nmaps, elevation, slope, step, roughness, traversability, memory):
        self._order_after_torch(memory)
        self._check(self._L.te_chain_batched(self._h, C.byref(g), C.byref(p), nmaps, _addr(elevation), _addr(slope),
                                             _addr(step), _addr(roughness), _addr(traversability), memory))

    def footprint(self, g, fp, traversability, slope, step, elevation, out, memory, slab=None, slope_fp=None, step_fp=None,
                  roughness=None, roughness_fp=None):
        self._order_after_torch(memory)
        if roughness is None and roughness_fp is None:
            self._check(self._L.te_footprint(self._h, C.byref(g), C.byref(slab) if slab is not None else None, C.byref(fp),
                                             _addr(traversability), _addr(slope), _addr(step), _addr(elevation), _addr(out),
                                             _addr(slope_fp), _addr(step_fp), memory))
        else:
            self._check(self._L.te_footprint2(self._h, C.byref(g), C.byref(slab) if slab is not None else None, C.byref(fp),
                                              _addr(traversability), _addr(slope), _addr(step), _addr(roughness), _addr(elevation),
                                              _addr(out), _addr(slope_fp), _addr(step_fp), _addr(roughness_fp), memory))

    def footprint_polygon(self, g, fp, polygon_xy, yaw, traversability, slope, step, elevation, out_x, out_rot, memory, slab=None, roughness=None):
        """TraversabilityMap::traversabilityFootprint(yaw): layers traversability_x / traversability_rot for the footprint polygon."""
        self._order_after_torch(memory)
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        self._check(self._L.te_footprint_polygon(self._h, C.byref(g), C.byref(slab) if slab is not None else None, C.byref(fp), len(pts),
                                                 pts.ctypes.data, float(yaw), _addr(traversability), _addr(slope), _addr(step), _addr(roughness),
                                                 _addr(elevation), _addr(out_x), _addr(out_rot), memory))

    def footprint_batched(self, g, fp, nmaps, traversability, slope, step, elevation, out, memory, slope_fp=None, step_fp=None,
                          roughness=None, roughness_fp=None):
        """footprint() for nmaps whole maps of geometry g stored back to back (the layout of chain_batched)."""
        self._order_after_torch(memory)
        self._check(self._L.te_footprint_batched(self._h, C.byref(g), C.byref(fp), nmaps, _addr(traversability), _addr(slope),
                                                 _addr(step), _addr(roughness), _addr(elevation), _addr(out), _addr(slope_fp),
                                                 _addr(step_fp), _addr(roughness_fp), memory))

    def footprint_polygon_batched(self, g, fp, nmaps, polygon_xy, yaw, traversability, slope, step, elevation, out_x, out_rot, memory,
                                  roughness=None):
        """footprint_polygon() for nmaps whole maps of geometry g stored back to back (the layout of chain_batched)."""
        self._order_after_torch(memory)
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        self._check(self._L.te_footprint_polygon_batched(self._h, C.byref(g), C.byref(fp), nmaps, len(pts), pts.ctypes.data, float(yaw),
                                                         _addr(traversability), _addr(slope), _addr(step), _addr(roughness),
                                                         _addr(elevation), _addr(out_x), _addr(out_rot), memory))

    def footprint_polygon_yaws(self, g, fp, nmaps, polygon_xy, yaws, traversability, slope, step, elevation, out, memory,
                               roughness=None):
        """footprint_polygon()'s traversability_rot at every yaw of `yaws` (host sequence) for nmaps whole maps of geometry g stored
        back to back (the layout of chain_batched).  `out` is (nyaws, nmaps, cols, rows) C-contiguous: out[k, m] is map m's layer
        at yaws[k]."""
        self._order_after_torch(memory)
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        ys = np.ascontiguousarray(yaws, dtype=np.float64).reshape(-1)
        self._check(self._L.te_footprint_polygon_yaws(self._h, C.byref(g), C.byref(fp), nmaps, len(pts), pts.ctypes.data, len(ys),
                                                      ys.ctypes.data if len(ys) else None, _addr(traversability), _addr(slope),
                                                      _addr(step), _addr(roughness), _addr(elevation), _addr(out), memory))

    def footprint_polygon_yaws_reduce(self, g, fp, nmaps, polygon_xy, yaws, traversability, slope, step, elevation, worst, best,
                                      best_yaw, memory, roughness=None):
        """Per-cell reductions of footprint_polygon_yaws over `yaws` without the stack: worst is the value of the first heading
        that minimises it, best that of the first that maximises it, best_yaw (int32) that heading's index.  Each output is
        (nmaps, cols, rows) C-contiguous, or None when not wanted (not all three)."""
        self._order_after_torch(memory)
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        ys = np.ascontiguousarray(yaws, dtype=np.float64).reshape(-1)
        self._check(self._L.te_footprint_polygon_yaws_reduce(self._h, C.byref(g), C.byref(fp), nmaps, len(pts), pts.ctypes.data, len(ys),
                                                             ys.ctypes.data if len(ys) else None, _addr(traversability), _addr(slope),
                                                             _addr(step), _addr(roughness), _addr(elevation), _addr(worst), _addr(best),
                                                             _addr(best_yaw), memory))

    def check_footprint_paths(self, g, footprint_layer, traversability_default, path_begin, poses_xy, robot_slope=None):
        """Host convenience: (is_safe uint8[npaths], traversability float64[npaths]); footprint_layer is a column-major host layer;
        robot_slope (optional layer) switches checkRobotInclination_ on."""
        f = np.asfortranarray(footprint_layer, dtype=np.float32)
        rs = np.asfortranarray(robot_slope, dtype=np.float32) if robot_slope is not None else None
        pb = np.ascontiguousarray(path_begin, dtype=np.int32)
        xy = np.ascontiguousarray(poses_xy, dtype=np.float64)
        n = len(pb) - 1
        safe, trav = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.float64)
        self._check(self._L.te_check_footprint_paths2(self._h, C.byref(g), f.ctypes.data, rs.ctypes.data if rs is not None else None,
                                                      traversability_default, n, pb.ctypes.data, xy.ctypes.data, safe.ctypes.data,
                                                      trav.ctypes.data, MEM_HOST))
        return safe, trav

    def check_footprint_paths_fresh(self, g, fp, traversability, slope, step, elevation, path_begin, poses_xy, radius, robot_slope=None,
                                    roughness=None, compute_untraversable_polygon=None, memory=MEM_HOST, is_safe=None,
                                    traversability_out=None, untraversable_capacity=None, untraversable_count=None,
                                    untraversable_xy=None):
        """te_check_footprint_paths_fresh: checkCircularFootprintPath on the chain layers as the reference's service answers it on a
        freshly computed map (empty traversability_footprint cache per path).  radius: FootprintPath.radius per path (float64);
        fp supplies offset, traversability_default, max_gap_width, critical_step_height, radius_is_integer_norm and
        verify_roughness.  MEM_HOST: numpy arguments, returns (is_safe uint8[npaths], traversability float64[npaths]).
        MEM_DEVICE: every argument is a device tensor (path_begin int32, poses_xy / radius float64,
        compute_untraversable_polygon uint8) and the results go to the caller's is_safe / traversability_out tensors.
        untraversable_capacity=V (te_check_footprint_paths_fresh2): the tuple gains the untraversable polygons, counts
        (int32[npaths]: vertex count, 0 none, -1 not computed) and xy (float64[npaths, V, 2]: the first min(count, V) vertices);
        in MEM_DEVICE they are the caller's untraversable_count / untraversable_xy tensors."""
        if untraversable_capacity is None:
            fn = self._L.te_check_footprint_paths_fresh
            extra = ()
        else:
            fn = self._L.te_check_footprint_paths_fresh2
        if memory == MEM_DEVICE:
            self._order_after_torch(memory)
            n = int(path_begin.numel()) - 1
            if untraversable_capacity is not None:
                extra = (int(untraversable_capacity), _addr(untraversable_count), _addr(untraversable_xy))
            self._check(fn(
                self._h, C.byref(g), C.byref(fp), _addr(traversability), _addr(slope), _addr(step), _addr(roughness), _addr(elevation),
                _addr(robot_slope), n, _addr(path_begin), _addr(poses_xy), _addr(radius), _addr(compute_untraversable_polygon),
                _addr(is_safe), _addr(traversability_out), *extra, MEM_DEVICE))
            if untraversable_capacity is None:
                return is_safe, traversability_out
            return is_safe, traversability_out, untraversable_count, untraversable_xy
        lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
        t, s, st, e, rs, r = (lay(a) for a in (traversability, slope, step, elevation, robot_slope, roughness))
        pb = np.ascontiguousarray(path_begin, dtype=np.int32)
        xy = np.ascontiguousarray(poses_xy, dtype=np.float64)
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        cup = None if compute_untraversable_polygon is None else np.ascontiguousarray(compute_untraversable_polygon, dtype=np.uint8)
        n = len(pb) - 1
        if len(rad) != n or (cup is not None and len(cup) != n):
            raise ValueError("radius / compute_untraversable_polygon need one entry per path")
        safe = np.zeros(n, dtype=np.uint8) if is_safe is None else is_safe
        trav = np.zeros(n, dtype=np.float64) if traversability_out is None else traversability_out
        if untraversable_capacity is not None:
            counts, uxy = _untraversable_outputs(n, untraversable_capacity)
            extra = (int(untraversable_capacity), counts.ctypes.data, uxy.ctypes.data)
        self._check(fn(
            self._h, C.byref(g), C.byref(fp), _addr(t), _addr(s), _addr(st), _addr(r), _addr(e), _addr(rs), n, pb.ctypes.data,
            xy.ctypes.data, rad.ctypes.data, _addr(cup), safe.ctypes.data, trav.ctypes.data, *extra, MEM_HOST))
        if untraversable_capacity is None:
            return safe, trav
        return safe, trav, counts, uxy

    def check_footprint_paths_polygon(self, g, fp, traversability, slope, step, elevation, footprint_xyz, path_begin, poses,
                                      robot_slope=None, roughness=None, conservative=None, memory=MEM_HOST, is_safe=None,
                                      traversability_out=None, area_out=None, compute_untraversable_polygon=None,
                                      untraversable_capacity=None, untraversable_count=None, untraversable_xy=None):
        """te_check_footprint_paths_polygon: checkPolygonalFootprintPath on the chain layers.  footprint_xyz: (n, 3) vertices
        (float32, host in both modes); poses: (nposes, 7) x y z qx qy qz qw; conservative: FootprintPath.conservative per path.
        fp supplies traversability_default, max_gap_width, critical_step_height and verify_roughness.  MEM_HOST: numpy arguments,
        returns (is_safe uint8, traversability float64, area float64) per path.  MEM_DEVICE: every other argument is a device
        tensor (path_begin int32, poses float64, conservative uint8) and the results go to the caller's is_safe /
        traversability_out / area_out tensors.  untraversable_capacity=V (te_check_footprint_paths_polygon2, with
        compute_untraversable_polygon uint8 per path): the tuple gains counts (int32[npaths]) and xy (float64[npaths, V, 2]) as
        in check_footprint_paths_fresh."""
        if untraversable_capacity is None:
            fn = self._L.te_check_footprint_paths_polygon
            extra = ()
        else:
            fn = self._L.te_check_footprint_paths_polygon2
        fxyz = np.ascontiguousarray(footprint_xyz, dtype=np.float32).reshape(-1, 3)
        if memory == MEM_DEVICE:
            self._order_after_torch(memory)
            n = int(path_begin.numel()) - 1
            nposes = int(poses.numel()) // 7
            if untraversable_capacity is not None:
                extra = (_addr(compute_untraversable_polygon), int(untraversable_capacity), _addr(untraversable_count),
                         _addr(untraversable_xy))
            self._check(fn(
                self._h, C.byref(g), C.byref(fp), _addr(traversability), _addr(slope), _addr(step), _addr(roughness), _addr(elevation),
                _addr(robot_slope), len(fxyz), fxyz.ctypes.data, n, nposes, _addr(path_begin), _addr(poses), _addr(conservative),
                _addr(is_safe), _addr(traversability_out), _addr(area_out), *extra, MEM_DEVICE))
            if untraversable_capacity is None:
                return is_safe, traversability_out, area_out
            return is_safe, traversability_out, area_out, untraversable_count, untraversable_xy
        lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
        t, s, st, e, rs, r = (lay(a) for a in (traversability, slope, step, elevation, robot_slope, roughness))
        pb = np.ascontiguousarray(path_begin, dtype=np.int32)
        ps = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
        cons = None if conservative is None else np.ascontiguousarray(conservative, dtype=np.uint8)
        n = len(pb) - 1
        if cons is not None and len(cons) != n:
            raise ValueError("conservative needs one entry per path")
        safe = np.zeros(n, dtype=np.uint8) if is_safe is None else is_safe
        trav = np.zeros(n, dtype=np.float64) if traversability_out is None else traversability_out
        area = np.zeros(n, dtype=np.float64) if area_out is None else area_out
        if untraversable_capacity is not None:
            cup = None if compute_untraversable_polygon is None else np.ascontiguousarray(compute_untraversable_polygon, dtype=np.uint8)
            if cup is not None and len(cup) != n:
                raise ValueError("compute_untraversable_polygon needs one entry per path")
            counts, uxy = _untraversable_outputs(n, untraversable_capacity)
            extra = (_addr(cup), int(untraversable_capacity), counts.ctypes.data, uxy.ctypes.data)
        self._check(fn(
            self._h, C.byref(g), C.byref(fp), _addr(t), _addr(s), _addr(st), _addr(r), _addr(e), _addr(rs), len(fxyz), fxyz.ctypes.data,
            n, len(ps), pb.ctypes.data, ps.ctypes.data, _addr(cons), safe.ctypes.data, trav.ctypes.data, area.ctypes.data, *extra,
            MEM_HOST))
        if untraversable_capacity is None:
            return safe, trav, area
        return safe, trav, area, counts, uxy

    def check_footprint_request(self, g, fp, traversability, slope, step, elevation, path_begin, poses, radius, footprint_begin,
                                footprint_xyz, max_footprint_vertices=None, robot_slope=None, roughness=None, conservative=None,
                                compute_untraversable_polygon=None, memory=MEM_HOST, is_safe=None, traversability_out=None,
                                area_out=None, untraversable_capacity=None, untraversable_count=None, untraversable_xy=None):
        """te_check_footprint_request: a whole CheckFootprintPath request, circular and polygonal paths mixed, in one call.
        poses: (nposes, 7) x y z qx qy qz qw for every path; radius: FootprintPath.radius per path (used by circular paths);
        footprint_xyz: (nvertices, 3) float32, path q's footprint = rows footprint_begin[q] .. footprint_begin[q+1]-1 (none:
        circular).  max_footprint_vertices (0..16) defaults to the longest footprint in MEM_HOST and to 16 in MEM_DEVICE.
        MEM_HOST: numpy arguments, returns (is_safe uint8, traversability float64, area float64) per path in request order.
        MEM_DEVICE: every argument is a device tensor (path_begin / footprint_begin int32, poses / radius float64, footprint_xyz
        float32, conservative / compute_untraversable_polygon uint8) and the results go to the caller's is_safe /
        traversability_out / area_out tensors.  untraversable_capacity=V: the tuple gains counts (int32[npaths]) and xy
        (float64[npaths, V, 2]) as in check_footprint_paths_fresh."""
        return self._request(None, g, fp, traversability, slope, step, elevation, path_begin, poses, radius, footprint_begin,
                             footprint_xyz, max_footprint_vertices, robot_slope, roughness, conservative, compute_untraversable_polygon,
                             memory, is_safe, traversability_out, area_out, untraversable_capacity, untraversable_count, untraversable_xy)

    def check_footprint_request_batched(self, g, fp, nmaps, traversability, slope, step, elevation, path_map, path_begin, poses,
                                        radius, footprint_begin, footprint_xyz, max_footprint_vertices=None, robot_slope=None,
                                        roughness=None, conservative=None, compute_untraversable_polygon=None, memory=MEM_HOST,
                                        is_safe=None, traversability_out=None, area_out=None, untraversable_capacity=None,
                                        untraversable_count=None, untraversable_xy=None):
        """te_check_footprint_request_batched: check_footprint_request() for the paths of nmaps whole maps of geometry g stored back
        to back (the layout of chain_batched: layers shaped (nmaps, cols, rows)); path q is on map path_map[q] (int32 per path).
        Keyword arguments and return values are those of check_footprint_request."""
        return self._request((int(nmaps), path_map), g, fp, traversability, slope, step, elevation, path_begin, poses, radius,
                             footprint_begin, footprint_xyz, max_footprint_vertices, robot_slope, roughness, conservative,
                             compute_untraversable_polygon, memory, is_safe, traversability_out, area_out, untraversable_capacity,
                             untraversable_count, untraversable_xy)

    def _request(self, batch, g, fp, traversability, slope, step, elevation, path_begin, poses, radius, footprint_begin, footprint_xyz,
                 max_footprint_vertices, robot_slope, roughness, conservative, compute_untraversable_polygon, memory, is_safe,
                 traversability_out, area_out, untraversable_capacity, untraversable_count, untraversable_xy):
        """The body of check_footprint_request (batch None) and check_footprint_request_batched (batch = (nmaps, path_map)): the
        batched entry takes nmaps after the parameters and path_map after robot_slope."""
        fn = self._L.te_check_footprint_request if batch is None else self._L.te_check_footprint_request_batched

        def lead(layers, path_map):
            """The arguments up to the path count: parameters, (nmaps,) the layers in argument order, (path_map)."""
            return [C.byref(g), C.byref(fp)] + ([] if batch is None else [batch[0]]) + [_addr(a) for a in layers] + \
                ([] if batch is None else [_addr(path_map)])

        maxv = 0 if untraversable_capacity is None else int(untraversable_capacity)
        if memory == MEM_DEVICE:
            self._order_after_torch(memory)
            n = int(path_begin.numel()) - 1
            mfv = 16 if max_footprint_vertices is None else int(max_footprint_vertices)
            self._check(fn(
                self._h, *lead([traversability, slope, step, roughness, elevation, robot_slope], None if batch is None else batch[1]),
                n, int(poses.numel()) // 7, _addr(path_begin), _addr(poses), _addr(radius),
                int(footprint_xyz.numel()) // 3, _addr(footprint_begin), _addr(footprint_xyz), mfv, _addr(conservative),
                _addr(compute_untraversable_polygon), _addr(is_safe), _addr(traversability_out), _addr(area_out), maxv,
                _addr(untraversable_count), _addr(untraversable_xy), MEM_DEVICE))
            if untraversable_capacity is None:
                return is_safe, traversability_out, area_out
            return is_safe, traversability_out, area_out, untraversable_count, untraversable_xy
        if batch is None:   # one column-major map
            lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
        else:               # (nmaps, cols, rows)
            lay = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
        t, s, st, e, rs, r = (lay(a) for a in (traversability, slope, step, elevation, robot_slope, roughness))
        pb = np.ascontiguousarray(path_begin, dtype=np.int32)
        ps = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        fb = np.ascontiguousarray(footprint_begin, dtype=np.int32)
        fxyz = np.ascontiguousarray(footprint_xyz, dtype=np.float32).reshape(-1, 3)
        pm = None if batch is None or batch[1] is None else np.ascontiguousarray(batch[1], dtype=np.int32)
        n = len(pb) - 1
        per_path = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint8)  # noqa: E731
        cons, cup = per_path(conservative), per_path(compute_untraversable_polygon)
        if len(rad) != n or len(fb) != n + 1 or any(a is not None and len(a) != n for a in (cons, cup, pm)):
            raise ValueError("radius / conservative / compute_untraversable_polygon / path_map need one entry per path, "
                             "footprint_begin npaths + 1")
        if max_footprint_vertices is None:
            max_footprint_vertices = int(np.diff(fb).max()) if n > 0 else 0
        safe = np.zeros(n, dtype=np.uint8) if is_safe is None else is_safe
        trav = np.zeros(n, dtype=np.float64) if traversability_out is None else traversability_out
        area = np.zeros(n, dtype=np.float64) if area_out is None else area_out
        counts, uxy = (None, None) if untraversable_capacity is None else _untraversable_outputs(n, maxv)
        self._check(fn(
            self._h, *lead([t, s, st, r, e, rs], pm), n, len(ps), pb.ctypes.data, ps.ctypes.data, rad.ctypes.data, len(fxyz), fb.ctypes.data, fxyz.ctypes.data, int(max_footprint_vertices), _addr(cons),
            _addr(cup), safe.ctypes.data, trav.ctypes.data, area.ctypes.data, maxv, _addr(counts), _addr(uxy), MEM_HOST))
        if untraversable_capacity is None:
            return safe, trav, area
        return safe, trav, area, counts, uxy

    def map(self):
        """A Map (te_map) owned by this context."""
        return Map(self)

    # ---- multi-GPU halo (te_halo_pull and the IPC helpers around it)
    def ipc_export(self, device_ptr) -> bytes:
        h = C.create_string_buffer(IPC_HANDLE_BYTES)
        self._check(self._L.te_ipc_export(_addr(device_ptr), h))
        return h.raw

    def ipc_open(self, handle: bytes) -> int:
        out = C.c_void_p()
        self._check(self._L.te_ipc_open(C.create_string_buffer(handle, IPC_HANDLE_BYTES), C.byref(out)))
        return out.value

    def ipc_close(self, ptr: int):
        self._check(self._L.te_ipc_close(ptr))

    def event_create_ipc(self):
        """(event, 64-byte handle) of an interprocess event recorded with event_record()."""
        ev, h = C.c_void_p(), C.create_string_buffer(64)
        self._check(self._L.te_event_create_ipc(self._h, C.byref(ev), h))
        return ev.value, h.raw

    def event_open_ipc(self, handle: bytes) -> int:
        ev = C.c_void_p()
        self._check(self._L.te_event_open_ipc(C.create_string_buffer(handle, 64), C.byref(ev)))
        return ev.value

    def event_record(self, event: int):
        self._check(self._L.te_event_record(self._h, event))

    def event_destroy(self, event: int):
        self._check(self._L.te_event_destroy(event))

    def halo_pull(self, g, slab, layer, left=None, right=None):
        self._order_after_torch(MEM_DEVICE)
        self._check(self._L.te_halo_pull(self._h, C.byref(g), C.byref(slab), _addr(layer),
                                         C.byref(left) if left is not None else None, C.byref(right) if right is not None else None))

    # Convenience for host numpy layers (column-major float32), used by tests.
    def chain_host(self, g, p, elevation, with_normals=False):
        e = np.asfortranarray(elevation, dtype=np.float32)
        assert e.shape == (g.rows, g.cols)
        o = {k: np.empty((g.rows, g.cols), np.float32, order="F") for k in ("slope", "step", "roughness", "traversability")}
        n = {k: np.empty((g.rows, g.cols), np.float32, order="F") for k in ("nx", "ny", "nz")} if with_normals else {}
        self.chain(g, p, e, o["slope"], o["step"], o["roughness"], o["traversability"], MEM_HOST, **n)
        o.update(n)
        return o


class Map:
    """te_map: the traversability layers, the traversability_footprint cache and the isTraversableForFilters memo kept on the
    device between calls, so that check_footprint_request answers as the reference's check_footprint_path service does over a
    sequence of requests.  Layers are numpy arrays in host memory (rows x cols, any order; copied column-major); the geometry's
    start index, if any, applies to them and to the layers read back.

    A Map may hold a batch of nmaps maps of one geometry (chain_batched / set_layers_batched): their layers are (nmaps, rows, cols)
    arrays, map k's layer a[k]; every output of the whole-map methods then has that leading nmaps axis, and the methods that address
    one map by position take a map index per path, window or position (the *_batched methods)."""

    def __init__(self, ctx: Context):
        self._ctx = ctx
        self._L = ctx._L
        h = C.c_void_p()
        self._check(self._L.te_map_create(ctx._h, C.byref(h)))
        self._h = h
        self._g = None
        self._n = 1

    @property
    def nmaps(self) -> int:
        """Maps held (1 until chain_batched / set_layers_batched gives it a batch)."""
        return self._n

    def _layer_out(self, count=None, dtype=np.float32):
        """An empty host output of `count` layers (None: one) of every map, laid out as the library writes them (per layer the
        maps back to back, each column-major), and the view returned to the caller: (rows, cols) for one map, (nmaps, rows, cols)
        for a batch, with a leading `count` axis when count is given."""
        rows, cols = self._shape()
        buf = np.empty((1 if count is None else count, self._n, cols, rows), dtype=dtype)
        view = buf.transpose(0, 1, 3, 2)
        if self._n == 1:
            view = view[:, 0]
        return buf, (view[0] if count is None else view)

    @staticmethod
    def _batch_layers(a):
        """(nmaps, rows, cols) host layers as the library reads them: map after map, each column-major."""
        return None if a is None else np.ascontiguousarray(np.asarray(a, dtype=np.float32).transpose(0, 2, 1))

    def _check(self, rc):
        self._ctx._check(rc)

    def close(self):
        if getattr(self, "_h", None):
            self._L.te_map_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _shape(self):
        return (self._g.rows, self._g.cols)

    def chain(self, g, p, elevation, outputs=False):
        """te_map_chain (computeTraversability): empties the cache.  outputs=True also returns the four layers as a dict."""
        fn = self._L.te_map_chain
        e = np.asfortranarray(elevation, dtype=np.float32)
        out = {k: np.empty((g.rows, g.cols), dtype=np.float32, order="F") for k in ("slope", "step", "roughness", "traversability")} \
            if outputs else {}
        self._check(fn(self._h, C.byref(g), C.byref(p), _addr(e), *(_addr(out.get(k)) for k in ("slope", "step", "roughness",
                                                                                                 "traversability")), MEM_HOST))
        self._g, self._n = g, 1
        return out if outputs else None

    def chain_batched(self, g, p, nmaps, elevation, outputs=False):
        """te_map_chain_batched (computeTraversability for every map): elevation (nmaps, rows, cols); empties every cache.
        outputs=True also returns the four layers as a dict of (nmaps, rows, cols) arrays."""
        fn = self._L.te_map_chain_batched
        e = self._batch_layers(elevation)
        out = {k: np.empty((int(nmaps), g.cols, g.rows), dtype=np.float32) for k in ("slope", "step", "roughness", "traversability")} \
            if outputs else {}
        self._check(fn(self._h, C.byref(g), C.byref(p), int(nmaps), _addr(e),
                       *(_addr(out.get(k)) for k in ("slope", "step", "roughness", "traversability")), MEM_HOST))
        self._g, self._n = g, int(nmaps)
        return {k: v.transpose(0, 2, 1) for k, v in out.items()} if outputs else None

    def set_layers(self, g, traversability, slope, step, elevation, roughness=None, robot_slope=None):
        """te_map_set_layers (setTraversabilityMap): empties the cache and the memo."""
        fn = self._L.te_map_set_layers
        lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
        t, s, st, r, e, rs = (lay(a) for a in (traversability, slope, step, roughness, elevation, robot_slope))
        self._check(fn(self._h, C.byref(g), _addr(t), _addr(s), _addr(st), _addr(r), _addr(e), _addr(rs), MEM_HOST))
        self._g, self._n = g, 1

    def set_layers_batched(self, g, nmaps, traversability, slope, step, elevation, roughness=None, robot_slope=None):
        """te_map_set_layers_batched (setTraversabilityMap for every map): each layer (nmaps, rows, cols); empties every cache and
        memo."""
        fn = self._L.te_map_set_layers_batched
        t, s, st, r, e, rs = (self._batch_layers(a) for a in (traversability, slope, step, roughness, elevation, robot_slope))
        self._check(fn(self._h, C.byref(g), int(nmaps), _addr(t), _addr(s), _addr(st), _addr(r), _addr(e), _addr(rs), MEM_HOST))
        self._g, self._n = g, int(nmaps)

    def footprint(self, fp):
        """te_map_footprint (traversabilityFootprint(radius, offset) on the cache); returns the cache afterwards."""
        fn = self._L.te_map_footprint
        if not self._g:
            self._check(fn(self._h, C.byref(fp), None, MEM_HOST))
        buf, out = self._layer_out()
        self._check(fn(self._h, C.byref(fp), _addr(buf), MEM_HOST))
        return out

    def footprint_polygon(self, fp, polygon_xy, yaw):
        """te_map_footprint_polygon: (traversability_x, traversability_rot) of the map's layers."""
        fn = self._L.te_map_footprint_polygon
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        (bx, ox), (brot, orot) = self._layer_out(), self._layer_out()
        self._check(fn(self._h, C.byref(fp), len(pts), pts.ctypes.data, float(yaw), _addr(bx), _addr(brot), MEM_HOST))
        return ox, orot

    def footprint_polygon_yaws(self, fp, polygon_xy, yaws):
        """te_map_footprint_polygon_yaws: (nyaws, rows, cols), layer k the traversability_rot at yaws[k] of the map's layers; on a
        batch (nyaws, nmaps, rows, cols)."""
        fn = self._L.te_map_footprint_polygon_yaws
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        ys = np.ascontiguousarray(yaws, dtype=np.float64).reshape(-1)
        buf, out = self._layer_out(len(ys))   # layer k of map m column-major at (k * nmaps + m) * rows * cols
        self._check(fn(self._h, C.byref(fp), len(pts), pts.ctypes.data, len(ys), ys.ctypes.data if len(ys) else None, _addr(buf),
                       MEM_HOST))
        return out

    def footprint_polygon_yaws_reduce(self, fp, polygon_xy, yaws):
        """te_map_footprint_polygon_yaws_reduce: (worst, best, best_yaw) over `yaws` of the map's layers, each (rows, cols) or, on
        a batch, (nmaps, rows, cols)."""
        fn = self._L.te_map_footprint_polygon_yaws_reduce
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        ys = np.ascontiguousarray(yaws, dtype=np.float64).reshape(-1)
        (bw, worst), (bb, best) = self._layer_out(), self._layer_out()
        by, best_yaw = self._layer_out(dtype=np.int32)
        self._check(fn(self._h, C.byref(fp), len(pts), pts.ctypes.data, len(ys), ys.ctypes.data if len(ys) else None, _addr(bw),
                       _addr(bb), _addr(by), MEM_HOST))
        return worst, best, best_yaw

    def check_footprint_request(self, fp, path_begin, poses, radius, footprint_begin, footprint_xyz, max_footprint_vertices=None,
                                conservative=None, compute_untraversable_polygon=None, untraversable_capacity=None):
        """te_map_check_footprint_request: Context.check_footprint_request in host memory on the map's layers and cache.
        Returns (is_safe, traversability, area) and, with untraversable_capacity=V, (counts, xy) too."""
        return self._request(fp, path_begin, poses, radius, footprint_begin, footprint_xyz, max_footprint_vertices, conservative,
                             compute_untraversable_polygon, untraversable_capacity)

    def check_footprint_request_batched(self, fp, path_map, path_begin, poses, radius, footprint_begin, footprint_xyz,
                                        max_footprint_vertices=None, conservative=None, compute_untraversable_polygon=None,
                                        untraversable_capacity=None):
        """te_map_check_footprint_request_batched: check_footprint_request with path q on map path_map[q] (int32 per path), each
        path on its own map's layers and cache, in request order."""
        return self._request(fp, path_begin, poses, radius, footprint_begin, footprint_xyz, max_footprint_vertices, conservative,
                             compute_untraversable_polygon, untraversable_capacity, path_map=path_map)

    def _request(self, fp, path_begin, poses, radius, footprint_begin, footprint_xyz, max_footprint_vertices, conservative,
                 compute_untraversable_polygon, untraversable_capacity, path_map=None):
        """The body of check_footprint_request (path_map None) and check_footprint_request_batched: the batched entry takes
        path_map after the parameters."""
        batched = path_map is not None
        fn = self._L.te_map_check_footprint_request_batched if batched else self._L.te_map_check_footprint_request
        pm = [np.ascontiguousarray(path_map, dtype=np.int32)] if batched else []
        pb = np.ascontiguousarray(path_begin, dtype=np.int32)
        ps = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        fb = np.ascontiguousarray(footprint_begin, dtype=np.int32)
        fxyz = np.ascontiguousarray(footprint_xyz, dtype=np.float32).reshape(-1, 3)
        n = len(pb) - 1
        per_path = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint8)  # noqa: E731
        cons, cup = per_path(conservative), per_path(compute_untraversable_polygon)
        if max_footprint_vertices is None:
            max_footprint_vertices = int(np.diff(fb).max()) if n > 0 else 0
        maxv = 0 if untraversable_capacity is None else int(untraversable_capacity)
        safe, trav, area = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.float64), np.zeros(n, dtype=np.float64)
        counts, uxy = (None, None) if untraversable_capacity is None else _untraversable_outputs(n, maxv)
        if batched and len(pm[0]) != n:
            raise ValueError("path_map needs one entry per path")
        self._check(fn(self._h, C.byref(fp), *(a.ctypes.data for a in pm), n, len(ps), pb.ctypes.data, ps.ctypes.data,
                       rad.ctypes.data, len(fxyz), fb.ctypes.data, fxyz.ctypes.data, int(max_footprint_vertices), _addr(cons),
                       _addr(cup), safe.ctypes.data, trav.ctypes.data, area.ctypes.data, maxv, _addr(counts), _addr(uxy)))
        if untraversable_capacity is None:
            return safe, trav, area
        return safe, trav, area, counts, uxy

    def check_footprint_request_device(self, fp, path_begin, poses, radius, footprint_begin, footprint_xyz, is_safe,
                                       traversability_out, area_out, max_checks, path_map=None, max_footprint_vertices=None,
                                       conservative=None, compute_untraversable_polygon=None, untraversable_capacity=None,
                                       untraversable_count=None, untraversable_xy=None):
        """te_map_check_footprint_request_device: check_footprint_request(_batched) with every argument a device tensor, as
        Context.check_footprint_request(memory=MEM_DEVICE) takes them (path_map int32 per path, None on a map of one map), results
        in the caller's tensors.  Asynchronous: ordered after torch's current stream, no host synchronisation.  max_checks sizes
        the work list of circle checks (te_b200.h).  max_footprint_vertices defaults to 16."""
        self._ctx._order_after_torch(MEM_DEVICE)
        n = int(path_begin.numel()) - 1
        mfv = 16 if max_footprint_vertices is None else int(max_footprint_vertices)
        maxv = 0 if untraversable_capacity is None else int(untraversable_capacity)
        self._check(self._L.te_map_check_footprint_request_device(
            self._h, C.byref(fp), _addr(path_map), n, int(poses.numel()) // 7, _addr(path_begin), _addr(poses), _addr(radius),
            int(footprint_xyz.numel()) // 3, _addr(footprint_begin), _addr(footprint_xyz), mfv, _addr(conservative),
            _addr(compute_untraversable_polygon), _addr(is_safe), _addr(traversability_out), _addr(area_out), maxv,
            _addr(untraversable_count), _addr(untraversable_xy), int(max_checks)))
        if untraversable_capacity is None:
            return is_safe, traversability_out, area_out
        return is_safe, traversability_out, area_out, untraversable_count, untraversable_xy

    def get_footprint(self):
        """te_map_get_footprint: the traversability_footprint cache (NaN = empty); (nmaps, rows, cols) on a batch."""
        fn = self._L.te_map_get_footprint
        if not self._g:
            self._check(fn(self._h, None, MEM_HOST))
        buf, out = self._layer_out()
        self._check(fn(self._h, _addr(buf), MEM_HOST))
        return out

    def clear_footprint(self):
        """te_map_clear_footprint (resetTraversabilityFootprintLayers)."""
        self._check(self._L.te_map_clear_footprint(self._h))

    def request_stats(self):
        """(candidate checks, distinct circles walked, cache cells stored) of the last request."""
        out = (C.c_int64 * 3)()
        self._check(self._L.te_map_request_stats(self._h, out))
        return tuple(int(v) for v in out)

    def get_layers(self, names, out=None, memory=MEM_HOST):
        """te_map_get_layers (publishTraversabilityMap): dict name -> (rows, cols) layer for `names` (LAYERS entries).  Host
        memory: numpy arrays, re-wrapped to the map's start index.  Device memory: `out` is a float32 device tensor of
        len(names) * rows * cols, filled asynchronously on the context stream in the map's default order; the dict holds views.
        On a batch every layer is (nmaps, rows, cols) (device memory: len(names) * nmaps * rows * cols floats)."""
        mask = layer_mask(names)
        order = [n for k, n in enumerate(LAYERS) if (mask >> k) & 1]
        rows, cols = self._shape() if self._g else (0, 0)
        if memory == MEM_HOST:
            out = np.empty((len(order), self._n, cols, rows), dtype=np.float32)   # per layer the maps back to back, column-major
        self._ctx._order_after_torch(memory)
        self._check(self._L.te_map_get_layers(self._h, mask, _addr(out), memory))
        if self._n == 1:
            v = out.reshape(len(order), cols, rows)
            return {n: v[k].T for k, n in enumerate(order)}
        v = out.reshape(len(order), self._n, cols, rows)
        return {n: v[k].swapaxes(1, 2) for k, n in enumerate(order)}

    def get_submaps(self, positions, lengths, names, out=None, memory=MEM_HOST):
        """te_map_get_submaps (the get_traversability_map service per window): one (info, layers) pair per window, info a
        SUBMAP_INFO_DTYPE record and layers a dict name -> (rows_k, cols_k) submap layer, or None for a failed window.  Host
        memory: numpy arrays (out=None: sized by submap_geometry).  Device memory: `out` is a float32 device tensor with room for
        every window, filled asynchronously on the context stream; the layers are views of it."""
        return self._submaps(None, positions, lengths, names, out, memory)

    def get_submaps_batched(self, win_map, positions, lengths, names, out=None, memory=MEM_HOST):
        """te_map_get_submaps_batched: get_submaps with window k taken from map win_map[k] (int32 per window)."""
        return self._submaps(win_map, positions, lengths, names, out, memory)

    def _submaps(self, win_map, positions, lengths, names, out, memory):
        mask = layer_mask(names)
        order = [n for k, n in enumerate(LAYERS) if (mask >> k) & 1]
        p, ln = _windows(positions, lengths)
        if out is None:
            if memory != MEM_HOST:
                raise ValueError("device memory needs an `out` tensor")
            geo = submap_geometry(self._g, p, ln) if self._g is not None else np.zeros(0, dtype=SUBMAP_INFO_DTYPE)
            out = np.empty(len(order) * int((geo["rows"].astype(np.int64) * geo["cols"]).sum()), dtype=np.float32)
        cap = out.size if isinstance(out, np.ndarray) else out.numel()
        info = np.zeros(len(p), dtype=SUBMAP_INFO_DTYPE)
        self._ctx._order_after_torch(memory)
        if win_map is None:
            fn = self._L.te_map_get_submaps
            self._check(fn(self._h, len(p), p.ctypes.data, ln.ctypes.data, mask, info.ctypes.data, _addr(out), cap, memory))
        else:
            wm = np.ascontiguousarray(win_map, dtype=np.int32).reshape(-1)
            if len(wm) != len(p):
                raise ValueError("win_map needs one entry per window")
            fn = self._L.te_map_get_submaps_batched
            self._check(fn(self._h, len(p), wm.ctypes.data, p.ctypes.data, ln.ctypes.data, mask, info.ctypes.data, _addr(out), cap,
                           memory))
        res = []
        for r in info:
            if not r["success"]:
                res.append((r, None))
                continue
            nr, nc, o = int(r["rows"]), int(r["cols"]), int(r["offset"])
            res.append((r, {n: out[o + k * nr * nc:o + (k + 1) * nr * nc].reshape(nc, nr).T for k, n in enumerate(order)}))
        return res

    def valid_at(self, xy, out=None, memory=MEM_HOST):
        """te_map_valid_at (mapHasValidTraversabilityAt per position): uint8 per (x, y) row of `xy`, 1 where getIndex finds the
        position in the map and traversability is finite there.  Device memory: xy a float64 (n, 2) device tensor and `out` a
        uint8 device tensor of n, filled asynchronously on the context stream."""
        if memory == MEM_HOST:
            xy = np.ascontiguousarray(xy, dtype=np.float64).reshape(-1, 2)
            out = np.zeros(len(xy), dtype=np.uint8)
        self._ctx._order_after_torch(memory)
        self._check(self._L.te_map_valid_at(self._h, len(xy), _addr(xy), _addr(out), memory))
        return out

    def valid_at_batched(self, pos_map, xy, out=None, memory=MEM_HOST):
        """te_map_valid_at_batched: valid_at with position q on map pos_map[q].  Host memory: numpy int32 pos_map (a map outside
        the batch raises).  Device memory: pos_map an int32 device tensor of n (a map outside the batch gives 0), xy and out as in
        valid_at."""
        if memory == MEM_HOST:
            xy = np.ascontiguousarray(xy, dtype=np.float64).reshape(-1, 2)
            pos_map = np.ascontiguousarray(pos_map, dtype=np.int32).reshape(-1)
            if len(pos_map) != len(xy):
                raise ValueError("pos_map needs one entry per position")
            out = np.zeros(len(xy), dtype=np.uint8)
        self._ctx._order_after_torch(memory)
        self._check(self._L.te_map_valid_at_batched(self._h, len(xy), _addr(pos_map), _addr(xy), _addr(out), memory))
        return out
