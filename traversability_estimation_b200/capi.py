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

# te_layer: bit k of a layer mask is LAYERS[k]; outputs that hold several layers have them in bit order.
LAYERS = ("traversability", "traversability_slope", "traversability_step", "traversability_roughness", "elevation", "robot_slope",
          "traversability_footprint")
# The elevation map's layers a te_map carries (Map.carry_layers), bits 8 .. 14 (bit 7 is unassigned), and uncertainty_range (bit
# 15: upper_bound - lower_bound, derived by Map.get_layers).
CARRIED_LAYERS = ("upper_bound", "lower_bound", "variance", "horizontal_variance_x", "horizontal_variance_y", "horizontal_variance_xy",
                  "time")
UNCERTAINTY_RANGE = "uncertainty_range"
# The traversability_footprint service's layers a te_map keeps (Map.footprint_polygon_keep), bits 16 and 17.
POLYGON_LAYERS = ("traversability_x", "traversability_rot")
LAYER_BITS = {**{n: k for k, n in enumerate(LAYERS)}, **{n: 8 + k for k, n in enumerate(CARRIED_LAYERS)}, UNCERTAINTY_RANGE: 15,
              **{n: 16 + k for k, n in enumerate(POLYGON_LAYERS)}}
# The layers isTraversableForFilters memoises its checks in, recorded by a te_map's requests and sweeps, bits 21 .. 23 (18 .. 20
# are unassigned).  Every method that takes layer names takes these too.
FOOTPRINT_MEMO_BITS = {"slope_footprint": 21, "step_footprint": 22, "roughness_footprint": 23}
_ALL_BITS = {**LAYER_BITS, **FOOTPRINT_MEMO_BITS}


def layer_mask(names) -> int:
    """The te_layer mask of layer names (any order; each once)."""
    names = list(names)
    unknown = [n for n in names if n not in _ALL_BITS]
    if unknown or len(set(names)) != len(names):
        raise ValueError(f"layer names {names}: each once, from {tuple(_ALL_BITS)}")
    return sum(1 << _ALL_BITS[n] for n in names)


_layer_mask_of = layer_mask  # for methods whose argument is named layer_mask


def layer_order(mask) -> list:
    """The layer names of a te_layer mask in bit order, the order of every output that holds several."""
    return [n for n, b in sorted(_ALL_BITS.items(), key=lambda x: x[1]) if (mask >> b) & 1]


class SubmapInfo(C.Structure):
    """te_submap_info."""
    _fields_ = [("success", C.c_int32), ("rows", C.c_int32), ("cols", C.c_int32), ("top_row", C.c_int32), ("top_col", C.c_int32),
                ("requested_row", C.c_int32), ("requested_col", C.c_int32), ("reserved", C.c_int32),
                ("length_x", C.c_double), ("length_y", C.c_double), ("position_x", C.c_double), ("position_y", C.c_double),
                ("offset", C.c_int64)]


# te_submap_info as a numpy record, for arrays of them
SUBMAP_INFO_DTYPE = np.dtype([(n, np.dtype(t._type_)) for n, t in SubmapInfo._fields_])
assert SUBMAP_INFO_DTYPE.itemsize == C.sizeof(SubmapInfo)


class OccupancyInfo(C.Structure):
    """te_occupancy_info: an OccupancyGrid's MapMetaData (width = rows, height = cols, origin = position - 0.5 * length)."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("resolution", C.c_float), ("reserved", C.c_int32),
                ("origin_x", C.c_double), ("origin_y", C.c_double)]


OCCUPANCY_INFO_DTYPE = np.dtype([(n, np.dtype(t._type_)) for n, t in OccupancyInfo._fields_])
assert OCCUPANCY_INFO_DTYPE.itemsize == C.sizeof(OccupancyInfo)


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
    "te_get_fixup_cells": (_R, [_P, _I, _U, _P, _P]),
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
    "te_map_chain_maps": (_R, [_P, _G, _CP, _I, _P, _P, _P, _P, _P, _P, _I]),
    "te_map_set_layers_maps": (_R, [_P, _G, _I, _P, _P, _P, _P, _P, _P, _P, _I]),
    "te_map_chain_batched_at": (_R, [_P, _G, _CP, _I, _P, _P, _P, _P, _P, _I, _P]),
    "te_map_set_layers_batched_at": (_R, [_P, _G, _I, _P, _P, _P, _P, _P, _P, _I, _P]),
    "te_map_chain_maps_at": (_R, [_P, _G, _CP, _I, _P, _P, _P, _P, _P, _P, _I, _P]),
    "te_map_set_layers_maps_at": (_R, [_P, _G, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "te_map_positions": (_R, [_P, _P]),
    "te_map_chain_batched_wrapped": (_R, [_P, _G, _CP, _I, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_set_layers_batched_wrapped": (_R, [_P, _G, _I, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_chain_maps_wrapped": (_R, [_P, _G, _CP, _I, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_set_layers_maps_wrapped": (_R, [_P, _G, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_start_indices": (_R, [_P, _P]),
    "te_image_geometry": (_R, [_I, _I, _D, _D, _D, _G]),
    "te_map_chain_image": (_R, [_P, _G, _CP, _I, _I, _P, _L, _L, _D, _D, _P, _P, _P, _P, _I]),
    "te_map_chain_image_maps": (_R, [_P, _G, _CP, _I, _P, _I, _P, _L, _L, _D, _D, _P, _P, _P, _P, _I]),
    "te_map_footprint": (_R, [_P, _FP, _P, _I]),
    "te_map_footprint_maps": (_R, [_P, _FP, _I, _P, _P, _I]),
    "te_map_footprint_polygon": (_R, [_P, _FP, _I, _P, _D, _P, _P, _I]),
    "te_map_footprint_polygon_yaws": (_R, [_P, _FP, _I, _P, _I, _P, _P, _I]),
    "te_map_footprint_polygon_yaws_reduce": (_R, [_P, _FP, _I, _P, _I, _P, _P, _P, _P, _I]),
    "te_map_footprint_polygon_keep": (_R, [_P, _FP, _I, _P, _I, _P, _I, _P, _P, _P, _I]),
    "te_map_check_footprint_request": (_R, [_P, _FP, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_check_footprint_request_batched": (_R, [_P, _FP, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_check_footprint_request_device": (_R, [_P, _FP, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P, _L]),
    "te_map_check_footprint_request_each": (_R, [_P, _FP, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P]),
    "te_map_check_footprint_request_device_each": (_R, [_P, _FP, _P, _I, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _P,
                                                        _L]),
    "te_map_footprint_each": (_R, [_P, _FP, _I, _P, _P, _I]),
    "te_map_get_footprint": (_R, [_P, _P, _I]),
    "te_map_get_memo": (_R, [_P, _P]),
    "te_map_clear_footprint": (_R, [_P]),
    "te_map_request_stats": (_R, [_P, _P]),
    "te_map_carry_layers": (_R, [_P, _I, _P, _U, _P, _I]),
    "te_submap_geometry": (_R, [_G, _I, _P, _P, _P]),
    "te_map_chain_submap": (_R, [_P, _G, _U, _P, _D, _D, _D, _D, _CP, _P, _I]),
    "te_map_chain_windows": (_R, [_P, _G, _G, _U, _P, _I, _P, _P, _CP, _I]),
    "te_map_get_layers": (_R, [_P, _U, _P, _I]),
    "te_map_get_submaps": (_R, [_P, _I, _P, _P, _U, _P, _P, _L, _I]),
    "te_map_get_submaps_batched": (_R, [_P, _I, _P, _P, _P, _U, _P, _P, _L, _I]),
    "te_map_valid_at": (_R, [_P, _I, _P, _P, _I]),
    "te_map_valid_at_batched": (_R, [_P, _I, _P, _P, _P, _I]),
    "te_map_at_poses": (_R, [_P, _P, _I, _P, _I, _P, _U, _P, _P, _I]),
    "te_occupancy_grid_info": (_R, [_G, _I, _P, _P]),
    "te_map_get_occupancy": (_R, [_P, _I, _P, _U, _P, _P, _P, _I]),
    "te_map_get_point_cloud": (_R, [_P, _I, _P, _I, _P, _U, _U, _P, _L, _P, _I]),
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


def occupancy_grid_info(g, positions=None):
    """te_occupancy_grid_info: the MapMetaData of the occupancy grids of maps of geometry `g`, as an array of OCCUPANCY_INFO_DTYPE
    records: one at g's position (positions None), or one per (x, y) row of `positions` (Map.positions() gives a batch's).  Host
    arithmetic, no GPU needed."""
    L = load_library()
    p = None if positions is None else np.ascontiguousarray(positions, dtype=np.float64).reshape(-1, 2)
    n = 1 if p is None else len(p)
    info = np.zeros(n, dtype=OCCUPANCY_INFO_DTYPE)
    rc = L.te_occupancy_grid_info(C.byref(g), n, _addr(p), info.ctypes.data)
    if rc != 0:
        raise TEError(rc, L.te_last_error().decode())
    return info


def point_cloud_fields(fields, point_layer="elevation"):
    """The PointCloud2 layout GridMapRosConverter::toPointCloud gives a cloud of the layers `fields` (names, in message order): one
    float32 field per entry at consecutive 4-byte offsets, the entry equal to point_layer replaced by x, y, z.  Returns the
    (name, offset) pairs and point_step (te_b200.h states the same rule for te_map_get_point_cloud)."""
    names = []
    for f in fields:
        names += ["x", "y", "z"] if f == point_layer else [f]
    return [(n, 4 * k) for k, n in enumerate(names)], 4 * len(names)


def point_cloud_dtype(layout, point_step):
    """The numpy structured dtype of one point of a point_cloud_fields layout: float32 fields at their offsets."""
    return np.dtype({"names": [n for n, _ in layout], "formats": [np.float32] * len(layout), "offsets": [o for _, o in layout],
                     "itemsize": point_step})


IMAGE_MONO8, IMAGE_MONO16 = 0, 1  # te_image encodings


def image_geometry(height, width, resolution, position=(0.0, 0.0)) -> Geometry:
    """te_image_geometry: the geometry initializeFromImage gives a height x width image (GridMap::setGeometry); host arithmetic,
    no GPU needed."""
    L = load_library()
    g = Geometry()
    rc = L.te_image_geometry(int(height), int(width), float(resolution), float(position[0]), float(position[1]), C.byref(g))
    if rc != 0:
        raise TEError(rc, L.te_last_error().decode())
    return g


def _images(images):
    """(array, nmaps, encoding, row_stride_bytes, image_stride_bytes) of uint8 / uint16 images shaped (rows, cols) or (n, rows,
    cols), row-major as an image is.  A view whose pixels are contiguous along each row (sliced, padded) is passed as it is; any
    other layout and a non-native byte order are copied."""
    a = np.asarray(images)
    if a.dtype.kind != "u" or a.dtype.itemsize not in (1, 2) or a.ndim not in (2, 3):
        raise ValueError(f"images: need uint8 or uint16 of shape (rows, cols) or (n, rows, cols), got {a.dtype} {a.shape}")
    if not a.dtype.isnative:
        a = a.astype(a.dtype.newbyteorder("="))
    if (a.strides[-1] != a.itemsize or a.strides[-2] < a.shape[-1] * a.itemsize
            or (a.ndim == 3 and a.strides[0] < a.shape[1] * a.strides[1])):  # also broadcast and reversed views
        a = np.ascontiguousarray(a)
    n = 1 if a.ndim == 2 else a.shape[0]
    return a, n, IMAGE_MONO8 if a.itemsize == 1 else IMAGE_MONO16, a.strides[-2], a.strides[0] if a.ndim == 3 else 0


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

    def fixup_cells(self, tier):
        """The tier-2 (tier=2) or tier-3 (tier=3) work list of the last fused launch as uint32 entries: cell index of the launch
        | do_n << 30 | do_s << 31, chunk padding dropped.  Only the last launch: a host-memory chain pipelined in column chunks
        reports its last chunk."""
        n = C.c_uint32()
        self._check(self._L.te_get_fixup_cells(self._h, tier, 0, None, C.byref(n)))
        out = np.zeros(n.value, dtype=np.uint32)
        self._check(self._L.te_get_fixup_cells(self._h, tier, n.value, out.ctypes.data if n.value else None, C.byref(n)))
        assert n.value == len(out), (n.value, len(out))
        return out

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

    @staticmethod
    def _positions(positions, n):
        """(n, 2) map positions (x, y) as the _at entries read them, or None."""
        if positions is None:
            return None
        xy = np.ascontiguousarray(positions, dtype=np.float64).reshape(-1)
        if xy.size != 2 * n:
            raise ValueError(f"positions: need {n} (x, y) pairs, got {xy.size} values")
        return xy

    def chain_batched(self, g, p, nmaps, elevation, outputs=False, positions=None, start_index=None, memory=MEM_HOST):
        """te_map_chain_batched (computeTraversability for every map): elevation (nmaps, rows, cols); empties every cache.
        outputs=True also returns the four layers as a dict of (nmaps, rows, cols) arrays.  positions (nmaps, 2): map m sits at
        positions[m] instead of g's position (te_map_chain_batched_at).  start_index (nmaps, 2): map m's layers (input and
        output) are in the circular-buffer order of start_index[m] (te_map_chain_batched_wrapped).  memory=MEM_DEVICE: elevation
        is a float32 device tensor of the nmaps maps back to back, each column-major (a batch too large to stage from the host),
        read in place; outputs must then be False."""
        if memory == MEM_HOST:
            e = self._batch_layers(elevation)
        elif outputs:
            raise ValueError("outputs=True copies the layers to host arrays: take them with get_layers in device memory")
        else:
            e = elevation
            self._ctx._order_after_torch(memory)
        out = {k: np.empty((int(nmaps), g.cols, g.rows), dtype=np.float32) for k in ("slope", "step", "roughness", "traversability")} \
            if outputs else {}
        xy = self._positions(positions, int(nmaps))
        args = (self._h, C.byref(g), C.byref(p), int(nmaps), _addr(e),
                *(_addr(out.get(k)) for k in ("slope", "step", "roughness", "traversability")), memory)
        self._update("te_map_chain_batched", args, xy, start_index, int(nmaps))
        self._g, self._n = g, int(nmaps)
        return {k: v.transpose(0, 2, 1) for k, v in out.items()} if outputs else None

    def set_layers(self, g, traversability, slope, step, elevation, roughness=None, robot_slope=None):
        """te_map_set_layers (setTraversabilityMap): empties the cache and the memo."""
        fn = self._L.te_map_set_layers
        lay = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)  # noqa: E731
        t, s, st, r, e, rs = (lay(a) for a in (traversability, slope, step, roughness, elevation, robot_slope))
        self._check(fn(self._h, C.byref(g), _addr(t), _addr(s), _addr(st), _addr(r), _addr(e), _addr(rs), MEM_HOST))
        self._g, self._n = g, 1

    def set_layers_batched(self, g, nmaps, traversability, slope, step, elevation, roughness=None, robot_slope=None, positions=None,
                           start_index=None):
        """te_map_set_layers_batched (setTraversabilityMap for every map): each layer (nmaps, rows, cols); empties every cache and
        memo.  positions (nmaps, 2): map m sits at positions[m] (te_map_set_layers_batched_at).  start_index (nmaps, 2): map m's
        layers are in the circular-buffer order of start_index[m] (te_map_set_layers_batched_wrapped)."""
        t, s, st, r, e, rs = (self._batch_layers(a) for a in (traversability, slope, step, roughness, elevation, robot_slope))
        xy = self._positions(positions, int(nmaps))
        args = (self._h, C.byref(g), int(nmaps), _addr(t), _addr(s), _addr(st), _addr(r), _addr(e), _addr(rs), MEM_HOST)
        self._update("te_map_set_layers_batched", args, xy, start_index, int(nmaps))
        self._g, self._n = g, int(nmaps)

    @staticmethod
    def _map_index(map_index):
        return np.ascontiguousarray(map_index, dtype=np.int32).reshape(-1)

    def chain_maps(self, g, p, map_index, elevation, outputs=False, positions=None, start_index=None):
        """te_map_chain_maps (computeTraversability for the maps map_index of the batch only): elevation (nsel, rows, cols), map
        j of it going to map map_index[j]; empties those maps' caches and keeps every other map as it was.  outputs=True also
        returns the four layers as a dict of (nsel, rows, cols) arrays in map_index order.  positions (nsel, 2): map map_index[j]
        moves to positions[j] (te_map_chain_maps_at).  start_index (nsel, 2): map map_index[j] comes (and its outputs go back)
        in the circular-buffer order of start_index[j] (te_map_chain_maps_wrapped)."""
        idx = self._map_index(map_index)
        e = self._batch_layers(elevation)
        out = {k: np.empty((len(idx), g.cols, g.rows), dtype=np.float32) for k in ("slope", "step", "roughness", "traversability")} \
            if outputs else {}
        xy = self._positions(positions, len(idx))
        args = (self._h, C.byref(g), C.byref(p), len(idx), _addr(idx), _addr(e),
                *(_addr(out.get(k)) for k in ("slope", "step", "roughness", "traversability")), MEM_HOST)
        self._update("te_map_chain_maps", args, xy, start_index, len(idx))
        return {k: v.transpose(0, 2, 1) for k, v in out.items()} if outputs else None

    _CHAIN_OUTPUTS = ("slope", "step", "roughness", "traversability")

    def chain_image(self, g, p, images, min_height, max_height, outputs=False):
        """te_map_chain_image (imageCallback: addLayerFromImage, then computeTraversability): images uint8 (mono8) or uint16 (mono16)
        of shape (rows, cols), or (n, rows, cols) for a batch of n maps.  outputs=True also returns the four layers as a dict, shaped
        as the images."""
        a, n, enc, rs, ims = _images(images)
        out = {k: np.empty((n, g.cols, g.rows), dtype=np.float32) for k in self._CHAIN_OUTPUTS} if outputs else {}
        self._check(self._L.te_map_chain_image(self._h, C.byref(g), C.byref(p), n, enc, _addr(a), rs, ims, float(min_height),
                                               float(max_height), *(_addr(out.get(k)) for k in self._CHAIN_OUTPUTS), MEM_HOST))
        self._g, self._n = g, n
        return {k: (v.transpose(0, 2, 1) if a.ndim == 3 else v[0].T) for k, v in out.items()} if outputs else None

    def chain_image_maps(self, g, p, map_index, images, min_height, max_height, outputs=False):
        """te_map_chain_image_maps (chain_image for the maps map_index of the batch only): images (nsel, rows, cols), image j
        going to map map_index[j]; keeps every other map as it was.  outputs=True also returns the four layers as a dict of
        (nsel, rows, cols) arrays in map_index order."""
        idx = self._map_index(map_index)
        a, _, enc, rs, ims = _images(images)
        out = {k: np.empty((len(idx), g.cols, g.rows), dtype=np.float32) for k in self._CHAIN_OUTPUTS} if outputs else {}
        self._check(self._L.te_map_chain_image_maps(self._h, C.byref(g), C.byref(p), len(idx), _addr(idx), enc, _addr(a), rs, ims,
                                                    float(min_height), float(max_height),
                                                    *(_addr(out.get(k)) for k in self._CHAIN_OUTPUTS), MEM_HOST))
        return {k: v.transpose(0, 2, 1) for k, v in out.items()} if outputs else None

    def set_layers_maps(self, g, map_index, traversability, slope, step, elevation, roughness=None, robot_slope=None, positions=None,
                        start_index=None):
        """te_map_set_layers_maps (setTraversabilityMap for the maps map_index only): each layer (nsel, rows, cols) in map_index
        order; the optional layers must be those the batch holds.  Empties those maps' caches and memos.  positions (nsel, 2): map
        map_index[j] moves to positions[j] (te_map_set_layers_maps_at).  start_index (nsel, 2): map map_index[j]'s layers are in
        the circular-buffer order of start_index[j] (te_map_set_layers_maps_wrapped)."""
        idx = self._map_index(map_index)
        t, s, st, r, e, rs = (self._batch_layers(a) for a in (traversability, slope, step, roughness, elevation, robot_slope))
        xy = self._positions(positions, len(idx))
        args = (self._h, C.byref(g), len(idx), _addr(idx), _addr(t), _addr(s), _addr(st), _addr(r), _addr(e), _addr(rs), MEM_HOST)
        self._update("te_map_set_layers_maps", args, xy, start_index, len(idx))

    def _update(self, entry, args, xy, start_index, n):
        """`entry`, or its _at entry when positions are given, or its _wrapped entry when start indices (n pairs) are given."""
        if start_index is None:
            return self._check(getattr(self._L, entry)(*args) if xy is None else getattr(self._L, entry + "_at")(*args, _addr(xy)))
        si = np.ascontiguousarray(start_index, dtype=np.int32).reshape(-1)
        if si.size != 2 * n:
            raise ValueError(f"start_index: need {n} (row, col) pairs, got {si.size} values")
        self._check(getattr(self._L, entry + "_wrapped")(*args, _addr(xy), _addr(si)))

    def start_indices(self):
        """te_map_start_indices: each map's circular-buffer start index, an (nmaps, 2) int32 array of (row, col)."""
        si = np.empty((self._n, 2), dtype=np.int32)
        self._check(self._L.te_map_start_indices(self._h, _addr(si)))
        return si

    def positions(self):
        """te_map_positions: where the maps sit, an (nmaps, 2) float64 array of (x, y)."""
        xy = np.empty((self._n, 2), dtype=np.float64)
        self._check(self._L.te_map_positions(self._h, _addr(xy)))
        return xy

    def carry_layers(self, names, layers, map_index=None, memory=MEM_HOST):
        """te_map_carry_layers (mapOut = mapIn for the layers the chain does not make): layers[k] becomes the map's layer names[k]
        ("robot_slope" or CARRIED_LAYERS entries, any order); None fills it with 0.0.  Leaves the cache and the memo as they are.
        map_index None: every map; otherwise the maps map_index only, and only layers the batch already holds.  Host memory: numpy
        layers, (rows, cols) for one map or (n, rows, cols) for n maps (the batch, or the selection in map_index order), in the
        map's start index.  Device memory: float32 device tensors of n * rows * cols, each map column-major in default order,
        read asynchronously on the context stream."""
        names, layers = list(names), list(layers)
        if len(names) != len(layers):
            raise ValueError(f"{len(names)} names but {len(layers)} layers")
        mask = layer_mask(names)
        given = dict(zip(names, layers))
        if memory == MEM_HOST:
            def host(a):
                if a is None:
                    return None
                a = np.asarray(a, dtype=np.float32)
                return np.asfortranarray(a) if a.ndim == 2 else self._batch_layers(a)
            given = {n: host(a) for n, a in given.items()}
        else:
            self._ctx._order_after_torch(memory)
        ordered = [given[n] for n in layer_order(mask)]   # the host pointer array holds them in bit order
        ptrs = (C.c_void_p * len(ordered))(*(_addr(a) for a in ordered))
        if map_index is None:
            self._check(self._L.te_map_carry_layers(self._h, 0, None, mask, ptrs, memory))
        else:
            idx = self._map_index(map_index)
            self._check(self._L.te_map_carry_layers(self._h, len(idx), _addr(idx), mask, ptrs, memory))

    def _source(self, layers, memory):
        """(mask, pointer array) of a source map's layers for chain_submap / chain_windows: layers a dict name -> layer, elevation
        and CARRIED_LAYERS entries.  Host memory: numpy (rows, cols) arrays in the source's buffer order (its start index), kept
        alive in the returned tuple.  Device memory: float32 device tensors of rows * cols, column-major in buffer order."""
        mask = layer_mask(list(layers))
        if memory == MEM_HOST:
            given = {n: np.asfortranarray(a, dtype=np.float32) for n, a in layers.items()}
        else:
            given = dict(layers)
            self._ctx._order_after_torch(memory)
        ordered = [given[n] for n in layer_order(mask)]
        return mask, (C.c_void_p * len(ordered))(*(_addr(a) for a in ordered)), ordered

    def chain_submap(self, src_g, layers, position, length, p, memory=MEM_HOST):
        """te_map_chain_submap (requestElevationMap -> setElevationMap -> computeTraversability): getSubmap(position, length) of
        the source map `src_g` (any start index), then the chain on its elevation and its other layers carried.  layers: a dict
        name -> source layer, "elevation" and any CARRIED_LAYERS (see _source).  Returns the window's SubmapInfo; when getSubmap
        fails (info.success == 0) the map is left as it was and nothing is raised, as the reference node skips that update.  The
        map then holds one map of the submap's geometry (start index 0)."""
        mask, ptrs, _keep = self._source(layers, memory)
        info = SubmapInfo()
        info.success = -1   # the library writes the record once every argument is checked
        rc = self._L.te_map_chain_submap(self._h, C.byref(src_g), mask, ptrs, float(position[0]), float(position[1]), float(length[0]),
                                         float(length[1]), C.byref(p), C.byref(info), memory)
        if rc != 0 and info.success != 0:
            self._check(rc)
        if rc == 0:
            self._g = Geometry(info.rows, info.cols, src_g.resolution, info.length_x, info.length_y, info.position_x, info.position_y,
                               0, 0)
            self._n = 1
        return info

    def chain_windows(self, g, src_g, layers, positions, p, map_index=None, memory=MEM_HOST):
        """te_map_chain_windows: one window of g's size per map, cut out of the source map `src_g` at the requested (robot)
        positions (n, 2) and chained, its other layers carried.  layers as in chain_submap.  map_index None reloads the whole batch
        with n maps; otherwise the maps map_index[j] get the window at positions[j] and every other map keeps its state."""
        mask, ptrs, _keep = self._source(layers, memory)
        xy = np.ascontiguousarray(positions, dtype=np.float64).reshape(-1, 2)
        idx = None if map_index is None else self._map_index(map_index)
        if idx is not None and len(idx) != len(xy):
            raise ValueError(f"{len(idx)} map indices but {len(xy)} positions")
        self._check(self._L.te_map_chain_windows(self._h, C.byref(g), C.byref(src_g), mask, ptrs, len(xy), _addr(idx), _addr(xy),
                                                 C.byref(p), memory))
        if idx is None:
            self._g, self._n = g, len(xy)

    def footprint_maps(self, fp, map_index):
        """te_map_footprint_maps (traversabilityFootprint(radius, offset) on the caches of the maps map_index only); returns those
        caches afterwards, (nsel, rows, cols) in map_index order."""
        idx = self._map_index(map_index)
        rows, cols = self._shape() if self._g else (0, 0)
        buf = np.empty((len(idx), cols, rows), dtype=np.float32)
        self._check(self._L.te_map_footprint_maps(self._h, C.byref(fp), len(idx), _addr(idx), _addr(buf), MEM_HOST))
        return buf.transpose(0, 2, 1)

    def _params(self, params):
        """A ctypes array of one FootprintParams per map of the te_map (the _each entries); such an array is passed as it is."""
        if isinstance(params, C.Array):
            if len(params) != self._n:
                raise ValueError(f"{len(params)} parameter sets for a te_map of {self._n} maps: need one per map")
            return params
        params = list(params)
        if len(params) != self._n:
            raise ValueError(f"{len(params)} parameter sets for a te_map of {self._n} maps: need one per map")
        return (FootprintParams * len(params))(*params)

    def footprint_each(self, params, map_index=None, memory=MEM_HOST, out=None):
        """te_map_footprint_each: traversabilityFootprint(radius, offset) on every map's cache (map_index None) or on the maps
        map_index only, map m with params[m] (one FootprintParams per map).  Host memory returns the swept caches afterwards, as
        footprint (whole batch) or footprint_maps (a selection) do; device memory fills `out` (a float32 device tensor of the swept
        maps' cells, or None) asynchronously on the context stream and returns it."""
        arr = self._params(params)
        idx = None if map_index is None else self._map_index(map_index)
        nsel = 0 if idx is None else len(idx)
        fn = self._L.te_map_footprint_each
        if memory != MEM_HOST:
            self._ctx._order_after_torch(memory)
            self._check(fn(self._h, arr, nsel, _addr(idx), _addr(out), memory))
            return out
        if idx is None:
            buf, res = self._layer_out()
        else:
            rows, cols = self._shape()
            buf = np.empty((nsel, cols, rows), dtype=np.float32)
            res = buf.transpose(0, 2, 1)
        self._check(fn(self._h, arr, nsel, _addr(idx), _addr(buf), MEM_HOST))
        return res

    def footprint(self, fp, out=None, memory=MEM_HOST):
        """te_map_footprint (traversabilityFootprint(radius, offset) on the cache); returns the cache afterwards.  Device memory:
        `out` is a float32 device tensor of every map's cells (or None: the cache stays on the device only), filled
        asynchronously on the context stream and returned."""
        fn = self._L.te_map_footprint
        if memory != MEM_HOST:
            self._ctx._order_after_torch(memory)
            self._check(fn(self._h, C.byref(fp), _addr(out), memory))
            return out
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

    def footprint_polygon_keep(self, fp, polygon_xy, yaws, map_index=None, outputs=False, memory=MEM_HOST):
        """te_map_footprint_polygon_keep (the traversability_footprint service, kept on the map): the swept maps (map_index None:
        every map) then hold traversability_x and traversability_rot at their yaws (a scalar for every swept map, or one per swept
        map in map_index order), which get_layers / get_submaps return.  Host memory: outputs=True returns copies of the swept
        maps' new layers (x, rot), each (rows, cols) for one map or (n, rows, cols) for n swept maps, in the map's start index.
        Device memory: outputs is False or a pair of float32 device tensors of n * rows * cols (None for one not wanted), filled
        asynchronously on the context stream in default order and returned."""
        pts = np.ascontiguousarray(polygon_xy, dtype=np.float64).reshape(-1, 2)
        ys = np.ascontiguousarray(yaws, dtype=np.float64).reshape(-1)
        idx = None if map_index is None else self._map_index(map_index)
        n = self._n if idx is None else len(idx)
        res = None
        if memory == MEM_HOST:
            rows, cols = self._shape() if self._g else (0, 0)
            bufs = (np.empty((n, cols, rows), np.float32), np.empty((n, cols, rows), np.float32)) if outputs else (None, None)
            if outputs:
                res = tuple(b.transpose(0, 2, 1)[0] if idx is None and self._n == 1 else b.transpose(0, 2, 1) for b in bufs)
        else:
            self._ctx._order_after_torch(memory)
            bufs = tuple(outputs) if outputs else (None, None)
            res = bufs if outputs else None
        self._check(self._L.te_map_footprint_polygon_keep(self._h, C.byref(fp), 0 if idx is None else len(idx), _addr(idx), len(pts),
                                                          pts.ctypes.data, len(ys), ys.ctypes.data if len(ys) else None,
                                                          _addr(bufs[0]), _addr(bufs[1]), memory))
        return res

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

    def check_footprint_request_each(self, params, path_map, path_begin, poses, radius, footprint_begin, footprint_xyz,
                                     max_footprint_vertices=None, conservative=None, compute_untraversable_polygon=None,
                                     untraversable_capacity=None):
        """te_map_check_footprint_request_each: check_footprint_request_batched with map m's paths checked with params[m] (one
        FootprintParams per map)."""
        return self._request(None, path_begin, poses, radius, footprint_begin, footprint_xyz, max_footprint_vertices, conservative,
                             compute_untraversable_polygon, untraversable_capacity, path_map=path_map, params=params)

    def _request(self, fp, path_begin, poses, radius, footprint_begin, footprint_xyz, max_footprint_vertices, conservative,
                 compute_untraversable_polygon, untraversable_capacity, path_map=None, params=None):
        """The body of check_footprint_request (path_map None), check_footprint_request_batched and check_footprint_request_each
        (params: one set per map instead of fp): the batched entries take path_map after the parameters."""
        batched = path_map is not None
        fn = self._L.te_map_check_footprint_request_batched if batched else self._L.te_map_check_footprint_request
        if params is not None:
            fn = self._L.te_map_check_footprint_request_each
        par = C.byref(fp) if params is None else self._params(params)
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
        self._check(fn(self._h, par, *(a.ctypes.data for a in pm), n, len(ps), pb.ctypes.data, ps.ctypes.data,
                       rad.ctypes.data, len(fxyz), fb.ctypes.data, fxyz.ctypes.data, int(max_footprint_vertices), _addr(cons),
                       _addr(cup), safe.ctypes.data, trav.ctypes.data, area.ctypes.data, maxv, _addr(counts), _addr(uxy)))
        if untraversable_capacity is None:
            return safe, trav, area
        return safe, trav, area, counts, uxy

    def check_footprint_request_device(self, fp, path_begin, poses, radius, footprint_begin, footprint_xyz, is_safe,
                                       traversability_out, area_out, max_checks, path_map=None, max_footprint_vertices=None,
                                       conservative=None, compute_untraversable_polygon=None, untraversable_capacity=None,
                                       untraversable_count=None, untraversable_xy=None, params=None):
        """te_map_check_footprint_request_device: check_footprint_request(_batched) with every argument a device tensor, as
        Context.check_footprint_request(memory=MEM_DEVICE) takes them (path_map int32 per path, None on a map of one map), results
        in the caller's tensors.  Asynchronous: ordered after torch's current stream, no host synchronisation.  max_checks sizes
        the work list of circle checks (te_b200.h).  max_footprint_vertices defaults to 16.  params (a host sequence of one
        FootprintParams per map, fp then unused): te_map_check_footprint_request_device_each."""
        self._ctx._order_after_torch(MEM_DEVICE)
        n = int(path_begin.numel()) - 1
        mfv = 16 if max_footprint_vertices is None else int(max_footprint_vertices)
        maxv = 0 if untraversable_capacity is None else int(untraversable_capacity)
        fn = self._L.te_map_check_footprint_request_device if params is None else self._L.te_map_check_footprint_request_device_each
        par = C.byref(fp) if params is None else self._params(params)
        self._check(fn(
            self._h, par, _addr(path_map), n, int(poses.numel()) // 7, _addr(path_begin), _addr(poses), _addr(radius),
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

    def get_memo(self):
        """te_map_get_memo: the isTraversableForFilters memo bytes (0 not evaluated, 1 passes, 2 blocked), uint8 (rows, cols), or
        (nmaps, rows, cols) on a batch, every map in default order."""
        rows, cols = self._shape()
        buf = np.empty((self._n, cols, rows), dtype=np.uint8)
        self._check(self._L.te_map_get_memo(self._h, buf.ctypes.data))
        out = buf.transpose(0, 2, 1)
        return out[0] if self._n == 1 else out

    def clear_footprint(self):
        """te_map_clear_footprint (resetTraversabilityFootprintLayers)."""
        self._check(self._L.te_map_clear_footprint(self._h))

    def request_stats(self):
        """(candidate checks, distinct circles walked, cache cells stored) of the last request."""
        out = (C.c_int64 * 3)()
        self._check(self._L.te_map_request_stats(self._h, out))
        return tuple(int(v) for v in out)

    def get_layers(self, names, out=None, memory=MEM_HOST):
        """te_map_get_layers (publishTraversabilityMap): dict name -> (rows, cols) layer for `names` (LAYER_BITS entries; the
        carried layers once carry_layers gave them, uncertainty_range = upper_bound - lower_bound computed on the device).  Host
        memory: numpy arrays, re-wrapped to the map's start index.  Device memory: `out` is a float32 device tensor of
        len(names) * rows * cols, filled asynchronously on the context stream in the map's default order; the dict holds views.
        On a batch every layer is (nmaps, rows, cols) (device memory: len(names) * nmaps * rows * cols floats)."""
        mask = layer_mask(names)
        order = layer_order(mask)
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
        order = layer_order(mask)
        p, ln = _windows(positions, lengths)
        if out is None:
            if memory != MEM_HOST:
                raise ValueError("device memory needs an `out` tensor")
            if self._g is None:
                geo = np.zeros(0, dtype=SUBMAP_INFO_DTYPE)
            else:   # each window on its own map's position (te_map_positions: g's unless an _at entry placed the map)
                wm = np.zeros(len(p), np.int64) if win_map is None else np.asarray(win_map, dtype=np.int64).reshape(-1)
                xy = self.positions()
                geo = np.zeros(len(p), dtype=SUBMAP_INFO_DTYPE)
                for m in np.unique(wm) if len(p) else ():
                    if not 0 <= m < self._n:   # the library refuses the call: nothing to size
                        continue
                    gm = Geometry.from_buffer_copy(self._g)
                    gm.position_x, gm.position_y = float(xy[m, 0]), float(xy[m, 1])
                    k = np.nonzero(wm == m)[0]
                    geo[k] = submap_geometry(gm, p[k], ln[k])
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

    def at_poses(self, poses, points, layer_mask, pose_map=None, out=None, valid=None, memory=MEM_HOST):
        """te_map_at_poses (GridMap::atPosition at robot-frame points around poses): returns (layers, valid), layers a dict name ->
        (nposes, npoints) values in te_layer bit order and valid (nposes, npoints) uint8 (1 where the point lies on its pose's
        map; the value is then the cell's, else NaN).  layer_mask: a te_layer mask or layer names.  poses: (nposes, 7) x y z qx qy
        qz qw; points: (npoints, 3) x y z; pose_map: map per pose (None on a map of one map).  Host memory: numpy arguments, out /
        valid allocated when None.  Device memory: poses float64, points float32 and pose_map int32 device tensors, `out` a
        float32 device tensor of nlayers * nposes * npoints and `valid` a uint8 device tensor of nposes * npoints or None, filled
        asynchronously on the context stream; the dict holds views of `out`."""
        mask = int(layer_mask) if isinstance(layer_mask, (int, np.integer)) else _layer_mask_of(layer_mask)
        order = layer_order(mask)
        if memory == MEM_HOST:
            poses = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 7)
            points = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
            if pose_map is not None:
                pose_map = np.ascontiguousarray(pose_map, dtype=np.int32).reshape(-1)
                if len(pose_map) != len(poses):
                    raise ValueError("pose_map needs one entry per pose")
            n, npts = len(poses), len(points)
            if out is None:
                out = np.empty(len(order) * n * npts, dtype=np.float32)
            if valid is None:
                valid = np.empty(n * npts, dtype=np.uint8)
        else:
            n, npts = int(poses.numel()) // 7, int(points.numel()) // 3
        self._ctx._order_after_torch(memory)
        self._check(self._L.te_map_at_poses(self._h, _addr(pose_map), n, _addr(poses), npts, _addr(points), mask, _addr(out),
                                            _addr(valid), memory))
        flat = out.reshape(-1)
        layers = {name: flat[k * n * npts:(k + 1) * n * npts].reshape(n, npts) for k, name in enumerate(order)}
        return layers, (None if valid is None else valid.reshape(n, npts))

    def get_occupancy(self, names, data_min, data_max, maps=None, out=None, memory=MEM_HOST):
        """te_map_get_occupancy (GridMapRosConverter::toOccupancyGrid): dict name -> int8 grid for `names` (LAYER_BITS entries),
        each (height, width) = (cols, rows) in C order, as OccupancyGrid.data reshapes, whatever the map's start index.  data_min /
        data_max: one float for every layer, or one per entry of `names`.  maps None: every map; otherwise the maps `maps` in that
        order.  On a batch, or with `maps`, every grid is (n, cols, rows).  Host memory: numpy arrays.  Device memory: `out` is an
        int8 device tensor of len(names) * n * rows * cols bytes, filled asynchronously on the context stream; the dict holds
        views."""
        names = list(names)
        mask = layer_mask(names)
        order = layer_order(mask)

        def per_layer(v, what):
            a = np.asarray(v, dtype=np.float32)
            if a.ndim == 0:
                return np.full(len(order), a, dtype=np.float32)
            if a.shape != (len(names),):
                raise ValueError(f"{what}: need one float or one per name ({len(names)}), got shape {a.shape}")
            return np.ascontiguousarray([a[names.index(n)] for n in order], dtype=np.float32)   # bit order

        lo, hi = per_layer(data_min, "data_min"), per_layer(data_max, "data_max")
        idx = None if maps is None else self._map_index(maps)
        n = self._n if idx is None else len(idx)
        rows, cols = self._shape() if self._g else (0, 0)
        if memory == MEM_HOST:
            out = np.empty(len(order) * n * rows * cols, dtype=np.int8)
        self._ctx._order_after_torch(memory)
        self._check(self._L.te_map_get_occupancy(self._h, 0 if idx is None else len(idx), _addr(idx), mask, _addr(lo), _addr(hi),
                                                 _addr(out), memory))
        if idx is None and self._n == 1:
            v = out.reshape(len(order), cols, rows)
        else:
            v = out.reshape(len(order), n, cols, rows)
        return {name: v[k] for k, name in enumerate(order)}

    def get_point_cloud(self, fields, point_layer="elevation", basic=(), nan_layers=(), maps=None, capacity=None, out=None,
                        offsets=None, memory=MEM_HOST):
        """te_map_get_point_cloud (GridMapRosConverter::toPointCloud): the clouds of the maps (maps None: every map; otherwise the
        maps `maps` in that order) with one float32 field per name of `fields` (message order), the point layer's entry replaced by
        x, y, z.  A name of `nan_layers` is a field holding NaN 0x7fc00000 (the published map's step_footprint / slope_footprint
        after computeTraversability); every other name is a LAYER_BITS or FOOTPRINT_MEMO_BITS entry (slope_footprint,
        step_footprint and roughness_footprint as the te_map recorded them).  basic: the map's basic layers.  Returns (layout,
        point_step, clouds), layout the (name, offset) pairs of point_cloud_fields.  Host memory: clouds is a list of one numpy
        structured array per map (point_cloud_dtype), in the reference's point order; capacity None sizes the call first, otherwise
        a cloud over `capacity` points raises.  Device memory: `out` a uint8 device tensor (capacity None: all of it) and `offsets`
        an int64 device tensor of n + 1, filled asynchronously on the context stream; clouds is (out, offsets)."""
        fields, nan_layers = list(fields), set(nan_layers)
        if len(set(fields)) != len(fields):
            raise ValueError(f"fields {fields}: each name once")
        bits = []
        for f in fields:
            if f not in nan_layers and f not in _ALL_BITS:
                raise ValueError(f"field {f!r}: neither a layer ({tuple(_ALL_BITS)}) nor one of nan_layers")
            bits.append(0 if f in nan_layers else 1 << _ALL_BITS[f])
        if point_layer not in _ALL_BITS:
            raise ValueError(f"point_layer {point_layer!r}: not a layer of {tuple(_ALL_BITS)}")
        fa = np.ascontiguousarray(bits, dtype=np.uint32)
        layout, step = point_cloud_fields(fields, point_layer)
        idx = None if maps is None else self._map_index(maps)
        n = self._n if idx is None else len(idx)
        fn = self._L.te_map_get_point_cloud
        args = (self._h, 0 if idx is None else len(idx), _addr(idx), len(fa), _addr(fa), 1 << _ALL_BITS[point_layer],
                layer_mask(basic) if len(basic) else 0)
        if memory != MEM_HOST:
            cap = out.numel() // step if capacity is None else int(capacity)
            self._ctx._order_after_torch(memory)
            self._check(fn(*args, _addr(out), cap, _addr(offsets), memory))
            return layout, step, (out, offsets)
        offsets = np.full(n + 1, -1, dtype=np.int64)
        if capacity is None:                      # a sizing call: offsets only
            rc = fn(*args, None, 0, _addr(offsets), memory)
            if rc != 0 and offsets[0] != 0:
                self._check(rc)
            capacity = int(offsets[-1])
        data = np.empty(int(capacity) * step, dtype=np.uint8)
        self._check(fn(*args, _addr(data), int(capacity), _addr(offsets), memory))
        dt = point_cloud_dtype(layout, step)
        return layout, step, [data[offsets[k] * step:offsets[k + 1] * step].view(dt) for k in range(n)]
