"""ctypes view of point_cloud_oracle.cpp (test infrastructure): GridMapRosConverter::toPointCloud on the CPU, and an independent
numpy restatement of it.  Layers are (rows, cols) arrays in the buffer order of a start index, as a GridMap message holds them."""
from __future__ import annotations

import ctypes as C

import numpy as np

import cpp_oracle

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cpp_oracle.load("point_cloud_oracle")
        L.teo_point_cloud.restype = C.c_longlong
        L.teo_point_cloud.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                                      C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def point_cloud(layers, fields, point_layer, resolution, length, position, basic=(), nan_layers=(), start=(0, 0)):
    """PointCloud2.data (uint8) and width of toPointCloud(map, fields, point_layer) on one map: layers, a dict name -> (rows, cols)
    float32 array in the buffer order of `start`, must hold every field not in nan_layers, the point layer and the basic layers."""
    lay = {n: np.asfortranarray(a, dtype=np.float32) for n, a in layers.items()}
    rows, cols = lay[point_layer].shape
    fields = list(fields)
    pe = fields.index(point_layer) if point_layer in fields else -1
    ptrs = (C.c_void_p * len(fields))(*[None if (f in nan_layers or k == pe) else lay[f].ctypes.data for k, f in enumerate(fields)])
    bptr = (C.c_void_p * max(1, len(basic)))(*[lay[b].ctypes.data for b in basic])
    words = len(fields) + (2 if pe >= 0 else 0)
    out = np.zeros(rows * cols * words, dtype=np.uint32)
    n = lib().teo_point_cloud(rows, cols, int(start[0]), int(start[1]), float(resolution), float(length[0]), float(length[1]),
                              float(position[0]), float(position[1]), len(fields), ptrs, pe, lay[point_layer].ctypes.data,
                              len(basic), bptr, out.ctypes.data)
    assert n >= 0
    return out[:n * words].view(np.uint8).copy(), int(n)


def point_cloud_numpy(layers, fields, point_layer, resolution, length, position, basic=(), nan_layers=(), start=(0, 0)):
    """The same, restated with numpy: a validity mask over the buffer-order cells, positions from the unwrapped indices, records
    assembled as columns of 4-byte words."""
    lay = {n: np.asarray(a, dtype=np.float32) for n, a in layers.items()}
    rows, cols = lay[point_layer].shape
    flat = {n: a.reshape(-1, order="F") for n, a in lay.items()}
    ok = np.isfinite(flat[point_layer])
    for b in basic:
        ok &= np.isfinite(flat[b])
    k = np.nonzero(ok)[0]
    i, j = k % rows, k // rows
    u = (i - start[0]) % rows
    v = (j - start[1]) % cols
    x = (position[0] + (0.5 * length[0] - 0.5 * resolution)) + resolution * (-u.astype(np.float64))
    y = (position[1] + (0.5 * length[1] - 0.5 * resolution)) + resolution * (-v.astype(np.float64))
    cols_out = []
    for f in fields:
        if f == point_layer:
            cols_out += [x.astype(np.float32).view(np.uint32), y.astype(np.float32).view(np.uint32), flat[f][k].view(np.uint32)]
        elif f in nan_layers:
            cols_out.append(np.full(len(k), 0x7fc00000, np.uint32))
        else:
            cols_out.append(flat[f][k].view(np.uint32))
    rec = np.stack(cols_out, axis=1) if cols_out else np.zeros((len(k), 0), np.uint32)
    return np.ascontiguousarray(rec).view(np.uint8).reshape(-1), len(k)


# The layers of the reference's published traversability map, in message order, as the fixture bag holds them (no basic layers);
# the three footprint layers are all NaN 0x7fc00000 after computeTraversability.
PUBLISHED = ["upper_bound", "lower_bound", "uncertainty_range", "elevation", "traversability_slope", "traversability_step",
             "traversability_roughness", "traversability", "step_footprint", "slope_footprint", "traversability_footprint"]
MEMO_LAYERS = ("step_footprint", "slope_footprint")


def fixture_bag(tmp_dir):
    """The grid_map_msgs/GridMap message of tests/golden/elevation_map.bag.xz, decoded into tmp_dir."""
    import lzma
    import os
    from bag import read_gridmap_bag
    raw = lzma.open(os.path.join(cpp_oracle.HERE, "golden", "elevation_map.bag.xz")).read()
    path = os.path.join(str(tmp_dir), "elevation_map.bag")
    with open(path, "wb") as f:
        f.write(raw)
    return read_gridmap_bag(path)
