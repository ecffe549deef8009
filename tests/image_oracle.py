"""ctypes view of image_oracle.cpp (test infrastructure): initializeFromImage's geometry and addLayerFromImage's elevation for
mono8 / mono16 images on the CPU.  Compiled on first use into a temporary directory (the source tree may be read-only), without
contraction."""
from __future__ import annotations

import ctypes as C

import numpy as np

import cpp_oracle

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cpp_oracle.load("image_oracle")
        L.teo_image_geometry.argtypes = [C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_void_p]
        L.teo_image_geometry.restype = None
        L.teo_image_layer.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_void_p]
        L.teo_image_layer.restype = None
        _lib = L
    return _lib


def image_geometry(height, width, resolution, position=(0.0, 0.0)):
    """dict rows, cols (int), length_x, length_y, position_x, position_y (float)."""
    out = np.zeros(6, dtype=np.float64)
    lib().teo_image_geometry(int(height), int(width), float(resolution), float(position[0]), float(position[1]), out.ctypes.data)
    return dict(rows=int(out[0]), cols=int(out[1]), length_x=out[2], length_y=out[3], position_x=out[4], position_y=out[5])


def elevation(images, min_height, max_height):
    """The elevation layer(s) of uint8 / uint16 images (rows, cols) or (n, rows, cols), as (rows, cols) / (n, rows, cols) float32."""
    a = np.asarray(images)
    assert a.dtype in (np.uint8, np.uint16) and a.ndim in (2, 3)
    batch = a.reshape((-1,) + a.shape[-2:])
    out = np.empty((len(batch), a.shape[-1], a.shape[-2]), dtype=np.float32)  # per image: cols x rows, i.e. column-major
    for k, im in enumerate(batch):
        im = np.ascontiguousarray(im)
        lib().teo_image_layer(im.itemsize, im.ctypes.data, im.shape[0], im.shape[1], im.strides[0], float(min_height),
                              float(max_height), out[k].ctypes.data)
    out = out.transpose(0, 2, 1)
    return out if a.ndim == 3 else out[0]
