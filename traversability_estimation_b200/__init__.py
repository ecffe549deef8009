"""H100-native traversability filter chain + footprint sweep (sm_90a CUDA behind a C ABI).

The product is `libte_b200.so` (include/te_b200.h); its reference-facing host side are the C++
filter plugin shells in `plugin/`.  This Python module is only a ctypes view of the same C ABI for
tests, `bench.py` and multi-process launch via torch.distributed — it adds no compute of its own
and there is no CPU fallback: loading fails loudly when the library is missing.
"""
from .capi import (ChainParams, Context, FootprintParams, Geometry, HaloPeer, Map, Slab, TEError,  # noqa: F401
                   KERNEL_AUTO, KERNEL_FUSED, KERNEL_GENERIC, MEM_DEVICE, MEM_HOST, build_library,
                   library_path, load_library)
