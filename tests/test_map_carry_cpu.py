"""The carried layers' names and bits in the ctypes view, without a GPU."""
import ctypes as C

import pytest


def test_carried_layer_bits(te):
    capi = te.capi
    assert capi.layer_mask(capi.CARRIED_LAYERS) == 0x7f00                      # TE_LAYER_CARRIED
    assert capi.layer_mask(["upper_bound", "lower_bound"]) == 0x300
    assert capi.layer_mask(["time", "robot_slope"]) == 0x4020
    assert capi.layer_mask([capi.UNCERTAINTY_RANGE]) == 0x8000
    assert 7 not in capi.LAYER_BITS.values()                                   # 1 << 7 stays unassigned
    assert capi.layer_order(0xffff & ~0x80) == list(capi.LAYERS) + list(capi.CARRIED_LAYERS) + ["uncertainty_range"]
    assert capi.layer_order(capi.layer_mask(["uncertainty_range", "elevation", "variance"])) == ["elevation", "variance",
                                                                                                 "uncertainty_range"]
    for names in (["upper_bound", "upper_bound"], ["uncertainty"], ["surface_normal_x"]):
        with pytest.raises(ValueError):
            capi.layer_mask(names)


def test_carry_without_a_map(te):
    L = te.load_library()
    ptrs = (C.c_void_p * 1)(None)
    assert L.te_map_carry_layers(None, 0, None, 0x100, ptrs, 0) == -1
