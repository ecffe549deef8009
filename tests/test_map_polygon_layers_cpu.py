"""traversability_x / traversability_rot as te_map layers in the ctypes view, without a GPU."""
import ctypes as C


def test_polygon_layer_bits(te):
    capi = te.capi
    assert capi.POLYGON_LAYERS == ("traversability_x", "traversability_rot")
    assert capi.LAYER_BITS["traversability_x"] == 16 and capi.LAYER_BITS["traversability_rot"] == 17
    assert capi.layer_mask(capi.POLYGON_LAYERS) == 0x30000
    assert capi.layer_mask(["traversability_rot", "elevation"]) == 0x20010
    assert 7 not in capi.LAYER_BITS.values()                                   # 1 << 7 stays unassigned
    assert sorted(capi.LAYER_BITS.values()) == [b for b in range(18) if b != 7]


def test_polygon_layers_come_after_uncertainty_range(te):
    capi = te.capi
    every = capi.layer_mask(list(capi.LAYER_BITS))
    assert every == 0x3ff7f
    assert capi.layer_order(every) == list(capi.LAYERS) + list(capi.CARRIED_LAYERS) + ["uncertainty_range", "traversability_x",
                                                                                       "traversability_rot"]
    assert capi.layer_order(capi.layer_mask(["traversability_rot", "uncertainty_range", "traversability"])) == [
        "traversability", "uncertainty_range", "traversability_rot"]


def test_keep_without_a_map(te):
    L = te.load_library()
    fp = te.FootprintParams.yaml_defaults()
    pts = (C.c_double * 8)(0.45, 0.3, 0.45, -0.3, -0.45, -0.3, -0.45, 0.3)
    yaw = (C.c_double * 1)(0.5)
    assert L.te_map_footprint_polygon_keep(None, C.byref(fp), 0, None, 4, pts, 1, yaw, None, None, te.MEM_HOST) == -1
