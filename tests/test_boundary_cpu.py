"""The drop-in boundary without a GPU: the C-ABI library loads and exports what include/te_b200.h declares,
fails loudly when no CUDA device exists, and the C++ plugin shells validate parameters like the reference."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "traversability_estimation_b200", "plugin")


def _declared():
    src = open(os.path.join(ROOT, "include", "te_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b(?:int|const char\*)\s+(te_[a-z0-9_]+)\s*\(", src)
    assert len(names) >= 18
    return names


def test_library_exports_every_declared_symbol(te):
    lib = te.load_library()
    missing = [n for n in _declared() if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.te_abi_version() == 1
    assert set(te.capi.EXPORTS) <= set(_declared())


@pytest.mark.parametrize("rows,cols,nmaps,sms", [(8192, 8192, 1, 148), (2048, 2048, 1, 148), (4096, 4096, 1, 148), (512, 512, 256, 148),
                                                  (192, 160, 1, 148), (60, 7, 1, 148), (8192, 2052, 1, 148), (1000, 333, 3, 132),
                                                  (8192, 1024, 1, 148), (8192, 4096, 1, 148), (8192, 6000, 1, 148), (16384, 16384, 1, 148)])
def test_fused_work_units_tile_every_map_exactly_once(te, rows, cols, nmaps, sms):
    """The fused kernel's queue of (level, map, segment, strip) units — decoded here the way the kernel decodes a unit id —
    covers every (map, strip, column) once, hands out longer segments first and ends on the unit count it reports."""
    import numpy as np
    plan = te.capi.fused_plan(rows, cols, nmaps, sms)
    strips, levels = plan["strips"], plan["levels"]
    assert strips == (rows + 59) // 60
    cover = np.zeros((nmaps, strips, cols), dtype=np.int32)
    unit = 0
    col_ends = [lv["col0"] for lv in levels[1:]] + [cols]
    lens = []
    for lv, c1 in zip(levels, col_ends):
        assert lv["unit0"] == unit
        upm = strips * lv["nseg"]
        for u in range(upm * nmaps):
            mapi, um = divmod(u, upm)
            seg, strip = divmod(um, strips)
            q0 = lv["col0"] + seg * lv["seg_len"]
            q1 = min(q0 + lv["seg_len"], c1)
            assert q0 < q1 <= cols
            cover[mapi, strip, q0:q1] += 1
        unit += upm * nmaps
        if lv["nseg"]:
            lens.append(lv["seg_len"])
    assert unit == plan["units"]
    assert (cover == 1).all()
    assert lens == sorted(lens, reverse=True) and min(lens) >= 8


def test_fused_plan_shapes_of_the_bench_configurations(te):
    """What plan_levels decides on an H100 (132 SMs x 12 warps) for the sizes the bench lines are quoted on: one long unit per
    warp first for the big single map, one round of one segment length for small launches, the tapering plan in between."""
    big = te.capi.fused_plan(8192, 8192, 1, 132)["levels"]
    assert (big[0]["seg_len"], big[0]["nseg"]) == (552, 11) and big[1]["seg_len"] == 24 and big[2]["seg_len"] == 16
    assert 137 * 11 <= 132 * 12                                    # at most one long unit per warp
    slab = te.capi.fused_plan(8192, 1024, 1, 132)
    assert slab["levels"][0]["seg_len"] == 96 and slab["units"] == 137 * 11 <= 132 * 12   # one round
    small = te.capi.fused_plan(2048, 2048, 1, 132)
    assert small["levels"][0]["seg_len"] == 48 and small["units"] <= 132 * 12
    batch = te.capi.fused_plan(512, 512, 256, 132)["levels"]
    assert batch[0]["seg_len"] == 96 and batch[1]["seg_len"] == 32  # many rounds: long segments first, short ones last


def test_fused_plan_rejects_bad_sizes(te):
    with pytest.raises(te.TEError):
        te.capi.fused_plan(0, 16)


def test_no_cpu_fallback(te):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(te.TEError) as e:
        te.Context(0)
    assert e.value.code == -3 and "no CPU fallback" in str(e.value)


def test_argument_validation_messages(te):
    lib = te.load_library()
    lib.te_last_error.restype = ctypes.c_char_p
    assert lib.te_create(None, 0) == -1
    assert b"null" in lib.te_last_error()
    assert lib.te_synchronize(None) == -1


def _harness():
    subprocess.check_call(["make", "-C", PLUGIN, "-s"])
    return os.path.join(PLUGIN, "test_plugins")


def test_plugin_configure_matches_reference_validation():
    r = subprocess.run([_harness(), "configure"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("PASS") >= 16 and "FAIL" not in r.stdout
    # the reference's own error strings (SlopeFilter.cpp:42, StepFilter.cpp:85)
    assert "Critical slope must be in the interval [0, PI/2]" in r.stderr


def test_plugin_update_fails_loudly_without_gpu():
    r = subprocess.run([_harness(), "nogpu"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "FAIL" not in r.stdout


def test_manifest_names_the_reference_plugins():
    xml = open(os.path.join(PLUGIN, "filter_plugins.xml")).read()
    for n in ("SlopeFilter", "StepFilter", "RoughnessFilter"):
        assert f'name="traversabilityFilters/{n}"' in xml
        assert f'type="filters::{n}<grid_map::GridMap>"' in xml
    assert xml.count('base_class_type="filters::FilterBase<grid_map::GridMap>"') == 4
    assert 'path="lib/libtraversability_estimation_filters"' in xml
