"""Properties of the recorded slope_footprint / step_footprint / roughness_footprint oracle (tests/memo_layers_oracle.cpp)."""
import numpy as np

import memo_layers_oracle as mo
import synth
from helpers import chain_layers, footprint_params, mixed_request, request_footprints
from oracle import binding as ob


def _map(rows=96, cols=80, res=0.02, seed=71):
    z = synth.terrain(rows, cols, res, seed, "mixed", (0.0, 0.0))
    og = ob.Geometry.make(rows, cols, res, (0.0, 0.0))
    L, rs = chain_layers(ob, og, z, seed)
    return og, L, rs


def _fp(verify, **kw):
    return footprint_params(ob, ob, verify, **kw)[1]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def test_sweep_on_empty_cache_is_the_predicate_layers():
    og, L, _ = _map()
    for verify in (0, 1):
        fo = _fp(verify)
        s = mo.State(og, L)
        s.sweep(fo)
        ref = ob.footprint(og, fo, L["traversability"], L["slope"], L["step"], L["elevation"], roughness=L["roughness"])
        for name, want in zip(mo.NAMES, ref[1:]):
            got = s.memo[name]
            assert np.array_equal(np.isnan(got), np.isnan(want)), (verify, name)
            assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]), (verify, name)


def test_request_writes_inside_visited_cells_only():
    og, L, rs = _map(seed=72)
    fo = _fp(1)
    rng = np.random.default_rng(3)
    fps = request_footprints(rng)
    R = mixed_request(rng, og, 40, fps, circular=0.6, cap_path=False)
    s = mo.State(og, dict(L, robot_slope=rs))
    s.request(fo, R, fps)
    written = ~np.isnan(s.memo["slope_footprint"]) | ~np.isnan(s.memo["step_footprint"]) | ~np.isnan(s.memo["roughness_footprint"])
    assert written.any() and not written.all()
    # a layer is written only where its input layer is exactly 0
    for name, key in zip(mo.NAMES, ("slope", "step", "roughness")):
        w = ~np.isnan(s.memo[name])
        assert (L[key][w] == 0.0).all(), name
        assert np.isin(s.memo[name][w], (0.0, 1.0)).all(), name
    # every walked centre is visited: a centre the request stored a value at, whose own layer is 0, holds its slope record
    walked = ~np.isnan(s.cache) & (L["slope"] == 0.0)
    assert (~np.isnan(s.memo["slope_footprint"][walked])).all()
    # a fresh sweep's layers hold every cell the request wrote, with the same values
    full = mo.State(og, L)
    full.sweep(fo)
    for name in mo.NAMES:
        w = ~np.isnan(s.memo[name])
        assert np.array_equal(s.memo[name][w], full.memo[name][w]), name


def test_clear_keeps_roughness():
    og, L, _ = _map(seed=73)
    fo = _fp(1)
    s = mo.State(og, L)
    s.sweep(fo)
    assert not np.isnan(s.memo["roughness_footprint"]).all()
    rough = s.memo["roughness_footprint"].copy()
    s.clear()
    assert np.isnan(s.memo["slope_footprint"]).all() and np.isnan(s.memo["step_footprint"]).all()
    assert np.array_equal(_bits(s.memo["roughness_footprint"]), _bits(rough))
