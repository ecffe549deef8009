"""te_submap_geometry without a GPU: GridMap::getSubmap's geometry, bit for bit against the CPU oracle (tests/submap_oracle.cpp),
and its argument errors."""
import ctypes as C

import numpy as np
import pytest

import submap_oracle as so

MAPS = [  # rows, cols, resolution, position, start index
    (200, 180, 0.02, (0.0, 0.0), (0, 0)),
    (97, 131, 0.05, (1.2345, -7.891), (13, 100)),
    (64, 64, 0.1, (-3.3, 2.7), (63, 1)),
    (1, 5, 0.04, (0.01, 0.0), (0, 4)),
]


def _maps(te, oracle):
    for rows, cols, res, pos, (sr, sc) in MAPS:
        g = te.Geometry.make(rows, cols, res, pos)
        g.start_row, g.start_col = sr, sc
        yield g, oracle.Geometry.make(rows, cols, res, pos)


def _windows(rng, g, n):
    """Centres inside, exactly on cell centres and edges, and outside; lengths of 0, below one cell, exact multiples of the
    resolution, 2.5 * res (checkForStep's window) and larger than the map."""
    res, L = g.resolution, np.array([g.length_x, g.length_y])
    P = np.array([g.position_x, g.position_y])
    i = rng.integers(0, g.rows, n)
    j = rng.integers(0, g.cols, n)
    cx = (g.position_x + (0.5 * g.length_x - 0.5 * res)) + res * (-i.astype(np.float64))   # grid_map cell centres
    cy = (g.position_y + (0.5 * g.length_y - 0.5 * res)) + res * (-j.astype(np.float64))
    kind = rng.integers(0, 4, n)
    pos = np.stack([cx, cy], 1)
    pos[kind == 1] += 0.5 * res * rng.choice([-1.0, 1.0], ((kind == 1).sum(), 2))                # cell edges
    pos[kind == 2] = P + rng.uniform(-0.5, 0.5, ((kind == 2).sum(), 2)) * L                     # anywhere inside
    pos[kind == 3] = P + rng.uniform(-0.9, 0.9, ((kind == 3).sum(), 2)) * L                     # often outside
    lk = rng.integers(0, 5, (n, 2))
    length = np.where(lk == 0, 0.0, np.where(lk == 1, rng.uniform(0, res, (n, 2)),
                      np.where(lk == 2, rng.integers(1, 40, (n, 2)) * res,
                               np.where(lk == 3, 2.5 * res, rng.uniform(1.0, 2.5, (n, 2)) * L))))
    return pos, length


def _same_records(got, want):
    for f in so.FIELDS:
        a, b = got[f], want[f]
        if f.startswith(("length", "position")):
            assert np.array_equal(a.astype(np.float64).view(np.uint64), b.view(np.uint64)), f
        else:
            assert np.array_equal(a.astype(np.int64), b), (f, np.nonzero(a != b)[0][:10])


def test_submap_geometry_matches_oracle_bit_for_bit(te, oracle):
    rng = np.random.default_rng(5)
    total = 0
    for g, og in _maps(te, oracle):
        pos, length = _windows(rng, g, 4000)
        got = te.capi.submap_geometry(g, pos, length)
        _same_records(got, so.submap_geometry(og, pos, length))
        # offsets count one layer per window; failed windows take no space and are all zeros otherwise
        size = got["rows"].astype(np.int64) * got["cols"]
        assert np.array_equal(got["offset"], np.concatenate([[0], np.cumsum(size)[:-1]]))
        bad = got["success"] == 0
        assert all((got[f][bad] == 0).all() for f in so.FIELDS)
        assert 0 < bad.sum() < len(bad) and (got["rows"][~bad] >= 1).all()
        # the circular-buffer start index changes nothing
        g0 = te.Geometry.make(g.rows, g.cols, g.resolution, (g.position_x, g.position_y))
        assert got.tobytes() == te.capi.submap_geometry(g0, pos, length).tobytes()
        total += len(pos)
    assert total >= 10000


def test_check_step_window_is_the_three_by_three_neighbourhood(te, oracle):
    """getSubmap(cell centre, 2.5 * res) is the 3 x 3 block around the cell, clipped at the map's edges (SURVEY.md A.1)."""
    g = te.Geometry.make(40, 30, 0.02, (0.1, -0.2))
    i, j = np.meshgrid(np.arange(40), np.arange(30), indexing="ij")
    i, j = i.ravel(), j.ravel()
    cx = (g.position_x + (0.5 * g.length_x - 0.5 * g.resolution)) + g.resolution * (-i.astype(np.float64))
    cy = (g.position_y + (0.5 * g.length_y - 0.5 * g.resolution)) + g.resolution * (-j.astype(np.float64))
    got = te.capi.submap_geometry(g, np.stack([cx, cy], 1), np.full((len(i), 2), 2.5 * g.resolution))
    assert (got["success"] == 1).all()
    assert np.array_equal(got["top_row"], np.maximum(i - 1, 0)) and np.array_equal(got["top_col"], np.maximum(j - 1, 0))
    assert np.array_equal(got["top_row"] + got["rows"], np.minimum(i + 2, 40))
    assert np.array_equal(got["top_col"] + got["cols"], np.minimum(j + 2, 30))
    assert np.array_equal(got["top_row"] + got["requested_row"], i) and np.array_equal(got["top_col"] + got["requested_col"], j)
    _same_records(got, so.submap_geometry(oracle.Geometry.make(40, 30, 0.02, (0.1, -0.2)), np.stack([cx, cy], 1),
                                          np.full((len(i), 2), 2.5 * g.resolution)))


@pytest.mark.parametrize("pos,length", [((0.0, np.nan), (1.0, 1.0)), ((np.inf, 0.0), (1.0, 1.0)), ((0.0, 0.0), (-0.01, 1.0)),
                                        ((0.0, 0.0), (1.0, np.nan)), ((0.0, 0.0), (np.inf, 1.0)), ((0.0, 0.0), (1.0, -np.inf))])
def test_submap_geometry_rejects_bad_windows_before_writing(te, pos, length):
    g = te.Geometry.make(50, 50, 0.02)
    L = te.load_library()
    p = np.array([[0.1, 0.1], pos], dtype=np.float64)
    ln = np.array([[0.2, 0.2], length], dtype=np.float64)
    info = np.full(2, 7, dtype=te.capi.SUBMAP_INFO_DTYPE)
    L.te_submap_geometry.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    assert L.te_submap_geometry(C.byref(g), 2, p.ctypes.data, ln.ctypes.data, info.ctypes.data) == -1
    assert (info["rows"] == 7).all() and (info["offset"] == 7).all()   # nothing written
    with pytest.raises(te.TEError) as e:
        te.capi.submap_geometry(g, p, ln)
    assert e.value.code == -1


def test_submap_geometry_argument_errors(te):
    L = te.load_library()
    L.te_submap_geometry.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    g = te.Geometry.make(50, 50, 0.02)
    p = np.zeros(2)
    info = np.zeros(1, dtype=te.capi.SUBMAP_INFO_DTYPE)
    assert L.te_submap_geometry(C.byref(g), -1, p.ctypes.data, p.ctypes.data, info.ctypes.data) == -1
    assert L.te_submap_geometry(C.byref(g), 1, None, p.ctypes.data, info.ctypes.data) == -1
    assert L.te_submap_geometry(C.byref(g), 1, p.ctypes.data, p.ctypes.data, None) == -1
    assert L.te_submap_geometry(None, 1, p.ctypes.data, p.ctypes.data, info.ctypes.data) == -1
    assert L.te_submap_geometry(C.byref(g), 0, None, None, None) == 0
    bad = te.Geometry.make(50, 50, 0.02)
    bad.start_row = 50                                   # start index outside the map
    assert L.te_submap_geometry(C.byref(bad), 1, p.ctypes.data, p.ctypes.data, info.ctypes.data) == -1
    with pytest.raises(ValueError):
        te.capi.submap_geometry(g, np.zeros((2, 2)), np.zeros((3, 2)))


def test_layer_mask_and_map_entries_without_a_map(te):
    assert te.capi.layer_mask(te.capi.LAYERS) == 0x7f
    assert te.capi.layer_mask(["elevation", "traversability"]) == 0x11
    for names in (["traversability", "traversability"], ["surface_normal_x"]):
        with pytest.raises(ValueError):
            te.capi.layer_mask(names)
    L = te.load_library()
    L.te_map_get_layers.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int]
    L.te_map_valid_at.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int]
    assert L.te_map_get_layers(None, 1, None, 0) == -1
    assert L.te_map_valid_at(None, 0, None, None, 0) == -1
