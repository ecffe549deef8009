"""Helpers shared by the te_map tests: closing the te_maps a test opens, snapshots of what a te_map holds, requests on a te_map, and
the submap windows of the GetGridMap tests."""
import numpy as np
import pytest

import paths_oracle as po
import submap_oracle as so
from helpers import assert_same_answers, assert_same_bits, footprint_arrays, same, same_polygons, subset

CAP = 64             # untraversable_capacity of the requests
MISSING_LAYER = -2   # te_b200.h TE_ERR_MISSING_LAYER


@pytest.fixture(autouse=True)
def close_maps(ctx, monkeypatch):
    """Every te_map a test opens is destroyed when it ends, failed or not, while the context still exists.  A test module
    imports it by name."""
    made, real = [], ctx.map
    monkeypatch.setattr(ctx, "map", lambda: made.append(real()) or made[-1])
    yield
    for m in made:
        m.close()


# ---- what a te_map holds ----------------------------------------------------------------------------------------------------

def all_layer_names(te):
    """Every layer name te_map_get_layers knows."""
    return list(te.capi.LAYERS) + list(te.capi.CARRIED_LAYERS) + [te.capi.UNCERTAINTY_RANGE] + list(te.capi.POLYGON_LAYERS)


def held(te, m, names=None, polygon=False, positions=False):
    """Every layer the te_map holds and its cache: (nmaps, rows, cols) arrays on a batch, (rows, cols) on one map.  names: the
    layers to read, all of which it must hold; None probes the chain and carried layers (and the polygon layers when `polygon`),
    for which the only error allowed is a missing layer.  positions: also the maps' positions."""
    if names is None:
        names = []
        for n in te.capi.LAYERS[:6] + te.capi.CARRIED_LAYERS + (te.capi.POLYGON_LAYERS if polygon else ()):
            try:
                m.get_layers([n])
                names.append(n)
            except te.TEError as e:
                assert e.code == MISSING_LAYER
    h = dict(m.get_layers(list(names)), cache=m.get_footprint())
    if positions:
        h["positions"] = m.positions()
    return h


def assert_same_held(a, b, what=""):
    """Two held snapshots: the same layers, each bit for bit, and the same positions."""
    assert set(a) == set(b), (what, sorted(set(a) ^ set(b)))
    for n in a:
        if n == "positions":
            assert np.array_equal(a[n], b[n]), what
        else:
            assert_same_bits(a[n], b[n], (what, n))


def assert_same_cache(a, b, what="cache", nan_bits=True):
    """Caches bit for bit; nan_bits=False lets any NaN match any NaN (the oracle's empty cell is not the library's NaN)."""
    equal = (a.view(np.uint32) == b.view(np.uint32)) | (not nan_bits and (np.isnan(a) & np.isnan(b)))
    assert equal.all(), (what, int(np.sum(~equal)))


# ---- requests ---------------------------------------------------------------------------------------------------------------

def ask(m, ft, R, path_map=None):
    """R (footprints R["fps"]) on te_map m: check_footprint_request, or check_footprint_request_batched with path_map."""
    fb, fx = footprint_arrays(R, R["fps"])
    kw = dict(max_footprint_vertices=16, conservative=R["cons"], compute_untraversable_polygon=R["cup"], untraversable_capacity=CAP)
    if path_map is None:
        return m.check_footprint_request(ft, R["begin"], R["poses"], R["radius"], fb, fx, **kw)
    return m.check_footprint_request_batched(ft, path_map, R["begin"], R["poses"], R["radius"], fb, fx, **kw)


def assert_batch_matches_singles(b, singles, ft, R, oracle_state=None):
    """One request on the batch b (path_map R["map"]) and, map by map, its paths on the single maps: answers, polygons and every
    cache identical.  oracle_state = (og, fo, per-map layers, per-map caches): each map's paths are also replayed on the CPU
    oracle, whose caches they update.  Returns the batch's answers."""
    got = ask(b, ft, R, R["map"])
    n = len(R["kind"])
    want = [np.zeros(n, np.uint8), np.zeros(n), np.zeros(n), np.zeros(n, np.int32), np.zeros((n, CAP, 2))]
    for k, s in enumerate(singles):
        idx = np.nonzero(R["map"] == k)[0]
        if not len(idx):
            continue
        Rk = subset(R, idx)
        for o, v in zip(want, ask(s, ft, Rk)):
            o[idx] = v
        if oracle_state is not None:
            og, fo, OL, caches = oracle_state
            fb, fx = footprint_arrays(Rk, R["fps"])
            ref = po.check_request(og, fo, OL[k], Rk["begin"], Rk["poses"], Rk["radius"], fb, fx, conservative=Rk["cons"], cup=Rk["cup"],
                                   cache=caches[k], capacity=CAP)
            assert np.array_equal(got[0][idx], ref[0]) and same(got[1][idx], ref[1]) and same(got[2][idx], ref[2]), k
            same_polygons(got[3][idx], got[4][idx], ref[3], ref[4], ("oracle polygons", k))
    assert_same_answers(got, want, "polygons")
    caches = b.get_footprint()
    assert caches.shape[0] == len(singles)
    for k, s in enumerate(singles):
        assert_same_cache(caches[k], s.get_footprint(), ("cache", k))
        if oracle_state is not None:
            assert_same_cache(caches[k], oracle_state[3][k], ("oracle cache", k), nan_bits=False)
    return got


# ---- GetGridMap submaps -----------------------------------------------------------------------------------------------------

def submap_windows(rng, n, g):
    """Windows of 0 to 1.5 m around centres inside, near the edges (straddling them) and outside the map of geometry g."""
    P, Lm = np.array([g.position_x, g.position_y]), np.array([g.length_x, g.length_y])
    kind = rng.integers(0, 3, n)
    pos = P + rng.uniform(-0.45, 0.45, (n, 2)) * Lm
    edge = kind == 1
    pos[edge] = P + rng.choice([-0.5, 0.5], (edge.sum(), 2)) * Lm + rng.uniform(-0.1, 0.1, (edge.sum(), 2))
    pos[kind == 2] = P + rng.uniform(-1.2, 1.2, ((kind == 2).sum(), 2)) * Lm
    length = rng.uniform(0.0, 1.5, (n, 2))
    length[rng.random(n) < 0.1] = 0.0
    length[rng.random(n) < 0.1] = 2.5 * g.resolution
    return pos, length


def check_submaps(res, want, full, names):
    """Every window: geometry as the oracle's, layers equal to the block of the default-order layers `full`."""
    assert len(res) == len(want["success"])
    for k, (info, lay) in enumerate(res):
        for f in so.FIELDS:
            assert info[f] == want[f][k] or (np.isnan(info[f]) and np.isnan(want[f][k])), (k, f)
        if not info["success"]:
            assert lay is None
            continue
        r0, c0, nr, nc = (int(info[f]) for f in ("top_row", "top_col", "rows", "cols"))
        assert list(lay) == [n for n in full if n in names]
        for n in lay:
            assert_same_bits(np.asarray(lay[n]), full[n][r0:r0 + nr, c0:c0 + nc], (k, n))
