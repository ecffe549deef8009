"""Properties of the sequential te_map oracle (tests/map_oracle.cpp): the check_footprint_path service loop on a persistent
traversability_footprint layer.  No GPU."""
import numpy as np

import map_oracle as mo
import synth
import untraversable_oracle as uo
from test_paths_fresh_gpu import _layers


def _map(oracle, rows=120, cols=110, res=0.02, seed=5):
    z = synth.terrain(rows, cols, res, seed, "mixed")
    og = oracle.Geometry.make(rows, cols, res)
    L, rs = _layers(oracle, og, z, seed)
    return og, L, rs


def _single_poses(og, rng, n):
    """n single-pose circular paths at distinct cells (x, y and a unit quaternion, 7 wide)."""
    cells = rng.choice(og.rows * og.cols, n, replace=False)
    xs = og.position_x + 0.5 * og.rows * og.resolution - (cells % og.rows + 0.5) * og.resolution
    ys = og.position_y + 0.5 * og.cols * og.resolution - (cells // og.rows + 0.5) * og.resolution
    poses = np.zeros((n, 7))
    poses[:, 0], poses[:, 1], poses[:, 6] = xs, ys, 1.0
    return np.arange(n + 1, dtype=np.int32), poses


def test_empty_cache_disjoint_cells_equal_fresh_oracle(oracle):
    og, L, rs = _map(oracle)
    fo = oracle.FootprintParams.yaml_defaults()
    rng = np.random.default_rng(1)
    begin, poses = _single_poses(og, rng, 200)
    radius = rng.choice([0.0, 0.1, 0.2, 0.3], 200)
    cup = (rng.random(200) < 0.5).astype(np.uint8)
    cache = mo.empty_cache(og)
    got = mo.check_request(og, fo, L, cache, begin, poses, radius, np.zeros(201, np.int32), np.zeros((0, 3), np.float32),
                           compute_untraversable_polygon=cup)
    want = uo.check_circular_paths_fresh2(og, fo, L["traversability"], L["slope"], L["step"], L["elevation"], begin,
                                          poses[:, :2].copy(), radius, compute_untraversable_polygon=cup)
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(got[1].view(np.uint64), want[1].view(np.uint64))
    assert np.array_equal(got[3], want[2])
    assert np.array_equal(got[4].view(np.uint64), want[3].view(np.uint64))
    assert np.isfinite(cache).sum() == 200   # every pose stored its cell


def test_annulus_blocker_is_unsafe_first_and_safe_after(oracle):
    """A first blocked cell between radius and radius + offset: untraversable on the first check, which still stores a positive
    value (TraversabilityMap.cpp:708, :714-717); the same path in the next request reads it back and passes (:673-675)."""
    og, L, rs = _map(oracle)
    fo = oracle.FootprintParams.yaml_defaults()
    rng = np.random.default_rng(2)
    begin, poses = _single_poses(og, rng, 400)
    radius = np.full(400, 0.1)
    cache = mo.empty_cache(og)
    args = (begin, poses, radius, np.zeros(401, np.int32), np.zeros((0, 3), np.float32))
    first = mo.check_request(og, fo, L, cache, *args)[0]
    second = mo.check_request(og, fo, L, cache, *args)[0]
    flipped = (first == 0) & (second == 1)
    assert flipped.sum() > 0
    assert np.all(second >= first)


def test_polygonal_paths_leave_the_cache_alone(oracle):
    og, L, rs = _map(oracle)
    fo = oracle.FootprintParams.yaml_defaults()
    rng = np.random.default_rng(3)
    begin, poses = _single_poses(og, rng, 30)
    fxyz = np.tile(np.array([[0.1, 0.05, 0.0], [-0.1, 0.05, 0.0], [-0.1, -0.05, 0.0], [0.1, -0.05, 0.0]], np.float32), (30, 1))
    cache = mo.empty_cache(og)
    cache[::7, ::5] = 0.25
    before = cache.copy()
    mo.check_request(og, fo, L, cache, begin, poses, np.full(30, 0.2), np.arange(0, 121, 4, dtype=np.int32), fxyz)
    assert np.array_equal(before.view(np.uint32), cache.view(np.uint32))
