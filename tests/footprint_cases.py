"""The maps of the footprint-parameter tests (test_footprint_params_gpu.py, test_footprint_params_cpu.py).

Chain layers block nearly every disk at large radii, so beside them there are built layers where one cell more or less in a
footprint shows: a traversability with a distinct value per cell (far_geometry.distinct_layer), about one invalid cell in 400, and
isolated zero-slope blockers that block alone with max_gap_width 0.001 (checkForSlope's critical count floor(2 gap / res) is then
0), spaced so that the first blocked cell of many disks falls on either side of the inner radius."""
import functools

import numpy as np

import far_geometry as fg
import synth
from helpers import chain_layers

LAYERS = ("traversability", "slope", "step", "elevation")
BUILT_GAP = dict(max_gap_width=0.001)   # the built maps' blockers block alone


@functools.lru_cache(maxsize=None)
def chain_map(oracle, res=0.02, rows=160, cols=140, seed=21):
    """The oracle chain's layers on synth terrain, roughness with zero patches."""
    og = oracle.Geometry.make(rows, cols, res)
    L, _ = chain_layers(oracle, og, synth.terrain(rows, cols, res, seed, "mixed"), seed)
    return L


@functools.lru_cache(maxsize=None)
def built_map(res=0.02, rows=160, cols=144, spacing=40, seed=3):
    """Distinct traversability with about one invalid cell in 400, and zero-slope blockers on a jittered lattice of `spacing`
    cells (at least one blocker)."""
    rng = np.random.default_rng(seed)
    t = fg.distinct_layer(rows, cols, seed)
    t[rng.random((rows, cols)) < 1.0 / 400] = np.nan
    slope = np.ones((rows, cols), np.float32, order="F")
    for a in range(spacing // 2, rows, spacing):
        for b in range(spacing // 2, cols, spacing):
            slope[min(a + int(rng.integers(-3, 4)), rows - 1), min(b + int(rng.integers(-3, 4)), cols - 1)] = 0.0
    one = np.ones((rows, cols), np.float32, order="F")
    return dict(traversability=t, slope=slope, step=one, roughness=one.copy(), elevation=np.zeros((rows, cols), np.float32, order="F"))


def unblocked(m):
    """m without its blockers: the reference for 'the result is not just the mean'."""
    return dict(m, slope=np.ones_like(m["slope"]))
