"""The extended-precision restatement of tier_exact.py and its rounding rule, pinned to the oracle without a GPU.

Near the origin the oracle's absolute-coordinate arithmetic carries no error that reaches a float32 rounding, so the correctly
rounded exact normal and roughness must be the oracle's layers on every cell of a partial window (the cells tier 2 recomputes),
except for cells within tier 2's delta of a rounding midpoint (explained, printed).  Cells whose scatter matrix is numerically
rank-deficient are left out: the reference's rank test decides those (tier 3), not the eigenvector.  The self-tests show the
rule has the power to see what the tolerance-based tests cannot: one float32 ulp, and a tier 2 that accumulates its z-moments in
float32."""
import numpy as np
import pytest

import tier_exact as tx
import window_masks as wm
from helpers import chain_params

SEED = 7
CASES = [("A", "tilt"), ("A", "nearflat"), ("B", "tilt")]
ROUGH_CRIT = 0.05


def _probe(oracle, shape, family):
    masks = wm.sample_masks(shape, 1 << 12, SEED) if len(wm.DISKS[shape]) > 12 else wm.all_masks(shape)
    z = wm.probe(shape, masks, family, SEED)
    rows, cols = z.shape
    res = wm.SHAPES[shape][0]
    ref = oracle.chain(oracle.Geometry.make(rows, cols, res), chain_params(oracle, **wm.chain_kwargs(shape)), z, with_normals=True)
    return z, res, ref


def _partial(z, shape, res):
    """Windows (reference coordinates) of the partial-window cells that are not rank-deficient, and the rank-deficient count."""
    i, j = np.nonzero(wm.partial_windows(np.isfinite(z), shape))
    win = tx.Windows(z, shape, i, j, res, tx.reference_coords(*z.shape, res, (0.0, 0.0)))
    rank = tx.Normals(win).rank
    return win.take(~rank), int(rank.sum())


def _normals(ref, win):
    return np.stack([ref[k][win.i, win.j] for k in ("nx", "ny", "nz")], -1)


def _check(win, ref, label):
    got_n = _normals(ref, win)
    bad_n, expl_n, mp_n = tx.check_normals(win, got_n)
    bad_r, expl_r, mp_r = tx.check_roughness(win, got_n, ref["roughness"][win.i, win.j], ROUGH_CRIT)
    print(f"\n{label}: {len(win.i)} cells; normals explained {expl_n.tolist()} (mpmath {mp_n}), roughness explained {expl_r} "
          f"(mpmath {mp_r})")
    assert len(bad_n) == 0, (label, bad_n[:10])
    assert len(bad_r) == 0, (label, bad_r[:10])
    # explained cells are the rare exception: a fixed budget of 1e-4 of the cells per layer
    assert expl_n.max() <= 1e-4 * len(win.i) + 1 and expl_r <= 1e-4 * len(win.i) + 1, (expl_n, expl_r)


@pytest.mark.parametrize("shape,family", CASES, ids=[f"{s}-{f}" for s, f in CASES])
def test_restatement_rounds_like_the_oracle_on_partial_windows(oracle, shape, family):
    z, res, ref = _probe(oracle, shape, family)
    win, rank = _partial(z, shape, res)
    assert len(win.i) > 500, len(win.i)
    print(f"\n{shape}-{family}: {rank} rank-deficient partial windows left to the rank test")
    _check(win, ref, f"{shape}-{family}")


def test_restatement_rounds_like_the_oracle_on_the_fixture(oracle, fixture_map):
    """The bag's elevation map at 0.03 m: the YAML disk is the 3 x 3 disk of shape B.  Every valid cell, full windows included."""
    m, d = fixture_map
    z = d["elevation"]
    res = m["resolution"]
    assert [o for o in tx.window_offsets("B") if o != (0, 0)] == [(k, l) for l in (-1, 0, 1) for k in (-1, 0, 1) if (k, l) != (0, 0)]
    g = oracle.Geometry.make(m["rows"], m["cols"], res)
    ref = oracle.chain(g, oracle.ChainParams.yaml_defaults(0), z, with_normals=True)
    i, j = np.nonzero(np.isfinite(z))
    win = tx.Windows(z, "B", i, j, res, tx.reference_coords(m["rows"], m["cols"], res, (0.0, 0.0)))
    win = win.take(~tx.Normals(win).rank)
    _check(win, ref, "fixture")


def test_rule_rejects_one_ulp_and_float32_moments(oracle):
    """Move the oracle's n_x, n_z and roughness by one ulp at a few hundred cells each: every moved cell must be rejected but
    those within delta of a midpoint.  A tier 2 with float32 z-moments must be rejected on a large share of the cells."""
    z, res, ref = _probe(oracle, "A", "tilt")
    win, _ = _partial(z, "A", res)
    rng = np.random.default_rng(3)
    got_n = _normals(ref, win)
    nrm = tx.Normals(win)
    movable = np.nonzero(~nrm.flat)[0]
    for d, name in ((0, "nx"), (2, "nz")):
        idx = rng.choice(movable, 300, replace=False)
        moved = got_n.copy()
        moved[:, d] = tx.ulp_step(got_n[:, d], idx, up=bool(d))
        bad, expl, _ = tx.check_normals(win, moved)
        print(f"\none ulp of {name} at {len(idx)} cells: {len(bad)} rejected, {expl.tolist()} explained")
        assert set(bad.tolist()) <= set(idx.tolist())
        assert len(bad) >= len(idx) - 2, (len(bad), len(idx))
    idx = rng.choice(len(win.i), 300, replace=False)
    rough = tx.ulp_step(ref["roughness"][win.i, win.j], idx, up=False)
    bad, expl, _ = tx.check_roughness(win, got_n, rough, ROUGH_CRIT)
    print(f"one ulp of the roughness at {len(idx)} cells: {len(bad)} rejected, {expl} explained")
    assert set(bad.tolist()) <= set(idx.tolist()) and len(bad) >= len(idx) - 2, len(bad)

    sub = win.take(rng.choice(movable, 2000, replace=False))
    f32 = tx.f32_moment_normals(sub)
    bad, expl, _ = tx.check_normals(sub, f32)
    print(f"float32 z-moments: {len(bad)} of {len(sub.i)} cells rejected, {expl.tolist()} explained")
    assert len(bad) >= 0.2 * len(sub.i), len(bad)
