"""The probe maps of window_masks.py, and the oracle's partial-window normals against an independent float64 restatement.

The oracle's behaviour on partial windows is one of its unpinned decisions (oracle/README.md items 1-3 and 5): nothing in the
reference's bag fixture has a hole in a normals window.  Here every block centre of the ShapeA probe map, one per mask of the
YAML disk, is solved a second way: its window scattered in centred coordinates and handed to numpy.linalg.eigh."""
import functools

import numpy as np
import pytest

import synth
import window_masks as wm

SEED = 7


@pytest.mark.parametrize("shape", ["A", "B"])
def test_probe_map_realises_every_mask_once(shape):
    masks = wm.all_masks(shape)
    for family in wm.FAMILIES:
        z = wm.probe(shape, masks, family, SEED)
        assert z.dtype == np.float32 and z.flags.f_contiguous
        assert z.shape == (5 * 2 ** (len(wm.DISKS[shape]) // 2),) * 2
        got = wm.decode(np.isfinite(z), shape)
        assert np.array_equal(np.sort(got), masks), family            # a permutation of 0 .. 2^n - 1
        if family == "inf":
            bad = z[~np.isfinite(z)]
            assert np.isnan(bad).any() and (bad == np.inf).any() and (bad == -np.inf).any()


def test_sampled_probe_map_realises_its_sample():
    masks = wm.sample_masks("tips", 1 << 16, SEED)
    assert len(np.unique(masks)) == 1 << 16
    z = wm.probe("tips", masks, "tilt", SEED)
    assert z.shape == (1280, 1280)
    assert np.array_equal(np.sort(wm.decode(np.isfinite(z), "tips")), masks)


def test_disks_and_partial_windows():
    assert len(wm.DISKS["A"]) == 20 and (2, 2) not in wm.DISKS["A"] and (2, 1) in wm.DISKS["A"]
    assert sorted(wm.DISKS["B"]) == sorted((k, l) for k in (-1, 0, 1) for l in (-1, 0, 1) if k or l)
    assert wm.DISKS["tips"] == wm.DISKS["A"]
    v = np.ones((10, 10), bool)
    v[4, 4] = False
    p = wm.partial_windows(v, "B")
    assert p.sum() == 8 + 36                      # the hole's 8 neighbours and the map's border ring
    assert not p[4, 4] and p[3, 3] and not p[2, 2] and p[0, 5]


# ---- the oracle against numpy.linalg.eigh on every ShapeA mask ---------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _shape_a_tilt():
    """Family 1 on the ShapeA probe map: the oracle's layers and normals at the block centres, and each centre's window
    (valid flags, centred float64 points)."""
    from oracle import binding as ob
    res = wm.SHAPES["A"][0]
    z = wm.probe("A", wm.all_masks("A"), "tilt", SEED)
    rows, cols = z.shape
    p = ob.ChainParams.yaml_defaults(0)
    for k, v in wm.chain_kwargs("A").items():
        setattr(p, k, v)
    ref = ob.chain(ob.Geometry.make(rows, cols, res), p, z, with_normals=True)
    ci, cj = wm.centres(rows, cols)
    at = {k: v[ci, cj] for k, v in ref.items()}
    X, Y = synth.cell_positions(rows, res), synth.cell_positions(cols, res)   # the oracle's cell-centre coordinates
    offs = [(0, 0)] + wm.DISKS["A"]
    ok = np.stack([np.isfinite(z[ci + k, cj + l]) for k, l in offs], axis=1)
    P = np.stack([np.stack([X[ci + k] - X[ci], Y[cj + l] - Y[cj], z[ci + k, cj + l].astype(np.float64) - z[ci, cj]], axis=1)
                  for k, l in offs], axis=1)
    P[~ok] = 0.0
    return at, ok, P, p.roughness_critical


def _scatter(ok, P):
    cnt = ok.sum(axis=1)
    mean = P.sum(axis=1) / cnt[:, None]
    D = np.where(ok[..., None], P - mean[:, None, :], 0.0)
    return cnt, D, np.einsum("nki,nkj->nij", D, D)


def _near_boundary(x, band):
    """x (float64) within `band` of a float32 rounding boundary (a midpoint between neighbouring float32 values)."""
    f = x.astype(np.float32)
    up = np.nextafter(f, np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    f = f.astype(np.float64)
    return (np.abs(x - 0.5 * (f + up)) < band) | (np.abs(x - 0.5 * (f + dn)) < band)


def test_oracle_partial_window_normals_against_eigh():
    at, ok, P, _ = _shape_a_tilt()
    cnt, _, S = _scatter(ok, P)
    lam, vec = np.linalg.eigh(S)
    n = vec[:, :, 0]
    n = np.where(n[:, 2:3] < 0.0, -n, n)
    well = (cnt >= 3) & (lam[:, 0] > 1e-9 * lam[:, 2]) & ((lam[:, 1] - lam[:, 0]) > 1e-6 * lam[:, 2])
    assert well.sum() > 0.99 * (cnt >= 3).sum(), (int(well.sum()), int((cnt >= 3).sum()))
    partial = well & (cnt < 21)
    assert partial.sum() == well.sum() - 1                         # every well-conditioned mask but the full one is partial
    worst, off = 0.0, 0
    for c, name in enumerate(("nx", "ny", "nz")):
        got, want = at[name][well], n[well, c]
        d = np.abs(got.astype(np.float64) - want)
        half = 0.5 * np.spacing(np.abs(got)).astype(np.float64)
        assert (d <= half + 1e-12).all(), (name, float((d / half).max()))   # half an ulp, up to the boundary band below
        differs = got != want.astype(np.float32)
        off += int(differs.sum())
        assert not (differs & ~_near_boundary(want, 1e-12)).any(), (name, int((differs & ~_near_boundary(want, 1e-12)).sum()))
        worst = max(worst, float(d.max()))
    print(f"\n{int(well.sum())} well-conditioned windows of {len(cnt)} masks; max |dn| {worst:.3g}; {off} components off by a "
          "float32 rounding-boundary tie")


def test_oracle_roughness_against_the_float32_normal():
    at, ok, P, crit = _shape_a_tilt()
    cnt, D, _ = _scatter(ok, P)
    N = np.stack([at["nx"], at["ny"], at["nz"]], axis=1).astype(np.float64)
    two = cnt >= 2
    r = np.sqrt((np.einsum("nki,ni->nk", D, N) ** 2).sum(axis=1) / np.maximum(cnt - 1, 1))
    want = np.where(r < crit, 1.0 - r / crit, 0.0).astype(np.float32)
    got = at["roughness"]
    ulps = np.abs(got[two].view(np.int32).astype(np.int64) - want[two].view(np.int32).astype(np.int64))
    assert ulps.max() <= 1, int(ulps.max())
    assert (got[~two] == 0.0).all()                                # one point: 0 / 0 fails the comparison -> 0.0


def test_oracle_rank_fallback_below_three_points():
    at, ok, _, _ = _shape_a_tilt()
    cnt = ok.sum(axis=1)
    few = cnt < 3
    assert few.sum() == 1 + 20                                      # the masks with no or one valid neighbour
    assert (at["nz"][few] == 1.0).all() and (at["nx"][few] == 0.0).all() and (at["ny"][few] == 0.0).all()
    assert (at["slope"][few] == 1.0).all()
