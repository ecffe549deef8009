"""Probe maps that put every validity pattern of a normals window under the chain.

A cell whose window has a hole or a map border in it takes a different path through the chain from a cell whose window is full
(tier 1 flags it, tier 2 recomputes it from popcounts of its 25-bit validity mask, tier 3 replays the reference's rank test), and
random terrain reaches only a few hundred of the 2^20 masks of the YAML disk.  A probe map of 5a x 5b cells is tiled into 5 x 5
blocks.  Each block's centre is valid and its disk neighbours are valid or not according to one mask; its other cells are valid
at random.  The disk of a centre lies inside its own block, so every block realises its mask exactly, and the other cells of the
map get partial windows of their own, many of them straddling two to four blocks.

Mask bit q is the disk neighbour DISKS[shape][q] = (k, l): row offset k, column offset l, in the order of the kernels' 25-bit
masks (bit (l + 2) * 5 + (k + 2), the centre left out).  Blocks are in row-major order."""
import numpy as np

# (resolution, normals = roughness radius, step first = second radius)
SHAPES = {
    "A": (0.02, 0.05, 0.04),        # the YAML: 20 neighbours; the step tips (+-2, 0), (0, +-2) lie on the circle
    "B": (0.025, 0.045, 0.03),      # 3 x 3 disk: 8 neighbours
    "tips": (0.021, 0.05, 0.042),   # the disk of A; step tips on the circle at a resolution that is no power of two
}

FAMILIES = ("tilt", "planar", "nearflat", "inf")


def disk(shape):
    """The normals disk's neighbour offsets (k, l) in mask-bit order."""
    res, rn, _ = SHAPES[shape]
    rr = (rn / res) ** 2
    out = []
    for l in range(-2, 3):
        for k in range(-2, 3):
            d = k * k + l * l
            assert abs(d - rr) > 1e-6, (shape, k, l)   # no offset of the normals disk sits on its circle
            if 0 < d < rr:
                out.append((k, l))
    return out


DISKS = {s: disk(s) for s in SHAPES}


def chain_kwargs(shape):
    """ChainParams fields of the shape."""
    _, rn, rs = SHAPES[shape]
    return dict(normals_radius=rn, roughness_radius=rn, step_first_radius=rs, step_second_radius=rs)


def all_masks(shape):
    return np.arange(1 << len(DISKS[shape]), dtype=np.int64)


def sample_masks(shape, n, seed):
    """n distinct masks of the shape, drawn with a seed."""
    return np.sort(np.random.default_rng(seed).choice(1 << len(DISKS[shape]), n, replace=False)).astype(np.int64)


def _grid(n):
    """Blocks (a, b) of a map holding n masks: a square of blocks."""
    a = int(round(np.sqrt(n)))
    assert a * a == n, n
    return a, a


def validity(shape, masks, seed):
    """(rows, cols) bool: the validity pattern of a probe map for `masks` (shuffled over the blocks with the seed)."""
    rng = np.random.default_rng(seed)
    a, b = _grid(len(masks))
    blk = rng.permutation(np.asarray(masks, np.int64)).reshape(a, b)
    V = rng.random((a, 5, b, 5)) < 0.5                        # cells outside every disk: valid at random
    V[:, 2, :, 2] = True
    for q, (k, l) in enumerate(DISKS[shape]):
        V[:, 2 + k, :, 2 + l] = ((blk >> q) & 1).astype(bool)
    return V.reshape(5 * a, 5 * b)


def decode(valid, shape):
    """The masks a validity pattern realises at its block centres, in block order; asserts every centre is valid."""
    rows, cols = valid.shape
    assert rows % 5 == 0 and cols % 5 == 0, valid.shape
    V = np.asarray(valid, bool).reshape(rows // 5, 5, cols // 5, 5)
    assert V[:, 2, :, 2].all()
    m = np.zeros((rows // 5, cols // 5), np.int64)
    for q, (k, l) in enumerate(DISKS[shape]):
        m |= V[:, 2 + k, :, 2 + l].astype(np.int64) << q
    return m.reshape(-1)


def centres(rows, cols):
    """Row and column index of every block centre, in block order."""
    i, j = np.meshgrid(np.arange(2, rows, 5), np.arange(2, cols, 5), indexing="ij")
    return i.reshape(-1), j.reshape(-1)


def probe(shape, masks, family, seed):
    """Column-major float32 elevation of a probe map: the validity pattern of `masks` and, per block, a surface of the family.

    tilt      a plane through the block centre inclined up to 1.2 rad in each direction, 1 mm of noise
    planar    an exactly planar block: slopes k/8 per cell, every z = f32(f32(sk*k + sl*l) * f32(res)) exact, some blocks flat
    nearflat  inclination up to 0.01 rad, noise of 1e-5 to 1e-4 m (the band where n_z's float32 rounding moves the slope)
    inf       the tilt surfaces with the holes NaN, +Inf or -Inf at random"""
    assert family in FAMILIES, family
    res = SHAPES[shape][0]
    rng = np.random.default_rng(seed + 1)
    V = validity(shape, masks, seed)
    rows, cols = V.shape
    a, b = rows // 5, cols // 5
    K = (np.arange(5) - 2.0).reshape(1, 5, 1, 1)
    L = (np.arange(5) - 2.0).reshape(1, 1, 1, 5)
    per = lambda draw: draw.reshape(a, 1, b, 1)   # noqa: E731  one value per block
    if family == "planar":
        sk = per(rng.integers(-16, 17, a * b) / 8.0)
        sl = per(rng.integers(-16, 17, a * b) / 8.0)
        flat = per(rng.random(a * b) < 0.05)
        sk, sl = np.where(flat, 0.0, sk), np.where(flat, 0.0, sl)
        z = ((sk * K + sl * L).astype(np.float32) * np.float32(res)).astype(np.float32)
    elif family == "nearflat":
        th, ph = per(rng.uniform(0.0, 0.01, a * b)), per(rng.uniform(0.0, 2 * np.pi, a * b))
        sigma = per(10.0 ** rng.uniform(-5.0, -4.0, a * b))
        z = res * np.tan(th) * (np.cos(ph) * K + np.sin(ph) * L) + sigma * rng.standard_normal((a, 5, b, 5))
    else:
        gk, gl = per(np.tan(rng.uniform(-1.2, 1.2, a * b))), per(np.tan(rng.uniform(-1.2, 1.2, a * b)))
        z = per(rng.uniform(-0.02, 0.02, a * b)) + res * (gk * K + gl * L) + 1e-3 * rng.standard_normal((a, 5, b, 5))
    z = np.asarray(z, np.float32).reshape(rows, cols)
    if family == "inf":
        z[~V] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), int((~V).sum()))
    else:
        z[~V] = np.nan
    return np.asfortranarray(z)


def partial_windows(valid, shape):
    """Valid cells whose normals window is partial: a disk neighbour is invalid or outside the map."""
    rows, cols = valid.shape
    pad = np.zeros((rows + 4, cols + 4), bool)
    pad[2:-2, 2:-2] = valid
    full = valid.copy()
    for k, l in DISKS[shape]:
        full &= pad[2 + k:2 + k + rows, 2 + l:2 + l + cols]
    return valid & ~full
