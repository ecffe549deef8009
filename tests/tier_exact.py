"""An extended-precision restatement of one chain cell's window fit, and the rounding rule its float32 layers are held to.

Tier 2 of the fused chain (k_fixup_t2, te_fixup.cu) recomputes the cells the fp32 stencil cannot certify in fp64 on window-centred
coordinates and claims an accuracy of about 1e-13 before it rounds to float32.  Its n_x, n_y, n_z and roughness must then be the
correctly rounded float32 of the EXACT value of the window, except where that value lies so close to a rounding midpoint that
tier 2's own error may carry it across.  This module states those exact values and the rule; CPU only.

Window.  The cells of the normals disk (window_masks.DISKS plus the centre) that are valid (finite) and inside the map, at offsets
from the centre cell: the reference's coordinates X[a] - X[i], Y[b] - Y[j] (oracle/te_oracle.cpp cell_coord), or the nominal
grid -res * k, -res * l that tier 2 computes on.  Both are exact in double: X[a] - X[i] by Sterbenz's lemma away from the origin
and with an error below 1e-17 m near it (far inside every delta below), -res * k because k is 1 or 2.  Elevation differences
z[a, b] - z[i, j] of float32 values are exact in double.  Near the origin the two offsets differ by ~1e-15 m; at far positions by
the reference's own coordinate rounding (ulp(|X|), 5e-10 m at LV95), which is why the tests of tier 2 use the nominal grid.

Normal.  The unit eigenvector of the smallest eigenvalue of the scatter matrix S = sum (p - mean)(p - mean)^T, signed n_z >= 0:
vectorised fp64 eigh screens every cell, and mpmath at 40 digits decides the cells where the screen is not conclusive.  A window
of fewer than 3 cells or with all elevations equal has the normal (0, 0, 1): the reference's rank test sends both there.

Roughness.  The layer 1 - r / crit (0 from r >= crit, and for a single cell) with r = sqrt(sum (N . (p - mean))^2 / (n - 1)) and
N the kernel's own float32 normal, which RoughnessFilter reads back from the layers.

Slope.  1 - acos(n_z) / crit of the float32 n_z (0 from acos(n_z) >= crit).

Delta.  te_fixup.cu documents tier 2 as accurate to ~1e-13 on the unit normal.  Its error is that of the scatter matrix (a few
roundings of sums of exact products: ~10 eps |S|) carried to the eigenvector by 1 / (lambda_1 - lambda_0), and that of Halley's
lambda_0 (stopped at 1e-15 trace(S)) carried the same way: with kappa = lambda_2 / (lambda_1 - lambda_0), at most ~1e-14 (1 +
kappa) absolutely.  DELTA_N = 1e-13 per unit of (1 + kappa) is the documented accuracy with that factor and a ten-fold margin.
The roughness sum is N^T S N in tier 2, off by ~10 eps sum_ij |N_i N_j S_ij| <= 3.3e-15 trace(S); DELTA_R = 1e-13 trace(S) holds it
with a thirty-fold margin, and it reaches the layer through r = sqrt(sum / (n - 1)) / crit."""
import math

import numpy as np

import window_masks as wm

DELTA_N = 1e-13      # absolute error of a tier-2 normal component per unit of (1 + kappa)
DELTA_R = 1e-13      # absolute error of tier 2's roughness sum per unit of trace(S)
MP_DPS = 40


# ---- coordinates and windows ------------------------------------------------------------------------------------------------------

def cell_coords(n, res, pos, length):
    """The reference's cell-centre coordinates of index 0 .. n-1 (cell_coord: (pos + offset) + res * (-idx))."""
    offset = 0.5 * length - 0.5 * res
    return (pos + offset) + res * (-np.arange(n, dtype=np.float64))


def reference_coords(rows, cols, res, pos):
    """(X, Y) of Geometry.make(rows, cols, res, pos)."""
    return cell_coords(rows, res, pos[0], rows * res), cell_coords(cols, res, pos[1], cols * res)


def window_offsets(shape):
    """(k, l) of the normals window of the shape: the centre and the disk, in mask-bit order after the centre."""
    return [(0, 0)] + list(wm.DISKS[shape])


class Windows:
    """The windows of cells (i, j) of the float32 map z: offsets U, V (m), elevation differences W (m) from the centre, and the
    validity mask M, each (ncells, m); invalid entries are 0.  coords=None: the nominal grid -res * k, -res * l; else (X, Y)."""

    def __init__(self, z, shape, i, j, res, coords=None):
        rows, cols = z.shape
        self.z, self.shape, self.res, self.coords = z, shape, res, coords
        self.i, self.j = np.asarray(i, np.int64), np.asarray(j, np.int64)
        self.off = window_offsets(shape)
        n, m = len(self.i), len(self.off)
        self.U, self.V, self.W = (np.zeros((n, m)) for _ in range(3))
        self.M = np.zeros((n, m), bool)
        zc = z[self.i, self.j].astype(np.float64)
        for q, (k, l) in enumerate(self.off):
            a, b = self.i + k, self.j + l
            inside = (a >= 0) & (a < rows) & (b >= 0) & (b < cols)
            v = np.full(n, np.nan)
            v[inside] = z[a[inside], b[inside]]
            ok = np.isfinite(v)
            self.M[:, q] = ok
            self.W[ok, q] = v[ok] - zc[ok]
            if coords is None:
                self.U[ok, q], self.V[ok, q] = -res * k, -res * l
            else:
                X, Y = coords
                self.U[ok, q] = X[a[ok]] - X[self.i[ok]]
                self.V[ok, q] = Y[b[ok]] - Y[self.j[ok]]
        self.n = self.M.sum(1)

    def take(self, sel):
        """The windows of the cells sel (index or bool array) only."""
        w = object.__new__(Windows)
        w.__dict__.update(self.__dict__)
        for k in ("i", "j", "U", "V", "W", "M", "n"):
            setattr(w, k, getattr(self, k)[sel])
        return w

    def scatter(self):
        """(ncells, 3, 3) scatter matrices in fp64 (centred on the window mean)."""
        n = np.maximum(self.n, 1)[:, None]
        P = np.stack([self.U, self.V, self.W], -1)                     # (ncells, m, 3)
        mean = P.sum(1) / n
        D = (P - mean[:, None, :]) * self.M[:, :, None]
        return np.einsum("cmi,cmj->cij", D, D), mean

    def mp_cell(self, c):
        """Exact points of cell c as mpmath (u, v, w) lists."""
        import mpmath
        out = []
        i, j = int(self.i[c]), int(self.j[c])
        zc = mpmath.mpf(float(self.z[i, j]))
        for q, (k, l) in enumerate(self.off):
            if not self.M[c, q]:
                continue
            if self.coords is None:
                u, v = -mpmath.mpf(self.res) * k, -mpmath.mpf(self.res) * l
            else:
                X, Y = self.coords
                u = mpmath.mpf(float(X[i + k])) - mpmath.mpf(float(X[i]))
                v = mpmath.mpf(float(Y[j + l])) - mpmath.mpf(float(Y[j]))
            out.append((u, v, mpmath.mpf(float(self.z[i + k, j + l])) - zc))
        return out


def _mp_scatter(pts):
    import mpmath
    n = len(pts)
    mean = [sum(p[d] for p in pts) / n for d in range(3)]
    S = mpmath.matrix(3, 3)
    for p in pts:
        q = [p[d] - mean[d] for d in range(3)]
        for r in range(3):
            for s in range(3):
                S[r, s] += q[r] * q[s]
    return S, mean


# ---- normals ----------------------------------------------------------------------------------------------------------------------

class Normals:
    """The exact normal of every window (fp64 screen; mpmath for the cells `decide` is asked about).

    n64 (ncells, 3): the fp64 normal; kappa: lambda_2 / (lambda_1 - lambda_0); flat: the normal is (0, 0, 1) by rule (fewer than
    3 cells, or all elevations equal); rank: lambda_0 <= 1e-9 trace(S), where the reference's rank test decides, not the
    eigenvector."""

    def __init__(self, win):
        self.win = win
        S, _ = win.scatter()
        lam, vec = np.linalg.eigh(S)
        n = vec[:, :, 0]
        n = np.where(n[:, 2:3] < 0, -n, n)
        self.flat = (win.n < 3) | (S[:, 2, 2] == 0.0)
        n[self.flat] = (0.0, 0.0, 1.0)
        self.n64 = n
        gap = lam[:, 1] - lam[:, 0]
        with np.errstate(divide="ignore", invalid="ignore"):
            self.kappa = np.where(gap > 0, lam[:, 2] / gap, np.inf)
        self.kappa[self.flat] = 0.0
        tr = lam.sum(1)
        self.rank = ~self.flat & ~(lam[:, 0] > 1e-9 * tr)
        self.S = S

    def delta(self):
        """Absolute rounding-rule delta of every component: DELTA_N (1 + kappa)."""
        return DELTA_N * (1.0 + self.kappa)

    def exact(self, c):
        """The normal of cell c at MP_DPS digits, as the nearest doubles."""
        import mpmath
        if self.flat[c]:
            return np.array([0.0, 0.0, 1.0])
        with mpmath.workdps(MP_DPS):
            S, _ = _mp_scatter(self.win.mp_cell(c))
            E, Q = mpmath.eigsy(S)
            s = min(range(3), key=lambda k: E[k])
            v = [Q[r, s] for r in range(3)]
            if v[2] < 0:
                v = [-x for x in v]
            return np.array([float(x) for x in v])


# ---- the rounding rule ------------------------------------------------------------------------------------------------------------

def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def rounding_range(exact, delta):
    """(lo, hi): the float32 roundings of exact - delta and exact + delta.  Rounding is monotone, so the floats in [lo, hi] are
    exactly the correct roundings of the values within delta of exact."""
    exact = np.asarray(exact, np.float64)
    return _f32(exact - delta), _f32(exact + delta)


def correctly_rounded(got, exact, delta):
    """(ok, explained) per cell: got (float32) must be the float32 nearest exact (a double, the exact value to well within
    delta), except where a value within delta (absolute, per cell) of exact rounds otherwise: where exact lies within delta of
    the midpoint between two floats, either neighbour passes (and where delta exceeds the spacing of the floats, as for a
    component of ~1e-16 that is zero by symmetry, every float in range).  explained: got passes, is not the nearest, and the
    floats around exact are farther apart than 2 delta (the midpoint exception proper; a value below that resolution is held to
    delta absolutely and not counted).  NaN passes against NaN only."""
    got = np.asarray(got, np.float32)
    exact = np.asarray(exact, np.float64)
    nan = np.isnan(exact)
    e = np.where(nan, 0.0, exact)
    lo, hi = rounding_range(e, delta)
    same = (got.view(np.uint32) == _f32(e).view(np.uint32)) & ~nan
    inside = (got >= lo) & (got <= hi) & ~nan
    return same | inside | (nan & np.isnan(got)), inside & ~same & resolvable(e, delta)


def resolvable(exact, delta):
    """Values whose float32 neighbours are farther apart than 2 delta."""
    return np.abs(np.spacing(_f32(exact))).astype(np.float64) > 2.0 * np.asarray(delta, np.float64)


def _screen(got, x64, delta, err):
    """The fp64 screen of the rule, x64 being the exact value to within err.  Returns (pass, fail): pass where got is a rounding
    of a value within delta - err of x64 (so within delta of the exact value), fail where it is none within delta + err; the
    other cells need the exact value."""
    lo_in, hi_in = rounding_range(x64, delta - err)
    lo_out, hi_out = rounding_range(x64, delta + err)
    ok = (got >= lo_in) & (got <= hi_in)
    return ok, ~((got >= lo_out) & (got <= hi_out))


# ---- roughness and slope ----------------------------------------------------------------------------------------------------------

def roughness_sum(win, N):
    """sum (N . (p - mean))^2 per window in fp64 (pointwise: the residuals are small, so the sum loses no relative accuracy)."""
    n = np.maximum(win.n, 1)[:, None]
    P = np.stack([win.U, win.V, win.W], -1)
    mean = P.sum(1) / n
    d = np.einsum("cmi,ci->cm", P - mean[:, None, :], N) * win.M
    return (d * d).sum(1)


def roughness_layer(sumsq, n, crit):
    """1 - r / crit of r = sqrt(sum / (n - 1)), 0 from r >= crit; 0 for a single cell (0 / 0 compares false)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.sqrt(sumsq / (n - 1.0))
        return np.where(r < crit, 1.0 - r / crit, 0.0), r


def roughness_delta(S, r, n, crit):
    """Absolute delta of tier 2's roughness layer: DELTA_R trace(S) of the sum, through r = sqrt(sum / (n - 1)) / crit, plus
    1e-14 for the few roundings after the sum (sqrt, 1 - r / crit: ~1e-16 each)."""
    ds = DELTA_R * np.trace(S, axis1=1, axis2=2) / np.maximum(n - 1.0, 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        dr = np.where(r > 0, np.minimum(ds / (2.0 * r), np.sqrt(ds)), np.sqrt(ds))
    return np.where(np.isfinite(r), (dr + 1e-15 * r) / crit, 0.0) + 1e-14   # r is NaN for a single cell: layer 0


def mp_roughness(win, c, N, crit):
    """The exact roughness layer of cell c with the normal N (3 doubles), as the nearest double."""
    import mpmath
    with mpmath.workdps(MP_DPS):
        pts = win.mp_cell(c)
        _, mean = _mp_scatter(pts)
        Nm = [mpmath.mpf(float(x)) for x in N]
        s = sum(sum(Nm[d] * (p[d] - mean[d]) for d in range(3)) ** 2 for p in pts)
        if len(pts) < 2:
            return 0.0
        r = mpmath.sqrt(s / (len(pts) - 1))
        return float(1 - r / mpmath.mpf(crit)) if r < crit else 0.0


def slope_exact(nz, crit):
    """1 - acos(nz) / crit of float32 n_z (0 from acos >= crit; NaN for NaN), and theta; fp64 (1 ulp acos)."""
    x = np.minimum(np.asarray(nz, np.float64), 1.0)
    th = np.arccos(x)
    return np.where(th < crit, 1.0 - th / crit, 0.0), th


def slope_bound_ok(got, nz, crit):
    """(ok, ratio): acos_t2's bound |got - exact| <= 1.7e-7 theta / crit + half an ulp of got, and exactly 0 from theta >=
    crit (1 + 2e-7); ratio = |got - exact| / bound.  Cells within 1e-12 of the bound are redone with mpmath's acos."""
    exact, th = slope_exact(nz, crit)
    g = np.asarray(got, np.float64)
    ulp = np.abs(np.nextafter(np.asarray(got, np.float32), np.float32(np.inf)).astype(np.float64) - g)
    bound = 1.7e-7 * th / crit + 0.5 * ulp
    err = np.abs(g - exact)
    close = np.nonzero(np.abs(err - bound) <= 1e-12)[0]
    if len(close):
        import mpmath
        with mpmath.workdps(MP_DPS):
            for c in close:
                t = mpmath.acos(mpmath.mpf(float(nz[c])))
                e = (1 - t / mpmath.mpf(crit)) if t < crit else mpmath.mpf(0)
                err[c] = float(abs(mpmath.mpf(float(g[c])) - e))
    ok = err <= bound
    ok &= ~((th >= crit * (1 + 2e-7)) & (g != 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(bound > 0, err / bound, 0.0)
    return ok, ratio


# ---- checking a kernel's normals and roughness ------------------------------------------------------------------------------------

def check_normals(win, got_n):
    """Hold got_n (ncells, 3) float32 to the rule.  Returns (bad cell indices, explained count per component, mpmath cells).

    The fp64 normal is the exact one to within ~1e-15 (1 + kappa), a hundredth of delta: _screen decides every cell it can, and
    the mpmath normal decides the rest."""
    nrm = Normals(win)
    got_n = np.asarray(got_n, np.float32)
    delta = nrm.delta()
    ok = np.ones(len(got_n), bool)
    fail = np.zeros(len(got_n), bool)
    expl = np.zeros(3, np.int64)
    for d in range(3):
        p, f = _screen(got_n[:, d], nrm.n64[:, d], delta, 0.1 * delta)
        ok &= p
        fail |= f
    ok |= nrm.flat & (got_n == np.float32([0, 0, 1])).all(1)
    for d in range(3):
        expl[d] = int((ok & (got_n[:, d].view(np.uint32) != _f32(nrm.n64[:, d]).view(np.uint32)) &
                       resolvable(nrm.n64[:, d], delta)).sum())
    bad = list(np.nonzero(fail & ~ok)[0])
    todo = np.nonzero(~ok & ~fail)[0]
    for c in todo:
        good, ex = correctly_rounded(got_n[c], nrm.exact(c), delta[c])
        if not good.all():
            bad.append(int(c))
        expl += ex
    return np.sort(np.asarray(bad, np.int64)), expl, len(todo)


def check_roughness(win, got_n, got_r, crit):
    """Hold the roughness layer got_r to the rule against the exact roughness of the kernel's own normal got_n.  Returns (bad
    cell indices, explained count, mpmath cells).  The pointwise fp64 layer is the exact one to within 2e-15."""
    N = np.asarray(got_n, np.float32).astype(np.float64)
    S, _ = win.scatter()
    layer, r = roughness_layer(roughness_sum(win, N), win.n.astype(np.float64), crit)
    delta = roughness_delta(S, r, win.n.astype(np.float64), crit)
    got_r = np.asarray(got_r, np.float32)
    ok, fail = _screen(got_r, layer, delta, 2e-15)
    expl = int((ok & (got_r.view(np.uint32) != _f32(layer).view(np.uint32)) & resolvable(layer, delta)).sum())
    bad = list(np.nonzero(fail & ~ok)[0])
    todo = np.nonzero(~ok & ~fail)[0]
    for c in todo:
        good, ex = correctly_rounded(got_r[c:c + 1], np.array([mp_roughness(win, c, N[c], crit)]), delta[c])
        if not good.all():
            bad.append(int(c))
        expl += int(ex.sum())
    return np.sort(np.asarray(bad, np.int64)), expl, len(todo)


def f32_moment_normals(win):
    """A tier 2 whose z-moments (sum w, sum w^2, sum u w, sum v w) are accumulated in float32: its float32 normal, for the rule's
    self-test."""
    f = np.float32
    n = np.maximum(win.n, 1).astype(np.float64)
    sw = np.zeros(len(n), f)
    sww, suw, svw = (np.zeros(len(n), f) for _ in range(3))
    for q in range(win.M.shape[1]):
        w = win.W[:, q].astype(f) * win.M[:, q]
        sw = (sw + w).astype(f)
        sww = (sww + w * w).astype(f)
        suw = (suw + win.U[:, q].astype(f) * w).astype(f)
        svw = (svw + win.V[:, q].astype(f) * w).astype(f)
    U, V, M = win.U, win.V, win.M
    su, sv = (U * M).sum(1), (V * M).sum(1)
    suu, svv, suv = (U * U * M).sum(1), (V * V * M).sum(1), (U * V * M).sum(1)
    sw, sww, suw, svw = (a.astype(np.float64) for a in (sw, sww, suw, svw))
    S = np.empty((len(n), 3, 3))
    S[:, 0, 0], S[:, 1, 1], S[:, 2, 2] = suu - su * su / n, svv - sv * sv / n, sww - sw * sw / n
    S[:, 0, 1] = S[:, 1, 0] = suv - su * sv / n
    S[:, 0, 2] = S[:, 2, 0] = suw - su * sw / n
    S[:, 1, 2] = S[:, 2, 1] = svw - sv * sw / n
    _, vec = np.linalg.eigh(S)
    v = vec[:, :, 0]
    v = np.where(v[:, 2:3] < 0, -v, v)
    return v.astype(np.float32)


def ulp_step(a, idx, up):
    """A copy of float32 array a with the cells idx moved one ulp up (up True) or down."""
    b = np.array(a, np.float32, copy=True)
    b[idx] = np.nextafter(b[idx], np.float32(np.inf) if up else np.float32(-np.inf))
    return b


def nz_check_limit(crit):
    """nz_check_limit() of te_fused.cu, as test_kernel_constants_cpu restates it: the s = 1 - n_z below which the fused kernel
    rounds n_z exactly like the reference or flags the cell."""
    if not crit < 1.0:
        return 7.2e-5
    t = 1.02 * crit + 2.0 ** -22 / math.sin(crit)
    return max(7.2e-5, 2.0 * math.sin(0.5 * t) ** 2)
