"""The cases of test_literal_params_gpu.py are not vacuous on the oracle, and the acos rule of its slope comparison is sound.

Every case of literal_cases.CASES records what makes it able to fail; here the oracle shows that it does: the positive axis flips
normals, the algorithms differ, on-circle radii put cells at distance exactly r on both sides of the test, a critical of 0 zeroes its
layer, and so on.  Then slope_explained must accept a cell whose float32 slope flips with a change of the double acos within its
error bound, and reject a one-step change of the float32 result anywhere else."""
import math

import numpy as np
import pytest

import literal_cases as lc
import synth


def _chain(oracle, c, **over):
    return oracle.chain(lc.geometry(oracle, c), lc.params(oracle, c, **over), lc.terrain(c), with_normals=True)


def _differ(a, b):
    """Cells where two float32 layers differ (a NaN matches a NaN)."""
    return int(((a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))).sum())


def _circle_test(c, name, k):
    """(inside, outside): centres whose cell k rows or k columns away passes / fails the circle test of radius `name`, with the
    oracle's coordinates and arithmetic (dx * dx + dy * dy <= r * r in double)."""
    r = c["params"][name]
    inside = outside = 0
    for n, p in ((c["rows"], c["pos"][0]), (c["cols"], c["pos"][1])):
        X = synth.cell_positions(n, c["res"], p)
        d = X[k:] - X[:-k]
        t = d * d + 0.0 * 0.0 <= r * r
        inside, outside = inside + int(t.sum()), outside + int((~t).sum())
    return inside, outside


def _few_windows(z):
    """Per valid cell of a few_valid map: (valid cells in its 3 x 3 window, whether they lie in one row or one column)."""
    rows, cols = z.shape
    out = {}
    for i, j in zip(*np.nonzero(np.isfinite(z))):
        pts = [(a, b) for a in range(max(0, i - 1), min(rows, i + 2)) for b in range(max(0, j - 1), min(cols, j + 2))
               if np.isfinite(z[a, b])]
        out[(i, j)] = (len(pts), len({a for a, _ in pts}) == 1 or len({b for _, b in pts}) == 1)
    return out


def _check(oracle, c, prop):
    name, *arg = prop
    ref = _chain(oracle, c)
    finite = np.isfinite(ref["nz"])
    if name == "axis":
        a = arg[0]
        for b in {0, 1, 2} - {a}:
            other = _chain(oracle, c, normals_positive_axis=b)
            n = _differ(ref["nz"], other["nz"])
            print(f"{c['name']}: axis {a} against {b}: {n} normals flipped")
            assert n > 0
        assert (ref[("nx", "ny", "nz")[a]][finite] >= 0).all()
    elif name == "alg":
        other = _chain(oracle, c, normals_algorithm=1 - c["params"].get("normals_algorithm", 0))
        n = sum(_differ(ref[k], other[k]) for k in ("nx", "ny", "nz"))
        print(f"{c['name']}: the other algorithm changes {n} normal components")
        assert n > 0
    elif name == "radius_zero":
        assert finite.any() and (ref["nz"][finite] == 1.0).all()   # one point in the window: the default normal (0, 0, 1)
    elif name in ("on_circle", "generous"):
        which, k = arg
        r = c["params"][which]
        inside, outside = _circle_test(c, which, k)
        print(f"{c['name']}: {which} = {r!r}, offset {k}: inside on {inside} centres, outside on {outside}")
        assert inside > 0
        if name == "generous":
            assert math.floor(r / c["res"]) < k and outside > 0   # only the generous reach scans the cells that get in
        elif c["pos"] == lc.LV95:
            assert outside > 0
    elif name == "big":
        R = math.floor(c["params"]["normals_radius"] / c["res"]) + 1
        assert (2 * R + 1) ** 2 > 64
    elif name == "param":
        which, layer, alt = arg
        other = _chain(oracle, c, **{which: alt})
        assert _differ(ref[layer], other[layer]) > 0
    elif name == "ncrit":
        for n in {1, 4, 1000} - {arg[0]}:
            assert _differ(ref["step"], _chain(oracle, c, step_critical_cells=n)["step"]) > 0
    elif name == "zero":
        v = ref[arg[0]][np.isfinite(ref[arg[0]])]
        assert v.size > 0 and (v == 0.0).all()
    elif name == "fuse":
        w = arg[0]
        want = np.float32(w) * ((ref["slope"] + ref["step"]) + ref["roughness"])
        assert _differ(ref["traversability"], want) == 0
        t = ref["traversability"]
        if math.isnan(w):
            assert np.isnan(t).all()
        else:
            assert (np.isfinite(t) & (t != 0.0)).any() == (w != 0.0)
    elif name == "holes":
        z = lc.terrain(c)
        assert abs(float(np.isnan(z).mean()) - arg[0]) < 0.02 and finite.any()
    elif name == "specials":
        z = lc.terrain(c)
        for v in (np.inf, -np.inf, np.float32(3e30), np.float32(-3e30)):
            assert (z == v).any()
        assert np.isnan(ref["nz"][np.isinf(z)]).all() and np.isfinite(ref["nz"][np.abs(z) == np.float32(3e30)]).all()
    elif name == "few":
        z = lc.terrain(c)
        win = _few_windows(z)
        kinds = set(win.values())
        assert {(1, True), (2, True), (3, True), (3, False)} <= kinds, kinds
        nz = ref["nz"]
        default = [nz[ij] == 1.0 for ij, (n, line) in win.items() if n < 3 or line]
        assert all(default)                                         # cnt < 3, collinear (mid ~ 0), or QR rank < 3
        plane = [nz[ij] for ij, (n, line) in win.items() if n == 3 and not line]
        if arg[0] == 1:
            assert all(v != 1.0 for v in plane)                     # raw moment: 3 points not on a line give their plane
        print(f"{c['name']}: {len(default)} default normals, {sum(v != 1.0 for v in plane)} of {len(plane)} plane normals")
    elif name == "dyadic":
        interior = ref["slope"][5:30, 5:25]
        assert (interior == 1.0).any() and (interior < 0.9).any()
    elif name == "shape":
        assert np.isfinite(ref["traversability"]).any()
    else:
        raise AssertionError(prop)


@pytest.mark.parametrize("case", lc.CASES, ids=lc.IDS)
def test_every_case_can_fail(oracle, case):
    assert case["fails"] and case["props"]
    assert lc.refusal(case) is not None, case["name"]   # the fused kernel refuses it: the literal kernels compute it under AUTO
    for prop in case["props"]:
        _check(oracle, case, prop)


def test_the_table_covers_the_issue_axes():
    ps = [c["params"] for c in lc.CASES]
    have = lambda k, v: any(p.get(k) == v for p in ps)  # noqa: E731
    for k, vals in (("normals_algorithm", (0, 1)), ("normals_positive_axis", (0, 1, 2)), ("step_critical_cells", (1, 4, 1000)),
                    ("slope_critical", (0.0, 1e-6, 0.05, 1.0, math.pi / 2)), ("step_critical", (0.0, 1e-6, 0.12, 10.0)),
                    ("roughness_critical", (0.0, 1e-6, 0.05, 10.0)), ("fuse_weight", (lc.YAML_W, 0.0, -1.0))):
        for v in vals:
            assert have(k, v), (k, v)
    assert any(math.isnan(p.get("fuse_weight", 0.0)) for p in ps)
    assert {c["res"] for c in lc.CASES} == set(lc.RESOLUTIONS)
    assert {c["pos"] for c in lc.CASES} == {(0.0, 0.0), lc.FAR, lc.LV95}
    assert {(c["rows"], c["cols"]) for c in lc.CASES} >= {(256, 256), (1, 1), (7, 9), (130, 50)}
    assert any(c["rows"] == 1 and c["cols"] > 1 for c in lc.CASES) and any(c["cols"] == 1 and c["rows"] > 1 for c in lc.CASES)
    assert max(p.get("step_first_radius", 0.04) + p.get("step_second_radius", 0.04) for p in ps) == pytest.approx(0.3)


# ---- the acos rule -----------------------------------------------------------------------------------------------------------

def _flip_inputs(crit, want=4):
    """Doubles x whose slope value changes with a one-ulp change of the double acos (a float32 rounding midpoint of 1 - theta/crit
    within an ulp of the exact acos), found next to cos of a midpoint."""
    rng = np.random.default_rng(int(crit * 1e6))
    found = []
    while len(found) < want:
        a = np.float32(rng.uniform(0.05, 0.95))
        m = (np.float64(a) + np.float64(np.nextafter(a, np.float32(1)))) / 2      # midpoint of two float32
        x0 = math.cos(crit * (1.0 - m))
        for d in range(-4, 5):
            x = float(np.float64(x0) + d * np.spacing(np.float64(x0)))
            if len(lc.slope_candidates(x, crit, 1)) > 1:
                found.append(x)
                break
    return found


@pytest.mark.parametrize("crit", [1.0, math.pi / 4, 0.436332])
def test_acos_rule_accepts_a_flip_within_an_ulp(crit):
    for x in _flip_inputs(crit):
        c = sorted(lc.slope_candidates(x, crit, 1))
        a, b = (np.uint32(v).view(np.float32) for v in c[:2])
        assert abs(int(c[0]) - int(c[1])) == 1                                 # adjacent floats
        assert lc.slope_explained(x, crit, a, b) == (True, 1)
        assert lc.slope_explained(x, crit, b, a) == (True, 1)


def test_acos_rule_accepts_the_branch_point():
    """theta within an ulp of crit: 0 on one side, the tiny 1 - theta/crit on the other."""
    x = 0.5403023058681398                                                       # cos(1)
    crit = lc._acos_exact(x)
    c = lc.slope_candidates(x, crit, 1)
    assert 0 in c and len(c) > 1
    tiny = np.uint32(max(c)).view(np.float32)
    assert 0.0 < tiny < 1e-15
    assert lc.slope_explained(x, crit, np.float32(0.0), tiny)[0]
    assert not lc.slope_explained(x, crit, np.float32(0.0), np.float32(1e-7))[0]


@pytest.mark.parametrize("crit", [1.0, math.pi / 4, 0.05, 1e-12])
def test_acos_rule_rejects_a_float32_step_elsewhere(crit):
    rng = np.random.default_rng(7)
    n = 0
    for x in rng.uniform(-1.0, 1.0, 400):
        c = lc.slope_candidates(x, crit)
        if len(c) != 1:
            continue
        v = np.uint32(next(iter(c))).view(np.float32)
        for w in (np.nextafter(v, np.float32(2)), np.nextafter(v, np.float32(-1))):
            assert not lc.slope_explained(x, crit, v, w)[0], (x, v, w)
        n += 1
    assert n > 350
    for x in (float("nan"), float("inf"), 1.5, -1.0000001):                      # no acos to explain anything
        assert not lc.slope_explained(x, crit, np.float32(0.0), np.float32(1e-45))[0]


def test_slope_mismatches_splits_cells():
    crit = 1.0
    x = np.array(_flip_inputs(crit, 2) + [0.25, 0.5])
    ref = np.array([lc.slope_expr(lc._acos_exact(v), crit) for v in x], np.float32)
    got = ref.copy()
    got[0] = np.uint32(sorted(lc.slope_candidates(x[0], crit, 1) - {int(ref[0].view(np.uint32))})[0]).view(np.float32)
    got[3] = np.nextafter(ref[3], np.float32(2))
    ok, no = lc.slope_mismatches(x, crit, got, ref)
    assert [c for c, _ in ok] == [0] and no == [3]
