"""The cases of the literal-kernel tests (test_literal_params_gpu.py, test_literal_params_cpu.py), and the rule by which a slope cell
may differ from the oracle's.

The literal kernels (KERNEL_GENERIC, and te_normals / te_step / te_roughness / te_slope) restate the oracle's double arithmetic
operation for operation, so every layer but the slope must equal the oracle's bit for bit.  The slope layer is
float32(theta < crit ? 1 - theta / crit : 0) with theta the double acos of n_z: CUDA's acos and glibc's may differ in the last
bits of theta, and where that moves the float32 result the two layers may differ by one step.  `slope_explained` accepts such a cell
only where the exact acos (mpmath, 50 digits) lies within ACOS_ULPS double ulps of a decision of the expression: a float32 rounding
midpoint of 1 - theta / crit, or the branch point theta == crit.

Each case records in `fails` what makes it able to fail, and in `props` the oracle properties test_literal_params_cpu.py asserts so
that the record holds (a property name, or (name, argument))."""
import functools
import math

import numpy as np

import synth

YAML_W = float(np.float32(1.0) / np.float32(3.0))
LV95 = (2_600_000.25, 1_200_000.75)
FAR = (12.5, -3.25)
RESOLUTIONS = (0.02, 0.025, 0.03, 0.05, 0.07, 0.1)

# Largest error of the double acos in ulps: 2 for CUDA's (CUDA C++ Programming Guide, double-precision functions), 1 for glibc's.
ACOS_ULPS = 2


# ---- the acos rule ---------------------------------------------------------------------------------------------------------------

def slope_expr(theta, crit):
    """The reference's slope value of a double theta, in IEEE double and float32 as SlopeFilter.cpp evaluates it."""
    theta, crit = np.float64(theta), np.float64(crit)
    with np.errstate(all="ignore"):
        return np.float32(np.float64(1.0) - theta / crit) if theta < crit else np.float32(0.0)


@functools.lru_cache(maxsize=None)
def _acos_exact(x):
    import mpmath
    with mpmath.workdps(50):
        return float(mpmath.acos(mpmath.mpf(x)))   # the double nearest the exact acos


def slope_candidates(x, crit, ulps=ACOS_ULPS):
    """The float32 values the slope expression takes for every double within `ulps` ulps of acos(x) (x finite, |x| <= 1)."""
    t = _acos_exact(float(x))
    lo = hi = np.float64(t)
    out = {slope_expr(t, crit).view(np.uint32).item()}
    for _ in range(ulps):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        out.add(slope_expr(lo, crit).view(np.uint32).item())
        out.add(slope_expr(hi, crit).view(np.uint32).item())
    return out


def slope_explained(x, crit, got, ref):
    """(ok, k): got != ref is explained by acos when both are values the expression takes within k <= ACOS_ULPS ulps of the exact
    acos of x; k is the least such distance (how close the cell lies to a decision)."""
    x = float(x)
    if not math.isfinite(x) or abs(x) > 1.0:
        return False, None
    g, r = np.float32(got).view(np.uint32).item(), np.float32(ref).view(np.uint32).item()
    for k in range(1, ACOS_ULPS + 1):
        c = slope_candidates(x, crit, k)
        if g in c and r in c:
            return True, k
    return False, None


def slope_mismatches(x, crit, got, ref):
    """Cells where the float32 slope layers got and ref differ (NaN matches NaN), split into (explained [(index, k)], unexplained
    [index]) by slope_explained."""
    x, got, ref = (np.asarray(a).reshape(-1) for a in (x, got, ref))
    bad = np.nonzero((got.view(np.uint32) != ref.view(np.uint32)) & ~(np.isnan(got) & np.isnan(ref)))[0]
    ok, no = [], []
    for c in bad:
        e, k = slope_explained(float(x[c]), crit, got[c], ref[c])
        (ok.append((int(c), k)) if e else no.append(int(c)))
    return ok, no


# ---- terrain ---------------------------------------------------------------------------------------------------------------------

def _rel(rows, cols, res, pos):
    """Cell-centre coordinates relative to the map position, as (rows, cols) arrays."""
    x = synth.cell_positions(rows, res, pos[0]) - pos[0]
    y = synth.cell_positions(cols, res, pos[1]) - pos[1]
    return np.broadcast_to(x[:, None], (rows, cols)), np.broadcast_to(y[None, :], (rows, cols))


def few_valid(rows, cols, res, seed):
    """NaN everywhere but groups of valid cells 9 cells apart: one cell, two, three in a line (on a line in 3-D too: equal
    heights), and three not on a line.  Every window of radius <= 1.5 cells sees one group at most."""
    rng = np.random.default_rng(seed)
    z = np.full((rows, cols), np.nan, np.float32)
    groups = [[(0, 0)], [(0, 0), (0, 1)], [(0, -1), (0, 0), (0, 1)], [(0, 0), (0, 1), (1, 0)]]
    q = 0
    for a in range(2, rows - 2, 9):
        for b in range(2, cols - 2, 9):
            h = np.float32(rng.uniform(-0.2, 0.2))
            for k, (da, db) in enumerate(groups[q % 4]):
                z[a + da, b + db] = h if q % 4 != 3 else np.float32(h + 0.01 * k * res / 0.02)
            q += 1
    return z


def terrain(c):
    """The elevation map of case c (float32, column-major)."""
    rows, cols, res, pos, kind, seed = c["rows"], c["cols"], c["res"], c["pos"], c["terrain"], c["seed"]
    if kind in ("gentle", "mixed", "rough"):
        z = synth.terrain(rows, cols, res, seed, kind, pos)
    elif kind == "pyramid":   # tilted in +x, -x, +y and -y: each axis flips some normals
        x, y = _rel(rows, cols, res, pos)
        z = (0.4 * np.abs(x - 0.1) + 0.3 * np.abs(y + 0.05)).astype(np.float32) + synth.fbm(rows, cols, res, seed, 0.05, position=pos)
    elif kind == "dyadic":    # an exactly representable tilted plane and an exactly flat plateau
        i, j = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
        z = (0.125 * i + 0.0625 * j).astype(np.float32) * np.float32(0.02)
        z[rows // 4:rows // 2, cols // 4:cols // 2] = np.float32(0.5)
    elif kind == "few":
        z = few_valid(rows, cols, res, seed)
    else:
        raise ValueError(kind)
    z = np.array(z, np.float32)
    rng = np.random.default_rng(seed + 1)
    if c.get("holes"):
        z[rng.random(z.shape) < c["holes"]] = np.nan
    if c.get("specials") and z.size > 64:
        for v in (np.inf, -np.inf, 3e30, -3e30):
            z.flat[rng.integers(0, z.size, 3)] = np.float32(v)
    return np.asfortranarray(z)


# ---- the cases -------------------------------------------------------------------------------------------------------------------

def _case(name, fails, props, rows=256, cols=256, res=0.02, pos=(0.0, 0.0), terrain="pyramid", seed=1, holes=0.0, specials=False,
          **params):
    return dict(name=name, fails=fails, props=tuple(props), rows=rows, cols=cols, res=res, pos=pos, terrain=terrain, seed=seed,
                holes=holes, specials=specials, params=params)


def _cases():
    C = []
    # normals: both algorithms x every positive axis, on terrain tilted both ways along x and y
    for alg in (0, 1):
        for axis in (0, 1, 2):
            res = RESOLUTIONS[alg * 3 + axis]
            C.append(_case(f"alg{alg}-axis{axis}", f"some n[{axis}] < 0 before the flip; the axis changes the normals",
                           [("axis", axis)] + ([("alg",)] if axis == 2 else []), rows=254 if axis == 2 else 256, res=res,
                           pos=(FAR, (0.0, 0.0), LV95)[axis],
                           seed=10 + axis, holes=0.05 if alg else 0.0, normals_algorithm=alg, normals_positive_axis=axis,
                           normals_radius=2.5 * res, roughness_radius=2.5 * res))
    # normals radii: 0, half a cell, exactly 1, 2, 3 cells, a reach of 4 and of 10 cells (windows over 64 cells)
    for q, (k, rmul) in enumerate(((0, 0.0), (0, 0.5), (1, 1.0), (2, 2.0), (3, 3.0), (4, 4.3), (10, 10.2))):
        res = RESOLUTIONS[q % 6]
        r = rmul * res
        props = [("radius_zero",)] if k == 0 else []
        if rmul == float(k) and k:
            props.append(("on_circle", "normals_radius", k))
        if k == 10:
            props.append(("big",))
        C.append(_case(f"normals-r{rmul:g}res-alg{q % 2}", f"normals window of {rmul:g} cells" + (
            ": cells at distance exactly r decided both ways" if rmul == k and k else ""), props or [("alg",)],
            rows=254 if q in (0, 2) else 256, res=res,
            pos=((0.0, 0.0), FAR, LV95)[q % 3], terrain=("mixed", "rough")[q % 2], seed=20 + q, normals_algorithm=q % 2,
            normals_radius=r, roughness_radius=r if q % 2 else 0.05))
    # a reach of exactly k cells that floor(r / res) misses: r = k * res * (1 - 1e-9), at LV95 inside on some centres only
    C.append(_case("normals-below-2res-lv95", "floor(r/res) = 1 but cells at offset 2 pass the circle test on some centres",
                   [("generous", "normals_radius", 2)], res=0.05, pos=LV95, terrain="mixed", seed=30, normals_algorithm=1,
                   normals_radius=2 * 0.05 * (1 - 1e-9), roughness_radius=2 * 0.05 * (1 - 1e-9)))
    C.append(_case("roughness-radius-differs", "roughness radius 0.09 against normals radius 0.03",
                   [("param", "roughness_radius", "roughness", 0.03)], res=0.03, pos=FAR, terrain="rough", seed=31,
                   normals_radius=0.03, roughness_radius=0.09))
    # step windows chosen independently
    for q, (r1, r2) in enumerate(((0.0, 0.04), (0.04, 0.0), (0.0, 0.0), ("2res", "3res"), (0.1, 0.2), (0.2, 0.1))):
        res = (0.02, 0.025, 0.03, 0.05, 0.05, 0.1)[q]
        a = 2 * res if r1 == "2res" else r1
        b = 3 * res if r2 == "3res" else r2
        props = [("param", "step_first_radius", "step", 0.04) if a == 0 else ("param", "step_second_radius", "step", 0.04)]
        if r1 == "2res":
            props += [("on_circle", "step_first_radius", 2), ("on_circle", "step_second_radius", 3)]
        C.append(_case(f"step-r1={a:g}-r2={b:g}", f"step windows {a:g} / {b:g} m at {res} m", props, res=res,
                       pos=((0.0, 0.0), FAR, LV95)[q % 3], terrain="rough", seed=40 + q,
                       normals_radius=3 * res, roughness_radius=3 * res, step_first_radius=a, step_second_radius=b,
                       step_critical=0.05))
    for ncrit in (1, 4, 1000):
        C.append(_case(f"step-cells-{ncrit}", f"step_critical_cells {ncrit} changes the step layer", [("ncrit", ncrit)],
                       res=0.025, terrain="rough", seed=50, normals_algorithm=1, step_critical_cells=ncrit,
                       step_first_radius=0.05, step_second_radius=0.075, step_critical=0.05))
    # criticals and the fuse weight (raw-moment normals, so that the fused kernel refuses them)
    for v in (0.0, 1e-6, 0.05, 1.0, math.pi / 2):
        C.append(_case(f"slope-crit-{v:g}", "slope_critical changes the slope layer",
                       [("param", "slope_critical", "slope", 0.5)] + ([("zero", "slope")] if v == 0 else []), res=0.025, terrain="rough",
                       seed=60, normals_algorithm=1, slope_critical=v))
    for name, layer, yaml, alt in (("step_critical", "step", 0.12, 0.01), ("roughness_critical", "roughness", 0.05, 0.2)):
        for v in (0.0, 1e-6, yaml, 10.0):
            C.append(_case(f"{name}-{v:g}", f"{name} changes the {layer} layer",
                           [("param", name, layer, alt if v > 1e-3 else 10.0)] + ([("zero", layer)] if v == 0 else []), res=0.02, terrain="rough", seed=61,
                           normals_positive_axis=1, **{name: v}, **({"roughness_radius": 0.06} if v == yaml else {})))
    for w in (YAML_W, 0.0, -1.0, float("nan")):
        C.append(_case(f"fuse-{w:g}", "the weight scales every traversability cell", [("fuse", w)], res=0.03, terrain="mixed",
                       seed=62, normals_algorithm=1, fuse_weight=w))
    # terrain: holes, non-finite and huge elevations, too few valid cells, exact planes
    for q, d in enumerate((0.0, 0.05, 0.5, 0.95)):
        C.append(_case(f"holes-{d:g}", f"NaN holes at density {d:g}", [("holes", d)], res=0.03, pos=FAR, terrain="gentle", seed=70 + q,
                       holes=d, normals_algorithm=1, normals_positive_axis=q % 3))
    C.append(_case("specials", "+-inf and +-3e30 cells: invalid cells and float32-overflowing moments", [("specials",)], res=0.02,
                   terrain="mixed", seed=75, specials=True, normals_algorithm=1))
    for alg in (0, 1):
        C.append(_case(f"few-valid-alg{alg}", "windows with 1, 2, 3 collinear and 3 non-collinear valid cells",
                       [("few", alg)], rows=130, cols=50, res=0.02, terrain="few", seed=80 + alg, normals_algorithm=alg,
                       normals_radius=0.03, roughness_radius=0.03))
    C.append(_case("dyadic-plane", "exact planes: the fixture's rank test decides on rounding noise", [("dyadic",)], rows=130, cols=96,
                   res=0.02, terrain="dyadic", seed=85))
    # awkward shapes and positions (rows % 4 != 0 refuses the fused kernel at the YAML parameters)
    for q, (rows, cols) in enumerate(((1, 1), (1, 37), (41, 1), (7, 9), (130, 50))):
        C.append(_case(f"shape-{rows}x{cols}", "windows clipped by every map edge", [("shape",)], rows=rows, cols=cols,
                       res=RESOLUTIONS[q], pos=((0.0, 0.0), FAR, LV95)[q % 3], terrain="mixed" if min(rows, cols) > 8 else "gentle",
                       seed=90 + q))
    return C


def refusal(c):
    """Why fused_eligible refuses case c (None: it may accept it)."""
    p, res = c["params"], c["res"]
    get = lambda k, d: p.get(k, d)  # noqa: E731
    if get("normals_algorithm", 0) != 0:
        return "raw-moment normals"
    if get("normals_positive_axis", 2) != 2:
        return "positive axis not z"
    if c["rows"] % 4:
        return "rows % 4 != 0"
    if not all(get(k, d) > 0 for k, d in (("slope_critical", 1.0), ("step_critical", 0.12), ("roughness_critical", 0.05))):
        return "a critical of 0"
    rn, rr = get("normals_radius", 0.05), get("roughness_radius", 0.05)
    if rn != rr:
        return "roughness window differs from the normals window"
    if math.floor(rn / res) > 2:
        return "normals reach over 2 cells"
    return None


CASES = _cases()
IDS = [c["name"] for c in CASES]


def params(mod, c, **over):
    """The ChainParams of `mod` (the library or the oracle) of case c, with the fields `over` set."""
    p = mod.ChainParams.yaml_defaults(0)
    for k, v in {**c["params"], **over}.items():
        setattr(p, k, v)
    return p


def geometry(mod, c):
    return mod.Geometry.make(c["rows"], c["cols"], c["res"], c["pos"])


# ---- two refused parameter sets of the batched, slab and position tests ----------------------------------------------------------

OTHER_SETS = {
    "raw-axis0": dict(normals_algorithm=1, normals_positive_axis=0),
    "reach4": dict(normals_radius=4.3 * 0.02, roughness_radius=4.3 * 0.02, step_first_radius=0.05, step_second_radius=0.03),
}
