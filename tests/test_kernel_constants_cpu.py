"""Host-side checks of numeric constants that the CUDA kernels hard-code (no GPU needed)."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED = os.path.join(ROOT, "traversability_estimation_b200", "csrc", "te_fused.cu")


def _acos_coefficients():
    src = open(FUSED).read()
    got = dict(re.findall(r"a\.k_p([0-7]) = B2\(([-0-9.eE]+)\)", src))
    assert sorted(got) == [str(k) for k in range(8)], got
    return [np.float32(float(got[str(k)])) for k in range(8)]


def test_fused_acos_polynomial_meets_its_stated_error():
    """acos2 in te_fused.cu: acos(x) = sqrt(1 - x) * P7(x) on [0, 1], evaluated in float32 (Horner, as the kernel does).
    The slope layer is 1 - acos(n_z)/crit, tolerance 1e-5 relative + 1e-6, for any slope_critical crit.  An error e of theta
    moves the layer by e/crit, so it is the RELATIVE error that has to stay far inside the tolerance: below crit,
    e/crit <= rel * theta/crit <= rel, whatever crit is.  te_fused.cu documents 2.2e-7 absolute / 1.7e-7 relative."""
    p = _acos_coefficients()
    x = np.concatenate([np.linspace(0.0, 1.0, 2_000_001), 1.0 - np.logspace(-7, -1, 200_001)]).astype(np.float32)
    acc = np.full_like(x, p[7])
    for k in range(6, -1, -1):
        acc = (acc * x + p[k]).astype(np.float32)  # FFMA rounds once, mul+add twice: this is the pessimistic evaluation
    approx = (np.sqrt((np.float32(1.0) - x).astype(np.float32)).astype(np.float32) * acc).astype(np.float32)
    exact = np.arccos(x.astype(np.float64))
    err = np.abs(approx.astype(np.float64) - exact)
    assert err.max() < 4.0e-7, err.max()
    rel = err[exact > 1e-3] / exact[exact > 1e-3]
    assert rel.max() < 3.0e-7, rel.max()
    assert approx[x == 1.0].max() == 0.0  # flat cells: slope layer exactly 1


def test_footprint_slope_threshold_constant():
    """checkForSlope's nSlopesCritical = floor(2 * (3 res) * (maxGapWidth / 3) / res^2) (TraversabilityMap.cpp:871-873) is
    29 at 0.02 m — the double expression evaluates to 29.999999999999996 — and 20 at 0.03 m; the oracle and the CUDA
    predicate kernel must evaluate it in this operand order."""
    def ncrit(res, gap=0.3):
        return int(np.floor(2.0 * (3.0 * res) * (gap / 3.0) / (res * res)))
    assert ncrit(0.02) == 29 and ncrit(0.03) == 20


def test_slope_stream_acos_constant_bank_coefficients_meet_their_stated_error():
    """k_slope_stream in te_generic.cu: acos(|x|) = sqrt(1 - |x|) * P14(|x|) in double.  The kernel rounds 1 - theta/critical
    to float32 only when it stands 1e-12 (times max(1, 1/critical)) clear of a rounding boundary and documents
    |error| <= 5.1e-14 rad for the polynomial, a 20-fold margin: check the coefficients the kernel holds in constant memory
    against an 80-bit reference (acos as 2 asin(sqrt((1 - a)/2)), which is well conditioned towards a = 1), evaluated with the
    kernel's Horner order in double."""
    src = open(os.path.join(ROOT, "traversability_estimation_b200", "csrc", "te_generic.cu")).read()
    body = re.search(r"c_acos14\[15\] = \{([^}]*)\}", src).group(1)
    c = [float(t) for t in body.replace("\n", " ").split(",")]
    assert len(c) == 15
    if np.finfo(np.longdouble).eps > 1e-18:
        import pytest
        pytest.skip("no extended-precision long double on this host")
    a = np.concatenate([np.linspace(0.0, 1.0, 2_000_001), 1.0 - np.logspace(-12, -1, 200_001)])
    p = np.full_like(a, c[0])
    for k in c[1:]:
        p = p * a + k          # double rounding per step: the pessimistic evaluation of the kernel's DFMAs
    theta = np.sqrt(1.0 - a) * p
    la = a.astype(np.longdouble)
    exact = 2 * np.arcsin(np.sqrt((1 - la) / 2))
    err = np.abs(theta.astype(np.longdouble) - exact)
    assert float(err.max()) <= 5.2e-14, float(err.max())
    assert theta[a == 1.0].max() == 0.0


def _nz_check_limit(crit):
    """Restates nz_check_limit() in te_fused.cu: the s = 1 - n_z below which finish_normal2 certifies the float32 rounding of
    n_z (k_nz_check), for slope_critical = crit: every theta up to just past crit below 1 rad, the calibrated 7.2e-5 from 1 rad."""
    import math
    if not crit < 1.0:
        return 7.2e-5
    t = 1.02 * crit + 2.0 ** -22 / math.sin(crit)
    return max(7.2e-5, 2.0 * math.sin(0.5 * t) ** 2)


SLOPE_CRITS = (1.3, 1.0, 0.999, np.pi / 4, 0.5, 0.436332, 0.3, 0.2, 0.1, 0.05)


def test_nz_rounding_check_covers_every_sensitive_nz():
    """Exhaustive over the float32 n_z in [0.5, 1): where the fused kernel does not certify the float32 rounding of n_z
    (s = 1 - n_z >= k_nz_check), one ulp of n_z must move the slope layer max(0, 1 - acos(n_z)/crit) by at most half its
    tolerance 1e-5 |layer| + 1e-6 (the tolerance of the smaller layer of the pair), including a step across the layer's 0
    branch.  At crit = 1 rad the band is the calibrated 7.2e-5 (DESIGN.md §4.1: 0.46 x tolerance measured on the 8192^2 map),
    so the YAML outputs keep every bit; below it the 7.2e-5 literal the kernel held before did not hold (ratios up to 24).
    Below 1 rad the band reaches past crit, which also covers the several-ulp fp32 error of n_z away from a rounding boundary."""
    src = open(FUSED).read()
    assert "a.k_nz_check = B2(nz_check_limit(p.slope_crit));" in src
    assert "lo(s) < A.k_nz_check" in src and "7.2e-5f" not in src
    n = 0.5 + np.arange(2 ** 23, dtype=np.float64) * 2.0 ** -24   # every float32 in [0.5, 1), ascending
    theta = np.arccos(n)
    worst = {}
    for crit in SLOPE_CRITS:
        thr = np.float32(_nz_check_limit(crit))                      # B2(): the kernel constant is the float32 rounding
        if crit >= 1.0:
            assert thr == np.float32(7.2e-5), thr
        assert thr < 0.5                                             # the check assumes the 2^-24 spacing of [0.5, 1)
        layer = np.maximum(0.0, 1.0 - theta / crit)
        move = layer[1:] - layer[:-1]                                # one ulp of n_z up from n[k]
        ratio = move / (1e-5 * layer[:-1] + 1e-6)
        # s >= thr is not checked: n_z = float32(1 - s) <= float32(1 - thr); a pair with its lower member there is exposed
        unchecked = n[:-1] <= float(np.float32(np.float32(1.0) - thr))
        worst[crit] = float(ratio[unchecked].max())
        assert worst[crit] <= 0.5, (crit, float(thr), worst[crit])
        old = ratio[n[:-1] <= float(np.float32(np.float32(1.0) - np.float32(7.2e-5)))].max()
        assert (old > 1.0) == (0.44 > crit), (crit, float(old))     # the band the literal left exposed beyond the tolerance
        if crit < 1.0:                                               # the band reaches past crit: the layer is 0 beyond it
            assert np.arccos(1.0 - float(thr)) > crit
    print(worst)
