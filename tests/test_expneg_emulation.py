"""The exponential boundary term's exp(-t) without a GPU: medpy_b200/csrc/gc_expneg.cuh compiled as host C++
(tests/emu/expneg_emu.cpp) against a 200-bit reference (mpmath).

exp_neg is a hand-written degree-13 polynomial with the scaling by 2^n done in the exponent field, a separate two-step
scaling for (nearly) subnormal results and a cut-off at t = 745.2; exp_neg_inrange is the same function without the range
handling, which the build uses where a whole warp's arguments lie in [0, 700].  Checked here:
  * <= 1 ulp of the exact exp(-t) on dense samples of [0, 708.39] (normal results), and <= 1 unit of the subnormal
    spacing 2^-1074 above, up to the cut-off;
  * the same bound a few ulps either side of every branch point: 1020.5 ln2 (the two-step scaling starts, n = -1021),
    1022 ln2 (results turn subnormal), 1074 ln2 and 1075 ln2 (the smallest subnormal, the underflow to 0), 745.2 (the
    cut-off), and of every point (k + 1/2) ln2 where n = rint(-t log2 e) steps;
  * special values: +inf -> 0, NaN -> NaN, +-0 -> 1;
  * exp_neg_inrange(t) has exp_neg(t)'s bits on [0, 700], 700 included.
numpy's exp is not correctly rounded either (it differs from the rounded 200-bit value on about 4% of uniform samples), so
the reference is mpmath, not numpy."""
import math

import numpy
import pytest

import expneg_ref as ref

T_NORMAL = 708.39            # below 1022 ln2 = 708.3964...: every exp(-t) is normal
T_CUT = 745.2


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return ref.build_emu(tmp_path_factory.mktemp("expneg"))


def _worst(emu, t):
    t = numpy.asarray(t, dtype=numpy.float64)
    w = emu.exp_neg(t)
    return ref.worst_ulps(w, [(x,) for x in t], ref.exp_neg_exact)


def test_dense_normal_range(emu):
    rng = numpy.random.default_rng(1)
    t = numpy.concatenate([rng.uniform(0.0, T_NORMAL, 20000), 10.0 ** rng.uniform(-30, 0, 2000),
                           numpy.linspace(0.0, T_NORMAL, 4001)])
    worst = _worst(emu, t)
    assert worst <= 1.0, worst


def test_dense_subnormal_range(emu):
    """Errors in units of the subnormal spacing: the result's ulp there, whatever its size."""
    rng = numpy.random.default_rng(2)
    t = numpy.concatenate([rng.uniform(T_NORMAL, T_CUT, 20000), numpy.linspace(T_NORMAL, T_CUT, 2001)])
    w = emu.exp_neg(t)
    assert (w >= 0.0).all()
    worst = ref.worst_ulps(w, [(x,) for x in t], ref.exp_neg_exact)
    assert worst <= 1.0, worst


@pytest.mark.parametrize("point", ["1020.5ln2", "1022ln2", "1074ln2", "1075ln2", "745.2", "700", "708.39"])
def test_branch_points(emu, point):
    """32 ulps either side of the point, and a few relative offsets from 1e-15 to 1e-9."""
    x = float(point) if "ln2" not in point else ref.ln2_multiple(float(point[:-3]))
    t = ref.neighbours(x, 32) + [x * (1.0 + s * 10.0 ** -e) for s in (-1, 1) for e in range(9, 16)]
    t = [v for v in t if v <= T_CUT]
    worst = _worst(emu, t)
    assert worst <= 1.0, (point, worst)
    # above the cut-off the function is 0, as the correctly rounded exp(-t) is there
    if point == "745.2":
        above = [v for v in ref.neighbours(x, 32) if v > T_CUT] + [745.3, 746.0, 800.0, 1e300]
        assert (emu.exp_neg(above) == 0.0).all()


def test_every_step_of_n(emu):
    """Either side of each (k + 1/2) ln2, where the reduction's n = rint(-t log2 e) steps from -k to -(k + 1): the
    reduced argument r sits at the end of its interval, where the polynomial's truncation error is largest."""
    t = [v for k in range(0, 1075) for v in ref.neighbours(ref.ln2_multiple(k + 0.5), 1)]
    t = [v for v in t if v <= T_CUT]
    worst = _worst(emu, t)
    assert worst <= 1.0, worst


def test_special_values(emu):
    w = emu.exp_neg([math.inf, math.nan, -math.nan, 0.0, -0.0])
    assert w[0] == 0.0 and not math.copysign(1.0, w[0]) < 0
    assert math.isnan(w[1]) and math.isnan(w[2])
    assert w[3] == 1.0 and w[4] == 1.0
    # the smallest arguments: exp(-t) rounds to 1 or to the double just below it
    tiny = numpy.array([5e-324, 1e-300, 2.0 ** -53, 2.0 ** -52, 1e-10])
    assert numpy.array_equal(emu.exp_neg(tiny), numpy.exp(-tiny))


def test_inrange_has_the_same_bits_on_0_700(emu):
    rng = numpy.random.default_rng(3)
    t = numpy.concatenate([rng.uniform(0.0, 700.0, 400000), 10.0 ** rng.uniform(-320, 2.845, 20000),
                           numpy.array(ref.neighbours(700.0, 64)), numpy.array([0.0, 5e-324, 2.2250738585072014e-308]),
                           numpy.array([v for k in range(0, 1010) for v in ref.neighbours(ref.ln2_multiple(k + 0.5), 2)])])
    t = t[(t >= 0.0) & (t <= 700.0)]
    assert t.max() == 700.0
    a, b = emu.exp_neg(t), emu.exp_neg_inrange(t)
    bad = numpy.flatnonzero(a.view(numpy.int64) != b.view(numpy.int64))
    assert bad.size == 0, (t[bad[:5]], a[bad[:5]], b[bad[:5]])
    assert (b >= 2.2250738585072014e-308).all()      # no DBL_MIN clamp is needed on the fast path
