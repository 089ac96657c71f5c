"""The exponential term's exp(-t) as host C++ (medpy_b200/csrc/gc_expneg.cuh through tests/emu/expneg_emu.cpp) and the
200-bit references the tests measure it and the device's pow against.  Used by test_expneg_emulation.py (no GPU) and
test_gpu_boundary_domain.py."""
import ctypes
import math
import os
import subprocess

import mpmath
import numpy

HERE = os.path.dirname(os.path.abspath(__file__))
PREC = 200
TINY = 2.0 ** -1074          # the subnormal spacing: the ulp of every result below 2^-1021
_P = ctypes.POINTER(ctypes.c_double)


class ExpNeg:
    """exp_neg / exp_neg_inrange / the whole exponential weight argument -> exp_neg, over float64 arrays."""

    def __init__(self, so):
        self._lib = ctypes.CDLL(so)
        for name in ("emu_exp_neg", "emu_exp_neg_inrange"):
            f = getattr(self._lib, name)
            f.restype = None
            f.argtypes = [_P, ctypes.c_longlong, _P]
        self._lib.emu_exp_term.restype = None
        self._lib.emu_exp_term.argtypes = [_P, ctypes.c_longlong, ctypes.c_double, ctypes.c_double, _P]

    def _run(self, name, t, *args):
        t = numpy.ascontiguousarray(t, dtype=numpy.float64)
        out = numpy.empty_like(t)
        getattr(self._lib, name)(t.ctypes.data_as(_P), t.size, *args, out.ctypes.data_as(_P))
        return out

    def exp_neg(self, t):
        return self._run("emu_exp_neg", t)

    def exp_neg_inrange(self, t):
        return self._run("emu_exp_neg_inrange", t)

    def term(self, x, sigma2):
        """exp_neg of the argument x^2 / sigma2 formed as the kernels form it (inv_sigma2 = 1 / sigma2 as the host forms
        it, gc_api.cu), before the DBL_MIN clamp of g_weight."""
        inv = 1.0 / sigma2 if sigma2 != 0.0 else 0.0
        return self._run("emu_exp_term", x, ctypes.c_double(inv), ctypes.c_double(sigma2))


def build_emu(directory):
    so = os.path.join(str(directory), "libexpneg_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-o", so,
                           os.path.join(HERE, "emu", "expneg_emu.cpp")])
    return ExpNeg(so)


def ulp_of(exact):
    """The spacing of the doubles around the real number `exact` (an mpf): 2^(e - 52) for 2^e <= |exact| < 2^(e + 1),
    and the subnormal spacing 2^-1074 below 2^-1021."""
    if exact == 0:
        return mpmath.mpf(TINY)
    _, e = mpmath.frexp(exact)          # exact = m * 2^e, 0.5 <= |m| < 1
    return mpmath.mpf(2) ** max(int(e) - 53, -1074)


def ulp_error(got, exact):
    """|got - exact| in units of the spacing of the doubles at `exact` (`got` a double, `exact` an mpf)."""
    with mpmath.workprec(PREC):
        return float(abs(mpmath.mpf(float(got)) - exact) / ulp_of(exact))


def exp_neg_exact(t):
    with mpmath.workprec(PREC):
        return mpmath.exp(-mpmath.mpf(float(t)))


def pow_exact(b, s):
    """b ** s for doubles b >= 0 and finite s, at 200 bits."""
    with mpmath.workprec(PREC):
        return mpmath.power(mpmath.mpf(float(b)), mpmath.mpf(float(s)))


def worst_ulps(got, args, exact_fn):
    """The largest ulp_error of got[i] against exact_fn(*args[i])."""
    worst = 0.0
    for g, a in zip(got, args):
        worst = max(worst, ulp_error(g, exact_fn(*a)))
    return worst


def ln2_multiple(k):
    """k * ln 2 rounded to the nearest double."""
    with mpmath.workprec(PREC):
        return float(mpmath.mpf(k) * mpmath.log(2))


def neighbours(x, steps):
    """x and the doubles up to `steps` ulps either side of it."""
    out = [x]
    lo = hi = x
    for _ in range(steps):
        lo = math.nextafter(lo, -math.inf)
        hi = math.nextafter(hi, math.inf)
        out += [lo, hi]
    return out
