// gc_expneg.cuh -- exp(-t) of the exponential boundary term, for t >= 0.
//
// Plain inline functions, compiled for the device by nvcc and for the host by tests/emu/expneg_emu.cpp, which checks them
// against a 200-bit reference over the whole domain, branch points and special values included.  The device code is the
// intrinsics below; the host build (-ffp-contract=off) performs the same correctly rounded operations.
#pragma once
#include "gc_exprange.cuh"

ER_HD double er_fma(double a, double b, double c)
{
#if defined(__CUDA_ARCH__)
    return __fma_rn(a, b, c);
#else
    return std::fma(a, b, c);
#endif
}
ER_HD double er_rint(double x) { return rint(x); }
ER_HD int er_hi(double x)
{
#if defined(__CUDA_ARCH__)
    return __double2hiint(x);
#else
    long long b;
    memcpy(&b, &x, 8);
    return (int)(b >> 32);
#endif
}
ER_HD int er_lo(double x)
{
#if defined(__CUDA_ARCH__)
    return __double2loint(x);
#else
    long long b;
    memcpy(&b, &x, 8);
    return (int)(unsigned)b;
#endif
}
ER_HD double er_hilo(int hi, int lo)
{
#if defined(__CUDA_ARCH__)
    return __hiloint2double(hi, lo);
#else
    const long long b = (long long)(((unsigned long long)(unsigned)hi << 32) | (unsigned)lo);
    double x;
    memcpy(&x, &b, 8);
    return x;
#endif
}

// the Taylor coefficients 1/k! of e^r, k = 0 .. 13: constant memory on the device, a plain array on the host
#define EXPN_COEFFS                                                                                                       \
    1.0, 1.0, 0.5, 1.6666666666666666e-01, 4.1666666666666664e-02, 8.3333333333333332e-03, 1.3888888888888889e-03,       \
        1.9841269841269841e-04, 2.4801587301587302e-05, 2.7557319223985893e-06, 2.7557319223985888e-07,                  \
        2.5052108385441720e-08, 2.0876756987868100e-09, 1.6059043836821613e-10
#if defined(__CUDACC__)
__constant__ double EXPN_C[14] = {EXPN_COEFFS};
#endif
ER_HD double expn_c(int k)
{
#if defined(__CUDA_ARCH__)
    return EXPN_C[k];
#else
    static const double c[14] = {EXPN_COEFFS};
    return c[k];
#endif
}

// exp(-t) for t >= 0 in ~25 instructions (CUDA's general exp() costs ~80 here, and K1 is bound by instruction issue):
// n = rint(-t*log2 e), r = -t - n*ln2 (two-step, exact product with the hi part), e^r by a degree-13 Taylor polynomial in
// Horner form (|r| <= 0.347: truncation 4e-18), result scaled by 2^n through the exponent field.  <= 1 ulp from the
// exact value on [0, 708.39] (normal results), and <= 1 unit of the subnormal spacing above; the (rare) subnormal range
// is scaled in two steps with one rounding, like ldexp; t > 745.2 gives 0 like exp does (the caller turns 0 into DBL_MIN,
// energy_voxel.py:235), +inf gives 0, NaN propagates.
ER_HD double exp_neg(double t)
{
    // branch-free: the three independent evaluations a voxel needs (+z, +y, +x pair) can be interleaved by the scheduler,
    // which hides the latency of the dependent DFMA chain.  Out-of-range arguments are computed on a clamped value and
    // selected away at the end.
    const double y = fmax(-t, -800.0);                       // NaN -> -800 here, restored by the last select
    const double n = er_rint(er_mul(y, 1.4426950408889634));
    double r = er_fma(-n, 6.93147180369123816490e-01, y);
    r = er_fma(-n, 1.90821492927058770002e-10, r);
    double p = expn_c(13);
#pragma unroll
    for (int k = 12; k >= 0; --k) p = er_fma(p, r, expn_c(k));
    const int ni = (int)n;
    const bool tiny = ni < -1020;                             // result (nearly) subnormal: scale in two exact/rounded-once steps
    const unsigned adj = (unsigned)(tiny ? ni + 64 : ni);
    double res = er_hilo((int)((unsigned)er_hi(p) + (adj << 20)), er_lo(p));
    res = er_mul(res, tiny ? 5.42101086242752217004e-20 : 1.0);      // 2^-64: one rounding, like ldexp
    res = (t <= 745.2) ? res : 0.0;
    return (t != t) ? t : res;
}

// The same function for arguments known to lie in [0, 700] (no NaN): none of the range handling, bit-identical results
// (y = -t needs no clamp, n >= -1010 keeps the scaled result normal, so the exponent-field add is exact and the result is
// positive -- no DBL_MIN clamp either).  Callers establish the range for the whole warp with one vote.
ER_HD double exp_neg_inrange(double t)
{
    const double y = -t;
    const double n = er_rint(er_mul(y, 1.4426950408889634));
    double r = er_fma(-n, 6.93147180369123816490e-01, y);
    r = er_fma(-n, 1.90821492927058770002e-10, r);
    double p = expn_c(13);
#pragma unroll
    for (int k = 12; k >= 0; --k) p = er_fma(p, r, expn_c(k));
    return er_hilo(er_hi(p) + ((int)n << 20), er_lo(p));
}
