// gc_exprange.cuh -- the range test of the exponential term's argument, per pair and per staged image block.
//
// The exponential boundary term without spacing has a fast path: where every argument t = x^2 / sigma^2 is <= 700 and
// not NaN, exp_neg_inrange gives exp_neg's doubles without any range handling, and every weight is >= DBL_MIN.  The
// lazy graph build (gc_build.cuh) needs no weight at all on that path -- rmask holds only the validity bits -- so it
// asks once per staged block instead of once per pair: block_exp_ordinary() on the min and max of the block's cells.
//
// Plain inline functions, compiled for the device by nvcc and for the host by tests/emu/exprange_emu.cpp, which checks
// on random and adversarial blocks that a block that passes holds no pair whose own test fails.
#pragma once
#include <cmath>
#include <cstring>

#if defined(__CUDACC__)
#define ER_HD __host__ __device__ __forceinline__
#else
#define ER_HD inline
#endif

// correctly rounded float64 operations (the host build compiles with -ffp-contract=off)
ER_HD double er_sub(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
ER_HD double er_mul(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
ER_HD double er_div(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// x of the pair (a, b) -- the values of its two cells as the build reads them (|I| under use_max): |a - b|, or
// max(|a|, |b|) under use_max
ER_HD double exp_pair_x(double a, double b, bool use_max)
{
    return use_max ? fmax(a, b) : fabs(er_sub(a, b));
}

// the argument x^2 / sigma^2 as g_weight<1> forms it: a product with the reciprocal while that is a positive number
// below 1e300, else the exact division by sigma2 = pow(sigma, 2) (so sigma == 0 still gives NaN for x == 0)
ER_HD double exp_arg(double x, double inv_sigma2, double sigma2)
{
    return (inv_sigma2 > 0.0 && inv_sigma2 < 1e300) ? er_mul(er_mul(x, x), inv_sigma2) : er_div(er_mul(x, x), sigma2);
}

// the per-pair test: the argument lies where exp_neg_inrange is exact (<= 700; NaN compares false)
ER_HD bool exp_arg_ordinary(double t)
{
    return t <= 700.0;
}

// One cell into a block's range: lo / hi over the cells that are not NaN, `nan` set by any that is.  Start from
// lo = +inf, hi = -inf, nan = false.
template <typename E>
ER_HD void block_range_add(E& lo, E& hi, bool& nan, E x)
{
    nan = nan || !(x == x);
    lo = x < lo ? x : lo;
    hi = x > hi ? x : hi;
}

// Whether every pair of cells of a block whose cells lie in [lo, hi] (as doubles; none NaN unless `nan`) passes the
// per-pair test.  Only the product form of the argument is taken (0 < inv_sigma2 < 1e300); otherwise no block passes.
//
// Why a block that passes holds no pair that fails, for cells a, b of the block:
//  * |a - b|: a - b lies in [lo - hi, hi - lo], and rounding to nearest is monotone and odd, so |RN(a - b)| <= RN(hi - lo);
//  * use_max: the build reads |I|, and max(|a|, |b|) <= max(|lo|, |hi|);
//  * x -> RN(RN(x * x) * c) is monotone on x >= 0 for c > 0, so the pair's argument is <= the block's;
//  * an infinite cell makes hi - lo or max(|lo|, |hi|) infinite or NaN, a NaN cell sets `nan`: either fails the test.
// With the same arithmetic on both sides the block's argument is an upper bound of every pair's, rounding included.
ER_HD bool block_exp_ordinary(double lo, double hi, bool nan, bool use_max, double inv_sigma2)
{
    if (nan || !(inv_sigma2 > 0.0 && inv_sigma2 < 1e300)) return false;
    const double x = use_max ? fmax(fabs(lo), fabs(hi)) : fabs(er_sub(hi, lo));
    return exp_arg_ordinary(er_mul(er_mul(x, x), inv_sigma2));
}

// The constant of the range test of a block whose staged box touches the images b0 .. b1 of a batch, whose exponential
// terms use sigma2[b] = pow(sigma_b, 2): the largest of their reciprocals 1 / sigma2[b] (formed as the host forms
// inv_sigma2), or 0 -- no block passes -- when one of them does not take the product form.  block_exp_ordinary is
// monotone in that constant (x -> RN(RN(x * x) * c) is monotone in c >= 0), so a block that passes under the largest
// constant passes under each image's own, and every pair lies inside one image: no pair of the block fails.
ER_HD double exp_table_inv_max(const double* sigma2, int b0, int b1)
{
    double m = 0.0;
    for (int b = b0; b <= b1; ++b) {
        const double inv = sigma2[b] != 0.0 ? er_div(1.0, sigma2[b]) : 0.0;
        if (!(inv > 0.0 && inv < 1e300)) return 0.0;
        m = inv > m ? inv : m;
    }
    return m;
}

// Order-preserving integer key of a float32's bits: key(a) < key(b) as signed ints whenever a < b, -0 just below +0, a
// positive NaN above +inf and a negative NaN below -inf.  The map is its own inverse.  The float32 block range of the lazy
// build reduces these keys with integer min / max (one instruction each, and __reduce_min_sync / __reduce_max_sync across
// a warp) instead of comparing floats and tracking NaN separately.
ER_HD int er_f32_key(int bits)
{
    return bits ^ ((bits >> 31) & 0x7fffffff);
}

// block_exp_ordinary on the smallest and largest key of a float32 block: the same verdict as the float fold above (lo /
// hi can differ from it only in the sign of a zero, which neither |hi - lo| nor max(|lo|, |hi|) sees)
ER_HD bool block_exp_ordinary_keys(int kmin, int kmax, bool use_max, double inv_sigma2)
{
    const bool nan = kmax > er_f32_key(0x7f800000) || kmin < er_f32_key((int)0xff800000u);
    float lo, hi;
    const int blo = er_f32_key(kmin), bhi = er_f32_key(kmax);
#if defined(__CUDA_ARCH__)
    lo = __int_as_float(blo);
    hi = __int_as_float(bhi);
#else
    memcpy(&lo, &blo, 4);
    memcpy(&hi, &bhi, 4);
#endif
    return block_exp_ordinary((double)lo, (double)hi, nan, use_max, inv_sigma2);
}
