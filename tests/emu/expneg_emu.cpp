// tests/emu/expneg_emu.cpp -- TEST INFRASTRUCTURE: medpy_b200/csrc/gc_expneg.cuh compiled for the host, so that the
// exponential term's exp(-t) can be checked against a high-precision reference without a GPU.
#include "../../medpy_b200/csrc/gc_expneg.cuh"

extern "C" void emu_exp_neg(const double* t, long long n, double* out)
{
    for (long long i = 0; i < n; ++i) out[i] = exp_neg(t[i]);
}
extern "C" void emu_exp_neg_inrange(const double* t, long long n, double* out)
{
    for (long long i = 0; i < n; ++i) out[i] = exp_neg_inrange(t[i]);
}
// the argument x^2 / sigma^2 as the n-link kernels form it (exp_arg, gc_exprange.cuh), then exp_neg
extern "C" void emu_exp_term(const double* x, long long n, double inv_sigma2, double sigma2, double* out)
{
    for (long long i = 0; i < n; ++i) out[i] = exp_neg(exp_arg(x[i], inv_sigma2, sigma2));
}
