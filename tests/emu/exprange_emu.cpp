// tests/emu/exprange_emu.cpp -- TEST INFRASTRUCTURE: medpy_b200/csrc/gc_exprange.cuh compiled for the host, so that the
// block range test of the lazy graph build can be checked against the per-pair test without a GPU.
#include "../../medpy_b200/csrc/gc_exprange.cuh"

// the value of a cell as the build reads it (build_val in gc_build.cuh): |I| in the image's type under use_max
template <typename E> static double cell_val(E x, bool use_max) { return (double)(use_max ? std::fabs(x) : x); }

// 1 when the block of n cells passes block_exp_ordinary (the fold the build kernel runs over its staged block)
template <typename E> static int block_ok(const E* cells, long long n, int use_max, double inv_sigma2)
{
    E lo = (E)INFINITY, hi = (E)-INFINITY;
    bool nan = false;
    for (long long i = 0; i < n; ++i) block_range_add<E>(lo, hi, nan, cells[i]);
    return block_exp_ordinary((double)lo, (double)hi, nan, use_max != 0, inv_sigma2) ? 1 : 0;
}

// 1 when every ordered pair of cells (a cell with itself included) passes the per-pair test
template <typename E> static int pairs_ok(const E* cells, long long n, int use_max, double inv_sigma2, double sigma2)
{
    for (long long i = 0; i < n; ++i) {
        const double a = cell_val<E>(cells[i], use_max != 0);
        for (long long j = 0; j < n; ++j) {
            const double b = cell_val<E>(cells[j], use_max != 0);
            if (!exp_arg_ordinary(exp_arg(exp_pair_x(a, b, use_max != 0), inv_sigma2, sigma2))) return 0;
        }
    }
    return 1;
}

extern "C" int emu_block_ok_f32(const float* c, long long n, int use_max, double inv_sigma2) { return block_ok<float>(c, n, use_max, inv_sigma2); }
extern "C" int emu_block_ok_f64(const double* c, long long n, int use_max, double inv_sigma2) { return block_ok<double>(c, n, use_max, inv_sigma2); }
extern "C" int emu_pairs_ok_f32(const float* c, long long n, int use_max, double inv_sigma2, double sigma2)
{
    return pairs_ok<float>(c, n, use_max, inv_sigma2, sigma2);
}
extern "C" int emu_pairs_ok_f64(const double* c, long long n, int use_max, double inv_sigma2, double sigma2)
{
    return pairs_ok<double>(c, n, use_max, inv_sigma2, sigma2);
}
