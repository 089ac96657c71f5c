// tests/emu/exprange_keys_emu.cpp -- TEST INFRASTRUCTURE: the float32 block range of the lazy graph build's lean kernel
// (integer keys, gc_exprange.cuh) next to the float fold it replaces, compiled for the host.
#include <cstdint>
#include "../../medpy_b200/csrc/gc_exprange.cuh"

// the float fold (k_build_tile)
extern "C" int emu_fold_ok_f32(const float* c, long long n, int use_max, double inv_sigma2)
{
    float lo = INFINITY, hi = -INFINITY;
    bool nan = false;
    for (long long i = 0; i < n; ++i) block_range_add<float>(lo, hi, nan, c[i]);
    return block_exp_ordinary((double)lo, (double)hi, nan, use_max != 0, inv_sigma2) ? 1 : 0;
}

// the key fold (k_build_lean): integer min / max of the keys, in any order
extern "C" int emu_keys_ok_f32(const float* c, long long n, int use_max, double inv_sigma2)
{
    int kmin = INT32_MAX, kmax = INT32_MIN;
    for (long long i = 0; i < n; ++i) {
        int b;
        memcpy(&b, &c[i], 4);
        const int k = er_f32_key(b);
        kmin = k < kmin ? k : kmin;
        kmax = k > kmax ? k : kmax;
    }
    return block_exp_ordinary_keys(kmin, kmax, use_max != 0, inv_sigma2) ? 1 : 0;
}

extern "C" int emu_key_f32(const float* c) { int b; memcpy(&b, c, 4); return er_f32_key(b); }
