// gc_expansion_cost.cuh -- what the alpha-expansion kernels of gc_expansion.cuh and gc_expansion_batch.cuh share: the
// pair-weight planes and the data cost D_p(k) (DESIGN.md §11).  Device functions only, no kernels.
#pragma once
#include "gc_terms.cuh"

struct ExpWeights {
    const double* w[4];      // canonical axes
};

template <typename C>
__device__ __forceinline__ double exp_cost(const C* __restrict__ costs, unsigned n, unsigned v, int k, int mark)
{
    double d = (double)costs[(size_t)k * n + v];
    if (mark && mark - 1 != k) d = __dadd_rn(d, 65535.0);
    return d;
}
