// gc_api_kernels.cuh -- kernels launched only by gc_api.cu (split from gc_terms.cuh, whose device functions every unit
// of the lattice C ABI shares): a kernel that is not a template is compiled into every unit that includes its header.
// k_sum_partials is launched by the other units through sum_partials() (gc_handle.cuh).
#pragma once
#include "gc_terms.cuh"

// acc[0] += sum(partials[0..n)) in a fixed order: 256 interleaved chains + tree (deterministic)
__global__ void k_sum_partials(const double* __restrict__ partials, unsigned n, double* __restrict__ acc)
{
    __shared__ double sh[256];
    unsigned tid = threadIdx.x;
    double s = 0.0;
    for (unsigned i = tid; i < n; i += 256) s = __dadd_rn(s, partials[i]);
    sh[tid] = s;
    __syncthreads();
    for (unsigned k = 128; k > 0; k >>= 1) {
        if (tid < k) sh[tid] = __dadd_rn(sh[tid], sh[tid + k]);
        __syncthreads();
    }
    if (tid == 0) acc[0] = __dadd_rn(acc[0], sh[0]);
}
