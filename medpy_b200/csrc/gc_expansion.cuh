// gc_expansion.cuh -- kernels of the alpha-expansion unit (gc_expansion.cu, DESIGN.md §11): a K-label segmentation cut
// as a sequence of binary moves (alpha-expansions or alpha-beta swaps) on the eager lattice handle.  Launched by
// gc_expansion.cu only.
//
// The labelling energy E(l) = sum_p D_p(l_p) + sum_pairs w_pq V(l_p, l_q):
//   D_p(k)  cost plane k at p widened to double, + GCGraph.MAX (65535) when p is marked with a label other than k
//   w_pq    the float64 weight graph_from_voxels puts on both arcs of the pair: k_boundary's own output, kept per axis in
//           w[d][p] for the pair (p, p + e_d) (0 on the last plane of d)
//   V       Potts (V = 1 - I) or a metric label distance (DESIGN.md §11, "Label distances"): the pair rule P
//           (gc_expansion_pair.cuh) the move and energy kernels are instantiated with
#pragma once
#include "gc_expansion_cost.cuh"

// One move for label `alpha`: exp_move_voxel at every voxel, the add_tweights constant as one fixed-order partial per
// block (summed by k_sum_partials)
template <typename P, typename C, int ND>
__global__ void __launch_bounds__(256)
k_exp_move(Lattice L, State<double> S, const C* __restrict__ costs, const uint8_t* __restrict__ markers,
           const uint8_t* __restrict__ labels, ExpWeights W, int alpha, double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[ND];
        decode<ND>(L, v, c);
        double tr = 0.0;
        m = __dadd_rn(m, exp_move_voxel<ND>(L, S, costs, markers, labels, W, pair, alpha, v, c, L.dim[0], tr));
        S.tr[v] = tr;
    }
    block_sum_store(m, partials);
}

// labels <- alpha where the cut put the voxel on the SINK side (mask 0); *switched += the voxels that changed
__global__ void __launch_bounds__(256)
k_exp_apply(unsigned n, const uint8_t* __restrict__ mask, uint8_t* __restrict__ labels, int alpha,
            unsigned long long* __restrict__ switched)
{
    unsigned cnt = 0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += step) {
        if (!mask[v] && labels[v] != alpha) { labels[v] = (uint8_t)alpha; ++cnt; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(switched, (unsigned long long)cnt);
}

// One swap move of (alpha, beta): swap_move_voxel at every voxel, the constant as k_exp_move forms it
template <typename P, typename C, int ND>
__global__ void __launch_bounds__(256)
k_swap_move(Lattice L, State<double> S, const C* __restrict__ costs, const uint8_t* __restrict__ markers,
            const uint8_t* __restrict__ labels, ExpWeights W, int alpha, int beta, double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[ND];
        decode<ND>(L, v, c);
        double tr = 0.0;
        m = __dadd_rn(m, swap_move_voxel<ND>(L, S, costs, markers, labels, W, pair, alpha, beta, v, c, L.dim[0], tr));
        S.tr[v] = tr;
    }
    block_sum_store(m, partials);
}

// labels of alpha or beta <- beta where the cut put the element on the SINK side (mask 0), alpha elsewhere; *switched +=
// the elements that changed
__global__ void __launch_bounds__(256)
k_swap_apply(unsigned n, const uint8_t* __restrict__ mask, uint8_t* __restrict__ labels, int alpha, int beta,
             unsigned long long* __restrict__ switched)
{
    unsigned cnt = 0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += step) {
        const int l = labels[v];
        if (l != alpha && l != beta) continue;
        const int to = mask[v] ? alpha : beta;
        if (l != to) { labels[v] = (uint8_t)to; ++cnt; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(switched, (unsigned long long)cnt);
}

// E(l) per block in a fixed order (exp_energy_voxel in grid-stride order); k_sum_partials adds the partials in a fixed
// order, so the same labels give the same bits
template <typename P, typename C, int ND>
__global__ void __launch_bounds__(256)
k_exp_energy(Lattice L, const C* __restrict__ costs, const uint8_t* __restrict__ markers, const uint8_t* __restrict__ labels,
             ExpWeights W, double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[ND];
        decode<ND>(L, v, c);
        m = __dadd_rn(m, exp_energy_voxel<ND>(L, costs, markers, labels, W, pair, v, c));
    }
    block_sum_store(m, partials);
}

// Initial labels: `init` where given (*bad = 1 where it contradicts a marker), else argmin_k D_p(k), ties to the lowest k
template <typename C>
__global__ void __launch_bounds__(256)
k_exp_init(unsigned n, int K, const C* __restrict__ costs, const uint8_t* __restrict__ markers,
           const uint8_t* __restrict__ init, uint8_t* __restrict__ labels, int* __restrict__ bad)
{
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += step) {
        const int mk = markers ? markers[v] : 0;
        int best = 0;
        if (init) {
            best = init[v];
            if (mk && mk - 1 != best) *bad = 1;
        } else {
            double bd = exp_cost(costs, n, v, 0, mk);
            for (int k = 1; k < K; ++k) {
                const double d = exp_cost(costs, n, v, k, mk);
                if (d < bd) { bd = d; best = k; }
            }
        }
        labels[v] = (uint8_t)best;
    }
}

// *bad = 1 where a cost is negative, NaN or infinite
template <typename C>
__global__ void __launch_bounds__(256)
k_exp_check_costs(unsigned n, const C* __restrict__ cost, int* __restrict__ bad)
{
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += step) {
        const double x = (double)cost[v];
        if (!(x >= 0.0) || isinf(x)) *bad = 1;
    }
}

// *bad = 1 where a label image entry exceeds `limit`
__global__ void __launch_bounds__(256)
k_exp_check_u8(unsigned n, const uint8_t* __restrict__ a, int limit, int* __restrict__ bad)
{
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += step)
        if (a[v] > limit) *bad = 1;
}
