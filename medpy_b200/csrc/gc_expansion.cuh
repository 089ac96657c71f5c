// gc_expansion.cuh -- kernels of the alpha-expansion unit (gc_expansion.cu, DESIGN.md §11): a K-label Potts segmentation
// cut as a sequence of binary moves on the eager lattice handle.  Launched by gc_expansion.cu only.
//
// The labelling energy E(l) = sum_p D_p(l_p) + sum_pairs w_pq [l_p != l_q]:
//   D_p(k)  cost plane k at p widened to double, + GCGraph.MAX (65535) when p is marked with a label other than k
//   w_pq    the float64 weight graph_from_voxels puts on both arcs of the pair: k_boundary's own output, kept per axis in
//           w[d][p] for the pair (p, p + e_d) (0 on the last plane of d)
//
// With a label distance V (DESIGN.md §11, "Label distances") the pair term is w_pq V(l_p, l_q): k_exp_move_m and
// k_exp_energy_m.
#pragma once
#include "gc_expansion_cost.cuh"
#include "gc_expansion_metric.cuh"

// One move for label `alpha` over the current labels: writes the eager handle's state exactly as mgc_add_tweights_dense +
// mgc_add_nweights_dense leave it on a fresh handle -- every capacity plane entry (0 where no arc), tr, and the
// add_tweights constant as one fixed-order partial per block (summed by k_sum_partials).  x_p = SINK means "p switches to
// alpha".  Per pair (p, q = p + e_d), by case:
//   l_p = l_q = alpha              nothing
//   exactly one end is alpha       w to the non-alpha end's sink link
//   l_p = l_q != alpha             arcs p->q and q->p of capacity w
//   l_p != l_q, neither is alpha   w to p's sink link, arc q->p of capacity w
// src_p = D_p(alpha), snk_p = D_p(l_p) + the contributions in the order axis 0..nd-1, within an axis the pair where p is
// the lower end first; then add_tweights(p, src_p, snk_p) on tr = 0.
template <typename C, int ND>
__global__ void __launch_bounds__(256)
k_exp_move(Lattice L, State<double> S, const C* __restrict__ costs, const uint8_t* __restrict__ markers,
           const uint8_t* __restrict__ labels, ExpWeights W, int alpha, double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[ND];
        decode<ND>(L, v, c);
        const int lp = labels[v];
        const int mk = markers ? markers[v] : 0;
        const double src = exp_cost(costs, L.n, v, alpha, mk);
        double snk = exp_cost(costs, L.n, v, lp, mk);
#pragma unroll
        for (int d = 0; d < ND; ++d) {
            double lo_c = 0.0, up_c = 0.0, fwd = 0.0, bwd = 0.0;
            if (c[d] + 1 < L.dim[d] && lp != alpha) {            // p is the lower end of (p, p + e_d)
                const double w = W.w[d][v];
                if (labels[v + L.stride[d]] == lp) fwd = w;
                else lo_c = w;
            }
            if (c[d] > 0 && lp != alpha) {                       // p is the upper end of (p - e_d, p)
                const unsigned o = v - L.stride[d];
                const double w = W.w[d][o];
                if (labels[o] == alpha) up_c = w;
                else bwd = w;
            }
            snk = __dadd_rn(snk, lo_c);
            snk = __dadd_rn(snk, up_c);
            S.cap[2 * d + 1][v] = fwd;
            S.cap[2 * d][v] = bwd;
        }
        double tr = 0.0;
        m = __dadd_rn(m, add_tweights_dev(tr, src, snk));
        S.tr[v] = tr;
    }
    block_sum_store(m, partials);
}

// k_exp_move with the pair term w_pq V(l_p, l_q) of a metric label distance (DESIGN.md §11, "Label distances"): each pair
// adds what exp_metric_pair says, in k_exp_move's order and to its planes.  A voxel labelled alpha has no arcs and no
// pair contributions, as there.
template <typename C, int ND>
__global__ void __launch_bounds__(256)
k_exp_move_m(Lattice L, State<double> S, const C* __restrict__ costs, const uint8_t* __restrict__ markers,
             const uint8_t* __restrict__ labels, ExpWeights W, const double* __restrict__ V, int K, int alpha,
             double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[ND];
        decode<ND>(L, v, c);
        const int lp = labels[v];
        const int mk = markers ? markers[v] : 0;
        const double src = exp_cost(costs, L.n, v, alpha, mk);
        double snk = exp_cost(costs, L.n, v, lp, mk);
#pragma unroll
        for (int d = 0; d < ND; ++d) {
            double lo_c = 0.0, up_c = 0.0, fwd = 0.0, bwd = 0.0;
            if (c[d] + 1 < L.dim[d] && lp != alpha) {            // p is the lower end of (p, p + e_d)
                const ExpPair r = exp_metric_pair(W.w[d][v], V, K, lp, labels[v + L.stride[d]], alpha);
                lo_c = r.lo;
                fwd = r.fwd;
            }
            if (c[d] > 0 && lp != alpha) {                       // p is the upper end of (p - e_d, p)
                const unsigned o = v - L.stride[d];
                const ExpPair r = exp_metric_pair(W.w[d][o], V, K, labels[o], lp, alpha);
                up_c = r.up;
                bwd = r.bwd;
            }
            snk = __dadd_rn(snk, lo_c);
            snk = __dadd_rn(snk, up_c);
            S.cap[2 * d + 1][v] = fwd;
            S.cap[2 * d][v] = bwd;
        }
        double tr = 0.0;
        m = __dadd_rn(m, add_tweights_dev(tr, src, snk));
        S.tr[v] = tr;
    }
    block_sum_store(m, partials);
}

// k_exp_energy with w_pq V(l_p, l_q) in place of w_pq for a lower-end pair whose labels differ
template <typename C, int ND>
__global__ void __launch_bounds__(256)
k_exp_energy_m(Lattice L, const C* __restrict__ costs, const uint8_t* __restrict__ markers, const uint8_t* __restrict__ labels,
               ExpWeights W, const double* __restrict__ V, int K, double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[ND];
        decode<ND>(L, v, c);
        const int lp = labels[v];
        double e = exp_cost(costs, L.n, v, lp, markers ? markers[v] : 0);
#pragma unroll
        for (int d = 0; d < ND; ++d) {
            if (c[d] + 1 < L.dim[d]) {
                const int lq = labels[v + L.stride[d]];
                if (lq != lp) e = __dadd_rn(e, exp_dist(W.w[d][v], V, K, lp, lq));
            }
        }
        m = __dadd_rn(m, e);
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

// E(l) per block in a fixed order (each voxel: D_p(l_p), then its lower-end pairs in axis order); k_sum_partials adds
// the partials in a fixed order, so the same labels give the same bits
template <typename C, int ND>
__global__ void __launch_bounds__(256)
k_exp_energy(Lattice L, const C* __restrict__ costs, const uint8_t* __restrict__ markers, const uint8_t* __restrict__ labels,
             ExpWeights W, double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[ND];
        decode<ND>(L, v, c);
        const int lp = labels[v];
        double e = exp_cost(costs, L.n, v, lp, markers ? markers[v] : 0);
#pragma unroll
        for (int d = 0; d < ND; ++d)
            if (c[d] + 1 < L.dim[d] && labels[v + L.stride[d]] != lp) e = __dadd_rn(e, W.w[d][v]);
        m = __dadd_rn(m, e);
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
