// gc_region_expansion.cuh -- kernels of the region alpha-expansion unit (gc_region_expansion.cu, DESIGN.md §11 "Region
// graphs"): a K-label segmentation of a region adjacency graph, each move cut by the sparse push-relabel (gc_sparse.cuh).
// Launched by gc_region_expansion.cu only.
//
// The graph is the CSR of the region pairs (row, head; each row in ascending neighbour id) with the pair's weight w on
// both of its arcs (wt).  The labelling energy E(l) = sum_r D_r(l_r) + sum_{pairs r<s} w_rs V(l_r, l_s), D_r(k) =
// costs[k * n + r] widened to double (markers are already in the costs), V Potts or a metric label distance: the pair
// rule P (gc_expansion_pair.cuh) the kernels are instantiated with.
#pragma once
#include "gc_expansion_pair.cuh"
#include "gc_terms.cuh"

// One move for label `alpha` over the current labels: writes the sparse solver's state exactly as a fresh mgc_sparse
// would hold it after sum_edge of every pair and add_tweights of every node -- every arc's capacity, tr, and the
// add_tweights constant as one fixed-order partial per block (summed by k_sum_partials).  x_u = SINK means "u switches to
// alpha".  Node u with a = l_u != alpha, arc u->v with b = l_v and weight w, in the row's order: u < v takes P's lower end
// of the pair (u, v), u > v its upper end of the pair (v, u), as (snk_u term, cap(u->v)); every such term is added, +0.0
// included, which can only turn a zero tr's sign (DESIGN.md §11, "Region graphs").  A node labelled alpha has no arcs and
// no pair contributions.  src_u = D_u(alpha), snk_u starts at D_u(a); then add_tweights(u, src_u, snk_u) on
// tr = 0.
template <typename P, typename C>
__global__ void __launch_bounds__(256)
k_rexp_move(int n, const int* __restrict__ row, const int* __restrict__ head, const double* __restrict__ wt,
            const C* __restrict__ costs, const uint8_t* __restrict__ labels, int alpha, double* __restrict__ cap,
            double* __restrict__ tr, double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const int step = gridDim.x * blockDim.x;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += step) {
        const int a = labels[u];
        const double src = (double)costs[(size_t)alpha * n + u];
        double snk = (double)costs[(size_t)a * n + u];
        const int end = row[u + 1];
        for (int e = row[u]; e < end; ++e) {
            double c = 0.0;
            if (a != alpha) {
                const int v = head[e];
                const int b = labels[v];
                double t = 0.0;
                if (u < v) pair.lower(wt[e], a, b, alpha, t, c);
                else       pair.upper(wt[e], b, a, alpha, t, c);
                snk = __dadd_rn(snk, t);
            }
            cap[e] = c;
        }
        double t = 0.0;
        m = __dadd_rn(m, add_tweights_dev(t, src, snk));
        tr[u] = t;
    }
    block_sum_store(m, partials);
}

// One swap move of (alpha, beta) over the current labels (DESIGN.md §11, "Swap moves"), written as k_rexp_move writes a
// move.  Only nodes labelled alpha or beta take part; x_u = SINK means "u takes beta".  A participant u has src_u =
// D_u(beta), snk_u = D_u(alpha); for each arc u -> v in the row's order, v labelled b: P's swap_fixed(w, b) to src_u and
// snk_u when v is no participant (no arc), else cap(u -> v) = P's swap_arc(w); then add_tweights(u, src_u, snk_u) on tr
// = 0.  Any other node has no arcs, tr = 0 and no constant.
template <typename P, typename C>
__global__ void __launch_bounds__(256)
k_rswap_move(int n, const int* __restrict__ row, const int* __restrict__ head, const double* __restrict__ wt,
             const C* __restrict__ costs, const uint8_t* __restrict__ labels, int alpha, int beta, double* __restrict__ cap,
             double* __restrict__ tr, double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const int step = gridDim.x * blockDim.x;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += step) {
        const int a = labels[u];
        const int end = row[u + 1];
        if (a != alpha && a != beta) {
            for (int e = row[u]; e < end; ++e) cap[e] = 0.0;
            tr[u] = 0.0;
            continue;
        }
        double src = (double)costs[(size_t)beta * n + u];
        double snk = (double)costs[(size_t)alpha * n + u];
        for (int e = row[u]; e < end; ++e) {
            const int b = labels[head[e]];
            double c = 0.0, ts = 0.0, tk = 0.0;
            if (b == alpha || b == beta) c = pair.swap_arc(wt[e], alpha, beta);
            else                         pair.swap_fixed(wt[e], b, alpha, beta, ts, tk);
            src = __dadd_rn(src, ts);
            snk = __dadd_rn(snk, tk);
            cap[e] = c;
        }
        double t = 0.0;
        m = __dadd_rn(m, add_tweights_dev(t, src, snk));
        tr[u] = t;
    }
    block_sum_store(m, partials);
}

// E(l) per block in a fixed order (each node: D_u(l_u), then its pairs to higher ids in the row's order); k_sum_partials
// adds the partials in a fixed order, so the same labels give the same bits
template <typename P, typename C>
__global__ void __launch_bounds__(256)
k_rexp_energy(int n, const int* __restrict__ row, const int* __restrict__ head, const double* __restrict__ wt,
              const C* __restrict__ costs, const uint8_t* __restrict__ labels, double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const int step = gridDim.x * blockDim.x;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += step) {
        const int a = labels[u];
        double e = (double)costs[(size_t)a * n + u];
        const int end = row[u + 1];
        for (int k = row[u]; k < end; ++k) {
            const int v = head[k];
            if (v > u) {
                const int b = labels[v];
                if (b != a) e = __dadd_rn(e, pair.energy(wt[k], a, b));
            }
        }
        m = __dadd_rn(m, e);
    }
    block_sum_store(m, partials);
}
