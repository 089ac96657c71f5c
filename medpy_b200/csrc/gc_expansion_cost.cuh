// gc_expansion_cost.cuh -- what the alpha-expansion kernels of gc_expansion.cuh and gc_expansion_batch.cuh share: the
// pair-weight planes, the data cost D_p(k), and the per-voxel work of a move and of the energy, which the single-image
// and batch kernels wrap in their own grid loops (DESIGN.md §11).  Device functions only, no kernels.
#pragma once
#include "gc_expansion_pair.cuh"
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

// The move for label `alpha` at voxel v over the current labels: every capacity plane entry of v (0 where no arc) and
// its tr, exactly as mgc_add_tweights_dense + mgc_add_nweights_dense leave them on a fresh handle; returns v's
// add_tweights constant.  x_p = SINK means "p switches to alpha".  c holds v's coordinates within its image, whose axis 0
// has `zext` planes.  Per pair (p, q = p + e_d), the rule P says what it adds seen from p (lower) and from q (upper); a
// voxel labelled alpha has no arcs and no pair contributions.  src_p = D_p(alpha), snk_p = D_p(l_p) + the contributions
// in the order axis 0..nd-1, within an axis the pair where p is the lower end first; then add_tweights(p, src_p, snk_p)
// on tr = 0.
template <int ND, typename P, typename C>
__device__ __forceinline__ double exp_move_voxel(const Lattice& L, const State<double>& S, const C* __restrict__ costs,
                                                 const uint8_t* __restrict__ markers, const uint8_t* __restrict__ labels,
                                                 const ExpWeights& W, const P& pair, int alpha, unsigned v,
                                                 const int (&c)[ND], int zext, double& tr)
{
    const int lp = labels[v];
    const int mk = markers ? markers[v] : 0;
    const double src = exp_cost(costs, L.n, v, alpha, mk);
    double snk = exp_cost(costs, L.n, v, lp, mk);
#pragma unroll
    for (int d = 0; d < ND; ++d) {
        double lo_c = 0.0, up_c = 0.0, fwd = 0.0, bwd = 0.0;
        if (c[d] + 1 < (d == 0 ? zext : L.dim[d]) && lp != alpha)         // p is the lower end of (p, p + e_d)
            pair.lower(W.w[d][v], lp, labels[v + L.stride[d]], alpha, lo_c, fwd);
        if (c[d] > 0 && lp != alpha) {                                      // p is the upper end of (p - e_d, p)
            const unsigned o = v - L.stride[d];
            pair.upper(W.w[d][o], labels[o], lp, alpha, up_c, bwd);
        }
        snk = __dadd_rn(snk, lo_c);
        snk = __dadd_rn(snk, up_c);
        S.cap[2 * d + 1][v] = fwd;
        S.cap[2 * d][v] = bwd;
    }
    return add_tweights_dev(tr, src, snk);
}

// The swap move of (alpha, beta), alpha < beta, at voxel v over the current labels (DESIGN.md §11, "Swap moves"): every
// capacity plane entry of v and its tr, as exp_move_voxel leaves them; returns v's add_tweights constant.  Only voxels
// labelled alpha or beta take part; x_p = SINK means "p takes beta", SOURCE "p takes alpha".  A participant has
// src_p = D_p(beta) and snk_p = D_p(alpha), plus for each neighbour q labelled c: P's swap_fixed(w, c) when q is no
// participant (ts to src_p, tk to snk_p, no arc), else the arc p -> q = P's swap_arc(w).  The sums run in the order axis
// 0..nd-1, within an axis the pair where p is the lower end first; then add_tweights(p, src_p, snk_p) on tr = 0.  Any
// other voxel reads nothing but its label: no arcs, tr = 0 and no constant.
template <int ND, typename P, typename C>
__device__ __forceinline__ double swap_move_voxel(const Lattice& L, const State<double>& S, const C* __restrict__ costs,
                                                  const uint8_t* __restrict__ markers, const uint8_t* __restrict__ labels,
                                                  const ExpWeights& W, const P& pair, int alpha, int beta, unsigned v,
                                                  const int (&c)[ND], int zext, double& tr)
{
    const int lp = labels[v];
    if (lp != alpha && lp != beta) {
#pragma unroll
        for (int d = 0; d < ND; ++d) {
            S.cap[2 * d + 1][v] = 0.0;
            S.cap[2 * d][v] = 0.0;
        }
        return 0.0;
    }
    const int mk = markers ? markers[v] : 0;
    double src = exp_cost(costs, L.n, v, beta, mk);
    double snk = exp_cost(costs, L.n, v, alpha, mk);
#pragma unroll
    for (int d = 0; d < ND; ++d) {
        double lo_s = 0.0, lo_k = 0.0, up_s = 0.0, up_k = 0.0, fwd = 0.0, bwd = 0.0;
        if (c[d] + 1 < (d == 0 ? zext : L.dim[d])) {                      // p is the lower end of (p, p + e_d)
            const int lq = labels[v + L.stride[d]];
            if (lq == alpha || lq == beta) fwd = pair.swap_arc(W.w[d][v], alpha, beta);
            else                           pair.swap_fixed(W.w[d][v], lq, alpha, beta, lo_s, lo_k);
        }
        if (c[d] > 0) {                                                     // p is the upper end of (p - e_d, p)
            const unsigned o = v - L.stride[d];
            const int lq = labels[o];
            if (lq == alpha || lq == beta) bwd = pair.swap_arc(W.w[d][o], alpha, beta);
            else                           pair.swap_fixed(W.w[d][o], lq, alpha, beta, up_s, up_k);
        }
        src = __dadd_rn(src, lo_s);
        src = __dadd_rn(src, up_s);
        snk = __dadd_rn(snk, lo_k);
        snk = __dadd_rn(snk, up_k);
        S.cap[2 * d + 1][v] = fwd;
        S.cap[2 * d][v] = bwd;
    }
    return add_tweights_dev(tr, src, snk);
}

// v's share of E(l): D_p(l_p), then its lower-end pairs in axis order.  c holds v's lattice coordinates; the axis-0 pairs
// are z_pairs', so none crosses a seam of a batch.
template <int ND, typename P, typename C>
__device__ __forceinline__ double exp_energy_voxel(const Lattice& L, const C* __restrict__ costs,
                                                   const uint8_t* __restrict__ markers, const uint8_t* __restrict__ labels,
                                                   const ExpWeights& W, const P& pair, unsigned v, const int (&c)[ND])
{
    const int lp = labels[v];
    double e = exp_cost(costs, L.n, v, lp, markers ? markers[v] : 0);
    if (z_pairs(L, c[0]) & 2u) {
        const int lq = labels[v + L.stride[0]];
        if (lq != lp) e = __dadd_rn(e, pair.energy(W.w[0][v], lp, lq));
    }
#pragma unroll
    for (int d = 1; d < ND; ++d) {
        if (c[d] + 1 < L.dim[d]) {
            const int lq = labels[v + L.stride[d]];
            if (lq != lp) e = __dadd_rn(e, pair.energy(W.w[d][v], lp, lq));
        }
    }
    return e;
}
