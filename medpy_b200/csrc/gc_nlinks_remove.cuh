// gc_nlinks_remove.cuh -- sum_edge calls with negated weights folded into the residual state of a solved lattice graph
// (mgc_remove_nweights_warm / mgc_remove_nweights_dense_warm).
//
// The calls lower capacities: call k is sum_edge(i[k], j[k], -cap[k], -rev_cap[k]) with nonnegative decrements.  On a solved
// graph an arc can carry more flow than its lowered capacity allows; the reference's BK has no defined meaning for that
// (it would run on negative residuals).  The defined result here is the one of a graph built from scratch with the
// decrements subtracted (Kohli and Torr's reparametrisation, DESIGN.md §4.6 "N-link decrements"):
//   0. the grouping of the increment fold, unchanged (k_nlinks_keys / k_weighted_heads / k_nlinks_items, or
//      k_nlinks_dense_heads for the dense form): the grouping kernels already refuse negative and non-finite values;
//   1. k_nlinks_remove_check: every arc pair's residual sum r(i->j) + r(j->i), which equals c(i->j) + c(j->i) under any
//      flow, must cover its total decrement up to NLINK_PAIR_TOL.  It runs before fold_items claims anything, so a failure
//      leaves the handle as it was;
//   2. after the claim, k_nlinks_remove_arcs lowers the two residuals of each pair.  Where a residual would go negative the
//      arc carries d more flow than its new capacity: that flow is cancelled (the residual becomes 0, the reverse one
//      loses d) and the item records the excess change d of its lower end (-d of its upper end);
//   3. the endpoint list, filled in atomic order, is sorted (tails_sort in gc_fold.cu); k_nlinks_remove_voxels visits each
//      endpoint once in ascending order and gathers the excess changes of its at most 2 * ND arcs in a fixed order (no
//      floating-point atomics and no order set by scheduling: the energy is reproducible bit for bit).  It recomputes the
//      arc bits and stores the new excess.  A voxel left with negative excess takes the shortfall from its terminal link:
//      its un-pushed source residual where it has one, and a raise of both terminal links by the rest, which lowers the
//      add_tweights constant;
//   4. fold_items rebuilds the push lists and the next solve starts with a full relabel reset.
#pragma once
#include "gc_nlinks.cuh"

#define FOLD_ERR_PAIRSUM 16     // a pair's total decrement exceeds its residual sum (read back by the second check)

// Relative tolerance of the pair check: a pair passes when its total decrement exceeds its residual sum by at most
// NLINK_PAIR_TOL * max(sum, decrement).  2^-44 is 256 units in the last place of that maximum; DESIGN.md §4.6 gives the
// rounding budget it covers.
#define NLINK_PAIR_TOL 0x1p-44

// the decrements of one arc pair summed in call order: df for lo -> hi, db for hi -> lo (a call (i, j) with i > j names
// the pair from its upper end, so its cap lowers hi -> lo and its rev_cap lo -> hi)
__device__ __forceinline__ void nlink_decrements(const NlinkItem& it, const int* __restrict__ order,
                                                 const int64_t* __restrict__ ids, const double* __restrict__ cap,
                                                 const double* __restrict__ rev, double& df, double& db)
{
    df = 0.0;
    db = 0.0;
    for (int j = it.first; j < it.first + it.count; ++j) {
        const int k = order ? order[j] : j;
        double f = cap[k], b = rev[k];
        if (ids && ids[k] != (int64_t)it.lo) { const double t = f; f = b; b = t; }
        df = __dadd_rn(df, f);
        db = __dadd_rn(db, b);
    }
}

// The residual of the arc tail -> tail +- stride[axis] (fwd: +) for the pair check.  Eager and 4-D handles hold it in
// cap[].  On a lazily built handle a tile that is not materialised (cmat[t] == 0; cmat == nullptr: every tile is) still
// has the build's weight on every arc: no push reaches a tile before it is materialised, and every tile an earlier n-link
// fold edited was claimed by it.  That weight is recomputed from the image as residual_read does (build_weight, or
// exp_caps6 for the exponential term without spacing); |a - b| and max(|a|, |b|) are symmetric, so it is the same double
// from either end of the pair.
template <typename E, int FN, int USE_MAX, int SPACING, bool BATCH>
__device__ __forceinline__ double remove_arc_residual(const LazyResidual<E, FN, USE_MAX, SPACING, BATCH>& A, const Lattice& L,
                                                      const Tiles& TL, const int* __restrict__ cmat, unsigned lo, int axis,
                                                      bool fwd)
{
    const unsigned hi = lo + nlink_pick(L.stride, axis, 3);
    const unsigned v = fwd ? lo : hi;
    int c[3];
    decode<3>(L, v, c);
    const int t = ((c[0] / TILE) * TL.nt[1] + c[1] / TILE) * TL.nt[2] + c[2] / TILE;
    if (!cmat || cmat[t]) return fwd ? nlink_pick(A.S.cap, 2 * axis + 1, 6)[v] : nlink_pick(A.S.cap, 2 * axis, 6)[v];
    const BoundaryParams P = BATCH ? params_at(A.P, L, c[0]) : A.P;      // a batch: the constants of the pair's image
    const bool use_max = USE_MAX >= 0 ? (USE_MAX != 0) : (P.use_max != 0);
    const bool spacing = SPACING >= 0 ? (SPACING != 0) : (P.inv_spacing_on != 0.0);
    const double a = build_val<E>(__ldg(A.img + lo), use_max);
    const E q = __ldg(A.img + hi);
    if (FN == 1 && SPACING == 0) {
        const double b = build_val<E>(q, use_max);
        const double x = exp_term_arg(P, use_max ? fmax(a, b) : fabs(__dsub_rn(a, b)));
        const double t6[6] = {x, x, x, x, x, x};
        double c6[6];
        exp_caps6(t6, false, 1u, c6);
        return c6[0];
    }
    return build_weight<FN, E>(P, a, q, use_max, spacing, nlink_pick(P.spacing, axis, 3));
}

template <int ND, bool BATCH>
__device__ __forceinline__ double remove_arc_residual(const EagerResidual<ND, BATCH>& A, const Lattice& L, const Tiles&, const int*,
                                                      unsigned lo, int axis, bool fwd)
{
    return fwd ? nlink_pick(A.S.cap, 2 * axis + 1, 2 * ND)[lo]
               : nlink_pick(A.S.cap, 2 * axis, 2 * ND)[lo + nlink_pick(L.stride, axis, ND)];
}

// One thread per arc pair: FOLD_ERR_PAIRSUM when df + db > r(lo->hi) + r(hi->lo) beyond the tolerance.  Reads only.
template <typename Access>
__global__ void __launch_bounds__(256)
k_nlinks_remove_check(Access A, Lattice L, Tiles TL, const int* __restrict__ cmat, const NlinkItem* __restrict__ items,
                      const int* __restrict__ ctl, const int* __restrict__ order, const int64_t* __restrict__ ids,
                      const double* __restrict__ cap, const double* __restrict__ rev, int* __restrict__ err)
{
    const int n = ctl[0];
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        const NlinkItem it = items[i];
        double df, db;
        nlink_decrements(it, order, ids, cap, rev, df, db);
        const double have = __dadd_rn(remove_arc_residual(A, L, TL, cmat, it.lo, it.axis, true),
                                      remove_arc_residual(A, L, TL, cmat, it.lo, it.axis, false));
        const double want = __dadd_rn(df, db);
        if (__dsub_rn(want, have) > NLINK_PAIR_TOL * fmax(have, want)) atomicOr(err, FOLD_ERR_PAIRSUM);
    }
}

// One thread per arc pair, after the claim: a = r(lo->hi) - df, b = r(hi->lo) - db.  a < 0: the arc lo -> hi carries
// d = -a more than its new capacity; cancelling it leaves a = 0, b - d, and moves excess d from hi back to lo (dx = d).
// b < 0 is the mirror case (dx = -d).  The check bounded a + b below by minus the tolerance, so what is left negative is
// a rounding: it is clamped to 0.  dx[item] is the excess change of lo (hi changes by -dx); both ends are listed once, in
// the order the atomics give (the host sorts the list before k_nlinks_remove_voxels).
template <int ND>
__global__ void __launch_bounds__(256)
k_nlinks_remove_arcs(Lattice L, State<double> S, const NlinkItem* __restrict__ items, int n, const int* __restrict__ order,
                     const int64_t* __restrict__ ids, const double* __restrict__ cap, const double* __restrict__ rev,
                     double* __restrict__ dx, unsigned* __restrict__ tbits, unsigned* __restrict__ tails,
                     int* __restrict__ ntails)
{
    const int step = (int)(gridDim.x * blockDim.x);
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += step) {
        const NlinkItem it = items[i];
        const unsigned hi = it.lo + nlink_pick(L.stride, it.axis, ND);
        double* __restrict__ cf = nlink_pick(S.cap, 2 * it.axis + 1, 2 * ND);
        double* __restrict__ cb = nlink_pick(S.cap, 2 * it.axis, 2 * ND);
        double df, db;
        nlink_decrements(it, order, ids, cap, rev, df, db);
        double a = __dsub_rn(cf[it.lo], df), b = __dsub_rn(cb[hi], db), d = 0.0;
        if (a < 0) { d = -a; b = __dsub_rn(b, d); a = 0.0; }
        else if (b < 0) { d = b; a = __dadd_rn(a, b); b = 0.0; }
        cf[it.lo] = a > 0 ? a : 0.0;
        cb[hi] = b > 0 ? b : 0.0;
        dx[i] = d;
        nlink_tail_once(it.lo, tbits, tails, ntails);
        nlink_tail_once(hi, tbits, tails, ntails);
    }
}

// the item of the arc pair (lo, axis), or -1: dense form (keys == nullptr, one axis) head[lo]; list form the first sorted
// key lo << 2 | axis, which heads an item if any of its calls had a nonzero decrement
__device__ __forceinline__ int remove_item_of(const unsigned long long* __restrict__ keys, const int* __restrict__ head,
                                              const int* __restrict__ pos, int n, unsigned lo, int axis)
{
    int p = (int)lo;
    if (keys) {
        const unsigned long long key = ((unsigned long long)lo << 2) | (unsigned)axis;
        p = lower_bound(keys, 0, n, key);
        if (p >= n || keys[p] != key) return -1;
    }
    return head[p] ? pos[p] - 1 : -1;
}

// One thread per listed endpoint v, the tails in ascending order.  Its excess changes are summed in a fixed order (arc
// by arc: along each axis v as the lower end, then as the upper end) into e' = e + de and stored; its arc bits are
// recomputed from cap[] (bits are cleared
// as well as set) before any read, as in k_nlinks_reclamp.  e' >= 0: a preflow the solver drains; the terminal link is
// not touched (a needless write would cost a rounding).  e' < 0: the shortfall s = -e' comes from the terminal link:
// f = A.read(v) (f.e = e') moves the absorbed sink flow into f.dk as every fold does, then the un-pushed source residual
// covers min(max(r, 0), s), and the rest is a raise of both terminal links by the same amount, which keeps the cut and
// lowers the constant by it: dk += min(max(r, 0), s) - s, r -= s, e = 0.  keys == nullptr: the dense form, whose only
// axis is `axis`.  The change of the add_tweights constant is summed into one partial per block for fold_items' sum and
// on a batch handle (Access::BATCH) stored per listed endpoint in tail_dk.
template <typename Access>
__global__ void __launch_bounds__(256)
k_nlinks_remove_voxels(Access A, Lattice L, const unsigned long long* __restrict__ keys, const int* __restrict__ head,
                       const int* __restrict__ pos, int ncalls, int axis, const double* __restrict__ dx,
                       const unsigned* __restrict__ tails, const int* __restrict__ ntails, double* __restrict__ partials,
                       double* __restrict__ tail_dk)
{
    constexpr int ND = Access::ND;
    constexpr unsigned ARCS = (1u << (2 * ND)) - 1u;
    const State<double>& S = A.S;
    const int n = *ntails;
    double m = 0.0;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned)n; i += gridDim.x * blockDim.x) {
        const unsigned v = tails[i];
        int c[ND];
        decode<ND>(L, v, c);
        double de = 0.0;
#pragma unroll 1
        for (int q = 0; q < 2 * ND; ++q) {
            const int a = q >> 1;
            const int ca = nlink_pick(c, a);
            const bool up = q & 1;                  // v as the upper end of the pair (lo = v - stride[a])
            if ((keys || a == axis) && (up ? ca > 0 : ca + 1 < nlink_pick(L.dim, a, ND))) {
                const int k = remove_item_of(keys, head, pos, ncalls, up ? v - nlink_pick(L.stride, a, ND) : v, a);
                if (k >= 0) de = up ? __dsub_rn(de, dx[k]) : __dadd_rn(de, dx[k]);
            }
        }
        S.rmask[v] = (uint8_t)((S.rmask[v] & ~ARCS) | nlink_arc_bits<ND>(S, v));
        const double e = __dadd_rn(S.excess[v], de);
        if (de != 0.0) S.excess[v] = e;
        double dk = 0.0;
        if (e < 0) {
            auto f = A.read(v);                       // f.e = e, stored above
            const double s = -f.e;
            const double rp = f.r > 0 ? f.r : 0.0;
            f.dk = __dadd_rn(f.dk, __dsub_rn(rp < s ? rp : s, s));
            f.r = __dsub_rn(f.r, s);
            f.e = 0.0;
            A.write(v, f);
            m = __dadd_rn(m, f.dk);
            dk = f.dk;
        }
        if constexpr (Access::BATCH) tail_dk[i] = dk;
    }
    block_sum_store(m, partials);
}
