// gc_expansion_pair.cuh -- the pair rules of the K-label move kernels (DESIGN.md §11): how one pair enters the move
// graph of an alpha-expansion or an alpha-beta swap and the energy, under Potts (PottsPair) or a label distance V
// (MetricPair, "Label distances").  The move and energy kernels of the voxel, batch and region units are templates over
// the rule, so each rule is an instantiation of its own: the Potts one loads no V and multiplies nothing.
// with_pair_rule picks the cost type and the rule of a handle at launch.
#pragma once
#include "gc_expansion_loop.hpp"

// A rule states what one pair adds to the move graph of alpha, seen from either end, and the pair's energy.  For the pair
// (p, q), p its lower end (the lattice pair p, p + e_d, or the lower region id), a = l_p, b = l_q and weight w:
//   lower(w, a, b, alpha, t, arc)   seen from p (a != alpha): t = t_lo to p's sink link, arc = fwd on arc p -> q
//   upper(w, a, b, alpha, t, arc)   seen from q (b != alpha): t = t_up to q's sink link, arc = bwd on arc q -> p
//   energy(w, a, b)                 the pair's energy when a != b
// The caller zeroes t and arc; a rule writes what the pair adds.
// For the swap move of (alpha, beta) (DESIGN.md §11, "Swap moves"), seen from a participant p (labelled alpha or beta):
//   swap_fixed(w, c, alpha, beta, ts, tk)   neighbour labelled c, not a participant: ts = e(beta, c) to p's src (paid
//                                           at SINK = beta), tk = e(alpha, c) to p's snk (paid at SOURCE = alpha)
//   swap_arc(w, alpha, beta)                neighbour a participant: the arc p -> q, e(alpha, beta) = e(beta, alpha)

// Potts, V = 1 - I: the table of DESIGN.md §11, "One move", with no V load and no multiply
struct PottsPair {
    __device__ __forceinline__ void lower(double w, int a, int b, int, double& t, double& arc) const
    {
        if (b == a) arc = w;
        else t = w;
    }
    __device__ __forceinline__ void upper(double w, int a, int, int alpha, double& t, double& arc) const
    {
        if (a == alpha) t = w;
        else arc = w;
    }
    __device__ __forceinline__ double energy(double w, int, int) const { return w; }
    __device__ __forceinline__ void swap_fixed(double w, int, int, int, double& ts, double& tk) const
    {
        ts = w;
        tk = w;
    }
    __device__ __forceinline__ double swap_arc(double w, int, int) const { return w; }
};

// What one pair (p, q), p its lower end, adds to the move graph of `alpha` under the metric V: `lo` to p's sink link, `up`
// to q's, `fwd` on arc p -> q and `bwd` on arc q -> p.  a = l_p, b = l_q, w the pair's weight, V the K x K distance
// (row-major, read through the read-only cache), e(x, y) = w * V[x][y]:
//   a = b = alpha              nothing
//   a = alpha != b             up = e(alpha, b)
//   a != alpha = b             lo = e(a, alpha)
//   a = b != alpha             fwd = e(a, alpha), bwd = e(alpha, b)
//   a != b, neither alpha      lo = min(e00, e01), up = e00 - lo, fwd = e01 - lo, bwd = max(e10 - up, 0)
// with e00 = e(a, b), e01 = e(a, alpha), e10 = e(alpha, b).  The four cut values are w V of the four outcomes; every entry
// is >= 0 in exact arithmetic (bwd by the triangle inequality through alpha), so the max only clamps a rounding.  V is
// symmetric (the host checks it bit for bit), so e(x, alpha) and e(alpha, x) are one load.  With V = 1 - I this is
// PottsPair bit for bit.
struct ExpPair {
    double lo, up, fwd, bwd;
};

__device__ __forceinline__ double exp_dist(double w, const double* __restrict__ V, int K, int x, int y)
{
    return __dmul_rn(w, __ldg(V + x * K + y));
}

__device__ __forceinline__ ExpPair exp_metric_pair(double w, const double* __restrict__ V, int K, int a, int b, int alpha)
{
    ExpPair r{0.0, 0.0, 0.0, 0.0};
    if (a == alpha) {
        if (b != alpha) r.up = exp_dist(w, V, K, alpha, b);
    } else if (b == alpha) {
        r.lo = exp_dist(w, V, K, a, alpha);
    } else if (a == b) {
        r.fwd = exp_dist(w, V, K, a, alpha);
        r.bwd = r.fwd;
    } else {
        const double e00 = exp_dist(w, V, K, a, b), e01 = exp_dist(w, V, K, a, alpha), e10 = exp_dist(w, V, K, alpha, b);
        r.lo = fmin(e00, e01);
        r.up = __dsub_rn(e00, r.lo);
        r.fwd = __dsub_rn(e01, r.lo);
        r.bwd = fmax(__dsub_rn(e10, r.up), 0.0);
    }
    return r;
}

// A label distance V (K x K, row-major, on the device).  Expansion moves take a metric, each end its half of
// exp_metric_pair; swap moves take any semi-metric (>= 0, symmetric, zero diagonal) and read V directly.
struct MetricPair {
    const double* V;
    int K;

    __device__ __forceinline__ void lower(double w, int a, int b, int alpha, double& t, double& arc) const
    {
        const ExpPair r = exp_metric_pair(w, V, K, a, b, alpha);
        t = r.lo;
        arc = r.fwd;
    }
    __device__ __forceinline__ void upper(double w, int a, int b, int alpha, double& t, double& arc) const
    {
        const ExpPair r = exp_metric_pair(w, V, K, a, b, alpha);
        t = r.up;
        arc = r.bwd;
    }
    __device__ __forceinline__ double energy(double w, int a, int b) const { return exp_dist(w, V, K, a, b); }
    __device__ __forceinline__ void swap_fixed(double w, int c, int alpha, int beta, double& ts, double& tk) const
    {
        ts = exp_dist(w, V, K, beta, c);
        tk = exp_dist(w, V, K, alpha, c);
    }
    __device__ __forceinline__ double swap_arc(double w, int alpha, int beta) const { return exp_dist(w, V, K, alpha, beta); }
};

// f(C{}, rule) with C the cost type of e's planes (float for MGC_F32, else double) and rule MetricPair over e.dist while a
// label distance is set, PottsPair otherwise.  A unit's build and energy hooks launch their kernel inside f.
template <typename F>
void with_pair_rule(const Expansion& e, F&& f)
{
    if (e.have_dist) {
        const MetricPair P{e.dist, e.K};
        if (e.cost_dtype == MGC_F32) f(float{}, P);
        else                         f(double{}, P);
    } else {
        if (e.cost_dtype == MGC_F32) f(float{}, PottsPair{});
        else                         f(double{}, PottsPair{});
    }
}
