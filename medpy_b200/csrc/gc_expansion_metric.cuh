// gc_expansion_metric.cuh -- the move graph of one pair under a metric label distance V (DESIGN.md §11, "Label
// distances"): the case table the metric move kernels of the voxel, batch and region units share.  Device functions
// only, no kernels.
#pragma once

// What one pair (p, q), p its lower end, adds to the move graph of `alpha`: `lo` to p's sink link, `up` to q's, `fwd` on
// arc p -> q and `bwd` on arc q -> p.  a = l_p, b = l_q, w the pair's weight, V the K x K distance (row-major, read
// through the read-only cache), e(x, y) = w * V[x][y]:
//   a = b = alpha              nothing
//   a = alpha != b             up = e(alpha, b)
//   a != alpha = b             lo = e(a, alpha)
//   a = b != alpha             fwd = e(a, alpha), bwd = e(alpha, b)
//   a != b, neither alpha      lo = min(e00, e01), up = e00 - lo, fwd = e01 - lo, bwd = max(e10 - up, 0)
// with e00 = e(a, b), e01 = e(a, alpha), e10 = e(alpha, b).  The four cut values are w V of the four outcomes; every entry
// is >= 0 in exact arithmetic (bwd by the triangle inequality through alpha), so the max only clamps a rounding.  V is
// symmetric (the host checks it bit for bit), so e(x, alpha) and e(alpha, x) are one load.  With V = 1 - I this is the
// Potts table of gc_expansion.cuh bit for bit.
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
