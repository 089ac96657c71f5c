// gc_nlinks.cuh -- sum_edge calls folded into the residual state of a solved lattice graph (mgc_add_nweights_warm /
// mgc_add_nweights_dense_warm).
//
// BK's sum_edge on a solved graph adds to the RESIDUAL capacities of the two arcs of a pair (a->r_cap += cap;
// a->sister->r_cap += rev_cap, graph.h:456-480) and the next maxflow() continues from that residual graph.  Here the same
// happens to the push-relabel state (DESIGN.md §4.6), with the steps of the t-link folds (gc_seeds.cuh):
//   0. the calls are grouped by arc on the device: key = lower endpoint << 2 | canonical axis, a stable radix sort of
//      (key, call index) pairs keeps the calls of one arc in call order, and a run-length pass makes one NlinkItem per
//      arc that has a nonzero increment (k_nlinks_keys / k_weighted_heads / k_nlinks_items; the dense form flags and
//      compacts the nonzero entries instead, k_nlinks_dense_heads).  On lazily built handles the tiles of BOTH endpoints
//      are listed once each;
//   1. those tiles are materialised before any capacity is written (fold_items), so the materialiser never overwrites an
//      edited arc;
//   2. k_nlinks_fold adds the increments of each arc in call order to the residual capacities cap[2a+1][lo] and cap[2a][hi]
//      and lists every tail whose out-capacity rose once, through a per-voxel bit;
//   3. after every arc update, k_nlinks_reclamp visits each listed tail once: the residual bits of the arcs that became
//      positive are set, and a tail that still holds an un-pushed source residual r(v) > 0 is read and written back through
//      the fold's residual access (LazyResidual / EagerResidual, gc_seeds.cuh), which pushes what the larger out-capacity
//      can carry -- without it that capacity would never see source flow;
//   4. fold_items rebuilds the push lists and the next solve starts with a full relabel reset.
// Only nonnegative, finite increments come here (the grouping checks them before anything is touched); the add_tweights
// constant does not change.
#pragma once
#include "gc_seeds.cuh"

// element k of a small array indexed by a runtime value, unrolled into selects so the kernel parameters stay in registers
// (a dynamic index would copy the whole parameter struct to local memory)
template <int N, typename T>
__device__ __forceinline__ T nlink_pick(const T (&a)[N], int k, int limit = N)
{
    T r = a[0];
#pragma unroll
    for (int x = 1; x < N; ++x)
        if (x < limit && x == k) r = a[x];
    return r;
}

// one arc pair lo -> lo + stride[axis] and its reverse: calls order[first .. first + count) (order == nullptr: the dense
// form, call `first` alone)
struct NlinkItem {
    unsigned lo;
    int axis;
    int first;
    int count;
};

// canonical axis of the pair (lo, lo + d): the axis a with d == stride[a] whose extent lo does not end; -1 if there is none
// (strides of extent-1 axes repeat a larger one, but lo is on their last plane).  Axis 0 takes z_pairs' rule, so on a
// batch lattice a pair across the seam between two images is no pair either.
template <int ND>
__device__ __forceinline__ int nlink_axis(const Lattice& L, unsigned lo, unsigned d)
{
    int c[ND];
    decode<ND>(L, lo, c);
    int a = -1;
#pragma unroll
    for (int k = 0; k < ND; ++k)
        if (d == L.stride[k] && (k == 0 ? (z_pairs(L, c[0]) & 2u) != 0u : c[k] + 1 < L.dim[k])) a = k;
    return a;
}

// list form: key = lo << 2 | axis, value = call index.  Ids out of range, non-neighbour pairs and bad weights set bits of
// *err (such a call gets key 0); the caller reads *err back before anything uses the items.
template <int ND>
__global__ void __launch_bounds__(256) k_nlinks_keys(Lattice L, const int64_t* __restrict__ ii, const int64_t* __restrict__ jj,
                                                     const double* __restrict__ cap, const double* __restrict__ rev, int n,
                                                     unsigned long long* __restrict__ keys, int* __restrict__ vals,
                                                     int* __restrict__ err)
{
    for (int k = (int)(blockIdx.x * blockDim.x + threadIdx.x); k < n; k += (int)(gridDim.x * blockDim.x)) {
        const int64_t i = ii[k], j = jj[k];
        unsigned long long key = 0ull;
        if (i < 0 || j < 0 || i >= (int64_t)L.n || j >= (int64_t)L.n) {
            atomicOr(err, FOLD_ERR_RANGE);
        } else {
            const unsigned lo = (unsigned)(i < j ? i : j);
            const int a = nlink_axis<ND>(L, lo, (unsigned)(i < j ? j - i : i - j));
            if (a < 0) atomicOr(err, FOLD_ERR_PAIR);
            else key = ((unsigned long long)lo << 2) | (unsigned)a;
        }
        const double c = cap[k], r = rev[k];
        if (!isfinite(c) || !isfinite(r)) atomicOr(err, FOLD_ERR_NONFINITE);
        else if (c < 0.0 || r < 0.0) atomicOr(err, FOLD_ERR_NEGATIVE);
        keys[k] = key;
        vals[k] = k;
    }
}

// dense form: 1 where the entry has a nonzero increment; entries on the last plane of the axis name no pair and are ignored
// (as mgc_add_nweights_dense ignores them).  The axis arrives as scalars, so no lattice array is indexed at run time:
// span = stride[axis] * dim[axis] (the stride of the next slower axis, or n for axis 0), span_magic its ceil(2^64 / span)
// (0: p < span for every p, or span == 1), last = span - stride[axis].  p lies on the last plane iff p mod span >= last.
// On a batch lattice axis 0 spans one image (zper * stride[0]), so the last plane of every image is ignored: its entries
// would name pairs across a seam (z_pairs).  Items, decrements and the pair check all come from these heads.
// SLAB: only an increment of an arc whose tail the slab owns counts (fwd: p owned, bwd: p + stride[axis] = p + span - last
// owned), so a pair inside a ghost plane, or one whose owned direction is zero, is no item; every entry is checked.
template <bool SLAB = false>
__global__ void __launch_bounds__(256) k_nlinks_dense_heads(unsigned n, unsigned span, unsigned long long span_magic,
                                                            unsigned last, const double* __restrict__ fwd,
                                                            const double* __restrict__ bwd, int* __restrict__ head,
                                                            int* __restrict__ err, SlabOwn own = {})
{
    for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const unsigned q = span_magic ? (unsigned)__umul64hi((unsigned long long)p, span_magic) : 0u;
        int h = 0;
        if (p - q * span < last) {
            const double f = fwd[p], b = bwd[p];
            if (!isfinite(f) || !isfinite(b)) atomicOr(err, FOLD_ERR_NONFINITE);
            else if (f < 0.0 || b < 0.0) atomicOr(err, FOLD_ERR_NEGATIVE);
            if constexpr (SLAB) h = ((f != 0.0 && own.voxel(p)) || (b != 0.0 && own.voxel(p + span - last))) ? 1 : 0;
            else h = (f != 0.0 || b != 0.0) ? 1 : 0;
        }
        head[p] = h;
    }
}

// sum_edge(i, j, 0, 0) changes nothing, so only arcs with a call of a nonzero increment become items: the list form flags
// the first sorted key of each such arc with k_weighted_heads (gc_seeds.cuh).
// pos = inclusive sum of the heads: the head at i is item pos[i] - 1, in ascending key order, and ctl[0] = pos[n - 1]
// items.  keys == nullptr: the dense form (pair i along `axis`, one call).  The tiles of both endpoints are listed once each
// (claim_tile_once), which keeps the claim list within TL.ntiles (see k_tweights_items); tflag == nullptr lists none (eager
// and 4-D handles).
__global__ void __launch_bounds__(256) k_nlinks_items(Lattice L, Tiles TL, const unsigned long long* __restrict__ keys, int axis,
                                                      const int* __restrict__ pos, int n, NlinkItem* __restrict__ items,
                                                      int* __restrict__ tflag, int* __restrict__ tiles, int* __restrict__ ctl)
{
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        if (i == n - 1) ctl[0] = pos[i];
        if (pos[i] == (i > 0 ? pos[i - 1] : 0)) continue;
        unsigned lo = (unsigned)i;
        int a = axis, cnt = 1;
        if (keys) {
            lo = (unsigned)(keys[i] >> 2);
            a = (int)(keys[i] & 3ull);
            cnt = lower_bound(keys, i, n, keys[i] + 1ull) - i;
        }
        items[pos[i] - 1] = NlinkItem{lo, a, i, cnt};
        if (tflag) {
            claim_tile_once(L, TL, lo, tflag, tiles, ctl);
            claim_tile_once(L, TL, lo + nlink_pick(L.stride, a, 3), tflag, tiles, ctl);
        }
    }
}

// lists tail v once: the first thread that sets its bit (tbits zeroed by the caller) appends it
__device__ __forceinline__ void nlink_tail_once(unsigned v, unsigned* __restrict__ tbits, unsigned* __restrict__ tails,
                                                int* __restrict__ ntails)
{
    const unsigned b = 1u << (v & 31u);
    if (!(atomicOr(&tbits[v >> 5], b) & b)) tails[atomicAdd(ntails, 1)] = v;
}

// One thread per arc pair: the increments added to the two residual capacities in call order, (r + a) + b, as BK's
// sum_edge does.  ids != nullptr: the list form, where a call (i, j) with i > j names the pair from its upper end, so its
// cap is the backward and its rev_cap the forward increment.  A zero increment is skipped (exact: r + 0 == r).  Nothing
// else is written here: the residual bits and the source re-clamp of the tails wait for k_nlinks_reclamp, after every
// arc of the call has its new capacity.  SLAB: an arc whose tail lies in a ghost plane is the neighbour slab's; its
// increments are dropped here, so no ghost voxel is written or listed for the re-clamp (whose source push would land in
// the ghost's excess, the outbox, and reach the neighbour as flow that no source sent).
template <int ND, bool SLAB = false>
__global__ void __launch_bounds__(256)
k_nlinks_fold(Lattice L, State<double> S, const NlinkItem* __restrict__ items, int n, const int* __restrict__ order,
              const int64_t* __restrict__ ids, const double* __restrict__ cap, const double* __restrict__ rev,
              unsigned* __restrict__ tbits, unsigned* __restrict__ tails, int* __restrict__ ntails, SlabOwn own = {})
{
    const int step = (int)(gridDim.x * blockDim.x);
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += step) {
        const NlinkItem it = items[i];
        const unsigned hi = it.lo + nlink_pick(L.stride, it.axis, ND);
        double* __restrict__ cf = nlink_pick(S.cap, 2 * it.axis + 1, 2 * ND);
        double* __restrict__ cb = nlink_pick(S.cap, 2 * it.axis, 2 * ND);
        double rf = cf[it.lo], rb = cb[hi];
        bool up_f = false, up_b = false;
        for (int j = it.first; j < it.first + it.count; ++j) {
            const int k = order ? order[j] : j;
            double f = cap[k], b = rev[k];
            if (ids && ids[k] != (int64_t)it.lo) { const double t = f; f = b; b = t; }
            if (f != 0.0) { rf = __dadd_rn(rf, f); up_f = true; }
            if (b != 0.0) { rb = __dadd_rn(rb, b); up_b = true; }
        }
        if constexpr (SLAB) { up_f = up_f && own.voxel(it.lo); up_b = up_b && own.voxel(hi); }
        if (up_f) { cf[it.lo] = rf; nlink_tail_once(it.lo, tbits, tails, ntails); }
        if (up_b) { cb[hi] = rb; nlink_tail_once(hi, tbits, tails, ntails); }
    }
}

// residual bits of a tail after the arc fold: every arc with capacity (the increments only add, so this only sets bits)
template <int ND>
__device__ __forceinline__ unsigned nlink_arc_bits(const State<double>& S, unsigned v)
{
    unsigned m = 0;
#pragma unroll
    for (int k = 0; k < 2 * ND; ++k)
        if (S.cap[k][v] > 0) m |= 1u << k;
    return m;
}

// One thread per listed tail: the new arc bits ORed into rmask first (4-D eager_write never stores rmask, and residual_write /
// 3-D eager_write keep bits 0..5 of what they read), then a tail with tr > 0 is read and, if r(v) > 0, written back.
// Lazily built handles: residual_read's co[] / lim0 are the capacities of the build, recomputed from the image: they
// describe how tr encodes the pushed source flow, not the current capacities, so they stay right after an n-link edit.
// residual_write then sees the new out-capacity: lim > lim0 pushes min(r, lim) more and keeps tr = u + lim0 (read back as
// u), otherwise source_excess(r, co) >= min(r, lim) as before.  A tail with r(v) <= 0 keeps its state (a rewrite would
// cost a rounding of a voxel with net inflow).  Eager and 4-D handles: tr > 0 is r(v) itself (the record of the first
// solve), and eager_write pushes min(r, lim) of the new out-capacity.  r > 0 needs tr > 0, which holds no sink flow, so
// the add_tweights constant does not move; each block stores a zero partial for fold_items' sum.
template <typename Access>
__global__ void __launch_bounds__(256)
k_nlinks_reclamp(Access A, const unsigned* __restrict__ tails, const int* __restrict__ ntails, double* __restrict__ partials)
{
    const State<double>& S = A.S;
    const int n = *ntails;
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        const unsigned v = tails[i];
        S.rmask[v] = (uint8_t)(S.rmask[v] | nlink_arc_bits<Access::ND>(S, v));
        if (S.tr[v] > 0) {
            const auto f = A.read(v);
            if (f.r > 0) A.write(v, f);
        }
    }
    block_sum_store(0.0, partials);
}
