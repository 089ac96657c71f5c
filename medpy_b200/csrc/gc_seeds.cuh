// gc_seeds.cuh -- seeds added to or erased from a solved lattice graph, and any add_tweights calls, folded into its
// residual state (mgc_add_seeds / mgc_remove_seeds / mgc_add_tweights_warm).
//
// The reference refines a cut by calling add_tweights(v, 65535, 0) / add_tweights(v, 0, 65535) on the new seed voxels of
// a solved GraphDouble and calling maxflow() again, and erases a seed with the inverse call add_tweights(v, -65535, 0) /
// add_tweights(v, 0, -65535): BK's add_tweights (graph.h:415-425) works on the RESIDUAL terminal capacity r(v) that the
// first maxflow() left, and the second maxflow() continues from that residual graph.  Here the same happens to the
// push-relabel state (DESIGN.md §4.6):
//   0. the calls are grouped by voxel on the device into TweightItems {v, first, count} in ascending voxel order, with
//      each touched tile listed once for the claim: seeds as keys v << 1 | bg, radix sorted (k_seed_keys / k_seed_heads);
//      a call list as (voxel, call index) pairs, stably radix sorted (k_tweights_keys / k_weighted_heads); the dense form
//      by a flag per voxel (k_tweights_dense_heads); then a scan and k_tweights_items;
//   1. on lazily built handles the tiles of the touched voxels are materialised first (k_caps_claim / k_caps_tiles), so
//      every touched voxel holds cap[], tr, excess and its sink-link state, and the fold below reads one representation
//      only.  The marker bit planes are never read again for a claimed tile, so they are not updated;
//   2. k_tlink_fold (one thread per item) reads r(v) from that state, replays the voxel's calls with add_tweights_dev --
//      the reference's arithmetic on r -- and writes r' back in the solver's representation.  The residual access is a
//      type: LazyResidual (residual_read / residual_write) on lazily built handles, EagerResidual (eager_read /
//      eager_write) on the others, once MGC_OPT_WARM had the first solve record their residual source capacities (the
//      end of this file).  The calls are a type as well: SeedCalls (the sorted seed keys) or ListCalls (src / snk);
//   3. k_seed_lists / k_seed_lists4 put every tile that holds excess back on the push lists; the next solve starts with a
//      full relabel reset.
#pragma once
#include "gc_build.cuh"
#include "gc_tiles4.cuh"

// error bits of a grouping, read back before anything touches the solver state
#define FOLD_ERR_RANGE 1        // a node id out of range
#define FOLD_ERR_NONFINITE 2    // a NaN or infinite weight
#define FOLD_ERR_PAIR 4         // a pair of ids that are not lattice neighbours (or i == j)
#define FOLD_ERR_NEGATIVE 8     // a negative n-link increment

// The voxels a z-slab handle owns, for the folds on it (DESIGN.md §4.6): local ids [lo, hi), its owned planes; the ghost
// planes lie outside.  A fold applies a t-link call to owned voxels only, and an n-link increment to the arcs whose tail
// is owned; the neighbour slab applies the rest to its own copy.  plane = voxels per axis-0 plane, the stride of axis 0.
// The grouping kernels take it behind a compile-time flag SLAB (false: every voxel is owned, the handle's kernels do not
// test it), as the batch kernels take BATCH.
struct SlabOwn {
    unsigned lo, hi, plane;
    __device__ __forceinline__ bool voxel(unsigned v) const { return v - lo < hi - lo; }
    // a t-link key of the grouping: the voxel itself
    __device__ __forceinline__ bool key(unsigned v) const { return voxel(v); }
    // an n-link key lo << 2 | axis: the pair has an owned end (an axis-0 pair reaches one plane up)
    __device__ __forceinline__ bool key(unsigned long long k) const
    {
        const unsigned v = (unsigned)(k >> 2);
        return (k & 3ull) == 0ull ? v + plane - lo < hi - lo + plane : voxel(v);
    }
};

// One voxel's calls: calls first .. first + count - 1 of the sorted grouping (the dense form: the single call `first`)
struct TweightItem {
    unsigned v;
    int first;
    int count;
    int pad;
};

// grouping keys v << 1 | bg (the lattice has < 2^31 voxels, so a key fits 32 bits); fg ids first, then bg ids.  An id out
// of range sets *err and gets key 0: the caller reads *err back before anything uses the items.
__global__ void __launch_bounds__(256) k_seed_keys(const int64_t* __restrict__ fg, int n_fg, const int64_t* __restrict__ bg,
                                                   int n_bg, int64_t n_vox, unsigned* __restrict__ keys, int* __restrict__ err)
{
    const int n = n_fg + n_bg;
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        const bool b = i >= n_fg;
        const int64_t v = b ? bg[i - n_fg] : fg[i];
        unsigned k = 0u;
        if (v < 0 || v >= n_vox) *err = FOLD_ERR_RANGE;
        else k = ((unsigned)v << 1) | (b ? 1u : 0u);
        keys[i] = k;
    }
}

// first index in [lo, hi) of the sorted keys whose key is >= x
template <typename K>
__device__ __forceinline__ int lower_bound(const K* __restrict__ keys, int lo, int hi, K x)
{
    while (lo < hi) {
        const int mid = lo + ((hi - lo) >> 1);
        if (keys[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// lists the tile of voxel v for the claim unless an earlier item did: tflag[t] (zeroed by the caller) flips once, ctl[2]
// counts the listed tiles
__device__ __forceinline__ void claim_tile_once(const Lattice& L, const Tiles& TL, unsigned v, int* __restrict__ tflag,
                                                int* __restrict__ tiles, int* __restrict__ ctl)
{
    int c[3];
    decode<3>(L, v, c);
    const int t = ((c[0] / TILE) * TL.nt[1] + c[1] / TILE) * TL.nt[2] + c[2] / TILE;
    if (tflag[t] == 0 && atomicExch(&tflag[t], 1) == 0) tiles[atomicAdd(&ctl[2], 1)] = t;
}

// 1 at the first sorted key of each voxel (a run of keys 2v, then 2v + 1); SLAB: of each owned voxel (a seed in a ghost
// plane is the neighbour slab's)
template <bool SLAB = false>
__global__ void __launch_bounds__(256) k_seed_heads(const unsigned* __restrict__ keys, int n, int* __restrict__ head,
                                                    SlabOwn own = {})
{
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        int h = (i == 0 || (keys[i] >> 1) != (keys[i - 1] >> 1)) ? 1 : 0;
        if constexpr (SLAB) h = h && own.voxel(keys[i] >> 1);
        head[i] = h;
    }
}

// Residual terminal capacity r(v) in the state of a materialised voxel (BK's tr_cap after the flow so far):
//   tr > 0 : tr - source_excess(tr, c_orig)   -- the source flow the build (or an earlier fold) pushed is
//            source_excess(tr, c_orig) exactly, c_orig = the voxel's capacities before any flow, from the image copy;
//   tr < 0 : tr + sink[v]                      -- sink capacity -tr minus the flow it absorbed (0 unless RM_SINKV);
//   tr = 0 : 0.
// The fold moves the absorbed flow into the add_tweights constant (it stays counted once: the energy is constant +
// absorbed flow), applies the seeds to r with the reference's arithmetic and writes r' back:
//   r' < 0 : tr = r' (a fresh sink link of capacity -r'), and the voxel's own excess goes through it at once
//            (sink[v] = min(excess, -r'), saturation exact as in the push kernel);
//   r' > 0 : a source residual of r'.  At least p = min(r', residual out-capacity (rounded up) x SOURCE_CLAMP_SLACK)
//            joins the excess -- the clamp of DESIGN.md §4.2 on the residual graph: whatever more the source link could
//            send has to leave through those arcs.  The rest must survive for a later fold (a background seed would count
//            it in the constant).  When that bound is within lim(c_orig) (no net inflow), source_excess(r', c_orig) is
//            pushed and tr = r', the build's own representation, read back exactly.  Otherwise p is pushed and
//            tr = u + lim(c_orig) for the rest u = r' - p > 0, whose source_excess is lim and whose residual reads back
//            as u to one rounding; tr = 0 when u = 0;
//   r' = 0 : tr = 0.
// `cap` is the seed capacity: +65535 adds seeds, -65535 erases them (add_tweights(v, -65535, 0) / (v, 0, -65535)).  An
// erase reaches every sign of r and r', and each branch above only assumes what holds for any sign: once r is read, the
// voxel carries no terminal flow (the absorbed flow is in the constant, the pushed source flow is in the network and out
// of r), so r' is the whole residual terminal capacity whatever produced it.
//   - r' < 0 after an fg erase on a source voxel (r < 65535; BK puts r - 65535 into the constant and leaves a sink link of
//     65535 - r): a fresh sink link, the same state a bg seed on a source voxel leaves;
//   - r' > 0 after a bg erase on a sink voxel, including one that absorbed flow: the sink bits are cleared (nm keeps bits
//     0..5 only), the absorbed flow already sits in the constant and sink[v] is not read without RM_SINKV; lim and lim0
//     depend on the capacities alone, so both sub-branches and their read-back hold as for an fg seed on a sink voxel;
//   - r' > 0 smaller than r after an fg erase on a source voxel: tr = r' with source_excess(r', c_orig) pushed on top of
//     the flow already pushed, which a later fold reads back as r' - source_excess(r', c_orig), the residual on top of
//     all the flow pushed so far;
//   - r' = 0: no terminal link, as for any seed that cancels.
// A materialised voxel's state read as BK's residual terminal capacity (residual_read), and r' written back in the
// solver's representation (residual_write): the two halves of every fold on a lazily built handle (LazyResidual).
struct Residual {
    double co[6];     // capacities before any flow
    double lim0;      // their sum rounded up, x SOURCE_CLAMP_SLACK
    double r;         // r(v); the fold applies its add_tweights calls to it
    double dk;        // change of the add_tweights constant: the absorbed sink flow, then the minima of the calls
    double e;         // excess
    unsigned rm;      // rmask
};

// BATCH: a batch lattice, whose voxels take the term constants of their own image (params_at); false compiles the
// single-image read with P itself.
template <typename E, int FN, int USE_MAX, int SPACING, bool BATCH>
__device__ __forceinline__ Residual residual_read(const Lattice& L, const State<double>& S, const E* __restrict__ img,
                                                  const BoundaryParams& P, unsigned v)
{
    const bool use_max = USE_MAX >= 0 ? (USE_MAX != 0) : (P.use_max != 0);
    const bool spacing = SPACING >= 0 ? (SPACING != 0) : (P.inv_spacing_on != 0.0);
    Residual f;
    int c[3];
    decode<3>(L, v, c);
    // capacities before any flow: the doubles k_caps_tiles computed from the same image copy, with the same term
    // constants (a batch: those of v's image)
    const unsigned valid = z_pairs(L, c[0]) | (c[1] > 0 ? 4u : 0u) | (c[1] + 1 < L.dim[1] ? 8u : 0u) |
                           (c[2] > 0 ? 16u : 0u) | (c[2] + 1 < L.dim[2] ? 32u : 0u);
    const BoundaryParams Pv = BATCH ? params_at(P, L, c[0]) : P;
    const double a = build_val<E>(__ldg(img + v), use_max);
    if (FN == 1 && SPACING == 0) {
        double t6[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            t6[k] = 0.0;
            if ((valid >> k) & 1u) {
                const double b = build_val<E>(__ldg(img + (unsigned)((int)v + dir_offset(L, k))), use_max);
                t6[k] = exp_term_arg(Pv, use_max ? fmax(a, b) : fabs(__dsub_rn(a, b)));
            }
        }
        exp_caps6(t6, false, valid, f.co);     // the general branch: the same doubles for ordinary arguments
    } else {
#pragma unroll
        for (int k = 0; k < 6; ++k)
            f.co[k] = ((valid >> k) & 1u)
                          ? build_weight<FN, E>(Pv, a, __ldg(img + (unsigned)((int)v + dir_offset(L, k))), use_max, spacing,
                                                P.spacing[k >> 1])
                          : 0.0;
    }
    double lim0 = __dadd_ru(0.0, f.co[0]);
    lim0 = __dadd_ru(lim0, f.co[1]); lim0 = __dadd_ru(lim0, f.co[2]); lim0 = __dadd_ru(lim0, f.co[3]);
    lim0 = __dadd_ru(lim0, f.co[4]); lim0 = __dadd_ru(lim0, f.co[5]);
    f.lim0 = lim0 * SOURCE_CLAMP_SLACK;

    const double tr = S.tr[v];
    f.rm = S.rmask[v];
    f.e = S.excess[v];
    f.dk = 0.0;
    f.r = 0.0;
    if (tr > 0) {
        f.r = __dsub_rn(tr, source_excess(tr, f.co));
    } else if (tr < 0) {
        const double sf = (f.rm & RM_SINKV) ? S.sink[v] : 0.0;
        f.r = __dadd_rn(tr, sf);
        f.dk = sf;
    }
    return f;
}

__device__ __forceinline__ void residual_write(const State<double>& S, unsigned v, const Residual& f)
{
    const double r = f.r;
    double e = f.e;
    unsigned nm = f.rm & 0x3fu;
    double trn = 0.0;
    if (r < 0) {
        trn = r;
        const double scap = -r;
        double sf;
        if (e >= scap) { sf = scap; e = __dsub_rn(e, scap); }
        else { sf = e; e = 0.0; }
        if (scap - sf > 0) nm |= RM_SINK;
        S.sink[v] = sf;
        nm |= RM_SINKV;
    } else if (r > 0) {
        double out = __dadd_ru(0.0, S.cap[0][v]);
        out = __dadd_ru(out, S.cap[1][v]); out = __dadd_ru(out, S.cap[2][v]); out = __dadd_ru(out, S.cap[3][v]);
        out = __dadd_ru(out, S.cap[4][v]); out = __dadd_ru(out, S.cap[5][v]);
        const double lim = out * SOURCE_CLAMP_SLACK;
        if (!(lim > f.lim0)) {
            // the usual case (no net inflow through the n-links): push source_excess(r', c_orig) >= min(r', lim) and
            // keep tr = r', which reads back as r' - source_excess(r', c_orig) bit for bit
            e = __dadd_rn(e, source_excess(r, f.co));
            trn = r;
        } else {
            const double p = r < lim ? r : lim;
            e = __dadd_rn(e, p);
            const double u = __dsub_rn(r, p);
            if (u > 0) trn = __dadd_rn(u, f.lim0);    // reads back as (u + lim0) - lim0: u to one rounding
        }
    }
    S.tr[v] = trn;
    S.excess[v] = e;
    S.rmask[v] = (uint8_t)nm;
}

// ---- general t-link folds (mgc_add_tweights_warm): add_tweights(v, src[k], snk[k]) with any finite values ----------------
// list form: key = voxel id, value = call index.  A stable radix sort of the pairs keeps a voxel's calls in call order.  An
// id out of range or a non-finite weight sets a bit of *err (an out-of-range id gets key 0).
__global__ void __launch_bounds__(256) k_tweights_keys(const int64_t* __restrict__ ids, const double* __restrict__ src,
                                                       const double* __restrict__ snk, int n, int64_t n_vox,
                                                       unsigned* __restrict__ keys, int* __restrict__ vals, int* __restrict__ err)
{
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        const int64_t v = ids[i];
        unsigned k = 0u;
        if (v < 0 || v >= n_vox) atomicOr(err, FOLD_ERR_RANGE);
        else k = (unsigned)v;
        if (!isfinite(src[i]) || !isfinite(snk[i])) atomicOr(err, FOLD_ERR_NONFINITE);
        keys[i] = k;
        vals[i] = i;
    }
}

// add_tweights(v, 0, 0) is an exact no-op in BK's arithmetic (the minimum is 0 and s - t gives tr back in both branches), so
// only voxels with a call of a nonzero weight become items, in both forms.
// list form: 1 at the first sorted key of each voxel that has such a call (order = the sorted call indices).  The n-link
// list form (gc_nlinks.cuh) groups its arcs the same way: a, b = cap, rev_cap there.  SLAB: only a key the slab owns
// heads an item (SlabOwn::key: an owned voxel, or a pair with an owned end).
template <typename K, bool SLAB = false>
__global__ void __launch_bounds__(256) k_weighted_heads(const K* __restrict__ keys, const int* __restrict__ order,
                                                        const double* __restrict__ a, const double* __restrict__ b, int n,
                                                        int* __restrict__ head, SlabOwn own = {})
{
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        int h = 0;
        bool first = i == 0 || keys[i] != keys[i - 1];
        if constexpr (SLAB) first = first && own.key(keys[i]);
        if (first) {
            const int e = lower_bound(keys, i, n, (K)(keys[i] + 1u));
            for (int j = i; j < e && !h; ++j) h = (a[order[j]] != 0.0 || b[order[j]] != 0.0) ? 1 : 0;
        }
        head[i] = h;
    }
}

// dense form: 1 where the call has a nonzero weight (SLAB: and the voxel is owned; every entry is checked)
template <bool SLAB = false>
__global__ void __launch_bounds__(256) k_tweights_dense_heads(const double* __restrict__ src, const double* __restrict__ snk,
                                                              int n, int* __restrict__ head, int* __restrict__ err,
                                                              SlabOwn own = {})
{
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        const double s = src[i], t = snk[i];
        if (!isfinite(s) || !isfinite(t)) atomicOr(err, FOLD_ERR_NONFINITE);
        int h = (s != 0.0 || t != 0.0) ? 1 : 0;
        if constexpr (SLAB) h = h && own.voxel((unsigned)i);
        head[i] = h;
    }
}

// pos = inclusive sum of the heads: the head at i is item pos[i] - 1, in ascending voxel order, and ctl[0] = pos[n - 1]
// items; the voxel of sorted key i is keys[i] >> shift (shift 1: the seed keys v << 1 | bg, whose fg keys precede the bg
// keys of a voxel).  keys == nullptr: the dense form (voxel i, one call).  Each touched tile is listed once, by the first
// item that flips tflag[t] (zeroed by the caller), and ctl[2] counts them: the claim list holds at most TL.ntiles entries
// whatever the number of calls.  That bound matters -- k_caps_claim enumerates count * 7 candidates in 32-bit arithmetic,
// and 7 * ntiles < 2^31 for every lattice below 2^31 voxels (ntiles = prod ceil(dim/8) <= n/8 + n^(2/3), taking the
// longest axis, c >= n^(1/3), at ceil(c/8)/c <= 1/8 + 1/c and the others at <= 1; so ntiles < 2^28 + 2^21), while one
// entry per item could pass 2^31 / 7 on a large erase.  The list order follows the atomics; k_caps_claim appends in atomic
// order anyway and each tile's materialisation does not depend on it.  tflag == nullptr lists no tiles (eager and 4-D
// handles: every voxel already holds its push state, and TL does not describe a 4-D lattice).
__global__ void __launch_bounds__(256) k_tweights_items(Lattice L, Tiles TL, const unsigned* __restrict__ keys, int shift,
                                                        const int* __restrict__ pos, int n, TweightItem* __restrict__ items,
                                                        int* __restrict__ tflag, int* __restrict__ tiles, int* __restrict__ ctl)
{
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += (int)(gridDim.x * blockDim.x)) {
        if (i == n - 1) ctl[0] = pos[i];
        if (pos[i] == (i > 0 ? pos[i - 1] : 0)) continue;
        unsigned v = (unsigned)i;
        int cnt = 1;
        if (keys) {
            v = keys[i] >> shift;
            cnt = lower_bound(keys, i, n, (v + 1u) << shift) - i;
        }
        items[pos[i] - 1] = TweightItem{v, i, cnt, 0};
        if (tflag) claim_tile_once(L, TL, v, tflag, tiles, ctl);
    }
}

// push lists after a fold: every materialised tile (cmat[t] = 1) holding an owned voxel with excess goes on the list its
// colour consumes next.  Excess stranded at voxels the last solve labelled HINF may reach a new sink link now; only
// materialised tiles can hold excess (mgc_add_seeds first materialises every tile whose source excess is still implicit).
// cmat == nullptr: an eager handle, every tile holds explicit state.
__global__ void __launch_bounds__(TILE_VOX) k_seed_lists(Lattice L, Tiles TL, State<double> S, const int* __restrict__ cmat,
                                                         int* __restrict__ pflag, WorkList pl0, WorkList pl1)
{
    for (int t = blockIdx.x; t < TL.ntiles; t += gridDim.x) {
        if (cmat && cmat[t] == 0) continue;    // block-uniform
        const TileCtx c = tile_ctx(L, TL, t);
        const int act = (c.own && S.excess[c.v] > 0) ? 1 : 0;
        if (__syncthreads_or(act) && threadIdx.x == 0) list_push(pflag, tile_color(c) ? pl1 : pl0, t);
    }
}

// ---- eager and 4-D handles (MGC_OPT_WARM) -------------------------------------------------------------------------------
// A handle that was not built lazily keeps no copy of its inputs, and cap[] holds residuals after the first push, so the
// source flow its state holds cannot be recomputed as residual_read does.  With MGC_OPT_WARM the first solve records it
// instead, before any push: tr > 0 becomes tr - e0, e0 = the source excess of the init (k_init_tile<T, true> /
// k_init_tile4<T, true> on the per-term path, k_warm_convert after the eager fused build).  tr then holds BK's own residual
// source capacity; once the excess is set nothing but these folds reads tr > 0 (DESIGN.md §4.6).
//   read : r = tr                  for tr > 0;
//          r = tr + absorbed       for tr < 0 (absorbed = sink[v] under RM_SINKV in 3-D; k_init_tile4 zeroes sink[], so
//                                  a 4-D voxel always holds it), moved into the add_tweights constant as in residual_read;
//          r = 0                   for tr = 0.
//   write: r' < 0 : as residual_write (a fresh sink link that takes the voxel's own excess at once);
//          r' > 0 : p = min(r', residual out-capacity rounded up x SOURCE_CLAMP_SLACK) joins the excess (r' itself when that
//                   sum is NaN, as in source_excess) and tr = r' - p, which the next fold reads back as the residual;
//          r' = 0 : tr = 0.
// 3-D state: 6 arcs, the sink-link bits RM_SINK / RM_SINKV in rmask.  4-D state: 8 arcs in rmask, the sink-residual bit in
// smask, and sink[] summed over every voxel by the read-out (so a voxel without a sink link gets sink[v] = 0).
struct EagerRead {
    double r;         // r(v)
    double dk;        // change of the add_tweights constant
    double e;         // excess
    unsigned rm;      // rmask
};

template <int ND>
__device__ __forceinline__ EagerRead eager_read(const State<double>& S, unsigned v)
{
    EagerRead f;
    const double tr = S.tr[v];
    f.rm = S.rmask[v];
    f.e = S.excess[v];
    f.dk = 0.0;
    f.r = 0.0;
    if (tr > 0) {
        f.r = tr;
    } else if (tr < 0) {
        const double sf = (ND == 4 || (f.rm & RM_SINKV)) ? S.sink[v] : 0.0;
        f.r = __dadd_rn(tr, sf);
        f.dk = sf;
    }
    return f;
}

template <int ND>
__device__ __forceinline__ void eager_write(const State<double>& S, uint8_t* __restrict__ smask, unsigned v,
                                            const EagerRead& f)
{
    const double r = f.r;
    double e = f.e;
    double trn = 0.0, sf = 0.0;
    bool sres = false;
    if (r < 0) {
        trn = r;
        const double scap = -r;
        if (e >= scap) { sf = scap; e = __dsub_rn(e, scap); }
        else { sf = e; e = 0.0; }
        sres = scap - sf > 0;
    } else if (r > 0) {
        double out = 0.0;
#pragma unroll
        for (int k = 0; k < 2 * ND; ++k) out = __dadd_ru(out, S.cap[k][v]);
        const double lim = out * SOURCE_CLAMP_SLACK;
        double p = r < lim ? r : lim;
        if (!(out == out)) p = r;
        e = __dadd_rn(e, p);
        trn = __dsub_rn(r, p);
    }
    S.tr[v] = trn;
    S.excess[v] = e;
    if (ND == 3) {
        unsigned nm = f.rm & 0x3fu;
        if (r < 0) {
            S.sink[v] = sf;
            nm |= RM_SINKV | (sres ? RM_SINK : 0u);
        }
        S.rmask[v] = (uint8_t)nm;
    } else {
        S.sink[v] = sf;
        smask[v] = sres ? 1 : 0;
    }
}

// ---- the fold ----------------------------------------------------------------------------------------------------------
// Residual access of a fold: read(v) gives r(v) and the voxel's state, write(v, f) stores r' back.  How tr holds the
// residual source capacity is the access type's business: a lazily built handle recomputes the pushed source flow from
// its image (residual_read), an eager or 4-D handle recorded r(v) itself at the first solve (eager_read).  The members
// are the fold kernels' first parameters.
// BATCH: a batch handle, whose fold kernels also store each entry's change of the add_tweights constant for the
// per-image sum (batch_fold_const); false compiles the single-handle kernels without it.
template <typename E, int FN, int USE_MAX, int SPACING, bool BATCH_>
struct LazyResidual {
    static constexpr int ND = 3;
    static constexpr bool BATCH = BATCH_;
    Lattice L;
    State<double> S;
    const E* img;
    BoundaryParams P;
    __device__ __forceinline__ Residual read(unsigned v) const { return residual_read<E, FN, USE_MAX, SPACING, BATCH>(L, S, img, P, v); }
    __device__ __forceinline__ void write(unsigned v, const Residual& f) const { residual_write(S, v, f); }
};

template <int ND_, bool BATCH_ = false>
struct EagerResidual {
    static constexpr int ND = ND_;
    static constexpr bool BATCH = BATCH_;
    State<double> S;
    uint8_t* smask;
    __device__ __forceinline__ EagerRead read(unsigned v) const { return eager_read<ND>(S, v); }
    __device__ __forceinline__ void write(unsigned v, const EagerRead& f) const { eager_write<ND>(S, smask, v, f); }
};

// The calls of a fold: get(j, s, t) gives add_tweights call j of the sorted grouping.  Read-only inputs are loaded through
// __ldg: a pointer inside a parameter struct carries no __restrict__.
// Seeds: sorted key j = v << 1 | bg is add_tweights(v, cap, 0) (fg) or add_tweights(v, 0, cap) (bg), cap = +-65535.
struct SeedCalls {
    const unsigned* keys;
    double cap;
    __device__ __forceinline__ void get(int j, double& s, double& t) const
    {
        const bool bg = (__ldg(keys + j) & 1u) != 0;
        s = bg ? 0.0 : cap;
        t = bg ? cap : 0.0;
    }
};

// mgc_add_tweights_warm: add_tweights(v, src[k], snk[k]), k = order[j] (the sorted call indices; nullptr: k = j)
struct ListCalls {
    const int* order;
    const double* src;
    const double* snk;
    __device__ __forceinline__ void get(int j, double& s, double& t) const
    {
        const int k = order ? __ldg(order + j) : j;
        s = __ldg(src + k);
        t = __ldg(snk + k);
    }
};

// One thread per touched voxel: r(v) read, its calls applied in order with the reference's arithmetic, r' written back;
// the change of the add_tweights constant summed into one partial per block, and on a batch handle (Access::BATCH),
// whose images keep their own constants, stored per item in item_dk.  residual_write and eager_write hold for any finite r and r',
// so any weights may come.
template <typename Access, typename Calls>
__global__ void __launch_bounds__(256)
k_tlink_fold(Access A, const TweightItem* __restrict__ items, int n, Calls C, double* __restrict__ partials,
             double* __restrict__ item_dk)
{
    double m = 0.0;
    const int step = (int)(gridDim.x * blockDim.x);
    for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x); i < n; i += step) {
        const TweightItem it = items[i];
        auto f = A.read(it.v);
        for (int j = it.first; j < it.first + it.count; ++j) {
            double s, t;
            C.get(j, s, t);
            f.dk = __dadd_rn(f.dk, add_tweights_dev(f.r, s, t));
        }
        A.write(it.v, f);
        m = __dadd_rn(m, f.dk);
        if constexpr (Access::BATCH) item_dk[i] = f.dk;
    }
    block_sum_store(m, partials);
}

// the eager fused build (k_build_tile<..., LAZY = 0>) wrote tr and the excess before MGC_OPT_WARM could be set: the same
// record as k_init_tile<T, true>, as a pass of its own at the first solve, before any push.  The capacity planes still hold
// the build's weights, so source_excess gives the build's e0 bit for bit.
__global__ void __launch_bounds__(256) k_warm_convert(Lattice L, State<double> S)
{
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += gridDim.x * blockDim.x) {
        const double tr = S.tr[v];
        if (tr > 0) {
            const double c[6] = {S.cap[0][v], S.cap[1][v], S.cap[2][v], S.cap[3][v], S.cap[4][v], S.cap[5][v]};
            S.tr[v] = __dsub_rn(tr, source_excess(tr, c));
        }
    }
}

// push lists after a fold on a 4-D handle (cf. k_seed_lists): every tile holding an owned voxel with excess goes on the
// list its colour (4-D checkerboard parity) consumes next
__global__ void __launch_bounds__(T4_VOX) k_seed_lists4(Lattice L, Tiles4 TL, State<double> S, int* __restrict__ pflag,
                                                        WorkList pl0, WorkList pl1)
{
    for (int t = blockIdx.x; t < TL.ntiles; t += gridDim.x) {
        const Tile4Ctx c = tile4_ctx(L, TL, t);
        const int act = (c.own && S.excess[c.v] > 0) ? 1 : 0;
        if (__syncthreads_or(act) && threadIdx.x == 0) list_push(pflag, tile4_color(c) ? pl1 : pl0, t);
    }
}
