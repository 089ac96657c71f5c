// gc_build.cuh -- the whole graph build as ONE pass over the lattice (3-D): n-link stencil + regional t-links + hard
// markers + solver-state initialisation, fused.
//
// Replaces, in one kernel, what the reference does in  energy_voxel.py:611-664 (__skeleton_base, one Python call
// per edge), graph.py:532-552 / :310-380 (set_tweights_all, set_source_nodes, set_sink_nodes -> Graph::add_tweights,
// graph.h:415-425) in the order graph_from_voxels applies them (generate.py:159-172: regional term, boundary term,
// foreground markers, background markers), plus what k_boundary / k_regional / k_markers / k_init_tile did in four
// passes here (with capacity planes written by one kernel and read straight back by the next).  Now every input byte is read once and every state byte written once:
//     read  image 4 + probability 4 + fg 1 + bg 1                         = 10 B/voxel (float32 inputs)
//     write six float64 capacities 48 + tr 8 + excess 8 + label 4 + rmask 1 = 69 B/voxel
// (the lazy variant, LAZY = 1 below, writes two marker bit planes instead of the capacities, tr and excess: 5.25 B/voxel,
// plus 8 B/voxel of image and probability copies for float32 inputs when the graph cannot read the inputs later)
// (`sink[]`, the absorbed-flow accumulator, is no longer zero-filled: bit RM_SINKV of rmask says whether a voxel's
// entry has been written, see gc_tiles.cuh.)
//
// Geometry: a 256-thread CTA builds an 8 (z) x 8 (y) x 32 (x) block = four 8^3 solver tiles in a row.  The image
// block with a one-voxel halo on every side (10 x 10 x 34, box 10 x 10 x BuildBox<E>::BX) is staged in shared memory by ONE
// `cp.async.bulk.tensor.3d` box copy against a per-call tensor map (SASS: UTMALDG + SYNCS; out-of-lattice parts are
// zero-filled by the TMA unit and masked by coordinates), or by plain loads when the image does not meet the 16-byte
// stride rule of tensor maps.  Thread (y, x) marches through z = -1 .. 7: per step it evaluates the three FORWARD
// pair weights of its voxel (+z, +y, +x) exactly once -- w(p, q) = g(|I_p - I_q|) or g(max(|I_p|, |I_q|)), float64,
// the arithmetic of gc_terms.cuh -- keeps the +z weight in a register for the next step (where it is the voxel's -z
// capacity), and publishes the +y / +x weights in a shared-memory plane from which the neighbours in y and x take
// their backward capacities.  The only weights evaluated twice are those on the block's low faces (12.5 %).
#pragma once
#include <climits>
#include <type_traits>
#include "gc_terms.cuh"
#include "gc_tiles.cuh"
#include "gc_tma.cuh"

#define BUILD_TZ 8
#define BUILD_TY 8
#define BUILD_TX 32
#define BUILD_THREADS 256
// Inner (x) extent of the staged image block.  Box starts are kept non-negative and 16-byte aligned along the innermost
// axis, so the copies never depend on how the TMA unit treats negative or unaligned innermost coordinates: the box starts
// BUILD_PAD = 16 / sizeof(E) elements in front of the block (x0 is a multiple of 32) instead of 1, or at 0 for the blocks
// on the low x face; the extent covers pad + 32 + 1 elements, rounded up to a multiple of 16 bytes.
// shared-memory offset of the staged t-link inputs: behind image block, weight planes, barrier, flags, reduction scratch
#define BUILD_TIN_OFFSET(img_pad) ((((img_pad) + (2 * 9 * 32 + 2 * 8 * 33 + 8 * 32 + 8 * 8) * 8 + 8 + 32 + 64) + 127) / 128 * 128)
template <typename E> struct BuildBox {
    static constexpr int PAD = 16 / (int)sizeof(E);
    static constexpr int BX = (PAD + 33 + PAD - 1) / PAD * PAD;      // f32 40, f64 36, u8 64, i16 48, i32 40
};
#define BUILD_HY 10
#define BUILD_HZ 10

// tensor maps of one build: image (halo box), probability map and the two marker volumes (8 x 8 x 32 blocks)
struct BuildMaps {
    CUtensorMap img, prob, fg, bg;
};

struct BuildArgs {
    const void* img;           // C-contiguous image over the local lattice (device)
    const void* prob;          // regional_probability_map input or nullptr
    int prob_f64;              // 1: prob is float64
    int compute_f32;           // products in float32 (numpy: float32 map * Python float)
    double alpha;
    const uint8_t* fg;         // marker volumes (bytes) or nullptr
    const uint8_t* bg;
    const unsigned* fg_bits;   // ... or bit-packed (bit v & 31 of word v >> 5), used when fg/bg are nullptr
    const unsigned* bg_bits;
    int use_tma;               // image block staged by TMA (else plain loads)
    int tma_prob;              // probability block (8 x 8 x 32) staged by TMA into shared memory
    int tma_mark;              // fg / bg byte blocks staged by TMA (bit 0: fg, bit 1: bg)
    int z_tile0;               // first z tile layer of this launch (chunked builds)
    int dbg;                   // diagnostics (MEDPY_GC_BUILD_DBG): 1 = do not load the probability map (constant 0.3)
    void* img_copy;            // lazy build: graph-owned copy of the image, or nullptr when the graph reads the input itself later
    void* prob_copy;           // lazy build: graph-owned copy of the probability map, in its own dtype, or nullptr (as img_copy)
    unsigned* fg_plane;        // lazy build: marker bit planes (nullptr: no such marker), see MarkerPlanes
    unsigned* bg_plane;
    int* cmat;                 // lazy build: per tile "push state materialised" flag, cleared here
};

// What k_caps_tiles needs to replay the t-links of a lazy build.  The marker planes are row-padded: bit x & 31 of word
// (z * Y + y) * words + x / 32, so that one warp row of the build (x0 .. x0 + 31 of row (z, y)) is one aligned word.
struct LazyTin {
    const void* prob;          // probability map copy or nullptr
    int prob_f64;
    int compute_f32;
    double alpha;
    const unsigned* fg;        // marker planes or nullptr
    const unsigned* bg;
    int words;                 // words per row: ceil(X / 32)
};

template <typename E>
__device__ __forceinline__ double build_val(E x, bool use_max)
{
    return use_max ? Elem<E>::val(Elem<E>::absv(x)) : Elem<E>::val(x);
}

template <int FN, typename E>
__device__ __forceinline__ double build_pair(const BoundaryParams& P, double a, E iq, bool use_max)
{
    const double b = build_val<E>(iq, use_max);
    const double x = use_max ? fmax(a, b) : fabs(__dsub_rn(a, b));
    return g_weight<FN>(P, x);
}

// One pair weight as every build path forms it (eager build, lazy build, capacity materialiser): the term's weight of the
// pair, divided by the axis spacing when there is one.  |a - b| and max(|a|, |b|) are symmetric, so the weight computed
// from either end of the pair is the same double.
template <int FN, typename E>
__device__ __forceinline__ double build_weight(const BoundaryParams& P, double a, E iq, bool use_max, bool spacing, double sp)
{
    double w = build_pair<FN, E>(P, a, iq, use_max);
    if (spacing) w = __ddiv_rn(w, sp);
    return w;
}

// The six capacities (-z, +z, -y, +y, -x, +x) of one voxel under the exponential term without spacing, from their
// arguments t[k]; bit k of `valid`: the pair exists.  `ordinary` must be warp-uniform (every argument of the warp <= 700,
// none NaN): both branches then give the same doubles as g_weight<1>, and an in-lattice weight is never below DBL_MIN.
__device__ __forceinline__ void exp_caps6(const double t[6], bool ordinary, unsigned valid, double c[6])
{
    if (ordinary) {
#pragma unroll
        for (int k = 0; k < 6; ++k) c[k] = exp_neg_inrange(t[k]);
    } else {
#pragma unroll
        for (int k = 0; k < 6; ++k) { const double w = exp_neg(t[k]); c[k] = w <= 0.0 ? DBL_MIN : w; }
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) if (!((valid >> k) & 1u)) c[k] = 0.0;
}

// The t-links of the build, replayed in the reference's order (regional term with float32 or float64 products,
// foreground markers, background markers) onto tr; returns the sum of the add_tweights minima.  The build and the
// materialiser both form tr here, so the lazy tr is the eager one bit for bit.
template <typename T>
__device__ __forceinline__ double tlink_replay(T& tr, bool has_prob, double p, bool f32, double alpha, unsigned fb)
{
    double mm = 0.0;
    if (has_prob) {
        double s, t;
        if (f32) {
            const float pf = (float)p;          // exact: the map is float32 when its products are
            const float af = (float)alpha;
            s = (double)__fmul_rn(pf, af);
            t = (double)__fmul_rn(__fsub_rn(1.0f, pf), af);
        } else {
            s = __dmul_rn(p, alpha);
            t = __dmul_rn(__dsub_rn(1.0, p), alpha);
        }
        mm = add_tweights_dev(tr, s, t);
    }
    if (fb & 1u) mm = __dadd_rn(mm, add_tweights_dev(tr, 65535.0, 0.0));
    if (fb & 2u) mm = __dadd_rn(mm, add_tweights_dev(tr, 0.0, 65535.0));
    return mm;
}

// residual-mask bits 0..5 of a voxel: its arcs with capacity
__device__ __forceinline__ unsigned cap_bits(const double c[6])
{
    return (c[0] > 0 ? 1u : 0u) | (c[1] > 0 ? 2u : 0u) | (c[2] > 0 ? 4u : 0u) | (c[3] > 0 ? 8u : 0u) |
           (c[4] > 0 ? 16u : 0u) | (c[5] > 0 ? 32u : 0u);
}

// source excess of a voxel with net terminal capacity tr > 0: clamped to the sum of its out-capacities rounded up,
// with SOURCE_CLAMP_SLACK head-room (DESIGN.md §4.2); 0 when tr <= 0
__device__ __forceinline__ double source_excess(double tr, const double c[6])
{
    double out = __dadd_ru(0.0, c[0]);
    out = __dadd_ru(out, c[1]); out = __dadd_ru(out, c[2]); out = __dadd_ru(out, c[3]);
    out = __dadd_ru(out, c[4]); out = __dadd_ru(out, c[5]);
    double e = 0.0;
    if (tr > 0) { const double lim = out * SOURCE_CLAMP_SLACK; e = tr < lim ? tr : lim; if (!(out == out)) e = tr; }
    return e;
}

// source_excess(tr, c) > 0 without the capacities, for a voxel whose in-lattice pairs are `pairs` (bit k: the pair across
// face k exists).  Every such pair has a weight > 0 (then the rounded-up sum is > 0 and so is the clamp), +inf or NaN
// (then the excess is tr itself), unless the build's weight check failed; so the excess is > 0 exactly when tr > 0 and
// the voxel has a pair.  A failed check can only make this claim excess that is not there, which is safe for its users.
__device__ __forceinline__ bool source_active(double tr, unsigned pairs)
{
    return tr > 0 && pairs != 0u;
}

// TIN = 1: the common configuration fixed at compile time -- float32 probability map with float32 products and both
// marker volumes as bytes, all three staged by TMA.  The generic form (TIN = 0) decides each of those per voxel with
// warp-uniform branches, whose bookkeeping costs instructions in this issue-heavy loop.
//
// LAZY = 1: neither the capacity planes nor tr nor excess are written (k_caps_tiles computes all three for the tiles the
// push path reaches); the kernel writes what recomputes them bit for bit instead -- the markers as two bit planes (one
// ballot per warp row) and, where the graph has no other copy of them to read later (img_copy / prob_copy not nullptr),
// copies of the image and of the probability map -- and clears cmat[] of its tiles.  rmask,
// height, partials and worklists are bit for bit what LAZY = 0 writes.  Under the exponential term without spacing every
// in-lattice weight is >= DBL_MIN, so for a voxel whose arguments are ordinary the n-link bits of rmask are the validity
// bits, and the clamped excess is > 0 exactly when tr > 0 and the voxel has an in-lattice arc.  One range test over the
// staged image block (block_exp_ordinary, gc_exprange.cuh) decides that for every pair of the block at once: in a block
// that passes, no z-step reads a neighbour cell, forms an argument or takes a vote.  A block that does not pass takes
// the warp vote per z-step, and a warp whose arguments are not ordinary evaluates all six weights per voxel (rmask
// depends on them; no z carry, no shared planes: a neighbouring warp may have skipped).  Other terms still evaluate
// every weight (weight check, rmask) but store none.
//
// The body builds block (bx, by, bz) of a launch of nbx x nby x (layers) blocks; k_build_tile runs it for its own CTA,
// k_build_refused for the blocks the lean kernel (below) refused.  `first`: the CTA's first block (the mbarrier is
// initialised), `parity`: the mbarrier phase of this block's copies.
template <typename E, typename T, int FN, int USE_MAX, int SPACING, int TIN, int LAZY>
__device__ __forceinline__ void
build_block(int bx, int by, int bz, int nbx, int nby, bool first, unsigned parity, unsigned char* smem_raw,
            const Lattice& L, const Tiles& TL, const State<T>& S, const BuildMaps& maps, const BuildArgs& A,
            const BoundaryParams& P, int* __restrict__ bad, double* __restrict__ partials, int* __restrict__ rflag,
            const WorkList& rl, int* __restrict__ pflag, const WorkList& pl0, const WorkList& pl1)
{
    constexpr int BUILD_BX = BuildBox<E>::BX, BUILD_PAD = BuildBox<E>::PAD;
    E* s_img = reinterpret_cast<E*>(smem_raw);                                   // [10][10][BUILD_BX]
    constexpr int IMG_BYTES = BUILD_HZ * BUILD_HY * BUILD_BX * (int)sizeof(E);
    constexpr int IMG_PAD = (IMG_BYTES + 127) / 128 * 128;
    double* s_wy = reinterpret_cast<double*>(smem_raw + IMG_PAD);                // [2][9][32]: +y weight of row y-1 .. 7
    double* s_wx = s_wy + 2 * 9 * 32;                                            // [2][8][33]: +x weight of column x-1 .. 31
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(s_wx + 2 * 8 * 33 + 8 * 32 + 8 * 8);
    int* s_flags = reinterpret_cast<int*>(bar + 1);                              // [4] needs, [4] has excess
    double* s_red = reinterpret_cast<double*>(s_flags + 8);                      // [8] block reduction
    // TMA-staged t-link inputs (LDGs issued from inside the store-saturated loop queue behind the stores; the async-proxy
    // copies are free of the LSU queue)
    unsigned char* s_prob = smem_raw + BUILD_TIN_OFFSET(IMG_PAD);                // [8][8][32] float or double, 128-B aligned
    unsigned char* s_fg = s_prob + BUILD_TZ * BUILD_TY * BUILD_TX * 8;           // [8][8][32] bytes
    unsigned char* s_bg = s_fg + BUILD_TZ * BUILD_TY * BUILD_TX;

    const int tid = threadIdx.x;
    const int lx = tid & 31, ly = tid >> 5;
    const int x0 = bx * BUILD_TX, y0 = by * BUILD_TY, z0 = (A.z_tile0 + bz) * BUILD_TZ;
    const bool use_max = USE_MAX >= 0 ? (USE_MAX != 0) : (P.use_max != 0);
    const bool spacing = SPACING >= 0 ? (SPACING != 0) : (P.inv_spacing_on != 0.0);
    constexpr bool LAZY_EXP = LAZY && FN == 1 && SPACING == 0;      // the lazy path that may skip the weights

    const int gy = y0 + ly, gx = x0 + lx;
    const bool col_in = gy < L.dim[1] && gx < L.dim[2];
    // t-link inputs of one voxel (probability, marker flags), fetched ONE z-step ahead of their use: otherwise the loop
    // stalled on these global loads (long scoreboard 7 of 15 cycles per issue) when they were read where they are needed
    struct TIn { double p; unsigned fb; };
    auto fetch = [&](int lz) -> TIn {
        TIn r{0.0, 0u};
        if (TIN == 1) {               // staged float32 probability (kept as the exact double image of the float) + staged marker bytes
            const int si = (lz * BUILD_TY + ly) * BUILD_TX + lx;
            r.p = (double)reinterpret_cast<const float*>(s_prob)[si];
            r.fb = (s_fg[si] ? 1u : 0u) | (s_bg[si] ? 2u : 0u);
            return r;
        }
        const int gz = z0 + lz;
        if (!(col_in && gz < L.dim[0])) return r;
        const unsigned v = (unsigned)gz * L.stride[0] + (unsigned)gy * L.stride[1] + (unsigned)gx;
        const int si = (lz * BUILD_TY + ly) * BUILD_TX + lx;          // index inside the staged 8 x 8 x 32 blocks
        if (A.prob) {
            if (A.tma_prob) r.p = A.prob_f64 ? reinterpret_cast<const double*>(s_prob)[si] : (double)reinterpret_cast<const float*>(s_prob)[si];
            else r.p = (A.dbg & 1) ? 0.3 : (A.prob_f64 ? reinterpret_cast<const double*>(A.prob)[v] : (double)reinterpret_cast<const float*>(A.prob)[v]);
        }
        if (A.fg_bits || A.bg_bits) {
            if (A.fg_bits) r.fb |= (A.fg_bits[v >> 5] >> (v & 31u)) & 1u;
            if (A.bg_bits) r.fb |= ((A.bg_bits[v >> 5] >> (v & 31u)) & 1u) << 1;
        } else {
            if (A.fg && ((A.tma_mark & 1) ? s_fg[si] : A.fg[v])) r.fb |= 1u;
            if (A.bg && ((A.tma_mark & 2) ? s_bg[si] : A.bg[v])) r.fb |= 2u;
        }
        return r;
    };
    const bool staged_tin = TIN == 1 || (A.use_tma && ((A.prob && A.tma_prob) || A.tma_mark));
    TIn cur{0.0, 0u};
    if (!staged_tin) cur = fetch(0);          // global loads: in flight while the image block is staged

    // ---- stage the image block with halo: local (hz, hy, hx) <-> global (z0 - 1 + hz, y0 - 1 + hy, x0 - 1 + hx) ----
    // TMA: the box starts at a non-negative, 16-byte aligned x (see BuildBox) and at non-negative y / z: blocks on a low
    // face start at 0 and the shared-memory index is shifted instead -- the halo cells in front of the lattice are never
    // read.  Parts of the box beyond the high faces are zero-filled by the TMA unit.  cx / cy / cz: shared-memory index of
    // the logical halo cell 0 (global x0 - 1, y0 - 1, z0 - 1) along each axis.
    const int cx = A.use_tma ? (x0 == 0 ? -1 : BUILD_PAD - 1) : 0;
    const int cy = (A.use_tma && y0 == 0) ? -1 : 0, cz = (A.use_tma && z0 == 0) ? -1 : 0;
    if (tid < 8) s_flags[tid] = 0;
    if (A.use_tma) {
        if (tid == 0) {
            if (first) {
                mbar_init(bar, 1);
                asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            } else {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the previous block's reads are done
            }
            const unsigned pbytes = (A.prob && A.tma_prob) ? (unsigned)(BUILD_TZ * BUILD_TY * BUILD_TX * (A.prob_f64 ? 8 : 4)) : 0u;
            const unsigned mbytes = (unsigned)(BUILD_TZ * BUILD_TY * BUILD_TX);
            mbar_expect_tx(bar, (unsigned)IMG_BYTES + pbytes + ((A.tma_mark & 1) ? mbytes : 0u) + ((A.tma_mark & 2) ? mbytes : 0u));
            tma_load_3d(s_img, &maps.img, bar, x0 - 1 - cx, y0 - 1 - cy, z0 - 1 - cz);
            if (pbytes) tma_load_3d(s_prob, &maps.prob, bar, x0, y0, z0);
            if (A.tma_mark & 1) tma_load_3d(s_fg, &maps.fg, bar, x0, y0, z0);
            if (A.tma_mark & 2) tma_load_3d(s_bg, &maps.bg, bar, x0, y0, z0);
        }
        __syncthreads();
        mbar_wait(bar, parity);
        if (staged_tin) cur = fetch(0);
    } else {
        // (LAZY_EXP stages whole rows of the box, as TMA does: the block's range test reads every cell)
        constexpr int SX = LAZY_EXP ? BUILD_BX : 34;
        const E* img = reinterpret_cast<const E*>(A.img);
        for (int i = tid; i < BUILD_HZ * BUILD_HY * SX; i += BUILD_THREADS) {
            const int hx = i % SX, r = i / SX, hy = r % BUILD_HY, hz = r / BUILD_HY;
            const int gz = z0 - 1 + hz, gy = y0 - 1 + hy, gx = x0 - 1 + hx;
            E val = (E)0;
            if (gz >= 0 && gy >= 0 && gx >= 0 && gz < L.dim[0] && gy < L.dim[1] && gx < L.dim[2])
                val = img[(unsigned)gz * L.stride[0] + (unsigned)gy * L.stride[1] + (unsigned)gx];
            s_img[(hz * BUILD_HY + hy) * BUILD_BX + hx] = val;
        }
        __syncthreads();
    }

    // ---- LAZY_EXP: one range test for the whole staged block instead of a warp vote per voxel and z-step.  Every cell
    // of the box counts -- halo, pad and zero fill included, which can only make the test stricter -- and
    // block_exp_ordinary (gc_exprange.cuh) states why a block that passes holds no pair whose own test would fail.  The
    // result is uniform over the CTA.  Scratch: the weight planes, which LAZY_EXP does not use.
    bool blk_ordinary = false;
    if constexpr (LAZY_EXP) {
        E lo = (E)INFINITY, hi = (E)-INFINITY;
        bool nan = false;
        for (int i = tid; i < IMG_BYTES / 16; i += BUILD_THREADS) {
            const uint4 q = reinterpret_cast<const uint4*>(s_img)[i];
            E e[16 / sizeof(E)];
            memcpy(e, &q, 16);
#pragma unroll
            for (int k = 0; k < (int)(16 / sizeof(E)); ++k) block_range_add<E>(lo, hi, nan, e[k]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const E olo = __shfl_xor_sync(0xffffffffu, lo, o), ohi = __shfl_xor_sync(0xffffffffu, hi, o);
            block_range_add<E>(lo, hi, nan, olo);
            block_range_add<E>(lo, hi, nan, ohi);
        }
        nan = __any_sync(0xffffffffu, nan);
        E* s_rng = reinterpret_cast<E*>(s_wy);                       // [8] warp minima, [8] warp maxima
        int* s_rnan = reinterpret_cast<int*>(s_wy + 16);             // [8] warp NaN flags
        if (lx == 0) { s_rng[ly] = lo; s_rng[8 + ly] = hi; s_rnan[ly] = nan ? 1 : 0; }
        __syncthreads();
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            block_range_add<E>(lo, hi, nan, s_rng[w]);
            block_range_add<E>(lo, hi, nan, s_rng[8 + w]);
            nan = nan || s_rnan[w] != 0;
        }
        blk_ordinary = block_exp_ordinary(Elem<E>::val(lo), Elem<E>::val(hi), nan, use_max,
                                          range_inv_sigma2(P, L, z0 - 1, z0 + BUILD_TZ));
    }

    const bool has_py = gy + 1 < L.dim[1], has_px = gx + 1 < L.dim[2];
    const double sp_z = spacing ? P.spacing[0] : 1.0, sp_y = spacing ? P.spacing[1] : 1.0, sp_x = spacing ? P.spacing[2] : 1.0;
    // (cells in front of the lattice do not exist when the box was clamped: their index is clamped too, the value is
    // never used -- every pair that would need it is invalid)
    auto at = [&](int hz, int hy, int hx) -> E {
        const int i = ((hz + cz) * BUILD_HY + (hy + cy)) * BUILD_BX + (hx + cx);
        return s_img[i < 0 ? 0 : i];
    };

    int isbad = 0;
    unsigned needs_any = 0, exc_any = 0;
    double msum = 0.0;
    // one pair weight: the term's constants of the pair's plane, value of the neighbour cell, validity, axis spacing
    auto pair_w = [&](const BoundaryParams& Q, double a, E iq, bool valid, double sp) -> double {
        const double w = build_weight<FN, E>(Q, a, iq, use_max, spacing, sp);
        // the exponential term without spacing is clamped to DBL_MIN and can never be <= 0 (NaN compares false)
        if (!(FN == 1 && SPACING == 0)) { if (valid && w <= 0.0) isbad = 1; }
        return valid ? w : 0.0;
    };
    // ---- prologue: the weights on the block's three LOW faces, spread over all threads (one z-face and one y-face
    // weight per thread, the 64 x-face weights on the first two warps) so that no warp carries extra work in the loop ----
    double* s_wyh = s_wx + 2 * 8 * 33;          // [8 z][32 x]: pair (y0 - 1, y0)
    double* s_wxh = s_wyh + 8 * 32;             // [8 z][8 y]:  pair (x0 - 1, x0)
    double wz_back = 0.0;
    if (!LAZY_EXP) {
        const bool vz = col_in && (z_pairs(L, z0) & 1u);
        wz_back = pair_w(params_at(P, L, z0), build_val<E>(at(0, ly + 1, lx + 1), use_max), at(1, ly + 1, lx + 1), vz, sp_z);
        // thread (ly, lx) -> y-face weight of plane z0 + ly at column x0 + lx
        const bool vy = y0 > 0 && gx < L.dim[2] && z0 + ly < L.dim[0];
        s_wyh[ly * 32 + lx] = pair_w(params_at(P, L, z0 + ly), build_val<E>(at(ly + 1, 0, lx + 1), use_max), at(ly + 1, 1, lx + 1), vy, sp_y);
        if (tid < 64) {
            const int fz = tid >> 3, fy = tid & 7;
            const bool vx = x0 > 0 && y0 + fy < L.dim[1] && z0 + fz < L.dim[0];
            s_wxh[fz * 8 + fy] = pair_w(params_at(P, L, z0 + fz), build_val<E>(at(fz + 1, fy + 1, 0), use_max), at(fz + 1, fy + 1, 1), vx, sp_x);
        }
    }

    // the in-lattice pairs of this thread's voxel in plane gz (bit k: the pair across face k exists)
    auto pairs_at = [&](int gz) -> unsigned {
        return z_pairs(L, gz) | (gy > 0 ? 4u : 0u) | (has_py ? 8u : 0u) | (gx > 0 ? 16u : 0u) | (has_px ? 32u : 0u);
    };
    const bool copies = A.img_copy != nullptr || A.prob_copy != nullptr;
    for (int lz = 0; lz < BUILD_TZ; ++lz) {
        const int gz = z0 + lz;
        const bool pin = col_in && gz < L.dim[0];            // block-uniform in z, per thread in y/x
        double* wyb = s_wy + (lz & 1) * 9 * 32;
        double* wxb = s_wx + (lz & 1) * 8 * 33;
        const int hz = lz + 1;
        const BoundaryParams Pz = params_at(P, L, gz);       // this plane's term constants (a batch: its image's)
        TIn nxt{0.0, 0u};
        if (lz + 1 < BUILD_TZ) nxt = fetch(lz + 1);
        // (the voxel's own value: read where a weight or an argument needs it)
        auto own_val = [&]() -> double { return build_val<E>(at(hz, ly + 1, lx + 1), use_max); };
        // ---- t-links: add_tweights replay in the reference's order (regional, fg, bg) ----
        auto tlinks = [&](T& tr) -> double {
            return tlink_replay<T>(tr, TIN == 1 || A.prob != nullptr, cur.p, TIN == 1 || A.compute_f32 != 0, A.alpha, cur.fb);
        };
        T tr = (T)0;
        double mm = 0.0;
        double c0 = 0.0, c1 = 0.0, c2 = 0.0, c3 = 0.0, c4 = 0.0, c5 = 0.0;
        double wz = 0.0, wy = 0.0, wx = 0.0;
        // LAZY_EXP: every argument of the warp is ordinary -- rmask then holds the validity bits and the excess follows
        // from tr (source_active) -- or else c0..c5 are the six weights
        bool lean = false;
        if constexpr (LAZY_EXP) {
            // the six weights are needed only when some argument of the warp is not ordinary (rmask would then depend on
            // the values): never in a block that passed its range test, else when the warp's vote fails
            if (pin) mm = tlinks(tr);
            lean = blk_ordinary;
            if (!lean) {
                const double a = own_val();
                auto arg = [&](E iq) -> double {
                    const double b = build_val<E>(iq, use_max);
                    return exp_term_arg(Pz, use_max ? fmax(a, b) : fabs(__dsub_rn(a, b)));
                };
                const double t[6] = {arg(at(hz - 1, ly + 1, lx + 1)), arg(at(hz + 1, ly + 1, lx + 1)), arg(at(hz, ly, lx + 1)),
                                     arg(at(hz, ly + 2, lx + 1)), arg(at(hz, ly + 1, lx)), arg(at(hz, ly + 1, lx + 2))};
                lean = __all_sync(0xffffffffu, t[0] <= 700.0 && t[1] <= 700.0 && t[2] <= 700.0 &&
                                               t[3] <= 700.0 && t[4] <= 700.0 && t[5] <= 700.0);
                if (!lean) {
                    double c[6];
                    exp_caps6(t, false, pin ? pairs_at(gz) : 0u, c);
                    c0 = c[0]; c1 = c[1]; c2 = c[2]; c3 = c[3]; c4 = c[4]; c5 = c[5];
                }
            }
        } else {
            // the three forward pair weights of this voxel: independent, branch-free evaluations
            const double a = own_val();
            if (FN == 1 && SPACING == 0) {
                // exponential term: form the three arguments, let the WARP agree that all of them are ordinary (<= 700, not
                // NaN -- true for every warp of a sane image) and evaluate without any range handling; the rare warp that
                // disagrees takes the general path.  Both paths give bit-identical weights for ordinary arguments.
                auto arg = [&](E iq) -> double {
                    const double b = build_val<E>(iq, use_max);
                    return exp_term_arg(Pz, use_max ? fmax(a, b) : fabs(__dsub_rn(a, b)));
                };
                const double tz = arg(at(hz + 1, ly + 1, lx + 1)), ty = arg(at(hz, ly + 2, lx + 1)), tx = arg(at(hz, ly + 1, lx + 2));
                if (__all_sync(0xffffffffu, tz <= 700.0 && ty <= 700.0 && tx <= 700.0)) {
                    wz = exp_neg_inrange(tz); wy = exp_neg_inrange(ty); wx = exp_neg_inrange(tx);
                } else {
                    wz = exp_neg(tz); wy = exp_neg(ty); wx = exp_neg(tx);
                    if (wz <= 0.0) wz = DBL_MIN;
                    if (wy <= 0.0) wy = DBL_MIN;
                    if (wx <= 0.0) wx = DBL_MIN;
                }
                if (!(pin && (z_pairs(L, gz) & 2u))) wz = 0.0;
                if (!(pin && has_py)) wy = 0.0;
                if (!(pin && has_px)) wx = 0.0;
            } else {
                wz = pair_w(Pz, a, at(hz + 1, ly + 1, lx + 1), pin && (z_pairs(L, gz) & 2u), sp_z);
                wy = pair_w(Pz, a, at(hz, ly + 2, lx + 1), pin && has_py, sp_y);
                wx = pair_w(Pz, a, at(hz, ly + 1, lx + 2), pin && has_px, sp_x);
            }
            wyb[(ly + 1) * 32 + lx] = wy;
            wxb[ly * 33 + lx + 1] = wx;
            __syncthreads();
        }
        if (pin) {
            const unsigned v = (unsigned)gz * L.stride[0] + (unsigned)gy * L.stride[1] + (unsigned)gx;
            if constexpr (!LAZY_EXP) {
                c0 = wz_back; c1 = wz; c3 = wy; c5 = wx;
                c2 = ly ? wyb[ly * 32 + lx] : s_wyh[lz * 32 + lx];
                c4 = lx ? wxb[ly * 33 + lx] : s_wxh[lz * 8 + ly];
                if (!LAZY) {
                    S.cap[0][v] = (T)c0; S.cap[1][v] = (T)c1; S.cap[2][v] = (T)c2;
                    S.cap[3][v] = (T)c3; S.cap[4][v] = (T)c4; S.cap[5][v] = (T)c5;
                }
                mm = tlinks(tr);
            }
            if (LAZY && copies) {
                if (A.img_copy) reinterpret_cast<E*>(A.img_copy)[v] = at(hz, ly + 1, lx + 1);
                if (A.prob_copy) {
                    if (TIN == 1 || !A.prob_f64) reinterpret_cast<float*>(A.prob_copy)[v] = (float)cur.p;
                    else reinterpret_cast<double*>(A.prob_copy)[v] = cur.p;
                }
            }
            const bool own = gz >= L.own0 && gz < L.own1;
            if (own) msum = __dadd_rn(msum, mm);
            if (!LAZY) S.tr[v] = tr;
            // ---- solver state (same arithmetic as k_init_tile and k_caps_tiles) ----
            const double trd = (double)tr;
            unsigned m;
            bool exc;
            if (LAZY_EXP && lean) {
                // every in-lattice weight is >= DBL_MIN: cap_bits gives the validity bits, and the clamped source excess
                // is > 0 exactly when source_active says so
                m = pairs_at(gz);
                exc = own && source_active(trd, m);
            } else {
                const double c[6] = {c0, c1, c2, c3, c4, c5};
                m = cap_bits(c);
                double e = source_excess(trd, c);
                if (!own) e = 0.0;
                if (!LAZY) S.excess[v] = (T)e;
                exc = e > 0;
            }
            if (trd < 0) m |= RM_SINK;
            S.rmask[v] = (uint8_t)m;
            const int h = (own && trd < 0) ? 1 : MGC_HINF;
            S.height[v] = h;
            if (own && (m & 0x3fu) != 0 && h == MGC_HINF) needs_any = 1u;
            if (exc) exc_any = 1u;
        }
        if (LAZY) {      // marker bit planes: one word per warp row and marker
            const unsigned bf = __ballot_sync(0xffffffffu, pin && (cur.fb & 1u)), bb = __ballot_sync(0xffffffffu, pin && (cur.fb & 2u));
            if (lx == 0 && gz < L.dim[0] && gy < L.dim[1]) {
                const unsigned w = ((unsigned)gz * (unsigned)L.dim[1] + (unsigned)gy) * (unsigned)nbx + (unsigned)bx;
                if (A.fg_plane) A.fg_plane[w] = bf;
                if (A.bg_plane) A.bg_plane[w] = bb;
            }
        }
        wz_back = wz;
        cur = nxt;
        // the planes of this step are read above; the next step writes the other buffer, the one after waits at its barrier
    }

    // ---- per solver tile flags and worklists (a warp row covers four 8^3 tiles: lanes 8j .. 8j+7) ----
    const unsigned bn = __ballot_sync(0xffffffffu, needs_any != 0), be = __ballot_sync(0xffffffffu, exc_any != 0);
    if (lx == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if ((bn >> (8 * j)) & 0xffu) atomicOr(&s_flags[j], 1);
            if ((be >> (8 * j)) & 0xffu) atomicOr(&s_flags[4 + j], 1);
        }
    }
    if (isbad) *bad = 1;
    // deterministic block sum of the add_tweights minima (fixed order: thread chain, warp shuffles, 8 warps)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) msum = __dadd_rn(msum, __shfl_down_sync(0xffffffffu, msum, o));
    if (lx == 0) s_red[ly] = msum;
    __syncthreads();
    if (tid == 0) {
        double t = s_red[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) t = __dadd_rn(t, s_red[w]);
        partials[((A.z_tile0 + bz) * nby + by) * nbx + bx] = t;
    }
    if (tid < 4) {
        const int tx = (x0 >> 3) + tid, ty = y0 >> 3, tz = z0 >> 3;
        if (tx < TL.nt[2] && ty < TL.nt[1] && tz < TL.nt[0]) {
            const int t = (tz * TL.nt[1] + ty) * TL.nt[2] + tx;
            const int any_needs = s_flags[tid], any_exc = s_flags[4 + tid];
            rflag[t] = any_needs;
            if (any_needs) rl.items[atomicAdd(rl.count, 1)] = t;
            pflag[t] = any_exc;
            if (LAZY) A.cmat[t] = 0;
            if (any_exc) {
                const WorkList& pl = ((tz + ty + tx) & 1) ? pl1 : pl0;
                pl.items[atomicAdd(pl.count, 1)] = t;
            }
        }
    }
}

template <typename E, typename T, int FN, int USE_MAX, int SPACING, int TIN = 0, int LAZY = 0>
__global__ void __launch_bounds__(BUILD_THREADS)
k_build_tile(Lattice L, Tiles TL, State<T> S, const __grid_constant__ BuildMaps maps, BuildArgs A, BoundaryParams P,
             int* __restrict__ bad, double* __restrict__ partials, int* __restrict__ rflag, WorkList rl,
             int* __restrict__ pflag, WorkList pl0, WorkList pl1)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    build_block<E, T, FN, USE_MAX, SPACING, TIN, LAZY>((int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z, (int)gridDim.x,
                                                       (int)gridDim.y, true, 0u, smem_raw, L, TL, S, maps, A, P, bad,
                                                       partials, rflag, rl, pflag, pl0, pl1);
}

template <typename E>
constexpr size_t build_smem_bytes()
{
    return (size_t)BUILD_TIN_OFFSET((BUILD_HZ * BUILD_HY * BuildBox<E>::BX * (int)sizeof(E) + 127) / 128 * 128) +
           (size_t)BUILD_TZ * BUILD_TY * BUILD_TX * (8 + 1 + 1);
}

// ---------------------------------------------------------------------------------------------------
// The lazy build under the exponential term without spacing, image block staged by TMA, as two launches (DESIGN.md §4.0):
//   k_build_lean    : stages every block and runs its range test; a block that passes is streamed by a loop that holds
//                     nothing but the lean path, a block that fails writes nothing and appends its index to a list;
//   k_build_refused : persistent CTAs run the k_build_tile body (range test, per-warp vote, six weights) on the listed
//                     blocks.  The launch follows on the same stream without a host synchronisation; it reads the
//                     list's length on the device and returns at once when nothing was refused.
// Both write exactly what k_build_tile<..., LAZY = 1> writes for their blocks.
// ---------------------------------------------------------------------------------------------------
template <typename E, int USE_MAX, int TIN>
__global__ void __launch_bounds__(BUILD_THREADS, 4)
k_build_refused(Lattice L, Tiles TL, State<double> S, const __grid_constant__ BuildMaps maps, BuildArgs A, BoundaryParams P,
                int* __restrict__ bad, double* __restrict__ partials, int* __restrict__ rflag, WorkList rl,
                int* __restrict__ pflag, WorkList pl0, WorkList pl1, const int* __restrict__ list,
                const int* __restrict__ count, int* __restrict__ total, int nbx, int nby)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int n = *count;
    if (blockIdx.x == 0 && threadIdx.x == 0 && n) atomicAdd(total, n);
    for (int i = blockIdx.x, it = 0; i < n; i += gridDim.x, ++it) {
        const int b = list[i];
        const int bx = b % nbx, r = b / nbx;
        build_block<E, double, 1, USE_MAX, 0, TIN, 1>(bx, r % nby, r / nby, nbx, nby, it == 0, (unsigned)it & 1u, smem_raw,
                                                      L, TL, S, maps, A, P, bad, partials, rflag, rl, pflag, pl0, pl1);
        __syncthreads();          // shared memory is restaged for the next block
    }
}

// shared memory of k_build_lean: image block with halo | probability block | fg block | bg block | barrier, tile flags,
// range and reduction scratch.  The add_tweights minima of the block (2048 doubles) overlay the image block once the
// range test and the image copy have read it; the image region is at least that large.
template <typename E, int TIN>
struct LeanSmem {
    static constexpr int IMG_BYTES = BUILD_HZ * BUILD_HY * BuildBox<E>::BX * (int)sizeof(E);
    static constexpr int MM_BYTES = BUILD_TZ * BUILD_TY * BUILD_TX * 8;
    static constexpr int PROB_OFF = (IMG_BYTES > MM_BYTES ? (IMG_BYTES + 127) / 128 * 128 : MM_BYTES);
    static constexpr int FG_OFF = PROB_OFF + BUILD_TZ * BUILD_TY * BUILD_TX * (TIN == 1 ? 4 : 8);
    static constexpr int BG_OFF = FG_OFF + BUILD_TZ * BUILD_TY * BUILD_TX;
    static constexpr int MISC_OFF = BG_OFF + BUILD_TZ * BUILD_TY * BUILD_TX;
    static constexpr int BYTES = MISC_OFF + 256;
};

// The range test of a staged block (block_exp_ordinary over every cell of the box), uniform over the CTA.  float32:
// integer keys (gc_exprange.cuh); other types: the float fold of k_build_tile.  `scratch`: 192 bytes of shared memory.
template <typename E>
__device__ __forceinline__ bool lean_range_test(const E* s_img, unsigned char* scratch, bool use_max, double inv_sigma2)
{
    constexpr int NV = LeanSmem<E, 0>::IMG_BYTES / 16;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if constexpr (std::is_same<E, float>::value) {
        int kmin = INT_MAX, kmax = INT_MIN;
        for (int i = tid; i < NV; i += BUILD_THREADS) {
            const int4 q = reinterpret_cast<const int4*>(s_img)[i];
            const int a = er_f32_key(q.x), b = er_f32_key(q.y), c = er_f32_key(q.z), d = er_f32_key(q.w);
            kmin = min(kmin, min(min(a, b), min(c, d)));
            kmax = max(kmax, max(max(a, b), max(c, d)));
        }
        kmin = __reduce_min_sync(0xffffffffu, kmin);
        kmax = __reduce_max_sync(0xffffffffu, kmax);
        int* s_k = reinterpret_cast<int*>(scratch);
        if (lane == 0) { s_k[w] = kmin; s_k[8 + w] = kmax; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 8; ++k) { kmin = min(kmin, s_k[k]); kmax = max(kmax, s_k[8 + k]); }
        return block_exp_ordinary_keys(kmin, kmax, use_max, inv_sigma2);
    } else {
        E lo = (E)INFINITY, hi = (E)-INFINITY;
        bool nan = false;
        for (int i = tid; i < NV; i += BUILD_THREADS) {
            const uint4 q = reinterpret_cast<const uint4*>(s_img)[i];
            E e[16 / sizeof(E)];
            memcpy(e, &q, 16);
#pragma unroll
            for (int k = 0; k < (int)(16 / sizeof(E)); ++k) block_range_add<E>(lo, hi, nan, e[k]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const E olo = __shfl_xor_sync(0xffffffffu, lo, o), ohi = __shfl_xor_sync(0xffffffffu, hi, o);
            block_range_add<E>(lo, hi, nan, olo);
            block_range_add<E>(lo, hi, nan, ohi);
        }
        nan = __any_sync(0xffffffffu, nan);
        E* s_rng = reinterpret_cast<E*>(scratch);                    // [8] warp minima, [8] warp maxima
        int* s_rnan = reinterpret_cast<int*>(scratch + 16 * sizeof(E));
        if (lane == 0) { s_rng[w] = lo; s_rng[8 + w] = hi; s_rnan[w] = nan ? 1 : 0; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            block_range_add<E>(lo, hi, nan, s_rng[k]);
            block_range_add<E>(lo, hi, nan, s_rng[8 + k]);
            nan = nan || s_rnan[k] != 0;
        }
        return block_exp_ordinary(Elem<E>::val(lo), Elem<E>::val(hi), nan, use_max, inv_sigma2);
    }
}

// bits k = 0..3 of the result: byte k of w is not zero
__device__ __forceinline__ unsigned nonzero_bytes4(unsigned w)
{
    return ((__vcmpne4(w, 0u) & 0x08040201u) * 0x01010101u) >> 24;
}

// The lean build.  Thread (z, y, g) of the block -- tid = (z * 8 + y) * 4 + g -- owns the 8 voxels x0 + 8g .. x0 + 8g + 7
// of row (z, y), the x-range of one 8^3 solver tile: it reads them with vector loads, replays their t-links, and writes
// rmask (one 8-byte store), height (two 16-byte stores), its byte of the marker words (a quad of threads covers one
// word) and, where the handle wants them, the image and map copies.  The block's add_tweights partial is formed in
// k_build_tile's order: every voxel's minimum goes to shared memory, and thread (y, x) then chains its column over z,
// followed by the same warp shuffle tree and the same fixed order over the 8 warps.  E: float or double (TMA-staged).
template <typename E, int TIN>
__global__ void __launch_bounds__(BUILD_THREADS, 6)
k_build_lean(Lattice L, Tiles TL, State<double> S, const __grid_constant__ BuildMaps maps, BuildArgs A, BoundaryParams P,
             double* __restrict__ partials, int* __restrict__ rflag, WorkList rl, int* __restrict__ pflag, WorkList pl0,
             WorkList pl1, int* __restrict__ refused, int* __restrict__ n_refused, int refuse_all)
{
    using LS = LeanSmem<E, TIN>;
    constexpr int BX = BuildBox<E>::BX, PAD = BuildBox<E>::PAD;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    E* s_img = reinterpret_cast<E*>(smem_raw);
    unsigned char* s_prob = smem_raw + LS::PROB_OFF;
    unsigned char* s_fg = smem_raw + LS::FG_OFF;
    unsigned char* s_bg = smem_raw + LS::BG_OFF;
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(smem_raw + LS::MISC_OFF);
    int* s_flags = reinterpret_cast<int*>(smem_raw + LS::MISC_OFF + 8);          // [4] needs, [4] has excess
    unsigned char* s_zp = smem_raw + LS::MISC_OFF + 40;                           // [8] z_pairs of the block's planes
    unsigned char* s_scr = smem_raw + LS::MISC_OFF + 64;                          // range test, then block reduction
    double* s_mm = reinterpret_cast<double*>(smem_raw);                           // [8 z][8 y][32 x], x ^ y swizzled

    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * BUILD_TX, y0 = blockIdx.y * BUILD_TY, z0 = (A.z_tile0 + (int)blockIdx.z) * BUILD_TZ;
    const int cx = x0 == 0 ? -1 : PAD - 1, cy = y0 == 0 ? -1 : 0, cz = z0 == 0 ? -1 : 0;
    const bool has_prob = TIN == 1 || A.prob != nullptr;
    if (tid < 8) s_flags[tid] = 0;
    // the axis-0 pair bits of the block's planes, formed once per plane here rather than per thread in the register-bound
    // state section below
    if (tid < BUILD_TZ) s_zp[tid] = (unsigned char)z_pairs(L, z0 + tid);
    if (tid == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned pbytes = (has_prob && A.tma_prob) ? (unsigned)(BUILD_TZ * BUILD_TY * BUILD_TX * (A.prob_f64 ? 8 : 4)) : 0u;
        const unsigned mbytes = (unsigned)(BUILD_TZ * BUILD_TY * BUILD_TX);
        mbar_expect_tx(bar, (unsigned)LS::IMG_BYTES + pbytes + ((A.tma_mark & 1) ? mbytes : 0u) + ((A.tma_mark & 2) ? mbytes : 0u));
        tma_load_3d(s_img, &maps.img, bar, x0 - 1 - cx, y0 - 1 - cy, z0 - 1 - cz);
        if (pbytes) tma_load_3d(s_prob, &maps.prob, bar, x0, y0, z0);
        if (A.tma_mark & 1) tma_load_3d(s_fg, &maps.fg, bar, x0, y0, z0);
        if (A.tma_mark & 2) tma_load_3d(s_bg, &maps.bg, bar, x0, y0, z0);
    }
    __syncthreads();
    mbar_wait(bar, 0u);

    if (!lean_range_test<E>(s_img, s_scr, P.use_max != 0, range_inv_sigma2(P, L, z0 - 1, z0 + BUILD_TZ)) || refuse_all) {
        if (tid == 0) refused[atomicAdd(n_refused, 1)] = ((int)blockIdx.z * (int)gridDim.y + (int)blockIdx.y) * (int)gridDim.x + (int)blockIdx.x;
        return;          // uniform over the CTA
    }

    const int g = tid & 3, ty = (tid >> 2) & 7, tz = tid >> 5;
    const int gy = y0 + ty, gz = z0 + tz, xb = x0 + 8 * g;
    const bool row_in = gz < L.dim[0] && gy < L.dim[1];
    const int nx = row_in ? min(8, L.dim[2] - xb) : 0;                 // in-lattice voxels of this thread (<= 0: none)
    const unsigned pin = nx >= 8 ? 0xffu : (nx > 0 ? (1u << nx) - 1u : 0u);
    const unsigned v = (unsigned)gz * L.stride[0] + (unsigned)gy * L.stride[1] + (unsigned)xb;
    const int si = (tz * BUILD_TY + ty) * BUILD_TX + 8 * g;             // index inside the staged 8 x 8 x 32 blocks

    // ---- the image copy: the last read of the image block, which the minima overlay (the range test's reads end at its
    // barrier) ----
    if (A.img_copy) {
        if (nx > 0) {
            const E* src = s_img + ((tz + 1 + cz) * BUILD_HY + (ty + 1 + cy)) * BX + (8 * g + 1 + cx);
            E* dst = reinterpret_cast<E*>(A.img_copy) + v;
            if (nx == 8 && (v % (16 / sizeof(E))) == 0) {
#pragma unroll
                for (int k = 0; k < (int)(8 * sizeof(E) / 16); ++k) reinterpret_cast<uint4*>(dst)[k] = reinterpret_cast<const uint4*>(src)[k];
            } else {
                for (int k = 0; k < nx; ++k) dst[k] = src[k];
            }
        }
        __syncthreads();
    }

    // ---- t-link inputs ----
    using PT = typename std::conditional<TIN == 1, float, double>::type;
    PT p[8];
    unsigned fgm = 0u, bgm = 0u;                     // bit k: voxel k carries the marker
    if constexpr (TIN == 1) {
        const float4 a = reinterpret_cast<const float4*>(s_prob + si * 4)[0], b = reinterpret_cast<const float4*>(s_prob + si * 4)[1];
        p[0] = a.x; p[1] = a.y; p[2] = a.z; p[3] = a.w; p[4] = b.x; p[5] = b.y; p[6] = b.z; p[7] = b.w;
        const uint2 f = *reinterpret_cast<const uint2*>(s_fg + si), q = *reinterpret_cast<const uint2*>(s_bg + si);
        fgm = nonzero_bytes4(f.x) | (nonzero_bytes4(f.y) << 4);
        bgm = nonzero_bytes4(q.x) | (nonzero_bytes4(q.y) << 4);
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            p[k] = 0.0;
            if (k >= nx) continue;
            const unsigned vk = v + (unsigned)k;
            if (A.prob) {
                if (A.tma_prob) p[k] = A.prob_f64 ? reinterpret_cast<const double*>(s_prob)[si + k] : (double)reinterpret_cast<const float*>(s_prob)[si + k];
                else p[k] = (A.dbg & 1) ? 0.3 : (A.prob_f64 ? reinterpret_cast<const double*>(A.prob)[vk] : (double)reinterpret_cast<const float*>(A.prob)[vk]);
            }
            if (A.fg_bits || A.bg_bits) {
                if (A.fg_bits) fgm |= ((A.fg_bits[vk >> 5] >> (vk & 31u)) & 1u) << k;
                if (A.bg_bits) bgm |= ((A.bg_bits[vk >> 5] >> (vk & 31u)) & 1u) << k;
            } else {
                if (A.fg && ((A.tma_mark & 1) ? s_fg[si + k] : A.fg[vk])) fgm |= 1u << k;
                if (A.bg && ((A.tma_mark & 2) ? s_bg[si + k] : A.bg[vk])) bgm |= 1u << k;
            }
        }
    }
    if (A.prob_copy && nx > 0) {
        if (TIN == 1 || !A.prob_f64) {
            float* dst = reinterpret_cast<float*>(A.prob_copy) + v;
            if (nx == 8 && (v & 3u) == 0) {
                reinterpret_cast<float4*>(dst)[0] = make_float4((float)p[0], (float)p[1], (float)p[2], (float)p[3]);
                reinterpret_cast<float4*>(dst)[1] = make_float4((float)p[4], (float)p[5], (float)p[6], (float)p[7]);
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) if (k < nx) dst[k] = (float)p[k];
            }
        } else {
            double* dst = reinterpret_cast<double*>(A.prob_copy) + v;
#pragma unroll
            for (int k = 0; k < 8; ++k) if (k < nx) dst[k] = (double)p[k];
        }
    }

    // ---- t-links and solver state ----
    const bool own = gz >= L.own0 && gz < L.own1;
    const unsigned zy = s_zp[tz] | (gy > 0 ? 4u : 0u) | (gy + 1 < L.dim[1] ? 8u : 0u);
    const bool f32 = TIN == 1 || A.compute_f32 != 0;
    unsigned rm_lo = 0u, rm_hi = 0u, sinkm = 0u;
    bool needs = false, exc = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        double tr = 0.0;
        const unsigned fb = ((fgm >> k) & 1u) | (((bgm >> k) & 1u) << 1);
        s_mm[(tz * BUILD_TY + ty) * BUILD_TX + ((8 * g + k) ^ ty)] = tlink_replay<double>(tr, has_prob, (double)p[k], f32, A.alpha, fb);
        const int gx = xb + k;
        // the in-lattice pairs (every weight of the block is >= DBL_MIN: they are the n-link bits of rmask)
        const unsigned pr = zy | (gx > 0 ? 16u : 0u) | (gx + 1 < L.dim[2] ? 32u : 0u);
        const unsigned m = pr | (tr < 0 ? RM_SINK : 0u);
        if (k < 4) rm_lo |= m << (8 * k); else rm_hi |= m << (8 * (k - 4));
        if (tr < 0) sinkm |= 1u << k;
        if ((pin >> k) & 1u) {
            if (own && pr != 0u && !(tr < 0)) needs = true;        // an arc, and the label is not the sink's 1
            if (own && source_active(tr, pr)) exc = true;
        }
    }
    if (nx > 0) {
        const int h_sink = own ? 1 : MGC_HINF;
        auto h_of = [&](int k) -> int { return ((sinkm >> k) & 1u) ? h_sink : MGC_HINF; };
        if (nx == 8 && (v & 7u) == 0) {
            *reinterpret_cast<uint2*>(S.rmask + v) = make_uint2(rm_lo, rm_hi);
        } else {
            for (int k = 0; k < nx; ++k) S.rmask[v + k] = (uint8_t)((k < 4 ? rm_lo >> (8 * k) : rm_hi >> (8 * (k - 4))) & 0xffu);
        }
        if (nx == 8 && (v & 3u) == 0) {
            reinterpret_cast<int4*>(S.height + v)[0] = make_int4(h_of(0), h_of(1), h_of(2), h_of(3));
            reinterpret_cast<int4*>(S.height + v)[1] = make_int4(h_of(4), h_of(5), h_of(6), h_of(7));
        } else {
            for (int k = 0; k < nx; ++k) S.height[v + k] = h_of(k);
        }
    }
    // marker bit planes: word (gz, gy) of this block is the bytes of the row's four threads
    {
        unsigned wf = (fgm & pin) << (8 * g), wb = (bgm & pin) << (8 * g);
        wf |= __shfl_xor_sync(0xffffffffu, wf, 1); wb |= __shfl_xor_sync(0xffffffffu, wb, 1);
        wf |= __shfl_xor_sync(0xffffffffu, wf, 2); wb |= __shfl_xor_sync(0xffffffffu, wb, 2);
        if (g == 0 && row_in) {
            const unsigned w = ((unsigned)gz * (unsigned)L.dim[1] + (unsigned)gy) * gridDim.x + blockIdx.x;
            if (A.fg_plane) A.fg_plane[w] = wf;
            if (A.bg_plane) A.bg_plane[w] = wb;
        }
    }
    // ---- per solver tile flags: lanes g, g + 4, ... of every warp cover tile g ----
    const unsigned bn = __ballot_sync(0xffffffffu, needs), be = __ballot_sync(0xffffffffu, exc);
    if ((tid & 31) == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (bn & (0x11111111u << j)) atomicOr(&s_flags[j], 1);
            if (be & (0x11111111u << j)) atomicOr(&s_flags[4 + j], 1);
        }
    }
    __syncthreads();

    // ---- the block's add_tweights partial, in k_build_tile's order ----
    {
        const int lx = tid & 31, ly = tid >> 5;
        const bool col_in = y0 + ly < L.dim[1] && x0 + lx < L.dim[2];
        double msum = 0.0;
#pragma unroll
        for (int lz = 0; lz < BUILD_TZ; ++lz) {
            const int cz2 = z0 + lz;
            if (col_in && cz2 < L.dim[0] && cz2 >= L.own0 && cz2 < L.own1)
                msum = __dadd_rn(msum, s_mm[(lz * BUILD_TY + ly) * BUILD_TX + (lx ^ ly)]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) msum = __dadd_rn(msum, __shfl_down_sync(0xffffffffu, msum, o));
        double* s_red = reinterpret_cast<double*>(s_scr);
        if (lx == 0) s_red[ly] = msum;
        __syncthreads();
        if (tid == 0) {
            double t = s_red[0];
#pragma unroll
            for (int w = 1; w < 8; ++w) t = __dadd_rn(t, s_red[w]);
            partials[((A.z_tile0 + (int)blockIdx.z) * (int)gridDim.y + (int)blockIdx.y) * (int)gridDim.x + (int)blockIdx.x] = t;
        }
    }
    if (tid < 4) {
        const int tx = (x0 >> 3) + tid, tyy = y0 >> 3, tzz = z0 >> 3;
        if (tx < TL.nt[2] && tyy < TL.nt[1] && tzz < TL.nt[0]) {
            const int t = (tzz * TL.nt[1] + tyy) * TL.nt[2] + tx;
            const int any_needs = s_flags[tid], any_exc = s_flags[4 + tid];
            rflag[t] = any_needs;
            if (any_needs) rl.items[atomicAdd(rl.count, 1)] = t;
            pflag[t] = any_exc;
            A.cmat[t] = 0;
            if (any_exc) {
                const WorkList& pl = ((tzz + tyy + tx) & 1) ? pl1 : pl0;
                pl.items[atomicAdd(pl.count, 1)] = t;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// The implicit push state of a lazy build, per voxel of a tile that is not materialised yet
// ---------------------------------------------------------------------------------------------------
// the in-lattice pairs of an in-lattice voxel (bit k: the pair across face k exists)
__device__ __forceinline__ unsigned tile_pairs(const Lattice& L, const TileCtx& c)
{
    const int gz = c.tz * TILE + c.lz, gy = c.ty * TILE + c.ly, gx = c.tx * TILE + c.lx;
    return z_pairs(L, gz) | (gy > 0 ? 4u : 0u) | (gy + 1 < L.dim[1] ? 8u : 0u) | (gx > 0 ? 16u : 0u) |
           (gx + 1 < L.dim[2] ? 32u : 0u);
}

// the t-link inputs of an in-lattice voxel: its probability (0 without a map) and marker bits (bit 0 fg, bit 1 bg)
__device__ __forceinline__ void lazy_tin_load(const Lattice& L, const LazyTin& tin, const TileCtx& c, double& p, unsigned& fb)
{
    const int gz = c.tz * TILE + c.lz, gy = c.ty * TILE + c.ly, gx = c.tx * TILE + c.lx;
    if (tin.prob) p = tin.prob_f64 ? reinterpret_cast<const double*>(tin.prob)[c.v] : (double)reinterpret_cast<const float*>(tin.prob)[c.v];
    const unsigned w = ((unsigned)gz * (unsigned)L.dim[1] + (unsigned)gy) * (unsigned)tin.words + ((unsigned)gx >> 5);
    if (tin.fg) fb |= (tin.fg[w] >> (gx & 31)) & 1u;
    if (tin.bg) fb |= ((tin.bg[w] >> (gx & 31)) & 1u) << 1;
}

// tr of the build, from those inputs
__device__ __forceinline__ double lazy_tr(const LazyTin& tin, double p, unsigned fb)
{
    double tr = 0.0;
    tlink_replay<double>(tr, tin.prob != nullptr, p, tin.compute_f32 != 0, tin.alpha, fb);
    return tr;
}

// whether an owned, in-lattice voxel of a tile that is not materialised holds excess: the build's source excess, since
// nothing else reaches such a tile (a push materialises its receivers first)
__device__ __forceinline__ bool lazy_has_excess(const Lattice& L, const LazyTin& tin, const TileCtx& c)
{
    double p = 0.0;
    unsigned fb = 0u;
    lazy_tin_load(L, tin, c, p, fb);
    return source_active(lazy_tr(tin, p, fb), tile_pairs(L, c));
}

// an active voxel: owned, at a finite label, with excess; `mat` = its tile's push state is materialised
template <typename T>
__device__ __forceinline__ bool voxel_active(const Lattice& L, const State<T>& S, const LazyTin& tin, const TileCtx& c, int h, bool mat)
{
    if (!c.own || h >= MGC_HINF) return false;
    return mat ? S.excess[c.v] > 0 : lazy_has_excess(L, tin, c);
}

// ---------------------------------------------------------------------------------------------------
// Label window of the push passes on an easy instance (sweep_mode == 0, DESIGN.md §4.3).  Before a colour's push launch,
//   k_window_min   : the lowest label over the active voxels of every listed tile, and the minimum gmin over the list;
//   k_window_split : tiles whose lowest active label is <= gmin + PUSH_WINDOW go to the list pushed (and materialised)
//                    now; the other tiles with an active voxel wait on the colour's next list (pflag stays set); tiles
//                    without one leave the lists.  After an exact relabel a voxel it labelled HINF never becomes active
//                    again; tiles that leave unmaterialised are kept for mgc_add_seeds.  After a relabel stopped at a
//                    label cap (`labels_capped`, the first relabel of a solve) HINF only means "deeper than the cap": such
//                    tiles wait on the next list too, and the next, exact, relabel labels them.
// Both read a tile that is not materialised yet through its implicit push state (cmat[t] == 0; cmat == nullptr: every
// tile is materialised).  They are in gc_solve_kernels.cuh with the materialiser; the host shares the constants below.
// ---------------------------------------------------------------------------------------------------
#define PUSH_WINDOW 8
// label cap of the first global relabel of an easy solve (no stop test reads it; only the window above uses its labels):
// the BFS labels the voxels within FIRST_RELABEL_CAP of the sink and leaves the rest HINF (relabel_visit)
#define FIRST_RELABEL_CAP 12
#define WIN_GMIN 0         // control words: lowest active label of the list
#define WIN_NOW 1          // ... count of the list pushed now
#define WIN_DEFERRED 2     // ... tile deferrals since the solve started
#define WIN_DROPPED 3      // ... tiles that left the lists since the solve started
#define WIN_NDROP 4        // ... tiles that left unmaterialised since the build (list `drop_items`)
