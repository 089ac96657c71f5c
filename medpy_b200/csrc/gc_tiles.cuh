// gc_tiles.cuh -- tile-resident solver kernels for the 3-D lattice (gc_tiles4.cuh holds the 4-D ones).  Every lattice
// handle, z-slabs included, runs the tile solver.
//
// The lattice is cut into 8x8x8 tiles.  A 512-thread CTA owns one tile for the duration of a visit, keeps the
// tile's state on chip (heights with a 1-voxel halo in shared memory; in the push kernel the six residual
// capacities, excess and sink-link state of each voxel in its thread's registers) and iterates there, so a
// visit costs one read and one write of the tile in HBM however many push/relabel or relaxation rounds it
// takes.  Work is driven by per-tile WORKLISTS: persistent CTAs (a small multiple of the SM count) pull tile
// ids from a device-side list with an atomic cursor; a tile is listed only if it may hold work (an active
// voxel / a label that may still drop), and kernels append to the list of the next pass themselves.
//
//  * k_init_tile          : solver state from the terms (source-excess clamp, residual mask, first labels) and
//                           the first worklists, fused in one pass over the lattice.
//  * k_relabel_reset      : start of a later global relabel: labels from the residual mask, new worklist
//                           (gc_solve_kernels.cuh, with the z-slab kernels in gc_slab_kernels.cuh).
//  * relabel_visit        : exact backward BFS from the sink (global relabel), one tile visit; k_bfs_coop
//                           (gc_persist.cuh) runs every pass in one cooperative launch.  Labels only decrease during it,
//                           so tiles run concurrently with benign races on the halo; a tile whose border labels
//                           dropped lists its face neighbours for the next pass.
//  * k_push_tile          : push/relabel discharge of one tile: synchronous rounds, "push then pull" through a
//                           shared-memory outflow buffer, so every state update is made by the voxel's own
//                           thread -- no shared-memory atomics, deterministic inside the tile.  Tiles are
//                           processed in two colours (3-D checkerboard): tiles of one colour are never
//                           face-adjacent, so a running tile is the only writer of its own voxels; flow
//                           crossing a face lands in the idle neighbour's arrays with global atomics (a corner
//                           voxel can receive from up to three running tiles).
#pragma once
#include "gc_common.cuh"

#define TILE 8
#define TILE_VOX 512
#define HALO_DIM 10
#define HALO_VOX 1000
#define RM_SINK 0x40u   // bit 6 of rmask: residual capacity towards the sink
#define RM_SINKV 0x80u  // bit 7 of rmask: sink[v] (flow absorbed so far) has been written; unset = 0, the array is never zero-filled

struct Tiles {
    int nt[3];      // tiles along z, y, x
    int ntiles;
    // tiles whose labels (or sink-link residual bits) were written since the last relabel reset: only these have to be
    // put back into the reset state (label 1 where a sink link is residual, HINF elsewhere) before the next BFS
    int* dflag;     // per tile: already on the dirty list (nullptr: tracking off)
    int* ditems;    // the dirty list
    int* dcount;
};

__device__ __forceinline__ void mark_dirty(const Tiles& TL, int t)
{
    if (TL.dflag && atomicExch(&TL.dflag[t], 1) == 0) TL.ditems[atomicAdd(TL.dcount, 1)] = t;
}

// worklists: items[] + count; kernels consume `cur` through an atomic cursor and append to `next`
struct WorkList {
    int* items;
    int* count;
};

// control block in device memory (ints): mgc_graph::d_tcount (gc_handle.cuh)
//   [0],[1]   relabel list counts          [2..5] push list counts [colour*2 + buffer]
//   [8]       work cursor                  [11] relabel list consumed next                [15] relabel passes
#define CTL_CURSOR 8
#define CTL_RLCUR 11
#define CTL_RELP 15

__device__ __forceinline__ int hidx(int z, int y, int x) { return (z * HALO_DIM + y) * HALO_DIM + x; }

template <int K>
__device__ __forceinline__ int hoff()
{
    constexpr int s = (K >> 1) == 0 ? HALO_DIM * HALO_DIM : ((K >> 1) == 1 ? HALO_DIM : 1);
    return (K & 1) ? s : -s;
}

struct TileCtx {
    int t;                 // tile id
    int tz, ty, tx;        // tile coordinates
    int lz, ly, lx;        // local coordinates of this thread's voxel
    bool inb;              // voxel inside the lattice
    bool own;              // ... and owned (not a ghost plane of a z-slab)
    unsigned v;            // flat index (valid when inb)
};

__device__ __forceinline__ TileCtx tile_ctx(const Lattice& L, const Tiles& TL, int t)
{
    TileCtx c;
    c.t = t;
    c.tx = t % TL.nt[2];
    int r = t / TL.nt[2];
    c.ty = r % TL.nt[1];
    c.tz = r / TL.nt[1];
    const int tid = threadIdx.x;
    c.lx = tid & 7; c.ly = (tid >> 3) & 7; c.lz = tid >> 6;
    const int gz = c.tz * TILE + c.lz, gy = c.ty * TILE + c.ly, gx = c.tx * TILE + c.lx;
    c.inb = gz < L.dim[0] && gy < L.dim[1] && gx < L.dim[2];
    c.v = c.inb ? (unsigned)gz * L.stride[0] + (unsigned)gy * L.stride[1] + (unsigned)gx : 0u;
    c.own = c.inb && gz >= L.own0 && gz < L.own1;
    return c;
}

__device__ __forceinline__ int tile_color(const TileCtx& c) { return (c.tz + c.ty + c.tx) & 1; }

// neighbour tile id across face k (only valid if it exists)
__device__ __forceinline__ int tile_nbr(const Tiles& TL, int t, int k)
{
    const int s = (k >> 1) == 0 ? TL.nt[1] * TL.nt[2] : ((k >> 1) == 1 ? TL.nt[2] : 1);
    return (k & 1) ? t + s : t - s;
}

// cooperative load of heights (own voxel + the six halo faces) into the 10^3 cube; out-of-lattice -> HINF
__device__ __forceinline__ int load_heights(const Lattice& L, const TileCtx& c, const int* __restrict__ height, int* sh)
{
    const int tid = threadIdx.x;
    // .cg loads: labels are read while other CTAs lower them (asynchronous BFS) -- never serve them from a stale L1 line
    int h0 = c.inb ? __ldcg(height + c.v) : MGC_HINF;
    sh[hidx(c.lz + 1, c.ly + 1, c.lx + 1)] = h0;
    if (tid < 384) {
        const int face = tid >> 6, a = (tid >> 3) & 7, b = tid & 7;
        int z, y, x;   // local coordinates in [-1, 8]
        switch (face) {
            case 0: z = -1; y = a; x = b; break;
            case 1: z = TILE; y = a; x = b; break;
            case 2: z = a; y = -1; x = b; break;
            case 3: z = a; y = TILE; x = b; break;
            case 4: z = a; y = b; x = -1; break;
            default: z = a; y = b; x = TILE; break;
        }
        const int gz = c.tz * TILE + z, gy = c.ty * TILE + y, gx = c.tx * TILE + x;
        int h = MGC_HINF;
        if (gz >= 0 && gy >= 0 && gx >= 0 && gz < L.dim[0] && gy < L.dim[1] && gx < L.dim[2])
            h = __ldcg(height + ((unsigned)gz * L.stride[0] + (unsigned)gy * L.stride[1] + (unsigned)gx));
        sh[hidx(z + 1, y + 1, x + 1)] = h;
    }
    return h0;
}

// append tile t to a worklist unless it is already flagged
__device__ __forceinline__ void list_push(int* __restrict__ flags, const WorkList& wl, int t)
{
    if (atomicExch(&flags[t], 1) == 0) wl.items[atomicAdd(wl.count, 1)] = t;
}

// persistent-CTA work fetch: returns the next tile id of `cur`, or -1 when the list is exhausted
__device__ __forceinline__ int fetch_tile(const WorkList& cur, int* __restrict__ cursor, int* s_slot)
{
    __syncthreads();                       // previous tile fully done (also protects s_slot reuse)
    if (threadIdx.x == 0) {
        const int i = atomicAdd(cursor, 1);
        *s_slot = (i < *(volatile int*)cur.count) ? cur.items[i] : -1;
    }
    __syncthreads();
    return *s_slot;
}

// ---------------------------------------------------------------------------------------------------
// init: one pass over every tile after the terms are in
//   excess = min(max(tr,0), roundup(sum of out-capacities))   (source-link clamp, DESIGN.md §4.2)
//   sink[] (flow absorbed so far) is NOT written: rmask bit RM_SINKV marks entries that hold a value
//   rmask, first labels (1 where a sink link exists, else HINF)
//   relabel worklist <- tiles holding an unlabelled voxel with residual out-arcs
//   push worklists   <- tiles holding a voxel with excess
// WARM (MGC_OPT_WARM): tr > 0 becomes tr - excess, BK's residual source capacity, which a later fold reads back as r(v)
// (gc_seeds.cuh).  Nothing else reads tr > 0 once the excess is set.
// ---------------------------------------------------------------------------------------------------
template <typename T, bool WARM = false>
__global__ void __launch_bounds__(TILE_VOX) k_init_tile(Lattice L, Tiles TL, State<T> S, int* __restrict__ rflag, WorkList rl,
                                                        int* __restrict__ pflag, WorkList pl0, WorkList pl1)
{
    const TileCtx c = tile_ctx(L, TL, blockIdx.x);
    int needs = 0, hasexc = 0;
    if (c.inb) {
        const double tr = (double)S.tr[c.v];
        unsigned m = 0;
        double out = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            const double ck = (double)S.cap[k][c.v];
            if (ck > 0) m |= 1u << k;
            out = __dadd_ru(out, ck);
        }
        double e = 0.0;
        if (tr > 0) { const double lim = out * SOURCE_CLAMP_SLACK; e = tr < lim ? tr : lim; if (!(out == out)) e = tr; }
        if (tr < 0) m |= RM_SINK;
        if (!c.own) e = 0.0;
        if (WARM && tr > 0) S.tr[c.v] = (T)(tr - e);
        S.excess[c.v] = (T)e;
        S.rmask[c.v] = (uint8_t)m;          // RM_SINKV clear: sink[v] counts as 0 without being written
        const int h = (c.own && tr < 0) ? 1 : MGC_HINF;
        S.height[c.v] = h;
        needs = (c.own && (m & 0x3fu) != 0 && h == MGC_HINF) ? 1 : 0;
        hasexc = e > 0 ? 1 : 0;
    }
    const int any_needs = __syncthreads_or(needs);
    const int any_exc = __syncthreads_or(hasexc);
    if (threadIdx.x == 0) {
        rflag[c.t] = any_needs;
        if (any_needs) rl.items[atomicAdd(rl.count, 1)] = c.t;
        pflag[c.t] = any_exc;
        if (any_exc) {
            const WorkList& pl = tile_color(c) ? pl1 : pl0;
            pl.items[atomicAdd(pl.count, 1)] = c.t;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// global relabel: one tile visit (k_bfs_coop of gc_persist.cuh runs the passes over the worklists)
// ---------------------------------------------------------------------------------------------------
// one tile visit of the global relabel: relax inside the tile until nothing changes, write back, list the face
// neighbours whose halo changed.  `sh` = HALO_VOX ints of shared memory.
// `cap`: no voxel is lowered to a label above it (it keeps HINF), and no neighbour is woken by a label that could only
// lower it above the cap.  Labels strictly decrease along a shortest residual path to the sink, so every voxel whose
// distance is <= cap still gets its exact distance; cap = MGC_HINF is the exact BFS.
__device__ __forceinline__ void relabel_visit(const Lattice& L, const Tiles& TL, const uint8_t* __restrict__ rmask,
                                              int* __restrict__ height, int* __restrict__ rflag, const WorkList& next,
                                              int t, int* sh, int cap)
{
    const TileCtx c = tile_ctx(L, TL, t);
    if (threadIdx.x == 0) rflag[t] = 0;        // may be listed again by a neighbour from now on
    const int h0 = load_heights(L, c, height, sh);
    const unsigned m = c.own ? (rmask[c.v] & 0x3fu) : 0u;
    __syncthreads();
    const int me = hidx(c.lz + 1, c.ly + 1, c.lx + 1);
    int h = h0;
    for (;;) {
        int changed = 0;
        if (m && h > 1) {
            int best = h;
            if (m & 1u)  { const int hw = sh[me + hoff<0>()] + 1; best = hw < best ? hw : best; }
            if (m & 2u)  { const int hw = sh[me + hoff<1>()] + 1; best = hw < best ? hw : best; }
            if (m & 4u)  { const int hw = sh[me + hoff<2>()] + 1; best = hw < best ? hw : best; }
            if (m & 8u)  { const int hw = sh[me + hoff<3>()] + 1; best = hw < best ? hw : best; }
            if (m & 16u) { const int hw = sh[me + hoff<4>()] + 1; best = hw < best ? hw : best; }
            if (m & 32u) { const int hw = sh[me + hoff<5>()] + 1; best = hw < best ? hw : best; }
            if (best < h && best <= cap) { h = best; sh[me] = h; changed = 1; }
        }
        if (!__syncthreads_or(changed)) break;
    }
    if (h != h0) {
        height[c.v] = h;
        // wake a face neighbour only if my new label can actually lower the voxel across the face: its label (from the
        // halo, and labels only ever decrease during a BFS) must exceed mine + 1.  Without this test every tile was
        // re-listed by each neighbour that settled after it -- most visits of a hard instance changed nothing.
        // A label at the cap wakes nobody: it could only lower a neighbour above the cap.
        if (h < cap) {
            if (c.lz == 0 && c.tz > 0 && sh[me + hoff<0>()] > h + 1) list_push(rflag, next, tile_nbr(TL, t, 0));
            if (c.lz == TILE - 1 && c.tz + 1 < TL.nt[0] && sh[me + hoff<1>()] > h + 1) list_push(rflag, next, tile_nbr(TL, t, 1));
            if (c.ly == 0 && c.ty > 0 && sh[me + hoff<2>()] > h + 1) list_push(rflag, next, tile_nbr(TL, t, 2));
            if (c.ly == TILE - 1 && c.ty + 1 < TL.nt[1] && sh[me + hoff<3>()] > h + 1) list_push(rflag, next, tile_nbr(TL, t, 3));
            if (c.lx == 0 && c.tx > 0 && sh[me + hoff<4>()] > h + 1) list_push(rflag, next, tile_nbr(TL, t, 4));
            if (c.lx == TILE - 1 && c.tx + 1 < TL.nt[2] && sh[me + hoff<5>()] > h + 1) list_push(rflag, next, tile_nbr(TL, t, 5));
        }
    }
    if (TL.dflag) {                          // labels of this tile changed: it has to be reset before the next BFS
        const int chg = __syncthreads_or(h != h0 ? 1 : 0);
        if (chg && threadIdx.x == 0) mark_dirty(TL, t);
    }
}

// ---------------------------------------------------------------------------------------------------
// push / relabel discharge of the tiles of one colour (persistent CTAs over that colour's worklist)
// ---------------------------------------------------------------------------------------------------
// One direction of the push phase.  K is a compile-time direction so everything stays in registers.
template <int K, typename T>
__device__ __forceinline__ void push_dir(const Lattice& L, const Tiles& TL, const State<T>& S, const TileCtx& c,
                                         const int* s_h, T* s_out, int me, int h, T& e, T& ck, int& minh,
                                         int* __restrict__ pflag, const WorkList& other_next, unsigned& nbr_listed,
                                         unsigned& dirty)
{
    T d = 0;
    if (ck > 0) {
        const int hw = s_h[me + hoff<K>()];
        if (hw < h && e > 0) {
            d = e < ck ? e : ck;
            ck -= d;
            e -= d;
            dirty |= (1u << K) | 64u;
        }
        if (ck > 0) minh = hw < minh ? hw : minh;
    }
    constexpr int AX = K >> 1;
    const int lc = (AX == 0 ? c.lz : (AX == 1 ? c.ly : c.lx)) + ((K & 1) ? 1 : -1);
    const bool inside = lc >= 0 && lc < TILE;
    if (inside) {
        s_out[K * TILE_VOX + threadIdx.x] = d;         // pulled by the neighbour's own thread
    } else if (d > 0) {
        // the neighbour tile has the other colour and is idle: update its voxel in HBM
        const unsigned w = (unsigned)((int)c.v + dir_offset(L, K));
        atomicAdd(&S.cap[K ^ 1][w], d);
        atomicAdd(&S.excess[w], d);
        // its residual mask gains the reverse arc (byte-wise OR through the containing 32-bit word)
        atomicOr(reinterpret_cast<unsigned*>(S.rmask) + (w >> 2), (1u << (K ^ 1)) << (8u * (w & 3u)));
        if (!(nbr_listed & (1u << K))) { nbr_listed |= 1u << K; list_push(pflag, other_next, tile_nbr(TL, c.t, K)); }
    }
}

template <int K, typename T>
__device__ __forceinline__ void pull_dir(const TileCtx& c, const T* s_out, T& e, T& ck, unsigned& dirty)
{
    constexpr int AX = K >> 1;
    constexpr int SG = (K & 1) ? 1 : -1;
    const int lc = (AX == 0 ? c.lz : (AX == 1 ? c.ly : c.lx)) + SG;
    if (lc >= 0 && lc < TILE) {
        constexpr int ST = AX == 0 ? 64 : (AX == 1 ? 8 : 1);
        // what my neighbour in direction K pushed towards me travelled along ITS direction K^1
        const T d = s_out[(K ^ 1) * TILE_VOX + (int)threadIdx.x + SG * ST];
        if (d > 0) {
            e += d;
            ck += d;   // my arc towards that neighbour is the reverse arc: it gains residual capacity
            dirty |= (1u << K) | 64u;
        }
    }
}

// one push/relabel discharge visit of tile t.  s_out = 6*TILE_VOX values, s_h = HALO_VOX ints of shared memory.
// `stg` (optional): the tile's six capacity planes + excess already staged in shared memory by TMA (gc_tma.cuh),
// plane p at stg + p * TILE_VOX, voxel order == thread order; nullptr = load from global memory here.
// `labels_capped`: the last global relabel stopped at a label cap, so a voxel at HINF may still reach the sink; a tile
// that keeps excess at such a voxel stays listed for the next (exact) relabel instead of leaving the lists.
template <typename T>
__device__ __forceinline__ void push_visit_staged(const Lattice& L, const Tiles& TL, const State<T>& S, int iters,
                                                  int* __restrict__ pflag, const WorkList& self_next, const WorkList& other_next,
                                                  int t, T* s_out, int* s_h, const double* stg, bool labels_capped = false)
{
    const TileCtx c = tile_ctx(L, TL, t);
    const int tid = threadIdx.x;
    const int me = hidx(c.lz + 1, c.ly + 1, c.lx + 1);
    if (tid == 0) pflag[t] = 0;
    const int h0 = load_heights(L, c, S.height, s_h);
    T e = 0, scap = 0, sf = 0, c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0;
    unsigned sinkv = 0;                     // RM_SINKV of this voxel (sink[v] holds a value)
    if (c.inb) {
        if (stg) {
            c0 = (T)stg[0 * TILE_VOX + tid]; c1 = (T)stg[1 * TILE_VOX + tid]; c2 = (T)stg[2 * TILE_VOX + tid];
            c3 = (T)stg[3 * TILE_VOX + tid]; c4 = (T)stg[4 * TILE_VOX + tid]; c5 = (T)stg[5 * TILE_VOX + tid];
            e = (T)stg[6 * TILE_VOX + tid];
        } else {
            e = S.excess[c.v];
            c0 = S.cap[0][c.v]; c1 = S.cap[1][c.v]; c2 = S.cap[2][c.v];
            c3 = S.cap[3][c.v]; c4 = S.cap[4][c.v]; c5 = S.cap[5][c.v];
        }
        const T tr = S.tr[c.v];
        if (tr < 0) {
            scap = -tr;
            sinkv = S.rmask[c.v] & RM_SINKV;
            if (sinkv) sf = S.sink[c.v];
        }
    }
    int h = h0;
    unsigned nbr_listed = 0, dirty = 0;     // dirty: bit k = cap k changed, 64 = excess, 128 = sink flow
    __syncthreads();

    for (int it = 0; it < iters; ++it) {
        // ---- push phase: decisions from the label snapshot, own registers updated, outflow published ----
        const int act = (c.own && e > 0 && h < MGC_HINF) ? 1 : 0;
        int newh = h;
        if (act) {
            if (scap > 0) {                      // the sink sits at height 0: always admissible
                const T rr = scap - sf;
                if (rr > 0) {
                    if (e < rr) { sf += e; e = 0; } else { e -= rr; sf = scap; }   // saturation is exact
                    dirty |= 64u | 128u;
                }
            }
            int minh = MGC_HINF;
            push_dir<0>(L, TL, S, c, s_h, s_out, me, h, e, c0, minh, pflag, other_next, nbr_listed, dirty);
            push_dir<1>(L, TL, S, c, s_h, s_out, me, h, e, c1, minh, pflag, other_next, nbr_listed, dirty);
            push_dir<2>(L, TL, S, c, s_h, s_out, me, h, e, c2, minh, pflag, other_next, nbr_listed, dirty);
            push_dir<3>(L, TL, S, c, s_h, s_out, me, h, e, c3, minh, pflag, other_next, nbr_listed, dirty);
            push_dir<4>(L, TL, S, c, s_h, s_out, me, h, e, c4, minh, pflag, other_next, nbr_listed, dirty);
            push_dir<5>(L, TL, S, c, s_h, s_out, me, h, e, c5, minh, pflag, other_next, nbr_listed, dirty);
            // excess left => no admissible arc left => relabel above the lowest residual neighbour
            if (e > 0) newh = (minh >= MGC_HINF) ? MGC_HINF : minh + 1;
        } else {
            s_out[0 * TILE_VOX + tid] = 0; s_out[1 * TILE_VOX + tid] = 0; s_out[2 * TILE_VOX + tid] = 0;
            s_out[3 * TILE_VOX + tid] = 0; s_out[4 * TILE_VOX + tid] = 0; s_out[5 * TILE_VOX + tid] = 0;
        }
        if (!__syncthreads_or(act)) break;       // nothing is active in this tile any more: done
        // ---- pull phase: every voxel collects what its in-tile neighbours sent; labels are published ----
        pull_dir<0>(c, s_out, e, c0, dirty); pull_dir<1>(c, s_out, e, c1, dirty); pull_dir<2>(c, s_out, e, c2, dirty);
        pull_dir<3>(c, s_out, e, c3, dirty); pull_dir<4>(c, s_out, e, c4, dirty); pull_dir<5>(c, s_out, e, c5, dirty);
        if (newh != h) { h = newh; s_h[me] = h; }
        __syncthreads();
    }

    // ---- write back what changed (this CTA is the only writer of its own voxels during this launch) ----
    if (c.inb && (dirty || h != h0)) {
        if (dirty & 64u) S.excess[c.v] = e;
        if (dirty & 1u) S.cap[0][c.v] = c0;
        if (dirty & 2u) S.cap[1][c.v] = c1;
        if (dirty & 4u) S.cap[2][c.v] = c2;
        if (dirty & 8u) S.cap[3][c.v] = c3;
        if (dirty & 16u) S.cap[4][c.v] = c4;
        if (dirty & 32u) S.cap[5][c.v] = c5;
        if (h != h0) S.height[c.v] = h;
        if (dirty & 128u) { S.sink[c.v] = sf; sinkv = RM_SINKV; }
        unsigned m = (c0 > 0 ? 1u : 0u) | (c1 > 0 ? 2u : 0u) | (c2 > 0 ? 4u : 0u) | (c3 > 0 ? 8u : 0u) |
                     (c4 > 0 ? 16u : 0u) | (c5 > 0 ? 32u : 0u) | ((scap - sf > 0) ? RM_SINK : 0u) | sinkv;
        S.rmask[c.v] = (uint8_t)m;
    }
    const int still = (c.own && e > 0 && (h < MGC_HINF || labels_capped)) ? 1 : 0;
    if (__syncthreads_or(still) && tid == 0) list_push(pflag, self_next, t);
    if (TL.dflag) {                          // a label or a sink-link residual bit of this tile changed
        const int chg = __syncthreads_or((c.inb && (h != h0 || (dirty & 128u))) ? 1 : 0);
        if (chg && tid == 0) mark_dirty(TL, t);
    }
}

template <typename T>
__global__ void __launch_bounds__(TILE_VOX, 2) k_push_tile(Lattice L, Tiles TL, State<T> S, int iters,
                                                           int* __restrict__ pflag, WorkList cur, int* __restrict__ cursor,
                                                           WorkList self_next, WorkList other_next, int labels_capped)
{
    __shared__ T s_out[6 * TILE_VOX];
    __shared__ int s_h[HALO_VOX];
    __shared__ int s_slot;
    for (;;) {
        const int t = fetch_tile(cur, cursor, &s_slot);
        if (t < 0) break;
        push_visit_staged<T>(L, TL, S, iters, pflag, self_next, other_next, t, s_out, s_h, nullptr, labels_capped != 0);
    }
}
