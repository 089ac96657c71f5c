// gc_tiles4.cuh -- tile-resident solver kernels for 4-D lattices (8-connected: the reference treats an n-D input as
// an n-D lattice, energy_voxel.py:637; BASELINE config 4 is 256x256x128x4 with the channel axis linked too).
//
// Same design as the 3-D kernels of gc_tiles.cuh -- a 512-thread CTA owns one tile for a visit, labels with a
// 1-voxel halo in shared memory, capacities/excess/sink state in the owning thread's registers, push-then-pull
// rounds through a shared outflow buffer, two-colour (4-D checkerboard) passes, worklists + persistent CTAs --
// with a 4 x 4 x 8 x 4 tile (axis 3 fastest: a tile row pair is 8 x 4 = 32 contiguous voxels = 256 B of float64).
// The residual mask needs 8 arc bits, so the "sink link residual" bit lives in a second byte array (smask).
#pragma once
#include "gc_tiles.cuh"

#define T4_VOX 512
#define H4_VOX 2160            // 6 * 6 * 10 * 6
#define H4_FACE_VOX 896        // 2*(4*8*4) + 2*(4*8*4) + 2*(4*4*4) + 2*(4*4*8)

struct Tiles4 {
    int nt[4];
    int ntiles;
};

__device__ __forceinline__ constexpr int t4_ext(int axis) { return axis == 2 ? 8 : 4; }
__device__ __forceinline__ constexpr int t4_toff(int axis) { return axis == 0 ? 128 : (axis == 1 ? 32 : (axis == 2 ? 4 : 1)); }
__device__ __forceinline__ constexpr int t4_hoff(int axis) { return axis == 0 ? 360 : (axis == 1 ? 60 : (axis == 2 ? 6 : 1)); }
__device__ __forceinline__ int h4idx(int a, int b, int c, int d) { return ((a * 6 + b) * 10 + c) * 6 + d; }

struct Tile4Ctx {
    int t;
    int tc[4];          // tile coordinates
    int l[4];           // local coordinates
    bool inb, own;
    unsigned v;
};

__device__ __forceinline__ Tile4Ctx tile4_ctx(const Lattice& L, const Tiles4& TL, int t)
{
    Tile4Ctx c;
    c.t = t;
    int r = t;
    c.tc[3] = r % TL.nt[3]; r /= TL.nt[3];
    c.tc[2] = r % TL.nt[2]; r /= TL.nt[2];
    c.tc[1] = r % TL.nt[1]; c.tc[0] = r / TL.nt[1];
    const int tid = threadIdx.x;
    c.l[3] = tid & 3; c.l[2] = (tid >> 2) & 7; c.l[1] = (tid >> 5) & 3; c.l[0] = tid >> 7;
    c.inb = true;
    unsigned v = 0;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int g = c.tc[a] * t4_ext(a) + c.l[a];
        c.inb = c.inb && g < L.dim[a];
        v += (unsigned)g * L.stride[a];
    }
    const int g0 = c.tc[0] * 4 + c.l[0];
    c.v = c.inb ? v : 0u;
    c.own = c.inb && g0 >= L.own0 && g0 < L.own1;
    return c;
}

__device__ __forceinline__ int tile4_color(const Tile4Ctx& c) { return (c.tc[0] + c.tc[1] + c.tc[2] + c.tc[3]) & 1; }

__device__ __forceinline__ int tile4_nbr(const Tiles4& TL, int t, int k)
{
    const int ax = k >> 1;
    const int s = ax == 0 ? TL.nt[1] * TL.nt[2] * TL.nt[3] : (ax == 1 ? TL.nt[2] * TL.nt[3] : (ax == 2 ? TL.nt[3] : 1));
    return (k & 1) ? t + s : t - s;
}

// labels of the tile (own voxel) and of its eight halo faces into the 6x6x10x6 array; out-of-lattice -> HINF
__device__ __forceinline__ int load_heights4(const Lattice& L, const Tile4Ctx& c, const int* __restrict__ height, int* sh)
{
    const int h0 = c.inb ? __ldcg(height + c.v) : MGC_HINF;
    sh[h4idx(c.l[0] + 1, c.l[1] + 1, c.l[2] + 1, c.l[3] + 1)] = h0;
    for (int i = threadIdx.x; i < H4_FACE_VOX; i += T4_VOX) {
        // faces in order: axis0 -,+ (128 each), axis1 -,+ (128), axis2 -,+ (64), axis3 -,+ (128)
        int f, j;
        if (i < 256) { f = i >> 7; j = i & 127; }
        else if (i < 512) { f = 2 + ((i - 256) >> 7); j = (i - 256) & 127; }
        else if (i < 640) { f = 4 + ((i - 512) >> 6); j = (i - 512) & 63; }
        else { f = 6 + ((i - 640) >> 7); j = (i - 640) & 127; }
        const int ax = f >> 1, hi = f & 1;
        int lc[4];
        // j enumerates the three other axes, fastest last
        if (ax == 0) { lc[3] = j & 3; lc[2] = (j >> 2) & 7; lc[1] = j >> 5; }
        else if (ax == 1) { lc[3] = j & 3; lc[2] = (j >> 2) & 7; lc[0] = j >> 5; }
        else if (ax == 2) { lc[3] = j & 3; lc[1] = (j >> 2) & 3; lc[0] = j >> 4; }
        else { lc[2] = j & 7; lc[1] = (j >> 3) & 3; lc[0] = j >> 5; }
        lc[ax] = hi ? t4_ext(ax) : -1;
        bool in = true;
        unsigned v = 0;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int g = c.tc[a] * t4_ext(a) + lc[a];
            in = in && g >= 0 && g < L.dim[a];
            v += (unsigned)g * L.stride[a];
        }
        sh[h4idx(lc[0] + 1, lc[1] + 1, lc[2] + 1, lc[3] + 1)] = in ? __ldcg(height + v) : MGC_HINF;
    }
    return h0;
}

// ---------------------------------------------------------------------------------------------------
// init (cf. k_init_tile; WARM: tr > 0 becomes tr - excess, BK's residual source capacity)
// ---------------------------------------------------------------------------------------------------
template <typename T, bool WARM = false>
__global__ void __launch_bounds__(T4_VOX) k_init_tile4(Lattice L, Tiles4 TL, State<T> S, uint8_t* __restrict__ smask,
                                                       int* __restrict__ rflag, WorkList rl, int* __restrict__ pflag,
                                                       WorkList pl0, WorkList pl1)
{
    const Tile4Ctx c = tile4_ctx(L, TL, blockIdx.x);
    int needs = 0, hasexc = 0;
    if (c.inb) {
        const double tr = (double)S.tr[c.v];
        unsigned m = 0;
        double out = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const double ck = (double)S.cap[k][c.v];
            if (ck > 0) m |= 1u << k;
            out = __dadd_ru(out, ck);
        }
        double e = 0.0;
        if (tr > 0) { const double lim = out * SOURCE_CLAMP_SLACK; e = tr < lim ? tr : lim; if (!(out == out)) e = tr; }
        if (!c.own) e = 0.0;
        if (WARM && tr > 0) S.tr[c.v] = (T)(tr - e);
        S.excess[c.v] = (T)e;
        S.sink[c.v] = (T)0;
        S.rmask[c.v] = (uint8_t)m;
        smask[c.v] = tr < 0 ? 1 : 0;
        const int h = (c.own && tr < 0) ? 1 : MGC_HINF;
        S.height[c.v] = h;
        needs = (c.own && m != 0 && h == MGC_HINF) ? 1 : 0;
        hasexc = e > 0 ? 1 : 0;
    }
    const int any_needs = __syncthreads_or(needs);
    const int any_exc = __syncthreads_or(hasexc);
    if (threadIdx.x == 0) {
        rflag[c.t] = any_needs;
        if (any_needs) rl.items[atomicAdd(rl.count, 1)] = c.t;
        pflag[c.t] = any_exc;
        if (any_exc) {
            const WorkList& pl = tile4_color(c) ? pl1 : pl0;
            pl.items[atomicAdd(pl.count, 1)] = c.t;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// global relabel: one tile visit (k_bfs_coop4 of gc_persist.cuh runs the passes over the worklists)
// ---------------------------------------------------------------------------------------------------
// one tile visit of the 4-D global relabel (cf. relabel_visit): relax inside the tile until nothing changes, write back,
// list the face neighbours whose halo changed.  `sh` = H4_VOX ints of shared memory.
__device__ __forceinline__ void relabel_visit4(const Lattice& L, const Tiles4& TL, const uint8_t* __restrict__ rmask,
                                               int* __restrict__ height, int* __restrict__ rflag, const WorkList& next, int t, int* sh)
{
    const Tile4Ctx c = tile4_ctx(L, TL, t);
    if (threadIdx.x == 0) rflag[t] = 0;
    const int h0 = load_heights4(L, c, height, sh);
    const unsigned m = c.own ? rmask[c.v] : 0u;
    __syncthreads();
    const int me = h4idx(c.l[0] + 1, c.l[1] + 1, c.l[2] + 1, c.l[3] + 1);
    int h = h0;
    for (;;) {
        int changed = 0;
        if (m && h > 1) {
            int best = h;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (m & (1u << k)) {
                    const int hw = sh[me + ((k & 1) ? t4_hoff(k >> 1) : -t4_hoff(k >> 1))] + 1;
                    best = hw < best ? hw : best;
                }
            }
            if (best < h) { h = best; sh[me] = h; changed = 1; }
        }
        if (!__syncthreads_or(changed)) break;
    }
    if (h != h0) {
        height[c.v] = h;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ax = k >> 1;
            const bool edge = (k & 1) ? (c.l[ax] == t4_ext(ax) - 1 && c.tc[ax] + 1 < TL.nt[ax]) : (c.l[ax] == 0 && c.tc[ax] > 0);
            // only if my new label can lower the voxel across the face (see relabel_visit)
            if (edge && sh[me + ((k & 1) ? t4_hoff(ax) : -t4_hoff(ax))] > h + 1) list_push(rflag, next, tile4_nbr(TL, t, k));
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// push / relabel discharge (cf. k_push_tile): cc[] is indexed only by unrolled constants -> registers
// ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(T4_VOX, 2) k_push_tile4(Lattice L, Tiles4 TL, State<T> S, uint8_t* __restrict__ smask, int iters,
                                                          int* __restrict__ pflag, WorkList cur, int* __restrict__ cursor,
                                                          WorkList self_next, WorkList other_next)
{
    __shared__ T s_out[8 * T4_VOX];
    __shared__ int s_h[H4_VOX];
    __shared__ int s_slot;
    for (;;) {
        const int t = fetch_tile(cur, cursor, &s_slot);
        if (t < 0) break;
        const Tile4Ctx c = tile4_ctx(L, TL, t);
        const int tid = threadIdx.x;
        const int me = h4idx(c.l[0] + 1, c.l[1] + 1, c.l[2] + 1, c.l[3] + 1);
        if (tid == 0) pflag[t] = 0;
        const int h0 = load_heights4(L, c, S.height, s_h);
        T e = 0, scap = 0, sf = 0;
        T cc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) cc[k] = c.inb ? S.cap[k][c.v] : (T)0;
        if (c.inb) {
            e = S.excess[c.v];
            const T tr = S.tr[c.v];
            if (tr < 0) { scap = -tr; sf = S.sink[c.v]; }
        }
        int h = h0;
        unsigned nbr_listed = 0, dirty = 0;   // dirty: bit k = cap k, 256 = excess, 512 = sink flow
        __syncthreads();

        for (int it = 0; it < iters; ++it) {
            const int act = (c.own && e > 0 && h < MGC_HINF) ? 1 : 0;
            int newh = h;
            if (act) {
                if (scap > 0) {
                    const T rr = scap - sf;
                    if (rr > 0) {
                        if (e < rr) { sf += e; e = 0; } else { e -= rr; sf = scap; }
                        dirty |= 256u | 512u;
                    }
                }
                int minh = MGC_HINF;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int ax = k >> 1, sg = (k & 1) ? 1 : -1;
                    T d = 0;
                    if (cc[k] > 0) {
                        const int hw = s_h[me + sg * t4_hoff(ax)];
                        if (hw < h && e > 0) {
                            d = e < cc[k] ? e : cc[k];
                            cc[k] -= d;
                            e -= d;
                            dirty |= (1u << k) | 256u;
                        }
                        if (cc[k] > 0) minh = hw < minh ? hw : minh;
                    }
                    const int lc = c.l[ax] + sg;
                    if (lc >= 0 && lc < t4_ext(ax)) {
                        s_out[k * T4_VOX + tid] = d;
                    } else if (d > 0) {
                        const unsigned w = (unsigned)((int)c.v + dir_offset(L, k));
                        atomicAdd(&S.cap[k ^ 1][w], d);
                        atomicAdd(&S.excess[w], d);
                        atomicOr(reinterpret_cast<unsigned*>(S.rmask) + (w >> 2), (1u << (k ^ 1)) << (8u * (w & 3u)));
                        if (!(nbr_listed & (1u << k))) { nbr_listed |= 1u << k; list_push(pflag, other_next, tile4_nbr(TL, t, k)); }
                    }
                }
                if (e > 0) newh = (minh >= MGC_HINF) ? MGC_HINF : minh + 1;
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) s_out[k * T4_VOX + tid] = 0;
            }
            if (!__syncthreads_or(act)) break;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int ax = k >> 1, sg = (k & 1) ? 1 : -1;
                const int lc = c.l[ax] + sg;
                if (lc >= 0 && lc < t4_ext(ax)) {
                    const T d = s_out[(k ^ 1) * T4_VOX + tid + sg * t4_toff(ax)];
                    if (d > 0) { e += d; cc[k] += d; dirty |= (1u << k) | 256u; }
                }
            }
            if (newh != h) { h = newh; s_h[me] = h; }
            __syncthreads();
        }

        if (c.inb && (dirty || h != h0)) {
            if (dirty & 256u) S.excess[c.v] = e;
            unsigned m = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (dirty & (1u << k)) S.cap[k][c.v] = cc[k];
                if (cc[k] > 0) m |= 1u << k;
            }
            if (h != h0) S.height[c.v] = h;
            if (dirty & 512u) S.sink[c.v] = sf;
            S.rmask[c.v] = (uint8_t)m;
            smask[c.v] = (scap - sf > 0) ? 1 : 0;
        }
        const int still = (c.own && e > 0 && h < MGC_HINF) ? 1 : 0;
        if (__syncthreads_or(still) && tid == 0) list_push(pflag, self_next, t);
    }
}

template <typename T>
__global__ void __launch_bounds__(T4_VOX) k_count_active_tiles4(Lattice L, Tiles4 TL, State<T> S, WorkList wl,
                                                                unsigned long long* __restrict__ count)
{
    const int n = *(volatile int*)wl.count;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const Tile4Ctx c = tile4_ctx(L, TL, wl.items[i]);
        const bool act = c.own && (S.excess[c.v] > 0) && (S.height[c.v] < MGC_HINF);
        const unsigned b = __ballot_sync(0xffffffffu, act);
        if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, (unsigned long long)__popc(b));
    }
}
