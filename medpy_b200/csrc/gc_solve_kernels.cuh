// gc_solve_kernels.cuh -- kernels launched only by gc_solve.cu, split from the headers whose device functions the other
// units of the lattice C ABI share (a kernel that is not a template is compiled into every unit that includes its
// header): the relabel resets of gc_tiles.cuh / gc_tiles4.cuh, and the materialiser, label window and stop test of
// gc_build.cuh, which read a lazy build's implicit push state.
#pragma once
#include "gc_build.cuh"
#include "gc_tiles4.cuh"

// later global relabels: labels from the (incrementally maintained) residual mask; 1 B read + 4 B written per voxel.
// One thread per 8-voxel x-run of a tile row, consecutive threads on consecutive runs (coalesced); rflag must be
// zero on entry (the host memsets it): a run that holds an unlabelled voxel with residual out-arcs lists its tile.
__global__ void __launch_bounds__(256) k_relabel_reset(Lattice L, Tiles TL, const uint8_t* __restrict__ rmask,
                                                       int* __restrict__ height, int* __restrict__ rflag, WorkList rl)
{
    const unsigned ntx = (unsigned)TL.nt[2];
    const unsigned nruns = (unsigned)L.dim[0] * (unsigned)L.dim[1] * ntx;
    for (unsigned r = blockIdx.x * blockDim.x + threadIdx.x; r < nruns; r += gridDim.x * blockDim.x) {
        const unsigned tx = r % ntx, zy = r / ntx;
        const unsigned gy = zy % (unsigned)L.dim[1], gz = zy / (unsigned)L.dim[1];
        const unsigned x0 = tx * TILE;
        const int nx = (int)min((unsigned)TILE, (unsigned)L.dim[2] - x0);
        const unsigned base = gz * L.stride[0] + gy * L.stride[1] + x0;
        const bool own = (int)gz >= L.own0 && (int)gz < L.own1;
        int needs = 0;
        if (nx == TILE && (base & 7u) == 0u) {
            const uint2 m8 = *reinterpret_cast<const uint2*>(rmask + base);
            int h[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const unsigned m = ((i < 4 ? m8.x : m8.y) >> (8 * (i & 3))) & 0xffu;
                h[i] = (own && (m & RM_SINK)) ? 1 : MGC_HINF;
                needs |= (own && (m & 0x3fu) != 0 && h[i] == MGC_HINF) ? 1 : 0;
            }
            int4* dst = reinterpret_cast<int4*>(height + base);
            dst[0] = make_int4(h[0], h[1], h[2], h[3]);
            dst[1] = make_int4(h[4], h[5], h[6], h[7]);
        } else {
            for (int i = 0; i < nx; ++i) {
                const unsigned m = rmask[base + i];
                const int h = (own && (m & RM_SINK)) ? 1 : MGC_HINF;
                height[base + i] = h;
                needs |= (own && (m & 0x3fu) != 0 && h == MGC_HINF) ? 1 : 0;
            }
        }
        if (needs) list_push(rflag, rl, (int)(((gz >> 3) * (unsigned)TL.nt[1] + (gy >> 3)) * ntx + tx));
    }
}

// the same reset restricted to the DIRTY tiles (Tiles::ditems): every other tile is still in the reset state, so an easy
// instance (regional term: the BFS only ever labels the few tiles around the objects) pays for those tiles instead of a
// 5 B/voxel pass over the lattice.  Persistent CTAs of one
// tile each; clears the dirty flags it consumes (the host zeroes the count afterwards).
__global__ void __launch_bounds__(TILE_VOX) k_relabel_reset_list(Lattice L, Tiles TL, const uint8_t* __restrict__ rmask,
                                                                 int* __restrict__ height, int* __restrict__ rflag, WorkList rl)
{
    const int n = *(volatile int*)TL.dcount;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int t = TL.ditems[i];
        const TileCtx c = tile_ctx(L, TL, t);
        int needs = 0;
        if (c.inb) {
            const unsigned m = rmask[c.v];
            const int h = (c.own && (m & RM_SINK)) ? 1 : MGC_HINF;
            height[c.v] = h;
            needs = (c.own && (m & 0x3fu) != 0 && h == MGC_HINF) ? 1 : 0;
        }
        const int any = __syncthreads_or(needs);
        if (threadIdx.x == 0) {
            TL.dflag[t] = 0;
            if (any) list_push(rflag, rl, t);
        }
    }
}

// labels from the residual masks; one CTA per tile
__global__ void __launch_bounds__(T4_VOX) k_relabel_reset4(Lattice L, Tiles4 TL, const uint8_t* __restrict__ rmask,
                                                           const uint8_t* __restrict__ smask, int* __restrict__ height,
                                                           int* __restrict__ rflag, WorkList rl)
{
    const Tile4Ctx c = tile4_ctx(L, TL, blockIdx.x);
    int needs = 0;
    if (c.inb) {
        const unsigned m = rmask[c.v];
        const int h = (c.own && smask[c.v]) ? 1 : MGC_HINF;
        height[c.v] = h;
        needs = (c.own && m != 0 && h == MGC_HINF) ? 1 : 0;
    }
    const int any_needs = __syncthreads_or(needs);
    if (threadIdx.x == 0) {
        rflag[c.t] = any_needs;
        if (any_needs) rl.items[atomicAdd(rl.count, 1)] = c.t;
    }
}

// ---------------------------------------------------------------------------------------------------
// Push-state materialiser of the lazy build: the six capacity planes, tr and excess of the tiles the push path is about
// to touch, from the graph-owned copies the build wrote.  Runs over a push worklist -- every listed tile and its six face
// neighbours, since a push writes across faces -- or, with wl.items == nullptr, over every tile.  A tile is materialised
// once per build.  Two launches:
//   k_caps_claim : claims each candidate tile (cmat[t]: 0 -> 1) and appends the claimed ones to a compact list;
//   k_caps_tiles : persistent CTAs take the listed tiles one by one through an atomic cursor (even load, whatever the
//                  list order), staging the image of the next tile in registers while the current one is computed.
// The values are the doubles the eager build writes: build_weight / exp_caps6 on the same operands, tlink_replay on the
// same inputs, source_excess on the capacities just computed.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_caps_claim(Tiles TL, int* __restrict__ cmat, WorkList wl, int* __restrict__ list,
                                                    int* __restrict__ count)
{
    const bool all = wl.items == nullptr;
    const int n = all ? TL.ntiles : *wl.count * 7;
    const int lane = threadIdx.x & 31;
    for (int base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31; base < n; base += gridDim.x * blockDim.x) {
        const int i = base + lane;
        int t = -1;
        if (i < n) {
            t = all ? i : wl.items[i / 7];
            const int k = all ? -1 : i % 7 - 1;          // -1: the listed tile, 0..5: its neighbour across face k
            if (k >= 0) {
                const int tx = t % TL.nt[2], r = t / TL.nt[2], ty = r % TL.nt[1], tz = r / TL.nt[1];
                const int ck = (k >> 1) == 0 ? tz : ((k >> 1) == 1 ? ty : tx);
                t = ((k & 1) ? ck + 1 < TL.nt[k >> 1] : ck > 0) ? tile_nbr(TL, t, k) : -1;
            }
        }
        const bool claim = t >= 0 && cmat[t] == 0 && atomicExch(&cmat[t], 1) == 0;
        const unsigned b = __ballot_sync(0xffffffffu, claim);
        int slot = 0;
        if (lane == 0 && b) slot = atomicAdd(count, __popc(b));
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (claim) list[slot + __popc(b & ((1u << lane) - 1u))] = t;
    }
}

template <typename E, int FN, int USE_MAX, int SPACING>
__global__ void __launch_bounds__(TILE_VOX, 2)
k_caps_tiles(Lattice L, Tiles TL, State<double> S, const E* __restrict__ img, BoundaryParams P, LazyTin tin,
             const int* __restrict__ list, const int* __restrict__ count, int* __restrict__ cursor, int* __restrict__ n_done)
{
    __shared__ E s_img[HALO_VOX];
    __shared__ int s_slot[2];
    const int tid = threadIdx.x;
    const int n = *count;
    if (blockIdx.x == 0 && tid == 0 && n) atomicAdd(n_done, n);
    const bool use_max = USE_MAX >= 0 ? (USE_MAX != 0) : (P.use_max != 0);
    const bool spacing = SPACING >= 0 ? (SPACING != 0) : (P.inv_spacing_on != 0.0);
    // this thread's image cells of tile t: its voxel and (tid < 384) one cell of the six face halos (edges and corners
    // are never read; out-of-lattice cells are never used)
    struct Cells { E own, halo; };
    auto load = [&](int t) -> Cells {
        Cells r{(E)0, (E)0};
        const TileCtx c = tile_ctx(L, TL, t);
        if (c.inb) r.own = img[c.v];
        if (tid < 384) {
            const int face = tid >> 6, fa = (tid >> 3) & 7, fb = tid & 7;
            int z, y, x;
            switch (face) {
                case 0: z = -1; y = fa; x = fb; break;
                case 1: z = TILE; y = fa; x = fb; break;
                case 2: z = fa; y = -1; x = fb; break;
                case 3: z = fa; y = TILE; x = fb; break;
                case 4: z = fa; y = fb; x = -1; break;
                default: z = fa; y = fb; x = TILE; break;
            }
            const int gz = c.tz * TILE + z, gy = c.ty * TILE + y, gx = c.tx * TILE + x;
            if (gz >= 0 && gy >= 0 && gx >= 0 && gz < L.dim[0] && gy < L.dim[1] && gx < L.dim[2])
                r.halo = img[(unsigned)gz * L.stride[0] + (unsigned)gy * L.stride[1] + (unsigned)gx];
        }
        return r;
    };
    auto halo_at = [&]() -> int {
        const int face = tid >> 6, fa = (tid >> 3) & 7, fb = tid & 7;
        switch (face) {
            case 0: return hidx(0, fa + 1, fb + 1);
            case 1: return hidx(TILE + 1, fa + 1, fb + 1);
            case 2: return hidx(fa + 1, 0, fb + 1);
            case 3: return hidx(fa + 1, TILE + 1, fb + 1);
            case 4: return hidx(fa + 1, fb + 1, 0);
            default: return hidx(fa + 1, fb + 1, TILE + 1);
        }
    };
    if (tid == 0) s_slot[0] = atomicAdd(cursor, 1);
    __syncthreads();
    int i = s_slot[0];
    Cells cur{(E)0, (E)0};
    if (i < n) cur = load(list[i]);
    for (int it = 1; i < n; ++it) {
        const int t = list[i];
        const TileCtx c = tile_ctx(L, TL, t);
        const int h = hidx(c.lz + 1, c.ly + 1, c.lx + 1);
        s_img[h] = cur.own;
        if (tid < 384) s_img[halo_at()] = cur.halo;
        if (tid == 0) s_slot[it & 1] = atomicAdd(cursor, 1);
        __syncthreads();
        // t-link inputs of this voxel, and the next tile's image: in flight while this tile is computed
        double p = 0.0;
        unsigned fb = 0u;
        if (c.inb) lazy_tin_load(L, tin, c, p, fb);
        const int inext = s_slot[it & 1];
        Cells nxt{(E)0, (E)0};
        if (inext < n) nxt = load(list[inext]);
        const unsigned valid = c.inb ? tile_pairs(L, c) : 0u;
        const BoundaryParams Pv = params_at(P, L, c.tz * TILE + c.lz);     // this voxel's term constants
        const double a = build_val<E>(s_img[h], use_max);
        const E q[6] = {s_img[h - HALO_DIM * HALO_DIM], s_img[h + HALO_DIM * HALO_DIM], s_img[h - HALO_DIM],
                        s_img[h + HALO_DIM], s_img[h - 1], s_img[h + 1]};
        double cap[6];
        if (FN == 1 && SPACING == 0) {
            double t6[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const double b = build_val<E>(q[k], use_max);
                // cells outside the lattice were never staged: their (unused) arguments are pinned to 0 so that they
                // cannot push the warp off the ordinary path
                t6[k] = ((valid >> k) & 1u) ? exp_term_arg(Pv, use_max ? fmax(a, b) : fabs(__dsub_rn(a, b))) : 0.0;
            }
            const bool ordinary = __all_sync(0xffffffffu, t6[0] <= 700.0 && t6[1] <= 700.0 && t6[2] <= 700.0 &&
                                                          t6[3] <= 700.0 && t6[4] <= 700.0 && t6[5] <= 700.0);
            exp_caps6(t6, ordinary, valid, cap);
        } else {
#pragma unroll
            for (int k = 0; k < 6; ++k)
                cap[k] = ((valid >> k) & 1u) ? build_weight<FN, E>(Pv, a, q[k], use_max, spacing, P.spacing[k >> 1]) : 0.0;
        }
        if (c.inb) {
            const double tr = lazy_tr(tin, p, fb);
            const double e = c.own ? source_excess(tr, cap) : 0.0;
#pragma unroll
            for (int k = 0; k < 6; ++k) S.cap[k][c.v] = cap[k];
            S.tr[c.v] = tr;
            S.excess[c.v] = e;
        }
        __syncthreads();          // s_img is restaged for the next tile
        cur = nxt;
        i = inext;
    }
}


template <typename T>
__global__ void __launch_bounds__(TILE_VOX) k_window_min(Lattice L, Tiles TL, State<T> S, const int* __restrict__ cmat, LazyTin tin,
                                                         WorkList cur, int* __restrict__ tmin, int* __restrict__ ctl)
{
    __shared__ int s_min[TILE_VOX / 32];
    const int n = *cur.count;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int t = cur.items[i];
        const TileCtx c = tile_ctx(L, TL, t);
        const bool mat = !cmat || cmat[t] != 0;
        const int h = c.own ? S.height[c.v] : MGC_HINF;
        int lo = voxel_active<T>(L, S, tin, c, h, mat) ? h : MGC_HINF;
        lo = __reduce_min_sync(0xffffffffu, lo);
        if ((threadIdx.x & 31) == 0) s_min[threadIdx.x >> 5] = lo;
        __syncthreads();
        if (threadIdx.x < 32) {
            int m = threadIdx.x < TILE_VOX / 32 ? s_min[threadIdx.x] : MGC_HINF;
            m = __reduce_min_sync(0xffffffffu, m);
            if (threadIdx.x == 0) {
                tmin[i] = m;
                if (m < MGC_HINF) atomicMin(ctl + WIN_GMIN, m);
            }
        }
        __syncthreads();
    }
}

// append t of every lane with `take` to a list, one atomic per warp; returns the ballot
__device__ __forceinline__ unsigned warp_append(const WorkList& wl, bool take, int t)
{
    const int lane = threadIdx.x & 31;
    const unsigned b = __ballot_sync(0xffffffffu, take);
    int slot = 0;
    if (lane == 0 && b) slot = atomicAdd(wl.count, __popc(b));
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (take) wl.items[slot + __popc(b & ((1u << lane) - 1u))] = t;
    return b;
}

__global__ void __launch_bounds__(256) k_window_split(WorkList cur, const int* __restrict__ tmin, const int* __restrict__ cmat,
                                                      int* __restrict__ pflag, WorkList now, WorkList later,
                                                      int* __restrict__ drop_items, int* __restrict__ ctl, int labels_capped)
{
    const int n = *cur.count;
    const int gmin = ctl[WIN_GMIN];
    const int lane = threadIdx.x & 31;
    for (int base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31; base < n; base += gridDim.x * blockDim.x) {
        const int i = base + lane;
        const int t = i < n ? cur.items[i] : -1;
        const int m = i < n ? tmin[i] : MGC_HINF;
        const bool act = t >= 0 && m < MGC_HINF;
        const bool drop = t >= 0 && !act && !labels_capped;
        if (drop) pflag[t] = 0;
        warp_append(now, act && m - gmin <= PUSH_WINDOW, t);
        const unsigned bl = warp_append(later, t >= 0 && !drop && !(act && m - gmin <= PUSH_WINDOW), t);
        warp_append(WorkList{drop_items, ctl + WIN_NDROP}, drop && cmat && cmat[t] == 0, t);
        const unsigned bd = __ballot_sync(0xffffffffu, drop);
        if (lane == 0) {
            if (bl) atomicAdd(ctl + WIN_DEFERRED, __popc(bl));
            if (bd) atomicAdd(ctl + WIN_DROPPED, __popc(bd));
        }
    }
}

// exact count of active voxels, scanning only the tiles of the worklists (a superset of the tiles that can hold one).
// Both colours' lists in one launch, four tiles in flight per CTA iteration (the loop is latency-bound with one tile
// per iteration), one atomic per warp at the end.  A listed tile that is not materialised (a window deferred it)
// counts its implicit source excess.
template <typename T>
__global__ void __launch_bounds__(TILE_VOX) k_count_active_tiles2(Lattice L, Tiles TL, State<T> S, const int* __restrict__ cmat,
                                                                  LazyTin tin, WorkList wa, WorkList wb,
                                                                  unsigned long long* __restrict__ count)
{
    const int na = *(volatile int*)wa.count, nb = *(volatile int*)wb.count;
    const int n = na + nb;
    unsigned mine = 0;
    for (int i0 = blockIdx.x * 4; i0 < n; i0 += gridDim.x * 4) {
        T e[4];
        int h[4], t[4];
        bool own[4], lazy[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = i0 + j;
            own[j] = false; lazy[j] = false; e[j] = 0; h[j] = MGC_HINF; t[j] = -1;
            if (i < n) {
                t[j] = i < na ? wa.items[i] : wb.items[i - na];
                const TileCtx c = tile_ctx(L, TL, t[j]);
                own[j] = c.own;
                lazy[j] = cmat && cmat[t[j]] == 0;
                if (c.own) { h[j] = S.height[c.v]; if (!lazy[j]) e[j] = S.excess[c.v]; }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (own[j] && lazy[j] && h[j] < MGC_HINF) e[j] = lazy_has_excess(L, tin, tile_ctx(L, TL, t[j])) ? (T)1 : (T)0;
            mine += (own[j] && e[j] > 0 && h[j] < MGC_HINF) ? 1u : 0u;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_down_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(count, (unsigned long long)mine);
}
