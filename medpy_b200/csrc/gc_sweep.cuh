// gc_sweep.cuh -- directional line sweeps for the global relabel (exact backward BFS) of HARD instances.
//
// The worklist BFS of gc_tiles.cuh / gc_persist.cuh costs one tile visit (4.5 KB of traffic, a dozen block barriers)
// per 8^3 tile and wavefront that crosses it; when the sink is far away from most of the lattice (boundary-only
// graphs: the only sink links are the background shell, BASELINE configs 2/4/5) every tile is visited several times
// and the BFS, not the pushes, is the solve, far below the HBM rate.  In exactly those
// instances most arcs are residual, so distances are almost Manhattan distances and propagate along straight lines.
// A sweep relaxes every line of one lattice axis in one direction SEQUENTIALLY (Gauss-Seidel along the line, all
// lines in parallel), which carries a label across the whole extent in one pass over memory at streaming rate
// (5 B read + <= 4 B written per voxel) instead of one tile layer per grid barrier.  One round = both directions of
// every axis.  Labels only ever decrease and every value written is the length of a real residual path, so the
// labels stay upper bounds of the true distances; k_relabel_check then lists the tiles that still hold a voxel
// whose label can drop and the worklist BFS finishes from there -- exactness is still established by the fixed
// point of the tile relaxation, the sweeps only bring almost every label to its final value first.
//
// Label semantics are those of relabel_visit: height[v] = 1 + min over residual arcs (v -> w) of height[w];
// bit k of rmask[v] says that arc k = 2*axis + (0: towards -1, 1: towards +1) leaving v is residual.  Only OWNED
// voxels are relabelled (ghost planes of a z-slab are inputs).
#pragma once
#include "gc_tiles.cuh"
#include "gc_tiles4.cuh"

#define SWEEP_UNROLL 16

__device__ __forceinline__ int sweep_inc(int h) { return h >= MGC_HINF ? MGC_HINF : h + 1; }

// ---------------------------------------------------------------------------------------------------
// lines along an axis that is NOT the fastest one: one thread per line, consecutive threads on consecutive
// x (coalesced); forward pass (information travels towards +axis) then backward pass, in one launch.
// `line` enumerates the lines: line = hi * stride + lo with lo = position inside one axis-plane (all faster axes)
// and hi = combined index of the slower axes, so the first voxel of the line is hi * dim * stride + lo.
// ---------------------------------------------------------------------------------------------------
template <bool FWD>
__device__ __forceinline__ void sweep_line(const uint8_t* __restrict__ rmask, int* __restrict__ height, unsigned base,
                                           unsigned stride, int D, int i_own0, int i_own1, unsigned bit)
{
    int carry = MGC_HINF;
    for (int i0 = 0; i0 < D; i0 += SWEEP_UNROLL) {
        int hb[SWEEP_UNROLL];
        unsigned mb[SWEEP_UNROLL];
#pragma unroll
        for (int u = 0; u < SWEEP_UNROLL; ++u) {
            const int j = i0 + u;
            if (j < D) {
                const int i = FWD ? j : D - 1 - j;
                const unsigned v = base + (unsigned)i * stride;
                hb[u] = __ldcg(height + v);
                mb[u] = rmask[v];
            }
        }
#pragma unroll
        for (int u = 0; u < SWEEP_UNROLL; ++u) {
            const int j = i0 + u;
            if (j < D) {
                const int i = FWD ? j : D - 1 - j;
                int h = hb[u];
                if ((mb[u] & bit) && i >= i_own0 && i < i_own1) {
                    const int cand = sweep_inc(carry);
                    if (cand < h) { h = cand; height[base + (unsigned)i * stride] = h; }
                }
                carry = h;
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_sweep_axis(Lattice L, const uint8_t* __restrict__ rmask, int* __restrict__ height, int axis)
{
    const unsigned stride = L.stride[axis];
    const int D = L.dim[axis];
    const unsigned nlines = L.n / (unsigned)D;
    const unsigned line = blockIdx.x * blockDim.x + threadIdx.x;
    if (line >= nlines) return;
    const unsigned hi = line / stride, lo = line - hi * stride;
    const unsigned base = hi * (unsigned)D * stride + lo;
    int i_own0 = 0, i_own1 = D;
    if (axis == 0) { i_own0 = L.own0; i_own1 = L.own1; }
    else {
        const int z = (int)(base / L.stride[0]);
        if (z < L.own0 || z >= L.own1) return;          // a line inside a ghost plane: nothing to relabel
    }
    // forward: voxel i receives from i-1 through its own arc towards -axis (bit 2*axis)
    sweep_line<true>(rmask, height, base, stride, D, i_own0, i_own1, 1u << (2 * axis));
    // backward: voxel i receives from i+1 through its arc towards +axis
    sweep_line<false>(rmask, height, base, stride, D, i_own0, i_own1, 1u << (2 * axis + 1));
}

// ---------------------------------------------------------------------------------------------------
// rows of the fastest axis: one warp per row, the row (segments of <= SWEEP_ROW_MAX voxels) staged in shared memory
// with coalesced loads; every lane then owns a contiguous chunk, relaxes it sequentially, the chunk summaries
// f(c) = min(a, c + b) ("label of my last voxel given the label c in front of my chunk") are composed across the
// lanes with a 5-step shuffle scan, and a second sequential pass applies the incoming label.
// ---------------------------------------------------------------------------------------------------
#define SWEEP_ROW_MAX 1024
#define SWEEP_ROW_PAD (SWEEP_ROW_MAX + SWEEP_ROW_MAX / 32)
#define SWEEP_WARPS 4

__device__ __forceinline__ int srow_idx(int x) { return x + (x >> 5); }   // one pad word per 32: lane chunks of 32 do not collide

// one direction over the staged segment [0, n): FWD = towards +x.  carry_in = label of the voxel in front of the
// segment (HINF if none); returns the label of the segment's last voxel in sweep direction.  `changed` accumulates.
template <bool FWD>
__device__ __forceinline__ int sweep_row_dir(int* sh, const uint8_t* sm, int n, int len, unsigned bit, int carry_in, int& changed)
{
    const int lane = threadIdx.x & 31;
    const int c0 = lane * len;
    const int cnt = max(0, min(len, n - c0));       // my elements: x = c0 .. c0+cnt-1 (ascending order)
    // ---- pass 1: local relaxation with nothing coming in
    int prev = MGC_HINF;
    int nopen = 0;             // leading elements (in sweep order) whose arc towards the predecessor is residual
    bool chain = true;
    for (int j = 0; j < cnt; ++j) {
        const int x = FWD ? c0 + j : c0 + cnt - 1 - j;
        int h = sh[srow_idx(x)];
        const bool open = (sm[x] & bit) != 0;
        if (open) {
            const int cand = sweep_inc(prev);
            if (cand < h) { h = cand; sh[srow_idx(x)] = h; changed = 1; }
        }
        if (chain) { if (open) ++nopen; else chain = false; }
        prev = h;
    }
    // summary: (a, b): last label = min(a, c + b), b = HINF if the chain is broken inside the chunk; empty chunk = identity
    int a = cnt ? prev : MGC_HINF;
    int b = cnt ? (nopen == cnt ? cnt : MGC_HINF) : 0;
    // ---- inclusive scan of the composition over lanes in sweep order (lane 0 first when FWD, lane 31 first otherwise)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int a1 = FWD ? __shfl_up_sync(0xffffffffu, a, o) : __shfl_down_sync(0xffffffffu, a, o);
        const int b1 = FWD ? __shfl_up_sync(0xffffffffu, b, o) : __shfl_down_sync(0xffffffffu, b, o);
        const bool has = FWD ? (lane >= o) : (lane + o < 32);
        if (has) {
            // (a, b) o (a1, b1): first (a1, b1) then me
            const int t = (a1 >= MGC_HINF || b >= MGC_HINF) ? MGC_HINF : min(a1 + b, MGC_HINF);
            a = min(a, t);
            b = (b1 >= MGC_HINF || b >= MGC_HINF) ? MGC_HINF : min(b1 + b, MGC_HINF);
        }
    }
    // label in front of my chunk: the composite of all earlier lanes applied to carry_in
    int pa = FWD ? __shfl_up_sync(0xffffffffu, a, 1) : __shfl_down_sync(0xffffffffu, a, 1);
    int pb = FWD ? __shfl_up_sync(0xffffffffu, b, 1) : __shfl_down_sync(0xffffffffu, b, 1);
    const bool first = FWD ? (lane == 0) : (lane == 31);
    int cin;
    if (first) cin = carry_in;
    else {
        const int t = (carry_in >= MGC_HINF || pb >= MGC_HINF) ? MGC_HINF : min(carry_in + pb, MGC_HINF);
        cin = min(pa, t);
    }
    // ---- pass 2: apply the incoming label along the open prefix of my chunk
    if (cin < MGC_HINF) {
        int c = cin;
        for (int j = 0; j < nopen; ++j) {
            const int x = FWD ? c0 + j : c0 + cnt - 1 - j;
            c = sweep_inc(c);
            if (c < sh[srow_idx(x)]) { sh[srow_idx(x)] = c; changed = 1; }
            else break;                 // from here on my own labels are at least as good (they grow by <= 1 per step)
        }
    }
    // label of the segment's last voxel in sweep direction: the full composite applied to carry_in, from the last lane
    const int la = __shfl_sync(0xffffffffu, a, FWD ? 31 : 0);
    const int lb = __shfl_sync(0xffffffffu, b, FWD ? 31 : 0);
    const int t = (carry_in >= MGC_HINF || lb >= MGC_HINF) ? MGC_HINF : min(carry_in + lb, MGC_HINF);
    return min(la, t);
}

__device__ __forceinline__ void srow_load(const uint8_t* __restrict__ rmask, const int* __restrict__ height, unsigned g0, int n,
                                          int* sh, uint8_t* sm)
{
    const int lane = threadIdx.x & 31;
    for (int x = lane; x < n; x += 32) { sh[srow_idx(x)] = __ldcg(height + g0 + x); sm[x] = rmask[g0 + x]; }
    __syncwarp();
}
__device__ __forceinline__ void srow_store(int* __restrict__ height, unsigned g0, int n, const int* sh)
{
    const int lane = threadIdx.x & 31;
    __syncwarp();
    for (int x = lane; x < n; x += 32) height[g0 + x] = sh[srow_idx(x)];
}

__global__ void __launch_bounds__(32 * SWEEP_WARPS) k_sweep_rows(Lattice L, const uint8_t* __restrict__ rmask, int* __restrict__ height)
{
    __shared__ int s_h[SWEEP_WARPS][SWEEP_ROW_PAD];
    __shared__ uint8_t s_m[SWEEP_WARPS][SWEEP_ROW_MAX];
    const int warp = threadIdx.x >> 5;
    int* sh = s_h[warp];
    uint8_t* sm = s_m[warp];
    const int ax = L.nd - 1;
    const int X = L.dim[ax];
    const unsigned nrows = L.n / (unsigned)X;
    const unsigned bit_m = 1u << (2 * ax), bit_p = 1u << (2 * ax + 1);
    const int nseg = (X + SWEEP_ROW_MAX - 1) / SWEEP_ROW_MAX;
    for (unsigned row = blockIdx.x * SWEEP_WARPS + warp; row < nrows; row += gridDim.x * SWEEP_WARPS) {
        const unsigned g = row * (unsigned)X;
        const int z = (int)(g / L.stride[0]);
        if (z < L.own0 || z >= L.own1) continue;
        if (nseg == 1) {
            const int len = (X + 31) >> 5;
            srow_load(rmask, height, g, X, sh, sm);
            int changed = 0;
            sweep_row_dir<true>(sh, sm, X, len, bit_m, MGC_HINF, changed);
            __syncwarp();
            sweep_row_dir<false>(sh, sm, X, len, bit_p, MGC_HINF, changed);
            if (__any_sync(0xffffffffu, changed)) srow_store(height, g, X, sh);
            __syncwarp();
        } else {
            int carry = MGC_HINF;
            for (int s = 0; s < nseg; ++s) {
                const int x0 = s * SWEEP_ROW_MAX, n = min(SWEEP_ROW_MAX, X - x0);
                srow_load(rmask, height, g + x0, n, sh, sm);
                int changed = 0;
                carry = sweep_row_dir<true>(sh, sm, n, (n + 31) >> 5, bit_m, carry, changed);
                if (__any_sync(0xffffffffu, changed)) srow_store(height, g + x0, n, sh);
                __syncwarp();
            }
            carry = MGC_HINF;
            for (int s = nseg - 1; s >= 0; --s) {
                const int x0 = s * SWEEP_ROW_MAX, n = min(SWEEP_ROW_MAX, X - x0);
                srow_load(rmask, height, g + x0, n, sh, sm);
                int changed = 0;
                carry = sweep_row_dir<false>(sh, sm, n, (n + 31) >> 5, bit_p, carry, changed);
                if (__any_sync(0xffffffffu, changed)) srow_store(height, g + x0, n, sh);
                __syncwarp();
            }
        }
    }
}

// short rows (fastest axis of <= SWEEP_SHORT voxels, e.g. the 4 channels of a multi-spectral 4-D image): one THREAD per
// row, forward then backward; consecutive threads read consecutive rows, so the loads still coalesce.
#define SWEEP_SHORT 32
__global__ void __launch_bounds__(256) k_sweep_rows_short(Lattice L, const uint8_t* __restrict__ rmask, int* __restrict__ height)
{
    const int ax = L.nd - 1;
    const int X = L.dim[ax];
    const unsigned nrows = L.n / (unsigned)X;
    const unsigned row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    const unsigned g = row * (unsigned)X;
    const int z = (int)(g / L.stride[0]);
    if (z < L.own0 || z >= L.own1) return;
    const unsigned bit_m = 1u << (2 * ax), bit_p = 1u << (2 * ax + 1);
    int h[SWEEP_SHORT];
    unsigned m[SWEEP_SHORT];
#pragma unroll
    for (int x = 0; x < SWEEP_SHORT; ++x) if (x < X) { h[x] = __ldcg(height + g + x); m[x] = rmask[g + x]; }
    unsigned changed = 0;
#pragma unroll
    for (int x = 1; x < SWEEP_SHORT; ++x)
        if (x < X && (m[x] & bit_m)) { const int c = sweep_inc(h[x - 1]); if (c < h[x]) { h[x] = c; changed |= 1u << x; } }
#pragma unroll
    for (int x = SWEEP_SHORT - 2; x >= 0; --x)
        if (x + 1 < X && (m[x] & bit_p)) { const int c = sweep_inc(h[x + 1]); if (c < h[x]) { h[x] = c; changed |= 1u << x; } }
#pragma unroll
    for (int x = 0; x < SWEEP_SHORT; ++x) if (x < X && (changed >> x) & 1u) height[g + x] = h[x];
}

// ---------------------------------------------------------------------------------------------------
// fixed-point check: lists (relabel worklist `rl`, flags `rflag`, both zeroed by the host) every 8^3 tile that holds
// an owned voxel whose label can still drop given its residual neighbours' labels.  One thread per voxel, neighbour
// labels from L1/L2 (5 B of HBM traffic per voxel).  3-D lattices only (the 8^3 tile numbering of gc_tiles.cuh).
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_relabel_check(Lattice L, Tiles TL, const uint8_t* __restrict__ rmask,
                                                       const int* __restrict__ height, int* __restrict__ rflag, WorkList rl)
{
    const unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= L.n) return;
    const unsigned m = rmask[v] & 0x3fu;
    if (!m) return;
    const int h = __ldcg(height + v);
    if (h <= 1) return;
    int c[3];
    decode<3>(L, v, c);
    if (c[0] < L.own0 || c[0] >= L.own1) return;
    int best = h;
#pragma unroll
    for (int k = 0; k < 6; ++k)
        if (m & (1u << k)) {
            const int hw = sweep_inc(__ldcg(height + (unsigned)((int)v + dir_offset(L, k))));
            best = hw < best ? hw : best;
        }
    if (best < h) {
        const int t = ((c[0] >> 3) * TL.nt[1] + (c[1] >> 3)) * TL.nt[2] + (c[2] >> 3);
        if (*(volatile int*)(rflag + t) == 0) list_push(rflag, rl, t);
    }
}

// 4-D lattices (4 x 4 x 8 x 4 tiles of gc_tiles4.cuh; all eight mask bits are arcs, the sink flag lives in smask and is
// not needed here: labels 1 are already in place)
__global__ void __launch_bounds__(256) k_relabel_check4(Lattice L, Tiles4 TL, const uint8_t* __restrict__ rmask,
                                                        const int* __restrict__ height, int* __restrict__ rflag, WorkList rl)
{
    const unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= L.n) return;
    const unsigned m = rmask[v];
    if (!m) return;
    const int h = __ldcg(height + v);
    if (h <= 1) return;
    int c[4];
    decode<4>(L, v, c);
    if (c[0] < L.own0 || c[0] >= L.own1) return;
    int best = h;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        if (m & (1u << k)) {
            const int hw = sweep_inc(__ldcg(height + (unsigned)((int)v + dir_offset(L, k))));
            best = hw < best ? hw : best;
        }
    if (best < h) {
        const int t = (((c[0] >> 2) * TL.nt[1] + (c[1] >> 2)) * TL.nt[2] + (c[2] >> 3)) * TL.nt[3] + (c[3] >> 2);
        if (*(volatile int*)(rflag + t) == 0) list_push(rflag, rl, t);
    }
}
