// gc_slab_kernels.cuh -- the z-slab kernels, launched only by gc_slab.cu: the border messages (k_slab_pack and the
// tile-aware unpacks) and the push-list relisting at the start of every distributed global relabel.
#pragma once
#include "gc_tiles.cuh"
#include "gc_tiles4.cuh"


// ---------------------------------------------------------------------------------------------------
// z-slab border messages (the tile-aware unpack is k_slab_unpack_tiles / k_slab_unpack_tiles4)
// ---------------------------------------------------------------------------------------------------
// pack: heights of my border plane + the flow parked in the ghost plane's excess (my outbox), which is cleared
template <typename T>
__global__ void k_slab_pack(unsigned plane, const int* __restrict__ height_border, T* __restrict__ excess_ghost,
                            int* __restrict__ h_out, double* __restrict__ f_out)
{
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= plane) return;
    h_out[i] = height_border[i];
    if (f_out) {                    // labels-only messages (relabel rounds: nothing was pushed since the last exchange) leave the outbox alone
        f_out[i] = (double)excess_ghost[i];
        excess_ghost[i] = 0;
    }
}

// ---------------------------------------------------------------------------------------------------
// z-slab border messages (written by k_slab_pack of gc_solver.cuh; k_slab_unpack_tiles4 is the 4-D form): ghost
// labels <- the neighbour's border labels; received flow joins the excess of the border voxel and the residual of its
// arc towards the ghost (the reverse of the arc the flow arrived on), and the border voxel's residual mask gains that
// arc.  The receiving tiles are put on the worklists -- the relabel list when a ghost label changed, the push list of
// the tile's colour when flow arrived.
// ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_slab_unpack_tiles(Lattice L, Tiles TL, State<T> S, int z_ghost, int z_border, int k_border_to_ghost,
                                    const int* __restrict__ h_in, const double* __restrict__ f_in,
                                    int* __restrict__ rflag, WorkList rl0, WorkList rl1, const int* __restrict__ rl_cur,
                                    int* __restrict__ pflag, WorkList pl0, WorkList pl1, int* __restrict__ changed)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L.plane) return;
    // the relabel list consumed next: the cooperative BFS keeps its selector in the control block
    const WorkList rl = *rl_cur ? rl1 : rl0;
    const int y = (int)(i / L.stride[1]), x = (int)(i % L.stride[1]);
    const unsigned vg = (unsigned)z_ghost * L.plane + i, vb = (unsigned)z_border * L.plane + i;
    const int tg = ((z_ghost / TILE) * TL.nt[1] + y / TILE) * TL.nt[2] + x / TILE;
    const int tb = ((z_border / TILE) * TL.nt[1] + y / TILE) * TL.nt[2] + x / TILE;
    const int hn = h_in[i];
    if (S.height[vg] != hn) {
        S.height[vg] = hn;
        mark_dirty(TL, tg);
        if (changed) *changed = 1;
        list_push(rflag, rl, tb);
        if (tg != tb) list_push(rflag, rl, tg);
    }
    const double f = f_in ? f_in[i] : 0.0;
    if (f > 0) {
        S.excess[vb] += (T)f;
        S.cap[k_border_to_ghost][vb] += (T)f;
        S.rmask[vb] |= (uint8_t)(1u << k_border_to_ghost);
        const int color = ((z_border / TILE) + y / TILE + x / TILE) & 1;
        list_push(pflag, color ? pl1 : pl0, tb);
    }
}

// ---------------------------------------------------------------------------------------------------
// z-slab border messages (cf. k_slab_unpack_tiles): ghost labels <- the neighbour's border labels, received flow joins
// the border voxel's excess and its arc towards the ghost; the receiving tiles go on the relabel list consumed next
// (ghost label changed) or on the push list of their colour (flow arrived).  4-D lattices keep no dirty tiles to mark.
// ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_slab_unpack_tiles4(Lattice L, Tiles4 TL, State<T> S, int z_ghost, int z_border, int k_border_to_ghost,
                                     const int* __restrict__ h_in, const double* __restrict__ f_in,
                                     int* __restrict__ rflag, WorkList rl0, WorkList rl1, const int* __restrict__ rl_cur,
                                     int* __restrict__ pflag, WorkList pl0, WorkList pl1, int* __restrict__ changed)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L.plane) return;
    const WorkList rl = *rl_cur ? rl1 : rl0;
    const unsigned r = i % L.stride[1];
    const int c1 = (int)(i / L.stride[1]), c2 = (int)(r / L.stride[2]), c3 = (int)(r % L.stride[2]);
    const unsigned vg = (unsigned)z_ghost * L.plane + i, vb = (unsigned)z_border * L.plane + i;
    const int tg = (((z_ghost >> 2) * TL.nt[1] + (c1 >> 2)) * TL.nt[2] + (c2 >> 3)) * TL.nt[3] + (c3 >> 2);
    const int tb = (((z_border >> 2) * TL.nt[1] + (c1 >> 2)) * TL.nt[2] + (c2 >> 3)) * TL.nt[3] + (c3 >> 2);
    const int hn = h_in[i];
    if (S.height[vg] != hn) {
        S.height[vg] = hn;
        if (changed) *changed = 1;
        list_push(rflag, rl, tb);
        if (tg != tb) list_push(rflag, rl, tg);
    }
    const double f = f_in ? f_in[i] : 0.0;
    if (f > 0) {
        S.excess[vb] += (T)f;
        S.cap[k_border_to_ghost][vb] += (T)f;
        S.rmask[vb] |= (uint8_t)(1u << k_border_to_ghost);
        const int color = ((z_border >> 2) + (c1 >> 2) + (c2 >> 3) + (c3 >> 2)) & 1;
        list_push(pflag, color ? pl1 : pl0, tb);
    }
}

// ---------------------------------------------------------------------------------------------------
// push lists at the start of a distributed global relabel: every tile holding an owned voxel with excess goes on the list
// its colour consumes next.  On one lattice a voxel the last relabel left at HINF never gets a finite label again, so its
// tile may leave the lists.  On a slab it can: a neighbour pushes into it across the border with a stale ghost label,
// and the reverse residual arc connects it to the sink at the next relabel.  The stop test counts only listed tiles.
// ---------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(TILE_VOX) k_slab_relist(Lattice L, Tiles TL, State<T> S, int* __restrict__ pflag,
                                                          WorkList pl0, WorkList pl1)
{
    for (int t = blockIdx.x; t < TL.ntiles; t += gridDim.x) {
        const TileCtx c = tile_ctx(L, TL, t);
        const int act = (c.own && S.excess[c.v] > 0) ? 1 : 0;
        if (__syncthreads_or(act) && threadIdx.x == 0) list_push(pflag, tile_color(c) ? pl1 : pl0, t);
    }
}

template <typename T>
__global__ void __launch_bounds__(T4_VOX) k_slab_relist4(Lattice L, Tiles4 TL, State<T> S, int* __restrict__ pflag,
                                                         WorkList pl0, WorkList pl1)
{
    for (int t = blockIdx.x; t < TL.ntiles; t += gridDim.x) {
        const Tile4Ctx c = tile4_ctx(L, TL, t);
        const int act = (c.own && S.excess[c.v] > 0) ? 1 : 0;
        if (__syncthreads_or(act) && threadIdx.x == 0) list_push(pflag, tile4_color(c) ? pl1 : pl0, t);
    }
}
