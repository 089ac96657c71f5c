// gc_persist.cuh -- the global relabel (worklist BFS) as ONE cooperative launch.
//
// A BFS driven from the host would need a device->host round trip per pass to learn whether the next worklist is
// empty; on hard instances (hundreds of short passes) those round trips would dominate.  k_bfs_coop (3-D) and
// k_bfs_coop4 (4-D) run all passes inside a single persistent cooperative kernel, separating them with grid-wide
// barriers; the list counts, the cursor and the list selector live in device memory.  A pass visits its tiles with
// relabel_visit (gc_tiles.cuh) / relabel_visit4 (gc_tiles4.cuh).
#pragma once
#include <cooperative_groups.h>
#include "gc_tiles.cuh"
#include "gc_tiles4.cuh"

namespace cg = cooperative_groups;

// control block: CTL_* (gc_tiles.cuh)
__device__ __forceinline__ int ld_ctl(const int* ctl, int i) { return *(const volatile int*)(ctl + i); }

// ---------------------------------------------------------------------------------------------------
// global relabel as one cooperative launch: all passes of the BFS with grid-wide barriers between them
// (`cap`: see relabel_visit; MGC_HINF = exact).
// The relabel visit needs 28 registers and 4 KB of shared memory, so 4 CTAs per SM are co-resident -- twice the
// parallelism of the push kernel -- and no pass costs a host round trip (count read-back, two memsets, launch).
// (A queue-driven asynchronous variant without barriers was tried and rejected: label-correcting order made tiles
//  converge to non-final labels over and over -- 50x more visits at 512^3.)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TILE_VOX, 4)
k_bfs_coop(Lattice L, Tiles TL, const uint8_t* __restrict__ rmask, int* __restrict__ height, int* __restrict__ rflag,
           int* __restrict__ items0, int* __restrict__ items1, int* __restrict__ ctl, int cap)
{
    __shared__ int sh[HALO_VOX];
    __shared__ int s_slot;
    cg::grid_group grid = cg::this_grid();
    const bool leader = blockIdx.x == 0 && threadIdx.x == 0;
    int rl_cur = ld_ctl(ctl, CTL_RLCUR);
    int n_rel = 0;
    for (;;) {
        if (ld_ctl(ctl, rl_cur) == 0) break;
        const WorkList cur{rl_cur ? items1 : items0, ctl + rl_cur};
        const WorkList nxt{rl_cur ? items0 : items1, ctl + (1 - rl_cur)};
        for (;;) {
            const int t = fetch_tile(cur, ctl + CTL_CURSOR, &s_slot);
            if (t < 0) break;
            relabel_visit(L, TL, rmask, height, rflag, nxt, t, sh, cap);
        }
        grid.sync();
        if (leader) { ctl[rl_cur] = 0; ctl[CTL_CURSOR] = 0; }
        rl_cur = 1 - rl_cur;
        n_rel++;
        grid.sync();
    }
    if (leader) { ctl[CTL_RLCUR] = rl_cur; ctl[CTL_RELP] = n_rel; }
}

// the same for 4-D lattices (4 x 4 x 8 x 4 tiles): grid barriers inside one cooperative launch instead of one launch +
// one host round trip per pass (r02 config 4: ~160 passes per solve)
__global__ void __launch_bounds__(T4_VOX, 3)
k_bfs_coop4(Lattice L, Tiles4 TL, const uint8_t* __restrict__ rmask, int* __restrict__ height, int* __restrict__ rflag,
            int* __restrict__ items0, int* __restrict__ items1, int* __restrict__ ctl)
{
    __shared__ int sh[H4_VOX];
    __shared__ int s_slot;
    cg::grid_group grid = cg::this_grid();
    const bool leader = blockIdx.x == 0 && threadIdx.x == 0;
    int rl_cur = ld_ctl(ctl, CTL_RLCUR);
    int n_rel = 0;
    for (;;) {
        if (ld_ctl(ctl, rl_cur) == 0) break;
        const WorkList cur{rl_cur ? items1 : items0, ctl + rl_cur};
        const WorkList nxt{rl_cur ? items0 : items1, ctl + (1 - rl_cur)};
        for (;;) {
            const int t = fetch_tile(cur, ctl + CTL_CURSOR, &s_slot);
            if (t < 0) break;
            relabel_visit4(L, TL, rmask, height, rflag, nxt, t, sh);
        }
        grid.sync();
        if (leader) { ctl[rl_cur] = 0; ctl[CTL_CURSOR] = 0; }
        rl_cur = 1 - rl_cur;
        n_rel++;
        grid.sync();
    }
    if (leader) { ctl[CTL_RLCUR] = rl_cur; ctl[CTL_RELP] = n_rel; }
}
