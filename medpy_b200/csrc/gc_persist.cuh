// gc_persist.cuh -- the whole max-flow as ONE cooperative launch.
//
// The host-driven loop of gc_api.cu (relabel passes, stop test, two-colour push passes) needs a device->host
// round trip per pass to learn whether the worklists are empty; on hard instances (hundreds of short passes)
// those round trips dominate.  k_solve_coop runs the same phases inside a single persistent cooperative kernel
// (as many 512-thread CTAs as are co-resident: 2 per SM), separating them with grid-wide barriers; list counts,
// the cursor and the stop test live in device memory, so the solver never leaves the GPU until it has converged.
// The phases call the very same tile bodies as the stand-alone kernels (gc_tiles.cuh).
#pragma once
#include <cooperative_groups.h>
#include "gc_tiles.cuh"
#include "gc_tiles4.cuh"

namespace cg = cooperative_groups;

// control block in device memory (ints): see gc_api.cu
//   [0],[1]   relabel list counts          [2..5] push list counts [colour*2 + buffer]
//   [8]       work cursor                  [9],[10] buffer each colour consumes next     [11] relabel list consumed next
//   [12]      status out (0 ok, 1 round cap hit)          [13] rounds      [14] push passes    [15] relabel passes
//   [16]      global relabels
#define CTL_CURSOR 8
#define CTL_SEL0 9
#define CTL_RLCUR 11
#define CTL_STATUS 12
#define CTL_ROUNDS 13
#define CTL_PUSHP 14
#define CTL_RELP 15
#define CTL_GREL 16

#define SOLVE_F_RESET 1   // start with a relabel reset (labels from rmask); otherwise labels/list are fresh
#define SOLVE_F_BFS 2     // run relabel passes until the list is empty
#define SOLVE_F_COUNT 4   // count active voxels into *active
#define SOLVE_F_PUSH 8    // run `passes0` two-colour push passes
#define SOLVE_F_LOOP 16   // full solve: (reset) bfs, count, stop-or-push, repeat with doubling passes

struct SolveLists {
    int* rl_items[2];
    int* pl_items[2][2];
};

__device__ __forceinline__ int ld_ctl(const int* ctl, int i) { return *(const volatile int*)(ctl + i); }

template <typename T>
__global__ void __launch_bounds__(TILE_VOX, 2)
k_solve_coop(Lattice L, Tiles TL, State<T> S, SolveLists SL, int* __restrict__ rflag, int* __restrict__ pflag,
             int* __restrict__ ctl, unsigned long long* __restrict__ active, unsigned long long* __restrict__ timers,
             int flags, int iters, int passes0, int passes_max, int max_rounds)
{
    __shared__ T s_out[6 * TILE_VOX];
    __shared__ int s_h[HALO_VOX];
    __shared__ int s_slot;
    cg::grid_group grid = cg::this_grid();
    const bool leader = blockIdx.x == 0 && threadIdx.x == 0;

    int sel[2] = {ld_ctl(ctl, CTL_SEL0), ld_ctl(ctl, CTL_SEL0 + 1)};
    int rl_cur = ld_ctl(ctl, CTL_RLCUR);
    int passes = passes0;
    bool do_reset = (flags & SOLVE_F_RESET) != 0;
    int rounds = 0, n_push = 0, n_rel = 0, n_grel = 0, status = 0;
    unsigned long long t_rel = 0, t_push = 0;

    auto RL = [&](int i) { return WorkList{SL.rl_items[i], ctl + i}; };
    auto PL = [&](int c, int b) { return WorkList{SL.pl_items[c][b], ctl + 2 + c * 2 + b}; };
    auto now = [&]() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; };

    for (;;) {
        unsigned long long t0 = now();
        // ---------------- global relabel ----------------
        if (flags & (SOLVE_F_BFS | SOLVE_F_LOOP)) {
            if (do_reset) {
                for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < TL.ntiles; i += gridDim.x * blockDim.x) rflag[i] = 0;
                if (leader) { ctl[0] = 0; ctl[1] = 0; }
                grid.sync();
                relabel_reset_body(L, TL, S.rmask, S.height, rflag, RL(0));
                rl_cur = 0;
                grid.sync();
            }
            do_reset = true;
            n_grel++;
            for (;;) {
                if (ld_ctl(ctl, rl_cur) == 0) break;
                const WorkList cur = RL(rl_cur), nxt = RL(1 - rl_cur);
                for (;;) {
                    const int t = fetch_tile(cur, ctl + CTL_CURSOR, &s_slot);
                    if (t < 0) break;
                    relabel_visit(L, TL, S.rmask, S.height, rflag, nxt, t, s_h, MGC_HINF);
                }
                grid.sync();
                if (leader) { ctl[rl_cur] = 0; ctl[CTL_CURSOR] = 0; }
                rl_cur = 1 - rl_cur;
                n_rel++;
                grid.sync();
            }
        }
        unsigned long long t1 = now();
        t_rel += t1 - t0;
        // ---------------- stop test ----------------
        if (flags & (SOLVE_F_COUNT | SOLVE_F_LOOP)) {
            if (leader) *active = 0ull;
            grid.sync();
            count_active_body<T>(L, TL, S, PL(0, sel[0]), active);
            count_active_body<T>(L, TL, S, PL(1, sel[1]), active);
            grid.sync();
            if (flags & SOLVE_F_LOOP) {
                if (*(volatile unsigned long long*)active == 0ull) break;
                if (rounds >= max_rounds) { status = 1; break; }
                rounds++;
            }
        }
        // ---------------- push passes ----------------
        if (flags & (SOLVE_F_PUSH | SOLVE_F_LOOP)) {
            unsigned long long t2 = now();
            for (int p = 0; p < passes; ++p) {
                for (int color = 0; color < 2; ++color) {
                    const WorkList cur = PL(color, sel[color]);
                    const WorkList self_next = PL(color, 1 - sel[color]);
                    const WorkList other_next = PL(1 - color, sel[1 - color]);
                    for (;;) {
                        const int t = fetch_tile(cur, ctl + CTL_CURSOR, &s_slot);
                        if (t < 0) break;
                        push_visit<T>(L, TL, S, iters, pflag, self_next, other_next, t, s_out, s_h);
                    }
                    grid.sync();
                    if (leader) { *cur.count = 0; ctl[CTL_CURSOR] = 0; }
                    sel[color] = 1 - sel[color];
                    grid.sync();
                }
                n_push++;
            }
            t_push += now() - t2;
            passes = passes * 2 > passes_max ? passes_max : passes * 2;
        }
        if (!(flags & SOLVE_F_LOOP)) break;
    }
    if (leader) {
        ctl[CTL_SEL0] = sel[0]; ctl[CTL_SEL0 + 1] = sel[1]; ctl[CTL_RLCUR] = rl_cur;
        ctl[CTL_STATUS] = status; ctl[CTL_ROUNDS] = rounds; ctl[CTL_PUSHP] = n_push; ctl[CTL_RELP] = n_rel; ctl[CTL_GREL] = n_grel;
        timers[0] = t_rel; timers[1] = t_push;
    }
}

// ---------------------------------------------------------------------------------------------------
// global relabel alone as one cooperative launch: all passes of the BFS with grid-wide barriers between them
// (`cap`: see relabel_visit; MGC_HINF = exact).
// The relabel visit needs 28 registers and 4 KB of shared memory, so 4 CTAs per SM are co-resident -- twice the
// parallelism k_solve_coop can offer (it is bounded by the push visit) -- while the per-pass host round trip
// (count read-back, two memsets, launch) of the list-driven host loop disappears.
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

// the same for 4-D lattices (4 x 4 x 8 x 4 tiles): replaces one launch + one host round trip PER PASS (r02 config 4:
// ~160 passes per solve) by grid barriers inside one cooperative launch
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
