// gc_solve.cu -- the tile solver of a lattice handle (gc_handle.cuh): the lazy push state, the solver driver from the
// first init to the read-out, and mgc_maxflow.
#include "gc_handle.cuh"
#include "gc_solver.cuh"
#include "gc_persist.cuh"
#include "gc_sweep.cuh"
#include "gc_solve_kernels.cuh"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>

// cuTensorMapEncodeTiled, resolved at run time so that the library does not link libcuda
tmap_encode_fn tensor_map_encoder()
{
    static tmap_encode_fn encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
            cudaGetLastError();
            return nullptr;
        }
        encode = (tmap_encode_fn)fn;
    }
    return encode;
}

namespace {
// rank-3 float64 tensor maps of cap[0..5] and excess with an 8x8x8 box over the local lattice (x fastest)
bool make_push_maps(mgc_graph* g)
{
    tmap_encode_fn encode = tensor_map_encoder();
    if (!encode) return false;
    const cuuint64_t X = (cuuint64_t)g->L.dim[2], Y = (cuuint64_t)g->L.dim[1], Z = (cuuint64_t)g->L.dim[0];
    if (X % 2) return false;                                   // global strides must be multiples of 16 B
    const cuuint64_t dims[3] = {X, Y, Z};
    const cuuint64_t strides[2] = {X * 8, X * Y * 8};
    const cuuint32_t box[3] = {TILE, TILE, TILE};
    const cuuint32_t estr[3] = {1, 1, 1};
    for (int p = 0; p < TMA_PLANES; ++p) {
        void* base = p < 6 ? (void*)g->S.cap[p] : (void*)g->S.excess;
        if (((uintptr_t)base) & 15) return false;
        if (encode(&g->maps.m[p], CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return false;
    }
    return true;
}
}  // namespace

// the environment options of the tile solver, the same for 3-D and 4-D lattices.  `bfs` is the cooperative BFS kernel
// of the lattice's tile shape, launched with `bfs_threads` threads per CTA: its occupancy sizes the grid.
int tile_solver_options(mgc_graph* g)
{
    const void* bfs = g->nd == 4 ? (const void*)k_bfs_coop4 : (const void*)k_bfs_coop;
    const int bfs_threads = g->nd == 4 ? T4_VOX : TILE_VOX;
    g->n_ctas = 2 * cached_sm_count(g->device);   // k_push_tile is built for 2 CTAs per SM
    if (const char* e1 = getenv("MEDPY_GC_ITERS")) if (atoi(e1) > 0) g->tile_iters = g->tile_iters_first = atoi(e1);
    if (const char* e2 = getenv("MEDPY_GC_PASSES0")) if (atoi(e2) > 0) g->passes0 = atoi(e2);
    if (const char* e3 = getenv("MEDPY_GC_PASSES_MAX")) if (atoi(e3) > 0) g->passes_max = atoi(e3);
    if (const char* e7 = getenv("MEDPY_GC_SWEEP")) g->use_sweeps = atoi(e7) != 0;
    if (const char* e8 = getenv("MEDPY_GC_SWEEP_FRAC")) if (atoi(e8) > 0) g->sweep_frac = atoi(e8);
    if (const char* e9 = getenv("MEDPY_GC_SWEEP_ROUNDS")) if (atoi(e9) > 0) g->sweep_rounds_max = atoi(e9);
    if (const char* e11 = getenv("MEDPY_GC_SWEEP_MIN_ROUNDS")) if (atoi(e11) > 0) g->sweep_rounds_min = atoi(e11);
    if (const char* e10 = getenv("MEDPY_GC_SWEEP_DONE_FRAC")) if (atoi(e10) > 0) g->sweep_done_frac = atoi(e10);
    if (const char* e12 = getenv("MEDPY_GC_BUILD_REFUSE_ALL")) g->build_refuse_all = atoi(e12) != 0;
    int coop = 0, nb = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, g->device);
    if (!coop || cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, bfs, bfs_threads, 0) != cudaSuccess || nb < 1) {
        cudaGetLastError();
        FAIL(MGC_E_CUDA, "the cooperative BFS of the tile solver cannot be launched on this device (no co-resident CTA)");
    }
    g->coop_bfs_grid = nb * cached_sm_count(g->device);
    return MGC_OK;
}

// 3-D lattices: the push kernel stages its tile planes with TMA (gc_tma.cuh) unless MEDPY_GC_TMA=0 or the tensor maps
// cannot be made
void push_tma_setup(mgc_graph* g)
{
    const char* e6 = getenv("MEDPY_GC_TMA");
    const size_t smem = 2 * TMA_STAGE_BYTES + 6 * TILE_VOX * sizeof(double) + 1024 * sizeof(int) + 64;
    if ((!e6 || atoi(e6) != 0) && make_push_maps(g) &&
        cudaFuncSetAttribute(k_push_tile_tma<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess)
        g->use_tma = true;
    else
        cudaGetLastError();
}

// terms that were never given leave their arrays unwritten: zero them before anything reads them
int materialise_zeros(mgc_graph* g)
{
    const size_t nb = (size_t)g->L.n;
    if (g->caps_fresh) {
        for (int k = 0; k < 2 * g->nd; ++k) CK(cudaMemsetAsync(g->S.cap[k], 0, nb * sizeof(double), g->stream));
        g->caps_fresh = false;
    }
    if (g->tr_fresh) {
        CK(cudaMemsetAsync(g->S.tr, 0, nb * sizeof(double), g->stream));
        g->tr_fresh = false;
    }
    return MGC_OK;
}

// materialise the tiles of a push worklist and their face neighbours (wl.items == nullptr: every tile), between a pair of
// events so that its time is kept apart from the push passes around it
int caps_launch(mgc_graph* g, WorkList wl)
{
    if (g->caps_ev_used + 2 > g->caps_ev.size()) g->caps_ev.resize(g->caps_ev_used + 2, nullptr);
    for (size_t i = g->caps_ev_used; i < g->caps_ev_used + 2; ++i) if (!g->caps_ev[i]) CK(cudaEventCreate(&g->caps_ev[i]));
    CK(cudaEventRecord(g->caps_ev[g->caps_ev_used], g->stream));
    CK(cudaMemsetAsync(g->d_flags + 4, 0, 2 * sizeof(int), g->stream));
    k_caps_claim<<<(unsigned)g->n_ctas * 4u, 256, 0, g->stream>>>(g->TL, g->cmat, wl, g->caps_list, g->d_flags + 4);
    int* count = g->d_flags + 4;              // [4] tiles claimed by this launch, [5] cursor
    int* done = g->d_flags + 3;               // tiles materialised since the build
    lazy_dispatch(g, [&](auto t) {
        using T = decltype(t);
        k_caps_tiles<typename T::E, T::FN, T::USE_MAX, T::SPACING><<<(unsigned)g->n_ctas, TILE_VOX, 0, g->stream>>>(
            g->L, g->TL, g->S, (const typename T::E*)g->caps_img, g->caps_P, g->caps_tin, g->caps_list, count, count + 1, done);
    });
    CK(cudaEventRecord(g->caps_ev[g->caps_ev_used + 1], g->stream));
    g->caps_ev_used += 2;
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    return MGC_OK;
}

// capacities, tr or excess are about to be read or written outside the push path: materialise the tiles that are not yet
int push_state_all(mgc_graph* g)
{
    if (!g->caps_lazy) return MGC_OK;
    g->caps_lazy = false;
    return caps_launch(g, WorkList{nullptr, nullptr});
}

// device ms of the materialiser launches since the last call, added to ms_caps; waits for the last of them
double caps_resolve(mgc_graph* g)
{
    double total = 0.0;
    if (g->caps_ev_used && cudaEventSynchronize(g->caps_ev[g->caps_ev_used - 1]) == cudaSuccess) {
        for (size_t i = 0; i + 1 < g->caps_ev_used; i += 2) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, g->caps_ev[i], g->caps_ev[i + 1]) == cudaSuccess) total += ms;
        }
    }
    g->caps_ev_used = 0;
    g->st.ms_caps += total;
    return total;
}

namespace {
int read_tcount(mgc_graph* g, int idx, int* out)
{
    CK(cudaMemcpyAsync(out, g->d_tcount + idx, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    return MGC_OK;
}
}  // namespace

// forget the dirty tiles (everything is in the reset state: fresh build / init, or a full reset just ran)
int dirty_clear(mgc_graph* g)
{
    if (g->nd == 3 && g->TL.dflag) {
        CK(cudaMemsetAsync(g->TL.dflag, 0, (size_t)g->TL.ntiles * sizeof(int), g->stream));
        CK(cudaMemsetAsync(g->TL.dcount, 0, sizeof(int), g->stream));
    }
    return MGC_OK;
}

// first call: solver state + first labels + first worklists in one pass (k_init_tile)
int init_tiles(mgc_graph* g)
{
    Nvtx range("mgc:init_state");
    { int rc0 = push_state_all(g); if (rc0) return rc0; }       // k_init_tile reads every capacity
    CK(cudaMemsetAsync(g->d_tcount, 0, 256, g->stream));
    g->pl_sel[0] = g->pl_sel[1] = 0;
    const bool warm = warm_wanted(g);      // tr > 0 becomes the residual source capacity (gc_seeds.cuh)
    cudaEventRecord(g->ev[4], g->stream);
    if (g->nd == 4) {
        if (warm) k_init_tile4<double, true><<<g->TL4.ntiles, T4_VOX, 0, g->stream>>>(g->L, g->TL4, g->S, g->smask, g->rflag, rl(g, 0),
                                                                                     g->pflag, pl(g, 0, 0), pl(g, 1, 0));
        else k_init_tile4<double><<<g->TL4.ntiles, T4_VOX, 0, g->stream>>>(g->L, g->TL4, g->S, g->smask, g->rflag, rl(g, 0), g->pflag,
                                                                           pl(g, 0, 0), pl(g, 1, 0));
    } else if (warm) {
        k_init_tile<double, true><<<g->TL.ntiles, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S, g->rflag, rl(g, 0), g->pflag,
                                                                            pl(g, 0, 0), pl(g, 1, 0));
    } else {
        k_init_tile<double><<<g->TL.ntiles, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S, g->rflag, rl(g, 0), g->pflag,
                                                                      pl(g, 0, 0), pl(g, 1, 0));
    }
    cudaEventRecord(g->ev[5], g->stream);
    g->init_timed = true;
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    g->state_init = true;
    g->labels_fresh = true;
    g->sweep_mode = -1;
    if (warm) {
        g->warm_state = true;
        g->flow_started = true;        // tr no longer holds the terms: no term may be added on top of it
    }
    return dirty_clear(g);
}

// exact global relabel by tile-wise relaxation; work is proportional to the tiles whose labels still move.
// begin: labels from the residual mask + a fresh worklist (skipped when k_init_tile just produced both)
int relabel_tiles_begin(mgc_graph* g)
{
    if (g->labels_fresh) {
        g->labels_fresh = false;
        CK(cudaMemsetAsync(g->d_tcount + CTL_RLCUR, 0, sizeof(int), g->stream));
        return MGC_OK;
    }
    CK(cudaMemsetAsync(g->d_tcount, 0, 2 * sizeof(int), g->stream));
    CK(cudaMemsetAsync(g->rflag, 0, (size_t)g->TL.ntiles * sizeof(int), g->stream));
    if (g->nd == 4) {
        k_relabel_reset4<<<g->TL4.ntiles, T4_VOX, 0, g->stream>>>(g->L, g->TL4, g->S.rmask, g->smask, g->S.height, g->rflag, rl(g, 0));
    } else {
        if (g->TL.dflag && g->sweep_mode == 0) {
            // easy instance: only the tiles written since the last reset (labels / sink-link bits) are not in the reset state
            k_relabel_reset_list<<<g->n_ctas * 2, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S.rmask, g->S.height, g->rflag, rl(g, 0));
            CK(cudaMemsetAsync(g->TL.dcount, 0, sizeof(int), g->stream));
        } else {
            const unsigned nruns = (unsigned)g->L.dim[0] * (unsigned)g->L.dim[1] * (unsigned)g->TL.nt[2];
            unsigned grid = (nruns + 255u) / 256u;
            if (grid > (unsigned)g->n_ctas * 8u) grid = (unsigned)g->n_ctas * 8u;
            k_relabel_reset<<<grid, 256, 0, g->stream>>>(g->L, g->TL, g->S.rmask, g->S.height, g->rflag, rl(g, 0));
            int rcd = dirty_clear(g);
            if (rcd) return rcd;
        }
    }
    g->st.kernel_launches++;
    CK(cudaMemsetAsync(g->d_tcount + CTL_RLCUR, 0, sizeof(int), g->stream));
    CK(cudaGetLastError());
    return MGC_OK;
}

namespace {
// run passes until the current worklist is empty; *any = 1 if any tile was visited
// one round of directional sweeps (both directions of every axis), then the list of tiles that are not at the fixed
// point yet (gc_sweep.cuh); *pending = number of such tiles (host synchronisation)
int relabel_sweep_round(mgc_graph* g, int* pending, bool with_check)
{
    const int last = g->nd - 1;
    for (int a = 0; a < last; ++a) {
        if (g->L.dim[a] < 2) continue;
        const unsigned nlines = g->L.n / (unsigned)g->L.dim[a];
        k_sweep_axis<<<(nlines + 255u) / 256u, 256, 0, g->stream>>>(g->L, g->S.rmask, g->S.height, a);
        g->st.kernel_launches++;
    }
    if (g->L.dim[last] >= 2 && g->L.dim[last] <= SWEEP_SHORT) {
        const unsigned nrows = g->L.n / (unsigned)g->L.dim[last];
        k_sweep_rows_short<<<(nrows + 255u) / 256u, 256, 0, g->stream>>>(g->L, g->S.rmask, g->S.height);
        g->st.kernel_launches++;
    } else if (g->L.dim[last] >= 2) {
        const unsigned nrows = g->L.n / (unsigned)g->L.dim[last];
        unsigned grid = (nrows + SWEEP_WARPS - 1) / SWEEP_WARPS;
        const unsigned cap = (unsigned)cached_sm_count(g->device) * 16u;
        if (grid > cap) grid = cap;
        k_sweep_rows<<<grid, 32 * SWEEP_WARPS, 0, g->stream>>>(g->L, g->S.rmask, g->S.height);
        g->st.kernel_launches++;
    }
    g->st.relabel_sweeps++;
    if (!with_check) { CK(cudaGetLastError()); return MGC_OK; }     // an early round: the next one follows without a verdict
    CK(cudaMemsetAsync(g->d_tcount, 0, 2 * sizeof(int), g->stream));
    CK(cudaMemsetAsync(g->rflag, 0, (size_t)g->TL.ntiles * sizeof(int), g->stream));
    if (g->nd == 4) k_relabel_check4<<<nblocks(g), 256, 0, g->stream>>>(g->L, g->TL4, g->S.rmask, g->S.height, g->rflag, rl(g, 0));
    else            k_relabel_check<<<nblocks(g), 256, 0, g->stream>>>(g->L, g->TL, g->S.rmask, g->S.height, g->rflag, rl(g, 0));
    g->st.kernel_launches++;
    CK(cudaMemsetAsync(g->d_tcount + CTL_RLCUR, 0, sizeof(int), g->stream));
    CK(cudaGetLastError());
    return read_tcount(g, 0, pending);
}
}  // namespace

// `first`: no stop test reads this relabel's labels (the first relabel of a solve, whose round skips the test).  On an
// easy instance of the 3-D tile solver such a relabel stops at g->first_cap (DESIGN.md §4.3).
int relabel_tiles_run(mgc_graph* g, int* any, bool want_any, bool first)
{
    *any = 0;
    g->relp_last = 0;
    g->relp_pending = false;
    if (g->use_sweeps && g->TL.ntiles >= 64 && g->sweep_mode != 0) {
        int pending = 0;
        int rc = read_tcount(g, 0, &pending);
        if (rc) return rc;
        // one decision per solve (one host synchronisation): an instance whose first relabel has to label most of the
        // lattice is a hard one at every later relabel too, an easy one (regional term: most voxels own a sink link) never is
        if (g->sweep_mode < 0) g->sweep_mode = pending > g->TL.ntiles / g->sweep_frac ? 1 : 0;
        if (pending > g->TL.ntiles / g->sweep_frac) {
            *any = 1;
            int prev = g->TL.ntiles + 1;
            const int rmin = g->sweep_rounds_min < g->sweep_rounds_max ? g->sweep_rounds_min : g->sweep_rounds_max;
            for (int r = 0; r < g->sweep_rounds_max; ++r) {
                // the first rounds run without the 5 B/voxel fixed-point check: nobody would act on its verdict
                const bool check = r + 1 >= rmin;
                rc = relabel_sweep_round(g, &pending, check);
                if (rc) return rc;
                if (!check) continue;
                if (pending <= g->TL.ntiles / g->sweep_done_frac) break;
                if ((long long)pending * 4 > (long long)prev * 3) break;      // a round that clears < 25 %: the rest is local detail
                prev = pending;
            }
        }
    }
    // the sweep decision is made above; the cap needs an easy instance of the 3-D tile solver, where the label window runs
    const bool capped = first && g->first_cap >= 2 && g->sweep_mode == 0 && g->nd == 3 && !g->slab;
    int cap = capped ? g->first_cap : MGC_HINF;
    g->labels_capped = capped;
    // all passes in one cooperative launch; the list selector lives in the control block (device side), so the
    // host does not have to synchronise unless the caller wants to know whether anything moved
    CK(cudaMemsetAsync(g->d_tcount + CTL_CURSOR, 0, sizeof(int), g->stream));
    int* it0 = g->rl_items[0]; int* it1 = g->rl_items[1];
    if (g->nd == 4) {
        void* args4[] = {&g->L, &g->TL4, &g->S.rmask, &g->S.height, &g->rflag, &it0, &it1, &g->d_tcount};
        CK(cudaLaunchCooperativeKernel((void*)k_bfs_coop4, dim3(g->coop_bfs_grid), dim3(T4_VOX), args4, 0, g->stream));
    } else {
        void* args[] = {&g->L, &g->TL, &g->S.rmask, &g->S.height, &g->rflag, &it0, &it1, &g->d_tcount, &cap};
        CK(cudaLaunchCooperativeKernel((void*)k_bfs_coop, dim3(g->coop_bfs_grid), dim3(TILE_VOX), args, 0, g->stream));
    }
    g->st.kernel_launches++;
    g->st.relabel_sweeps++;     // passes are counted on the device (ctl[CTL_RELP]); one launch here
    if (want_any) {
        int relp = 0;
        CK(cudaMemcpyAsync(&relp, g->d_tcount + CTL_RELP, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        if (relp != 0) *any = 1;
        g->relp_last = relp;
        g->st.relabel_passes += relp;
    } else {
        g->relp_pending = true;     // read back by relabel_passes_fetch / _collect
    }
    return MGC_OK;
}

namespace {
// BFS passes of the last relabel_tiles_run.  The cooperative BFS leaves them in the control block: _fetch enqueues their copy
// to pinned memory (after the relabel's timing event, so the adaptive schedule does not see the copy), _collect reads them
// once the stream has passed it (`*enqueued`: a copy was enqueued and needs a stream synchronisation).
int relabel_passes_fetch(mgc_graph* g, bool* enqueued)
{
    *enqueued = false;
    if (!g->relp_pending) return MGC_OK;
    if (!g->h_bad) { g->relp_pending = false; return MGC_OK; }       // no pinned slot: the count is not kept
    CK(cudaMemcpyAsync(g->h_bad + 4, g->d_tcount + CTL_RELP, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
    *enqueued = true;
    return MGC_OK;
}

int relabel_passes_collect(mgc_graph* g)
{
    if (g->relp_pending) {
        g->relp_last = ((volatile int*)g->h_bad)[4];
        g->st.relabel_passes += g->relp_last;
        g->relp_pending = false;
    }
    return g->relp_last;
}

// one colour: consume its current list; still-active tiles go to its alternate list, receivers of cross-face flow
// to the list the other colour consumes next
// tiles whose push state may still be implicit (nullptr: every tile is materialised)
const int* lazy_cmat(const mgc_graph* g) { return g->caps_lazy ? g->cmat : nullptr; }

// label window of an easy instance (DESIGN.md §4.3): of the colour's current list, the tiles whose lowest active label is
// within PUSH_WINDOW of the list's lowest go to win_items; the other tiles with an active voxel move to the colour's next
// list, the rest leave the lists -- or wait on the next list too while the labels are capped.  Returns the list to push now.
int window_filter(mgc_graph* g, int color, int a, WorkList* now)
{
    const WorkList cur = pl(g, color, a);
    *now = WorkList{g->win_items, g->win_ctl + WIN_NOW};
    CK(cudaMemsetAsync(g->win_ctl + WIN_GMIN, 0x7f, sizeof(int), g->stream));      // above every label
    CK(cudaMemsetAsync(g->win_ctl + WIN_NOW, 0, sizeof(int), g->stream));
    k_window_min<double><<<g->n_ctas * 2, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S, lazy_cmat(g), g->caps_tin, cur, g->win_tmin, g->win_ctl);
    k_window_split<<<g->n_ctas, 256, 0, g->stream>>>(cur, g->win_tmin, lazy_cmat(g), g->pflag, *now, pl(g, color, 1 - a),
                                                     g->drop_items, g->win_ctl, g->labels_capped ? 1 : 0);
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    return MGC_OK;
}

int push_color(mgc_graph* g, int color)
{
    g->flow_started = true;
    const int a = g->pl_sel[color], oa = g->pl_sel[1 - color];
    WorkList cur = pl(g, color, a);
    if (g->sweep_mode == 0 && g->nd == 3 && !g->slab) {
        const int rc = window_filter(g, color, a, &cur);
        if (rc) return rc;
    }
    if (g->caps_lazy) {
        // the pushers are the listed tiles, the receivers of cross-face flow their face neighbours: materialise those.  A
        // hard instance (sweeps at every relabel) pushes through most of the lattice: everything at once, then no more
        const int rc = g->sweep_mode == 1 ? push_state_all(g) : caps_launch(g, cur);
        if (rc) return rc;
    }
    CK(cudaMemsetAsync(cursor(g), 0, sizeof(int), g->stream));
    const int capped = g->labels_capped ? 1 : 0;
    if (g->nd == 4) {
        k_push_tile4<double><<<g->n_ctas, T4_VOX, 0, g->stream>>>(g->L, g->TL4, g->S, g->smask, g->iters_now, g->pflag, cur,
                                                                  cursor(g), pl(g, color, 1 - a), pl(g, 1 - color, oa));
    } else if (g->use_tma) {
        const size_t smem = 2 * TMA_STAGE_BYTES + 6 * TILE_VOX * sizeof(double) + 1024 * sizeof(int) + 64;
        k_push_tile_tma<double><<<g->n_ctas, TILE_VOX, smem, g->stream>>>(g->L, g->TL, g->S, g->maps, g->iters_now, g->pflag,
                                                                          cur, cursor(g), pl(g, color, 1 - a),
                                                                          pl(g, 1 - color, oa), capped);
    } else
    k_push_tile<double><<<g->n_ctas, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S, g->iters_now, g->pflag, cur,
                                                               cursor(g), pl(g, color, 1 - a), pl(g, 1 - color, oa), capped);
    CK(cudaMemsetAsync(g->d_tcount + 2 + color * 2 + a, 0, sizeof(int), g->stream));   // consumed list is empty again
    g->pl_sel[color] = 1 - a;
    g->st.kernel_launches++;
    return MGC_OK;
}

// `passes` two-colour passes: colour 0's list, then colour 1's
int push_passes(mgc_graph* g, int passes)
{
    for (int p = 0; p < passes; ++p) {
        int rc = push_color(g, 0);
        if (rc) return rc;
        rc = push_color(g, 1);
        if (rc) return rc;
    }
    g->st.push_sweeps += passes;
    CK(cudaGetLastError());
    return MGC_OK;
}
}  // namespace

int push_tiles(mgc_graph* g, int passes)
{
    Nvtx range("mgc:push_passes");
    cudaEventRecord(g->ev[2], g->stream);
    int rc = push_passes(g, passes);
    if (rc) return rc;
    if (g->slab) return MGC_OK;      // slabs are stepped asynchronously: no per-call timing synchronisation
    cudaEventRecord(g->ev[3], g->stream);
    CK(cudaEventSynchronize(g->ev[3]));
    { float ms = 0; cudaEventElapsedTime(&ms, g->ev[2], g->ev[3]); g->st.ms_push += (double)ms - caps_resolve(g); }
    return MGC_OK;
}

// active voxels, counted exactly over the two pending push lists (a superset of the tiles that can hold one)
int count_active_tiles_enqueue(mgc_graph* g, unsigned long long* dst)
{
    CK(cudaMemsetAsync(dst, 0, sizeof(unsigned long long), g->stream));
    if (g->nd == 4) {
        for (int color = 0; color < 2; ++color)
            k_count_active_tiles4<double><<<g->n_ctas * 2, T4_VOX, 0, g->stream>>>(g->L, g->TL4, g->S, pl(g, color, g->pl_sel[color]), dst);
        g->st.kernel_launches += 2;
    } else {
        k_count_active_tiles2<double><<<g->n_ctas * 2, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S, lazy_cmat(g), g->caps_tin,
                                                                                 pl(g, 0, g->pl_sel[0]), pl(g, 1, g->pl_sel[1]), dst);
        g->st.kernel_launches++;
    }
    CK(cudaGetLastError());
    return MGC_OK;
}

int count_active_tiles(mgc_graph* g, int64_t* out)
{
    int rc = count_active_tiles_enqueue(g, g->d_count);
    if (rc) return rc;
    unsigned long long c = 0;
    CK(cudaMemcpyAsync(&c, g->d_count, sizeof(c), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    *out = (int64_t)c;
    g->st.active_last = (int64_t)c;
    return MGC_OK;
}

namespace {
// MEDPY_GC_DEBUG=1: device-side invariants; `after` = compare flow conservation with the excess recorded before the solve
int debug_invariants(mgc_graph* g, bool after)
{
    if (!g->debug_checks) return MGC_OK;
    { int rc0 = push_state_all(g); if (rc0) return rc0; }
    double* d = g->d_scalars + 4;        // [4] excess, [5] absorbed, [6] violations
    CK(cudaMemsetAsync(d, 0, 3 * sizeof(double), g->stream));
    if (g->nd == 3) k_debug_invariants<3, double, true><<<nblocks(g), 256, 0, g->stream>>>(g->L, g->S, d);
    else            k_debug_invariants<4, double, false><<<nblocks(g), 256, 0, g->stream>>>(g->L, g->S, d);
    double h[3] = {0, 0, 0};
    CK(cudaMemcpyAsync(h, d, sizeof(h), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    if (h[2] != 0.0) {
        g->err = "debug check: " + std::to_string((long long)h[2]) + " invariant violation(s) (negative capacity / excess, absorbed flow out of range or stale residual mask)";
        return MGC_E_STATE;
    }
    if (!after) { g->debug_excess0 = h[0] + h[1]; return MGC_OK; }
    const double scale = fabs(g->debug_excess0) > 1.0 ? fabs(g->debug_excess0) : 1.0;
    if (!g->slab && !(fabs(h[0] + h[1] - g->debug_excess0) <= 1e-9 * scale)) {
        char buf[200];
        snprintf(buf, sizeof(buf), "debug check: flow not conserved: excess %.17g + absorbed %.17g != initial %.17g", h[0], h[1], g->debug_excess0);
        g->err = buf;
        return MGC_E_STATE;
    }
    return MGC_OK;
}

int solve_tiles(mgc_graph* g)
{
    int rc = materialise_zeros(g);
    if (rc) return rc;
    if (!g->state_init) {
        rc = init_tiles(g);
        if (rc) return rc;
    }
    if (g->win_ctl) CK(cudaMemsetAsync(g->win_ctl + WIN_DEFERRED, 0, 2 * sizeof(int), g->stream));    // per-solve window counts
    // One host synchronisation per round: relabel (reset + BFS), stop test and the previous round's push passes are all
    // enqueued back to back; the host waits once, reads the active count and the CUDA-event times of both phases and
    // decides.  The stop test of the FIRST round is skipped (a graph that was just built almost always has active
    // voxels; if it has none the push pass is a no-op and the next round's test ends the solve).
    int passes = g->passes0;
    int64_t rounds = 0;
    bool push_open = false;
    int passes_done = 0;
    unsigned long long active_fallback = 0;
    unsigned long long* h_active = g->h_bad ? (unsigned long long*)g->h_bad + 1 : &active_fallback;      // pinned
    for (;;) {
        cudaEventRecord(g->ev[2], g->stream);
        {
            Nvtx range("mgc:global_relabel");
            rc = relabel_tiles_begin(g);
            if (rc) return rc;
            int any = 0;
            rc = relabel_tiles_run(g, &any, false, rounds == 0 && g->skip_first_test);
            if (rc) return rc;
        }
        cudaEventRecord(g->ev[3], g->stream);
        g->st.global_relabels++;
        bool relp_copy = false;
        rc = relabel_passes_fetch(g, &relp_copy);
        if (rc) return rc;
        const bool test = rounds > 0 || !g->skip_first_test;
        if (test) {
            rc = count_active_tiles_enqueue(g, g->d_count);
            if (rc) return rc;
            CK(cudaMemcpyAsync(h_active, g->d_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, g->stream));
        }
        CK(cudaEventSynchronize(g->ev[3]));
        if (test || relp_copy) CK(cudaStreamSynchronize(g->stream));
        float ms = 0;
        const double caps_ms = caps_resolve(g);      // materialiser launches inside the push span: timed apart
        if (g->init_timed) {          // k_init_tile of the per-term path: its events are reused for the push spans below
            if (cudaEventElapsedTime(&ms, g->ev[4], g->ev[5]) == cudaSuccess) g->st.ms_init = ms;
            g->init_timed = false;
        }
        cudaEventElapsedTime(&ms, g->ev[2], g->ev[3]);
        const double t_rel = ms;
        g->st.ms_relabel += ms;
        const int relp = relabel_passes_collect(g);
        if (rounds == 0) { g->st.ms_relabel_first += ms; g->st.relabel_passes_first += relp; }
        double t_pass = 0.0;
        if (push_open) {
            cudaEventElapsedTime(&ms, g->ev[4], g->ev[5]);
            const double push_ms = (double)ms - caps_ms;
            g->st.ms_push += push_ms;
            t_pass = push_ms / (passes_done > 0 ? passes_done : 1);
            push_open = false;
            // next round: at most double, and no more push time than one global relabel costs (measured, not guessed):
            // easy instances keep relabelling often, hard ones (long BFS, cheap passes) push longer between relabels
            int want = t_pass > 1e-4 ? (int)(t_rel / t_pass + 0.999) : passes * 2;
            if (want < 1) want = 1;
            if (want > passes * 2) want = passes * 2;
            passes = want > g->passes_max ? g->passes_max : want;
        }
        if (test) {
            g->st.active_last = (int64_t)*h_active;
            if (*h_active == 0ull) break;
        }
        if (++rounds > g->max_rounds) FAIL(MGC_E_NOCONV, "push-relabel did not converge within the round cap");
        g->iters_now = rounds == 1 ? g->tile_iters_first : g->tile_iters;
        {
            Nvtx range("mgc:push_passes");
            cudaEventRecord(g->ev[4], g->stream);
            rc = push_passes(g, passes);
            if (rc) return rc;
            cudaEventRecord(g->ev[5], g->stream);
            passes_done = passes;
            push_open = true;
        }
    }
    g->init_timed = false;       // ev[4..5] were reused for the push spans
    return MGC_OK;
}
}  // namespace

int readout(mgc_graph* g, double* energy_part)
{
    Nvtx range("mgc:readout");
    // clean tiles hold the reset labels while no sweep has lowered labels unmarked (the partial reset relies on the same)
    const bool clean = g->nd == 3 && !g->slab && g->TL.dflag && g->sweep_mode != 1 && g->L.dim[2] % 4 == 0;
    if (clean) k_readout<double, true, true><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, g->mask_dev, g->partials, g->TL.dflag,
                                                                                g->TL.nt[1], g->TL.nt[2]);
    else if (g->nd == 3) k_readout<double, true><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, g->mask_dev, g->partials);
    else                 k_readout<double, false><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, g->mask_dev, g->partials);
    CK(cudaMemsetAsync(g->d_scalars + 1, 0, sizeof(double), g->stream));
    sum_partials(g, g->partials, rblocks(g), g->d_scalars + 1);
    g->st.kernel_launches += 2;
    double sc[2] = {0, 0};
    int fl[5] = {0, 0, 0, 0, 0};     // d_flags[3..7]: [0] tiles materialised, [4] build blocks refused
    int win[2] = {0, 0};             // WIN_DEFERRED, WIN_DROPPED of this solve
    CK(cudaMemcpyAsync(sc, g->d_scalars, sizeof(sc), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaMemcpyAsync(fl, g->d_flags + 3, sizeof(fl), cudaMemcpyDeviceToHost, g->stream));
    if (g->win_ctl) CK(cudaMemcpyAsync(win, g->win_ctl + WIN_DEFERRED, sizeof(win), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    g->st.flow_const = sc[0];
    g->st.tiles_materialised = fl[0];
    g->st.build_blocks_refused = fl[4];
    g->st.tiles_deferred += win[0];
    g->st.tiles_dropped += win[1];
    *energy_part = sc[0] + sc[1];
    if (g->init_timed) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, g->ev[4], g->ev[5]) == cudaSuccess) g->st.ms_init = ms;
        g->init_timed = false;
    }
    return MGC_OK;
}

namespace {
struct Timer {
    mgc_graph* g;
    double* acc;
    Timer(mgc_graph* g_, double* acc_) : g(g_), acc(acc_) { cudaEventRecord(g->ev[0], g->stream); }
    void stop_sync()
    {
        cudaEventRecord(g->ev[1], g->stream);
        cudaEventSynchronize(g->ev[1]);
        float ms = 0;
        cudaEventElapsedTime(&ms, g->ev[0], g->ev[1]);
        *acc += ms;
    }
};
}  // namespace

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

int mgc_maxflow(mgc_graph* g, double* energy)
{
    if (!g) return MGC_E_ARG;
    if (g->slab) FAIL(MGC_E_STATE, "z-slab handles are stepped with mgc_slab_*");
    CK(cudaSetDevice(g->device));
    if (g->solved) { if (energy) *energy = g->energy; return MGC_OK; }
    { int rc0 = check_pending(g); if (rc0) return rc0; }
    resolve_term_span(g);
    {
        Timer t(g, &g->st.ms_solve);
        int rc = warm_prepare(g); if (rc) return rc;
        if (g->debug_checks) {
            rc = materialise_zeros(g); if (rc) return rc;
            if (!g->state_init) { rc = init_tiles(g); if (rc) return rc; }
            rc = debug_invariants(g, false); if (rc) return rc;
        }
        rc = solve_tiles(g);
        if (rc) return rc;
        rc = debug_invariants(g, true);
        if (rc) return rc;
        t.stop_sync();
    }
    {
        Timer t(g, &g->st.ms_readout);
        double e = 0.0;
        int rc = readout(g, &e);
        if (rc) return rc;
        g->energy = e;
        g->st.energy = e;
        t.stop_sync();
    }
    caps_resolve(g);
    g->solved = true;
    if (energy) *energy = g->energy;
    return MGC_OK;
}

}  // extern "C"
