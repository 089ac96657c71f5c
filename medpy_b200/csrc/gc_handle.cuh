// gc_handle.cuh -- the lattice handle (struct mgc_graph) and what the units of its C ABI share.  Host-side and internal;
// the public ABI is include/medpy_b200_graphcut.h.  The units:
//   gc_api.cu        device and pinned pools, input staging, create / destroy / reset, the per-term entry points, the
//                    gradient, the getters
//   gc_build_api.cu  the fused graph build (mgc_build_voxel_graph)
//   gc_solve.cu      the lazy push state, the tile-solver driver, mgc_maxflow
//   gc_fold.cu       the folds into the residual state (seeds, t-links, n-links)
//   gc_slab.cu       z-slab stepping and the NCCL slab solve
//   gc_batch.cu      batches of independent images: create, build, per-image constants and energies
// Each kernel is compiled into exactly one of them: a unit includes the kernel-only header of the kernels it launches
// (gc_<unit>_kernels.cuh, gc_persist.cuh, gc_sweep.cuh, ...), and k_sum_partials, which several launch, is behind
// sum_partials().  Process-wide state (pools, the cub launch counts, the NCCL binding) is defined in one unit each.
#pragma once
#include "gc_host.hpp"
#include "gc_common.cuh"
#include "gc_terms.cuh"
#include "gc_tiles.cuh"
#include "gc_tiles4.cuh"
#include "gc_tma.cuh"
#include "gc_build.cuh"

#include <nccl.h>
#include <nvtx3/nvToolsExt.h>

#include <cstdint>
#include <string>
#include <type_traits>
#include <vector>

struct Buf {
    void* p = nullptr;
    size_t bytes = 0;
};

struct mgc_graph {
    int device = 0;
    int user_ndim = 0;
    int nd = 3;             // canonical axes
    int shift = 0;          // canonical axis = user axis + shift
    int64_t user_shape[4] = {1, 1, 1, 1};
    Lattice L{};
    bool slab = false;
    bool ghost_lo = false, ghost_hi = false;
    int64_t global_dim0 = 0, z0 = 0, z1 = 0;

    State<double> S{};
    std::vector<Buf> owned_bufs;       // everything allocated from the pool
    Buf scratch[5];                    // staged (contiguous) copies of input arrays: 0 prob/src, 1 fg/snk, 2 image, 4 bg
    Buf raw;                           // raw span of a strided host array
    uint8_t* mask_dev = nullptr;
    double* partials = nullptr;        // per-block partial sums
    unsigned n_partials = 0;
    void* minmax_buf = nullptr;        // 3 x 1024 partial min/max/absmax
    double* d_scalars = nullptr;       // [0] flow_const, [1] absorbed, [2..3] minmax out
    int* d_flags = nullptr;            // [0] bad weight, [3] tiles materialised, [4..5] materialiser claim count / cursor,
                                       // [6] blocks refused by the last lean build launch, [7] ... by the whole build
    unsigned long long* d_count = nullptr;
    int64_t device_bytes = 0;

    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaEvent_t ev[6] = {};
    // host -> device staging runs on its own stream so that the copy of the next term overlaps the kernel of the
    // previous one; the host only waits for the COPY (its pointer is borrowed for the call), never for the kernel
    cudaStream_t up_stream = nullptr;
    cudaEvent_t ev_up = nullptr;
    cudaEvent_t ev_slot[5] = {};       // main-stream point after which a staging slot may be overwritten (3 = raw span)
    bool slot_used[5] = {false, false, false, false, false};
    cudaEvent_t ev_chunk[2] = {};      // chunked fused build: upload stream -> main stream hand-over (alternating)
    cudaEvent_t ev_terms[2] = {};      // span of the term kernels since the last reset
    bool terms_open = false;
    // deferred weight verdict (MGC_OPT_DEFER_WEIGHT_CHECK)
    bool defer_check = false;
    bool bad_pending = false;
    int* h_bad = nullptr;              // pinned
    cudaEvent_t ev_bad = nullptr;
    cudaEvent_t ev_b[2] = {};          // the boundary kernel alone

    bool init_timed = false;           // ev[4..5] bracket the last k_init_tile
    bool boundary_timed = false;       // ev[2..3]... the boundary kernel's own events (ev_b) await reading
    bool caps_fresh = true;            // capacity arrays not written yet since create/reset (hold garbage)
    bool tr_fresh = true;              // same for tr[]
    bool state_init = false;
    bool flow_started = false;         // push kernels have run since the last reset: cap[] holds residuals, not the terms
    bool debug_checks = false;         // MEDPY_GC_DEBUG=1: device-side invariant + flow-conservation checks around every solve
    double debug_excess0 = 0.0;        // clamped source excess the solve started from
    bool fuse_build = true;            // mgc_build_voxel_graph uses the single-pass k_build_tile (MEDPY_GC_FUSE=0: four passes)
    // lazy exponential build staged by TMA: every block goes to k_build_refused, none is streamed by k_build_lean
    // (MEDPY_GC_BUILD_REFUSE_ALL=1; for tests that compare the two paths on one volume)
    bool build_refuse_all = false;
    int* build_refused = nullptr;      // blocks k_build_lean refused (indices into its grid), one entry per build block
    // lazy push state: the fused 3-D build writes no capacity planes, no tr and no excess; k_caps_tiles computes them per
    // tile, from copies of the build's inputs, for the tiles the push path reaches (MEDPY_GC_LAZY_CAPS=0: the build
    // writes them all)
    bool lazy_caps = true;
    bool caps_lazy = false;            // the last build was lazy and some tiles are not materialised yet
    // the last build was the lazy fused build and nothing else changed the terms since: mgc_add_seeds / mgc_remove_seeds /
    // mgc_add_tweights_warm may fold t-link calls into the residual state.  Unlike caps_lazy this stays true once every
    // tile is materialised (hard instances).
    bool lazy_built = false;
    // MGC_OPT_WARM: the other tile-solver handles (eager fused build, per-term path, 4-D lattices, z-slabs) record their
    // residual source capacities in tr at the first solve, which lets the same folds work on them (gc_seeds.cuh).  Kept
    // across mgc_reset, like defer_check.
    bool warm_opt = false;
    bool warm_state = false;           // tr holds BK's residual source capacity: recorded since the last init
    int* cmat = nullptr;              // per tile: push state materialised since the last lazy build
    int* caps_list = nullptr;          // tiles claimed by the current materialiser launch
    // The inputs below (with caps_P and caps_tin) live as long as the handle's last lazy build: besides the materialiser,
    // the seed folds depend on them -- they recompute a seeded voxel's capacities before any flow from caps_img to know
    // the source flow its state already holds (gc_seeds.cuh).  Dropping them breaks the warm re-solve.
    Buf img_copy;                      // the image the lazy build saw, in its own dtype (a staging buffer of the build, or
                                       // a copy its kernel wrote)
    Buf prob_copy;                     // ... its probability map, in its own dtype
    Buf mark_planes[2];                // ... its fg / bg markers as bit planes (LazyTin)
    // what the materialiser and the folds read: img_copy, or the caller's device image (MGC_OPT_KEEP_DEVICE_INPUTS);
    // caps_tin.prob likewise.  Forgotten by mgc_reset, the per-term calls and every build that is not lazy.
    const void* caps_img = nullptr;
    bool keep_device_inputs = false;   // MGC_OPT_KEEP_DEVICE_INPUTS
    Buf fold_buf;                      // folds: control words, inputs, keys, runs, touched tiles, items, cub scratch
    cudaEvent_t ev_fold[4] = {};       // spans of the grouping and of claim + fold + list fix-up
    int caps_dtype = MGC_F32;
    BoundaryParams caps_P{};           // the boundary term of the lazy build
    LazyTin caps_tin{};                // its t-link terms
    std::vector<cudaEvent_t> caps_ev;  // start / end of every materialiser launch since the last caps_resolve
    size_t caps_ev_used = 0;
    int build_chunks = 8;              // host inputs: z-chunks whose upload overlaps the build of the previous chunk
    bool solved = false;
    bool has_nlinks = false;
    double energy = 0.0;
    std::vector<uint8_t> host_mask;
    bool host_mask_valid = false;

    // tile solver (3-D lattices)
    Tiles TL{};
    Tiles4 TL4{};                      // 4-D lattices: 4x4x8x4 tiles (gc_tiles4.cuh)
    uint8_t* smask = nullptr;          // 4-D: residual sink link flag (the 8 arc bits fill rmask)
    int* pflag = nullptr;              // push: tile is already on the list its colour consumes next
    int* rflag = nullptr;              // relabel: tile is already on the next relabel list
    int* rl_items[2] = {nullptr, nullptr};     // relabel worklists (double buffered)
    int* pl_items[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // push worklists [colour][buffer]
    int* d_tcount = nullptr;           // [0..1] relabel counts, [2..5] push counts [colour*2+buffer], [8] cursor
    int pl_sel[2] = {0, 0};            // buffer each colour consumes next
    // label window of the push passes on easy instances (k_window_min / k_window_split): per list position the lowest
    // active label of the tile, the list pushed now, control words (WIN_*), the tiles dropped before they were materialised
    int* win_tmin = nullptr;
    int* win_items = nullptr;
    int* win_ctl = nullptr;
    int* drop_items = nullptr;
    bool labels_fresh = false;         // labels + relabel list 0 come straight from k_init_tile
    int n_ctas = 264;                  // persistent CTAs per tile-kernel launch
    int coop_bfs_grid = 0;             // co-resident CTAs of k_bfs_coop / k_bfs_coop4
    bool use_tma = false;              // push kernel stages its tile planes with TMA (gc_tma.cuh)
    PushMaps maps{};                   // tensor maps of cap[0..5] and excess
    int tile_iters = 8;                // synchronous push/relabel rounds per tile visit
    int tile_iters_first = 4;          // ... in the first round after init (mostly stranded excess drains locally)
    int iters_now = 8;
    int passes0 = 1, passes_max = 32;  // two-colour passes per round: starts at passes0, at most doubles per round
    // directional line sweeps in front of the worklist BFS (gc_sweep.cuh): used when more than 1/sweep_frac of the
    // tiles are waiting for labels (hard instances: the sink is far from most of the lattice)
    bool skip_first_test = true;       // MEDPY_GC_FIRST_TEST=1 restores the stop test of the first round
    // label cap of a relabel that no stop test reads (the first of an easy solve, DESIGN.md §4.3): its labels only feed
    // the label window of round 1's push passes.  MEDPY_GC_FIRST_CAP=0 keeps it exact, =N caps it at N (N >= 2)
    int first_cap = FIRST_RELABEL_CAP;
    bool labels_capped = false;        // the last global relabel stopped at first_cap: HINF means "deeper than the cap"
    int relp_last = 0;                 // BFS passes of the last relabel_tiles_run ...
    bool relp_pending = false;         // ... still in the control block (cooperative BFS, not read back yet)
    int sweep_mode = -1;               // decided at the first relabel of a solve: 1 = hard instance (sweep at every relabel), 0 = worklist BFS only
    bool use_sweeps = true;
    int sweep_frac = 8;                // sweep when pending tiles > ntiles / sweep_frac
    int sweep_rounds_min = 1;          // rounds before the first fixed-point check (MEDPY_GC_SWEEP_MIN_ROUNDS); one round +
                                       // check + worklist BFS is the usual sequence
    int sweep_rounds_max = 4;
    int sweep_done_frac = 16;          // hand over to the worklist BFS when violating tiles <= ntiles / sweep_done_frac

    // tuning
    int64_t max_rounds = 100000;

    // z-slab solve inside the library (mgc_slab_comm_init / mgc_slab_solve): NCCL communicator of the slab ranks, border
    // message buffers [labels int32 | pad | flow float64] per neighbour and direction, stop-test scalars
    ncclComm_t comm = nullptr;
    int comm_rank = 0, comm_world = 1;
    char* msg[4] = {nullptr, nullptr, nullptr, nullptr};   // send_lo, send_hi, recv_lo, recv_hi (device)
    size_t msg_h_bytes = 0, msg_bytes = 0;
    long long* d_stat = nullptr;       // [changed in round A, changed in round B, active voxels] (device, all-reduced in place)
    long long* h_stat = nullptr;       // pinned mirror
    double* d_esum = nullptr;          // energy all-reduce
    int64_t slab_exchanges = 0, slab_relabel_rounds = 0, slab_push_passes = 0, slab_global_relabels = 0;
    // per-phase device time of the last mgc_slab_solve (CUDA events on the stream, resolved at the end of the solve):
    // [0] local BFS (reset + relax), [1] border exchanges (pack + NCCL send/recv + unpack), [2] stop test (count + all-reduce),
    // [3] push passes, [4] read-out + energy all-reduce; [5] = host time blocked in stream synchronisations (ms)
    std::vector<cudaEvent_t> ph_events;
    std::vector<int> ph_kind;
    size_t ph_used = 0;
    double slab_phase_ms[6] = {0, 0, 0, 0, 0, 0};

    // batch of independent images stacked along axis 0 (mgc_create_batch, DESIGN.md §3.1; L.zper planes per image)
    int64_t batch = 0;                 // images (0: not a batch handle)
    int batch_ndim = 0;                // dimensions of one image (1..3)
    int batch_chunks = 1;              // blocks per image of the per-image reductions
    bool batch_built = false;          // the state comes from mgc_build_voxel_batch (cleared by mgc_reset); with
                                       // MGC_OPT_WARM the warm folds edit it and its per-image constants (batch_warm)
    double* batch_buf = nullptr;       // [B] term constants (BoundaryParams::ktab) | [B] add_tweights constants |
                                       // [B] energies | [2B] min / max read-outs | [B * batch_chunks] partials
    std::vector<double> batch_k_host;  // the term constants of the next build (NaN: M computed on the device)

    mgc_stats st{};
    std::string err;
};

// ---- gc_api.cu ------------------------------------------------------------------------------------------
extern thread_local std::string g_create_error;   // mgc_last_error(nullptr): the last failure without a handle
size_t dtype_size(int dt);
int alloc_buf(mgc_graph* g, size_t bytes, void** out);
int ensure_scratch(mgc_graph* g, Buf& b, size_t bytes);
int upload(mgc_graph* g, void* dst, const void* src, size_t bytes, int slot);
void slots_release(mgc_graph* g, unsigned mask);
int stage_input(mgc_graph* g, const mgc_array* a, int slot, const void** out);
void sum_partials(mgc_graph* g, const double* partials, unsigned n, double* out);
void resolve_term_span(mgc_graph* g);
int check_pending(mgc_graph* g);
int boundary_params(mgc_graph* g, int kind, int dtype, const void* img, double sigma, const double* spacing, double norm, BoundaryParams* out);
int minmax_dtype(mgc_graph* g, int dtype, const void* img, unsigned n, double* out);

// ---- gc_solve.cu ----------------------------------------------------------------------------------------
typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
tmap_encode_fn tensor_map_encoder();
int tile_solver_options(mgc_graph* g);
void push_tma_setup(mgc_graph* g);
int materialise_zeros(mgc_graph* g);
int caps_launch(mgc_graph* g, WorkList wl);
int push_state_all(mgc_graph* g);
double caps_resolve(mgc_graph* g);
int dirty_clear(mgc_graph* g);
int init_tiles(mgc_graph* g);
int relabel_tiles_begin(mgc_graph* g);
int relabel_tiles_run(mgc_graph* g, int* any, bool want_any = true, bool first = false);
int push_tiles(mgc_graph* g, int passes);
int count_active_tiles_enqueue(mgc_graph* g, unsigned long long* dst);
int count_active_tiles(mgc_graph* g, int64_t* out);
int readout(mgc_graph* g, double* energy_part);

// ---- gc_build_api.cu ------------------------------------------------------------------------------------
int voxel_build(mgc_graph* g, const mgc_voxel_terms* t);

// ---- gc_batch.cu ----------------------------------------------------------------------------------------
int batch_constants(mgc_graph* g, int dtype, const void* d_img, BoundaryParams* P);
int batch_tconst(mgc_graph* g, const BuildArgs& A);
void batch_sum(mgc_graph* g, const double* partials, unsigned n, double* out);
int batch_view(mgc_graph* g, const mgc_array* a, int slot, mgc_array* out);
size_t batch_fold_chunks(int max_count);
int batch_fold_const(mgc_graph* g, const unsigned* vox, int vstride, const int* count, int max_count, const double* dk,
                     double* part, int* span);

// ---- gc_fold.cu -----------------------------------------------------------------------------------------
int warm_prepare(mgc_graph* g);

// ---- gc_slab.cu -----------------------------------------------------------------------------------------
void slab_comm_release(mgc_graph* g);

// ---- inline helpers ---------------------------------------------------------------------------------------
// The one refusal of every call a batch handle does not take: MGC_E_STATE with this message (else MGC_OK).  The warm
// folds take it too, unless the handle has MGC_OPT_WARM and a state from mgc_build_voxel_batch (batch_warm).
inline int batch_refused(const mgc_graph* g)
{
    if (!g->batch) return MGC_OK;
    const_cast<mgc_graph*>(g)->err = "batch handles take their terms from mgc_build_voxel_batch only: the per-term calls "
                                     "and the z-slab calls are not available on them, and the warm edits need "
                                     "MGC_OPT_WARM set before mgc_build_voxel_batch";
    return MGC_E_STATE;
}

// a batch handle whose state the warm folds may edit: MGC_OPT_WARM was set, and the state comes from the batch build
// (the per-image constants exist and stay valid until mgc_reset)
inline bool batch_warm(const mgc_graph* g) { return g->batch && g->warm_opt && g->batch_built; }

// NVTX range per phase (build / relabel / push / readout / exchange): visible in nsys / ncu timelines, a no-op without a
// profiler attached (SURVEY.md §5.1)
struct Nvtx {
    explicit Nvtx(const char* name) { nvtxRangePushA(name); }
    ~Nvtx() { nvtxRangePop(); }
};

inline unsigned nblocks(const mgc_graph* g) { return (g->L.n + 255u) / 256u; }
// grid of the grid-stride reduction kernels (partials per launch)
inline unsigned rblocks(const mgc_graph* g) { const unsigned nb = nblocks(g); return nb < REDUCE_BLOCKS ? nb : REDUCE_BLOCKS; }

inline WorkList rl(mgc_graph* g, int i) { return WorkList{g->rl_items[i], g->d_tcount + i}; }
inline WorkList pl(mgc_graph* g, int color, int buf) { return WorkList{g->pl_items[color][buf], g->d_tcount + 2 + color * 2 + buf}; }
inline int* cursor(mgc_graph* g) { return g->d_tcount + 8; }

// MGC_OPT_WARM applies: a tile-solver handle whose state does not come from the lazy fused build (z-slabs included: they
// build eagerly, and their folds apply only what the slab owns, DESIGN.md §4.6)
inline bool warm_wanted(const mgc_graph* g) { return g->warm_opt && !g->lazy_built; }

// term kernels are not synchronised one by one: their span on the stream is measured between the first term after a
// reset and the last term before the solve, and read when the solve synchronises anyway
struct TermSpan {
    mgc_graph* g;
    explicit TermSpan(mgc_graph* g_) : g(g_)
    {
        if (!g->terms_open) { cudaEventRecord(g->ev_terms[0], g->stream); g->terms_open = true; }
    }
    void stop(unsigned slot_mask) { slots_release(g, slot_mask); cudaEventRecord(g->ev_terms[1], g->stream); }
};

// ---- lazy push state: k_caps_tiles over a push worklist or over every tile -----------------------------------------
// The instantiation of the lazy build's boundary term, as a tag type: E = the image dtype, FN / USE_MAX / SPACING fixed
// (>= 0) or read from BoundaryParams at run time (-1).
template <typename E_, int FN_, int USE_MAX_, int SPACING_>
struct LazyTerm {
    using E = E_;
    static constexpr int FN = FN_, USE_MAX = USE_MAX_, SPACING = SPACING_;
};

// f(LazyTerm<...>{}) for the handle's caps_dtype / caps_P: <1, 1, 0> and <1, 0, 0> for float images with the exponential
// term without spacing, <-1, -1, -1> for every other case.  k_caps_tiles and the lazy folds are instantiated here only.
template <typename F>
void lazy_dispatch(const mgc_graph* g, F&& f)
{
    auto by_dtype = [&](auto e) {
        using E = decltype(e);
        const BoundaryParams& P = g->caps_P;
        if constexpr (!std::is_integral<E>::value) {
            if (P.fn == 1 && P.inv_spacing_on == 0.0) {
                if (P.use_max) f(LazyTerm<E, 1, 1, 0>{});
                else           f(LazyTerm<E, 1, 0, 0>{});
                return;
            }
        }
        f(LazyTerm<E, -1, -1, -1>{});
    };
    switch (g->caps_dtype) {
        case MGC_F32: by_dtype(float{}); break;
        case MGC_F64: by_dtype(double{}); break;
        case MGC_U8: by_dtype(uint8_t{}); break;
        case MGC_I16: by_dtype(int16_t{}); break;
        default: by_dtype(int32_t{}); break;
    }
}
