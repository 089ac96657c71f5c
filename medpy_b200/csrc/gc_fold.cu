// gc_fold.cu -- folds into the residual state of a solved lattice handle (gc_handle.cuh): mgc_add_seeds /
// mgc_remove_seeds / mgc_add_tweights_warm / mgc_add_nweights*_warm / mgc_remove_nweights*_warm, and warm_prepare, which
// records the residual source capacities of an MGC_OPT_WARM handle.
#include "gc_handle.cuh"
#include "gc_nlinks_remove.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <chrono>
#include <functional>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>
#include <vector>

// MGC_OPT_WARM: put tr into BK's representation before the first push (a no-op where it is already, or where the option
// does not apply).  The per-term path does it in k_init_tile; after the eager fused build, which wrote the state before
// the option could be read, k_warm_convert does it in a pass of its own (8 B of tr read per voxel, plus the six capacities
// and the write of tr where tr > 0).
int warm_prepare(mgc_graph* g)
{
    if (!warm_wanted(g) || g->warm_state) return MGC_OK;
    if (g->flow_started) FAIL(MGC_E_STATE, "MGC_OPT_WARM was set after the first solve: reset() the graph and rebuild it");
    // no push has run: a 4-D init (the only other source of 4-D state) is simply run again, recording this time
    if (!g->state_init || g->nd == 4) {
        int rc = materialise_zeros(g);
        if (rc) return rc;
        return init_tiles(g);
    }
    Nvtx range("mgc:warm_convert");
    unsigned grid = nblocks(g);
    if (grid > (unsigned)g->n_ctas * 8u) grid = (unsigned)g->n_ctas * 8u;
    k_warm_convert<<<grid, 256, 0, g->stream>>>(g->L, g->S);
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    g->warm_state = true;
    g->flow_started = true;
    return MGC_OK;
}

namespace {

// f(A) with the residual access of a fold on this handle (gc_seeds.cuh): LazyResidual with the lazy build's instantiation,
// or (eager: an MGC_OPT_WARM handle) EagerResidual<3> / <4>; batch handles (3-D lattices) take the BATCH variants
template <typename F>
void residual_dispatch(const mgc_graph* g, bool eager, F&& f)
{
    if (eager) {
        if (g->nd == 4)     f(EagerResidual<4>{g->S, g->smask});
        else if (g->batch)  f(EagerResidual<3, true>{g->S, g->smask});
        else                f(EagerResidual<3>{g->S, g->smask});
        return;
    }
    lazy_dispatch(g, [&](auto t) {
        using T = decltype(t);
        using E = typename T::E;
        // a batch replays each voxel's capacities with its image's constants and stores each entry's constant change;
        // single handles keep the plain kernels
        if (g->batch) f(LazyResidual<E, T::FN, T::USE_MAX, T::SPACING, true>{g->L, g->S, (const E*)g->caps_img, g->caps_P});
        else          f(LazyResidual<E, T::FN, T::USE_MAX, T::SPACING, false>{g->L, g->S, (const E*)g->caps_img, g->caps_P});
    });
}

// f(std::bool_constant<SLAB>{}, own): the grouping and n-link kernels of a z-slab handle (SLAB = true) take its owned
// voxels and drop what lies in its ghost planes (SlabOwn, gc_seeds.cuh); every other handle keeps the kernels without
// the test
template <typename F>
void slab_dispatch(const mgc_graph* g, F&& f)
{
    if (g->slab) f(std::true_type{}, SlabOwn{(unsigned)g->L.own0 * g->L.plane, (unsigned)g->L.own1 * g->L.plane, g->L.plane});
    else         f(std::false_type{}, SlabOwn{});
}

// MEDPY_GC_DEBUG=1 on a z-slab handle: after a fold the ghost planes' excess -- the outbox of flow pushed towards the
// neighbour, emptied by every exchange -- is still zero, so the next exchange sends nothing the fold made up
int slab_outbox_check(mgc_graph* g)
{
    if (!g->slab || !g->debug_checks) return MGC_OK;
    const size_t P = g->L.plane;
    std::vector<double> box(P);
    for (int side = 0; side < 2; ++side) {
        if (!(side == 0 ? g->ghost_lo : g->ghost_hi)) continue;
        const size_t ghost = side == 0 ? (size_t)(g->L.own0 - 1) * P : (size_t)g->L.own1 * P;
        CK(cudaMemcpyAsync(box.data(), g->S.excess + ghost, P * sizeof(double), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        for (double x : box)
            if (x != 0.0) FAIL(MGC_E_CUDA, "debug check: a fold left flow in a ghost plane's excess (the z-slab's outbox)");
    }
    return MGC_OK;
}

}  // namespace

// ---- folds into the residual state (mgc_add_seeds / mgc_remove_seeds / mgc_add_tweights_warm / mgc_add_nweights*_warm /
// mgc_remove_nweights*_warm)
// The cub calls of a fold's grouping: the radix sort of its keys (FOLD_SORT_KEYS: the keys alone, FOLD_SORT_PAIRS: keys
// and call indices, stable; FOLD_SCAN: no sort), then the inclusive sum of the heads.  tmp == nullptr only sizes them:
// *bytes is the larger scratch size of the two.
enum { FOLD_SORT_KEYS = 0, FOLD_SORT_PAIRS = 1, FOLD_SCAN = 2, FOLD_SORT_TAILS = 3 };
template <typename Key>
static cudaError_t fold_sort(int sort, void* tmp, size_t* bytes, Key* keys, Key* skeys, int* vals, int* svals, int n,
                             int end_bit, cudaStream_t s)
{
    size_t tb = *bytes;
    cudaError_t e = cudaSuccess;
    if constexpr (sizeof(Key) == 4)             // seeds sort 32-bit keys only
        if (sort == FOLD_SORT_KEYS) e = cub::DeviceRadixSort::SortKeys(tmp, tb, keys, skeys, n, 0, end_bit, s);
    if (sort == FOLD_SORT_PAIRS) e = cub::DeviceRadixSort::SortPairs(tmp, tb, keys, skeys, vals, svals, n, 0, end_bit, s);
    if (!tmp && sort != FOLD_SCAN) *bytes = tb;
    return e;
}

static cudaError_t fold_scan(void* tmp, size_t* bytes, int* head, int* pos, int n, cudaStream_t s)
{
    size_t tb = *bytes;
    const cudaError_t e = cub::DeviceScan::InclusiveSum(tmp, tb, head, pos, n, s);
    if (!tmp) *bytes = std::max(*bytes, tb);
    return e;
}

// Number of kernels the cub calls of a fold's grouping enqueue, so that kernel_launches counts them too.  cub decides it
// on the host from (n, end_bit) and the device; the calls are captured on a capture-only stream of the device (nothing
// runs) and the kernel nodes of the captured graph counted.  The stream lives for the process and the counts are cached,
// so a call pays only the capture of a few launches.
// `key` names the calls (device, sort kind, key size, n, end_bit); enqueue(s) issues them on the capture stream s.
static int cub_launches(mgc_graph* g, const std::tuple<int, int, int, int, int>& key,
                        const std::function<cudaError_t(cudaStream_t)>& enqueue, int* out)
{
    static std::mutex mu;
    static std::map<int, cudaStream_t> streams;
    static std::map<std::tuple<int, int, int, int, int>, int> counts;
    std::lock_guard<std::mutex> lock(mu);
    auto it = counts.find(key);
    if (it != counts.end()) { *out = it->second; return MGC_OK; }
    cudaStream_t& s = streams[g->device];
    if (!s) CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed);
    if (e == cudaSuccess) {
        const cudaError_t e2 = enqueue(s);
        e = cudaStreamEndCapture(s, &graph);
        if (e == cudaSuccess) e = e2;
    }
    size_t nn = 0;
    std::vector<cudaGraphNode_t> nodes;
    if (e == cudaSuccess) e = cudaGraphGetNodes(graph, nullptr, &nn);
    if (e == cudaSuccess) { nodes.resize(nn); e = cudaGraphGetNodes(graph, nodes.data(), &nn); }
    int k = 0;
    for (size_t i = 0; e == cudaSuccess && i < nn; ++i) {
        cudaGraphNodeType t;
        e = cudaGraphNodeGetType(nodes[i], &t);
        if (e == cudaSuccess && t == cudaGraphNodeTypeKernel) ++k;
    }
    if (graph) cudaGraphDestroy(graph);
    CK(e);
    if (counts.size() > 4096) counts.clear();
    counts[key] = k;
    *out = k;
    return MGC_OK;
}

template <typename Key>
static int fold_cub_launches(mgc_graph* g, int sort, int n, int end_bit, void* tmp, size_t tmp_bytes, Key* keys, Key* skeys,
                             int* vals, int* svals, int* head, int* pos, int* out)
{
    return cub_launches(g, std::make_tuple(g->device, sort, (int)sizeof(Key), n, end_bit), [&](cudaStream_t s) {
        size_t tb = tmp_bytes;
        const cudaError_t e1 = fold_sort(sort, tmp, &tb, keys, skeys, vals, svals, n, end_bit, s);
        tb = tmp_bytes;
        return e1 == cudaSuccess ? fold_scan(tmp, &tb, head, pos, n, s) : e1;
    }, out);
}

// The tail list of an n-link decrement fold in ascending voxel order: the first *ntails of `count` slots hold the listed
// tails in the order the atomics gave them, the rest 0xffffffff; sorted on the bits below `end_bit` = bits_for(n), the
// smallest end_bit with n < 2^end_bit, which put every voxel id below the fill.  tmp == nullptr only sizes the sort
// (*bytes).
static cudaError_t tails_sort(void* tmp, size_t* bytes, const unsigned* tails, unsigned* stails, int count, int end_bit,
                              cudaStream_t s)
{
    return cub::DeviceRadixSort::SortKeys(tmp, *bytes, tails, stails, count, 0, end_bit, s);
}

// preconditions of every fold into the residual state: the copies of the lazy fused build are what the fold reads, or
// (MGC_OPT_WARM, *eager = true) the residual source capacities the first solve records in tr on any other tile-solver
// handle, z-slabs included
static int warm_check(mgc_graph* g, bool* eager)
{
    *eager = false;
    if (g->batch && !batch_warm(g)) return batch_refused(g);
    if (!g->slab && g->lazy_built && g->state_init && g->nd == 3) return MGC_OK;
    if (warm_wanted(g)) { *eager = true; return MGC_OK; }
    if (g->slab)
        FAIL(MGC_E_STATE, "a warm re-solve of a z-slab handle needs MGC_OPT_WARM set before its first solve; reset() it and "
                          "rebuild the graph with the edits instead");
    FAIL(MGC_E_STATE, "a warm re-solve needs a lazily built 3-D handle (mgc_build_voxel_graph on a 1-D..3-D lattice with a "
                      "boundary term, tile solver, lazy capacities); on this handle reset() it and rebuild the graph with "
                      "the seeds instead");
}

// The steps of a fold after its grouping (fold_run).  The grouping was enqueued after ev_fold[0] and left d_ctl = [item
// count | FOLD_ERR_* bits | touched-tile count] and the touched tiles in `tiles`; fold(grid, n_items) enqueues the fold
// kernel, which stores one partial of the add_tweights constant per block.  `nonfinite` and `negative` are the messages of
// FOLD_ERR_NONFINITE and FOLD_ERR_NEGATIVE, which name the kind of weight.  check (optional) enqueues a check of the calls
// against the current state that may set FOLD_ERR_PAIRSUM in d_ctl[1]; it runs after the first read-back, before anything
// is claimed or written, and its bits come back in a second read-back (only the folds that have one pay for it).
static int fold_items(mgc_graph* g, int* d_ctl, int* tiles, const std::function<int(unsigned, int)>& fold,
                      const char* nonfinite, const char* negative, const std::function<int()>* check)
{
    CK(cudaEventRecord(g->ev_fold[1], g->stream));
    // the item count and the error bits in one synchronisation, before the claim and the fold are enqueued
    int h_ctl[2] = {0, 0};
    CK(cudaMemcpyAsync(h_ctl, d_ctl, sizeof(h_ctl), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    if (h_ctl[1] & FOLD_ERR_RANGE) FAIL(MGC_E_ARG, "node id out of range");
    if (h_ctl[1] & FOLD_ERR_PAIR) FAIL(MGC_E_ARG, "node ids are not lattice neighbours");
    if (h_ctl[1] & FOLD_ERR_NONFINITE) FAIL(MGC_E_ARG, nonfinite);
    if (h_ctl[1] & FOLD_ERR_NEGATIVE) FAIL(MGC_E_WEIGHT, negative);
    const int ni = h_ctl[0];
    if (ni == 0) return MGC_OK;                // only add_tweights(v, 0, 0) calls: the state, mask and energy stay
    const bool eager = !g->lazy_built;         // MGC_OPT_WARM handle (warm_check passed)
    if (eager) {
        // not solved yet: the init and the record of the residual source capacities come first, so the fold reads the
        // same representation as after a solve
        int rc = warm_prepare(g);
        if (rc) return rc;
    }
    if (check) {
        // the check reads the state warm_prepare left (the init a first solve runs anyway) and writes nothing
        int rc = (*check)();
        if (rc) return rc;
        int bits = 0;
        CK(cudaMemcpyAsync(&bits, d_ctl + 1, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        if (bits & FOLD_ERR_PAIRSUM)
            FAIL(MGC_E_WEIGHT, "an n-link decrement exceeds what its arc pair holds: r(i->j) + r(j->i), which equals "
                               "c(i->j) + c(j->i), is below cap + rev_cap");
    }
    CK(cudaEventRecord(g->ev_fold[2], g->stream));
    // 1. every touched voxel's tile (and its face neighbours) holds cap[], tr, excess and the sink-link state from here on
    if (g->caps_lazy) {
        // Source excess is still implicit on the tiles that are listed but not materialised (before the first solve, or
        // deferred by the label window of the last one) and on the tiles the window dropped unmaterialised.  A new sink
        // link may drain it: materialise them, step 3 rebuilds the lists from cmat.
        int rc;
        for (int color = 0; color < 2; ++color) { rc = caps_launch(g, pl(g, color, g->pl_sel[color])); if (rc) return rc; }
        rc = caps_launch(g, WorkList{g->drop_items, g->win_ctl + WIN_NDROP});
        if (rc) return rc;
        CK(cudaMemsetAsync(g->win_ctl + WIN_NDROP, 0, sizeof(int), g->stream));
        rc = caps_launch(g, WorkList{tiles, d_ctl + 2});
        if (rc) return rc;
    }
    // 2. the fold, its change of the add_tweights constant summed in a fixed order into flow_const (on a batch handle the
    // fold also adds each image's share into that image's constant, batch_fold_const)
    unsigned grid = (unsigned)((ni + 255) / 256);
    if (grid > REDUCE_BLOCKS) grid = REDUCE_BLOCKS;
    { int rc = fold(grid, ni); if (rc) return rc; }
    sum_partials(g, g->partials, grid, g->d_scalars);
    // 3. solver state for the next solve: fresh push lists over every materialised tile with excess (every tile of an
    // eager handle; TL.ntiles is the 4-D tile count on a 4-D handle); labels from a full relabel reset (sweep_mode = -1: a
    // fold can remove a sink link, so the last solve's labels bound nothing).  On a z-slab only owned excess lists a tile:
    // the ghost planes' excess is the outbox, and the fold wrote none of it.
    CK(cudaMemsetAsync(g->d_tcount, 0, 256, g->stream));
    CK(cudaMemsetAsync(g->pflag, 0, (size_t)g->TL.ntiles * sizeof(int), g->stream));
    g->pl_sel[0] = g->pl_sel[1] = 0;
    {
        unsigned lgrid = (unsigned)g->n_ctas * 4u;
        if (lgrid > (unsigned)g->TL.ntiles) lgrid = (unsigned)g->TL.ntiles;
        if (g->nd == 4) k_seed_lists4<<<lgrid, T4_VOX, 0, g->stream>>>(g->L, g->TL4, g->S, g->pflag, pl(g, 0, 0), pl(g, 1, 0));
        else k_seed_lists<<<lgrid, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S, eager ? nullptr : g->cmat, g->pflag,
                                                             pl(g, 0, 0), pl(g, 1, 0));
    }
    g->st.kernel_launches += 3;
    CK(cudaGetLastError());
    CK(cudaEventRecord(g->ev_fold[3], g->stream));
    CK(cudaEventSynchronize(g->ev_fold[3]));
    {
        // two device spans: the grouping, then claim + fold + list fix-up (the read-back between them is not counted)
        float ms0 = 0, ms1 = 0;
        if (cudaEventElapsedTime(&ms0, g->ev_fold[0], g->ev_fold[1]) == cudaSuccess &&
            cudaEventElapsedTime(&ms1, g->ev_fold[2], g->ev_fold[3]) == cudaSuccess)
            g->st.ms_seeds += ms0 + ms1;
        g->st.ms_caps -= caps_resolve(g);          // the claim is part of ms_seeds, not of the solve's materialisation
    }
    g->labels_fresh = false;
    g->sweep_mode = -1;
    g->solved = false;
    g->host_mask_valid = false;
    g->st.seed_folds++;
    return slab_outbox_check(g);
}

// One fold call as its entry point describes it to fold_run: the argument checks, the inputs, and how the grouping keys
// its calls.  The rest of a fold is the same for seeds, t-links and n-links.
struct FoldCall {
    const char* range;            // NVTX range
    const char* bad;              // MGC_E_ARG message of malformed arrays or counts (nullptr: well formed)
    const char* too_many;         // MGC_E_ARG message of more than 2^31 - 1 calls
    const char* negative;         // MGC_E_WEIGHT message of a negative n-link weight
    int64_t count;                // calls: seed ids, add_tweights or sum_edge calls, or dense entries
    int32_t mem;                  // memory space of in[]
    bool dense;                   // one entry per voxel (count == the voxel count)
    const void* in[4];            // input arrays of 8-byte elements, in[k] with in_n[k] of them (nullptr: unused)
    int64_t in_n[4];
    const mgc_array* arrays[2];   // dense inputs as caller arrays, staged into in[2] / in[3] through slots 0 / 1
    int sort;                     // FOLD_SORT_KEYS / FOLD_SORT_PAIRS / FOLD_SCAN
    int key_shift;                // a key is voxel << key_shift | low bits: it has the bits of n << key_shift - 1
    int axis;                     // k_nlinks_items: the axis of the dense form
    bool item_flows;              // one double per item for the fold (n-link decrements: the excess change of an arc)
};

// The device buffers of a fold in fold_buf, 16-byte aligned pieces in this order
template <typename Key, typename Item>
struct FoldBufs {
    int* ctl;                     // [item count | FOLD_ERR_* bits | touched-tile count | tail count]
    const void* in[4];            // the inputs on the device: host arrays uploaded, device arrays in place
    Key* keys;                    // list forms: the keys of the calls, and sorted
    Key* skeys;
    int* vals;                    // pair sorts: the call indices, and sorted (each key's calls in call order)
    int* svals;
    int* head;                    // item heads, and their inclusive sum
    int* pos;
    int* tflag;                   // lazy handles: per-tile flags, and the touched tiles for the claim
    int* tiles;
    Item* items;
    unsigned* tbits;              // n-links: per-voxel tail bits, and the tails for the re-clamp
    unsigned* tails;
    double* dx;                   // item_flows: one double per item
    unsigned* stails;             // item_flows: the tails in ascending order (tails_sort)
    double* dk;                   // batch handles: the change of the add_tweights constant per item (or per sorted tail),
    double* dk_part;              // ... and the chunk sums and run images of its per-image sum (batch_fold_const)
    int* dk_span;
    void* tmp;                    // cub scratch
    size_t tmp_bytes;
};

// A bump allocator of 16-byte aligned pieces over one buffer; base == nullptr only measures the pieces
struct Bump {
    char* base;
    size_t used;
    template <typename T>
    T* take(size_t count)
    {
        T* p = base ? (T*)(base + used) : nullptr;
        used += (count * sizeof(T) + 15) / 16 * 16;
        return p;
    }
};

// A fold: the checks, the grouping of the calls into items on the device, then fold_items.  An item of NlinkItem names an
// arc: both ends are listed for the claim and its tails re-clamped.  group(b, grid) enqueues the keys, the sort
// (fold_sort) and the heads of the calls; fold(b, grid, n_items) the fold kernel(s); check(b, eager) (optional) the check
// fold_items runs before the claim.
template <typename Key, typename Item, typename Group, typename Fold, typename Check = std::nullptr_t>
static int fold_run(mgc_graph* g, const FoldCall& c, Group&& group, Fold&& fold, Check&& check = nullptr)
{
    constexpr bool arcs = std::is_same<Item, NlinkItem>::value;
    if (!g) return MGC_E_ARG;
    if (c.bad) FAIL(MGC_E_ARG, c.bad);
    if (c.count > (int64_t)INT32_MAX) FAIL(MGC_E_ARG, c.too_many);
    if (c.mem != MGC_MEM_HOST && c.mem != MGC_MEM_DEVICE) FAIL(MGC_E_ARG, "bad memory space");
    bool eager = false;
    { int rc0 = warm_check(g, &eager); if (rc0) return rc0; }
    if (c.dense && c.count && c.count != (int64_t)g->L.n) FAIL(MGC_E_ARG, "the dense form takes one weight pair per voxel");
    CK(cudaSetDevice(g->device));
    { int rc0 = check_pending(g); if (rc0) return rc0; }
    const void* in[4] = {c.in[0], c.in[1], c.in[2], c.in[3]};
    for (int k = 0; k < 2; ++k) {
        if (!c.arrays[k]) continue;
        // a batch's dense arrays are over (B, ...image): first as an array over its (B * Z, Y, X) lattice
        mgc_array view;
        const mgc_array* a = c.arrays[k];
        if (g->batch) { int rc0 = batch_view(g, a, k, &view); if (rc0) return rc0; a = &view; }
        int rc0 = stage_input(g, a, k, &in[2 + k]);
        if (rc0) return rc0;
    }
    int rc = MGC_OK;
    if (c.count) {                              // else nothing to fold: the solved state, mask and energy stay as they are
        const auto host_t0 = std::chrono::steady_clock::now();
        const int n = (int)c.count;
        // sort only the bits a key of this lattice can have
        const int end_bit = bits_for(((uint64_t)g->L.n << c.key_shift) - 1ull);
        size_t tmp_bytes = 0;
        CK(fold_sort(c.sort, nullptr, &tmp_bytes, (Key*)nullptr, (Key*)nullptr, nullptr, nullptr, n, end_bit, g->stream));
        CK(fold_scan(nullptr, &tmp_bytes, nullptr, nullptr, n, g->stream));
        if (c.item_flows) {
            // the largest tail sort the fold can need (tails_sort; fold_run's callers size it again before the sort)
            size_t tb = 0;
            CK(tails_sort(nullptr, &tb, nullptr, nullptr, (int)std::min(2 * (size_t)n, (size_t)g->L.n),
                          bits_for(g->L.n), g->stream));
            tmp_bytes = std::max(tmp_bytes, tb);
        }
        // no host slots for device inputs, no keys or call indices in a dense form, no tiles on an eager handle (nothing
        // to claim), no tails but for n-links
        const bool host = c.mem == MGC_MEM_HOST;
        const size_t ntl = eager ? 0 : (size_t)g->TL.ntiles;
        const size_t nk = c.sort == FOLD_SCAN ? 0 : (size_t)n;
        const size_t nv = c.sort == FOLD_SORT_PAIRS ? (size_t)n : 0;
        const size_t claims = std::min((arcs ? 2 : 1) * (size_t)n, ntl);
        const size_t ntails = arcs ? std::min(2 * (size_t)n, (size_t)g->L.n) : 0;
        const size_t nbits = arcs ? ((size_t)g->L.n + 31) / 32 : 0;
        FoldBufs<Key, Item> b{};
        auto layout = [&](Bump m) {
            b.ctl = m.take<int>(4);
            for (int k = 0; k < 4; ++k)
                b.in[k] = host && c.in[k] ? m.take<int64_t>((size_t)c.in_n[k]) : in[k];
            b.keys = m.take<Key>(nk);
            b.skeys = m.take<Key>(nk);
            b.vals = m.take<int>(nv);
            b.svals = m.take<int>(nv);
            b.head = m.take<int>(n);
            b.pos = m.take<int>(n);
            b.tflag = m.take<int>(ntl);
            b.tiles = m.take<int>(claims);
            b.items = m.take<Item>(n);
            b.tbits = m.take<unsigned>(nbits);
            b.tails = m.take<unsigned>(ntails);
            b.dx = m.take<double>(c.item_flows ? (size_t)n : 0);
            b.stails = m.take<unsigned>(c.item_flows ? ntails : 0);
            const size_t nd = g->batch ? std::max((size_t)n, ntails) : 0;
            b.dk = nd ? m.take<double>(nd) : nullptr;
            b.dk_part = nd ? m.take<double>(2 * batch_fold_chunks((int)nd)) : nullptr;
            b.dk_span = nd ? m.take<int>(batch_fold_chunks((int)nd)) : nullptr;
            b.tmp = m.take<char>(tmp_bytes);
            b.tmp_bytes = tmp_bytes;
            return m.used;
        };
        rc = ensure_scratch(g, g->fold_buf, layout(Bump{nullptr, 0}));
        if (rc) return rc;
        layout(Bump{(char*)g->fold_buf.p, 0});
        int cub_launches = 0;
        rc = fold_cub_launches(g, c.sort, n, end_bit, b.tmp, tmp_bytes, b.keys, b.skeys, b.vals, b.svals, b.head, b.pos,
                               &cub_launches);
        if (rc) return rc;
        for (auto& ev : g->ev_fold) if (!ev) CK(cudaEventCreate(&ev));
        Nvtx range(c.range);
        g->st.ms_seeds_host += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count();
        // 0. grouping on the device; nothing below touches the solver state until the checks of the calls have passed.
        // Host arrays go straight from the caller into their device slots: no host pass over them.
        CK(cudaEventRecord(g->ev_fold[0], g->stream));
        for (int k = 0; k < 4; ++k)
            if (host && c.in[k] && c.in_n[k])
                CK(cudaMemcpyAsync((void*)b.in[k], c.in[k], (size_t)c.in_n[k] * 8, cudaMemcpyHostToDevice, g->stream));
        CK(cudaMemsetAsync(b.ctl, 0, 4 * sizeof(int), g->stream));
        CK(cudaMemsetAsync(b.tflag, 0, ntl * sizeof(int), g->stream));
        if (arcs) CK(cudaMemsetAsync(b.tbits, 0, nbits * 4, g->stream));
        const unsigned kgrid = (unsigned)std::min<int64_t>(((int64_t)n + 255) / 256, (int64_t)g->n_ctas * 8);
        rc = group(b, kgrid, [&]() { return fold_sort(c.sort, b.tmp, &tmp_bytes, b.keys, b.skeys, b.vals, b.svals, n,
                                                      end_bit, g->stream); });
        if (rc) return rc;
        CK(fold_scan(b.tmp, &tmp_bytes, b.head, b.pos, n, g->stream));
        int* tflag = eager ? nullptr : b.tflag;
        const Key* skeys = c.sort == FOLD_SCAN ? nullptr : b.skeys;
        if constexpr (arcs)
            k_nlinks_items<<<kgrid, 256, 0, g->stream>>>(g->L, g->TL, skeys, c.axis, b.pos, n, b.items, tflag, b.tiles, b.ctl);
        else
            k_tweights_items<<<kgrid, 256, 0, g->stream>>>(g->L, g->TL, skeys, c.key_shift, b.pos, n, b.items, tflag, b.tiles,
                                                           b.ctl);
        g->st.kernel_launches += (c.sort == FOLD_SCAN ? 2 : 3) + cub_launches;
        CK(cudaGetLastError());
        std::function<int()> chk;
        if constexpr (!std::is_same<std::decay_t<Check>, std::nullptr_t>::value) chk = [&]() { return check(b, eager); };
        auto fold_call = [&](unsigned grid, int ni) -> int {
            if constexpr (std::is_void<decltype(fold(b, eager, grid, ni))>::value) { fold(b, eager, grid, ni); return MGC_OK; }
            else return fold(b, eager, grid, ni);
        };
        rc = fold_items(g, b.ctl, b.tiles, fold_call,
                        arcs ? "an n-link weight is NaN or infinite" : "a t-link weight is NaN or infinite",
                        c.negative ? c.negative : "negative n-link weights are not allowed (a warm fold only raises capacities)",
                        chk ? &chk : nullptr);
    }
    if (c.arrays[0]) slots_release(g, 3u);     // the grouping and the fold read the staging slots
    return rc;
}

// The t-link fold over a grouping's items, then on a batch handle the per-image sum of their constant changes (the
// items are in ascending voxel order, TweightItem::v first)
template <typename Calls>
static int tlink_fold(mgc_graph* g, const FoldBufs<unsigned, TweightItem>& b, bool eager, unsigned grid, int ni,
                      const Calls& calls)
{
    residual_dispatch(g, eager, [&](auto A) {
        k_tlink_fold<<<grid, 256, 0, g->stream>>>(A, b.items, ni, calls, g->partials, b.dk);
    });
    if (!g->batch) return MGC_OK;
    return batch_fold_const(g, reinterpret_cast<const unsigned*>(b.items), (int)(sizeof(TweightItem) / sizeof(unsigned)),
                            b.ctl, ni, b.dk, b.dk_part, b.dk_span);
}

extern "C" {

// mgc_add_seeds (cap = 65535) and mgc_remove_seeds (cap = -65535): add_tweights(v, cap, 0) for every fg id in list order,
// then add_tweights(v, 0, cap) for every bg id, folded into the handle's current state.  Key = v << 1 | (background):
// sorted, a voxel's fg seeds precede its bg seeds, the reference's order for one voxel (a voxel's t-link only depends on
// its own calls).
static int seeds_fold(mgc_graph* g, const int64_t* fg_ids, int64_t n_fg, const int64_t* bg_ids, int64_t n_bg, int32_t mem,
                      double cap)
{
    const bool bad = n_fg < 0 || n_bg < 0 || (n_fg && !fg_ids) || (n_bg && !bg_ids);
    FoldCall c{};
    c.range = cap > 0 ? "mgc:add_seeds" : "mgc:remove_seeds";
    c.bad = bad ? "bad seed lists" : nullptr;
    c.too_many = "more than 2^31 - 1 seeds in one call";
    c.count = bad ? 0 : n_fg + n_bg;
    c.mem = mem;
    c.in[0] = fg_ids; c.in_n[0] = n_fg;
    c.in[1] = bg_ids; c.in_n[1] = n_bg;
    c.sort = FOLD_SORT_KEYS;
    c.key_shift = 1;
    return fold_run<unsigned, TweightItem>(g, c,
        [&](const FoldBufs<unsigned, TweightItem>& b, unsigned kgrid, auto sort) {
            k_seed_keys<<<kgrid, 256, 0, g->stream>>>((const int64_t*)b.in[0], (int)n_fg, (const int64_t*)b.in[1], (int)n_bg,
                                                      (int64_t)g->L.n, b.keys, b.ctl + 1);
            CK(sort());
            slab_dispatch(g, [&](auto slab, SlabOwn own) {
                k_seed_heads<decltype(slab)::value><<<kgrid, 256, 0, g->stream>>>(b.skeys, (int)(n_fg + n_bg), b.head, own);
            });
            return MGC_OK;
        },
        [&](const FoldBufs<unsigned, TweightItem>& b, bool eager, unsigned grid, int ni) {
            return tlink_fold(g, b, eager, grid, ni, SeedCalls{b.skeys, cap});
        });
}

int mgc_add_seeds(mgc_graph* g, const int64_t* fg_ids, int64_t n_fg, const int64_t* bg_ids, int64_t n_bg, int32_t mem)
{
    return seeds_fold(g, fg_ids, n_fg, bg_ids, n_bg, mem, 65535.0);
}

int mgc_remove_seeds(mgc_graph* g, const int64_t* fg_ids, int64_t n_fg, const int64_t* bg_ids, int64_t n_bg, int32_t mem)
{
    return seeds_fold(g, fg_ids, n_fg, bg_ids, n_bg, mem, -65535.0);
}

// list form: (voxel id, call index) pairs, stably sorted so a voxel's calls keep their order, then run-length encoded;
// dense form (ids == nullptr): the voxels with a nonzero weight, compacted by a scan of their flags.  In both, a voxel
// whose calls all have zero weights is no item (add_tweights(v, 0, 0) changes nothing).
int mgc_add_tweights_warm(mgc_graph* g, const int64_t* ids, const double* src, const double* snk, int64_t count, int32_t mem)
{
    const bool dense = ids == nullptr;
    FoldCall c{};
    c.range = "mgc:add_tweights_warm";
    c.bad = count < 0 || (count && (!src || !snk)) ? "bad t-link arrays" : nullptr;
    c.too_many = "more than 2^31 - 1 add_tweights calls in one call";
    c.count = count;
    c.mem = mem;
    c.dense = dense;
    c.in[0] = ids; c.in_n[0] = count;
    c.in[1] = src; c.in_n[1] = count;
    c.in[2] = snk; c.in_n[2] = count;
    c.sort = dense ? FOLD_SCAN : FOLD_SORT_PAIRS;
    return fold_run<unsigned, TweightItem>(g, c,
        [&](const FoldBufs<unsigned, TweightItem>& b, unsigned kgrid, auto sort) {
            const double* d_src = (const double*)b.in[1];
            const double* d_snk = (const double*)b.in[2];
            if (dense) {
                slab_dispatch(g, [&](auto slab, SlabOwn own) {
                    k_tweights_dense_heads<decltype(slab)::value><<<kgrid, 256, 0, g->stream>>>(d_src, d_snk, (int)count,
                                                                                              b.head, b.ctl + 1, own);
                });
                return MGC_OK;
            }
            k_tweights_keys<<<kgrid, 256, 0, g->stream>>>((const int64_t*)b.in[0], d_src, d_snk, (int)count, (int64_t)g->L.n,
                                                          b.keys, b.vals, b.ctl + 1);
            CK(sort());
            slab_dispatch(g, [&](auto slab, SlabOwn own) {
                k_weighted_heads<unsigned, decltype(slab)::value><<<kgrid, 256, 0, g->stream>>>(b.skeys, b.svals, d_src, d_snk,
                                                                                              (int)count, b.head, own);
            });
            return MGC_OK;
        },
        [&](const FoldBufs<unsigned, TweightItem>& b, bool eager, unsigned grid, int ni) {
            const ListCalls calls{dense ? nullptr : b.svals, (const double*)b.in[1], (const double*)b.in[2]};
            return tlink_fold(g, b, eager, grid, ni, calls);
        });
}

// sum_edge calls folded into the handle's current state (gc_nlinks.cuh).  ii != nullptr: the list form, call k is
// sum_edge(ii[k], jj[k], cap[k], rev[k]) with every array in `mem`: (arc key, call index) pairs, key = lo << 2 | axis,
// stably sorted, then run-length encoded.  ii == nullptr: the dense form along canonical axis `axis`, entry p of the
// staged cap / rev (count = the voxel count) holds the increments of p -> p + e_axis and back; the pairs with a nonzero
// increment are compacted by a scan of their flags.  The grouping is the same for increments and decrements
// (nweights_group); only the fold differs.
using NlinkBufs = FoldBufs<unsigned long long, NlinkItem>;

static int nweights_group(mgc_graph* g, const FoldCall& c, const NlinkBufs& b, unsigned kgrid,
                          const std::function<cudaError_t()>& sort)
{
    const int axis = c.axis;
    const int n = (int)c.count;
    const double* d_cap = (const double*)b.in[2];
    const double* d_rev = (const double*)b.in[3];
    if (c.dense) {
        // axis 0 spans the lattice, or one image of a batch (k_nlinks_dense_heads)
        unsigned span = axis == 0 ? g->L.n : g->L.stride[axis - 1];
        unsigned long long magic = axis == 0 ? 0ull : g->L.magic[axis - 1];
        if (axis == 0 && g->L.zper) {
            span = (unsigned)g->L.zper * g->L.stride[0];
            magic = span <= 1 ? 0ull : (~0ull / span) + 1ull;
        }
        slab_dispatch(g, [&](auto slab, SlabOwn own) {
            k_nlinks_dense_heads<decltype(slab)::value><<<kgrid, 256, 0, g->stream>>>(g->L.n, span, magic,
                                                                                    span - g->L.stride[axis], d_cap, d_rev,
                                                                                    b.head, b.ctl + 1, own);
        });
        return MGC_OK;
    }
    const int64_t* d_i = (const int64_t*)b.in[0];
    const int64_t* d_j = (const int64_t*)b.in[1];
    if (g->nd == 4) k_nlinks_keys<4><<<kgrid, 256, 0, g->stream>>>(g->L, d_i, d_j, d_cap, d_rev, n, b.keys, b.vals, b.ctl + 1);
    else            k_nlinks_keys<3><<<kgrid, 256, 0, g->stream>>>(g->L, d_i, d_j, d_cap, d_rev, n, b.keys, b.vals, b.ctl + 1);
    CK(sort());
    slab_dispatch(g, [&](auto slab, SlabOwn own) {
        k_weighted_heads<unsigned long long, decltype(slab)::value><<<kgrid, 256, 0, g->stream>>>(b.skeys, b.svals, d_cap,
                                                                                                d_rev, n, b.head, own);
    });
    return MGC_OK;
}

static int nweights_fold(mgc_graph* g, FoldCall& c, int axis)
{
    const bool dense = c.dense;
    c.sort = dense ? FOLD_SCAN : FOLD_SORT_PAIRS;
    c.key_shift = 2;
    c.axis = axis;
    return fold_run<unsigned long long, NlinkItem>(g, c,
        [&](const NlinkBufs& b, unsigned kgrid, auto sort) { return nweights_group(g, c, b, kgrid, sort); },
        [&](const NlinkBufs& b, bool eager, unsigned grid, int ni) {
            // the arcs first, then each tail once: the re-clamp reads the out-capacity after every increment of the call
            const int* order = dense ? nullptr : b.svals;
            const int64_t* ids = dense ? nullptr : (const int64_t*)b.in[0];
            const double* d_cap = (const double*)b.in[2];
            const double* d_rev = (const double*)b.in[3];
            int* ntails = b.ctl + 3;
            slab_dispatch(g, [&](auto slab, SlabOwn own) {
                constexpr bool S = decltype(slab)::value;
                if (g->nd == 4) k_nlinks_fold<4, S><<<grid, 256, 0, g->stream>>>(g->L, g->S, b.items, ni, order, ids, d_cap, d_rev, b.tbits, b.tails, ntails, own);
                else            k_nlinks_fold<3, S><<<grid, 256, 0, g->stream>>>(g->L, g->S, b.items, ni, order, ids, d_cap, d_rev, b.tbits, b.tails, ntails, own);
            });
            g->st.kernel_launches++;
            residual_dispatch(g, eager, [&](auto A) {
                k_nlinks_reclamp<<<grid, 256, 0, g->stream>>>(A, b.tails, ntails, g->partials);
            });
        });
}

// sum_edge calls with negated weights (gc_nlinks_remove.cuh): the grouping of nweights_fold, the pair check before the
// claim, then the arcs (one excess change per item in dx) and each endpoint once.
static int nweights_remove_fold(mgc_graph* g, FoldCall& c, int axis)
{
    const bool dense = c.dense;
    c.sort = dense ? FOLD_SCAN : FOLD_SORT_PAIRS;
    c.key_shift = 2;
    c.axis = axis;
    c.negative = "negative n-link decrements are not allowed (a removal takes nonnegative amounts off the capacities)";
    c.item_flows = true;
    const int n = (int)c.count;
    auto calls = [&](const NlinkBufs& b, const int*& order, const int64_t*& ids) {
        order = dense ? nullptr : b.svals;
        ids = dense ? nullptr : (const int64_t*)b.in[0];
    };
    return fold_run<unsigned long long, NlinkItem>(g, c,
        [&](const NlinkBufs& b, unsigned kgrid, auto sort) { return nweights_group(g, c, b, kgrid, sort); },
        [&](const NlinkBufs& b, bool eager, unsigned grid, int ni) -> int {
            const int* order; const int64_t* ids;
            calls(b, order, ids);
            const double* d_cap = (const double*)b.in[2];
            const double* d_rev = (const double*)b.in[3];
            int* ntails = b.ctl + 3;
            // the tails are listed in atomic order; they are sorted before the voxel pass, so each one lands in the same
            // thread and block on every run and the per-block sums of the constant are reproducible
            const int nt = (int)std::min(2 * (int64_t)ni, (int64_t)g->L.n);
            const int tbit = bits_for(g->L.n);
            CK(cudaMemsetAsync(b.tails, 0xff, (size_t)nt * sizeof(unsigned), g->stream));
            if (g->nd == 4) k_nlinks_remove_arcs<4><<<grid, 256, 0, g->stream>>>(g->L, g->S, b.items, ni, order, ids, d_cap, d_rev, b.dx, b.tbits, b.tails, ntails);
            else            k_nlinks_remove_arcs<3><<<grid, 256, 0, g->stream>>>(g->L, g->S, b.items, ni, order, ids, d_cap, d_rev, b.dx, b.tbits, b.tails, ntails);
            g->st.kernel_launches++;
            size_t tb = 0;
            CK(tails_sort(nullptr, &tb, b.tails, b.stails, nt, tbit, g->stream));
            if (tb > b.tmp_bytes) FAIL(MGC_E_CUDA, "the tail sort needs more scratch than was sized");
            int sort_launches = 0;
            int rc = cub_launches(g, std::make_tuple(g->device, (int)FOLD_SORT_TAILS, 4, nt, tbit), [&](cudaStream_t s) {
                size_t t = b.tmp_bytes;
                return tails_sort(b.tmp, &t, b.tails, b.stails, nt, tbit, s);
            }, &sort_launches);
            if (rc) return rc;
            tb = b.tmp_bytes;
            CK(tails_sort(b.tmp, &tb, b.tails, b.stails, nt, tbit, g->stream));
            g->st.kernel_launches += sort_launches;
            const unsigned long long* skeys = dense ? nullptr : b.skeys;
            residual_dispatch(g, eager, [&](auto A) {
                k_nlinks_remove_voxels<<<grid, 256, 0, g->stream>>>(A, g->L, skeys, b.head, b.pos, n, axis, b.dx, b.stails,
                                                                    ntails, g->partials, b.dk);
            });
            // a batch: the shortfalls the terminal links covered, per image (the sorted tails are in ascending order)
            return g->batch ? batch_fold_const(g, b.stails, 1, ntails, nt, b.dk, b.dk_part, b.dk_span) : MGC_OK;
        },
        [&](const NlinkBufs& b, bool eager) {
            // after the first read-back: the item count is on the device in b.ctl[0]
            const int* order; const int64_t* ids;
            calls(b, order, ids);
            const int* cmat = eager || !g->caps_lazy ? nullptr : g->cmat;
            unsigned grid = (unsigned)std::min<int64_t>(((int64_t)n + 255) / 256, (int64_t)g->n_ctas * 8);
            residual_dispatch(g, eager, [&](auto A) {
                k_nlinks_remove_check<<<grid, 256, 0, g->stream>>>(A, g->L, g->TL, cmat, b.items, b.ctl, order, ids,
                                                                   (const double*)b.in[2], (const double*)b.in[3],
                                                                   b.ctl + 1);
            });
            g->st.kernel_launches++;
            CK(cudaGetLastError());
            return MGC_OK;
        });
}

static void nweights_list_call(FoldCall& c, const char* range, const int64_t* i, const int64_t* j, const double* cap,
                               const double* rev_cap, int64_t count, int32_t mem)
{
    c.range = range;
    c.bad = count < 0 || (count && (!i || !j || !cap || !rev_cap)) ? "bad n-link arrays" : nullptr;
    c.too_many = "more than 2^31 - 1 sum_edge calls in one call";
    c.count = count;
    c.mem = mem;
    c.in[0] = i; c.in_n[0] = count;
    c.in[1] = j; c.in_n[1] = count;
    c.in[2] = cap; c.in_n[2] = count;
    c.in[3] = rev_cap; c.in_n[3] = count;
}

static int nweights_dense_call(mgc_graph* g, FoldCall& c, const char* range, int32_t axis, const mgc_array* fwd,
                               const mgc_array* bwd)
{
    if (!g || !fwd || !bwd) return MGC_E_ARG;
    if (axis < 0 || axis >= g->user_ndim) FAIL(MGC_E_ARG, "bad axis");
    if (fwd->dtype != MGC_F64 || bwd->dtype != MGC_F64) FAIL(MGC_E_ARG, "dense n-weights must be float64");
    c.range = range;
    c.count = (int64_t)g->L.n;
    c.mem = MGC_MEM_DEVICE;
    c.dense = true;
    c.arrays[0] = fwd;
    c.arrays[1] = bwd;
    return MGC_OK;
}

int mgc_add_nweights_warm(mgc_graph* g, const int64_t* i, const int64_t* j, const double* cap, const double* rev_cap,
                          int64_t count, int32_t mem)
{
    FoldCall c{};
    nweights_list_call(c, "mgc:add_nweights_warm", i, j, cap, rev_cap, count, mem);
    return nweights_fold(g, c, 0);
}

int mgc_add_nweights_dense_warm(mgc_graph* g, int32_t axis, const mgc_array* fwd, const mgc_array* bwd)
{
    FoldCall c{};
    int rc = nweights_dense_call(g, c, "mgc:add_nweights_dense_warm", axis, fwd, bwd);
    if (rc) return rc;
    return nweights_fold(g, c, axis + g->shift);
}

// n-link decrements on a z-slab handle: refused whatever the pairs.  A decrement of a pair across a slab border needs the
// residual of the arc the neighbour owns, and the pair check's verdict is known on the owning slab only, so refusing a bad
// call on every slab alike would take a two-phase collective.  Refusing them all keeps the answer the same however the
// volume is partitioned.
static int slab_decrement_refused(mgc_graph* g)
{
    if (!g || !g->slab) return MGC_OK;
    FAIL(MGC_E_STATE, "n-link decrements are not available on z-slab handles (a pair across a slab border needs the "
                      "neighbour's residual); reset() the slabs and rebuild the graph without the weight instead");
}

int mgc_remove_nweights_warm(mgc_graph* g, const int64_t* i, const int64_t* j, const double* cap, const double* rev_cap,
                             int64_t count, int32_t mem)
{
    if (int rc = slab_decrement_refused(g)) return rc;
    FoldCall c{};
    nweights_list_call(c, "mgc:remove_nweights_warm", i, j, cap, rev_cap, count, mem);
    return nweights_remove_fold(g, c, 0);
}

int mgc_remove_nweights_dense_warm(mgc_graph* g, int32_t axis, const mgc_array* fwd, const mgc_array* bwd)
{
    if (int rc = slab_decrement_refused(g)) return rc;
    FoldCall c{};
    int rc = nweights_dense_call(g, c, "mgc:remove_nweights_dense_warm", axis, fwd, bwd);
    if (rc) return rc;
    return nweights_remove_fold(g, c, axis + g->shift);
}

}  // extern "C"
