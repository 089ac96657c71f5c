// gc_sparse_api.cu -- host side of the C ABI for general sparse graphs (include/medpy_b200_graphcut.h, section "general
// sparse graphs"; SURVEY.md §8 row f4).
//
// mgc_sparse keeps what the reference's Graph<> keeps on the host while a graph is assembled (gc_sparse_host.hpp) and
// runs the max-flow on the device (gc_sparse.cuh).  With MGC_OPT_WARM the device state of the first solve stays resident
// and later calls fold into it (gc_sparse_warm.cuh); the stable radix sort that groups a fold's calls is
// cub::DeviceRadixSort (gc_sort.cuh).
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/medpy_b200_graphcut.h"
#include "gc_host.hpp"
#include "gc_sort.cuh"
#include "gc_sparse_host.hpp"
#include "gc_sparse_warm.cuh"

namespace {

thread_local std::string g_sp_create_error;

// The device arrays of a solve: the push-relabel state, the loop's flag words, active-node count, mask and absorbed
// flow, and on a warm handle `sent` and the edge fold's tail flags.
struct SparseDev {
    int n = 0, m2 = 0;
    int *row = nullptr, *head = nullptr, *sis = nullptr, *height = nullptr, *flags = nullptr;
    double *cap = nullptr, *tr = nullptr, *excess = nullptr, *sunk = nullptr, *sent = nullptr, *abs = nullptr;
    uint8_t *mask = nullptr, *tail = nullptr;
    unsigned long long* count = nullptr;

    template <typename T>
    static void get(cudaError_t& e, T*& p, size_t count)
    {
        if (e == cudaSuccess) e = cudaMalloc(&p, (count ? count : 1) * sizeof(T));
    }
    cudaError_t alloc(int nodes, int arcs, bool warm)
    {
        n = nodes;
        m2 = arcs;
        cudaError_t e = cudaSuccess;
        get(e, row, (size_t)n + 1); get(e, head, (size_t)m2); get(e, sis, (size_t)m2); get(e, cap, (size_t)m2);
        get(e, tr, (size_t)n); get(e, excess, (size_t)n); get(e, sunk, (size_t)n); get(e, height, (size_t)n);
        get(e, mask, (size_t)n); get(e, flags, 2); get(e, abs, 1); get(e, count, 1);
        if (warm) { get(e, sent, (size_t)n); get(e, tail, (size_t)n); }
        return e;
    }
    void release()
    {
        void* ps[] = {row, head, sis, height, flags, cap, tr, excess, sunk, sent, abs, mask, tail, count};
        for (void* p : ps)
            if (p) cudaFree(p);
        *this = SparseDev{};
    }
    SparseState state() const { return SparseState{n, m2, row, head, sis, cap, tr, excess, sunk, height}; }
    SparseWarm warm() const { return SparseWarm{n, row, head, cap, tr, excess, sunk, sent}; }
};

// two events around a timed section on the legacy default stream, destroyed with the scope
struct Events {
    cudaEvent_t start = nullptr, stop = nullptr;
    Events() = default;
    Events(const Events&) = delete;
    ~Events() { for (cudaEvent_t e : {start, stop}) if (e) cudaEventDestroy(e); }
    cudaError_t begin()
    {
        cudaError_t e = cudaEventCreate(&start);
        if (e == cudaSuccess) e = cudaEventCreate(&stop);
        return e == cudaSuccess ? cudaEventRecord(start, 0) : e;
    }
    cudaError_t elapsed(float* ms) const { return cudaEventElapsedTime(ms, start, stop); }
};

}  // namespace

struct mgc_sparse {
    int device = 0;
    SparseHost host;                                   // the graph's calls as the reference's Graph<> keeps them
    bool solved = false;
    double energy = 0.0;
    std::vector<uint8_t> mask;
    int push_steps = 4;                                // push steps per node and launch
    int sweeps_per_round = 16;                         // push launches between two global relabels
    int relax_batch = 8;                               // relaxation launches per "changed" read-back
    int64_t max_rounds = 1000000;
    double max_seconds = 600.0;                        // wall-clock cap of one solve (MEDPY_GC_SPARSE_TIMEOUT overrides)
    mgc_stats st{};
    std::string err;
    // MGC_OPT_WARM (gc_sparse_warm.cuh): the device state of the first solve stays resident and later calls fold into it
    bool warm = false;
    bool solved_once = false;                          // solved since create / reset: the option can no longer change
    bool resident = false;                             // `dev` holds the state of a warm solve
    bool warm_bad = false;                             // that solve's graph held a NaN or infinite capacity: no folds
    double wconst = 0.0;                               // constant of the resident state (energy = wconst + absorbed)
    SparseDev dev;                                     // a cold solve's arrays for the call, a warm one's until reset
    void release()
    {
        if (!resident) return;
        cudaSetDevice(device);
        dev.release();
        resident = false;
    }
    ~mgc_sparse() { release(); }
};

namespace {

// The push-relabel loop from the first exact global relabel to the stop test, then the read-out: the whole solve of a
// warm re-solve, the rest of a first solve after its init.
int sparse_loop(mgc_sparse* g, const Events& ev, double base)
{
    const SparseState S = g->dev.state();
    int* d_flags = g->dev.flags;
    const int n = S.n;
    const unsigned blocks = grid_for(n);
    int64_t rounds = 0;
    long long active = 0;
    const auto t_start = std::chrono::steady_clock::now();
    for (;;) {
        // exact global relabel: backward BFS from the sink by in-place relaxation
        k_sp_relabel_init<<<blocks, 256>>>(S);
        g->st.kernel_launches++;
        g->st.global_relabels++;
        for (;;) {
            CK(cudaMemsetAsync(d_flags, 0, sizeof(int), 0));
            for (int r = 0; r < g->relax_batch; ++r) k_sp_relax<<<blocks, 256>>>(S, d_flags);
            g->st.kernel_launches += g->relax_batch;
            g->st.relabel_sweeps += g->relax_batch;
            int changed = 0;
            CK(cudaMemcpy(&changed, d_flags, sizeof(int), cudaMemcpyDeviceToHost));
            if (!changed) break;
        }
        // stop test, only ever right after an exact relabel
        CK(cudaMemsetAsync(g->dev.count, 0, sizeof(unsigned long long), 0));
        k_sp_count_active<<<blocks, 256>>>(S, g->dev.count);
        g->st.kernel_launches++;
        unsigned long long c = 0;
        CK(cudaMemcpy(&c, g->dev.count, sizeof(c), cudaMemcpyDeviceToHost));
        active = (long long)c;
        if (!active) break;
        const double elapsed = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
        if (++rounds > g->max_rounds || elapsed > g->max_seconds)
            FAIL(MGC_E_NOCONV, "sparse push-relabel did not converge within " + std::to_string(rounds) + " rounds / " +
                                     std::to_string(elapsed) + " s (" + std::to_string(active) + " active nodes left)");
        for (int s = 0; s < g->sweeps_per_round; ++s) k_sp_push<<<blocks, 256>>>(S, g->push_steps, d_flags + 1);
        g->st.kernel_launches += g->sweeps_per_round;
        g->st.push_sweeps += g->sweeps_per_round;
    }
    k_sp_readout<<<1, 256>>>(S, g->dev.mask, g->dev.abs);
    g->st.kernel_launches++;
    CK(cudaEventRecord(ev.stop, 0));
    CK(cudaGetLastError());
    g->mask.assign((size_t)n, 0);
    double absorbed = 0.0;
    CK(cudaMemcpy(g->mask.data(), g->dev.mask, (size_t)n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&absorbed, g->dev.abs, sizeof(double), cudaMemcpyDeviceToHost));
    float ms = 0.f;
    CK(ev.elapsed(&ms));
    g->energy = base + absorbed;
    g->solved = true;
    g->solved_once = true;
    g->st.n_voxels = n;
    g->st.ms_solve = ms;
    g->st.active_last = active;
    g->st.flow_const = g->host.flow_const;
    g->st.energy = g->energy;
    g->st.device_bytes = (int64_t)((size_t)S.m2 * 16 + (size_t)n * (g->warm ? 41 : 33));
    return MGC_OK;
}

// the first solve since create / reset: CSR on the host, upload, init, loop
int sparse_first_solve(mgc_sparse* g)
{
    const SparseHost& h = g->host;
    const int n = (int)h.n;
    const int64_t np = (int64_t)h.plo.size();
    if (2 * np >= (int64_t)INT32_MAX) FAIL(MGC_E_ARG, "too many arcs for 32-bit arc ids");
    const int m2 = (int)(2 * np);
    std::vector<int> row, head, sis;
    std::vector<double> cap;
    h.csr(row, head, sis, cap);
    SparseDev& d = g->dev;
    CK(d.alloc(n, m2, g->warm));
    CK(cudaMemcpy(d.row, row.data(), ((size_t)n + 1) * sizeof(int), cudaMemcpyHostToDevice));
    if (m2) {
        CK(cudaMemcpy(d.head, head.data(), (size_t)m2 * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d.sis, sis.data(), (size_t)m2 * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d.cap, cap.data(), (size_t)m2 * sizeof(double), cudaMemcpyHostToDevice));
    }
    CK(cudaMemcpy(d.tr, h.tr.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
    if (g->warm) CK(cudaMemset(d.tail, 0, (size_t)n));
    Events ev;
    CK(ev.begin());
    const unsigned blocks = grid_for(n);
    if (g->warm) k_spw_init<<<blocks, 256>>>(d.warm());
    else         k_sp_init<<<blocks, 256>>>(d.state());
    g->st.kernel_launches++;
    if (!g->warm) return sparse_loop(g, ev, h.flow_const);
    // warm: the state stays resident whether the loop converges or not; so do the pairs' arc offsets
    g->resident = true;
    g->wconst = h.flow_const;
    bool bad = false;
    for (int v = 0; v < n && !bad; ++v) bad = !std::isfinite(h.tr[(size_t)v]);
    for (int a = 0; a < m2 && !bad; ++a) bad = !std::isfinite(cap[(size_t)a]);
    g->warm_bad = bad;
    g->host.record_offsets();
    return sparse_loop(g, ev, g->wconst);
}

int sparse_solve(mgc_sparse* g)
{
    CK(cudaSetDevice(g->device));
    if (g->resident) {
        Events ev;
        CK(ev.begin());
        return sparse_loop(g, ev, g->wconst);
    }
    const int rc = sparse_first_solve(g);
    if (!g->resident) g->dev.release();             // a cold solve's arrays live for the call
    return rc;
}

// ---- folds into the resident state of a warm handle ------------------------------------------------------------
template <typename T>
int warm_upload(mgc_sparse* g, DevScope& dev, const T* h, size_t count, T** d)
{
    CK(dev.alloc(d, count));
    if (count) CK(cudaMemcpy(*d, h, count * sizeof(T), cudaMemcpyHostToDevice));
    return MGC_OK;
}

// The calls are grouped on the device: (key, call index) pairs through a stable radix sort, so each key's calls keep
// their order; the first slot of every run of equal keys does the work (gc_sparse_warm.cuh).
int warm_sort(mgc_sparse* g, DevScope& dev, unsigned* keys, long long m, unsigned key_max, unsigned** keys_sorted,
              unsigned** order)
{
    unsigned* idx;
    CK(dev.alloc(&idx, (size_t)m));
    CK(dev.alloc(keys_sorted, (size_t)m));
    CK(dev.alloc(order, (size_t)m));
    lab_iota(idx, m);
    g->st.kernel_launches++;
    CK(radix_sort(dev, keys, *keys_sorted, (int)m, bits_for(key_max), idx, *order));
    g->st.kernel_launches += 4;
    return MGC_OK;
}

int warm_group(mgc_sparse* g, DevScope& dev, const std::vector<unsigned>& h_keys, unsigned key_max, unsigned** keys_sorted,
               unsigned** order)
{
    unsigned* keys;
    RC(warm_upload(g, dev, h_keys.data(), h_keys.size(), &keys));
    return warm_sort(g, dev, keys, (long long)h_keys.size(), key_max, keys_sorted, order);
}

// resolved n-link calls on the device, grouped by pair
struct DevCalls {
    unsigned *keys, *order;
    int *lo, *hi, *olo, *ohi;
    double *c_lh, *c_hl;
};

int warm_calls(mgc_sparse* g, DevScope& dev, const SparseCalls& c, DevCalls& d)
{
    const size_t m = c.pk.size();
    const int64_t np = (int64_t)g->host.plo.size();
    RC(warm_group(g, dev, c.pk, (unsigned)(np > 0 ? np - 1 : 0), &d.keys, &d.order));
    RC(warm_upload(g, dev, c.lo.data(), m, &d.lo));
    RC(warm_upload(g, dev, c.hi.data(), m, &d.hi));
    RC(warm_upload(g, dev, c.olo.data(), m, &d.olo));
    RC(warm_upload(g, dev, c.ohi.data(), m, &d.ohi));
    RC(warm_upload(g, dev, c.c_lh.data(), m, &d.c_lh));
    RC(warm_upload(g, dev, c.c_hl.data(), m, &d.c_hl));
    return MGC_OK;
}

// constant of a fold: fixed-order per-block partials summed by one block
int warm_constant(mgc_sparse* g, DevScope& dev, const double* partials, long long nb, double* out)
{
    double* d_out;
    CK(dev.alloc(&d_out, 1));
    k_spw_sum_partials<<<1, 256>>>(partials, nb, d_out);
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, d_out, sizeof(double), cudaMemcpyDeviceToHost));
    return MGC_OK;
}

// the end of a timed fold: its time and count into the stats
int fold_done(mgc_sparse* g, const Events& ev)
{
    CK(cudaEventRecord(ev.stop, 0));
    CK(cudaEventSynchronize(ev.stop));
    float ms = 0.f;
    ev.elapsed(&ms);
    g->st.seed_folds++;
    g->st.ms_seeds += ms;
    return MGC_OK;
}

int warm_fold_tweights(mgc_sparse* g, int64_t count, const int32_t* nodes, const double* src, const double* snk)
{
    CK(cudaSetDevice(g->device));
    Events ev;
    CK(ev.begin());
    DevScope dev;
    std::vector<unsigned> keys((size_t)count);
    for (int64_t k = 0; k < count; ++k) keys[(size_t)k] = (unsigned)(nodes ? nodes[k] : k);
    unsigned *ks, *order;
    RC(warm_group(g, dev, keys, (unsigned)(g->host.n - 1), &ks, &order));
    double *d_src, *d_snk, *partials;
    const long long nb = (count + 255) / 256;
    RC(warm_upload(g, dev, src, (size_t)count, &d_src));
    RC(warm_upload(g, dev, snk, (size_t)count, &d_snk));
    CK(dev.alloc(&partials, (size_t)nb));
    k_spw_tlink_fold<<<(unsigned)nb, 256>>>(g->dev.warm(), ks, order, count, d_src, d_snk, partials);
    g->st.kernel_launches++;
    double dk = 0.0;
    RC(warm_constant(g, dev, partials, nb, &dk));
    g->wconst += dk;
    return fold_done(g, ev);
}

// sum_edge calls resolved to pairs; the pairs from `first_fresh` on are new, in creation order
int warm_fold_edges(mgc_sparse* g, const SparseCalls& c, int64_t first_fresh)
{
    CK(cudaSetDevice(g->device));
    Events ev;
    CK(ev.begin());
    DevScope dev;
    const SparseHost& h = g->host;
    SparseDev& d = g->dev;
    const int n = (int)h.n;
    const unsigned blocks = grid_for(n);
    const int64_t np = (int64_t)h.plo.size();
    const int64_t q = np - first_fresh;
    if (q > 0) {
        // device CSR re-assembly: every residual carried over, old arcs first, new pairs after them in creation order
        // (the arc order a cold build of the same call sequence gives)
        int *d_qlo, *d_qhi, *d_qol, *d_qoh;
        RC(warm_upload(g, dev, h.plo.data() + first_fresh, (size_t)q, &d_qlo));
        RC(warm_upload(g, dev, h.phi.data() + first_fresh, (size_t)q, &d_qhi));
        RC(warm_upload(g, dev, h.olo.data() + first_fresh, (size_t)q, &d_qol));
        RC(warm_upload(g, dev, h.ohi.data() + first_fresh, (size_t)q, &d_qoh));
        unsigned* cnt;
        unsigned long long* off;
        CK(dev.alloc(&cnt, (size_t)n));
        CK(dev.alloc(&off, (size_t)n + 1));
        CK(cudaMemset(cnt, 0, (size_t)n * sizeof(unsigned)));
        const unsigned qb = (unsigned)((q + 255) / 256);
        k_spw_count_new<<<qb, 256>>>(d_qlo, d_qhi, q, cnt);
        k_spw_degree<<<blocks, 256>>>(d.row, n, cnt);
        lab_scan_blocks(cnt, (long long)n, off);
        g->st.kernel_launches += 3;
        const int m2n = (int)(2 * np);
        DevScope fresh;                                 // the new arrays trade places with the old, which it then frees
        int *row, *head, *sis;
        double* cap;
        CK(fresh.alloc(&row, (size_t)n + 1));
        CK(fresh.alloc(&head, (size_t)m2n));
        CK(fresh.alloc(&sis, (size_t)m2n));
        CK(fresh.alloc(&cap, (size_t)m2n));
        k_spw_row<<<blocks, 256>>>(off, n, row);
        k_spw_move<<<blocks, 256>>>(n, d.row, d.head, d.sis, d.cap, row, head, sis, cap);
        k_spw_new_pairs<<<qb, 256>>>(d_qlo, d_qhi, d_qol, d_qoh, q, row, head, sis, cap);
        g->st.kernel_launches += 3;
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        fresh.trade(row, d.row);
        fresh.trade(head, d.head);
        fresh.trade(sis, d.sis);
        fresh.trade(cap, d.cap);
        d.m2 = m2n;
    }
    const long long m = (long long)c.pk.size();
    DevCalls a;
    RC(warm_calls(g, dev, c, a));
    const SparseWarm W = d.warm();
    k_spw_pair_inc<<<(unsigned)((m + 255) / 256), 256>>>(W, a.keys, a.order, m, a.lo, a.hi, a.olo, a.ohi, a.c_lh, a.c_hl, d.tail);
    k_spw_reclamp<<<blocks, 256>>>(W, d.tail);
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    return fold_done(g, ev);
}

// remove_edges_warm calls resolved to pairs, the decrements oriented lo->hi / hi->lo
int warm_fold_decrements(mgc_sparse* g, const SparseCalls& c)
{
    CK(cudaSetDevice(g->device));
    DevScope dev;
    const long long m = (long long)c.pk.size();
    DevCalls a;
    RC(warm_calls(g, dev, c, a));
    int* refused;
    CK(dev.alloc(&refused, 1));
    CK(cudaMemset(refused, 0, sizeof(int)));
    const SparseWarm W = g->dev.warm();
    const unsigned mb = (unsigned)((m + 255) / 256);
    k_spw_pair_check<<<mb, 256>>>(W, a.keys, a.order, m, a.lo, a.hi, a.olo, a.ohi, a.c_lh, a.c_hl, refused);
    g->st.kernel_launches++;
    int bad = 0;
    CK(cudaMemcpy(&bad, refused, sizeof(int), cudaMemcpyDeviceToHost));
    if (bad)
        FAIL(MGC_E_WEIGHT, "remove_edges_warm: a pair's decrements exceed its capacities r(i->j) + r(j->i) (the graph is "
                             "unchanged)");
    // arcs, then every end once in ascending node order with its changes in a fixed order
    unsigned *end_key, *end_ks, *end_order;
    double *end_dx, *partials;
    CK(dev.alloc(&end_key, (size_t)(2 * m)));
    CK(dev.alloc(&end_dx, (size_t)(2 * m)));
    k_spw_pair_dec<<<mb, 256>>>(W, a.keys, a.order, m, a.lo, a.hi, a.olo, a.ohi, a.c_lh, a.c_hl, end_key, end_dx);
    g->st.kernel_launches++;
    RC(warm_sort(g, dev, end_key, 2 * m, 0xffffffffu, &end_ks, &end_order));
    const long long nb = (2 * m + 255) / 256;
    CK(dev.alloc(&partials, (size_t)nb));
    k_spw_ends<<<(unsigned)nb, 256>>>(W, end_ks, end_order, 2 * m, end_dx, partials);
    g->st.kernel_launches++;
    double dk = 0.0;
    RC(warm_constant(g, dev, partials, nb, &dk));
    g->wconst += dk;
    g->st.seed_folds++;
    return MGC_OK;
}

const char* const warm_bad_msg =
    "the first solve of this warm graph held a NaN or infinite capacity or t-link, so it has no residual state to fold "
    "into: reset() and rebuild the graph";

// sum_edge calls on a solved warm handle: the host mirror accumulates as on a cold graph, the resident state folds
int warm_sum_edges(mgc_sparse* g, int64_t count, const int32_t* i, const int32_t* j, const double* cap, const double* rev_cap)
{
    if (g->warm_bad) FAIL(MGC_E_STATE, warm_bad_msg);
    for (int64_t k = 0; k < count; ++k) {
        if (!std::isfinite(cap[k]) || !std::isfinite(rev_cap[k])) FAIL(MGC_E_ARG, "edge capacities hold NaN or infinite values");
        if (cap[k] < 0 || rev_cap[k] < 0)
            FAIL(MGC_E_ARG, "a negative capacity cannot fold into a solved graph: lower capacities with remove_edges_warm");
    }
    if (count == 0) return MGC_OK;
    if (2 * ((int64_t)g->host.plo.size() + count) >= (int64_t)INT32_MAX) FAIL(MGC_E_ARG, "too many arcs for 32-bit arc ids");
    const int64_t first_fresh = (int64_t)g->host.plo.size();
    SparseCalls c;
    g->host.resolve(count, i, j, cap, rev_cap, true, c);
    g->host.add(c);
    g->solved = false;
    return warm_fold_edges(g, c, first_fresh);
}

}  // namespace

extern "C" {

int mgc_sparse_create(int64_t n_nodes, int32_t device, mgc_sparse** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    if (n_nodes < 1 || n_nodes >= (int64_t)INT32_MAX) { g_sp_create_error = "node count must be in [1, 2^31-2]"; return MGC_E_ARG; }
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count < 1) {
        cudaGetLastError();
        g_sp_create_error = "no CUDA device available (this library has no CPU solver)";
        return MGC_E_CUDA;
    }
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
    if (device >= count) { g_sp_create_error = "invalid CUDA device ordinal"; return MGC_E_ARG; }
    mgc_sparse* g = new mgc_sparse();
    g->device = device;
    g->host = SparseHost(n_nodes);
    if (const char* e = std::getenv("MEDPY_GC_SPARSE_TIMEOUT")) { const double v = std::atof(e); if (v > 0) g->max_seconds = v; }
    if (const char* e = std::getenv("MEDPY_GC_SPARSE_SWEEPS")) { const int v = std::atoi(e); if (v > 0) g->sweeps_per_round = v; }
    *out = g;
    return MGC_OK;
}

void mgc_sparse_destroy(mgc_sparse* g) { delete g; }

int mgc_sparse_reset(mgc_sparse* g)
{
    if (!g) return MGC_E_ARG;
    g->host = SparseHost(g->host.n);
    g->solved = false;
    g->energy = 0.0;
    g->mask.clear();
    g->st = mgc_stats{};
    g->release();                   // the warm option itself stays
    g->solved_once = false;
    g->warm_bad = false;
    g->wconst = 0.0;
    return MGC_OK;
}

int mgc_sparse_set_option(mgc_sparse* g, int32_t option, int64_t value)
{
    if (!g) return MGC_E_ARG;
    if (option != MGC_OPT_WARM) FAIL(MGC_E_ARG, "unknown option for a sparse graph");
    if (g->solved_once || g->resident)
        FAIL(MGC_E_STATE, "MGC_OPT_WARM must be set before the first maxflow(): reset() the graph and rebuild it");
    g->warm = value != 0;
    return MGC_OK;
}

const char* mgc_sparse_last_error(const mgc_sparse* g) { return g ? g->err.c_str() : g_sp_create_error.c_str(); }

int mgc_sparse_sum_edges(mgc_sparse* g, int64_t count, const int32_t* i, const int32_t* j, const double* cap, const double* rev_cap)
{
    if (!g) return MGC_E_ARG;
    if (count < 0 || (count > 0 && (!i || !j || !cap || !rev_cap))) FAIL(MGC_E_ARG, "null edge arrays");
    for (int64_t k = 0; k < count; ++k) {
        const int64_t a = i[k], b = j[k];
        if (a < 0 || b < 0 || a >= g->host.n || b >= g->host.n)
            FAIL(MGC_E_ARG, "Invalid node id in edge (" + std::to_string(a) + ", " + std::to_string(b) + "). Valid values are 0 to " +
                                  std::to_string(g->host.n - 1) + ".");
        if (a == b) FAIL(MGC_E_ARG, "The node_from (" + std::to_string(a) + ") can not be equal to the node_to (" + std::to_string(b) + ") (self-connections are forbidden in graph-cuts).");
    }
    if (g->resident) return warm_sum_edges(g, count, i, j, cap, rev_cap);
    g->host.sum_edges(count, i, j, cap, rev_cap);
    if (count) g->solved = false;
    return MGC_OK;
}

int mgc_sparse_add_tweights(mgc_sparse* g, int64_t count, const int32_t* nodes, const double* src, const double* snk)
{
    if (!g) return MGC_E_ARG;
    if (count < 0 || (count > 0 && (!src || !snk))) FAIL(MGC_E_ARG, "null t-weight arrays");
    if (!nodes && count > g->host.n) FAIL(MGC_E_ARG, "more t-weights than nodes");
    if (nodes)
        for (int64_t k = 0; k < count; ++k)
            if (nodes[k] < 0 || nodes[k] >= g->host.n)
                FAIL(MGC_E_ARG, "Invalid node id of " + std::to_string(nodes[k]) + ". Valid values are 0 to " + std::to_string(g->host.n - 1) + ".");
    if (g->resident) {
        if (g->warm_bad) FAIL(MGC_E_STATE, warm_bad_msg);
        for (int64_t k = 0; k < count; ++k)
            if (!std::isfinite(src[k]) || !std::isfinite(snk[k])) FAIL(MGC_E_ARG, "t-weights hold NaN or infinite values");
        if (count == 0) return MGC_OK;
        int rc = warm_fold_tweights(g, count, nodes, src, snk);
        if (rc) return rc;
    }
    g->host.add_tweights(count, nodes, src, snk);
    if (count) g->solved = false;
    return MGC_OK;
}

int mgc_sparse_remove_edges_warm(mgc_sparse* g, int64_t count, const int32_t* i, const int32_t* j, const double* cap,
                                 const double* rev_cap)
{
    if (!g) return MGC_E_ARG;
    if (!g->warm)
        FAIL(MGC_E_STATE, "remove_edges_warm needs a graph created with the warm option (MGC_OPT_WARM): reset() the graph "
                            "and rebuild it without the weight instead");
    if (count < 0 || (count > 0 && (!i || !j || !cap || !rev_cap))) FAIL(MGC_E_ARG, "null edge arrays");
    for (int64_t k = 0; k < count; ++k) {
        if (i[k] < 0 || j[k] < 0 || i[k] >= g->host.n || j[k] >= g->host.n || i[k] == j[k])
            FAIL(MGC_E_ARG, "invalid node ids (" + std::to_string(i[k]) + ", " + std::to_string(j[k]) + ")");
        if (!std::isfinite(cap[k]) || !std::isfinite(rev_cap[k])) FAIL(MGC_E_ARG, "decrements hold NaN or infinite values");
        if (cap[k] < 0 || rev_cap[k] < 0) FAIL(MGC_E_WEIGHT, "decrements are nonnegative amounts");
    }
    if (g->resident && g->warm_bad) FAIL(MGC_E_STATE, warm_bad_msg);
    if (count == 0) return MGC_OK;
    SparseCalls c;
    const int64_t k = g->host.resolve(count, i, j, cap, rev_cap, false, c);
    if (k >= 0)
        FAIL(MGC_E_ARG, "no edge between nodes " + std::to_string(i[k]) + " and " + std::to_string(j[k]) +
                              ": remove_edges_warm lowers existing capacities");
    // per pair: the decrements summed in call order, pairs in order of their first call
    std::vector<unsigned> pairs;
    std::vector<double> sl, sh;
    SparseHost::pair_sums(c, pairs, sl, sh);
    if (g->resident) {
        RC(warm_fold_decrements(g, c));
    } else {
        // before the first solve: the same pair rule on the accumulated capacities
        for (size_t q = 0; q < pairs.size(); ++q)
            if (spw_pair_refused(g->host.cap_lh[pairs[q]], g->host.cap_hl[pairs[q]], sl[q], sh[q]))
                FAIL(MGC_E_WEIGHT, "remove_edges_warm: a pair's decrements exceed its capacities c(i->j) + c(j->i) (the graph "
                                     "is unchanged)");
    }
    g->host.lower(pairs, sl, sh);
    g->solved = false;
    return MGC_OK;
}

int mgc_sparse_maxflow(mgc_sparse* g, double* energy)
{
    if (!g) return MGC_E_ARG;
    if (!g->solved) {
        int rc = sparse_solve(g);
        if (rc) return rc;
    }
    if (energy) *energy = g->energy;
    return MGC_OK;
}

int mgc_sparse_get_mask(mgc_sparse* g, uint8_t* out)
{
    if (!g || !out) return MGC_E_ARG;
    if (!g->solved) { int rc = sparse_solve(g); if (rc) return rc; }
    std::memcpy(out, g->mask.data(), (size_t)g->host.n);
    return MGC_OK;
}

int mgc_sparse_what_segment(mgc_sparse* g, int64_t node, int32_t* segment)
{
    if (!g || !segment) return MGC_E_ARG;
    if (node < 0 || node >= g->host.n) FAIL(MGC_E_ARG, "node id out of range");
    if (!g->solved) { int rc = sparse_solve(g); if (rc) return rc; }
    *segment = g->mask[(size_t)node] ? MGC_SOURCE : MGC_SINK;
    return MGC_OK;
}

int mgc_sparse_get_edge(const mgc_sparse* g, int64_t i, int64_t j, double* cap)
{
    if (!g || !cap) return MGC_E_ARG;
    SparseHost& h = const_cast<mgc_sparse*>(g)->host;
    h.ensure_index();                                   // the index is a cache: building it does not change the graph
    *cap = 0.0;
    if (i < 0 || j < 0 || i >= h.n || j >= h.n || i == j) return MGC_OK;
    const bool fwd = i < j;
    const int64_t p = h.find((int32_t)(fwd ? i : j), (int32_t)(fwd ? j : i));
    if (p >= 0) *cap = fwd ? h.cap_lh[(size_t)p] : h.cap_hl[(size_t)p];
    return MGC_OK;
}

int mgc_sparse_get_trcap(const mgc_sparse* g, int64_t node, double* trcap)
{
    if (!g || !trcap || node < 0 || node >= g->host.n) return MGC_E_ARG;
    *trcap = g->host.tr[(size_t)node];
    return MGC_OK;
}

int mgc_sparse_get_node_num(const mgc_sparse* g, int64_t* n) { if (!g || !n) return MGC_E_ARG; *n = g->host.n; return MGC_OK; }
int mgc_sparse_get_arc_num(const mgc_sparse* g, int64_t* n) { if (!g || !n) return MGC_E_ARG; *n = 2 * (int64_t)g->host.plo.size(); return MGC_OK; }
int mgc_sparse_get_stats(const mgc_sparse* g, mgc_stats* out) { if (!g || !out) return MGC_E_ARG; *out = g->st; return MGC_OK; }

}  // extern "C"