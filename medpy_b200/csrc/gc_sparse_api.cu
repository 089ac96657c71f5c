// gc_sparse_api.cu -- host side of the C ABI for general sparse graphs and label images
// (include/medpy_b200_graphcut.h, sections "general sparse graphs" and "label images"; SURVEY.md §8 rows f3/f4).
//
// mgc_sparse keeps what the reference's Graph<> keeps on the host while a graph is assembled -- the arc pairs in
// insertion order with accumulated capacities (graph.h:427-480) and tr_cap / flow per add_tweights (graph.h:415-425);
// these are O(1) updates per call exactly like the reference's -- and runs the max-flow on the device
// (gc_sparse.cuh).  mgc_labels keeps a label image resident in HBM and reduces voxel-scale data to the region
// adjacency graph there (gc_labels.cuh); only per-region / per-region-pair results ever reach the host.
// The stable radix sort that orders the contributions by key is cub::DeviceRadixSort (CUDA toolkit).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <unordered_map>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cuda_runtime.h>

#include "../../include/medpy_b200_graphcut.h"
#include "gc_host.hpp"
#include "gc_labels.cuh"
#include "gc_sparse.cuh"
#include "gc_sparse_warm.cuh"

namespace {

thread_local std::string g_sp_create_error;
thread_local std::string g_lab_create_error;

// device allocations of one call, released together
struct DevScope {
    std::vector<void*> ptrs;
    ~DevScope() { for (void* p : ptrs) cudaFree(p); }
    template <typename T>
    cudaError_t alloc(T** out, size_t count)
    {
        void* p = nullptr;
        cudaError_t e = cudaMalloc(&p, (count ? count : 1) * sizeof(T));
        if (e == cudaSuccess) ptrs.push_back(p);
        *out = (T*)p;
        return e;
    }
};

// grid of the grid-stride kernels: one block per LAB_BLOCK items, at most 32 blocks per SM of the current device
unsigned grid_for(long long n)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
    const long long cap = 32LL * cached_sm_count(dev);
    long long b = (n + LAB_BLOCK - 1) / LAB_BLOCK;
    if (b < 1) b = 1;
    return (unsigned)(b < cap ? b : cap);
}

}  // namespace

// =================================================================================================================
// sparse graph
// =================================================================================================================
struct mgc_sparse {
    int device = 0;
    int64_t n = 0;
    std::vector<double> tr;                            // net terminal capacity per node
    double flow_const = 0.0;                           // sum of the add_tweights minima (graph.h:423)
    std::unordered_map<uint64_t, int64_t> pair_of;     // (lo << 32 | hi) -> index into the pair arrays (built on demand)
    bool indexed = true;                               // pair_of covers every pair
    std::vector<int32_t> plo, phi;                     // node pairs in insertion order, lo < hi
    std::vector<double> cap_lh, cap_hl;                // capacity lo->hi, hi->lo
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
    std::vector<int32_t> olo, ohi;                     // per pair: node-local offsets of its arcs lo->hi and hi->lo
    std::vector<int32_t> deg;                          // arcs per node
    int m2 = 0;                                        // resident arcs
    struct {
        int *row = nullptr, *head = nullptr, *sis = nullptr, *height = nullptr, *flags = nullptr;
        double *cap = nullptr, *tr = nullptr, *excess = nullptr, *sunk = nullptr, *sent = nullptr, *abs = nullptr;
        uint8_t *mask = nullptr, *tail = nullptr;
        unsigned long long* count = nullptr;
    } dev;
    void release()
    {
        if (!resident) return;
        cudaSetDevice(device);
        void* ps[] = {dev.row, dev.head, dev.sis, dev.height, dev.flags, dev.cap, dev.tr, dev.excess, dev.sunk, dev.sent,
                      dev.abs, dev.mask, dev.tail, dev.count};
        for (void* p : ps) cudaFree(p);
        dev = {};
        resident = false;
    }
    ~mgc_sparse() { release(); }
};

namespace {

void sparse_ensure_index(mgc_sparse* g)
{
    if (g->indexed) return;
    g->pair_of.clear();
    g->pair_of.reserve(g->plo.size() * 2);
    for (size_t p = 0; p < g->plo.size(); ++p)
        g->pair_of.emplace(((uint64_t)(uint32_t)g->plo[p] << 32) | (uint32_t)g->phi[p], (int64_t)p);
    g->indexed = true;
}

// The push-relabel loop from the first exact global relabel to the stop test, then the read-out: the whole solve of a
// warm re-solve, the rest of a first solve after its init.
int sparse_loop(mgc_sparse* g, const SparseState& S, int* d_flags, unsigned long long* d_count, uint8_t* d_mask,
                double* d_abs, cudaEvent_t ev0, cudaEvent_t ev1, double base)
{
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
        CK(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), 0));
        k_sp_count_active<<<blocks, 256>>>(S, d_count);
        g->st.kernel_launches++;
        unsigned long long c = 0;
        CK(cudaMemcpy(&c, d_count, sizeof(c), cudaMemcpyDeviceToHost));
        active = (long long)c;
        if (!active) break;
        const double elapsed = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
        if (++rounds > g->max_rounds || elapsed > g->max_seconds) {
            cudaEventDestroy(ev0); cudaEventDestroy(ev1);
            FAIL(MGC_E_NOCONV, "sparse push-relabel did not converge within " + std::to_string(rounds) + " rounds / " +
                                     std::to_string(elapsed) + " s (" + std::to_string(active) + " active nodes left)");
        }
        for (int s = 0; s < g->sweeps_per_round; ++s) k_sp_push<<<blocks, 256>>>(S, g->push_steps, d_flags + 1);
        g->st.kernel_launches += g->sweeps_per_round;
        g->st.push_sweeps += g->sweeps_per_round;
    }
    k_sp_readout<<<1, 256>>>(S, d_mask, d_abs);
    g->st.kernel_launches++;
    CK(cudaEventRecord(ev1, 0));
    CK(cudaGetLastError());
    g->mask.assign((size_t)n, 0);
    double absorbed = 0.0;
    CK(cudaMemcpy(g->mask.data(), d_mask, (size_t)n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&absorbed, d_abs, sizeof(double), cudaMemcpyDeviceToHost));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ev0, ev1));
    cudaEventDestroy(ev0);
    cudaEventDestroy(ev1);
    g->energy = base + absorbed;
    g->solved = true;
    g->solved_once = true;
    g->st.n_voxels = n;
    g->st.ms_solve = ms;
    g->st.active_last = active;
    g->st.flow_const = g->flow_const;
    g->st.energy = g->energy;
    g->st.device_bytes = (int64_t)((size_t)S.m2 * 16 + (size_t)n * (g->warm ? 41 : 33));
    return MGC_OK;
}

SparseState warm_state(const mgc_sparse* g)
{
    SparseState S{};
    S.n = (int)g->n; S.m2 = g->m2; S.row = g->dev.row; S.head = g->dev.head; S.sis = g->dev.sis; S.cap = g->dev.cap;
    S.tr = g->dev.tr; S.excess = g->dev.excess; S.sunk = g->dev.sunk; S.height = g->dev.height;
    return S;
}

SparseWarm warm_view(const mgc_sparse* g)
{
    SparseWarm W{};
    W.n = (int)g->n; W.row = g->dev.row; W.head = g->dev.head; W.cap = g->dev.cap; W.tr = g->dev.tr;
    W.excess = g->dev.excess; W.sunk = g->dev.sunk; W.sent = g->dev.sent;
    return W;
}

// a warm handle with a resident state: the loop only
int sparse_resolve(mgc_sparse* g)
{
    CK(cudaSetDevice(g->device));
    cudaEvent_t ev0, ev1;
    CK(cudaEventCreate(&ev0));
    CK(cudaEventCreate(&ev1));
    CK(cudaEventRecord(ev0, 0));
    return sparse_loop(g, warm_state(g), g->dev.flags, g->dev.count, g->dev.mask, g->dev.abs, ev0, ev1, g->wconst);
}

int sparse_solve(mgc_sparse* g)
{
    if (g->resident) return sparse_resolve(g);
    CK(cudaSetDevice(g->device));
    const int n = (int)g->n;
    const int64_t np = (int64_t)g->plo.size();
    if (2 * np >= (int64_t)INT32_MAX) FAIL(MGC_E_ARG, "too many arcs for 32-bit arc ids");
    const int m2 = (int)(2 * np);
    // CSR in insertion order of the pairs (the order add_edge appends arcs to a node's list, graph.h:443-452)
    std::vector<int> row((size_t)n + 1, 0), head((size_t)m2), sis((size_t)m2);
    std::vector<double> cap((size_t)m2);
    for (int64_t p = 0; p < np; ++p) { row[(size_t)g->plo[p] + 1]++; row[(size_t)g->phi[p] + 1]++; }
    for (int v = 0; v < n; ++v) row[(size_t)v + 1] += row[(size_t)v];
    {
        std::vector<int> fill(row.begin(), row.end() - 1);
        for (int64_t p = 0; p < np; ++p) {
            const int a = fill[(size_t)g->plo[p]]++, b = fill[(size_t)g->phi[p]]++;
            head[(size_t)a] = g->phi[p]; head[(size_t)b] = g->plo[p];
            sis[(size_t)a] = b; sis[(size_t)b] = a;
            cap[(size_t)a] = g->cap_lh[p]; cap[(size_t)b] = g->cap_hl[p];
        }
    }
    DevScope dev;
    SparseState S{};
    int *d_row, *d_head, *d_sis, *d_height, *d_flags;
    double *d_cap, *d_tr, *d_excess, *d_sunk, *d_abs;
    uint8_t* d_mask;
    unsigned long long* d_count;
    CK(dev.alloc(&d_row, (size_t)n + 1));
    CK(dev.alloc(&d_head, (size_t)m2));
    CK(dev.alloc(&d_sis, (size_t)m2));
    CK(dev.alloc(&d_cap, (size_t)m2));
    CK(dev.alloc(&d_tr, (size_t)n));
    CK(dev.alloc(&d_excess, (size_t)n));
    CK(dev.alloc(&d_sunk, (size_t)n));
    CK(dev.alloc(&d_height, (size_t)n));
    CK(dev.alloc(&d_mask, (size_t)n));
    CK(dev.alloc(&d_flags, 2));
    CK(dev.alloc(&d_abs, 1));
    CK(dev.alloc(&d_count, 1));
    CK(cudaMemcpy(d_row, row.data(), ((size_t)n + 1) * sizeof(int), cudaMemcpyHostToDevice));
    if (m2) {
        CK(cudaMemcpy(d_head, head.data(), (size_t)m2 * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_sis, sis.data(), (size_t)m2 * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_cap, cap.data(), (size_t)m2 * sizeof(double), cudaMemcpyHostToDevice));
    }
    CK(cudaMemcpy(d_tr, g->tr.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
    S.n = n; S.m2 = m2; S.row = d_row; S.head = d_head; S.sis = d_sis; S.cap = d_cap; S.tr = d_tr;
    S.excess = d_excess; S.sunk = d_sunk; S.height = d_height;

    double* d_sent = nullptr;
    uint8_t* d_tail = nullptr;
    if (g->warm) {
        CK(dev.alloc(&d_sent, (size_t)n));
        CK(dev.alloc(&d_tail, (size_t)n));
        CK(cudaMemset(d_tail, 0, (size_t)n));
    }
    cudaEvent_t ev0, ev1;
    CK(cudaEventCreate(&ev0));
    CK(cudaEventCreate(&ev1));
    CK(cudaEventRecord(ev0, 0));
    const unsigned blocks = grid_for(n);
    if (g->warm) {
        SparseWarm W{};
        W.n = n; W.row = d_row; W.head = d_head; W.cap = d_cap; W.tr = d_tr; W.excess = d_excess; W.sunk = d_sunk; W.sent = d_sent;
        k_spw_init<<<blocks, 256>>>(W);
    } else {
        k_sp_init<<<blocks, 256>>>(S);
    }
    g->st.kernel_launches++;
    if (!g->warm) return sparse_loop(g, S, d_flags, d_count, d_mask, d_abs, ev0, ev1, g->flow_const);
    // warm: the state stays resident whether the loop converges or not; so do the pairs' arc offsets
    g->dev.row = d_row; g->dev.head = d_head; g->dev.sis = d_sis; g->dev.height = d_height; g->dev.flags = d_flags;
    g->dev.cap = d_cap; g->dev.tr = d_tr; g->dev.excess = d_excess; g->dev.sunk = d_sunk; g->dev.sent = d_sent;
    g->dev.abs = d_abs; g->dev.mask = d_mask; g->dev.tail = d_tail; g->dev.count = d_count;
    dev.ptrs.clear();
    g->resident = true;
    g->m2 = m2;
    g->wconst = g->flow_const;
    bool bad = false;
    for (int v = 0; v < n && !bad; ++v) bad = !std::isfinite(g->tr[(size_t)v]);
    for (int a = 0; a < m2 && !bad; ++a) bad = !std::isfinite(cap[(size_t)a]);
    g->warm_bad = bad;
    g->deg.assign((size_t)n, 0);
    g->olo.resize((size_t)np);
    g->ohi.resize((size_t)np);
    for (int64_t p = 0; p < np; ++p) {
        g->olo[(size_t)p] = g->deg[(size_t)g->plo[p]]++;
        g->ohi[(size_t)p] = g->deg[(size_t)g->phi[p]]++;
    }
    return sparse_loop(g, S, d_flags, d_count, d_mask, d_abs, ev0, ev1, g->wconst);
}

// ---- folds into the resident state of a warm handle ------------------------------------------------------------
int warm_sort(mgc_sparse* g, DevScope& dev, unsigned* keys, unsigned* idx, long long m, unsigned key_max,
              unsigned* keys_sorted, unsigned* order, bool iota);

// The calls are grouped on the device: (key, call index) pairs through a stable radix sort, so each key's calls keep
// their order; the first slot of every run of equal keys does the work (gc_sparse_warm.cuh).
int warm_group(mgc_sparse* g, DevScope& dev, const unsigned* h_keys, long long m, unsigned key_max,
               unsigned** keys_sorted, unsigned** order)
{
    unsigned *keys, *idx;
    CK(dev.alloc(&keys, (size_t)m));
    CK(dev.alloc(&idx, (size_t)m));
    CK(dev.alloc(keys_sorted, (size_t)m));
    CK(dev.alloc(order, (size_t)m));
    if (h_keys) CK(cudaMemcpy(keys, h_keys, (size_t)m * sizeof(unsigned), cudaMemcpyHostToDevice));
    return warm_sort(g, dev, keys, idx, m, key_max, *keys_sorted, *order, true);
}

int warm_sort(mgc_sparse* g, DevScope& dev, unsigned* keys, unsigned* idx, long long m, unsigned key_max,
              unsigned* keys_sorted, unsigned* order, bool iota)
{
    const unsigned mb = (unsigned)((m + 255) / 256);
    if (iota) { k_spw_iota<<<mb, 256>>>(idx, m); g->st.kernel_launches++; }
    const int end_bit = bits_for(key_max);
    size_t tb = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keys_sorted, idx, order, (int)m, 0, end_bit, 0));
    char* tmp;
    CK(dev.alloc(&tmp, tb));
    CK(cub::DeviceRadixSort::SortPairs(tmp, tb, keys, keys_sorted, idx, order, (int)m, 0, end_bit, 0));
    g->st.kernel_launches += 4;
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

template <typename T>
int warm_upload(mgc_sparse* g, DevScope& dev, const std::vector<T>& h, T** d)
{
    CK(dev.alloc(d, h.size()));
    if (!h.empty()) CK(cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    return MGC_OK;
}

int warm_fold_tweights(mgc_sparse* g, int64_t count, const int32_t* nodes, const double* src, const double* snk)
{
    CK(cudaSetDevice(g->device));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0, 0));
    DevScope dev;
    std::vector<unsigned> keys((size_t)count);
    for (int64_t k = 0; k < count; ++k) keys[(size_t)k] = (unsigned)(nodes ? nodes[k] : k);
    unsigned *ks, *order;
    RC(warm_group(g, dev, keys.data(), count, (unsigned)(g->n - 1), &ks, &order));
    double *d_src, *d_snk, *partials;
    const long long nb = (count + 255) / 256;
    CK(dev.alloc(&d_src, (size_t)count));
    CK(dev.alloc(&d_snk, (size_t)count));
    CK(dev.alloc(&partials, (size_t)nb));
    CK(cudaMemcpy(d_src, src, (size_t)count * sizeof(double), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_snk, snk, (size_t)count * sizeof(double), cudaMemcpyHostToDevice));
    k_spw_tlink_fold<<<(unsigned)nb, 256>>>(warm_view(g), ks, order, count, d_src, d_snk, partials);
    g->st.kernel_launches++;
    double dk = 0.0;
    RC(warm_constant(g, dev, partials, nb, &dk));
    g->wconst += dk;
    CK(cudaEventRecord(e1, 0));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    g->st.seed_folds++;
    g->st.ms_seeds += ms;
    return MGC_OK;
}

// one call per pair index `pk` (lo / hi / offsets per call, capacities oriented lo->hi / hi->lo); `fresh` lists the
// pairs the calls created, in creation order
int warm_fold_edges(mgc_sparse* g, const std::vector<unsigned>& pk, const std::vector<int32_t>& lo, const std::vector<int32_t>& hi,
                    const std::vector<int32_t>& olo, const std::vector<int32_t>& ohi, const std::vector<double>& c_lh,
                    const std::vector<double>& c_hl, int64_t first_fresh)
{
    CK(cudaSetDevice(g->device));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0, 0));
    DevScope dev;
    const int n = (int)g->n;
    const unsigned blocks = grid_for(n);
    const int64_t np = (int64_t)g->plo.size();
    const int64_t q = np - first_fresh;
    if (q > 0) {
        // device CSR re-assembly: every residual carried over, old arcs first, new pairs after them in creation order
        // (the arc order a cold build of the same call sequence gives)
        const int m2n = (int)(2 * np);
        std::vector<int32_t> qlo(g->plo.begin() + first_fresh, g->plo.end()), qhi(g->phi.begin() + first_fresh, g->phi.end());
        std::vector<int32_t> qol(g->olo.begin() + first_fresh, g->olo.end()), qoh(g->ohi.begin() + first_fresh, g->ohi.end());
        int *d_qlo, *d_qhi, *d_qol, *d_qoh;
        RC(warm_upload(g, dev, qlo, &d_qlo));
        RC(warm_upload(g, dev, qhi, &d_qhi));
        RC(warm_upload(g, dev, qol, &d_qol));
        RC(warm_upload(g, dev, qoh, &d_qoh));
        unsigned* cnt;
        unsigned long long* off;
        CK(dev.alloc(&cnt, (size_t)n));
        CK(dev.alloc(&off, (size_t)n + 1));
        CK(cudaMemset(cnt, 0, (size_t)n * sizeof(unsigned)));
        const unsigned qb = (unsigned)((q + 255) / 256);
        k_spw_count_new<<<qb, 256>>>(d_qlo, d_qhi, q, cnt);
        k_spw_degree<<<blocks, 256>>>(g->dev.row, n, cnt);
        k_lab_scan_blocks<<<1, 1024>>>(cnt, (long long)n, off);
        g->st.kernel_launches += 3;
        int *row, *head, *sis;
        double* cap;
        {
            DevScope keep;
            CK(keep.alloc(&row, (size_t)n + 1));
            CK(keep.alloc(&head, (size_t)m2n));
            CK(keep.alloc(&sis, (size_t)m2n));
            CK(keep.alloc(&cap, (size_t)m2n));
            k_spw_row<<<blocks, 256>>>(off, n, row);
            k_spw_move<<<blocks, 256>>>(n, g->dev.row, g->dev.head, g->dev.sis, g->dev.cap, row, head, sis, cap);
            k_spw_new_pairs<<<qb, 256>>>(d_qlo, d_qhi, d_qol, d_qoh, q, row, head, sis, cap);
            g->st.kernel_launches += 3;
            CK(cudaGetLastError());
            CK(cudaDeviceSynchronize());
            keep.ptrs.clear();
        }
        cudaFree(g->dev.row); cudaFree(g->dev.head); cudaFree(g->dev.sis); cudaFree(g->dev.cap);
        g->dev.row = row; g->dev.head = head; g->dev.sis = sis; g->dev.cap = cap;
        g->m2 = m2n;
    }
    const long long m = (long long)pk.size();
    unsigned *ks, *order;
    RC(warm_group(g, dev, pk.data(), m, (unsigned)(np > 0 ? np - 1 : 0), &ks, &order));
    int *d_lo, *d_hi, *d_ol, *d_oh;
    double *d_cl, *d_ch;
    RC(warm_upload(g, dev, lo, &d_lo));
    RC(warm_upload(g, dev, hi, &d_hi));
    RC(warm_upload(g, dev, olo, &d_ol));
    RC(warm_upload(g, dev, ohi, &d_oh));
    RC(warm_upload(g, dev, c_lh, &d_cl));
    RC(warm_upload(g, dev, c_hl, &d_ch));
    const SparseWarm W = warm_view(g);
    k_spw_pair_inc<<<(unsigned)((m + 255) / 256), 256>>>(W, ks, order, m, d_lo, d_hi, d_ol, d_oh, d_cl, d_ch, g->dev.tail);
    k_spw_reclamp<<<blocks, 256>>>(W, g->dev.tail);
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    CK(cudaEventRecord(e1, 0));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    g->st.seed_folds++;
    g->st.ms_seeds += ms;
    return MGC_OK;
}

int warm_fold_decrements(mgc_sparse* g, const std::vector<unsigned>& pk, const std::vector<int32_t>& lo, const std::vector<int32_t>& hi,
                         const std::vector<int32_t>& olo, const std::vector<int32_t>& ohi, const std::vector<double>& d_lh,
                         const std::vector<double>& d_hl)
{
    CK(cudaSetDevice(g->device));
    DevScope dev;
    const long long m = (long long)pk.size();
    const int64_t np = (int64_t)g->plo.size();
    unsigned *ks, *order;
    RC(warm_group(g, dev, pk.data(), m, (unsigned)(np > 0 ? np - 1 : 0), &ks, &order));
    int *d_lo, *d_hi, *d_ol, *d_oh, *refused;
    double *d_l, *d_h;
    RC(warm_upload(g, dev, lo, &d_lo));
    RC(warm_upload(g, dev, hi, &d_hi));
    RC(warm_upload(g, dev, olo, &d_ol));
    RC(warm_upload(g, dev, ohi, &d_oh));
    RC(warm_upload(g, dev, d_lh, &d_l));
    RC(warm_upload(g, dev, d_hl, &d_h));
    CK(dev.alloc(&refused, 1));
    CK(cudaMemset(refused, 0, sizeof(int)));
    const SparseWarm W = warm_view(g);
    const unsigned mb = (unsigned)((m + 255) / 256);
    k_spw_pair_check<<<mb, 256>>>(W, ks, order, m, d_lo, d_hi, d_ol, d_oh, d_l, d_h, refused);
    g->st.kernel_launches++;
    int bad = 0;
    CK(cudaMemcpy(&bad, refused, sizeof(int), cudaMemcpyDeviceToHost));
    if (bad)
        FAIL(MGC_E_WEIGHT, "remove_edges_warm: a pair's decrements exceed its capacities r(i->j) + r(j->i) (the graph is "
                             "unchanged)");
    // arcs, then every end once in ascending node order with its changes in a fixed order
    unsigned *end_key, *end_idx, *end_ks, *end_order;
    double *end_dx, *partials;
    CK(dev.alloc(&end_key, (size_t)(2 * m)));
    CK(dev.alloc(&end_idx, (size_t)(2 * m)));
    CK(dev.alloc(&end_ks, (size_t)(2 * m)));
    CK(dev.alloc(&end_order, (size_t)(2 * m)));
    CK(dev.alloc(&end_dx, (size_t)(2 * m)));
    k_spw_pair_dec<<<mb, 256>>>(W, ks, order, m, d_lo, d_hi, d_ol, d_oh, d_l, d_h, end_key, end_dx);
    g->st.kernel_launches++;
    RC(warm_sort(g, dev, end_key, end_idx, 2 * m, 0xffffffffu, end_ks, end_order, true));
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

// calls checked (ids by the caller) and resolved to pairs: pk[k] = pair of call k, the capacities oriented lo->hi, hi->lo
int warm_resolve(mgc_sparse* g, int64_t count, const int32_t* i, const int32_t* j, const double* cap, const double* rev_cap,
                 bool create, std::vector<unsigned>& pk, std::vector<int32_t>& lo, std::vector<int32_t>& hi,
                 std::vector<double>& c_lh, std::vector<double>& c_hl)
{
    sparse_ensure_index(g);
    pk.resize((size_t)count); lo.resize((size_t)count); hi.resize((size_t)count);
    c_lh.resize((size_t)count); c_hl.resize((size_t)count);
    for (int64_t k = 0; k < count; ++k) {
        const bool fwd = i[k] < j[k];
        const int32_t a = fwd ? i[k] : j[k], b = fwd ? j[k] : i[k];
        const uint64_t key = ((uint64_t)(uint32_t)a << 32) | (uint32_t)b;
        auto it = g->pair_of.find(key);
        int64_t p;
        if (it != g->pair_of.end()) {
            p = it->second;
        } else if (create) {
            p = (int64_t)g->plo.size();
            g->pair_of.emplace(key, p);
            g->plo.push_back(a); g->phi.push_back(b);
            g->cap_lh.push_back(0.0); g->cap_hl.push_back(0.0);
            if (g->resident) { g->olo.push_back(g->deg[(size_t)a]++); g->ohi.push_back(g->deg[(size_t)b]++); }
        } else {
            FAIL(MGC_E_ARG, "no edge between nodes " + std::to_string(i[k]) + " and " + std::to_string(j[k]) +
                                  ": remove_edges_warm lowers existing capacities");
        }
        pk[(size_t)k] = (unsigned)p;
        lo[(size_t)k] = a; hi[(size_t)k] = b;
        c_lh[(size_t)k] = fwd ? cap[k] : rev_cap[k];
        c_hl[(size_t)k] = fwd ? rev_cap[k] : cap[k];
    }
    return MGC_OK;
}

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
    if (2 * ((int64_t)g->plo.size() + count) >= (int64_t)INT32_MAX) FAIL(MGC_E_ARG, "too many arcs for 32-bit arc ids");
    const int64_t first_fresh = (int64_t)g->plo.size();
    std::vector<unsigned> pk;
    std::vector<int32_t> lo, hi;
    std::vector<double> c_lh, c_hl;
    RC(warm_resolve(g, count, i, j, cap, rev_cap, true, pk, lo, hi, c_lh, c_hl));
    std::vector<int32_t> ol((size_t)count), oh((size_t)count);
    for (int64_t k = 0; k < count; ++k) {
        const size_t p = pk[(size_t)k];
        g->cap_lh[p] += c_lh[(size_t)k];          // a new pair starts at 0: add_edge's r_cap = cap (graph.h:449-450)
        g->cap_hl[p] += c_hl[(size_t)k];
        ol[(size_t)k] = g->olo[p]; oh[(size_t)k] = g->ohi[p];
    }
    g->solved = false;
    return warm_fold_edges(g, pk, lo, hi, ol, oh, c_lh, c_hl, first_fresh);
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
    g->n = n_nodes;
    g->tr.assign((size_t)n_nodes, 0.0);
    if (const char* e = std::getenv("MEDPY_GC_SPARSE_TIMEOUT")) { const double v = std::atof(e); if (v > 0) g->max_seconds = v; }
    if (const char* e = std::getenv("MEDPY_GC_SPARSE_SWEEPS")) { const int v = std::atoi(e); if (v > 0) g->sweeps_per_round = v; }
    *out = g;
    return MGC_OK;
}

void mgc_sparse_destroy(mgc_sparse* g) { delete g; }

int mgc_sparse_reset(mgc_sparse* g)
{
    if (!g) return MGC_E_ARG;
    std::fill(g->tr.begin(), g->tr.end(), 0.0);
    g->flow_const = 0.0;
    g->pair_of.clear();
    g->indexed = true;
    g->plo.clear(); g->phi.clear(); g->cap_lh.clear(); g->cap_hl.clear();
    g->solved = false;
    g->energy = 0.0;
    g->mask.clear();
    g->st = mgc_stats{};
    g->release();                   // the warm option itself stays
    g->solved_once = false;
    g->warm_bad = false;
    g->wconst = 0.0;
    g->olo.clear(); g->ohi.clear(); g->deg.clear();
    g->m2 = 0;
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
        if (a < 0 || b < 0 || a >= g->n || b >= g->n)
            FAIL(MGC_E_ARG, "Invalid node id in edge (" + std::to_string(a) + ", " + std::to_string(b) + "). Valid values are 0 to " +
                                  std::to_string(g->n - 1) + ".");
        if (a == b) FAIL(MGC_E_ARG, "The node_from (" + std::to_string(a) + ") can not be equal to the node_to (" + std::to_string(b) + ") (self-connections are forbidden in graph-cuts).");
    }
    if (g->resident) return warm_sum_edges(g, count, i, j, cap, rev_cap);
    // A batch of distinct pairs in strictly increasing (i, j) order with i < j -- what the region adjacency reduction
    // delivers (mgc_labels_fetch_edges) -- landing in an empty graph needs no look-ups: append, index later if ever needed.
    if (g->plo.empty() && count > 0) {
        bool sorted_unique = true;
        uint64_t prev = 0;
        for (int64_t k = 0; k < count && sorted_unique; ++k) {
            const uint64_t key = ((uint64_t)(uint32_t)i[k] << 32) | (uint32_t)j[k];
            sorted_unique = i[k] < j[k] && (k == 0 || key > prev);
            prev = key;
        }
        if (sorted_unique) {
            g->plo.assign(i, i + count);
            g->phi.assign(j, j + count);
            g->cap_lh.assign(cap, cap + count);
            g->cap_hl.assign(rev_cap, rev_cap + count);
            g->pair_of.clear();
            g->indexed = false;
            g->solved = false;
            return MGC_OK;
        }
    }
    sparse_ensure_index(g);
    for (int64_t k = 0; k < count; ++k) {
        const bool fwd = i[k] < j[k];
        const int32_t lo = fwd ? i[k] : j[k], hi = fwd ? j[k] : i[k];
        const uint64_t key = ((uint64_t)(uint32_t)lo << 32) | (uint32_t)hi;
        auto it = g->pair_of.find(key);
        const double c_lh = fwd ? cap[k] : rev_cap[k], c_hl = fwd ? rev_cap[k] : cap[k];
        if (it == g->pair_of.end()) {
            g->pair_of.emplace(key, (int64_t)g->plo.size());
            g->plo.push_back(lo); g->phi.push_back(hi);
            g->cap_lh.push_back(c_lh); g->cap_hl.push_back(c_hl);      // add_edge: r_cap = cap (graph.h:449-450)
        } else {
            g->cap_lh[(size_t)it->second] += c_lh;                       // sum_edge: r_cap += cap (graph.h:472-476)
            g->cap_hl[(size_t)it->second] += c_hl;
        }
    }
    if (count) g->solved = false;
    return MGC_OK;
}

int mgc_sparse_add_tweights(mgc_sparse* g, int64_t count, const int32_t* nodes, const double* src, const double* snk)
{
    if (!g) return MGC_E_ARG;
    if (count < 0 || (count > 0 && (!src || !snk))) FAIL(MGC_E_ARG, "null t-weight arrays");
    if (!nodes && count > g->n) FAIL(MGC_E_ARG, "more t-weights than nodes");
    if (nodes)
        for (int64_t k = 0; k < count; ++k)
            if (nodes[k] < 0 || nodes[k] >= g->n)
                FAIL(MGC_E_ARG, "Invalid node id of " + std::to_string(nodes[k]) + ". Valid values are 0 to " + std::to_string(g->n - 1) + ".");
    if (g->resident) {
        if (g->warm_bad) FAIL(MGC_E_STATE, warm_bad_msg);
        for (int64_t k = 0; k < count; ++k)
            if (!std::isfinite(src[k]) || !std::isfinite(snk[k])) FAIL(MGC_E_ARG, "t-weights hold NaN or infinite values");
        if (count == 0) return MGC_OK;
        int rc = warm_fold_tweights(g, count, nodes, src, snk);
        if (rc) return rc;
    }
    for (int64_t k = 0; k < count; ++k) {
        const size_t v = (size_t)(nodes ? nodes[k] : k);
        double s = src[k], t = snk[k];
        const double delta = g->tr[v];                 // graph.h:418-424
        if (delta > 0) s += delta; else t -= delta;
        g->flow_const += (s < t) ? s : t;
        g->tr[v] = s - t;
    }
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
        if (i[k] < 0 || j[k] < 0 || i[k] >= g->n || j[k] >= g->n || i[k] == j[k])
            FAIL(MGC_E_ARG, "invalid node ids (" + std::to_string(i[k]) + ", " + std::to_string(j[k]) + ")");
        if (!std::isfinite(cap[k]) || !std::isfinite(rev_cap[k])) FAIL(MGC_E_ARG, "decrements hold NaN or infinite values");
        if (cap[k] < 0 || rev_cap[k] < 0) FAIL(MGC_E_WEIGHT, "decrements are nonnegative amounts");
    }
    if (g->resident && g->warm_bad) FAIL(MGC_E_STATE, warm_bad_msg);
    if (count == 0) return MGC_OK;
    std::vector<unsigned> pk;
    std::vector<int32_t> lo, hi;
    std::vector<double> d_lh, d_hl;
    RC(warm_resolve(g, count, i, j, cap, rev_cap, false, pk, lo, hi, d_lh, d_hl));
    // per pair: the decrements summed in call order, pairs in order of their first call
    std::unordered_map<unsigned, size_t> slot;
    std::vector<unsigned> pairs;
    std::vector<double> sl, sh;
    for (int64_t k = 0; k < count; ++k) {
        auto ins = slot.emplace(pk[(size_t)k], pairs.size());
        if (ins.second) { pairs.push_back(pk[(size_t)k]); sl.push_back(0.0); sh.push_back(0.0); }
        sl[ins.first->second] += d_lh[(size_t)k];
        sh[ins.first->second] += d_hl[(size_t)k];
    }
    if (g->resident) {
        std::vector<int32_t> ol((size_t)count), oh((size_t)count);
        for (int64_t k = 0; k < count; ++k) { ol[(size_t)k] = g->olo[pk[(size_t)k]]; oh[(size_t)k] = g->ohi[pk[(size_t)k]]; }
        RC(warm_fold_decrements(g, pk, lo, hi, ol, oh, d_lh, d_hl));
    } else {
        // before the first solve: the same pair rule on the accumulated capacities
        for (size_t q = 0; q < pairs.size(); ++q)
            if (spw_pair_refused(g->cap_lh[pairs[q]], g->cap_hl[pairs[q]], sl[q], sh[q]))
                FAIL(MGC_E_WEIGHT, "remove_edges_warm: a pair's decrements exceed its capacities c(i->j) + c(j->i) (the graph "
                                     "is unchanged)");
    }
    for (size_t q = 0; q < pairs.size(); ++q) {
        const size_t p = pairs[q];
        const double a = g->cap_lh[p] - sl[q], b = g->cap_hl[p] - sh[q];
        g->cap_lh[p] = a < 0 ? 0.0 : a;
        g->cap_hl[p] = b < 0 ? 0.0 : b;
    }
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
    std::memcpy(out, g->mask.data(), (size_t)g->n);
    return MGC_OK;
}

int mgc_sparse_what_segment(mgc_sparse* g, int64_t node, int32_t* segment)
{
    if (!g || !segment) return MGC_E_ARG;
    if (node < 0 || node >= g->n) FAIL(MGC_E_ARG, "node id out of range");
    if (!g->solved) { int rc = sparse_solve(g); if (rc) return rc; }
    *segment = g->mask[(size_t)node] ? MGC_SOURCE : MGC_SINK;
    return MGC_OK;
}

int mgc_sparse_get_edge(const mgc_sparse* g, int64_t i, int64_t j, double* cap)
{
    if (!g || !cap) return MGC_E_ARG;
    sparse_ensure_index(const_cast<mgc_sparse*>(g));   // the index is a cache: building it does not change the graph
    *cap = 0.0;
    if (i < 0 || j < 0 || i >= g->n || j >= g->n || i == j) return MGC_OK;
    const bool fwd = i < j;
    const uint64_t key = ((uint64_t)(uint32_t)(fwd ? i : j) << 32) | (uint32_t)(fwd ? j : i);
    auto it = g->pair_of.find(key);
    if (it != g->pair_of.end()) *cap = fwd ? g->cap_lh[(size_t)it->second] : g->cap_hl[(size_t)it->second];
    return MGC_OK;
}

int mgc_sparse_get_trcap(const mgc_sparse* g, int64_t node, double* trcap)
{
    if (!g || !trcap || node < 0 || node >= g->n) return MGC_E_ARG;
    *trcap = g->tr[(size_t)node];
    return MGC_OK;
}

int mgc_sparse_get_node_num(const mgc_sparse* g, int64_t* n) { if (!g || !n) return MGC_E_ARG; *n = g->n; return MGC_OK; }
int mgc_sparse_get_arc_num(const mgc_sparse* g, int64_t* n) { if (!g || !n) return MGC_E_ARG; *n = 2 * (int64_t)g->plo.size(); return MGC_OK; }
int mgc_sparse_get_stats(const mgc_sparse* g, mgc_stats* out) { if (!g || !out) return MGC_E_ARG; *out = g->st; return MGC_OK; }

}  // extern "C"

// =================================================================================================================
// label images
// =================================================================================================================
struct mgc_labels {
    int device = 0;
    LabGeom G{};
    int64_t shape[4] = {1, 1, 1, 1};
    int* labels = nullptr;          // dense int32, C order
    bool owns_labels = false;
    int64_t k = 0;                  // regions
    std::vector<int32_t> ei, ej;    // last boundary result, sorted by (i, j)
    std::vector<double> ew, er;
    int64_t kernel_launches = 0;
    std::string err;
};

#undef CK
#undef FAIL
#define LBCK(call)                                                                                 \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            l->err = std::string(#call) + ": " + cudaGetErrorString(_e);                           \
            cudaGetLastError();                                                                    \
            return MGC_E_CUDA;                                                                     \
        }                                                                                          \
    } while (0)
#define LBFAIL(code, msg)                                                                          \
    do {                                                                                           \
        l->err = (msg);                                                                            \
        return (code);                                                                             \
    } while (0)

namespace {

// Dense, C-ordered device copy of `a` over the handle's shape.  *out points into `a` itself when it already is a dense
// device array, otherwise into memory owned by `scope`.
template <typename E>
int lab_stage(mgc_labels* l, const mgc_array* a, DevScope& scope, const E** out)
{
    if (!a || !a->data) LBFAIL(MGC_E_ARG, "null array");
    const size_t es = sizeof(E);
    LabStrides st{};
    bool contiguous = true;
    long long span = (long long)es, expect = (long long)es;
    for (int d = l->G.nd - 1; d >= 0; --d) {
        long long s = (long long)a->strides[d];
        if (l->G.dim[d] > 1) {
            if (s <= 0) LBFAIL(MGC_E_ARG, "array strides must be positive (pass a contiguous copy)");
            if (s != expect) contiguous = false;
            span += (l->G.dim[d] - 1) * s;
        } else {
            s = 0;
        }
        st.s[d] = s;
        expect *= l->G.dim[d];
    }
    const size_t bytes = (size_t)l->G.n * es;
    if (contiguous && a->mem == MGC_MEM_DEVICE) { *out = (const E*)a->data; return MGC_OK; }
    E* dst = nullptr;
    LBCK(scope.alloc(&dst, (size_t)l->G.n));
    if (contiguous) {
        LBCK(cudaMemcpy(dst, a->data, bytes, cudaMemcpyHostToDevice));
        *out = dst;
        return MGC_OK;
    }
    const char* src = (const char*)a->data;
    if (a->mem == MGC_MEM_HOST) {
        char* raw = nullptr;
        LBCK(scope.alloc(&raw, (size_t)span));
        LBCK(cudaMemcpy(raw, a->data, (size_t)span, cudaMemcpyHostToDevice));
        src = raw;
    }
    k_lab_gather<E><<<(unsigned)((l->G.n + LAB_BLOCK - 1) / LAB_BLOCK), LAB_BLOCK>>>(l->G, src, st, dst);
    l->kernel_launches++;
    LBCK(cudaGetLastError());
    *out = dst;
    return MGC_OK;
}

template <typename E, int MODE>
int lab_boundary_run(mgc_labels* l, const E* grad, double directedness)
{
    DevScope dev;
    const long long items = (long long)l->G.nd * l->G.n;
    const long long nb = (items + LAB_BLOCK - 1) / LAB_BLOCK;
    if (nb >= (long long)INT32_MAX) LBFAIL(MGC_E_ARG, "label image too large");
    unsigned* block_count;
    unsigned long long* block_off;
    LBCK(dev.alloc(&block_count, (size_t)nb));
    LBCK(dev.alloc(&block_off, (size_t)nb + 1));
    k_lab_pair_count<<<(unsigned)nb, LAB_BLOCK>>>(l->G, l->labels, MODE == 2 ? 1 : 0, block_count);
    k_lab_scan_blocks<<<1, 1024>>>(block_count, nb, block_off);
    l->kernel_launches += 2;
    LBCK(cudaGetLastError());
    unsigned long long m_u = 0;
    LBCK(cudaMemcpy(&m_u, block_off + nb, sizeof(m_u), cudaMemcpyDeviceToHost));
    const long long m = (long long)m_u;
    l->ei.clear(); l->ej.clear(); l->ew.clear(); l->er.clear();
    if (m == 0) return MGC_OK;
    if (m >= (1ll << 32)) LBFAIL(MGC_E_ARG, "more than 2^32 border voxel pairs");
    unsigned long long *keys, *keys_sorted;
    unsigned *perm = nullptr, *perm_sorted = nullptr;
    double *wf = nullptr, *wr = nullptr, *wf_s = nullptr, *wr_s = nullptr;
    LBCK(dev.alloc(&keys, (size_t)m));
    LBCK(dev.alloc(&keys_sorted, (size_t)m));
    if (MODE >= 1) { LBCK(dev.alloc(&wf, (size_t)m)); LBCK(dev.alloc(&wf_s, (size_t)m)); }
    if (MODE == 2) { LBCK(dev.alloc(&wr, (size_t)m)); LBCK(dev.alloc(&wr_s, (size_t)m)); }
    k_lab_pair_emit<E, MODE><<<(unsigned)nb, LAB_BLOCK>>>(l->G, l->labels, grad, directedness < 0 ? -directedness : directedness,
                                                          directedness < 0 ? 1 : 0, block_off, keys, wf, wr);
    l->kernel_launches++;
    LBCK(cudaGetLastError());
    // stable sort by key: contributions of one region pair stay in the reference's order
    const unsigned mblocks = (unsigned)((m + LAB_BLOCK - 1) / LAB_BLOCK);
    const int end_bit = 32 + bits_for((unsigned long long)l->k);
    if (MODE >= 1) {
        LBCK(dev.alloc(&perm, (size_t)m));
        LBCK(dev.alloc(&perm_sorted, (size_t)m));
        k_lab_iota<<<mblocks, LAB_BLOCK>>>(perm, m);
        size_t tb = 0;
        LBCK(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keys_sorted, perm, perm_sorted, m, 0, end_bit, 0));
        char* tmp;
        LBCK(dev.alloc(&tmp, tb));
        LBCK(cub::DeviceRadixSort::SortPairs(tmp, tb, keys, keys_sorted, perm, perm_sorted, m, 0, end_bit, 0));
        k_lab_permute<<<mblocks, LAB_BLOCK>>>(wf, perm_sorted, m, wf_s);
        if (MODE == 2) k_lab_permute<<<mblocks, LAB_BLOCK>>>(wr, perm_sorted, m, wr_s);
        l->kernel_launches += 3;
    } else {
        size_t tb = 0;
        LBCK(cub::DeviceRadixSort::SortKeys(nullptr, tb, keys, keys_sorted, m, 0, end_bit, 0));
        char* tmp;
        LBCK(dev.alloc(&tmp, tb));
        LBCK(cub::DeviceRadixSort::SortKeys(tmp, tb, keys, keys_sorted, m, 0, end_bit, 0));
    }
    LBCK(cudaGetLastError());
    // one output slot per run of equal keys, in key order (heads per block -> scan -> slot)
    unsigned* head_count;
    unsigned long long* head_off;
    LBCK(dev.alloc(&head_count, (size_t)mblocks));
    LBCK(dev.alloc(&head_off, (size_t)mblocks + 1));
    k_lab_seg_head_count<<<mblocks, LAB_BLOCK>>>(keys_sorted, m, head_count);
    k_lab_scan_blocks<<<1, 1024>>>(head_count, (long long)mblocks, head_off);
    unsigned long long u = 0;
    LBCK(cudaMemcpy(&u, head_off + mblocks, sizeof(u), cudaMemcpyDeviceToHost));
    unsigned long long* out_key;
    double *out_f, *out_r;
    LBCK(dev.alloc(&out_key, (size_t)u));
    LBCK(dev.alloc(&out_f, (size_t)u));
    LBCK(dev.alloc(&out_r, (size_t)u));
    k_lab_seg_reduce<<<mblocks, LAB_BLOCK>>>(keys_sorted, wf_s, wr_s, m, head_off, out_key, out_f, out_r);
    l->kernel_launches += 3;
    LBCK(cudaGetLastError());
    std::vector<unsigned long long> hk((size_t)u);
    l->ew.resize((size_t)u); l->er.resize((size_t)u);
    LBCK(cudaMemcpy(hk.data(), out_key, (size_t)u * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    LBCK(cudaMemcpy(l->ew.data(), out_f, (size_t)u * sizeof(double), cudaMemcpyDeviceToHost));
    LBCK(cudaMemcpy(l->er.data(), out_r, (size_t)u * sizeof(double), cudaMemcpyDeviceToHost));
    l->ei.resize((size_t)u); l->ej.resize((size_t)u);
    for (size_t t = 0; t < (size_t)u; ++t) {
        l->ei[t] = (int32_t)(hk[t] >> 32);
        l->ej[t] = (int32_t)(hk[t] & 0xffffffffull);
    }
    return MGC_OK;
}

template <typename E>
int lab_boundary_dispatch(mgc_labels* l, int kind, const mgc_array* values, double directedness)
{
    DevScope scope;
    const E* grad = nullptr;
    int rc = lab_stage<E>(l, values, scope, &grad);
    if (rc) return rc;
    if (kind == MGC_LABELS_STAWIASKI) return lab_boundary_run<E, 1>(l, grad, 0.0);
    return lab_boundary_run<E, 2>(l, grad, directedness);
}

// V = element type the sums are formed in (double: bincount; float/double: numpy.sum of a float array)
template <typename E, typename V, bool PAIRWISE>
int lab_region_sums_run(mgc_labels* l, const mgc_array* values, double* sums, int64_t* counts)
{
    DevScope dev;
    const E* vals_in = nullptr;
    int rc = lab_stage<E>(l, values, dev, &vals_in);
    if (rc) return rc;
    const long long n = l->G.n;
    if (n >= (long long)INT32_MAX) LBFAIL(MGC_E_ARG, "label image too large");
    unsigned *keys, *keys_sorted;
    V *vals, *vals_sorted;
    double* d_sums;
    long long* d_counts;
    LBCK(dev.alloc(&keys, (size_t)n));
    LBCK(dev.alloc(&keys_sorted, (size_t)n));
    LBCK(dev.alloc(&vals, (size_t)n));
    LBCK(dev.alloc(&vals_sorted, (size_t)n));
    LBCK(dev.alloc(&d_sums, (size_t)l->k));
    LBCK(dev.alloc(&d_counts, (size_t)l->k));
    const unsigned blocks = (unsigned)((n + LAB_BLOCK - 1) / LAB_BLOCK);
    k_lab_region_items<E, V><<<blocks, LAB_BLOCK>>>(l->labels, vals_in, n, keys, vals);
    size_t tb = 0;
    const int end_bit = bits_for((unsigned long long)l->k);
    LBCK(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keys_sorted, vals, vals_sorted, n, 0, end_bit, 0));
    char* tmp;
    LBCK(dev.alloc(&tmp, tb));
    LBCK(cub::DeviceRadixSort::SortPairs(tmp, tb, keys, keys_sorted, vals, vals_sorted, n, 0, end_bit, 0));
    if (PAIRWISE) k_lab_region_reduce_pairwise<V><<<blocks, LAB_BLOCK>>>(keys_sorted, vals_sorted, n, d_sums, d_counts);
    else          k_lab_region_reduce<<<blocks, LAB_BLOCK>>>(keys_sorted, (const double*)vals_sorted, n, d_sums, d_counts);
    l->kernel_launches += 2;
    LBCK(cudaGetLastError());
    std::vector<long long> hc((size_t)l->k);
    LBCK(cudaMemcpy(sums, d_sums, (size_t)l->k * sizeof(double), cudaMemcpyDeviceToHost));
    LBCK(cudaMemcpy(hc.data(), d_counts, (size_t)l->k * sizeof(long long), cudaMemcpyDeviceToHost));
    if (counts) for (int64_t r = 0; r < l->k; ++r) counts[r] = (int64_t)hc[(size_t)r];
    return MGC_OK;
}

}  // namespace

extern "C" {

int mgc_labels_create(int32_t ndim, const int64_t* shape, const mgc_array* labels, int32_t device, mgc_labels** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    if (ndim < 1 || ndim > MGC_MAX_NDIM || !shape || !labels) { g_lab_create_error = "label images must have 1 to 4 dimensions"; return MGC_E_ARG; }
    if (labels->dtype != MGC_I32) { g_lab_create_error = "label image must be int32"; return MGC_E_ARG; }
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count < 1) {
        cudaGetLastError();
        g_lab_create_error = "no CUDA device available (this library has no CPU path)";
        return MGC_E_CUDA;
    }
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
    if (device >= count) { g_lab_create_error = "invalid CUDA device ordinal"; return MGC_E_ARG; }
    mgc_labels* l = new mgc_labels();
    l->device = device;
    l->G.nd = ndim;
    long long n = 1;
    for (int d = 0; d < 4; ++d) { l->G.dim[d] = 1; l->G.stride[d] = 1; }
    for (int d = 0; d < ndim; ++d) {
        if (shape[d] < 1) { g_lab_create_error = "empty label image"; delete l; return MGC_E_LABELS; }
        l->G.dim[d] = shape[d];
        l->shape[d] = shape[d];
        n *= shape[d];
    }
    if (n >= (long long)INT32_MAX) { g_lab_create_error = "label image too large (2^31 voxels)"; delete l; return MGC_E_ARG; }
    l->G.n = n;
    long long acc = 1;
    for (int d = ndim - 1; d >= 0; --d) { l->G.stride[d] = acc; acc *= l->G.dim[d]; }
    auto fail = [&](int code) { g_lab_create_error = l->err; mgc_labels_destroy(l); return code; };
    if (cudaSetDevice(device) != cudaSuccess) { l->err = "cudaSetDevice failed"; return fail(MGC_E_CUDA); }
    {
        DevScope scope;
        const int* p = nullptr;
        int rc = lab_stage<int>(l, labels, scope, &p);
        if (rc) return fail(rc);
        if (!scope.ptrs.empty()) {
            // the dense copy is the last block the staging allocated: keep it, release the rest with the scope
            l->labels = (int*)p;
            l->owns_labels = true;
            scope.ptrs.erase(std::find(scope.ptrs.begin(), scope.ptrs.end(), (void*)p));
        } else {
            l->labels = (int*)p;        // dense device array of the caller: read in place
        }
        // __check_label_image: min == 1 and every id up to max present
        int* mm = nullptr;
        unsigned long long* cnt = nullptr;
        if (scope.alloc(&mm, 2) != cudaSuccess || scope.alloc(&cnt, 1) != cudaSuccess) { l->err = "device allocation failed"; return fail(MGC_E_NOMEM); }
        const int init[2] = {INT32_MAX, INT32_MIN};
        cudaMemcpy(mm, init, sizeof(init), cudaMemcpyHostToDevice);
        k_lab_minmax<<<grid_for(n), LAB_BLOCK>>>(l->labels, n, mm);
        int got[2] = {0, 0};
        if (cudaMemcpy(got, mm, sizeof(got), cudaMemcpyDeviceToHost) != cudaSuccess) { l->err = std::string("label scan failed: ") + cudaGetErrorString(cudaGetLastError()); return fail(MGC_E_CUDA); }
        const char* msg = "The supplied label image does either not contain any regions or they are not labeled consecutively starting from 1.";
        if (got[0] != 1 || got[1] < 1) { l->err = msg; return fail(MGC_E_LABELS); }
        uint8_t* present = nullptr;
        if (scope.alloc(&present, (size_t)got[1]) != cudaSuccess) { l->err = "device allocation failed"; return fail(MGC_E_NOMEM); }
        cudaMemset(present, 0, (size_t)got[1]);
        cudaMemset(cnt, 0, sizeof(unsigned long long));
        k_lab_presence<<<grid_for(n), LAB_BLOCK>>>(l->labels, n, present);
        k_lab_count_u8<<<grid_for(got[1]), LAB_BLOCK>>>(present, got[1], cnt);
        unsigned long long c = 0;
        if (cudaMemcpy(&c, cnt, sizeof(c), cudaMemcpyDeviceToHost) != cudaSuccess) { l->err = std::string("label scan failed: ") + cudaGetErrorString(cudaGetLastError()); return fail(MGC_E_CUDA); }
        l->kernel_launches += 3;
        if ((long long)c != (long long)got[1]) { l->err = msg; return fail(MGC_E_LABELS); }
        l->k = got[1];
    }
    *out = l;
    return MGC_OK;
}

void mgc_labels_destroy(mgc_labels* l)
{
    if (!l) return;
    if (l->owns_labels && l->labels) { cudaSetDevice(l->device); cudaFree(l->labels); }
    delete l;
}

const char* mgc_labels_last_error(const mgc_labels* l) { return l ? l->err.c_str() : g_lab_create_error.c_str(); }

int mgc_labels_region_count(const mgc_labels* l, int64_t* k) { if (!l || !k) return MGC_E_ARG; *k = l->k; return MGC_OK; }

int mgc_labels_boundary(mgc_labels* l, int32_t kind, const mgc_array* values, double directedness, int64_t* n_edges)
{
    if (!l) return MGC_E_ARG;
    LBCK(cudaSetDevice(l->device));
    int rc;
    if (kind == MGC_LABELS_ADJACENCY) {
        rc = lab_boundary_run<float, 0>(l, nullptr, 0.0);
    } else if (kind == MGC_LABELS_STAWIASKI || kind == MGC_LABELS_STAWIASKI_DIRECTED) {
        if (!values) LBFAIL(MGC_E_ARG, "the boundary term needs the gradient image");
        switch (values->dtype) {
            case MGC_F32: rc = lab_boundary_dispatch<float>(l, kind, values, directedness); break;
            case MGC_F64: rc = lab_boundary_dispatch<double>(l, kind, values, directedness); break;
            case MGC_U8: rc = lab_boundary_dispatch<uint8_t>(l, kind, values, directedness); break;
            case MGC_I16: rc = lab_boundary_dispatch<int16_t>(l, kind, values, directedness); break;
            case MGC_I32: rc = lab_boundary_dispatch<int32_t>(l, kind, values, directedness); break;
            default: LBFAIL(MGC_E_ARG, "unsupported dtype");
        }
    } else {
        LBFAIL(MGC_E_ARG, "unknown label boundary term");
    }
    if (rc) return rc;
    if (n_edges) *n_edges = (int64_t)l->ei.size();
    return MGC_OK;
}

int mgc_labels_fetch_edges(const mgc_labels* l, int32_t* i, int32_t* j, double* w_ij, double* w_ji)
{
    if (!l) return MGC_E_ARG;
    const size_t u = l->ei.size();
    if (u && (!i || !j)) return MGC_E_ARG;
    if (u) {
        std::memcpy(i, l->ei.data(), u * sizeof(int32_t));
        std::memcpy(j, l->ej.data(), u * sizeof(int32_t));
        if (w_ij) std::memcpy(w_ij, l->ew.data(), u * sizeof(double));
        if (w_ji) std::memcpy(w_ji, l->er.data(), u * sizeof(double));
    }
    return MGC_OK;
}

int mgc_labels_region_sums(mgc_labels* l, const mgc_array* values, int32_t mode, double* sums, int64_t* counts)
{
    if (!l || !values || !sums) return MGC_E_ARG;
    LBCK(cudaSetDevice(l->device));
    const bool pw = (mode == MGC_SUM_PAIRWISE);
    switch (values->dtype) {
        case MGC_F32: return pw ? lab_region_sums_run<float, float, true>(l, values, sums, counts)
                                : lab_region_sums_run<float, double, false>(l, values, sums, counts);
        case MGC_F64: return pw ? lab_region_sums_run<double, double, true>(l, values, sums, counts)
                                : lab_region_sums_run<double, double, false>(l, values, sums, counts);
        case MGC_U8: return lab_region_sums_run<uint8_t, double, false>(l, values, sums, counts);
        case MGC_I16: return lab_region_sums_run<int16_t, double, false>(l, values, sums, counts);
        case MGC_I32: return lab_region_sums_run<int32_t, double, false>(l, values, sums, counts);
        default: LBFAIL(MGC_E_ARG, "unsupported dtype");
    }
}

int mgc_labels_region_flags(mgc_labels* l, const mgc_array* markers, uint8_t* flags)
{
    if (!l || !markers || !flags) return MGC_E_ARG;
    if (markers->dtype != MGC_U8) LBFAIL(MGC_E_ARG, "markers must be uint8 / bool");
    LBCK(cudaSetDevice(l->device));
    DevScope dev;
    const uint8_t* m = nullptr;
    int rc = lab_stage<uint8_t>(l, markers, dev, &m);
    if (rc) return rc;
    uint8_t* d_flags;
    LBCK(dev.alloc(&d_flags, (size_t)l->k));
    LBCK(cudaMemset(d_flags, 0, (size_t)l->k));
    k_lab_region_flags<<<grid_for(l->G.n), LAB_BLOCK>>>(l->labels, m, l->G.n, d_flags);
    l->kernel_launches++;
    LBCK(cudaGetLastError());
    LBCK(cudaMemcpy(flags, d_flags, (size_t)l->k, cudaMemcpyDeviceToHost));
    return MGC_OK;
}

int mgc_labels_apply(mgc_labels* l, const uint8_t* per_region, uint8_t* out, int32_t out_mem)
{
    if (!l || !per_region || !out) return MGC_E_ARG;
    LBCK(cudaSetDevice(l->device));
    DevScope dev;
    uint8_t *d_reg, *d_out = out;
    LBCK(dev.alloc(&d_reg, (size_t)l->k));
    LBCK(cudaMemcpy(d_reg, per_region, (size_t)l->k, cudaMemcpyHostToDevice));
    if (out_mem == MGC_MEM_HOST) LBCK(dev.alloc(&d_out, (size_t)l->G.n));
    k_lab_apply<<<grid_for(l->G.n), LAB_BLOCK>>>(l->labels, d_reg, l->G.n, d_out);
    l->kernel_launches++;
    LBCK(cudaGetLastError());
    if (out_mem == MGC_MEM_HOST) LBCK(cudaMemcpy(out, d_out, (size_t)l->G.n, cudaMemcpyDeviceToHost));
    else LBCK(cudaDeviceSynchronize());
    return MGC_OK;
}

}  // extern "C"
