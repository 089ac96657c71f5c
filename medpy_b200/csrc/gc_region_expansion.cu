// gc_region_expansion.cu -- C ABI of the region alpha-expansion segmentation (mgc_region_expansion_*,
// include/medpy_b200_graphcut.h; DESIGN.md §11 "Region graphs").  A handle owns one sparse graph (mgc_sparse) whose
// device arrays hold the CSR of the region pairs for the handle's life (gc_sparse_held.hpp): every move writes only the
// capacities and t-links there (k_rexp_move) and is a cold solve of the sparse push-relabel.  Everything runs on the
// legacy default stream, the sparse solver's.  The loop is gc_expansion_loop.cu's, with B = 1.
#include "gc_host.hpp"
#include "gc_expansion_loop.hpp"
#include "gc_region_expansion.cuh"
#include "gc_sparse_held.hpp"
#include "gc_sparse_host.hpp"

#include <cmath>
#include <string>
#include <vector>

namespace {
// the grid of the per-node kernels: one block per 256 regions, at most REDUCE_BLOCKS (the partials' length)
unsigned rexp_blocks(int64_t n)
{
    const unsigned nb = (unsigned)((n + 255) / 256);
    return nb < REDUCE_BLOCKS ? nb : REDUCE_BLOCKS;
}
}  // namespace

struct mgc_region_expansion : Expansion {
    std::string msg;                    // the handle's error string: Expansion::err refers to it (bound, not read, before
                                        // it is constructed)
    mgc_sparse* sp;                     // every move is cut on it
    SparseHeld H{};                     // its device topology, capacities and t-links
    double* wt = nullptr;               // the pair weight on each arc of H
    double* partials = nullptr;         // REDUCE_BLOCKS per-block partials
    double* d_base = nullptr;           // the move's add_tweights constant
    std::vector<void*> bufs;            // what alloc() handed out

    mgc_region_expansion(mgc_sparse* sp, int device, int64_t n, int K)
        : Expansion(msg, "mgc_region_expansion", device, 0, (unsigned)n, rexp_blocks(n), K, 1), sp(sp)
    {
    }
    ~mgc_region_expansion() override
    {
        if (wt) cudaFree(wt);
        for (void* p : bufs) cudaFree(p);
        mgc_sparse_destroy(sp);
    }

    int alloc(size_t bytes, void** out) override;
    // a 1-D array of n entries with unit stride, as every per-region argument is passed: read where it is
    int stage(const mgc_array* a, size_t es, const char* what, const void** out) override;
    int build(const ExpMove& m) override;
    int solve(const uint8_t** mask) override;
    int energy() override;
};

namespace {
thread_local std::string g_rexp_create_error;

int sparse_failed(mgc_region_expansion* g, int rc)
{
    g->err = mgc_sparse_last_error(g->sp);
    return rc;
}

// the CSR of `count` pairs (host arrays, already checked) held on the sparse handle, their weights on both arcs
int hold_pairs(mgc_region_expansion* g, int64_t count, const int32_t* i, const int32_t* j, const double* w)
{
    SparseHost h((int)g->n);
    h.sum_edges(count, i, j, w, w);                 // ascending distinct pairs: taken as they are
    std::vector<int> row, head, sis;
    std::vector<double> cap;
    h.csr(row, head, sis, cap);                     // pairs in ascending order: every row in ascending neighbour id
    if (g->wt) { cudaFree(g->wt); g->wt = nullptr; }
    int rc = sparse_hold(g->sp, row, head, sis, &g->H);
    if (rc) return sparse_failed(g, rc);
    CK(cudaMalloc(&g->wt, (cap.empty() ? 1 : cap.size()) * sizeof(double)));
    if (!cap.empty()) CK(cudaMemcpy(g->wt, cap.data(), cap.size() * sizeof(double), cudaMemcpyHostToDevice));
    return MGC_OK;
}
}  // namespace

int mgc_region_expansion::alloc(size_t bytes, void** out)
{
    mgc_region_expansion* const g = this;
    CK(cudaMalloc(out, bytes));
    bufs.push_back(*out);
    return MGC_OK;
}

int mgc_region_expansion::stage(const mgc_array* a, size_t es, const char* what, const void** out)
{
    mgc_region_expansion* const g = this;
    if (!a->data || (n != 1 && a->strides[0] != (int64_t)es))
        FAIL(MGC_E_ARG, std::string(what) + ": one contiguous entry per region expected");
    *out = a->data;
    return MGC_OK;
}

int mgc_region_expansion::build(const ExpMove& m)
{
    mgc_region_expansion* const g = this;
    with_pair_rule(*this, [&](auto c, auto pair) {
        using C = decltype(c);
        if (m.beta >= 0)
            k_rswap_move<<<blocks, 256>>>(H.n, H.row, H.head, wt, (const C*)costs, labels, m.alpha, m.beta, H.cap, H.tr,
                                          partials, pair);
        else
            k_rexp_move<<<blocks, 256>>>(H.n, H.row, H.head, wt, (const C*)costs, labels, m.alpha, H.cap, H.tr, partials,
                                         pair);
    });
    CK(cudaGetLastError());
    CK(cudaMemsetAsync(d_base, 0, sizeof(double), 0));
    sum_partials_on(0, partials, blocks, d_base);       // the add_tweights constant
    CK(cudaGetLastError());
    return MGC_OK;
}

int mgc_region_expansion::solve(const uint8_t** mask)
{
    mgc_region_expansion* const g = this;
    double base = 0.0, cut = 0.0;
    CK(cudaMemcpy(&base, d_base, sizeof(double), cudaMemcpyDeviceToHost));
    const int rc = sparse_solve_held(sp, base, &cut, mask);
    return rc ? sparse_failed(this, rc) : MGC_OK;
}

int mgc_region_expansion::energy()
{
    mgc_region_expansion* const g = this;
    CK(cudaMemsetAsync(d_energy, 0, sizeof(double), 0));
    with_pair_rule(*this, [&](auto c, auto pair) {
        using C = decltype(c);
        k_rexp_energy<<<blocks, 256>>>(H.n, H.row, H.head, wt, (const C*)costs, labels, partials, pair);
    });
    CK(cudaGetLastError());
    sum_partials_on(0, partials, blocks, d_energy);
    return MGC_OK;
}

extern "C" {

int mgc_region_expansion_create(int64_t regions, int32_t labels, int32_t device, mgc_region_expansion** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    int rc = expansion_check_labels(labels, g_rexp_create_error);
    if (rc) return rc;
    if (regions < 1 || regions >= (int64_t)INT32_MAX) { g_rexp_create_error = "region count must be in [1, 2^31-2]"; return MGC_E_ARG; }
    mgc_sparse* sp = nullptr;
    rc = mgc_sparse_create(regions, device, &sp);
    if (rc) { g_rexp_create_error = mgc_sparse_last_error(nullptr); return rc; }
    if (device < 0 && cudaGetDevice(&device) != cudaSuccess) { cudaGetLastError(); device = 0; }
    mgc_region_expansion* g = new mgc_region_expansion(sp, device, regions, labels);
    rc = g->setup();
    if (!rc) rc = g->alloc(REDUCE_BLOCKS * sizeof(double), (void**)&g->partials);
    if (!rc) rc = g->alloc(sizeof(double), (void**)&g->d_base);
    if (!rc) rc = hold_pairs(g, 0, nullptr, nullptr, nullptr);   // no pairs until set_pairs
    if (rc) { g_rexp_create_error = g->err; mgc_region_expansion_destroy(g); return rc; }
    *out = g;
    return MGC_OK;
}

void mgc_region_expansion_destroy(mgc_region_expansion* g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    delete g;
}

const char* mgc_region_expansion_last_error(const mgc_region_expansion* g) { return g ? g->err.c_str() : g_rexp_create_error.c_str(); }

int mgc_region_expansion_set_cost(mgc_region_expansion* g, int32_t label, const mgc_array* cost)
{
    return g ? g->set_cost(label, cost) : MGC_E_ARG;
}

int mgc_region_expansion_set_pairs(mgc_region_expansion* g, int64_t count, const int32_t* i, const int32_t* j,
                                   const double* w)
{
    if (!g) return MGC_E_ARG;
    if (count < 0 || (count > 0 && (!i || !j || !w))) FAIL(MGC_E_ARG, "null pair arrays");
    if (2 * count >= (int64_t)INT32_MAX) FAIL(MGC_E_ARG, "too many pairs for 32-bit arc ids");
    for (int64_t k = 0; k < count; ++k) {
        if (i[k] < 0 || i[k] >= j[k] || j[k] >= (int64_t)g->n)
            FAIL(MGC_E_ARG, "pair " + std::to_string(k) + " (" + std::to_string(i[k]) + ", " + std::to_string(j[k]) +
                                ") is not 0 <= i < j < " + std::to_string(g->n));
        if (k && (i[k] < i[k - 1] || (i[k] == i[k - 1] && j[k] <= j[k - 1])))
            FAIL(MGC_E_ARG, "pairs must be strictly ascending in (i, j): pair " + std::to_string(k) + " is not");
        if (!std::isfinite(w[k]) || !(w[k] >= 0.0)) FAIL(MGC_E_ARG, "pair weights must be finite and >= 0");
    }
    g->ran = false;
    return hold_pairs(g, count, i, j, w);
}

int mgc_region_expansion_set_init(mgc_region_expansion* g, const mgc_array* init) { return g ? g->set_init(init) : MGC_E_ARG; }
int mgc_region_expansion_set_moves(mgc_region_expansion* g, int32_t kind) { return g ? g->set_moves(kind) : MGC_E_ARG; }
int mgc_region_expansion_set_label_distance(mgc_region_expansion* g, const double* dist)
{
    return g ? g->set_label_distance(dist) : MGC_E_ARG;
}

int mgc_region_expansion_run(mgc_region_expansion* g, int32_t max_cycles) { return g ? g->run(max_cycles) : MGC_E_ARG; }
int mgc_region_expansion_get_labels(mgc_region_expansion* g, uint8_t* out, int32_t mem) { return g ? g->get_labels(out, mem) : MGC_E_ARG; }
int mgc_region_expansion_get_stats(const mgc_region_expansion* g, mgc_expansion_stats* out) { return g ? g->get_stats(out) : MGC_E_ARG; }
int mgc_region_expansion_get_switched(const mgc_region_expansion* g, int64_t* out) { return g ? g->get_switched(out) : MGC_E_ARG; }

}  // extern "C"
