// gc_region_expansion.cu -- C ABI of the region alpha-expansion segmentation (mgc_region_expansion_*,
// include/medpy_b200_graphcut.h; DESIGN.md §11 "Region graphs").  A handle owns one sparse graph (mgc_sparse) whose
// device arrays hold the CSR of the region pairs for the handle's life (gc_sparse_held.hpp): every move writes only the
// capacities and t-links there (k_rexp_move) and is a cold solve of the sparse push-relabel.  Everything runs on the
// legacy default stream, the sparse solver's.
#include "gc_host.hpp"
#include "gc_region_expansion.cuh"
#include "gc_sparse_held.hpp"
#include "gc_sparse_host.hpp"

#include <cmath>
#include <string>
#include <vector>

struct mgc_region_expansion {
    int device = 0;
    int n = 0;                          // regions
    int K = 0;
    mgc_sparse* sp = nullptr;           // every move is cut on it
    SparseHeld H{};                     // its device topology, capacities and t-links
    double* wt = nullptr;               // the pair weight on each arc of H
    int cost_dtype = -1;                // MGC_F32 / MGC_F64 (fixed by the first cost set)
    void* costs = nullptr;              // K planes of n entries
    std::vector<uint8_t> cost_set;
    uint8_t* labels = nullptr;
    uint8_t* init = nullptr;
    bool have_init = false;
    double* partials = nullptr;         // REDUCE_BLOCKS per-block partials
    double* d_scalars = nullptr;        // [0] the move's add_tweights constant, [1] the energy
    unsigned long long* d_switched = nullptr;
    int* d_bad = nullptr;
    cudaEvent_t ev[6] = {};             // [0..3] one move: build | solve | apply; [4..5] the whole run
    bool ran = false;
    mgc_expansion_stats st{};
    std::vector<int64_t> switched;      // per move
    std::string err;
};

namespace {
thread_local std::string g_rexp_create_error;

// the grid of the per-node kernels: one block per 256 regions, at most REDUCE_BLOCKS (the partials' length)
unsigned rexp_blocks(int n)
{
    const unsigned nb = (unsigned)((n + 255) / 256);
    return nb < REDUCE_BLOCKS ? nb : REDUCE_BLOCKS;
}

// a 1-D array of n entries with unit stride, as every per-region argument is passed
bool one_per_region(const mgc_region_expansion* g, const mgc_array* a, size_t es)
{
    return a && a->data && (g->n == 1 || a->strides[0] == (int64_t)es);
}

int sparse_failed(mgc_region_expansion* g, int rc)
{
    g->err = mgc_sparse_last_error(g->sp);
    return rc;
}

// the CSR of `count` pairs (host arrays, already checked) held on the sparse handle, their weights on both arcs
int hold_pairs(mgc_region_expansion* g, int64_t count, const int32_t* i, const int32_t* j, const double* w)
{
    SparseHost h(g->n);
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

void move_launch(mgc_region_expansion* g, int alpha, unsigned nb)
{
    const SparseHeld& H = g->H;
    if (g->cost_dtype == MGC_F32)
        k_rexp_move<float><<<nb, 256>>>(H.n, H.row, H.head, g->wt, (const float*)g->costs, g->labels, alpha, H.cap, H.tr,
                                        g->partials);
    else
        k_rexp_move<double><<<nb, 256>>>(H.n, H.row, H.head, g->wt, (const double*)g->costs, g->labels, alpha, H.cap,
                                         H.tr, g->partials);
}

void energy_launch(mgc_region_expansion* g, unsigned nb)
{
    const SparseHeld& H = g->H;
    if (g->cost_dtype == MGC_F32)
        k_rexp_energy<float><<<nb, 256>>>(H.n, H.row, H.head, g->wt, (const float*)g->costs, g->labels, g->partials);
    else
        k_rexp_energy<double><<<nb, 256>>>(H.n, H.row, H.head, g->wt, (const double*)g->costs, g->labels, g->partials);
}

float elapsed(cudaEvent_t a, cudaEvent_t b)
{
    float ms = 0.0f;
    return cudaEventElapsedTime(&ms, a, b) == cudaSuccess ? ms : 0.0f;
}

int read_bad(mgc_region_expansion* g, int* bad)
{
    CK(cudaMemcpy(bad, g->d_bad, sizeof(int), cudaMemcpyDeviceToHost));
    return MGC_OK;
}
}  // namespace

extern "C" {

int mgc_region_expansion_create(int64_t regions, int32_t labels, int32_t device, mgc_region_expansion** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    if (labels < 2 || labels > 255) { g_rexp_create_error = "the number of labels must be 2..255"; return MGC_E_ARG; }
    if (regions < 1 || regions >= (int64_t)INT32_MAX) { g_rexp_create_error = "region count must be in [1, 2^31-2]"; return MGC_E_ARG; }
    mgc_sparse* sp = nullptr;
    int rc = mgc_sparse_create(regions, device, &sp);
    if (rc) { g_rexp_create_error = mgc_sparse_last_error(nullptr); return rc; }
    if (device < 0 && cudaGetDevice(&device) != cudaSuccess) { cudaGetLastError(); device = 0; }
    mgc_region_expansion* g = new mgc_region_expansion();
    g->device = device;
    g->n = (int)regions;
    g->K = labels;
    g->sp = sp;
    g->cost_set.assign((size_t)labels, 0);
    rc = [&]() -> int {
        CK(cudaSetDevice(device));
        CK(cudaMalloc(&g->labels, (size_t)g->n));
        CK(cudaMalloc(&g->init, (size_t)g->n));
        CK(cudaMalloc(&g->partials, REDUCE_BLOCKS * sizeof(double)));
        CK(cudaMalloc(&g->d_scalars, 2 * sizeof(double)));
        CK(cudaMalloc(&g->d_switched, sizeof(unsigned long long)));
        CK(cudaMalloc(&g->d_bad, sizeof(int)));
        for (auto& ev : g->ev) CK(cudaEventCreate(&ev));
        return hold_pairs(g, 0, nullptr, nullptr, nullptr);   // no pairs until set_pairs
    }();
    if (rc) { g_rexp_create_error = g->err; mgc_region_expansion_destroy(g); return rc; }
    *out = g;
    return MGC_OK;
}

void mgc_region_expansion_destroy(mgc_region_expansion* g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    for (auto& ev : g->ev) if (ev) cudaEventDestroy(ev);
    for (void* p : {(void*)g->wt, g->costs, (void*)g->labels, (void*)g->init, (void*)g->partials, (void*)g->d_scalars,
                    (void*)g->d_switched, (void*)g->d_bad})
        if (p) cudaFree(p);
    mgc_sparse_destroy(g->sp);
    delete g;
}

const char* mgc_region_expansion_last_error(const mgc_region_expansion* g)
{
    return g ? g->err.c_str() : g_rexp_create_error.c_str();
}

int mgc_region_expansion_set_cost(mgc_region_expansion* g, int32_t label, const mgc_array* cost)
{
    if (!g || !cost) return MGC_E_ARG;
    if (label < 0 || label >= g->K) FAIL(MGC_E_ARG, "label out of range");
    if (cost->dtype != MGC_F32 && cost->dtype != MGC_F64) FAIL(MGC_E_ARG, "costs must be float32 or float64");
    if (g->cost_dtype >= 0 && cost->dtype != g->cost_dtype) FAIL(MGC_E_ARG, "every cost row must have the same dtype");
    const size_t es = cost->dtype == MGC_F32 ? 4 : 8, bytes = (size_t)g->n * es;
    if (!one_per_region(g, cost, es)) FAIL(MGC_E_ARG, "costs: one contiguous entry per region expected");
    CK(cudaSetDevice(g->device));
    if (!g->costs) {
        CK(cudaMalloc(&g->costs, (size_t)g->K * bytes));
        g->cost_dtype = cost->dtype;
    }
    g->cost_set[(size_t)label] = 0;
    g->ran = false;
    void* dst = (char*)g->costs + (size_t)label * bytes;
    CK(cudaMemcpy(dst, cost->data, bytes, cudaMemcpyDefault));
    CK(cudaMemset(g->d_bad, 0, sizeof(int)));
    exp_check_costs_launch(0, rexp_blocks(g->n), (unsigned)g->n, g->cost_dtype, dst, g->d_bad);
    CK(cudaGetLastError());
    int bad = 0;
    RC(read_bad(g, &bad));
    if (bad) FAIL(MGC_E_ARG, "costs must be finite and >= 0");
    g->cost_set[(size_t)label] = 1;
    return MGC_OK;
}

int mgc_region_expansion_set_pairs(mgc_region_expansion* g, int64_t count, const int32_t* i, const int32_t* j,
                                   const double* w)
{
    if (!g) return MGC_E_ARG;
    if (count < 0 || (count > 0 && (!i || !j || !w))) FAIL(MGC_E_ARG, "null pair arrays");
    if (2 * count >= (int64_t)INT32_MAX) FAIL(MGC_E_ARG, "too many pairs for 32-bit arc ids");
    for (int64_t k = 0; k < count; ++k) {
        if (i[k] < 0 || i[k] >= j[k] || j[k] >= g->n)
            FAIL(MGC_E_ARG, "pair " + std::to_string(k) + " (" + std::to_string(i[k]) + ", " + std::to_string(j[k]) +
                                ") is not 0 <= i < j < " + std::to_string(g->n));
        if (k && (i[k] < i[k - 1] || (i[k] == i[k - 1] && j[k] <= j[k - 1])))
            FAIL(MGC_E_ARG, "pairs must be strictly ascending in (i, j): pair " + std::to_string(k) + " is not");
        if (!std::isfinite(w[k]) || !(w[k] >= 0.0)) FAIL(MGC_E_ARG, "pair weights must be finite and >= 0");
    }
    g->ran = false;
    return hold_pairs(g, count, i, j, w);
}

int mgc_region_expansion_set_init(mgc_region_expansion* g, const mgc_array* init)
{
    if (!g || !init) return MGC_E_ARG;
    if (init->dtype != MGC_U8) FAIL(MGC_E_ARG, "init must be uint8");
    if (!one_per_region(g, init, 1)) FAIL(MGC_E_ARG, "init: one contiguous entry per region expected");
    CK(cudaSetDevice(g->device));
    g->have_init = false;
    g->ran = false;
    CK(cudaMemcpy(g->init, init->data, (size_t)g->n, cudaMemcpyDefault));
    CK(cudaMemset(g->d_bad, 0, sizeof(int)));
    exp_check_u8_launch(0, rexp_blocks(g->n), (unsigned)g->n, g->init, g->K - 1, g->d_bad);
    CK(cudaGetLastError());
    int bad = 0;
    RC(read_bad(g, &bad));
    if (bad) FAIL(MGC_E_ARG, "init holds a value above " + std::to_string(g->K - 1));
    g->have_init = true;
    return MGC_OK;
}

int mgc_region_expansion_run(mgc_region_expansion* g, int32_t max_cycles)
{
    if (!g) return MGC_E_ARG;
    if (max_cycles < 1) FAIL(MGC_E_ARG, "max_cycles must be >= 1");
    for (int k = 0; k < g->K; ++k)
        if (!g->cost_set[(size_t)k]) FAIL(MGC_E_STATE, "the costs of label " + std::to_string(k) + " are not set");
    CK(cudaSetDevice(g->device));
    g->ran = false;
    g->st = mgc_expansion_stats{};
    g->switched.clear();
    const unsigned nb = rexp_blocks(g->n);
    const unsigned n = (unsigned)g->n;
    CK(cudaEventRecord(g->ev[4], 0));
    exp_init_launch(0, nb, n, g->K, g->cost_dtype, g->costs, g->have_init ? g->init : nullptr, g->labels, g->d_bad);
    CK(cudaGetLastError());
    for (int cycle = 0; cycle < max_cycles; ++cycle) {
        int64_t changed = 0;
        for (int alpha = 0; alpha < g->K; ++alpha) {
            CK(cudaEventRecord(g->ev[0], 0));
            move_launch(g, alpha, nb);
            CK(cudaGetLastError());
            CK(cudaMemsetAsync(g->d_scalars, 0, sizeof(double), 0));
            sum_partials_on(0, g->partials, nb, g->d_scalars);       // the add_tweights constant
            CK(cudaGetLastError());
            CK(cudaEventRecord(g->ev[1], 0));
            double base = 0.0, cut = 0.0;
            CK(cudaMemcpy(&base, g->d_scalars, sizeof(double), cudaMemcpyDeviceToHost));
            const uint8_t* mask = nullptr;
            int rc = sparse_solve_held(g->sp, base, &cut, &mask);
            if (rc) return sparse_failed(g, rc);
            CK(cudaEventRecord(g->ev[2], 0));
            CK(cudaMemsetAsync(g->d_switched, 0, sizeof(unsigned long long), 0));
            exp_apply_launch(0, nb, n, mask, g->labels, alpha, g->d_switched);
            CK(cudaGetLastError());
            CK(cudaEventRecord(g->ev[3], 0));
            unsigned long long sw = 0;
            CK(cudaMemcpy(&sw, g->d_switched, sizeof(sw), cudaMemcpyDeviceToHost));
            g->st.ms_build += elapsed(g->ev[0], g->ev[1]);
            g->st.ms_solve += elapsed(g->ev[1], g->ev[2]);
            g->st.ms_apply += elapsed(g->ev[2], g->ev[3]);
            g->switched.push_back((int64_t)sw);
            changed += (int64_t)sw;
            g->st.moves++;
        }
        g->st.cycles++;
        if (!changed) { g->st.converged = 1; break; }
    }
    CK(cudaMemsetAsync(g->d_scalars + 1, 0, sizeof(double), 0));
    energy_launch(g, nb);
    CK(cudaGetLastError());
    sum_partials_on(0, g->partials, nb, g->d_scalars + 1);
    CK(cudaGetLastError());
    CK(cudaEventRecord(g->ev[5], 0));
    CK(cudaMemcpy(&g->st.energy, g->d_scalars + 1, sizeof(double), cudaMemcpyDeviceToHost));
    g->st.ms_total = elapsed(g->ev[4], g->ev[5]);
    g->ran = true;
    return MGC_OK;
}

int mgc_region_expansion_get_labels(mgc_region_expansion* g, uint8_t* out, int32_t mem)
{
    if (!g || !out) return MGC_E_ARG;
    if (!g->ran) FAIL(MGC_E_STATE, "call mgc_region_expansion_run first");
    CK(cudaSetDevice(g->device));
    CK(cudaMemcpy(out, g->labels, (size_t)g->n, mem == MGC_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost));
    return MGC_OK;
}

int mgc_region_expansion_get_stats(const mgc_region_expansion* g, mgc_expansion_stats* out)
{
    if (!g || !out) return MGC_E_ARG;
    if (!g->ran) { const_cast<mgc_region_expansion*>(g)->err = "call mgc_region_expansion_run first"; return MGC_E_STATE; }
    *out = g->st;
    return MGC_OK;
}

int mgc_region_expansion_get_switched(const mgc_region_expansion* g, int64_t* out)
{
    if (!g || !out) return MGC_E_ARG;
    if (!g->ran) { const_cast<mgc_region_expansion*>(g)->err = "call mgc_region_expansion_run first"; return MGC_E_STATE; }
    for (size_t k = 0; k < g->switched.size(); ++k) out[k] = g->switched[k];
    return MGC_OK;
}

}  // extern "C"
