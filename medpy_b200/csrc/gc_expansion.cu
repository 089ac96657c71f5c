// gc_expansion.cu -- C ABI of the alpha-expansion segmentation (mgc_expansion_*, include/medpy_b200_graphcut.h; DESIGN.md
// §11).  A handle owns one eager lattice handle (mgc_graph) and cuts every move on it: the move kernel writes the state
// mgc_add_tweights_dense + mgc_add_nweights_dense would leave on a fresh handle, and mgc_maxflow solves it unchanged.
#include "gc_handle.cuh"
#include "gc_expansion.cuh"

#include <string>
#include <vector>

struct mgc_expansion {
    mgc_graph* g = nullptr;            // the lattice every move is cut on; its pool owns the buffers below
    int K = 0;
    int cost_dtype = -1;               // MGC_F32 / MGC_F64 of the cost planes (fixed by the first plane set)
    void* costs = nullptr;             // K planes of n elements
    std::vector<uint8_t> cost_set;
    double* w = nullptr;               // nd planes: w[d * n + p] = weight of the pair (p, p + e_d), 0 without one
    uint8_t* labels = nullptr;
    uint8_t* markers = nullptr;        // 0 none, m > 0: label m - 1
    uint8_t* init = nullptr;
    bool have_markers = false, have_init = false;
    unsigned long long* d_switched = nullptr;
    double* d_energy = nullptr;
    int* d_bad = nullptr;
    cudaEvent_t ev[6] = {};            // [0..3] one move: build | solve | apply; [4..5] the whole run
    bool ran = false;
    mgc_expansion_stats st{};
    std::vector<int64_t> switched;     // per move
};

namespace {
thread_local std::string g_exp_create_error;

template <typename C, int ND>
void move_launch(mgc_expansion* e, int alpha)
{
    mgc_graph* g = e->g;
    ExpWeights W{};
    for (int d = 0; d < ND; ++d) W.w[d] = e->w + (size_t)d * g->L.n;
    k_exp_move<C, ND><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const C*)e->costs, e->have_markers ? e->markers : nullptr,
                                                         e->labels, W, alpha, g->partials);
}

template <typename C, int ND>
void energy_launch(mgc_expansion* e)
{
    mgc_graph* g = e->g;
    ExpWeights W{};
    for (int d = 0; d < ND; ++d) W.w[d] = e->w + (size_t)d * g->L.n;
    k_exp_energy<C, ND><<<rblocks(g), 256, 0, g->stream>>>(g->L, (const C*)e->costs, e->have_markers ? e->markers : nullptr,
                                                           e->labels, W, g->partials);
}

template <int ND>
void by_dtype(mgc_expansion* e, int alpha)
{
    if (e->cost_dtype == MGC_F32) { if (alpha >= 0) move_launch<float, ND>(e, alpha); else energy_launch<float, ND>(e); }
    else                          { if (alpha >= 0) move_launch<double, ND>(e, alpha); else energy_launch<double, ND>(e); }
}

// alpha >= 0: the move kernel for alpha; -1: the energy kernel
void dispatch(mgc_expansion* e, int alpha)
{
    if (e->g->nd == 3) by_dtype<3>(e, alpha);
    else               by_dtype<4>(e, alpha);
}

// a uint8 label image staged into dst, refused (MGC_E_ARG) when an entry exceeds `limit`
int stage_u8(mgc_expansion* e, const mgc_array* a, uint8_t* dst, int limit, const char* what)
{
    mgc_graph* g = e->g;
    if (!a) return MGC_E_ARG;
    if (a->dtype != MGC_U8) FAIL(MGC_E_ARG, std::string(what) + " must be uint8");
    CK(cudaSetDevice(g->device));
    const void* p = nullptr;
    int rc = stage_input(g, a, 0, &p);
    if (rc) return rc;
    CK(cudaMemsetAsync(e->d_bad, 0, sizeof(int), g->stream));
    k_exp_check_u8<<<rblocks(g), 256, 0, g->stream>>>(g->L.n, (const uint8_t*)p, limit, e->d_bad);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(dst, p, g->L.n, cudaMemcpyDeviceToDevice, g->stream));
    slots_release(g, 1u);
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, e->d_bad, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    if (bad) FAIL(MGC_E_ARG, std::string(what) + " holds a value above " + std::to_string(limit));
    return MGC_OK;
}

float elapsed(cudaEvent_t a, cudaEvent_t b)
{
    float ms = 0.0f;
    return cudaEventElapsedTime(&ms, a, b) == cudaSuccess ? ms : 0.0f;
}
}  // namespace

// ---- gc_host.hpp: the element-wise kernels for the region and batch expansion units -------------------------------------------
void exp_init_launch(cudaStream_t s, unsigned blocks, unsigned n, int K, int dtype, const void* costs, const uint8_t* init,
                     uint8_t* labels, int* bad)
{
    if (dtype == MGC_F32) k_exp_init<float><<<blocks, 256, 0, s>>>(n, K, (const float*)costs, nullptr, init, labels, bad);
    else                  k_exp_init<double><<<blocks, 256, 0, s>>>(n, K, (const double*)costs, nullptr, init, labels, bad);
}

void exp_init_marked_launch(cudaStream_t s, unsigned blocks, unsigned n, int K, int dtype, const void* costs,
                            const uint8_t* markers, const uint8_t* init, uint8_t* labels, int* bad)
{
    if (dtype == MGC_F32) k_exp_init<float><<<blocks, 256, 0, s>>>(n, K, (const float*)costs, markers, init, labels, bad);
    else                  k_exp_init<double><<<blocks, 256, 0, s>>>(n, K, (const double*)costs, markers, init, labels, bad);
}

void exp_apply_launch(cudaStream_t s, unsigned blocks, unsigned n, const uint8_t* mask, uint8_t* labels, int alpha,
                      unsigned long long* switched)
{
    k_exp_apply<<<blocks, 256, 0, s>>>(n, mask, labels, alpha, switched);
}

void exp_check_costs_launch(cudaStream_t s, unsigned blocks, unsigned n, int dtype, const void* cost, int* bad)
{
    if (dtype == MGC_F32) k_exp_check_costs<float><<<blocks, 256, 0, s>>>(n, (const float*)cost, bad);
    else                  k_exp_check_costs<double><<<blocks, 256, 0, s>>>(n, (const double*)cost, bad);
}

void exp_check_u8_launch(cudaStream_t s, unsigned blocks, unsigned n, const uint8_t* a, int limit, int* bad)
{
    k_exp_check_u8<<<blocks, 256, 0, s>>>(n, a, limit, bad);
}

extern "C" {

int mgc_expansion_create(int32_t ndim, const int64_t* shape, int32_t labels, int32_t device, mgc_expansion** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    if (labels < 2 || labels > 255) { g_exp_create_error = "the number of labels must be 2..255"; return MGC_E_ARG; }
    mgc_graph* g = nullptr;
    int rc = mgc_create(ndim, shape, device, &g);
    if (rc) { g_exp_create_error = mgc_last_error(nullptr); return rc; }
    mgc_expansion* e = new mgc_expansion();
    e->g = g;
    e->K = labels;
    e->cost_set.assign((size_t)labels, 0);
    const size_t n = g->L.n;
    void* p = nullptr;
    rc = alloc_buf(g, (size_t)g->nd * n * sizeof(double), &p); e->w = (double*)p;
    if (!rc) { rc = alloc_buf(g, n, &p); e->labels = (uint8_t*)p; }
    if (!rc) { rc = alloc_buf(g, 64, &p); e->d_switched = (unsigned long long*)p; }
    if (!rc) { rc = alloc_buf(g, 64, &p); e->d_energy = (double*)p; }
    if (!rc) { rc = alloc_buf(g, 64, &p); e->d_bad = (int*)p; }
    // no boundary term: w = 0, every pair free
    if (!rc && cudaMemsetAsync(e->w, 0, (size_t)g->nd * n * sizeof(double), g->stream) != cudaSuccess) {
        g->err = "cudaMemsetAsync of the pair weights failed";
        rc = MGC_E_CUDA;
    }
    for (auto& ev : e->ev) cudaEventCreate(&ev);
    if (rc) { g_exp_create_error = g->err; mgc_expansion_destroy(e); return rc; }
    *out = e;
    return MGC_OK;
}

void mgc_expansion_destroy(mgc_expansion* e)
{
    if (!e) return;
    if (e->g) cudaSetDevice(e->g->device);
    for (auto& ev : e->ev) if (ev) cudaEventDestroy(ev);
    mgc_destroy(e->g);
    delete e;
}

const char* mgc_expansion_last_error(const mgc_expansion* e)
{
    return e ? e->g->err.c_str() : g_exp_create_error.c_str();
}

int mgc_expansion_set_cost(mgc_expansion* e, int32_t label, const mgc_array* cost)
{
    if (!e || !cost) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (label < 0 || label >= e->K) FAIL(MGC_E_ARG, "label out of range");
    if (cost->dtype != MGC_F32 && cost->dtype != MGC_F64) FAIL(MGC_E_ARG, "costs must be float32 or float64");
    if (e->cost_dtype >= 0 && cost->dtype != e->cost_dtype) FAIL(MGC_E_ARG, "every cost plane must have the same dtype");
    CK(cudaSetDevice(g->device));
    const size_t es = dtype_size(cost->dtype), bytes = (size_t)g->L.n * es;
    if (!e->costs) {
        int rc = alloc_buf(g, (size_t)e->K * bytes, &e->costs);
        if (rc) return rc;
        e->cost_dtype = cost->dtype;
    }
    const void* p = nullptr;
    int rc = stage_input(g, cost, 0, &p);
    if (rc) return rc;
    CK(cudaMemsetAsync(e->d_bad, 0, sizeof(int), g->stream));
    if (cost->dtype == MGC_F32) k_exp_check_costs<float><<<rblocks(g), 256, 0, g->stream>>>(g->L.n, (const float*)p, e->d_bad);
    else                        k_exp_check_costs<double><<<rblocks(g), 256, 0, g->stream>>>(g->L.n, (const double*)p, e->d_bad);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync((char*)e->costs + (size_t)label * bytes, p, bytes, cudaMemcpyDeviceToDevice, g->stream));
    slots_release(g, 1u);
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, e->d_bad, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    if (bad) FAIL(MGC_E_ARG, "costs must be finite and >= 0");
    e->cost_set[(size_t)label] = 1;
    e->ran = false;
    return MGC_OK;
}

int mgc_expansion_set_boundary(mgc_expansion* e, int32_t kind, const mgc_array* image, double sigma, const double* spacing,
                               double norm)
{
    if (!e) return MGC_E_ARG;
    mgc_graph* g = e->g;
    // the weights are what mgc_add_boundary writes on a fresh handle: arc p -> p + e_d of the FRESH stencil holds w, 0 on
    // the last plane of d
    int rc = mgc_reset(g);
    if (!rc) rc = mgc_add_boundary(g, kind, image, sigma, spacing, norm);
    if (!rc) {
        for (int d = 0; d < g->nd; ++d)
            CK(cudaMemcpyAsync(e->w + (size_t)d * g->L.n, g->S.cap[2 * d + 1], (size_t)g->L.n * sizeof(double),
                               cudaMemcpyDeviceToDevice, g->stream));
        CK(cudaStreamSynchronize(g->stream));
    }
    const std::string err = g->err;
    const int rc2 = mgc_reset(g);
    g->err = err;
    e->ran = false;
    return rc ? rc : rc2;
}

int mgc_expansion_set_markers(mgc_expansion* e, const mgc_array* markers)
{
    if (!e) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (!e->markers) {
        void* p = nullptr;
        int rc = alloc_buf(g, g->L.n, &p);
        if (rc) return rc;
        e->markers = (uint8_t*)p;
    }
    e->have_markers = false;
    e->ran = false;
    int rc = stage_u8(e, markers, e->markers, e->K, "markers");
    if (!rc) e->have_markers = true;
    return rc;
}

int mgc_expansion_set_init(mgc_expansion* e, const mgc_array* init)
{
    if (!e) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (!e->init) {
        void* p = nullptr;
        int rc = alloc_buf(g, g->L.n, &p);
        if (rc) return rc;
        e->init = (uint8_t*)p;
    }
    e->have_init = false;
    e->ran = false;
    int rc = stage_u8(e, init, e->init, e->K - 1, "init");
    if (!rc) e->have_init = true;
    return rc;
}

int mgc_expansion_run(mgc_expansion* e, int32_t max_cycles)
{
    if (!e) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (max_cycles < 1) FAIL(MGC_E_ARG, "max_cycles must be >= 1");
    for (int k = 0; k < e->K; ++k)
        if (!e->cost_set[(size_t)k]) FAIL(MGC_E_STATE, "the cost plane of label " + std::to_string(k) + " is not set");
    CK(cudaSetDevice(g->device));
    e->ran = false;
    e->st = mgc_expansion_stats{};
    e->switched.clear();
    const unsigned nb = rblocks(g);
    CK(cudaEventRecord(e->ev[4], g->stream));
    CK(cudaMemsetAsync(e->d_bad, 0, sizeof(int), g->stream));
    if (e->cost_dtype == MGC_F32)
        k_exp_init<float><<<nb, 256, 0, g->stream>>>(g->L.n, e->K, (const float*)e->costs, e->have_markers ? e->markers : nullptr,
                                                     e->have_init ? e->init : nullptr, e->labels, e->d_bad);
    else
        k_exp_init<double><<<nb, 256, 0, g->stream>>>(g->L.n, e->K, (const double*)e->costs, e->have_markers ? e->markers : nullptr,
                                                      e->have_init ? e->init : nullptr, e->labels, e->d_bad);
    CK(cudaGetLastError());
    if (e->have_init && e->have_markers) {
        int bad = 0;
        CK(cudaMemcpyAsync(&bad, e->d_bad, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        if (bad) FAIL(MGC_E_ARG, "init gives a marked voxel another label than its marker");
    }
    for (int cycle = 0; cycle < max_cycles; ++cycle) {
        int64_t changed = 0;
        for (int alpha = 0; alpha < e->K; ++alpha) {
            int rc = mgc_reset(g);
            if (rc) return rc;
            CK(cudaEventRecord(e->ev[0], g->stream));
            dispatch(e, alpha);
            CK(cudaGetLastError());
            sum_partials(g, g->partials, nb, g->d_scalars);     // the add_tweights constant, as finish_flow_const forms it
            g->caps_fresh = false;
            g->tr_fresh = false;
            g->has_nlinks = true;
            g->st.kernel_launches += 2;
            CK(cudaEventRecord(e->ev[1], g->stream));
            double flow = 0.0;
            rc = mgc_maxflow(g, &flow);
            if (rc) return rc;
            CK(cudaEventRecord(e->ev[2], g->stream));
            CK(cudaMemsetAsync(e->d_switched, 0, sizeof(unsigned long long), g->stream));
            k_exp_apply<<<nb, 256, 0, g->stream>>>(g->L.n, g->mask_dev, e->labels, alpha, e->d_switched);
            CK(cudaGetLastError());
            CK(cudaEventRecord(e->ev[3], g->stream));
            unsigned long long sw = 0;
            CK(cudaMemcpyAsync(&sw, e->d_switched, sizeof(sw), cudaMemcpyDeviceToHost, g->stream));
            CK(cudaStreamSynchronize(g->stream));
            e->st.ms_build += elapsed(e->ev[0], e->ev[1]);
            e->st.ms_solve += elapsed(e->ev[1], e->ev[2]);
            e->st.ms_apply += elapsed(e->ev[2], e->ev[3]);
            e->switched.push_back((int64_t)sw);
            changed += (int64_t)sw;
            e->st.moves++;
        }
        e->st.cycles++;
        if (!changed) { e->st.converged = 1; break; }
    }
    CK(cudaMemsetAsync(e->d_energy, 0, sizeof(double), g->stream));
    dispatch(e, -1);
    CK(cudaGetLastError());
    sum_partials(g, g->partials, nb, e->d_energy);
    CK(cudaEventRecord(e->ev[5], g->stream));
    CK(cudaMemcpyAsync(&e->st.energy, e->d_energy, sizeof(double), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    e->st.ms_total = elapsed(e->ev[4], e->ev[5]);
    e->ran = true;
    return MGC_OK;
}

int mgc_expansion_get_labels(mgc_expansion* e, uint8_t* out, int32_t mem)
{
    if (!e || !out) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (!e->ran) FAIL(MGC_E_STATE, "call mgc_expansion_run first");
    CK(cudaSetDevice(g->device));
    CK(cudaMemcpyAsync(out, e->labels, g->L.n, mem == MGC_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                       g->stream));
    CK(cudaStreamSynchronize(g->stream));
    return MGC_OK;
}

int mgc_expansion_get_stats(const mgc_expansion* e, mgc_expansion_stats* out)
{
    if (!e || !out) return MGC_E_ARG;
    if (!e->ran) { e->g->err = "call mgc_expansion_run first"; return MGC_E_STATE; }
    *out = e->st;
    return MGC_OK;
}

int mgc_expansion_get_switched(const mgc_expansion* e, int64_t* out)
{
    if (!e || !out) return MGC_E_ARG;
    if (!e->ran) { e->g->err = "call mgc_expansion_run first"; return MGC_E_STATE; }
    for (size_t i = 0; i < e->switched.size(); ++i) out[i] = e->switched[i];
    return MGC_OK;
}

}  // extern "C"
