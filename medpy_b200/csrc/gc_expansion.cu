// gc_expansion.cu -- C ABI of the K-label segmentation by alpha-expansion or alpha-beta swap moves (mgc_expansion_*,
// include/medpy_b200_graphcut.h; DESIGN.md §11).  A handle owns one eager lattice handle (mgc_graph) and cuts every move on it: the move kernel writes the state
// mgc_add_tweights_dense + mgc_add_nweights_dense would leave on a fresh handle, and mgc_maxflow solves it unchanged.
// The loop is gc_expansion_loop.cu's, with B = 1; this unit also compiles the element-wise kernels it launches.
#include "gc_handle.cuh"
#include "gc_expansion.cuh"
#include "gc_expansion_loop.hpp"

#include <string>

struct mgc_expansion : Expansion {
    mgc_graph* g;                      // the lattice every move is cut on; its pool owns the buffers
    double* w = nullptr;               // nd planes: w[d * n + p] = weight of the pair (p, p + e_d), 0 without one

    mgc_expansion(mgc_graph* g, int K) : Expansion(g->err, "mgc_expansion", g->device, g->stream, g->L.n, rblocks(g), K, 1), g(g) {}
    ~mgc_expansion() override { mgc_destroy(g); }

    int alloc(size_t bytes, void** out) override { return alloc_buf(g, bytes, out); }
    int stage(const mgc_array* a, size_t, const char*, const void** out) override { return stage_input(g, a, 0, out); }
    void release() override { slots_release(g, 1u); }
    int reset() override { return mgc_reset(g); }
    int build(const ExpMove& m) override;
    int solve(const uint8_t** mask) override;
    int energy() override;

    ExpWeights weights() const
    {
        ExpWeights W{};
        for (int d = 0; d < g->nd; ++d) W.w[d] = w + (size_t)d * n;
        return W;
    }
};

namespace {
thread_local std::string g_exp_create_error;
}  // namespace

int mgc_expansion::build(const ExpMove& m)
{
    const uint8_t* mk = have_markers ? markers : nullptr;
    const int alpha = m.alpha, beta = m.beta;
    with_pair_rule(*this, [&](auto c, auto pair) {
        using C = decltype(c);
        using P = decltype(pair);
        if (beta >= 0) {
            if (g->nd == 3)
                k_swap_move<P, C, 3><<<blocks, 256, 0, g->stream>>>(g->L, g->S, (const C*)costs, mk, labels, weights(),
                                                                   alpha, beta, g->partials, pair);
            else
                k_swap_move<P, C, 4><<<blocks, 256, 0, g->stream>>>(g->L, g->S, (const C*)costs, mk, labels, weights(),
                                                                   alpha, beta, g->partials, pair);
        } else if (g->nd == 3)
            k_exp_move<P, C, 3><<<blocks, 256, 0, g->stream>>>(g->L, g->S, (const C*)costs, mk, labels, weights(), alpha,
                                                              g->partials, pair);
        else
            k_exp_move<P, C, 4><<<blocks, 256, 0, g->stream>>>(g->L, g->S, (const C*)costs, mk, labels, weights(), alpha,
                                                              g->partials, pair);
    });
    CK(cudaGetLastError());
    sum_partials(g, g->partials, blocks, g->d_scalars);     // the add_tweights constant, as finish_flow_const forms it
    g->caps_fresh = false;
    g->tr_fresh = false;
    g->has_nlinks = true;
    g->st.kernel_launches += 2;
    return MGC_OK;
}

int mgc_expansion::solve(const uint8_t** mask)
{
    double flow = 0.0;
    RC(mgc_maxflow(g, &flow));
    *mask = g->mask_dev;
    return MGC_OK;
}

int mgc_expansion::energy()
{
    CK(cudaMemsetAsync(d_energy, 0, sizeof(double), g->stream));
    const uint8_t* mk = have_markers ? markers : nullptr;
    with_pair_rule(*this, [&](auto c, auto pair) {
        using C = decltype(c);
        using P = decltype(pair);
        if (g->nd == 3)
            k_exp_energy<P, C, 3><<<blocks, 256, 0, g->stream>>>(g->L, (const C*)costs, mk, labels, weights(), g->partials, pair);
        else
            k_exp_energy<P, C, 4><<<blocks, 256, 0, g->stream>>>(g->L, (const C*)costs, mk, labels, weights(), g->partials, pair);
    });
    CK(cudaGetLastError());
    sum_partials(g, g->partials, blocks, d_energy);
    return MGC_OK;
}

// ---- gc_expansion_loop.hpp: the element-wise kernels the loop launches -----------------------------------------------
void exp_init_launch(cudaStream_t s, unsigned blocks, unsigned n, int K, int dtype, const void* costs, const uint8_t* markers,
                     const uint8_t* init, uint8_t* labels, int* bad)
{
    if (dtype == MGC_F32) k_exp_init<float><<<blocks, 256, 0, s>>>(n, K, (const float*)costs, markers, init, labels, bad);
    else                  k_exp_init<double><<<blocks, 256, 0, s>>>(n, K, (const double*)costs, markers, init, labels, bad);
}

void exp_apply_launch(cudaStream_t s, unsigned blocks, unsigned n, const uint8_t* mask, uint8_t* labels, int alpha,
                      unsigned long long* switched)
{
    k_exp_apply<<<blocks, 256, 0, s>>>(n, mask, labels, alpha, switched);
}

void swap_apply_launch(cudaStream_t s, unsigned blocks, unsigned n, const uint8_t* mask, uint8_t* labels, int alpha, int beta,
                       unsigned long long* switched)
{
    k_swap_apply<<<blocks, 256, 0, s>>>(n, mask, labels, alpha, beta, switched);
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
    int rc = expansion_check_labels(labels, g_exp_create_error);
    if (rc) return rc;
    mgc_graph* g = nullptr;
    rc = mgc_create(ndim, shape, device, &g);
    if (rc) { g_exp_create_error = mgc_last_error(nullptr); return rc; }
    mgc_expansion* e = new mgc_expansion(g, labels);
    const size_t n = g->L.n;
    void* p = nullptr;
    rc = alloc_buf(g, (size_t)g->nd * n * sizeof(double), &p); e->w = (double*)p;
    // no boundary term: w = 0, every pair free
    if (!rc && cudaMemsetAsync(e->w, 0, (size_t)g->nd * n * sizeof(double), g->stream) != cudaSuccess) {
        g->err = "cudaMemsetAsync of the pair weights failed";
        rc = MGC_E_CUDA;
    }
    if (!rc) rc = e->setup();
    if (rc) { g_exp_create_error = g->err; mgc_expansion_destroy(e); return rc; }
    *out = e;
    return MGC_OK;
}

void mgc_expansion_destroy(mgc_expansion* e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    delete e;
}

const char* mgc_expansion_last_error(const mgc_expansion* e) { return e ? e->err.c_str() : g_exp_create_error.c_str(); }
int mgc_expansion_set_cost(mgc_expansion* e, int32_t label, const mgc_array* cost) { return e ? e->set_cost(label, cost) : MGC_E_ARG; }

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

int mgc_expansion_set_markers(mgc_expansion* e, const mgc_array* markers) { return e ? e->set_markers(markers) : MGC_E_ARG; }
int mgc_expansion_set_init(mgc_expansion* e, const mgc_array* init) { return e ? e->set_init(init) : MGC_E_ARG; }
int mgc_expansion_set_moves(mgc_expansion* e, int32_t kind) { return e ? e->set_moves(kind) : MGC_E_ARG; }
int mgc_expansion_set_label_distance(mgc_expansion* e, const double* dist) { return e ? e->set_label_distance(dist) : MGC_E_ARG; }
int mgc_expansion_run(mgc_expansion* e, int32_t max_cycles) { return e ? e->run(max_cycles) : MGC_E_ARG; }
int mgc_expansion_get_labels(mgc_expansion* e, uint8_t* out, int32_t mem) { return e ? e->get_labels(out, mem) : MGC_E_ARG; }
int mgc_expansion_get_stats(const mgc_expansion* e, mgc_expansion_stats* out) { return e ? e->get_stats(out) : MGC_E_ARG; }
int mgc_expansion_get_switched(const mgc_expansion* e, int64_t* out) { return e ? e->get_switched(out) : MGC_E_ARG; }

}  // extern "C"
