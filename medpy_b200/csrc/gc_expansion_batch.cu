// gc_expansion_batch.cu -- C ABI of the batched alpha-expansion segmentation (mgc_expansion_batch_*,
// include/medpy_b200_graphcut.h; DESIGN.md §11 "Batches").  A handle owns one batch lattice handle (mgc_create_batch) and
// cuts every move of all B images on it at once: the move kernel writes the state of the B move graphs, mgc_maxflow
// solves it unchanged, and the images stay independent because no arc crosses a seam.  An image whose cycle switched
// nothing is frozen: its later move graphs are empty and its labels stay, which is where its own run would have stopped.
// The loop is gc_expansion_loop.cu's.
#include "gc_handle.cuh"
#include "gc_expansion_batch.cuh"
#include "gc_expansion_loop.hpp"

#include <string>
#include <vector>

struct mgc_expansion_batch : Expansion {
    mgc_graph* g;                      // the batch lattice every move is cut on; its pool owns the buffers
    double* w = nullptr;               // 3 planes: w[d * n + p] = weight of the pair (p, p + e_d), 0 without one
    uint8_t* d_active = nullptr;       // [B] 1 while the image is not frozen
    double* d_part = nullptr;          // [B * batch_chunks] energy partials

    mgc_expansion_batch(mgc_graph* g, int K)
        : Expansion(g->err, "mgc_expansion_batch", g->device, g->stream, g->L.n, rblocks(g), K, (int)g->batch), g(g)
    {
    }
    ~mgc_expansion_batch() override { mgc_destroy(g); }

    int alloc(size_t bytes, void** out) override { return alloc_buf(g, bytes, out); }
    // (B, *image) with any positive strides: a strided device array is gathered on the device
    int stage(const mgc_array* a, size_t, const char*, const void** out) override
    {
        mgc_array view;
        RC(batch_view(g, a, 0, &view));
        return stage_input(g, &view, 0, out);
    }
    void release() override { slots_release(g, 1u); }
    int reset() override { return mgc_reset(g); }
    int build(const ExpMove& m) override;
    int solve(const uint8_t** mask) override
    {
        double flow = 0.0;
        RC(mgc_maxflow(g, &flow));
        *mask = g->mask_dev;
        return MGC_OK;
    }
    void apply(const uint8_t* mask, const ExpMove& m) override
    {
        if (m.beta < 0) k_bexp_apply<<<blocks, 256, 0, g->stream>>>(g->L, mask, labels, d_active, m.alpha, d_switched);
        else k_bswap_apply<<<blocks, 256, 0, g->stream>>>(g->L, mask, labels, d_active, m.alpha, m.beta, d_switched);
    }
    int freeze(const std::vector<uint8_t>& active) override
    {
        CK(cudaMemcpyAsync(d_active, active.data(), (size_t)B, cudaMemcpyHostToDevice, g->stream));
        return MGC_OK;
    }
    int energy() override;

    ExpWeights weights() const
    {
        ExpWeights W{};
        for (int d = 0; d < 3; ++d) W.w[d] = w + (size_t)d * n;
        return W;
    }
};

namespace {
thread_local std::string g_bexp_create_error;
}  // namespace

int mgc_expansion_batch::build(const ExpMove& m)
{
    const uint8_t* mk = have_markers ? markers : nullptr;
    with_pair_rule(*this, [&](auto c, auto pair) {
        using C = decltype(c);
        if (m.beta >= 0)
            k_bswap_move<<<blocks, 256, 0, g->stream>>>(g->L, g->S, (const C*)costs, mk, labels, weights(), d_active,
                                                       m.alpha, m.beta, g->partials, pair);
        else
            k_bexp_move<<<blocks, 256, 0, g->stream>>>(g->L, g->S, (const C*)costs, mk, labels, weights(), d_active,
                                                      m.alpha, g->partials, pair);
    });
    CK(cudaGetLastError());
    sum_partials(g, g->partials, blocks, g->d_scalars);     // the add_tweights constant of the active images
    g->caps_fresh = false;
    g->tr_fresh = false;
    g->has_nlinks = true;
    g->st.kernel_launches += 2;
    return MGC_OK;
}

int mgc_expansion_batch::energy()
{
    const unsigned chunks = (unsigned)g->batch_chunks;
    const uint8_t* mk = have_markers ? markers : nullptr;
    with_pair_rule(*this, [&](auto c, auto pair) {
        using C = decltype(c);
        k_bexp_energy<<<(unsigned)B * chunks, 256, 0, g->stream>>>(g->L, (const C*)costs, mk, labels, weights(), chunks,
                                                                  d_part, pair);
    });
    CK(cudaGetLastError());
    batch_sum(g, d_part, (unsigned)g->batch_chunks, d_energy);
    return MGC_OK;
}

extern "C" {

int mgc_expansion_batch_create(int32_t ndim, const int64_t* image_shape, int64_t batch, int32_t labels, int32_t device,
                               mgc_expansion_batch** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    int rc = expansion_check_labels(labels, g_bexp_create_error);
    if (rc) return rc;
    mgc_graph* g = nullptr;
    rc = mgc_create_batch(ndim, image_shape, batch, device, &g);
    if (rc) { g_bexp_create_error = mgc_last_error(nullptr); return rc; }
    // the pair weights come from one eager fused batch build: the capacity planes k_boundary writes, whatever
    // MEDPY_GC_FUSE / MEDPY_GC_LAZY_CAPS say for the caller's own handles
    g->fuse_build = true;
    g->lazy_caps = false;
    mgc_expansion_batch* e = new mgc_expansion_batch(g, labels);
    const size_t n = g->L.n;
    void* p = nullptr;
    rc = alloc_buf(g, 3 * n * sizeof(double), &p); e->w = (double*)p;
    if (!rc) { rc = alloc_buf(g, (size_t)batch, &p); e->d_active = (uint8_t*)p; }
    if (!rc) { rc = alloc_buf(g, (size_t)batch * (size_t)g->batch_chunks * sizeof(double), &p); e->d_part = (double*)p; }
    // no boundary term: w = 0, every pair free
    if (!rc && cudaMemsetAsync(e->w, 0, 3 * n * sizeof(double), g->stream) != cudaSuccess) {
        g->err = "cudaMemsetAsync of the pair weights failed";
        rc = MGC_E_CUDA;
    }
    if (!rc) rc = e->setup();
    if (rc) { g_bexp_create_error = g->err; mgc_expansion_batch_destroy(e); return rc; }
    *out = e;
    return MGC_OK;
}

void mgc_expansion_batch_destroy(mgc_expansion_batch* e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    delete e;
}

const char* mgc_expansion_batch_last_error(const mgc_expansion_batch* e) { return e ? e->err.c_str() : g_bexp_create_error.c_str(); }

int mgc_expansion_batch_set_cost(mgc_expansion_batch* e, int32_t label, const mgc_array* cost)
{
    return e ? e->set_cost(label, cost) : MGC_E_ARG;
}

int mgc_expansion_batch_set_boundary(mgc_expansion_batch* e, int32_t kind, const mgc_array* image, const double* sigmas,
                                     const double* spacing, const double* norms)
{
    if (!e || !image || !sigmas || !norms) return MGC_E_ARG;
    mgc_graph* g = e->g;
    // the weights are the forward capacity planes of one eager batch build with the boundary term alone: per image what
    // mgc_add_boundary writes on a fresh handle of that image, 0 across the seams
    mgc_voxel_terms t{};
    t.boundary_kind = kind;
    t.image = image;
    t.spacing = spacing;
    t.compute_dtype = MGC_F64;
    int rc = mgc_reset(g);
    if (!rc) rc = mgc_build_voxel_batch(g, &t, sigmas, norms);
    if (!rc) {
        for (int d = 0; d < 3; ++d)
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

int mgc_expansion_batch_set_markers(mgc_expansion_batch* e, const mgc_array* markers) { return e ? e->set_markers(markers) : MGC_E_ARG; }
int mgc_expansion_batch_set_init(mgc_expansion_batch* e, const mgc_array* init) { return e ? e->set_init(init) : MGC_E_ARG; }
int mgc_expansion_batch_set_moves(mgc_expansion_batch* e, int32_t kind) { return e ? e->set_moves(kind) : MGC_E_ARG; }
int mgc_expansion_batch_set_label_distance(mgc_expansion_batch* e, const double* dist)
{
    return e ? e->set_label_distance(dist) : MGC_E_ARG;
}

int mgc_expansion_batch_run(mgc_expansion_batch* e, int32_t max_cycles) { return e ? e->run(max_cycles) : MGC_E_ARG; }
int mgc_expansion_batch_get_labels(mgc_expansion_batch* e, uint8_t* out, int32_t mem) { return e ? e->get_labels(out, mem) : MGC_E_ARG; }
int mgc_expansion_batch_get_stats(const mgc_expansion_batch* e, mgc_expansion_stats* out) { return e ? e->get_stats(out) : MGC_E_ARG; }

int mgc_expansion_batch_get_image_stats(const mgc_expansion_batch* e, mgc_expansion_stats* out)
{
    return e ? e->get_image_stats(out) : MGC_E_ARG;
}

int mgc_expansion_batch_get_switched(const mgc_expansion_batch* e, int64_t* out) { return e ? e->get_switched(out) : MGC_E_ARG; }

int mgc_expansion_batch_get_weights(mgc_expansion_batch* e, int32_t axis, double* out, int32_t mem)
{
    if (!e || !out) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (axis < 0 || axis >= g->batch_ndim) FAIL(MGC_E_ARG, "axis must name an image axis");
    CK(cudaSetDevice(g->device));
    const int d = 3 - g->batch_ndim + axis;
    CK(cudaMemcpyAsync(out, e->w + (size_t)d * g->L.n, (size_t)g->L.n * sizeof(double),
                       mem == MGC_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    return MGC_OK;
}

}  // extern "C"
