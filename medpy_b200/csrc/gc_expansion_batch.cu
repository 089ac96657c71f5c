// gc_expansion_batch.cu -- C ABI of the batched alpha-expansion segmentation (mgc_expansion_batch_*,
// include/medpy_b200_graphcut.h; DESIGN.md §11 "Batches").  A handle owns one batch lattice handle (mgc_create_batch) and
// cuts every move of all B images on it at once: the move kernel writes the state of the B move graphs, mgc_maxflow
// solves it unchanged, and the images stay independent because no arc crosses a seam.  An image whose cycle switched
// nothing is frozen: its later move graphs are empty and its labels stay, which is where its own run would have stopped.
#include "gc_handle.cuh"
#include "gc_expansion_batch.cuh"

#include <string>
#include <vector>

struct mgc_expansion_batch {
    mgc_graph* g = nullptr;            // the batch lattice every move is cut on; its pool owns the buffers below
    int K = 0;
    int B = 0;
    int cost_dtype = -1;               // MGC_F32 / MGC_F64 of the cost planes (fixed by the first plane set)
    void* costs = nullptr;             // K planes of n = B * N elements
    std::vector<uint8_t> cost_set;
    double* w = nullptr;               // 3 planes: w[d * n + p] = weight of the pair (p, p + e_d), 0 without one
    uint8_t* labels = nullptr;
    uint8_t* markers = nullptr;        // 0 none, m > 0: label m - 1
    uint8_t* init = nullptr;
    bool have_markers = false, have_init = false;
    uint8_t* d_active = nullptr;       // [B] 1 while the image is not frozen
    unsigned long long* d_switched = nullptr;   // [B] voxels the current move switched per image
    double* d_energy = nullptr;        // [B]
    double* d_part = nullptr;          // [B * batch_chunks] energy partials
    int* d_bad = nullptr;
    cudaEvent_t ev[6] = {};            // [0..3] one move: build | solve | apply; [4..5] the whole run
    bool ran = false;
    mgc_expansion_stats st{};                  // the batch loop
    std::vector<mgc_expansion_stats> per;      // per image
    std::vector<int64_t> switched;             // moves x B, row-major
};

namespace {
thread_local std::string g_bexp_create_error;

ExpWeights weights_of(const mgc_expansion_batch* e)
{
    ExpWeights W{};
    for (int d = 0; d < 3; ++d) W.w[d] = e->w + (size_t)d * e->g->L.n;
    return W;
}

template <typename C>
void move_launch(mgc_expansion_batch* e, int alpha)
{
    mgc_graph* g = e->g;
    k_bexp_move<C><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const C*)e->costs, e->have_markers ? e->markers : nullptr,
                                                      e->labels, weights_of(e), e->d_active, alpha, g->partials);
}

template <typename C>
void energy_launch(mgc_expansion_batch* e)
{
    mgc_graph* g = e->g;
    const unsigned chunks = (unsigned)g->batch_chunks;
    k_bexp_energy<C><<<(unsigned)e->B * chunks, 256, 0, g->stream>>>(g->L, (const C*)e->costs,
                                                                    e->have_markers ? e->markers : nullptr, e->labels,
                                                                    weights_of(e), chunks, e->d_part);
}

// a (B, *image) uint8 label image staged into dst, refused (MGC_E_ARG) when an entry exceeds `limit`
int stage_u8(mgc_expansion_batch* e, const mgc_array* a, uint8_t* dst, int limit, const char* what)
{
    mgc_graph* g = e->g;
    if (!a) return MGC_E_ARG;
    if (a->dtype != MGC_U8) FAIL(MGC_E_ARG, std::string(what) + " must be uint8");
    CK(cudaSetDevice(g->device));
    mgc_array view;
    int rc = batch_view(g, a, 0, &view);
    if (rc) return rc;
    const void* p = nullptr;
    rc = stage_input(g, &view, 0, &p);
    if (rc) return rc;
    CK(cudaMemsetAsync(e->d_bad, 0, sizeof(int), g->stream));
    exp_check_u8_launch(g->stream, rblocks(g), g->L.n, (const uint8_t*)p, limit, e->d_bad);
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

extern "C" {

int mgc_expansion_batch_create(int32_t ndim, const int64_t* image_shape, int64_t batch, int32_t labels, int32_t device,
                               mgc_expansion_batch** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    if (labels < 2 || labels > 255) { g_bexp_create_error = "the number of labels must be 2..255"; return MGC_E_ARG; }
    mgc_graph* g = nullptr;
    int rc = mgc_create_batch(ndim, image_shape, batch, device, &g);
    if (rc) { g_bexp_create_error = mgc_last_error(nullptr); return rc; }
    // the pair weights come from one eager fused batch build: the capacity planes k_boundary writes, whatever
    // MEDPY_GC_FUSE / MEDPY_GC_LAZY_CAPS say for the caller's own handles
    g->fuse_build = true;
    g->lazy_caps = false;
    mgc_expansion_batch* e = new mgc_expansion_batch();
    e->g = g;
    e->K = labels;
    e->B = (int)batch;
    e->cost_set.assign((size_t)labels, 0);
    const size_t n = g->L.n;
    void* p = nullptr;
    rc = alloc_buf(g, 3 * n * sizeof(double), &p); e->w = (double*)p;
    if (!rc) { rc = alloc_buf(g, n, &p); e->labels = (uint8_t*)p; }
    if (!rc) { rc = alloc_buf(g, (size_t)batch, &p); e->d_active = (uint8_t*)p; }
    if (!rc) { rc = alloc_buf(g, (size_t)batch * sizeof(unsigned long long), &p); e->d_switched = (unsigned long long*)p; }
    if (!rc) { rc = alloc_buf(g, (size_t)batch * sizeof(double), &p); e->d_energy = (double*)p; }
    if (!rc) { rc = alloc_buf(g, (size_t)batch * (size_t)g->batch_chunks * sizeof(double), &p); e->d_part = (double*)p; }
    if (!rc) { rc = alloc_buf(g, 64, &p); e->d_bad = (int*)p; }
    // no boundary term: w = 0, every pair free
    if (!rc && cudaMemsetAsync(e->w, 0, 3 * n * sizeof(double), g->stream) != cudaSuccess) {
        g->err = "cudaMemsetAsync of the pair weights failed";
        rc = MGC_E_CUDA;
    }
    for (auto& ev : e->ev) cudaEventCreate(&ev);
    if (rc) { g_bexp_create_error = g->err; mgc_expansion_batch_destroy(e); return rc; }
    *out = e;
    return MGC_OK;
}

void mgc_expansion_batch_destroy(mgc_expansion_batch* e)
{
    if (!e) return;
    if (e->g) cudaSetDevice(e->g->device);
    for (auto& ev : e->ev) if (ev) cudaEventDestroy(ev);
    mgc_destroy(e->g);
    delete e;
}

const char* mgc_expansion_batch_last_error(const mgc_expansion_batch* e)
{
    return e ? e->g->err.c_str() : g_bexp_create_error.c_str();
}

int mgc_expansion_batch_set_cost(mgc_expansion_batch* e, int32_t label, const mgc_array* cost)
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
    // (B, *image) with any positive strides: a strided device array is gathered on the device
    mgc_array view;
    int rc = batch_view(g, cost, 0, &view);
    if (rc) return rc;
    const void* p = nullptr;
    rc = stage_input(g, &view, 0, &p);
    if (rc) return rc;
    CK(cudaMemsetAsync(e->d_bad, 0, sizeof(int), g->stream));
    exp_check_costs_launch(g->stream, rblocks(g), g->L.n, cost->dtype, p, e->d_bad);
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

int mgc_expansion_batch_set_markers(mgc_expansion_batch* e, const mgc_array* markers)
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

int mgc_expansion_batch_set_init(mgc_expansion_batch* e, const mgc_array* init)
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

int mgc_expansion_batch_run(mgc_expansion_batch* e, int32_t max_cycles)
{
    if (!e) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (max_cycles < 1) FAIL(MGC_E_ARG, "max_cycles must be >= 1");
    for (int k = 0; k < e->K; ++k)
        if (!e->cost_set[(size_t)k]) FAIL(MGC_E_STATE, "the cost plane of label " + std::to_string(k) + " is not set");
    CK(cudaSetDevice(g->device));
    const int B = e->B, K = e->K;
    e->ran = false;
    e->st = mgc_expansion_stats{};
    e->per.assign((size_t)B, mgc_expansion_stats{});
    e->switched.clear();
    const unsigned nb = rblocks(g);
    CK(cudaEventRecord(e->ev[4], g->stream));
    CK(cudaMemsetAsync(e->d_bad, 0, sizeof(int), g->stream));
    exp_init_marked_launch(g->stream, nb, g->L.n, K, e->cost_dtype, e->costs, e->have_markers ? e->markers : nullptr,
                           e->have_init ? e->init : nullptr, e->labels, e->d_bad);
    CK(cudaGetLastError());
    if (e->have_init && e->have_markers) {
        int bad = 0;
        CK(cudaMemcpyAsync(&bad, e->d_bad, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        if (bad) FAIL(MGC_E_ARG, "init gives a marked voxel another label than its marker");
    }
    std::vector<uint8_t> active((size_t)B, 1);
    std::vector<unsigned long long> sw((size_t)B);
    std::vector<int64_t> changed((size_t)B);
    CK(cudaMemcpyAsync(e->d_active, active.data(), (size_t)B, cudaMemcpyHostToDevice, g->stream));
    int live = B;
    for (int cycle = 0; cycle < max_cycles && live; ++cycle) {
        std::fill(changed.begin(), changed.end(), 0);
        for (int alpha = 0; alpha < K; ++alpha) {
            int rc = mgc_reset(g);
            if (rc) return rc;
            CK(cudaEventRecord(e->ev[0], g->stream));
            if (e->cost_dtype == MGC_F32) move_launch<float>(e, alpha);
            else                          move_launch<double>(e, alpha);
            CK(cudaGetLastError());
            sum_partials(g, g->partials, nb, g->d_scalars);     // the add_tweights constant of the active images
            g->caps_fresh = false;
            g->tr_fresh = false;
            g->has_nlinks = true;
            g->st.kernel_launches += 2;
            CK(cudaEventRecord(e->ev[1], g->stream));
            double flow = 0.0;
            rc = mgc_maxflow(g, &flow);
            if (rc) return rc;
            CK(cudaEventRecord(e->ev[2], g->stream));
            CK(cudaMemsetAsync(e->d_switched, 0, (size_t)B * sizeof(unsigned long long), g->stream));
            k_bexp_apply<<<nb, 256, 0, g->stream>>>(g->L, g->mask_dev, e->labels, e->d_active, alpha, e->d_switched);
            CK(cudaGetLastError());
            CK(cudaEventRecord(e->ev[3], g->stream));
            CK(cudaMemcpyAsync(sw.data(), e->d_switched, (size_t)B * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                               g->stream));
            CK(cudaStreamSynchronize(g->stream));
            e->st.ms_build += elapsed(e->ev[0], e->ev[1]);
            e->st.ms_solve += elapsed(e->ev[1], e->ev[2]);
            e->st.ms_apply += elapsed(e->ev[2], e->ev[3]);
            for (int b = 0; b < B; ++b) {
                e->switched.push_back((int64_t)sw[(size_t)b]);
                changed[(size_t)b] += (int64_t)sw[(size_t)b];
            }
            e->st.moves++;
        }
        e->st.cycles++;
        // an image whose cycle switched nothing is at a fixed point: its own run stops here
        bool froze = false;
        for (int b = 0; b < B; ++b) {
            if (!active[(size_t)b]) continue;
            mgc_expansion_stats& s = e->per[(size_t)b];
            s.cycles++;
            s.moves += K;
            if (!changed[(size_t)b]) { s.converged = 1; active[(size_t)b] = 0; --live; froze = true; }
        }
        if (froze && live) CK(cudaMemcpyAsync(e->d_active, active.data(), (size_t)B, cudaMemcpyHostToDevice, g->stream));
    }
    e->st.converged = live ? 0 : 1;
    if (e->cost_dtype == MGC_F32) energy_launch<float>(e);
    else                          energy_launch<double>(e);
    CK(cudaGetLastError());
    batch_sum(g, e->d_part, (unsigned)g->batch_chunks, e->d_energy);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e->ev[5], g->stream));
    std::vector<double> energy((size_t)B);
    CK(cudaMemcpyAsync(energy.data(), e->d_energy, (size_t)B * sizeof(double), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    e->st.ms_total = elapsed(e->ev[4], e->ev[5]);
    for (int b = 0; b < B; ++b) {
        e->per[(size_t)b].energy = energy[(size_t)b];
        e->st.energy += energy[(size_t)b];          // in image order
    }
    e->ran = true;
    return MGC_OK;
}

int mgc_expansion_batch_get_labels(mgc_expansion_batch* e, uint8_t* out, int32_t mem)
{
    if (!e || !out) return MGC_E_ARG;
    mgc_graph* g = e->g;
    if (!e->ran) FAIL(MGC_E_STATE, "call mgc_expansion_batch_run first");
    CK(cudaSetDevice(g->device));
    CK(cudaMemcpyAsync(out, e->labels, g->L.n, mem == MGC_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                       g->stream));
    CK(cudaStreamSynchronize(g->stream));
    return MGC_OK;
}

int mgc_expansion_batch_get_stats(const mgc_expansion_batch* e, mgc_expansion_stats* out)
{
    if (!e || !out) return MGC_E_ARG;
    if (!e->ran) { e->g->err = "call mgc_expansion_batch_run first"; return MGC_E_STATE; }
    *out = e->st;
    return MGC_OK;
}

int mgc_expansion_batch_get_image_stats(const mgc_expansion_batch* e, mgc_expansion_stats* out)
{
    if (!e || !out) return MGC_E_ARG;
    if (!e->ran) { e->g->err = "call mgc_expansion_batch_run first"; return MGC_E_STATE; }
    for (size_t b = 0; b < e->per.size(); ++b) out[b] = e->per[b];
    return MGC_OK;
}

int mgc_expansion_batch_get_switched(const mgc_expansion_batch* e, int64_t* out)
{
    if (!e || !out) return MGC_E_ARG;
    if (!e->ran) { e->g->err = "call mgc_expansion_batch_run first"; return MGC_E_STATE; }
    for (size_t i = 0; i < e->switched.size(); ++i) out[i] = e->switched[i];
    return MGC_OK;
}

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
