// gc_api.cu -- C-ABI of libmedpy_b200_gc.so (include/medpy_b200_graphcut.h): the device and pinned pools, input staging,
// handle lifecycle, the per-term entry points, the gradient and the getters.  The lattice handle and the other units of
// its ABI are described in gc_handle.cuh.  sm_90a only; there is no CPU path: without a CUDA device every entry point
// fails with MGC_E_CUDA.
#include "gc_handle.cuh"
#include "gc_api_kernels.cuh"
#include "gc_gradient.cuh"

#include <cmath>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

thread_local std::string g_create_error;

// ---------------------------------------------------------------------------------------------------
// device memory pool: graph_from_voxels creates a new graph per call (generate.py:120); handing freed
// blocks to the next handle keeps cudaMalloc (milliseconds per GB) out of the steady state.
// ---------------------------------------------------------------------------------------------------
namespace {
std::mutex g_pool_mu;
std::map<std::pair<int, size_t>, std::vector<void*>> g_pool;

size_t round_up(size_t b) { const size_t g = size_t(1) << 21; return (b + g - 1) / g * g; }

cudaError_t pool_alloc(int dev, size_t bytes, void** out)
{
    bytes = round_up(bytes);
    {
        std::lock_guard<std::mutex> lk(g_pool_mu);
        auto it = g_pool.find({dev, bytes});
        if (it != g_pool.end() && !it->second.empty()) {
            *out = it->second.back();
            it->second.pop_back();
            return cudaSuccess;
        }
    }
    cudaError_t e = cudaMalloc(out, bytes);
    if (e != cudaSuccess) {
        // release cached blocks and retry once
        std::lock_guard<std::mutex> lk(g_pool_mu);
        for (auto& kv : g_pool) if (kv.first.first == dev) { for (void* p : kv.second) cudaFree(p); kv.second.clear(); }
        cudaGetLastError();
        e = cudaMalloc(out, bytes);
    }
    return e;
}

void pool_free(int dev, size_t bytes, void* p)
{
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_pool_mu);
    g_pool[{dev, round_up(bytes)}].push_back(p);
}

// pinned host blocks (mask read-back buffers handed to the binding): same pooling idea as device memory
std::map<size_t, std::vector<void*>> g_host_pool;
std::map<void*, size_t> g_host_live;

}  // namespace

size_t dtype_size(int dt)
{
    switch (dt) {
        case MGC_F32: return 4;
        case MGC_F64: return 8;
        case MGC_U8: return 1;
        case MGC_I16: return 2;
        case MGC_I32: return 4;
        default: return 0;
    }
}

int alloc_buf(mgc_graph* g, size_t bytes, void** out)
{
    void* p = nullptr;
    cudaError_t e = pool_alloc(g->device, bytes, &p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        g->err = std::string("device allocation of ") + std::to_string(bytes) + " bytes failed: " + cudaGetErrorString(e);
        return MGC_E_NOMEM;
    }
    g->owned_bufs.push_back({p, bytes});
    g->device_bytes += (int64_t)round_up(bytes);
    *out = p;
    return MGC_OK;
}

int ensure_scratch(mgc_graph* g, Buf& b, size_t bytes)
{
    if (b.bytes >= bytes) return MGC_OK;
    if (b.p) {
        // a kernel or copy that is still in flight may be using the old block: drain before it goes back to the pool
        if (g->stream) cudaStreamSynchronize(g->stream);
        if (g->up_stream) cudaStreamSynchronize(g->up_stream);
        pool_free(g->device, b.bytes, b.p);
        g->device_bytes -= (int64_t)round_up(b.bytes);
    }
    b.p = nullptr; b.bytes = 0;
    void* p = nullptr;
    cudaError_t e = pool_alloc(g->device, bytes, &p);
    if (e != cudaSuccess) { cudaGetLastError(); g->err = "scratch allocation failed"; return MGC_E_NOMEM; }
    b.p = p; b.bytes = bytes;
    g->device_bytes += (int64_t)round_up(bytes);
    return MGC_OK;
}

namespace {
// Bring an input array into a C-contiguous device buffer over the local lattice.  Returns a device pointer
// valid until the next stage_input on the same slot.
template <typename E>
int gather_launch(mgc_graph* g, const char* src, const Strides4& st, E* dst)
{
    // exact Fortran order over a 3-D lattice (the layout medpy.io.load hands out): coalesced tiled transpose
    const int Z = g->L.dim[0], Y = g->L.dim[1], X = g->L.dim[2];
    if (g->nd == 3 && Z > 1 && X > 1 && Y <= 65535 && (Z + 31) / 32 <= 65535 &&
        st.s[0] == (long long)sizeof(E) && (Y == 1 || st.s[1] == (long long)sizeof(E) * Z) && st.s[2] == (long long)sizeof(E) * Z * Y) {
        const dim3 grid((unsigned)((X + 31) / 32), (unsigned)Y, (unsigned)((Z + 31) / 32));
        k_gather_fortran3<E><<<grid, 256, 0, g->stream>>>(Z, Y, X, reinterpret_cast<const E*>(src), dst);
        g->st.kernel_launches++;
        return MGC_OK;
    }
    if (g->nd == 3) k_gather<E, 3><<<nblocks(g), 256, 0, g->stream>>>(g->L, src, st, dst);
    else            k_gather<E, 4><<<nblocks(g), 256, 0, g->stream>>>(g->L, src, st, dst);
    g->st.kernel_launches++;
    return MGC_OK;
}
}  // namespace

// host -> device copy on the upload stream: waits until the staging slot's previous reader is done, makes the
// main stream wait for the copy, and blocks the HOST only until the copy itself has finished.
int upload(mgc_graph* g, void* dst, const void* src, size_t bytes, int slot)
{
    if (g->slot_used[slot]) CK(cudaStreamWaitEvent(g->up_stream, g->ev_slot[slot], 0));
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, g->up_stream));
    CK(cudaEventRecord(g->ev_up, g->up_stream));
    CK(cudaStreamWaitEvent(g->stream, g->ev_up, 0));
    CK(cudaEventSynchronize(g->ev_up));
    return MGC_OK;
}

// call after the kernel(s) that read the staging slots have been launched
void slots_release(mgc_graph* g, unsigned mask)
{
    // only the slots this call's kernels actually read: marking the others would make the NEXT call's upload wait for
    // this call's kernel although it targets a different buffer
    for (int i = 0; i < 5; ++i)
        if (mask & (1u << i)) { cudaEventRecord(g->ev_slot[i], g->stream); g->slot_used[i] = true; }
}

int stage_input(mgc_graph* g, const mgc_array* a, int slot, const void** out)
{
    const size_t es = dtype_size(a->dtype);
    if (!es) FAIL(MGC_E_ARG, "unsupported dtype");
    if (!a->data) FAIL(MGC_E_ARG, "null array");
    // canonical strides
    Strides4 st{};
    bool contiguous = true;
    long long span = (long long)es;
    long long expect = (long long)es;
    for (int d = g->nd - 1; d >= 0; --d) {
        long long s = 0;
        int ud = d - g->shift;
        if (ud >= 0) s = (long long)a->strides[ud];
        if (g->L.dim[d] > 1) {
            if (s <= 0) FAIL(MGC_E_ARG, "array strides must be positive (pass a contiguous copy)");
            if (s != expect) contiguous = false;
            span += (long long)(g->L.dim[d] - 1) * s;
        } else {
            s = 0;
        }
        st.s[d] = s;
        expect *= g->L.dim[d];
    }
    const size_t bytes = (size_t)g->L.n * es;
    if (contiguous && a->mem == MGC_MEM_DEVICE) { *out = a->data; return MGC_OK; }
    int rc = ensure_scratch(g, g->scratch[slot], bytes);
    if (rc) return rc;
    if (contiguous) {
        rc = upload(g, g->scratch[slot].p, a->data, bytes, slot);
        if (rc) return rc;
        *out = g->scratch[slot].p;
        return MGC_OK;
    }
    const char* src = (const char*)a->data;
    if (a->mem == MGC_MEM_HOST) {
        rc = ensure_scratch(g, g->raw, (size_t)span);
        if (rc) return rc;
        rc = upload(g, g->raw.p, a->data, (size_t)span, 3);
        if (rc) return rc;
        src = (const char*)g->raw.p;
    }
    else if (g->slot_used[slot]) CK(cudaStreamWaitEvent(g->stream, g->ev_slot[slot], 0));
    switch (a->dtype) {
        case MGC_F32: gather_launch<float>(g, src, st, (float*)g->scratch[slot].p); break;
        case MGC_F64: gather_launch<double>(g, src, st, (double*)g->scratch[slot].p); break;
        case MGC_U8: gather_launch<uint8_t>(g, src, st, (uint8_t*)g->scratch[slot].p); break;
        case MGC_I16: gather_launch<int16_t>(g, src, st, (int16_t*)g->scratch[slot].p); break;
        case MGC_I32: gather_launch<int32_t>(g, src, st, (int32_t*)g->scratch[slot].p); break;
    }
    CK(cudaGetLastError());
    // the gather is the last reader of the raw span: the next upload into it (same call, e.g. bg after fg) must wait
    if (a->mem == MGC_MEM_HOST) { CK(cudaEventRecord(g->ev_slot[3], g->stream)); g->slot_used[3] = true; }
    *out = g->scratch[slot].p;
    return MGC_OK;
}

// the one launcher of k_sum_partials: *out += the fixed-order sum of partials[0..n)
void sum_partials(mgc_graph* g, const double* partials, unsigned n, double* out)
{
    k_sum_partials<<<1, 256, 0, g->stream>>>(partials, n, out);
}

void sum_partials_on(cudaStream_t s, const double* partials, unsigned n, double* out)
{
    k_sum_partials<<<1, 256, 0, s>>>(partials, n, out);
}

namespace {
int finish_flow_const(mgc_graph* g)
{
    sum_partials(g, g->partials, rblocks(g), g->d_scalars);
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    return MGC_OK;
}

void invalidate(mgc_graph* g)
{
    g->lazy_built = false;             // terms changed outside the lazy build
    g->caps_img = nullptr;             // ... so no later call reads its inputs (work already queued may still read them)
    g->caps_tin.prob = nullptr;
    g->state_init = false;
    g->warm_state = false;
    g->solved = false;
    g->host_mask_valid = false;
}
}  // namespace

void resolve_term_span(mgc_graph* g)
{
    if (!g->terms_open) return;
    if (cudaEventSynchronize(g->ev_terms[1]) == cudaSuccess) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, g->ev_terms[0], g->ev_terms[1]) == cudaSuccess) g->st.ms_terms += ms;
        if (g->boundary_timed && cudaEventElapsedTime(&ms, g->ev_b[0], g->ev_b[1]) == cudaSuccess) g->st.ms_boundary = ms;
        g->boundary_timed = false;
    }
    g->terms_open = false;
}

// deliver a deferred weight verdict: waits for the boundary kernel that produced it
int check_pending(mgc_graph* g)
{
    if (!g->bad_pending) return MGC_OK;
    g->bad_pending = false;
    CK(cudaEventSynchronize(g->ev_bad));
    if (*g->h_bad) FAIL(MGC_E_WEIGHT, "Negative or zero weights are not allowed.");
    return MGC_OK;
}

namespace {
int create_impl(int32_t ndim, const int64_t* shape, int64_t z0, int64_t z1, bool slab, int32_t device, mgc_graph** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    if (ndim < 1 || ndim > MGC_MAX_NDIM || !shape) { g_create_error = "ndim must be 1..4"; return MGC_E_ARG; }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        g_create_error = std::string("no usable CUDA device (this library has no CPU path): ") + cudaGetErrorString(e);
        return MGC_E_CUDA;
    }
    if (device < 0) cudaGetDevice(&device);
    if (device >= ndev) { g_create_error = "bad device ordinal"; return MGC_E_ARG; }
    e = cudaSetDevice(device);
    if (e != cudaSuccess) { g_create_error = cudaGetErrorString(e); return MGC_E_CUDA; }

    mgc_graph* g = new mgc_graph();
    g->device = device;
    g->user_ndim = ndim;
    g->nd = ndim == 4 ? 4 : 3;
    g->shift = g->nd - ndim;
    for (int d = 0; d < ndim; ++d) {
        if (shape[d] < 1) { g_create_error = "extents must be >= 1"; delete g; return MGC_E_ARG; }
        g->user_shape[d] = shape[d];
    }
    int64_t dims[4] = {1, 1, 1, 1};
    for (int d = 0; d < ndim; ++d) dims[d + g->shift] = shape[d];
    g->slab = slab;
    int own0 = 0, own1 = (int)dims[0];
    if (slab) {
        if (g->shift != 0 || z0 < 0 || z1 > shape[0] || z0 >= z1) { g_create_error = "bad slab"; delete g; return MGC_E_ARG; }
        g->global_dim0 = shape[0]; g->z0 = z0; g->z1 = z1;
        g->ghost_lo = z0 > 0; g->ghost_hi = z1 < shape[0];
        dims[0] = (z1 - z0) + (g->ghost_lo ? 1 : 0) + (g->ghost_hi ? 1 : 0);
        own0 = g->ghost_lo ? 1 : 0;
        own1 = own0 + (int)(z1 - z0);
    }
    int64_t n = 1;
    for (int d = 0; d < g->nd; ++d) n *= dims[d];
    if (n >= (int64_t(1) << 31)) { g_create_error = "lattice too large for one device handle (>= 2^31 voxels)"; delete g; return MGC_E_ARG; }
    g->L.nd = g->nd;
    unsigned s = (unsigned)n;
    for (int d = 0; d < 4; ++d) { g->L.dim[d] = 1; g->L.stride[d] = 1; }
    for (int d = 0; d < g->nd; ++d) { g->L.dim[d] = (int)dims[d]; s /= (unsigned)dims[d]; g->L.stride[d] = s; }
    for (int d = 0; d < 4; ++d) {
        const unsigned long long st = g->L.stride[d];
        // ceil(2^64 / st) = floor((2^64 - 1) / st) + 1 for st > 1 that does not divide 2^64 ... and also when it does
        g->L.magic[d] = st <= 1 ? 0ull : (~0ull / st) + 1ull;
    }
    g->L.n = (unsigned)n;
    g->L.plane = g->L.stride[0];
    g->L.own0 = own0; g->L.own1 = own1;

    int rc = MGC_OK;
    const size_t nb = (size_t)n;
    void* p = nullptr;
    for (int k = 0; k < 2 * g->nd && !rc; ++k) { rc = alloc_buf(g, nb * sizeof(double), &p); g->S.cap[k] = (double*)p; }
    if (!rc) { rc = alloc_buf(g, nb * sizeof(double), &p); g->S.excess = (double*)p; }
    if (!rc) { rc = alloc_buf(g, nb * sizeof(double), &p); g->S.sink = (double*)p; }
    if (!rc) { rc = alloc_buf(g, nb * sizeof(double), &p); g->S.tr = (double*)p; }
    if (!rc) { rc = alloc_buf(g, nb * sizeof(int), &p); g->S.height = (int*)p; }
    if (!rc) { rc = alloc_buf(g, nb, &p); g->S.rmask = (uint8_t*)p; }
    if (!rc) { rc = alloc_buf(g, nb, &p); g->mask_dev = (uint8_t*)p; }
    g->n_partials = nblocks(g);
    if (g->nd == 3) {   // k_build_tile writes one partial per 8 x 8 x 32 block
        const unsigned nbuild = (unsigned)((g->L.dim[0] + 7) / 8) * (unsigned)((g->L.dim[1] + 7) / 8) * (unsigned)((g->L.dim[2] + 31) / 32);
        if (nbuild > g->n_partials) g->n_partials = nbuild;
        if (!rc) { rc = alloc_buf(g, (size_t)nbuild * sizeof(int), &p); g->build_refused = (int*)p; }
    }
    if (!rc) { rc = alloc_buf(g, (size_t)g->n_partials * sizeof(double), &p); g->partials = (double*)p; }
    if (!rc) { rc = alloc_buf(g, 3 * 1024 * sizeof(double), &p); g->minmax_buf = p; }
    if (!rc) { rc = alloc_buf(g, 64, &p); g->d_scalars = (double*)p; }
    if (!rc) { rc = alloc_buf(g, 64, &p); g->d_flags = (int*)p; }
    if (!rc) { rc = alloc_buf(g, 64, &p); g->d_count = (unsigned long long*)p; }
    if (!rc && g->nd == 3) {
        for (int d = 0; d < 3; ++d) g->TL.nt[d] = (g->L.dim[d] + TILE - 1) / TILE;
        g->TL.ntiles = g->TL.nt[0] * g->TL.nt[1] * g->TL.nt[2];
        const size_t tb = (size_t)g->TL.ntiles * sizeof(int);
        if (!rc) { rc = alloc_buf(g, tb, &p); g->pflag = (int*)p; }
        if (!rc) { rc = alloc_buf(g, tb, &p); g->rflag = (int*)p; }
        if (!rc) { rc = alloc_buf(g, tb, &p); g->cmat = (int*)p; }
        if (!rc) { rc = alloc_buf(g, tb, &p); g->caps_list = (int*)p; }
        for (int i = 0; i < 2 && !rc; ++i) { rc = alloc_buf(g, tb, &p); g->rl_items[i] = (int*)p; }
        for (int i = 0; i < 4 && !rc; ++i) { rc = alloc_buf(g, tb, &p); g->pl_items[i >> 1][i & 1] = (int*)p; }
        if (!rc) { rc = alloc_buf(g, 256, &p); g->d_tcount = (int*)p; }
        if (!rc) { rc = alloc_buf(g, tb, &p); g->win_tmin = (int*)p; }
        if (!rc) { rc = alloc_buf(g, tb, &p); g->win_items = (int*)p; }
        if (!rc) { rc = alloc_buf(g, tb, &p); g->drop_items = (int*)p; }
        if (!rc) { rc = alloc_buf(g, 64, &p); g->win_ctl = (int*)p; }
        if (!rc && cudaMemset(g->win_ctl, 0, 64) != cudaSuccess) { g->err = "cudaMemset of the window control words failed"; rc = MGC_E_CUDA; }
        {   // dirty-tile tracking for the partial relabel reset (MEDPY_GC_PARTIAL_RESET=0: off)
            const char* ed = getenv("MEDPY_GC_PARTIAL_RESET");
            g->TL.dflag = nullptr; g->TL.ditems = nullptr; g->TL.dcount = nullptr;
            if (!rc && (!ed || atoi(ed) != 0)) {
                rc = alloc_buf(g, tb, &p); g->TL.dflag = (int*)p;
                if (!rc) { rc = alloc_buf(g, tb, &p); g->TL.ditems = (int*)p; }
                if (!rc) { rc = alloc_buf(g, 64, &p); g->TL.dcount = (int*)p; }
            }
        }
        if (!rc) rc = tile_solver_options(g);
        push_tma_setup(g);
    }
    if (!rc && g->nd == 4) {
        const int ext[4] = {4, 4, 8, 4};
        g->TL4.ntiles = 1;
        for (int d = 0; d < 4; ++d) { g->TL4.nt[d] = (g->L.dim[d] + ext[d] - 1) / ext[d]; g->TL4.ntiles *= g->TL4.nt[d]; }
        g->TL.ntiles = g->TL4.ntiles;   // list sizes / shared helpers
        const size_t tb = (size_t)g->TL4.ntiles * sizeof(int);
        if (!rc) { rc = alloc_buf(g, tb, &p); g->pflag = (int*)p; }
        if (!rc) { rc = alloc_buf(g, tb, &p); g->rflag = (int*)p; }
        for (int i = 0; i < 2 && !rc; ++i) { rc = alloc_buf(g, tb, &p); g->rl_items[i] = (int*)p; }
        for (int i = 0; i < 4 && !rc; ++i) { rc = alloc_buf(g, tb, &p); g->pl_items[i >> 1][i & 1] = (int*)p; }
        if (!rc) { rc = alloc_buf(g, 256, &p); g->d_tcount = (int*)p; }
        if (!rc) { rc = alloc_buf(g, nb, &p); g->smask = (uint8_t*)p; }
        if (!rc) rc = tile_solver_options(g);
    }
    if (rc) { g_create_error = g->err; mgc_destroy(g); return rc; }
    if (cudaStreamCreate(&g->stream) != cudaSuccess) { g_create_error = "cudaStreamCreate failed"; mgc_destroy(g); return MGC_E_CUDA; }
    g->own_stream = true;
    for (auto& ev : g->ev) cudaEventCreate(&ev);
    cudaStreamCreateWithFlags(&g->up_stream, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&g->ev_up, cudaEventDisableTiming);
    for (auto& ev : g->ev_slot) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    for (auto& ev : g->ev_chunk) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    for (auto& ev : g->ev_terms) cudaEventCreate(&ev);
    if (const char* f0 = getenv("MEDPY_GC_DEBUG")) g->debug_checks = atoi(f0) != 0;
    if (const char* f3 = getenv("MEDPY_GC_FIRST_TEST")) g->skip_first_test = atoi(f3) == 0;
    if (const char* f5 = getenv("MEDPY_GC_FIRST_CAP")) g->first_cap = atoi(f5) >= 2 ? atoi(f5) : 0;
    if (const char* f1 = getenv("MEDPY_GC_FUSE")) g->fuse_build = atoi(f1) != 0;
    if (const char* f4 = getenv("MEDPY_GC_LAZY_CAPS")) g->lazy_caps = atoi(f4) != 0;
    if (const char* f2 = getenv("MEDPY_GC_CHUNKS")) if (atoi(f2) > 0) g->build_chunks = atoi(f2);
    cudaEventCreateWithFlags(&g->ev_bad, cudaEventDisableTiming);
    for (auto& ev : g->ev_b) cudaEventCreate(&ev);
    // [0] weight verdict, [2..3] active count, [4] BFS passes of the last cooperative relabel.  From the pinned pool: cudaHostAlloc / cudaFreeHost per handle (one handle per
    // graph_from_voxels call) are heavyweight driver calls that synchronise the device
    { void* hp = nullptr; g->h_bad = (mgc_host_alloc(64, &hp) == MGC_OK) ? (int*)hp : nullptr; }
    g->st.n_voxels = (int64_t)n;
    rc = mgc_reset(g);
    if (rc) { g_create_error = g->err; mgc_destroy(g); return rc; }
    *out = g;
    return MGC_OK;
}

template <typename E, int ND, bool FRESH>
void boundary_launch_nd(mgc_graph* g, const E* img, const BoundaryParams& P)
{
    const dim3 grid(nblocks(g)), block(256);
    // specialised instances: exponential term, no spacing, float32 / float64 images (every BASELINE configuration)
    if (P.fn == 1 && P.inv_spacing_on == 0.0 && (sizeof(E) == 4 || sizeof(E) == 8) && !std::is_integral<E>::value) {
        if (P.use_max) k_boundary<E, ND, double, FRESH, 1, 1, 0><<<grid, block, 0, g->stream>>>(g->L, g->S, img, P, g->d_flags);
        else           k_boundary<E, ND, double, FRESH, 1, 0, 0><<<grid, block, 0, g->stream>>>(g->L, g->S, img, P, g->d_flags);
        return;
    }
    k_boundary<E, ND, double, FRESH><<<grid, block, 0, g->stream>>>(g->L, g->S, img, P, g->d_flags);
}

template <typename E>
int boundary_launch(mgc_graph* g, const E* img, const BoundaryParams& P)
{
    if (g->caps_fresh) {
        if (g->nd == 3) boundary_launch_nd<E, 3, true>(g, img, P);
        else            boundary_launch_nd<E, 4, true>(g, img, P);
    } else {
        if (g->nd == 3) boundary_launch_nd<E, 3, false>(g, img, P);
        else            boundary_launch_nd<E, 4, false>(g, img, P);
    }
    g->caps_fresh = false;
    g->st.kernel_launches++;
    return MGC_OK;
}

// out[0] = |max - min|, out[1] = max |x| over img[0..n), in the input dtype (device)
template <typename E>
int minmax_launch(mgc_graph* g, const E* img, unsigned n, double* out)
{
    unsigned nb = g->n_partials < 1024u ? g->n_partials : 1024u;
    if (nb > (n + 255u) / 256u) nb = (n + 255u) / 256u;
    E* pm = (E*)g->minmax_buf;
    E* px = pm + 1024;
    E* pa = px + 1024;
    k_minmax_partial<E><<<nb, 256, 0, g->stream>>>(img, n, pm, px, pa);
    k_minmax_final<E><<<1, 32, 0, g->stream>>>(pm, px, pa, nb, out);
    g->st.kernel_launches += 2;
    return MGC_OK;
}
}  // namespace

int minmax_dtype(mgc_graph* g, int dtype, const void* img, unsigned n, double* out)
{
    switch (dtype) {
        case MGC_F32: return minmax_launch<float>(g, (const float*)img, n, out);
        case MGC_F64: return minmax_launch<double>(g, (const double*)img, n, out);
        case MGC_U8: return minmax_launch<uint8_t>(g, (const uint8_t*)img, n, out);
        case MGC_I16: return minmax_launch<int16_t>(g, (const int16_t*)img, n, out);
        case MGC_I32: return minmax_launch<int32_t>(g, (const int32_t*)img, n, out);
    }
    return MGC_OK;
}

// parameters of one of the eight boundary terms; the linear normaliser is computed on the device (K0) when `norm` is NaN
int boundary_params(mgc_graph* g, int kind, int dtype, const void* img, double sigma, const double* spacing, double norm, BoundaryParams* out)
{
    BoundaryParams P{};
    P.fn = kind & 3;
    // boundary_maximum_division computes the difference variant (energy_voxel.py:347)
    P.use_max = (kind >= 4 && kind != MGC_BOUNDARY_MAXIMUM_DIVISION) ? 1 : 0;
    P.sigma = (P.fn == 1) ? pow(sigma, 2) : sigma;   // math.pow(sigma, 2), energy_voxel.py:231
    P.inv_sigma2 = (P.fn == 1 && P.sigma != 0.0) ? 1.0 / P.sigma : 0.0;
    P.inv_spacing_on = spacing ? 1.0 : 0.0;
    for (int d = 0; d < 4; ++d) P.spacing[d] = 1.0;
    if (spacing) for (int d = 0; d < g->user_ndim; ++d) P.spacing[d + g->shift] = spacing[d];
    P.norm = norm;
    if (P.fn == 0 && std::isnan(norm)) {
        if (g->slab) FAIL(MGC_E_ARG, "z-slab handles need the global normaliser of the linear terms");
        int rc = minmax_dtype(g, dtype, img, g->L.n, g->d_scalars + 2);
        if (rc) return rc;
        double mm[2];
        CK(cudaMemcpyAsync(mm, g->d_scalars + 2, sizeof(mm), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        P.norm = (kind == MGC_BOUNDARY_MAXIMUM_LINEAR) ? mm[1] : mm[0];
    }
    *out = P;
    return MGC_OK;
}

template <typename E, int ND>
static cudaError_t gradient_launch(const int64_t* shape, const E* img, float* out, long long n)
{
    GradCtx<ND> G;
    long long st = 1;
    for (int d = ND - 1; d >= 0; --d) { G.dim[d] = (int)shape[d]; G.stride[d] = st; st *= shape[d]; }
    k_gradient_magnitude<E, ND><<<(unsigned)((n + 255) / 256), 256>>>(G, n, img, out);
    return cudaGetLastError();
}

template <typename E>
static cudaError_t gradient_dispatch(int nd, const int64_t* shape, const E* img, float* out, long long n)
{
    switch (nd) {
        case 1: return gradient_launch<E, 1>(shape, img, out, n);
        case 2: return gradient_launch<E, 2>(shape, img, out, n);
        case 3: return gradient_launch<E, 3>(shape, img, out, n);
        default: return gradient_launch<E, 4>(shape, img, out, n);
    }
}

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

int mgc_abi_version(void) { return MGC_ABI_VERSION; }

const char* mgc_last_error(const mgc_graph* g) { return g ? g->err.c_str() : g_create_error.c_str(); }

int mgc_create(int32_t ndim, const int64_t* shape, int32_t device, mgc_graph** out)
{
    return create_impl(ndim, shape, 0, 0, false, device, out);
}

int mgc_create_slab(int32_t ndim, const int64_t* shape, int64_t z0, int64_t z1, int32_t device, mgc_graph** out)
{
    if (ndim < 3) { g_create_error = "z-slab handles need ndim >= 3"; return MGC_E_ARG; }
    return create_impl(ndim, shape, z0, z1, true, device, out);
}

void mgc_destroy(mgc_graph* g)
{
    if (!g) return;
    cudaSetDevice(g->device);
    if (g->stream) cudaStreamSynchronize(g->stream);
    for (auto& b : g->owned_bufs) pool_free(g->device, b.bytes, b.p);
    for (auto& b : g->scratch) if (b.p) pool_free(g->device, b.bytes, b.p);
    if (g->raw.p) pool_free(g->device, g->raw.bytes, g->raw.p);
    if (g->img_copy.p) pool_free(g->device, g->img_copy.bytes, g->img_copy.p);
    if (g->prob_copy.p) pool_free(g->device, g->prob_copy.bytes, g->prob_copy.p);
    for (auto& b : g->mark_planes) if (b.p) pool_free(g->device, b.bytes, b.p);
    if (g->fold_buf.p) pool_free(g->device, g->fold_buf.bytes, g->fold_buf.p);
    for (auto& ev : g->ev_fold) if (ev) cudaEventDestroy(ev);
    for (auto& ev : g->ev) if (ev) cudaEventDestroy(ev);
    for (auto& ev : g->caps_ev) if (ev) cudaEventDestroy(ev);
    for (auto& ev : g->ev_slot) if (ev) cudaEventDestroy(ev);
    for (auto& ev : g->ev_terms) if (ev) cudaEventDestroy(ev);
    for (auto& ev : g->ev_chunk) if (ev) cudaEventDestroy(ev);
    if (g->ev_up) cudaEventDestroy(g->ev_up);
    if (g->ev_bad) cudaEventDestroy(g->ev_bad);
    for (auto& ev : g->ev_b) if (ev) cudaEventDestroy(ev);
    for (auto& ev : g->ph_events) if (ev) cudaEventDestroy(ev);
    if (g->h_bad) mgc_host_free(g->h_bad);
    if (g->h_stat) mgc_host_free(g->h_stat);
    slab_comm_release(g);
    if (g->up_stream) { cudaStreamSynchronize(g->up_stream); cudaStreamDestroy(g->up_stream); }
    if (g->own_stream && g->stream) cudaStreamDestroy(g->stream);
    delete g;
}

int mgc_reset(mgc_graph* g)
{
    if (!g) return MGC_E_ARG;
    CK(cudaSetDevice(g->device));
    // no memset of the big arrays: the first n-link / t-link term overwrites them (FRESH kernels)
    g->caps_fresh = true;
    g->tr_fresh = true;
    g->caps_lazy = false;
    CK(cudaMemsetAsync(g->d_scalars, 0, 64, g->stream));
    CK(cudaMemsetAsync(g->d_flags, 0, 64, g->stream));
    invalidate(g);
    g->flow_started = false;
    g->has_nlinks = false;
    g->batch_built = false;
    g->energy = 0.0;
    int64_t n = g->st.n_voxels;
    g->st = mgc_stats{};
    g->st.n_voxels = n;
    g->terms_open = false;
    g->bad_pending = false;
    return MGC_OK;
}

int mgc_gradient_magnitude_prewitt(int32_t ndim, const int64_t* shape, const mgc_array* image, float* out,
                                   int32_t out_mem, int32_t device)
{
    if (ndim < 1 || ndim > 4 || !shape || !image || !image->data || !out) { g_create_error = "bad arguments"; return MGC_E_ARG; }
    const size_t es = dtype_size(image->dtype);
    if (!es) { g_create_error = "unsupported dtype"; return MGC_E_ARG; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        g_create_error = "no usable CUDA device (this library has no CPU path)";
        return MGC_E_CUDA;
    }
    if (device < 0) cudaGetDevice(&device);
    cudaSetDevice(device);
    long long n = 1;
    bool contiguous = true;
    long long expect = (long long)es;
    for (int d = ndim - 1; d >= 0; --d) {
        if (shape[d] < 1) { g_create_error = "extents must be >= 1"; return MGC_E_ARG; }
        if (shape[d] > 1 && image->strides[d] != expect) contiguous = false;
        expect *= shape[d];
        n *= shape[d];
    }
    if (!contiguous) { g_create_error = "gradient input must be C-contiguous (the host layer copies otherwise)"; return MGC_E_ARG; }
    void* d_in = nullptr;
    void* d_out = nullptr;
    const size_t in_bytes = (size_t)n * es, out_bytes = (size_t)n * sizeof(float);
    cudaError_t e = cudaSuccess;
    if (image->mem == MGC_MEM_HOST) {
        if ((e = pool_alloc(device, in_bytes, &d_in)) != cudaSuccess) { cudaGetLastError(); g_create_error = "device allocation failed"; return MGC_E_NOMEM; }
        e = cudaMemcpy(d_in, image->data, in_bytes, cudaMemcpyHostToDevice);
    }
    const void* src = image->mem == MGC_MEM_HOST ? d_in : image->data;
    float* dst = out;
    if (e == cudaSuccess && out_mem == MGC_MEM_HOST) {
        if ((e = pool_alloc(device, out_bytes, &d_out)) == cudaSuccess) dst = (float*)d_out;
    }
    if (e == cudaSuccess) {
        switch (image->dtype) {
            case MGC_F32: e = gradient_dispatch<float>(ndim, shape, (const float*)src, dst, n); break;
            case MGC_F64: e = gradient_dispatch<double>(ndim, shape, (const double*)src, dst, n); break;
            case MGC_U8: e = gradient_dispatch<uint8_t>(ndim, shape, (const uint8_t*)src, dst, n); break;
            case MGC_I16: e = gradient_dispatch<int16_t>(ndim, shape, (const int16_t*)src, dst, n); break;
            default: e = gradient_dispatch<int32_t>(ndim, shape, (const int32_t*)src, dst, n); break;
        }
    }
    if (e == cudaSuccess && out_mem == MGC_MEM_HOST) e = cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (d_in) pool_free(device, in_bytes, d_in);
    if (d_out) pool_free(device, out_bytes, d_out);
    if (e != cudaSuccess) { cudaGetLastError(); g_create_error = std::string("gradient kernel failed: ") + cudaGetErrorString(e); return MGC_E_CUDA; }
    return MGC_OK;
}

int mgc_host_alloc(size_t bytes, void** out)
{
    if (!out || !bytes) return MGC_E_ARG;
    const size_t rb = round_up(bytes);
    std::lock_guard<std::mutex> lk(g_pool_mu);
    auto it = g_host_pool.find(rb);
    void* p = nullptr;
    if (it != g_host_pool.end() && !it->second.empty()) { p = it->second.back(); it->second.pop_back(); }
    else if (cudaHostAlloc(&p, rb, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); g_create_error = "pinned host allocation failed"; return MGC_E_NOMEM; }
    g_host_live[p] = rb;
    *out = p;
    return MGC_OK;
}

void mgc_host_free(void* p)
{
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_pool_mu);
    auto it = g_host_live.find(p);
    if (it == g_host_live.end()) return;
    g_host_pool[it->second].push_back(p);
    g_host_live.erase(it);
}

// Give cached blocks back to the driver: every device block of the size-keyed pool (all devices) and every pinned host block
// that is not handed out.  Handles that are alive keep what they hold.
int mgc_trim_pools(void)
{
    std::lock_guard<std::mutex> lk(g_pool_mu);
    int cur = 0;
    cudaGetDevice(&cur);
    for (auto& kv : g_pool) {
        if (kv.second.empty()) continue;
        cudaSetDevice(kv.first.first);
        for (void* p : kv.second) cudaFree(p);
        kv.second.clear();
    }
    cudaSetDevice(cur);
    for (auto& kv : g_host_pool) { for (void* p : kv.second) cudaFreeHost(p); kv.second.clear(); }
    cudaGetLastError();
    return MGC_OK;
}

int mgc_set_option(mgc_graph* g, int32_t option, int64_t value)
{
    if (!g) return MGC_E_ARG;
    if (option == MGC_OPT_DEFER_WEIGHT_CHECK) { g->defer_check = value != 0; return MGC_OK; }
    if (option == MGC_OPT_KEEP_DEVICE_INPUTS) { g->keep_device_inputs = value != 0; return MGC_OK; }
    if (option == MGC_OPT_WARM) {
        // the record is taken before the first push; a lazily built handle folds without it, so there it changes nothing now
        // (on a batch handle the option also admits the folds at all, batch_warm)
        const bool on = value != 0;
        if (on != g->warm_opt && g->flow_started && !g->lazy_built)
            FAIL(MGC_E_STATE, "MGC_OPT_WARM is set before the first solve (the residual source capacities are recorded at "
                              "its start): reset() the handle and rebuild the graph to change it");
        g->warm_opt = on;
        return MGC_OK;
    }
    FAIL(MGC_E_ARG, "unknown option");
}

int mgc_check(mgc_graph* g)
{
    if (!g) return MGC_E_ARG;
    return check_pending(g);
}

int mgc_set_stream(mgc_graph* g, void* cuda_stream)
{
    if (!g) return MGC_E_ARG;
    CK(cudaStreamSynchronize(g->stream));
    if (g->own_stream) { cudaStreamDestroy(g->stream); g->own_stream = false; }
    g->stream = (cudaStream_t)cuda_stream;
    return MGC_OK;
}

int mgc_synchronize(mgc_graph* g)
{
    if (!g) return MGC_E_ARG;
    CK(cudaStreamSynchronize(g->stream));
    return MGC_OK;
}

int mgc_add_regional_probability(mgc_graph* g, const mgc_array* prob, double alpha, int32_t compute_dtype)
{
    if (!g || !prob) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (g->flow_started) FAIL(MGC_E_STATE, "the graph has been solved (its capacities hold residuals): reset() it before adding terms");
    if (prob->dtype != MGC_F32 && prob->dtype != MGC_F64) FAIL(MGC_E_ARG, "probability map must be float32 or float64");
    if (compute_dtype != MGC_F32 && compute_dtype != MGC_F64) FAIL(MGC_E_ARG, "compute dtype must be float32 or float64");
    CK(cudaSetDevice(g->device));
    { int rc0 = push_state_all(g); if (rc0) return rc0; }       // the term adds to tr
    TermSpan t(g);
    const void* p = nullptr;
    int rc = stage_input(g, prob, 0, &p);
    if (rc) return rc;
    rc = check_pending(g);
    if (rc) return rc;
    if (prob->dtype == MGC_F32 && (g->L.n % 4u) == 0u && ((uintptr_t)p % 16u) == 0u)
        k_regional_f32x4<double><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const float4*)p, alpha, compute_dtype == MGC_F32, g->tr_fresh ? 1 : 0, g->partials);
    else if (prob->dtype == MGC_F32)
        k_regional<float, double><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const float*)p, alpha, compute_dtype == MGC_F32, g->tr_fresh ? 1 : 0, g->partials);
    else
        k_regional<double, double><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const double*)p, alpha, 0, g->tr_fresh ? 1 : 0, g->partials);
    g->tr_fresh = false;
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    rc = finish_flow_const(g);
    if (rc) return rc;
    invalidate(g);
    t.stop(1u);
    return MGC_OK;
}

int mgc_add_tweights_dense(mgc_graph* g, const mgc_array* src, const mgc_array* snk)
{
    if (!g || !src || !snk) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (g->flow_started) FAIL(MGC_E_STATE, "the graph has been solved (its capacities hold residuals): reset() it before adding terms");
    if (src->dtype != MGC_F64 || snk->dtype != MGC_F64) FAIL(MGC_E_ARG, "dense t-weights must be float64");
    CK(cudaSetDevice(g->device));
    { int rc0 = push_state_all(g); if (rc0) return rc0; }       // the term adds to tr
    TermSpan t(g);
    const void *ps = nullptr, *pk = nullptr;
    int rc = stage_input(g, src, 0, &ps);
    if (rc) return rc;
    rc = stage_input(g, snk, 1, &pk);
    if (rc) return rc;
    rc = check_pending(g);
    if (rc) return rc;
    k_tweights_dense<double><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const double*)ps, (const double*)pk, g->tr_fresh ? 1 : 0, g->partials);
    g->tr_fresh = false;
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    rc = finish_flow_const(g);
    if (rc) return rc;
    invalidate(g);
    t.stop(3u);
    return MGC_OK;
}

int mgc_add_markers(mgc_graph* g, const mgc_array* fg, const mgc_array* bg)
{
    if (!g) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (!fg && !bg) return MGC_OK;
    if (g->flow_started) FAIL(MGC_E_STATE, "the graph has been solved (its capacities hold residuals): reset() it before adding terms");
    if ((fg && fg->dtype != MGC_U8) || (bg && bg->dtype != MGC_U8)) FAIL(MGC_E_ARG, "markers must be uint8 / bool");
    CK(cudaSetDevice(g->device));
    { int rc0 = push_state_all(g); if (rc0) return rc0; }       // the term adds to tr
    TermSpan t(g);
    const void *pf = nullptr, *pb = nullptr;
    int rc = MGC_OK;
    if (fg) { rc = stage_input(g, fg, 1, &pf); if (rc) return rc; }
    if (bg) { rc = stage_input(g, bg, 4, &pb); if (rc) return rc; }
    rc = check_pending(g);      // after the uploads: they overlapped the boundary kernel whose verdict this is
    if (rc) return rc;
    const bool vec16 = !g->tr_fresh && (g->L.n % 16u) == 0u && ((uintptr_t)pf % 16u) == 0u && ((uintptr_t)pb % 16u) == 0u;
    if (vec16)
        k_markers16<double><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const uint4*)pf, (const uint4*)pb, g->partials);
    else
        k_markers<double><<<rblocks(g), 256, 0, g->stream>>>(g->L, g->S, (const uint8_t*)pf, (const uint8_t*)pb, g->tr_fresh ? 1 : 0, g->partials);
    g->tr_fresh = false;
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    rc = finish_flow_const(g);
    if (rc) return rc;
    invalidate(g);
    t.stop(0x12u);
    return MGC_OK;
}

int mgc_add_boundary(mgc_graph* g, int32_t kind, const mgc_array* image, double sigma, const double* spacing, double norm)
{
    if (!g || !image) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (kind < 0 || kind > 7) FAIL(MGC_E_ARG, "unknown boundary term");
    if (g->flow_started) FAIL(MGC_E_STATE, "the graph has been solved (its capacities hold residuals): reset() it before adding terms");
    CK(cudaSetDevice(g->device));
    { int rc0 = check_pending(g); if (rc0) return rc0; }
    { int rc0 = push_state_all(g); if (rc0) return rc0; }       // the term adds to every capacity
    TermSpan t(g);
    const void* img = nullptr;
    int rc = stage_input(g, image, 2, &img);
    if (rc) return rc;
    BoundaryParams P{};
    rc = boundary_params(g, kind, image->dtype, img, sigma, spacing, norm, &P);
    if (rc) return rc;
    CK(cudaMemsetAsync(g->d_flags, 0, sizeof(int), g->stream));
    cudaEventRecord(g->ev_b[0], g->stream);
    switch (image->dtype) {
        case MGC_F32: boundary_launch<float>(g, (const float*)img, P); break;
        case MGC_F64: boundary_launch<double>(g, (const double*)img, P); break;
        case MGC_U8: boundary_launch<uint8_t>(g, (const uint8_t*)img, P); break;
        case MGC_I16: boundary_launch<int16_t>(g, (const int16_t*)img, P); break;
        case MGC_I32: boundary_launch<int32_t>(g, (const int32_t*)img, P); break;
    }
    cudaEventRecord(g->ev_b[1], g->stream);
    CK(cudaGetLastError());
    invalidate(g);
    g->has_nlinks = true;
    g->boundary_timed = true;
    if (g->defer_check && g->h_bad && image->mem == MGC_MEM_HOST) {
        // verdict later: the next call's host->device copy overlaps this kernel (see MGC_OPT_DEFER_WEIGHT_CHECK)
        CK(cudaMemcpyAsync(g->h_bad, g->d_flags, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaEventRecord(g->ev_bad, g->stream));
        g->bad_pending = true;
        t.stop(4u);
        return MGC_OK;
    }
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, g->d_flags, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
    t.stop(4u);
    CK(cudaStreamSynchronize(g->stream));      // the weight check must be reported by this call (ValueError)
    if (bad) FAIL(MGC_E_WEIGHT, "Negative or zero weights are not allowed.");
    return MGC_OK;
}

int mgc_add_nweights_dense(mgc_graph* g, int32_t axis, const mgc_array* fwd, const mgc_array* bwd)
{
    if (!g || !fwd || !bwd) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (g->flow_started) FAIL(MGC_E_STATE, "the graph has been solved (its capacities hold residuals): reset() it before adding terms");
    if (axis < 0 || axis >= g->user_ndim) FAIL(MGC_E_ARG, "bad axis");
    if (fwd->dtype != MGC_F64 || bwd->dtype != MGC_F64) FAIL(MGC_E_ARG, "dense n-weights must be float64");
    CK(cudaSetDevice(g->device));
    { int rc0 = check_pending(g); if (rc0) return rc0; }
    { int rc0 = push_state_all(g); if (rc0) return rc0; }       // the term adds to the capacities of one axis
    TermSpan t(g);
    const void *pf = nullptr, *pb = nullptr;
    int rc = stage_input(g, fwd, 0, &pf);
    if (rc) return rc;
    rc = stage_input(g, bwd, 1, &pb);
    if (rc) return rc;
    if (g->caps_fresh) {
        const size_t nbz = (size_t)g->L.n;
        for (int k = 0; k < 2 * g->nd; ++k) CK(cudaMemsetAsync(g->S.cap[k], 0, nbz * sizeof(double), g->stream));
        g->caps_fresh = false;
    }
    CK(cudaMemsetAsync(g->d_flags, 0, sizeof(int), g->stream));
    const int ca = axis + g->shift;
    if (g->nd == 3) k_nweights_dense<3, double><<<nblocks(g), 256, 0, g->stream>>>(g->L, g->S, ca, (const double*)pf, (const double*)pb, g->d_flags);
    else            k_nweights_dense<4, double><<<nblocks(g), 256, 0, g->stream>>>(g->L, g->S, ca, (const double*)pf, (const double*)pb, g->d_flags);
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, g->d_flags, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
    t.stop(3u);
    CK(cudaStreamSynchronize(g->stream));
    invalidate(g);
    g->has_nlinks = true;
    if (bad) FAIL(MGC_E_WEIGHT, "Negative or zero weights are not allowed.");
    return MGC_OK;
}

int mgc_get_mask(mgc_graph* g, uint8_t* out, int32_t mem)
{
    if (!g || !out) return MGC_E_ARG;
    if (!g->solved) FAIL(MGC_E_STATE, "call maxflow first");
    CK(cudaSetDevice(g->device));
    const size_t owned_n = (size_t)(g->L.own1 - g->L.own0) * g->L.plane;
    const uint8_t* src = g->mask_dev + (size_t)g->L.own0 * g->L.plane;
    CK(cudaMemcpyAsync(out, src, owned_n, mem == MGC_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    return MGC_OK;
}

int mgc_what_segment(mgc_graph* g, int64_t node, int32_t* segment)
{
    if (!g || !segment) return MGC_E_ARG;
    if (!g->solved) FAIL(MGC_E_STATE, "call maxflow first");
    if (node < 0 || node >= (int64_t)g->L.n) FAIL(MGC_E_ARG, "node id out of range");
    if (!g->host_mask_valid) {
        g->host_mask.resize(g->L.n);
        CK(cudaMemcpyAsync(g->host_mask.data(), g->mask_dev, g->L.n, cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        g->host_mask_valid = true;
    }
    *segment = g->host_mask[(size_t)node] ? MGC_SOURCE : MGC_SINK;
    return MGC_OK;
}

int mgc_get_edge(mgc_graph* g, int64_t i, int64_t j, double* cap)
{
    if (!g || !cap) return MGC_E_ARG;
    const int64_t n = (int64_t)g->L.n;
    if (i < 0 || j < 0 || i >= n || j >= n || i == j) FAIL(MGC_E_ARG, "bad node ids");
    *cap = 0.0;
    if (g->caps_fresh) return MGC_OK;
    CK(cudaSetDevice(g->device));
    { int rc0 = push_state_all(g); if (rc0) return rc0; }
    int c[4] = {0, 0, 0, 0};
    unsigned r = (unsigned)i;
    for (int d = 0; d < g->nd; ++d) { c[d] = (int)(r / g->L.stride[d]); r %= g->L.stride[d]; }
    for (int k = 0; k < 2 * g->nd; ++k) {
        const int d = k >> 1;
        const int64_t off = (k & 1) ? (int64_t)g->L.stride[d] : -(int64_t)g->L.stride[d];
        const int cn = c[d] + ((k & 1) ? 1 : -1);
        if (cn < 0 || cn >= g->L.dim[d]) continue;
        if (i + off == j) {
            CK(cudaMemcpyAsync(cap, g->S.cap[k] + i, sizeof(double), cudaMemcpyDeviceToHost, g->stream));
            CK(cudaStreamSynchronize(g->stream));
            caps_resolve(g);
            return MGC_OK;
        }
    }
    return MGC_OK;  // not lattice neighbours: 0, like get_edge on a missing arc (graph.h:482-497)
}

int mgc_get_trcap(mgc_graph* g, int64_t node, double* trcap)
{
    if (!g || !trcap) return MGC_E_ARG;
    if (node < 0 || node >= (int64_t)g->L.n) FAIL(MGC_E_ARG, "node id out of range");
    if (g->tr_fresh) { *trcap = 0.0; return MGC_OK; }
    CK(cudaSetDevice(g->device));
    { int rc0 = push_state_all(g); if (rc0) return rc0; }       // tr before the flow, excess after it
    if (!g->state_init || !g->flow_started) {      // no flow yet: the net terminal capacity exactly as add_tweights left it
        CK(cudaMemcpyAsync(trcap, g->S.tr + node, sizeof(double), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaStreamSynchronize(g->stream));
        return MGC_OK;
    }
    double e = 0, s = 0;
    uint8_t rm = 0x80u;
    CK(cudaMemcpyAsync(&e, g->S.excess + node, sizeof(double), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaMemcpyAsync(&s, g->S.sink + node, sizeof(double), cudaMemcpyDeviceToHost, g->stream));
    if (g->nd == 3) CK(cudaMemcpyAsync(&rm, g->S.rmask + node, 1, cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    if (!(rm & 0x80u)) s = 0;        // RM_SINKV clear: nothing absorbed yet, the entry was never written
    double tr = 0;
    CK(cudaMemcpyAsync(&tr, g->S.tr + node, sizeof(double), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    *trcap = (tr < 0 && -tr - s > 0) ? -(-tr - s) : e;
    return MGC_OK;
}

int mgc_get_node_num(const mgc_graph* g, int64_t* n)
{
    if (!g || !n) return MGC_E_ARG;
    *n = (int64_t)g->L.n;
    return MGC_OK;
}

int mgc_get_arc_num(const mgc_graph* g, int64_t* n)
{
    if (!g || !n) return MGC_E_ARG;
    int64_t e = 0;
    if (g->has_nlinks)
        for (int d = 0; d < g->nd; ++d)
            if (g->L.dim[d] > 1) e += ((int64_t)g->L.n / g->L.dim[d]) * (g->L.dim[d] - 1);
    *n = 2 * e;
    return MGC_OK;
}

int mgc_get_stats(const mgc_graph* g, mgc_stats* out)
{
    if (!g || !out) return MGC_E_ARG;
    *out = g->st;
    out->device_bytes = g->device_bytes;
    return MGC_OK;
}

}  // extern "C"
