// gc_batch.cu -- batches of independent images in one lattice handle (DESIGN.md §3.1): mgc_create_batch,
// mgc_build_voxel_batch, mgc_get_batch_energies, the per-image term constants of the build and the per-image read-out.
//
// B images of canonical shape (Z, Y, X) are stacked along axis 0 into one (B * Z, Y, X) lattice with Lattice::zper = Z.
// z_pairs (gc_common.cuh) severs the pairs across the seams, so every seam arc has capacity 0 and no rmask bit: the
// solver, which only sees capacities and rmask bits, computes B independent minimum cuts without knowing about images.
#include "gc_handle.cuh"

#include <algorithm>
#include <cmath>

namespace {
// The per-image reductions run one block per (image b, chunk c) on a 1-D grid, block b * chunks + c, so that a batch
// of any size fits the grid (gridDim.y / z stop at 65535); chunk c of image b covers its voxels c * 256 + t, stepping by
// chunks * 256, and stores partials[b * chunks + c].
//
// The add_tweights minima of the image's voxels, replayed from the build's t-link inputs exactly as the build replays them
// (tlink_replay)
__global__ void __launch_bounds__(256) k_batch_tconst(Lattice L, BuildArgs A, unsigned chunks, double* __restrict__ partials)
{
    const unsigned per = (unsigned)L.zper * L.plane, base = (blockIdx.x / chunks) * per, c = blockIdx.x % chunks;
    double m = 0.0;
    for (unsigned i = c * blockDim.x + threadIdx.x; i < per; i += chunks * blockDim.x) {
        const unsigned v = base + i;
        double p = 0.0;
        unsigned fb = 0u;
        if (A.prob) p = A.prob_f64 ? reinterpret_cast<const double*>(A.prob)[v] : (double)reinterpret_cast<const float*>(A.prob)[v];
        if (A.fg_bits) fb |= (A.fg_bits[v >> 5] >> (v & 31u)) & 1u;
        if (A.bg_bits) fb |= ((A.bg_bits[v >> 5] >> (v & 31u)) & 1u) << 1;
        if (A.fg && A.fg[v]) fb |= 1u;
        if (A.bg && A.bg[v]) fb |= 2u;
        double tr = 0.0;
        m = __dadd_rn(m, tlink_replay<double>(tr, A.prob != nullptr, p, A.compute_f32 != 0, A.alpha, fb));
    }
    block_sum_store(m, partials);
}

// the flow the image's sink links absorbed (sink[v] where rmask bit RM_SINKV is set, as k_readout reads it)
__global__ void __launch_bounds__(256) k_batch_sink(Lattice L, State<double> S, unsigned chunks, double* __restrict__ partials)
{
    const unsigned per = (unsigned)L.zper * L.plane, base = (blockIdx.x / chunks) * per, c = blockIdx.x % chunks;
    double m = 0.0;
    for (unsigned i = c * blockDim.x + threadIdx.x; i < per; i += chunks * blockDim.x) {
        const unsigned v = base + i;
        if (S.rmask[v] & RM_SINKV) m = __dadd_rn(m, S.sink[v]);
    }
    block_sum_store(m, partials);
}

// out[b] = add[b] (0 without `add`) + the fixed-order sum of partials[b * n .. (b + 1) * n); one block per image
__global__ void __launch_bounds__(256) k_batch_sum(const double* __restrict__ partials, unsigned n, const double* __restrict__ add,
                                                   double* __restrict__ out)
{
    __shared__ double sh[256];
    const unsigned tid = threadIdx.x;
    const double* p = partials + (size_t)blockIdx.x * n;
    double s = 0.0;
    for (unsigned i = tid; i < n; i += 256) s = __dadd_rn(s, p[i]);
    sh[tid] = s;
    __syncthreads();
    for (unsigned k = 128; k > 0; k >>= 1) {
        if (tid < k) sh[tid] = __dadd_rn(sh[tid], sh[tid + k]);
        __syncthreads();
    }
    if (tid == 0) out[blockIdx.x] = add ? __dadd_rn(add[blockIdx.x], sh[0]) : sh[0];
}

// ktab[b] = the image's linear normaliser M where the caller left NaN: mm[2b] = |max - min|, mm[2b + 1] = max |x|
// (k_minmax_final); `which` selects the second (boundary_maximum_linear)
__global__ void k_batch_norms(double* __restrict__ ktab, const double* __restrict__ mm, int B, int which)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B && ktab[b] != ktab[b]) ktab[b] = mm[2 * b + which];
}

// The change a fold made to the add_tweights constant, per image: tconst[b] += the sum of dk[i] over the fold's entries i
// < *count in image b.  The entries are in ascending voxel order (vox[i * vstride] is entry i's voxel), so each image's
// entries form one run.  Two passes over fixed chunks of FOLD_CHUNK entries, so the same calls give the same bits and no
// chain of dependent steps grows with the length of a run:
//   k_batch_fold_chunks: one block per chunk sums every piece of a run inside the chunk with a segmented Hillis-Steele
//     scan (eight fixed steps).  A run that starts and ends in the chunk goes straight into tconst[b]; the piece at the
//     chunk's start of a run that began earlier is cont[c]; the piece at its end of a run that goes on is head[c], with
//     span[c] = b (else -1);
//   k_batch_fold_spans: one block per chunk with span[c] = b finds the end of b's run (a binary search over the entries)
//     and adds head[c] + the cont[] of the chunks the run covers, summed by the block in a fixed tree.
// Each image is written by one thread of one block.  The work is proportional to the entries, not to B.
constexpr unsigned FOLD_CHUNK = 256;

__device__ __forceinline__ int fold_image(const Lattice& L, const unsigned* __restrict__ vox, int vstride, unsigned i)
{
    return image_of(L, (int)div_stride(L, __ldg(vox + (size_t)i * (unsigned)vstride), 0));
}

__global__ void __launch_bounds__(FOLD_CHUNK) k_batch_fold_chunks(Lattice L, const unsigned* __restrict__ vox, int vstride,
                                                                  const int* __restrict__ count,
                                                                  const double* __restrict__ dk, double* __restrict__ tconst,
                                                                  double* __restrict__ cont, double* __restrict__ head,
                                                                  int* __restrict__ span)
{
    __shared__ double sv[FOLD_CHUNK];
    __shared__ unsigned char sf[FOLD_CHUNK];
    __shared__ int s_first;                    // the image of the chunk's first entry if its run began earlier, else -1
    const unsigned n = (unsigned)*count;       // < 2^31: no index below overflows
    const unsigned t = threadIdx.x;
    for (unsigned c = blockIdx.x; c * FOLD_CHUNK < n; c += gridDim.x) {
        const unsigned i = c * FOLD_CHUNK + t;
        const bool in = i < n;
        int b = -1;
        double v = 0.0;
        bool start = false;                    // the run of b starts at i
        if (in) {
            b = fold_image(L, vox, vstride, i);
            start = i == 0 || fold_image(L, vox, vstride, i - 1) != b;
            v = dk[i];
        }
        if (t == 0) { s_first = start ? -1 : b; span[c] = -1; }
        bool f = t == 0 || start;              // a piece starts at t
        sv[t] = v;
        sf[t] = f;
        __syncthreads();
        for (unsigned d = 1; d < FOLD_CHUNK; d <<= 1) {
            double pv = 0.0;
            bool pf = true;
            if (t >= d) { pv = sv[t - d]; pf = sf[t - d] != 0; }
            __syncthreads();
            if (!f) { v = __dadd_rn(pv, v); f = pf; }
            sv[t] = v;
            sf[t] = f;
            __syncthreads();
        }
        if (in) {
            const bool ends = i + 1 == n || fold_image(L, vox, vstride, i + 1) != b;     // the run of b ends at i
            if (ends || t + 1 == FOLD_CHUNK) {                                          // i ends its piece
                if (b == s_first) cont[c] = v;
                else if (ends) tconst[b] = __dadd_rn(tconst[b], v);
                else { head[c] = v; span[c] = b; }
            }
        }
        __syncthreads();                       // s_first and the scan arrays are reused by the next chunk
    }
}

__global__ void __launch_bounds__(FOLD_CHUNK) k_batch_fold_spans(Lattice L, const unsigned* __restrict__ vox, int vstride,
                                                                 const int* __restrict__ count,
                                                                 const double* __restrict__ cont,
                                                                 const double* __restrict__ head,
                                                                 const int* __restrict__ span, double* __restrict__ tconst)
{
    __shared__ double sh[FOLD_CHUNK];
    __shared__ unsigned s_last;
    const unsigned n = (unsigned)*count;
    const unsigned t = threadIdx.x;
    for (unsigned c = blockIdx.x; c * FOLD_CHUNK < n; c += gridDim.x) {
        const int b = span[c];                 // block-uniform
        if (b < 0) continue;
        if (t == 0) {
            // the first entry past b's run, in (c + 1) * FOLD_CHUNK .. n: the images are ascending
            unsigned lo = (c + 1) * FOLD_CHUNK, hi = n;
            while (lo < hi) {
                const unsigned mid = lo + ((hi - lo) >> 1);
                if (fold_image(L, vox, vstride, mid) <= b) lo = mid + 1; else hi = mid;
            }
            s_last = (lo - 1) / FOLD_CHUNK;    // the chunk of the run's last entry
        }
        __syncthreads();
        double s = 0.0;
        for (unsigned k = c + 1 + t; k <= s_last; k += FOLD_CHUNK) s = __dadd_rn(s, cont[k]);
        sh[t] = s;
        __syncthreads();
        for (unsigned k = FOLD_CHUNK / 2; k > 0; k >>= 1) {
            if (t < k) sh[t] = __dadd_rn(sh[t], sh[t + k]);
            __syncthreads();
        }
        if (t == 0) tconst[b] = __dadd_rn(tconst[b], __dadd_rn(head[c], sh[0]));
        __syncthreads();                       // s_last and sh are reused by the next chunk
    }
}

double* ktab_of(mgc_graph* g) { return g->batch_buf; }
double* tconst_of(mgc_graph* g) { return g->batch_buf + g->batch; }
double* energy_of(mgc_graph* g) { return g->batch_buf + 2 * g->batch; }
double* mm_of(mgc_graph* g) { return g->batch_buf + 3 * g->batch; }
double* part_of(mgc_graph* g) { return g->batch_buf + 5 * g->batch; }
}  // namespace

// A (B, ...) input array as a C-contiguous array over the batch lattice (B * Z, Y, X): the array itself with the
// lattice's strides when it is one, else a copy gathered into the staging slot (what stage_input does for a strided
// input of a single image; the build, or the dense fold that stages the result, then reads the slot in place).
int batch_view(mgc_graph* g, const mgc_array* a, int slot, mgc_array* out)
{
    const size_t es = dtype_size(a->dtype);
    if (!es) FAIL(MGC_E_ARG, "unsupported dtype");
    if (!a->data) FAIL(MGC_E_ARG, "null array");
    const int nd = g->batch_ndim;
    const int dim4[4] = {(int)g->batch, g->L.zper, g->L.dim[1], g->L.dim[2]};
    Strides4 st{};
    st.s[0] = a->strides[0];
    for (int u = 1; u <= nd; ++u) st.s[4 - nd + u - 1] = a->strides[u];
    bool contiguous = true;
    long long expect = (long long)es, span = (long long)es;
    for (int d = 3; d >= 0; --d) {
        if (dim4[d] > 1) {
            if (st.s[d] <= 0) FAIL(MGC_E_ARG, "array strides must be positive (pass a contiguous copy)");
            if (st.s[d] != expect) contiguous = false;
            span += (long long)(dim4[d] - 1) * st.s[d];
        } else {
            st.s[d] = 0;
        }
        expect *= dim4[d];
    }
    *out = *a;
    for (int d = 0; d < MGC_MAX_NDIM; ++d) out->strides[d] = 0;
    out->strides[2] = (int64_t)es;
    out->strides[1] = (int64_t)(es * (size_t)g->L.dim[2]);
    out->strides[0] = (int64_t)(es * (size_t)g->L.plane);
    if (contiguous) return MGC_OK;
    int rc = ensure_scratch(g, g->scratch[slot], (size_t)g->L.n * es);
    if (rc) return rc;
    const char* src = (const char*)a->data;
    if (a->mem == MGC_MEM_HOST) {
        rc = ensure_scratch(g, g->raw, (size_t)span);
        if (rc) return rc;
        rc = upload(g, g->raw.p, a->data, (size_t)span, 3);
        if (rc) return rc;
        src = (const char*)g->raw.p;
    }
    // the gather decodes the voxel index over the 4-D (B, Z, Y, X) shape
    Lattice L4 = g->L;
    unsigned s = g->L.n;
    for (int d = 0; d < 4; ++d) {
        L4.dim[d] = dim4[d];
        s /= (unsigned)dim4[d];
        L4.stride[d] = s;
        L4.magic[d] = s <= 1 ? 0ull : (~0ull / s) + 1ull;
    }
    const unsigned nb = (g->L.n + 255u) / 256u;
    void* dst = g->scratch[slot].p;
    switch (a->dtype) {
        case MGC_F32: k_gather<float, 4><<<nb, 256, 0, g->stream>>>(L4, src, st, (float*)dst); break;
        case MGC_F64: k_gather<double, 4><<<nb, 256, 0, g->stream>>>(L4, src, st, (double*)dst); break;
        case MGC_U8: k_gather<uint8_t, 4><<<nb, 256, 0, g->stream>>>(L4, src, st, (uint8_t*)dst); break;
        case MGC_I16: k_gather<int16_t, 4><<<nb, 256, 0, g->stream>>>(L4, src, st, (int16_t*)dst); break;
        default: k_gather<int32_t, 4><<<nb, 256, 0, g->stream>>>(L4, src, st, (int32_t*)dst); break;
    }
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    if (a->mem == MGC_MEM_HOST) { CK(cudaEventRecord(g->ev_slot[3], g->stream)); g->slot_used[3] = true; }
    out->data = dst;
    out->mem = MGC_MEM_DEVICE;
    return MGC_OK;
}

// Chunks of the per-image constant sum for a fold of at most max_count entries (the size of `part`: 2 doubles each, and
// of `span`: 1 int each)
size_t batch_fold_chunks(int max_count) { return ((size_t)(max_count > 0 ? max_count : 0) + FOLD_CHUNK - 1) / FOLD_CHUNK; }

// The per-image constant sum after a fold's kernels, on the fold's entries (at most max_count; their count is on the
// device); part / span: scratch of batch_fold_chunks(max_count) chunks
int batch_fold_const(mgc_graph* g, const unsigned* vox, int vstride, const int* count, int max_count, const double* dk,
                     double* part, int* span)
{
    const size_t chunks = batch_fold_chunks(max_count);
    if (!chunks) return MGC_OK;
    const unsigned grid = (unsigned)std::min<size_t>(chunks, (size_t)g->n_ctas * 4u);
    double* cont = part;
    double* head = part + chunks;
    k_batch_fold_chunks<<<grid, FOLD_CHUNK, 0, g->stream>>>(g->L, vox, vstride, count, dk, tconst_of(g), cont, head, span);
    k_batch_fold_spans<<<grid, FOLD_CHUNK, 0, g->stream>>>(g->L, vox, vstride, count, cont, head, span, tconst_of(g));
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    return MGC_OK;
}

// The term-constant table of a batch build (BoundaryParams::ktab): the host values of mgc_build_voxel_batch, and for the
// linear terms the normaliser M of every image whose entry is NaN, reduced on the device over that image alone
int batch_constants(mgc_graph* g, int dtype, const void* d_img, BoundaryParams* P)
{
    const int B = (int)g->batch;
    CK(cudaMemcpyAsync(ktab_of(g), g->batch_k_host.data(), (size_t)B * sizeof(double), cudaMemcpyHostToDevice, g->stream));
    if (P->fn == 0) {
        const unsigned per = g->L.n / (unsigned)B;
        const size_t es = dtype_size(dtype);
        bool any = false;
        for (int b = 0; b < B; ++b) {
            if (!std::isnan(g->batch_k_host[b])) continue;
            int rc = minmax_dtype(g, dtype, (const char*)d_img + (size_t)b * per * es, per, mm_of(g) + 2 * b);
            if (rc) return rc;
            any = true;
        }
        if (any) {
            k_batch_norms<<<(B + 255) / 256, 256, 0, g->stream>>>(ktab_of(g), mm_of(g), B, P->use_max ? 1 : 0);
            g->st.kernel_launches++;
        }
        CK(cudaGetLastError());
    }
    P->ktab = ktab_of(g);
    return MGC_OK;
}

// out[b] = the fixed-order sum of partials[b * n .. (b + 1) * n), for every image b (k_batch_sum)
void batch_sum(mgc_graph* g, const double* partials, unsigned n, double* out)
{
    k_batch_sum<<<(unsigned)g->batch, 256, 0, g->stream>>>(partials, n, nullptr, out);
    g->st.kernel_launches++;
}

// the per-image add_tweights constants of the build whose t-link inputs A holds
int batch_tconst(mgc_graph* g, const BuildArgs& A)
{
    const unsigned chunks = (unsigned)g->batch_chunks;
    k_batch_tconst<<<(unsigned)g->batch * chunks, 256, 0, g->stream>>>(g->L, A, chunks, part_of(g));
    k_batch_sum<<<(unsigned)g->batch, 256, 0, g->stream>>>(part_of(g), (unsigned)g->batch_chunks, nullptr, tconst_of(g));
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    return MGC_OK;
}

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

int mgc_create_batch(int32_t ndim, const int64_t* image_shape, int64_t batch, int32_t device, mgc_graph** out)
{
    if (!out) return MGC_E_ARG;
    *out = nullptr;
    if (ndim < 1 || ndim > 3 || !image_shape) { g_create_error = "batch images are 1-D..3-D"; return MGC_E_ARG; }
    if (batch < 1) { g_create_error = "a batch holds at least one image"; return MGC_E_ARG; }
    int64_t dims[3] = {1, 1, 1};
    for (int d = 0; d < ndim; ++d) {
        if (image_shape[d] < 1) { g_create_error = "extents must be >= 1"; return MGC_E_ARG; }
        dims[d + 3 - ndim] = image_shape[d];
    }
    const int64_t limit = (int64_t(1) << 31) - 1;
    if (dims[0] > limit / dims[1] / dims[2] || dims[0] * dims[1] * dims[2] > limit / batch) {
        g_create_error = "batch too large for one handle: images x voxels per image must stay below 2^31";
        return MGC_E_ARG;
    }
    const int64_t shape[3] = {batch * dims[0], dims[1], dims[2]};
    mgc_graph* g = nullptr;
    int rc = mgc_create(3, shape, device, &g);
    if (rc) return rc;
    g->batch = batch;
    g->batch_ndim = ndim;
    g->L.zper = (int)dims[0];
    g->L.zmagic = dims[0] <= 1 ? 0ull : (~0ull / (unsigned long long)dims[0]) + 1ull;
    const int64_t per = dims[0] * dims[1] * dims[2];
    const int64_t chunks = (per + 2047) / 2048;
    g->batch_chunks = (int)(chunks < 1 ? 1 : (chunks > 64 ? 64 : chunks));
    void* p = nullptr;
    rc = alloc_buf(g, (size_t)batch * (5 + (size_t)g->batch_chunks) * sizeof(double), &p);
    if (rc) { g_create_error = g->err; mgc_destroy(g); return rc; }
    g->batch_buf = (double*)p;
    *out = g;
    return MGC_OK;
}

int mgc_build_voxel_batch(mgc_graph* g, const mgc_voxel_terms* t, const double* sigmas, const double* norms)
{
    if (!g || !t) return MGC_E_ARG;
    if (!g->batch) FAIL(MGC_E_STATE, "not a batch handle (mgc_create_batch)");
    if (!g->fuse_build) FAIL(MGC_E_STATE, "batch builds need the fused graph build (MEDPY_GC_FUSE=0 switches it off)");
    if (g->flow_started || !g->caps_fresh || !g->tr_fresh || g->state_init)
        FAIL(MGC_E_STATE, "a batch handle is built once: reset() it before building it again");
    if (t->boundary_kind < 0 || t->boundary_kind > 7) FAIL(MGC_E_ARG, "a batch needs one of the eight boundary terms");
    if (!t->image) FAIL(MGC_E_ARG, "boundary term without image");
    if (t->fg_bits || t->bg_bits) FAIL(MGC_E_ARG, "a batch takes its markers as uint8 arrays");
    CK(cudaSetDevice(g->device));
    const int B = (int)g->batch;
    const int fn = t->boundary_kind & 3;
    g->batch_k_host.resize((size_t)B);
    bool any_nan = false;
    for (int b = 0; b < B; ++b) {
        const double sigma = sigmas ? sigmas[b] : t->sigma;
        const double norm = norms ? norms[b] : t->norm;
        g->batch_k_host[b] = fn == 0 ? norm : (fn == 1 ? pow(sigma, 2) : sigma);    // as boundary_params forms them
        any_nan = any_nan || (fn == 0 && std::isnan(norm));
    }
    mgc_voxel_terms u = *t;
    double sp[3] = {1.0, 1.0, 1.0};            // image axes -> lattice axes (leading axes of 1-D and 2-D images: no pairs)
    if (t->spacing) {
        for (int d = 0; d < g->batch_ndim; ++d) sp[3 - g->batch_ndim + d] = t->spacing[d];
        u.spacing = sp;
    }
    mgc_array img, prob, fg, bg;
    int rc = batch_view(g, t->image, 2, &img); if (rc) return rc;
    u.image = &img;
    if (t->prob) { rc = batch_view(g, t->prob, 0, &prob); if (rc) return rc; u.prob = &prob; }
    if (t->fg) { rc = batch_view(g, t->fg, 1, &fg); if (rc) return rc; u.fg = &fg; }
    if (t->bg) { rc = batch_view(g, t->bg, 4, &bg); if (rc) return rc; u.bg = &bg; }
    // (a NaN normaliser keeps host images out of the chunked upload: the images are reduced before the build starts)
    u.norm = any_nan ? NAN : 0.0;
    g->batch_built = false;
    rc = voxel_build(g, &u);
    g->batch_built = rc == MGC_OK;
    return rc;
}

int mgc_get_batch_energies(mgc_graph* g, double* out)
{
    if (!g || !out) return MGC_E_ARG;
    if (!g->batch) FAIL(MGC_E_STATE, "not a batch handle (mgc_create_batch)");
    // the per-image add_tweights constants exist only for a state mgc_build_voxel_batch made
    if (!g->batch_built) FAIL(MGC_E_STATE, "the batch handle has not been built since it was created or reset: call mgc_build_voxel_batch");
    if (!g->solved) FAIL(MGC_E_STATE, "call maxflow first");
    CK(cudaSetDevice(g->device));
    const unsigned chunks = (unsigned)g->batch_chunks;
    k_batch_sink<<<(unsigned)g->batch * chunks, 256, 0, g->stream>>>(g->L, g->S, chunks, part_of(g));
    k_batch_sum<<<(unsigned)g->batch, 256, 0, g->stream>>>(part_of(g), (unsigned)g->batch_chunks, tconst_of(g), energy_of(g));
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, energy_of(g), (size_t)g->batch * sizeof(double), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    return MGC_OK;
}

}  // extern "C"
