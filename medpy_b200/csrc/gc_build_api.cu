// gc_build_api.cu -- the fused graph build of a lattice handle (gc_handle.cuh): mgc_build_voxel_graph and the launches
// of the build kernels of gc_build.cuh.
#include "gc_handle.cuh"

#include <atomic>
#include <cmath>
#include <cstdlib>
#include <thread>
#include <type_traits>
#include <utility>

namespace {
// ---- fused graph build (gc_build.cuh) ------------------------------------------------------------------
// rank-3 tensor map of the image with the 10 x 10 x BUILD_BX halo box; false when the 16-byte rules are not met
bool make_image_map(mgc_graph* g, const void* img, int dtype, CUtensorMap* out)
{
    tmap_encode_fn encode = tensor_map_encoder();
    if (!encode) return false;
    const size_t es = dtype_size(dtype);
    const cuuint64_t X = (cuuint64_t)g->L.dim[2], Y = (cuuint64_t)g->L.dim[1], Z = (cuuint64_t)g->L.dim[0];
    if ((X * es) % 16 || ((uintptr_t)img & 15)) return false;
    CUtensorMapDataType dt;
    switch (dtype) {
        case MGC_F32: dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32; break;
        case MGC_F64: dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT64; break;
        case MGC_U8: dt = CU_TENSOR_MAP_DATA_TYPE_UINT8; break;
        case MGC_I16: dt = CU_TENSOR_MAP_DATA_TYPE_UINT16; break;     // moved as raw 2-byte words
        default: dt = CU_TENSOR_MAP_DATA_TYPE_INT32; break;
    }
    const cuuint64_t dims[3] = {X, Y, Z};
    const cuuint64_t strides[2] = {X * es, X * Y * es};
    cuuint32_t bx = 0;
    switch (dtype) {
        case MGC_F32: bx = BuildBox<float>::BX; break;
        case MGC_F64: bx = BuildBox<double>::BX; break;
        case MGC_U8: bx = BuildBox<uint8_t>::BX; break;
        case MGC_I16: bx = BuildBox<int16_t>::BX; break;
        default: bx = BuildBox<int32_t>::BX; break;
    }
    const cuuint32_t box[3] = {bx, BUILD_HY, BUILD_HZ};
    const cuuint32_t estr[3] = {1, 1, 1};
    return encode(out, dt, 3, const_cast<void*>(img), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// rank-3 tensor map of a C-contiguous array over the local lattice with an 8 x 8 x 32 box (probability map, marker bytes)
bool make_block_map(mgc_graph* g, const void* ptr, int dtype, CUtensorMap* out)
{
    tmap_encode_fn encode = tensor_map_encoder();
    if (!encode || !ptr) return false;
    const size_t es = dtype_size(dtype);
    const cuuint64_t X = (cuuint64_t)g->L.dim[2], Y = (cuuint64_t)g->L.dim[1], Z = (cuuint64_t)g->L.dim[0];
    if ((X * es) % 16 || ((uintptr_t)ptr & 15)) return false;
    const CUtensorMapDataType dt = dtype == MGC_F64 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : (dtype == MGC_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8);
    const cuuint64_t dims[3] = {X, Y, Z};
    const cuuint64_t strides[2] = {X * es, X * Y * es};
    const cuuint32_t box[3] = {BUILD_TX, BUILD_TY, BUILD_TZ};
    const cuuint32_t estr[3] = {1, 1, 1};
    return encode(out, dt, 3, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// The lazy build under the exponential term without spacing, image staged by TMA: k_build_lean over the whole grid, then
// k_build_refused on the blocks it refused (gc_build.cuh).  No host synchronisation: the second launch reads the count.
template <typename E, int USE_MAX, int TIN>
int build_launch_split(mgc_graph* g, const BuildMaps& imap, const BuildArgs& A, const BoundaryParams& P, int nz_layers)
{
    auto lean = k_build_lean<E, TIN>;
    auto ref = k_build_refused<E, USE_MAX, TIN>;
    const size_t smem_lean = LeanSmem<E, TIN>::BYTES, smem_ref = build_smem_bytes<E>();
    static int ref_ctas = 0;             // per instantiation: persistent CTAs of the refused launch
    if (!ref_ctas) {
        cudaFuncSetAttribute(lean, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_lean);
        cudaFuncSetAttribute(ref, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ref);
        int nb = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, ref, BUILD_THREADS, smem_ref) != cudaSuccess || nb < 1) {
            cudaGetLastError();
            nb = 1;
        }
        ref_ctas = nb * cached_sm_count(g->device);
    }
    const int nbx = (g->L.dim[2] + BUILD_TX - 1) / BUILD_TX, nby = (g->L.dim[1] + BUILD_TY - 1) / BUILD_TY;
    int* count = g->d_flags + 6;         // blocks refused by this lean launch
    int* total = g->d_flags + 7;         // ... by every lean launch of the build
    CK(cudaMemsetAsync(count, 0, sizeof(int), g->stream));
    lean<<<dim3((unsigned)nbx, (unsigned)nby, (unsigned)nz_layers), BUILD_THREADS, smem_lean, g->stream>>>(
        g->L, g->TL, g->S, imap, A, P, g->partials, g->rflag, rl(g, 0), g->pflag, pl(g, 0, 0), pl(g, 1, 0), g->build_refused,
        count, g->build_refuse_all ? 1 : 0);
    CK(cudaGetLastError());
    const int nblk = nbx * nby * nz_layers;
    ref<<<(unsigned)(nblk < ref_ctas ? nblk : ref_ctas), BUILD_THREADS, smem_ref, g->stream>>>(
        g->L, g->TL, g->S, imap, A, P, g->d_flags, g->partials, g->rflag, rl(g, 0), g->pflag, pl(g, 0, 0), pl(g, 1, 0),
        g->build_refused, count, total, nbx, nby);
    g->st.kernel_launches += 2;
    CK(cudaGetLastError());
    return MGC_OK;
}

template <typename E, int FN, int USE_MAX, int SPACING, int TIN, int LAZY>
int build_launch_inst(mgc_graph* g, const BuildMaps& imap, const BuildArgs& A, const BoundaryParams& P, int nz_layers)
{
    if constexpr (LAZY && FN == 1 && SPACING == 0 && USE_MAX >= 0 && (std::is_same<E, float>::value || std::is_same<E, double>::value))
        if (A.use_tma) return build_launch_split<E, USE_MAX, TIN>(g, imap, A, P, nz_layers);
    auto kern = k_build_tile<E, double, FN, USE_MAX, SPACING, TIN, LAZY>;
    const size_t smem = build_smem_bytes<E>();
    static bool attr_done = false;       // per instantiation
    if (!attr_done) { cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr_done = true; }
    const dim3 grid((unsigned)((g->L.dim[2] + BUILD_TX - 1) / BUILD_TX), (unsigned)((g->L.dim[1] + BUILD_TY - 1) / BUILD_TY), (unsigned)nz_layers);
    kern<<<grid, BUILD_THREADS, smem, g->stream>>>(g->L, g->TL, g->S, imap, A, P, g->d_flags, g->partials, g->rflag, rl(g, 0), g->pflag,
                                                     pl(g, 0, 0), pl(g, 1, 0));
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    return MGC_OK;
}

template <typename E, int LAZY>
int build_launch(mgc_graph* g, const BuildMaps& imap, const BuildArgs& A, const BoundaryParams& P, int nz_layers)
{
    if constexpr (!std::is_integral<E>::value) {
        if (P.fn == 1 && P.inv_spacing_on == 0.0) {
            if constexpr (std::is_same<E, float>::value) {
                // float32 image + float32 probability map + byte markers, everything staged by TMA: the compile-time variant
                const bool fast = A.use_tma && A.prob && !A.prob_f64 && A.compute_f32 && A.tma_prob && A.tma_mark == 3 &&
                                  !A.fg_bits && !A.bg_bits && A.dbg == 0;
                if (fast) {
                    if (P.use_max) return build_launch_inst<E, 1, 1, 0, 1, LAZY>(g, imap, A, P, nz_layers);
                    return build_launch_inst<E, 1, 0, 0, 1, LAZY>(g, imap, A, P, nz_layers);
                }
            }
            if (P.use_max) return build_launch_inst<E, 1, 1, 0, 0, LAZY>(g, imap, A, P, nz_layers);
            return build_launch_inst<E, 1, 0, 0, 0, LAZY>(g, imap, A, P, nz_layers);
        }
    }
    return build_launch_inst<E, -1, -1, -1, 0, LAZY>(g, imap, A, P, nz_layers);
}

template <int LAZY>
int build_launch_dtype(mgc_graph* g, int dtype, const BuildMaps& imap, const BuildArgs& A, const BoundaryParams& P, int nz_layers)
{
    switch (dtype) {
        case MGC_F32: return build_launch<float, LAZY>(g, imap, A, P, nz_layers);
        case MGC_F64: return build_launch<double, LAZY>(g, imap, A, P, nz_layers);
        case MGC_U8: return build_launch<uint8_t, LAZY>(g, imap, A, P, nz_layers);
        case MGC_I16: return build_launch<int16_t, LAZY>(g, imap, A, P, nz_layers);
        default: return build_launch<int32_t, LAZY>(g, imap, A, P, nz_layers);
    }
}

// gridDim.z is at most 65535 layers of 8 planes: a longer lattice (a batch of many 2-D images) takes several launches,
// each starting at its own z_tile0 (the kernels index partials, flags and marker planes by the global layer)
int build_launch_any(mgc_graph* g, bool lazy, int dtype, const BuildMaps& imap, const BuildArgs& A, const BoundaryParams& P, int nz_layers)
{
    constexpr int MAX_LAYERS = 65535;
    BuildArgs Al = A;
    for (int l = 0; l < nz_layers; l += MAX_LAYERS) {
        Al.z_tile0 = A.z_tile0 + l;
        const int nl = nz_layers - l < MAX_LAYERS ? nz_layers - l : MAX_LAYERS;
        const int rc = lazy ? build_launch_dtype<1>(g, dtype, imap, Al, P, nl) : build_launch_dtype<0>(g, dtype, imap, Al, P, nl);
        if (rc) return rc;
    }
    return MGC_OK;
}

// C-contiguous over the local lattice?
bool c_contiguous(const mgc_graph* g, const mgc_array* a)
{
    long long expect = (long long)dtype_size(a->dtype);
    for (int d = g->nd - 1; d >= 0; --d) {
        const int ud = d - g->shift;
        if (g->L.dim[d] > 1) {
            if (ud < 0 || (long long)a->strides[ud] != expect) return false;
        }
        expect *= g->L.dim[d];
    }
    return true;
}

bool can_fuse(const mgc_graph* g) { return g->nd == 3 && g->fuse_build; }
// lazy capacities need the per-tile worklists of one whole lattice: no z-slabs
bool can_lazy(const mgc_graph* g) { return can_fuse(g) && !g->slab && g->lazy_caps && g->cmat; }
}  // namespace

// mgc_build_voxel_graph, and mgc_build_voxel_batch with its arrays over the batch lattice (a batch handle reads its term
// constants from the table batch_constants fills, and its per-image add_tweights constants are summed after the build)
int voxel_build(mgc_graph* g, const mgc_voxel_terms* t)
{
    if (g->flow_started) FAIL(MGC_E_STATE, "the graph has been solved (its capacities hold residuals): reset() it before adding terms");
    const bool has_bits = t->fg_bits || t->bg_bits;
    if (has_bits && (t->fg || t->bg)) FAIL(MGC_E_ARG, "pass the markers either as byte arrays or bit-packed, not both");
    if (t->boundary_kind > 7) FAIL(MGC_E_ARG, "unknown boundary term");
    if (t->boundary_kind >= 0 && !t->image) FAIL(MGC_E_ARG, "boundary term without image");
    const bool fresh = g->caps_fresh && g->tr_fresh && !g->state_init;
    if (!(fresh && can_fuse(g) && t->boundary_kind >= 0)) {
        // the same terms through the one-pass-per-term entry points, in the reference's order (generate.py:159-172)
        if (has_bits) FAIL(MGC_E_ARG, "bit-packed markers need the fused build (fresh 1-D..3-D tile-solver handle with a boundary term)");
        int rc = MGC_OK;
        if (t->prob) { rc = mgc_add_regional_probability(g, t->prob, t->alpha, t->compute_dtype); if (rc) return rc; }
        if (t->boundary_kind >= 0) { rc = mgc_add_boundary(g, t->boundary_kind, t->image, t->sigma, t->spacing, t->norm); if (rc) return rc; }
        return mgc_add_markers(g, t->fg, t->bg);
    }
    if (t->prob && t->prob->dtype != MGC_F32 && t->prob->dtype != MGC_F64) FAIL(MGC_E_ARG, "probability map must be float32 or float64");
    if (t->prob && t->compute_dtype != MGC_F32 && t->compute_dtype != MGC_F64) FAIL(MGC_E_ARG, "compute dtype must be float32 or float64");
    if (t->prob && t->compute_dtype == MGC_F32 && t->prob->dtype != MGC_F32) FAIL(MGC_E_ARG, "float32 products need a float32 probability map");
    if ((t->fg && t->fg->dtype != MGC_U8) || (t->bg && t->bg->dtype != MGC_U8)) FAIL(MGC_E_ARG, "markers must be uint8 / bool");
    if (!dtype_size(t->image->dtype)) FAIL(MGC_E_ARG, "unsupported dtype");
    CK(cudaSetDevice(g->device));
    { int rc0 = check_pending(g); if (rc0) return rc0; }
    Nvtx range("mgc:build_voxel_graph");
    TermSpan span(g);

    const size_t n = (size_t)g->L.n;
    const size_t plane = (size_t)g->L.plane;
    const int Z = g->L.dim[0];
    const int nzt = (Z + BUILD_TZ - 1) / BUILD_TZ;
    const size_t es_img = dtype_size(t->image->dtype), es_prob = t->prob ? dtype_size(t->prob->dtype) : 0;
    const size_t words = (n + 31) / 32;

    // ---- chunked path: contiguous HOST arrays, upload of z-chunk c+1 overlaps the build of chunk c ----
    bool chunked = g->build_chunks > 1 && nzt >= 2 && t->image->mem == MGC_MEM_HOST && c_contiguous(g, t->image) &&
                   !(( t->boundary_kind & 3) == 0 && std::isnan(t->norm));
    if (t->prob) chunked = chunked && t->prob->mem == MGC_MEM_HOST && c_contiguous(g, t->prob);
    if (t->fg) chunked = chunked && t->fg->mem == MGC_MEM_HOST && c_contiguous(g, t->fg);
    if (t->bg) chunked = chunked && t->bg->mem == MGC_MEM_HOST && c_contiguous(g, t->bg);
    if (has_bits) chunked = chunked && t->bits_mem == MGC_MEM_HOST;

    const void *d_img = nullptr, *d_prob = nullptr, *d_fg = nullptr, *d_bg = nullptr;
    int rc = MGC_OK;
    if (!chunked) {
        rc = stage_input(g, t->image, 2, &d_img); if (rc) return rc;
        if (t->prob) { rc = stage_input(g, t->prob, 0, &d_prob); if (rc) return rc; }
        if (t->fg) { rc = stage_input(g, t->fg, 1, &d_fg); if (rc) return rc; }
        if (t->bg) { rc = stage_input(g, t->bg, 4, &d_bg); if (rc) return rc; }
        if (has_bits) {
            if (t->bits_ready_words && t->bits_mem == MGC_MEM_HOST) {
                while (*t->bits_ready_words < (int64_t)words) std::this_thread::yield();
                std::atomic_thread_fence(std::memory_order_acquire);
            }
            const uint32_t* src[2] = {t->fg_bits, t->bg_bits};
            const void** dst[2] = {&d_fg, &d_bg};
            const int slot[2] = {1, 4};
            for (int i = 0; i < 2; ++i) {
                if (!src[i]) continue;
                if (t->bits_mem == MGC_MEM_DEVICE) { *dst[i] = src[i]; continue; }
                rc = ensure_scratch(g, g->scratch[slot[i]], words * 4); if (rc) return rc;
                rc = upload(g, g->scratch[slot[i]].p, src[i], words * 4, slot[i]); if (rc) return rc;
                *dst[i] = g->scratch[slot[i]].p;
            }
        }
    } else {
        rc = ensure_scratch(g, g->scratch[2], n * es_img); if (rc) return rc;
        if (t->prob) { rc = ensure_scratch(g, g->scratch[0], n * es_prob); if (rc) return rc; }
        if (t->fg || t->fg_bits) { rc = ensure_scratch(g, g->scratch[1], has_bits ? words * 4 : n); if (rc) return rc; }
        if (t->bg || t->bg_bits) { rc = ensure_scratch(g, g->scratch[4], has_bits ? words * 4 : n); if (rc) return rc; }
        d_img = g->scratch[2].p;
        if (t->prob) d_prob = g->scratch[0].p;
        if (t->fg || t->fg_bits) d_fg = g->scratch[1].p;
        if (t->bg || t->bg_bits) d_bg = g->scratch[4].p;
        const int slots[4] = {0, 1, 2, 4};
        for (int i = 0; i < 4; ++i) if (g->slot_used[slots[i]]) CK(cudaStreamWaitEvent(g->up_stream, g->ev_slot[slots[i]], 0));
    }

    BoundaryParams P{};
    rc = boundary_params(g, t->boundary_kind, t->image->dtype, d_img, t->sigma, t->spacing, g->batch ? 0.0 : t->norm, &P);
    if (rc) return rc;
    if (g->batch) { rc = batch_constants(g, t->image->dtype, d_img, &P); if (rc) return rc; }

    BuildArgs A{};
    A.img = d_img;
    A.prob = d_prob;
    A.prob_f64 = (t->prob && t->prob->dtype == MGC_F64) ? 1 : 0;
    A.compute_f32 = (t->prob && t->compute_dtype == MGC_F32) ? 1 : 0;
    A.alpha = t->alpha;
    if (has_bits) { A.fg_bits = (const unsigned*)d_fg; A.bg_bits = (const unsigned*)d_bg; }
    else { A.fg = (const uint8_t*)d_fg; A.bg = (const uint8_t*)d_bg; }
    BuildMaps imap{};
    A.use_tma = make_image_map(g, d_img, t->image->dtype, &imap.img) ? 1 : 0;
    if (const char* e = getenv("MEDPY_GC_BUILD_TMA")) if (atoi(e) == 0) A.use_tma = 0;
    int tin_tma = A.use_tma;                 // t-link inputs through TMA as well (MEDPY_GC_BUILD_TMA=2: image only)
    if (const char* e = getenv("MEDPY_GC_BUILD_TMA")) if (atoi(e) == 2) tin_tma = 0;
    if (tin_tma) {
        if (d_prob && make_block_map(g, d_prob, t->prob->dtype, &imap.prob)) A.tma_prob = 1;
        if (!has_bits) {
            if (d_fg && make_block_map(g, d_fg, MGC_U8, &imap.fg)) A.tma_mark |= 1;
            if (d_bg && make_block_map(g, d_bg, MGC_U8, &imap.bg)) A.tma_mark |= 2;
        }
    }
    if (const char* e = getenv("MEDPY_GC_BUILD_DBG")) A.dbg = atoi(e);
    const bool lazy = can_lazy(g);
    const int mark_words = (g->L.dim[2] + 31) / 32;
    // Where the materialiser and the folds read the image and the map of a lazy build later:
    //   STAGED   -- the staging buffer of this call (host or gathered input) becomes the copy: swapped after the build;
    //   BORROWED -- the caller's contiguous device array itself (MGC_OPT_KEEP_DEVICE_INPUTS);
    //   COPIED   -- a copy the build kernel writes as it goes.
    enum { COPIED, STAGED, BORROWED };
    auto source_of = [&](const mgc_array* a, const void* d, int slot) {
        if (d == g->scratch[slot].p) return STAGED;
        return (g->keep_device_inputs && a->mem == MGC_MEM_DEVICE && d == a->data) ? BORROWED : COPIED;
    };
    const int img_src = lazy ? source_of(t->image, d_img, 2) : COPIED;
    // (MEDPY_GC_BUILD_DBG=1 builds from a constant map: only a copy holds what the build saw)
    const int prob_src = (lazy && t->prob && !(A.dbg & 1)) ? source_of(t->prob, d_prob, 0) : COPIED;
    if (lazy) {
        if (img_src == COPIED) { rc = ensure_scratch(g, g->img_copy, n * es_img); if (rc) return rc; A.img_copy = g->img_copy.p; }
        if (t->prob && prob_src == COPIED) { rc = ensure_scratch(g, g->prob_copy, n * es_prob); if (rc) return rc; A.prob_copy = g->prob_copy.p; }
        const size_t plane_bytes = (size_t)g->L.dim[0] * (size_t)g->L.dim[1] * (size_t)mark_words * 4;
        if (t->fg || t->fg_bits) { rc = ensure_scratch(g, g->mark_planes[0], plane_bytes); if (rc) return rc; A.fg_plane = (unsigned*)g->mark_planes[0].p; }
        if (t->bg || t->bg_bits) { rc = ensure_scratch(g, g->mark_planes[1], plane_bytes); if (rc) return rc; A.bg_plane = (unsigned*)g->mark_planes[1].p; }
        A.cmat = g->cmat;
        CK(cudaMemsetAsync(g->d_flags + 3, 0, sizeof(int), g->stream));      // tiles materialised
        CK(cudaMemsetAsync(g->win_ctl + WIN_NDROP, 0, sizeof(int), g->stream));   // tiles dropped unmaterialised
    }

    CK(cudaMemsetAsync(g->d_tcount, 0, 256, g->stream));
    CK(cudaMemsetAsync(g->d_flags, 0, sizeof(int), g->stream));
    CK(cudaMemsetAsync(g->d_flags + 7, 0, sizeof(int), g->stream));     // blocks refused by the lean build
    { int rcd = dirty_clear(g); if (rcd) return rcd; }
    g->pl_sel[0] = g->pl_sel[1] = 0;
    cudaEventRecord(g->ev_b[0], g->stream);
    if (!chunked) {
        A.z_tile0 = 0;
        rc = build_launch_any(g, lazy, t->image->dtype, imap, A, P, nzt);
        if (rc) return rc;
    } else {
        int nchunks = g->build_chunks < nzt ? g->build_chunks : nzt;
        const int per = (nzt + nchunks - 1) / nchunks;
        nchunks = (nzt + per - 1) / per;
        const char* h_img = (const char*)t->image->data;
        int prev_l0 = 0, prev_nl = 0;
        for (int c = 0; c < nchunks; ++c) {
            const int l0 = c * per, l1 = (l0 + per < nzt) ? l0 + per : nzt;
            const size_t z0 = (size_t)l0 * BUILD_TZ, z1 = ((size_t)l1 * BUILD_TZ < (size_t)Z) ? (size_t)l1 * BUILD_TZ : (size_t)Z;
            const size_t v0 = z0 * plane, nv = (z1 - z0) * plane;
            CK(cudaMemcpyAsync((char*)g->scratch[2].p + v0 * es_img, h_img + v0 * es_img, nv * es_img, cudaMemcpyHostToDevice, g->up_stream));
            if (c > 0) {
                // chunk c-1 needs the first image plane of chunk c (its +z neighbours) and its own prob / markers
                CK(cudaEventRecord(g->ev_chunk[c & 1], g->up_stream));
                CK(cudaStreamWaitEvent(g->stream, g->ev_chunk[c & 1], 0));
                A.z_tile0 = prev_l0;
                rc = build_launch_any(g, lazy, t->image->dtype, imap, A, P, prev_nl);
                if (rc) { cudaStreamSynchronize(g->up_stream); return rc; }     // the host arrays are borrowed: no copy may outlive the call
            }
            if (t->prob) CK(cudaMemcpyAsync((char*)g->scratch[0].p + v0 * es_prob, (const char*)t->prob->data + v0 * es_prob, nv * es_prob, cudaMemcpyHostToDevice, g->up_stream));
            if (has_bits) {
                const size_t w0 = v0 / 32, w1 = (v0 + nv + 31) / 32;
                if (t->bits_ready_words) {        // producer thread still packing: wait until this chunk's words exist
                    const int64_t need = (int64_t)(w1 < words ? w1 : words);
                    while (*t->bits_ready_words < need) std::this_thread::yield();   // packing runs at memory speed, far ahead of PCIe
                    std::atomic_thread_fence(std::memory_order_acquire);
                }
                if (t->fg_bits) CK(cudaMemcpyAsync((uint32_t*)g->scratch[1].p + w0, t->fg_bits + w0, (w1 - w0) * 4, cudaMemcpyHostToDevice, g->up_stream));
                if (t->bg_bits) CK(cudaMemcpyAsync((uint32_t*)g->scratch[4].p + w0, t->bg_bits + w0, (w1 - w0) * 4, cudaMemcpyHostToDevice, g->up_stream));
            } else {
                if (t->fg) CK(cudaMemcpyAsync((char*)g->scratch[1].p + v0, (const char*)t->fg->data + v0, nv, cudaMemcpyHostToDevice, g->up_stream));
                if (t->bg) CK(cudaMemcpyAsync((char*)g->scratch[4].p + v0, (const char*)t->bg->data + v0, nv, cudaMemcpyHostToDevice, g->up_stream));
            }
            prev_l0 = l0; prev_nl = l1 - l0;
        }
        CK(cudaEventRecord(g->ev_up, g->up_stream));
        CK(cudaStreamWaitEvent(g->stream, g->ev_up, 0));
        A.z_tile0 = prev_l0;
        rc = build_launch_any(g, lazy, t->image->dtype, imap, A, P, prev_nl);
        if (rc) { cudaStreamSynchronize(g->up_stream); return rc; }
        CK(cudaEventSynchronize(g->ev_up));       // the host arrays are only borrowed for this call
    }
    cudaEventRecord(g->ev_b[1], g->stream);
    {   // flow constant: one partial per build block, fixed order
        const unsigned nbuild = (unsigned)nzt * (unsigned)((g->L.dim[1] + BUILD_TY - 1) / BUILD_TY) * (unsigned)((g->L.dim[2] + BUILD_TX - 1) / BUILD_TX);
        sum_partials(g, g->partials, nbuild, g->d_scalars);
        g->st.kernel_launches++;
        CK(cudaGetLastError());
    }
    if (g->batch) { rc = batch_tconst(g, A); if (rc) return rc; }
    g->caps_fresh = false;
    g->tr_fresh = false;
    g->caps_lazy = lazy;
    g->lazy_built = lazy;
    g->warm_state = false;
    g->st.seed_folds = 0;
    g->st.ms_seeds = 0.0;
    g->st.ms_seeds_host = 0.0;
    g->caps_dtype = t->image->dtype;
    g->caps_P = P;
    // a staged input becomes the copy and the old copy the staging buffer; span.stop below records the slot's event after
    // the build, so the next upload into that buffer waits for whatever already queued still reads the old copy
    if (img_src == STAGED) std::swap(g->scratch[2], g->img_copy);
    if (prob_src == STAGED) std::swap(g->scratch[0], g->prob_copy);
    g->caps_img = !lazy ? nullptr : (img_src == BORROWED ? d_img : g->img_copy.p);
    const void* caps_prob = !(lazy && t->prob) ? nullptr : (prob_src == BORROWED ? d_prob : g->prob_copy.p);
    g->caps_tin = LazyTin{caps_prob, A.prob_f64, A.compute_f32, A.alpha, A.fg_plane, A.bg_plane, mark_words};
    g->has_nlinks = true;
    g->boundary_timed = true;
    g->state_init = true;
    g->solved = false;
    g->host_mask_valid = false;
    g->labels_fresh = true;
    g->sweep_mode = -1;
    g->init_timed = false;
    g->st.ms_init = 0.0;
    span.stop(0x17u);
    if (g->defer_check && g->h_bad) {
        CK(cudaMemcpyAsync(g->h_bad, g->d_flags, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
        CK(cudaEventRecord(g->ev_bad, g->stream));
        g->bad_pending = true;
        return MGC_OK;
    }
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, g->d_flags, sizeof(int), cudaMemcpyDeviceToHost, g->stream));
    CK(cudaStreamSynchronize(g->stream));
    if (bad) FAIL(MGC_E_WEIGHT, "Negative or zero weights are not allowed.");
    return MGC_OK;
}

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

int mgc_can_fuse(const mgc_graph* g) { return g && can_fuse(g) ? 1 : 0; }

int mgc_build_voxel_graph(mgc_graph* g, const mgc_voxel_terms* t)
{
    if (!g || !t) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    return voxel_build(g, t);
}

}  // extern "C"
