// gc_labels_api.cu -- host side of the C ABI for label images (include/medpy_b200_graphcut.h, section "label images";
// SURVEY.md §8 row f3).
//
// mgc_labels keeps a label image resident in HBM and reduces voxel-scale data to the region adjacency graph there
// (gc_labels.cuh); only per-region / per-region-pair results ever reach the host.  The stable radix sort that orders the
// contributions by key is cub::DeviceRadixSort (gc_sort.cuh).  The kernels of gc_labels.cuh are compiled here only;
// lab_iota() and lab_scan_blocks() launch the two the sparse unit needs as well.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/medpy_b200_graphcut.h"
#include "gc_host.hpp"
#include "gc_labels.cuh"
#include "gc_sort.cuh"

static_assert(LAB_BLOCK == 256, "grid_for() counts blocks of 256 threads");

void lab_iota(unsigned* a, long long m) { k_lab_iota<<<(unsigned)((m + LAB_BLOCK - 1) / LAB_BLOCK), LAB_BLOCK>>>(a, m); }

void lab_scan_blocks(const unsigned* cnt, long long nb, unsigned long long* out) { k_lab_scan_blocks<<<1, 1024>>>(cnt, nb, out); }

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

namespace {

thread_local std::string g_lab_create_error;

// Dense, C-ordered device copy of `a` over the handle's shape.  *out points into `a` itself when it already is a dense
// device array, otherwise into memory owned by `scope`.
template <typename E>
int lab_stage(mgc_labels* g, const mgc_array* a, DevScope& scope, const E** out)
{
    if (!a || !a->data) FAIL(MGC_E_ARG, "null array");
    const size_t es = sizeof(E);
    LabStrides st{};
    bool contiguous = true;
    long long span = (long long)es, expect = (long long)es;
    for (int d = g->G.nd - 1; d >= 0; --d) {
        long long s = (long long)a->strides[d];
        if (g->G.dim[d] > 1) {
            if (s <= 0) FAIL(MGC_E_ARG, "array strides must be positive (pass a contiguous copy)");
            if (s != expect) contiguous = false;
            span += (g->G.dim[d] - 1) * s;
        } else {
            s = 0;
        }
        st.s[d] = s;
        expect *= g->G.dim[d];
    }
    const size_t bytes = (size_t)g->G.n * es;
    if (contiguous && a->mem == MGC_MEM_DEVICE) { *out = (const E*)a->data; return MGC_OK; }
    E* dst = nullptr;
    CK(scope.alloc(&dst, (size_t)g->G.n));
    if (contiguous) {
        CK(cudaMemcpy(dst, a->data, bytes, cudaMemcpyHostToDevice));
        *out = dst;
        return MGC_OK;
    }
    const char* src = (const char*)a->data;
    if (a->mem == MGC_MEM_HOST) {
        char* raw = nullptr;
        CK(scope.alloc(&raw, (size_t)span));
        CK(cudaMemcpy(raw, a->data, (size_t)span, cudaMemcpyHostToDevice));
        src = raw;
    }
    k_lab_gather<E><<<(unsigned)((g->G.n + LAB_BLOCK - 1) / LAB_BLOCK), LAB_BLOCK>>>(g->G, src, st, dst);
    g->kernel_launches++;
    CK(cudaGetLastError());
    *out = dst;
    return MGC_OK;
}

template <typename E, int MODE>
int lab_boundary_run(mgc_labels* g, const E* grad, double directedness)
{
    DevScope dev;
    const long long items = (long long)g->G.nd * g->G.n;
    const long long nb = (items + LAB_BLOCK - 1) / LAB_BLOCK;
    if (nb >= (long long)INT32_MAX) FAIL(MGC_E_ARG, "label image too large");
    unsigned* block_count;
    unsigned long long* block_off;
    CK(dev.alloc(&block_count, (size_t)nb));
    CK(dev.alloc(&block_off, (size_t)nb + 1));
    k_lab_pair_count<<<(unsigned)nb, LAB_BLOCK>>>(g->G, g->labels, MODE == 2 ? 1 : 0, block_count);
    k_lab_scan_blocks<<<1, 1024>>>(block_count, nb, block_off);
    g->kernel_launches += 2;
    CK(cudaGetLastError());
    unsigned long long m_u = 0;
    CK(cudaMemcpy(&m_u, block_off + nb, sizeof(m_u), cudaMemcpyDeviceToHost));
    const long long m = (long long)m_u;
    g->ei.clear(); g->ej.clear(); g->ew.clear(); g->er.clear();
    if (m == 0) return MGC_OK;
    if (m >= (1ll << 32)) FAIL(MGC_E_ARG, "more than 2^32 border voxel pairs");
    unsigned long long *keys, *keys_sorted;
    unsigned *perm = nullptr, *perm_sorted = nullptr;
    double *wf = nullptr, *wr = nullptr, *wf_s = nullptr, *wr_s = nullptr;
    CK(dev.alloc(&keys, (size_t)m));
    CK(dev.alloc(&keys_sorted, (size_t)m));
    if (MODE >= 1) { CK(dev.alloc(&wf, (size_t)m)); CK(dev.alloc(&wf_s, (size_t)m)); }
    if (MODE == 2) { CK(dev.alloc(&wr, (size_t)m)); CK(dev.alloc(&wr_s, (size_t)m)); }
    k_lab_pair_emit<E, MODE><<<(unsigned)nb, LAB_BLOCK>>>(g->G, g->labels, grad, directedness < 0 ? -directedness : directedness,
                                                          directedness < 0 ? 1 : 0, block_off, keys, wf, wr);
    g->kernel_launches++;
    CK(cudaGetLastError());
    // stable sort by key: contributions of one region pair stay in the reference's order
    const unsigned mblocks = (unsigned)((m + LAB_BLOCK - 1) / LAB_BLOCK);
    const int end_bit = 32 + bits_for((unsigned long long)g->k);
    if (MODE >= 1) {
        CK(dev.alloc(&perm, (size_t)m));
        CK(dev.alloc(&perm_sorted, (size_t)m));
        k_lab_iota<<<mblocks, LAB_BLOCK>>>(perm, m);
        CK(radix_sort(dev, keys, keys_sorted, m, end_bit, perm, perm_sorted));
        k_lab_permute<<<mblocks, LAB_BLOCK>>>(wf, perm_sorted, m, wf_s);
        if (MODE == 2) k_lab_permute<<<mblocks, LAB_BLOCK>>>(wr, perm_sorted, m, wr_s);
        g->kernel_launches += 3;
    } else {
        CK(radix_sort(dev, keys, keys_sorted, m, end_bit));
    }
    CK(cudaGetLastError());
    // one output slot per run of equal keys, in key order (heads per block -> scan -> slot)
    unsigned* head_count;
    unsigned long long* head_off;
    CK(dev.alloc(&head_count, (size_t)mblocks));
    CK(dev.alloc(&head_off, (size_t)mblocks + 1));
    k_lab_seg_head_count<<<mblocks, LAB_BLOCK>>>(keys_sorted, m, head_count);
    k_lab_scan_blocks<<<1, 1024>>>(head_count, (long long)mblocks, head_off);
    unsigned long long u = 0;
    CK(cudaMemcpy(&u, head_off + mblocks, sizeof(u), cudaMemcpyDeviceToHost));
    unsigned long long* out_key;
    double *out_f, *out_r;
    CK(dev.alloc(&out_key, (size_t)u));
    CK(dev.alloc(&out_f, (size_t)u));
    CK(dev.alloc(&out_r, (size_t)u));
    k_lab_seg_reduce<<<mblocks, LAB_BLOCK>>>(keys_sorted, wf_s, wr_s, m, head_off, out_key, out_f, out_r);
    g->kernel_launches += 3;
    CK(cudaGetLastError());
    std::vector<unsigned long long> hk((size_t)u);
    g->ew.resize((size_t)u); g->er.resize((size_t)u);
    CK(cudaMemcpy(hk.data(), out_key, (size_t)u * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g->ew.data(), out_f, (size_t)u * sizeof(double), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g->er.data(), out_r, (size_t)u * sizeof(double), cudaMemcpyDeviceToHost));
    g->ei.resize((size_t)u); g->ej.resize((size_t)u);
    for (size_t t = 0; t < (size_t)u; ++t) {
        g->ei[t] = (int32_t)(hk[t] >> 32);
        g->ej[t] = (int32_t)(hk[t] & 0xffffffffull);
    }
    return MGC_OK;
}

template <typename E>
int lab_boundary_dispatch(mgc_labels* g, int kind, const mgc_array* values, double directedness)
{
    DevScope scope;
    const E* grad = nullptr;
    int rc = lab_stage<E>(g, values, scope, &grad);
    if (rc) return rc;
    if (kind == MGC_LABELS_STAWIASKI) return lab_boundary_run<E, 1>(g, grad, 0.0);
    return lab_boundary_run<E, 2>(g, grad, directedness);
}

// V = element type the sums are formed in (double: bincount; float/double: numpy.sum of a float array)
template <typename E, typename V, bool PAIRWISE>
int lab_region_sums_run(mgc_labels* g, const mgc_array* values, double* sums, int64_t* counts)
{
    DevScope dev;
    const E* vals_in = nullptr;
    int rc = lab_stage<E>(g, values, dev, &vals_in);
    if (rc) return rc;
    const long long n = g->G.n;
    if (n >= (long long)INT32_MAX) FAIL(MGC_E_ARG, "label image too large");
    unsigned *keys, *keys_sorted;
    V *vals, *vals_sorted;
    double* d_sums;
    long long* d_counts;
    CK(dev.alloc(&keys, (size_t)n));
    CK(dev.alloc(&keys_sorted, (size_t)n));
    CK(dev.alloc(&vals, (size_t)n));
    CK(dev.alloc(&vals_sorted, (size_t)n));
    CK(dev.alloc(&d_sums, (size_t)g->k));
    CK(dev.alloc(&d_counts, (size_t)g->k));
    const unsigned blocks = (unsigned)((n + LAB_BLOCK - 1) / LAB_BLOCK);
    k_lab_region_items<E, V><<<blocks, LAB_BLOCK>>>(g->labels, vals_in, n, keys, vals);
    CK(radix_sort(dev, keys, keys_sorted, n, bits_for((unsigned long long)g->k), vals, vals_sorted));
    if (PAIRWISE) k_lab_region_reduce_pairwise<V><<<blocks, LAB_BLOCK>>>(keys_sorted, vals_sorted, n, d_sums, d_counts);
    else          k_lab_region_reduce<<<blocks, LAB_BLOCK>>>(keys_sorted, (const double*)vals_sorted, n, d_sums, d_counts);
    g->kernel_launches += 2;
    CK(cudaGetLastError());
    std::vector<long long> hc((size_t)g->k);
    CK(cudaMemcpy(sums, d_sums, (size_t)g->k * sizeof(double), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hc.data(), d_counts, (size_t)g->k * sizeof(long long), cudaMemcpyDeviceToHost));
    if (counts) for (int64_t r = 0; r < g->k; ++r) counts[r] = (int64_t)hc[(size_t)r];
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
    mgc_labels* g = new mgc_labels();
    g->device = device;
    g->G.nd = ndim;
    long long n = 1;
    for (int d = 0; d < 4; ++d) { g->G.dim[d] = 1; g->G.stride[d] = 1; }
    for (int d = 0; d < ndim; ++d) {
        if (shape[d] < 1) { g_lab_create_error = "empty label image"; delete g; return MGC_E_LABELS; }
        g->G.dim[d] = shape[d];
        g->shape[d] = shape[d];
        n *= shape[d];
    }
    if (n >= (long long)INT32_MAX) { g_lab_create_error = "label image too large (2^31 voxels)"; delete g; return MGC_E_ARG; }
    g->G.n = n;
    long long acc = 1;
    for (int d = ndim - 1; d >= 0; --d) { g->G.stride[d] = acc; acc *= g->G.dim[d]; }
    auto fail = [&](int code) { g_lab_create_error = g->err; mgc_labels_destroy(g); return code; };
    if (cudaSetDevice(device) != cudaSuccess) { g->err = "cudaSetDevice failed"; return fail(MGC_E_CUDA); }
    {
        DevScope scope;
        const int* p = nullptr;
        int rc = lab_stage<int>(g, labels, scope, &p);
        if (rc) return fail(rc);
        if (!scope.ptrs.empty()) {
            // the dense copy is the last block the staging allocated: keep it, release the rest with the scope
            g->labels = (int*)p;
            g->owns_labels = true;
            scope.keep(p);
        } else {
            g->labels = (int*)p;        // dense device array of the caller: read in place
        }
        // __check_label_image: min == 1 and every id up to max present
        int* mm = nullptr;
        unsigned long long* cnt = nullptr;
        if (scope.alloc(&mm, 2) != cudaSuccess || scope.alloc(&cnt, 1) != cudaSuccess) { g->err = "device allocation failed"; return fail(MGC_E_NOMEM); }
        const int init[2] = {INT32_MAX, INT32_MIN};
        cudaMemcpy(mm, init, sizeof(init), cudaMemcpyHostToDevice);
        k_lab_minmax<<<grid_for(n), LAB_BLOCK>>>(g->labels, n, mm);
        int got[2] = {0, 0};
        if (cudaMemcpy(got, mm, sizeof(got), cudaMemcpyDeviceToHost) != cudaSuccess) { g->err = std::string("label scan failed: ") + cudaGetErrorString(cudaGetLastError()); return fail(MGC_E_CUDA); }
        const char* msg = "The supplied label image does either not contain any regions or they are not labeled consecutively starting from 1.";
        if (got[0] != 1 || got[1] < 1) { g->err = msg; return fail(MGC_E_LABELS); }
        uint8_t* present = nullptr;
        if (scope.alloc(&present, (size_t)got[1]) != cudaSuccess) { g->err = "device allocation failed"; return fail(MGC_E_NOMEM); }
        cudaMemset(present, 0, (size_t)got[1]);
        cudaMemset(cnt, 0, sizeof(unsigned long long));
        k_lab_presence<<<grid_for(n), LAB_BLOCK>>>(g->labels, n, present);
        k_lab_count_u8<<<grid_for(got[1]), LAB_BLOCK>>>(present, got[1], cnt);
        unsigned long long c = 0;
        if (cudaMemcpy(&c, cnt, sizeof(c), cudaMemcpyDeviceToHost) != cudaSuccess) { g->err = std::string("label scan failed: ") + cudaGetErrorString(cudaGetLastError()); return fail(MGC_E_CUDA); }
        g->kernel_launches += 3;
        if ((long long)c != (long long)got[1]) { g->err = msg; return fail(MGC_E_LABELS); }
        g->k = got[1];
    }
    *out = g;
    return MGC_OK;
}

void mgc_labels_destroy(mgc_labels* g)
{
    if (!g) return;
    if (g->owns_labels && g->labels) { cudaSetDevice(g->device); cudaFree(g->labels); }
    delete g;
}

const char* mgc_labels_last_error(const mgc_labels* g) { return g ? g->err.c_str() : g_lab_create_error.c_str(); }

int mgc_labels_region_count(const mgc_labels* g, int64_t* k) { if (!g || !k) return MGC_E_ARG; *k = g->k; return MGC_OK; }

int mgc_labels_boundary(mgc_labels* g, int32_t kind, const mgc_array* values, double directedness, int64_t* n_edges)
{
    if (!g) return MGC_E_ARG;
    CK(cudaSetDevice(g->device));
    int rc;
    if (kind == MGC_LABELS_ADJACENCY) {
        rc = lab_boundary_run<float, 0>(g, nullptr, 0.0);
    } else if (kind == MGC_LABELS_STAWIASKI || kind == MGC_LABELS_STAWIASKI_DIRECTED) {
        if (!values) FAIL(MGC_E_ARG, "the boundary term needs the gradient image");
        switch (values->dtype) {
            case MGC_F32: rc = lab_boundary_dispatch<float>(g, kind, values, directedness); break;
            case MGC_F64: rc = lab_boundary_dispatch<double>(g, kind, values, directedness); break;
            case MGC_U8: rc = lab_boundary_dispatch<uint8_t>(g, kind, values, directedness); break;
            case MGC_I16: rc = lab_boundary_dispatch<int16_t>(g, kind, values, directedness); break;
            case MGC_I32: rc = lab_boundary_dispatch<int32_t>(g, kind, values, directedness); break;
            default: FAIL(MGC_E_ARG, "unsupported dtype");
        }
    } else {
        FAIL(MGC_E_ARG, "unknown label boundary term");
    }
    if (rc) return rc;
    if (n_edges) *n_edges = (int64_t)g->ei.size();
    return MGC_OK;
}

int mgc_labels_fetch_edges(const mgc_labels* g, int32_t* i, int32_t* j, double* w_ij, double* w_ji)
{
    if (!g) return MGC_E_ARG;
    const size_t u = g->ei.size();
    if (u && (!i || !j)) return MGC_E_ARG;
    if (u) {
        std::memcpy(i, g->ei.data(), u * sizeof(int32_t));
        std::memcpy(j, g->ej.data(), u * sizeof(int32_t));
        if (w_ij) std::memcpy(w_ij, g->ew.data(), u * sizeof(double));
        if (w_ji) std::memcpy(w_ji, g->er.data(), u * sizeof(double));
    }
    return MGC_OK;
}

int mgc_labels_region_sums(mgc_labels* g, const mgc_array* values, int32_t mode, double* sums, int64_t* counts)
{
    if (!g || !values || !sums) return MGC_E_ARG;
    CK(cudaSetDevice(g->device));
    const bool pw = (mode == MGC_SUM_PAIRWISE);
    switch (values->dtype) {
        case MGC_F32: return pw ? lab_region_sums_run<float, float, true>(g, values, sums, counts)
                                : lab_region_sums_run<float, double, false>(g, values, sums, counts);
        case MGC_F64: return pw ? lab_region_sums_run<double, double, true>(g, values, sums, counts)
                                : lab_region_sums_run<double, double, false>(g, values, sums, counts);
        case MGC_U8: return lab_region_sums_run<uint8_t, double, false>(g, values, sums, counts);
        case MGC_I16: return lab_region_sums_run<int16_t, double, false>(g, values, sums, counts);
        case MGC_I32: return lab_region_sums_run<int32_t, double, false>(g, values, sums, counts);
        default: FAIL(MGC_E_ARG, "unsupported dtype");
    }
}

int mgc_labels_region_flags(mgc_labels* g, const mgc_array* markers, uint8_t* flags)
{
    if (!g || !markers || !flags) return MGC_E_ARG;
    if (markers->dtype != MGC_U8) FAIL(MGC_E_ARG, "markers must be uint8 / bool");
    CK(cudaSetDevice(g->device));
    DevScope dev;
    const uint8_t* m = nullptr;
    int rc = lab_stage<uint8_t>(g, markers, dev, &m);
    if (rc) return rc;
    uint8_t* d_flags;
    CK(dev.alloc(&d_flags, (size_t)g->k));
    CK(cudaMemset(d_flags, 0, (size_t)g->k));
    k_lab_region_flags<<<grid_for(g->G.n), LAB_BLOCK>>>(g->labels, m, g->G.n, d_flags);
    g->kernel_launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpy(flags, d_flags, (size_t)g->k, cudaMemcpyDeviceToHost));
    return MGC_OK;
}

int mgc_labels_apply(mgc_labels* g, const uint8_t* per_region, uint8_t* out, int32_t out_mem)
{
    if (!g || !per_region || !out) return MGC_E_ARG;
    CK(cudaSetDevice(g->device));
    DevScope dev;
    uint8_t *d_reg, *d_out = out;
    CK(dev.alloc(&d_reg, (size_t)g->k));
    CK(cudaMemcpy(d_reg, per_region, (size_t)g->k, cudaMemcpyHostToDevice));
    if (out_mem == MGC_MEM_HOST) CK(dev.alloc(&d_out, (size_t)g->G.n));
    k_lab_apply<<<grid_for(g->G.n), LAB_BLOCK>>>(g->labels, d_reg, g->G.n, d_out);
    g->kernel_launches++;
    CK(cudaGetLastError());
    if (out_mem == MGC_MEM_HOST) CK(cudaMemcpy(out, d_out, (size_t)g->G.n, cudaMemcpyDeviceToHost));
    else CK(cudaDeviceSynchronize());
    return MGC_OK;
}

}  // extern "C"
