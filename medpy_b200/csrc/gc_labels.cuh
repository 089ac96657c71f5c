// gc_labels.cuh -- region adjacency graph of a label image, built on the device (SURVEY.md §8 row f3).
//
// Replaces the voxel-pair Python loops of medpy/graphcut/energy_label.py: boundary_stawiaski (:123-214, one
// set_nweight call per border voxel pair), boundary_stawiaski_directed (:217-342), __compute_edges_nd (:411-441,
// used by boundary_difference_of_means :33-120), scipy.ndimage.mean over the regions (:92) and the per-region sums
// of regional_atlas (:345-396).
//
// Everything is a keyed reduction over voxels or voxel pairs.  The reference accumulates with `r_cap += w`
// (graph.h:472-476) in a fixed order -- axis by axis, C order inside an axis -- and float64 addition is not
// associative, so the reduction here keeps that order: contributions are written in reference order (order
// preserving compaction: block counts -> exclusive scan -> in-block scan), stably sorted by key, and every key's run
// is then summed front to back by one thread.  The sums are therefore bit-identical to the reference's and
// independent of the launch geometry.
#pragma once
#include <cfloat>
#include <cstdint>

#include <cuda_runtime.h>

#include "gc_pairwise.cuh"

#define LAB_BLOCK 256

struct LabGeom {
    int nd;                 // canonical axes (1..4)
    long long n;            // voxels
    long long dim[4];
    long long stride[4];    // element strides, C order
};

// strided -> dense copy of an input array (any of the ABI's element types), logical C order
struct LabStrides { long long s[4]; };   // BYTE strides per canonical axis

template <typename E>
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_gather(LabGeom G, const char* __restrict__ src, LabStrides st, E* __restrict__ dst)
{
    const long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (p >= G.n) return;
    long long off = 0, r = p;
    for (int d = 0; d < G.nd; ++d) {
        const long long c = r / G.stride[d];
        r -= c * G.stride[d];
        off += c * st.s[d];
    }
    dst[p] = *reinterpret_cast<const E*>(src + off);
}

// ---------------------------------------------------------------------------------------------------------------
// __check_label_image (energy_label.py:444-456): ids must be exactly 1..K
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_minmax(const int* __restrict__ labels, long long n, int* __restrict__ mm)
{
    int lo = INT32_MAX, hi = INT32_MIN;
    for (long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x; p < n; p += (long long)gridDim.x * LAB_BLOCK) {
        const int l = labels[p];
        lo = l < lo ? l : lo;
        hi = l > hi ? l : hi;
    }
    for (int o = 16; o > 0; o >>= 1) {
        const int a = __shfl_down_sync(0xffffffffu, lo, o), b = __shfl_down_sync(0xffffffffu, hi, o);
        lo = a < lo ? a : lo;
        hi = b > hi ? b : hi;
    }
    if ((threadIdx.x & 31) == 0) { atomicMin(&mm[0], lo); atomicMax(&mm[1], hi); }
}

// present[l-1] = 1 for every label that occurs (labels already known to lie in 1..K)
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_presence(const int* __restrict__ labels, long long n, uint8_t* __restrict__ present)
{
    for (long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x; p < n; p += (long long)gridDim.x * LAB_BLOCK)
        present[labels[p] - 1] = 1;
}

__global__ void __launch_bounds__(LAB_BLOCK) k_lab_count_u8(const uint8_t* __restrict__ a, long long n, unsigned long long* __restrict__ count)
{
    unsigned long long c = 0;
    for (long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x; p < n; p += (long long)gridDim.x * LAB_BLOCK) c += a[p] ? 1u : 0u;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

// ---------------------------------------------------------------------------------------------------------------
// border voxel pairs, in the reference's order
// ---------------------------------------------------------------------------------------------------------------
// Item idx in [0, nd*n): axis d = idx / n (axis-major, like `for dim in range(ndim)`), voxel p = idx % n (C order
// inside the axis, like the sliced arrays).  The item is a border pair when p has a successor q = p + stride_d along
// d and the two labels differ.  `dup_first`: numpy.vectorize evaluates its function one extra time on the first
// element of its inputs to find the output type (no otypes given, energy_label.py:325-328), so the directed term
// adds the first pair of every axis TWICE when it is a border pair; the copy directly precedes the pair itself.
__device__ __forceinline__ unsigned lab_pair_items(const LabGeom& G, const int* __restrict__ labels, long long idx, int dup_first,
                                                   long long* p_out, long long* q_out)
{
    if (idx >= (long long)G.nd * G.n) return 0u;
    const int d = (int)(idx / G.n);
    const long long p = idx - (long long)d * G.n;
    const long long c = (p / G.stride[d]) % G.dim[d];
    if (c >= G.dim[d] - 1) return 0u;
    const long long q = p + G.stride[d];
    if (labels[p] == labels[q]) return 0u;
    *p_out = p;
    *q_out = q;
    return (dup_first && p == 0) ? 2u : 1u;
}

// exclusive prefix of `c` over the 256 threads of the block; *total = block sum
__device__ __forceinline__ unsigned lab_block_scan(unsigned c, unsigned* total)
{
    __shared__ unsigned wsum[LAB_BLOCK / 32];
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (unsigned)o) incl += t;
    }
    if (lane == 31u) wsum[warp] = incl;
    __syncthreads();
    unsigned base = 0, all = 0;
#pragma unroll
    for (unsigned w = 0; w < LAB_BLOCK / 32; ++w) {
        const unsigned s = wsum[w];
        if (w < warp) base += s;
        all += s;
    }
    *total = all;
    return base + incl - c;
}

__global__ void __launch_bounds__(LAB_BLOCK) k_lab_pair_count(LabGeom G, const int* __restrict__ labels, int dup_first,
                                                               unsigned* __restrict__ block_count)
{
    const long long idx = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    long long p, q;
    const unsigned c = lab_pair_items(G, labels, idx, dup_first, &p, &q);
    unsigned total;
    lab_block_scan(c, &total);
    if (threadIdx.x == 0) block_count[blockIdx.x] = total;
}

// exclusive scan of the block counts (one block, each thread owns a contiguous chunk); out[nb] = grand total
__global__ void __launch_bounds__(1024) k_lab_scan_blocks(const unsigned* __restrict__ cnt, long long nb, unsigned long long* __restrict__ out)
{
    __shared__ unsigned long long part[1024];
    const int tid = threadIdx.x;
    const long long chunk = (nb + 1023) / 1024;
    const long long b0 = (long long)tid * chunk;
    const long long b1 = b0 + chunk < nb ? b0 + chunk : nb;
    unsigned long long s = 0;
    for (long long b = b0; b < b1; ++b) s += cnt[b];
    part[tid] = s;
    __syncthreads();
    if (tid == 0) {
        unsigned long long acc = 0;
        for (int t = 0; t < 1024; ++t) { const unsigned long long v = part[t]; part[t] = acc; acc += v; }
        out[nb] = acc;
    }
    __syncthreads();
    unsigned long long acc = part[tid];
    for (long long b = b0; b < b1; ++b) { out[b] = acc; acc += cnt[b]; }
}

// g(max(|a|,|b|)) = (1/(1+x))^2 floored at DBL_MIN (energy_label.py:206-211,297-301), in the two arithmetics the
// reference ends up using (pinned by tests/golden/golden_labels_v1.npz):
//  * "native": numpy scalars of the gradient's dtype under numpy-2 promotion -- `1.0 + val` and `1.0 / (...)` stay
//    float32 for a float32 gradient, every other dtype goes to float64; numpy.abs wraps at the integer minimum.
//    Used by boundary_stawiaski and by the probing call numpy.vectorize makes on element 0.
//  * "pyfloat": the ufunc loop of numpy.vectorize runs over dtype=object copies, i.e. Python floats / ints: float64
//    arithmetic, abs() without wrap-around.  Used by boundary_stawiaski_directed.
// math.pow(r, 2) is taken as the correctly rounded r*r: exact for a float32 r; for a float64 r libm's pow is within
// one ulp of it (tests allow that ulp on float64 / integer gradients and demand equality on float32 ones).
template <typename E> struct LabAbs;
template <> struct LabAbs<float>   { __device__ static float  f(float x)   { return fabsf(x); } };
template <> struct LabAbs<double>  { __device__ static double f(double x)  { return fabs(x); } };
template <> struct LabAbs<uint8_t> { __device__ static uint8_t f(uint8_t x) { return x; } };
template <> struct LabAbs<int16_t> { __device__ static int16_t f(int16_t x) { return (int16_t)(x < 0 ? -x : x); } };
template <> struct LabAbs<int32_t> { __device__ static int32_t f(int32_t x) { return x < 0 ? (int32_t)(0u - (unsigned)x) : x; } };

template <typename E> struct LabIsF32 { static const bool v = false; };
template <> struct LabIsF32<float> { static const bool v = true; };

__device__ __forceinline__ double lab_floor_min(double w) { return (DBL_MIN > w) ? DBL_MIN : w; }   // max(w, float_info.min); NaN stays

// The two maxima differ only on NaN: boundary_stawiaski takes numpy.maximum (NaN if either operand is NaN), the
// directed term Python's max(a, b) (b only when b > a: a NaN second operand is dropped).
template <typename E> __device__ __forceinline__ E lab_max_numpy(E a, E b) { return (a != a) ? a : ((b != b || b > a) ? b : a); }
template <typename E> __device__ __forceinline__ E lab_max_python(E a, E b) { return b > a ? b : a; }

// NUMPY_MAX: the maximum of the two magnitudes as boundary_stawiaski takes it, otherwise as the directed term's probe
template <typename E, bool NUMPY_MAX>
__device__ __forceinline__ double lab_weight_native(E a, E b)
{
    const E va = LabAbs<E>::f(a), vb = LabAbs<E>::f(b);
    const E val = NUMPY_MAX ? lab_max_numpy<E>(va, vb) : lab_max_python<E>(va, vb);
    if (LabIsF32<E>::v) {
        const float s = __fadd_rn(1.0f, (float)val);
        const float r = __fdiv_rn(1.0f, s);
        return lab_floor_min(__dmul_rn((double)r, (double)r));
    }
    const double s = __dadd_rn(1.0, (double)val);
    const double r = __ddiv_rn(1.0, s);
    return lab_floor_min(__dmul_rn(r, r));
}

template <typename E>
__device__ __forceinline__ double lab_weight_pyfloat(E a, E b)
{
    const double val = lab_max_python<double>(fabs((double)a), fabs((double)b));
    const double r = __ddiv_rn(1.0, __dadd_rn(1.0, val));
    return lab_floor_min(__dmul_rn(r, r));
}

// The c records of border pair (p, q) from slot block_off[blockIdx.x] + ex on.  MODE 0: adjacency only (weights unused), 1: boundary_stawiaski,
// 2: boundary_stawiaski_directed.  key = (lo << 32) | hi with lo < hi the 0-based node ids; wf accumulates cap(lo -> hi),
// wr cap(hi -> lo)
template <typename E, int MODE>
__device__ __forceinline__ void lab_pair_write(const int* __restrict__ labels, const E* __restrict__ grad, double beta,
                                               int dark_to_light, long long p, long long q, unsigned c,
                                               const unsigned long long* __restrict__ block_off, unsigned ex,
                                               unsigned long long* __restrict__ keys,
                                               double* __restrict__ wf, double* __restrict__ wr)
{
    const int k1 = labels[p] - 1, k2 = labels[q] - 1;            // set_nweight(key1 - 1, key2 - 1, there, back)
    const bool fwd = k1 < k2;
    const unsigned long long lo = (unsigned long long)(fwd ? k1 : k2), hi = (unsigned long long)(fwd ? k2 : k1);
    const unsigned long long pos = block_off[blockIdx.x] + ex;
    for (unsigned r = 0; r < c; ++r) {
        keys[pos + r] = (lo << 32) | hi;
        if (MODE == 1) {
            wf[pos + r] = lab_weight_native<E, true>(grad[p], grad[q]);
        } else if (MODE == 2) {
            const E v1 = grad[p], v2 = grad[q];
            const bool probe = (c == 2u && r == 0u);             // the extra call numpy.vectorize makes on element 0
            const double w = probe ? lab_weight_native<E, false>(v1, v2) : lab_weight_pyfloat<E>(v1, v2);
            const double wb = __dadd_rn(w, beta);
            const double capped = (wb < 1.0) ? wb : 1.0;         // min(1, weight + beta)
            const bool first_gets_beta = dark_to_light ? !(v1 > v2) : (v1 > v2);
            const double there = first_gets_beta ? capped : w;
            const double back = first_gets_beta ? w : capped;
            wf[pos + r] = fwd ? there : back;
            wr[pos + r] = fwd ? back : there;
        }
    }
}

template <typename E, int MODE>
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_pair_emit(LabGeom G, const int* __restrict__ labels, const E* __restrict__ grad,
                                                              double beta, int dark_to_light,
                                                              const unsigned long long* __restrict__ block_off,
                                                              unsigned long long* __restrict__ keys, double* __restrict__ wf,
                                                              double* __restrict__ wr)
{
    const long long idx = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    long long p = 0, q = 0;
    const unsigned c = lab_pair_items(G, labels, idx, MODE == 2, &p, &q);
    unsigned total;
    const unsigned ex = lab_block_scan(c, &total);
    if (!c) return;
    lab_pair_write<E, MODE>(labels, grad, beta, dark_to_light, p, q, c, block_off, ex, keys, wf, wr);
}

// ---------------------------------------------------------------------------------------------------------------
// a batch of label images (mgc_labels_create_batch)
// ---------------------------------------------------------------------------------------------------------------
// The images' voxels are concatenated image after image, each image in its own C order, and the staged labels hold
// label + node_off[b] (global node id + 1).  The kernels above that only read labels -- region items, flags, apply --
// therefore run unchanged on the concatenation.  The border-pair item space is image-major, then axis-major, then C
// order inside the image (image b owns items [nd * vox_off[b], nd * vox_off[b+1])); a pair never crosses images.
struct LabBatch {
    int B;                          // images
    int nd;                         // axes of every image (1..4)
    const long long* vox_off;       // [B+1] exclusive prefix of the images' voxel counts
    const int* dim;                 // [4*B] extents per image, padded with 1
};

// The images that units [blockIdx.x * LAB_BLOCK, +LAB_BLOCK) of a block touch (`per` units per voxel: 1 for voxels, nd
// for border-pair items), staged in shared memory: a block of 256 units touches at most 256 images, and every unit then
// finds its image by a binary search here instead of in global memory.
struct LabWindow {
    int b0, count;                  // images b0 .. b0 + count - 1
    long long vox[LAB_BLOCK + 1];   // their vox_off entries (count + 1)
    int dim[LAB_BLOCK][4];
};

// largest i in [0, count) with off[i] <= x (off ascending, off[0] <= x)
__device__ __forceinline__ int lab_batch_find(const long long* off, int count, long long x)
{
    int lo = 0, hi = count;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

// every thread of the block calls it; units in [0, total)
__device__ __forceinline__ void lab_batch_window(const LabBatch& L, int per, long long total, LabWindow& w)
{
    if (threadIdx.x == 0) {
        const long long s = (long long)blockIdx.x * LAB_BLOCK;
        const long long e = (s + LAB_BLOCK < total ? s + LAB_BLOCK : total) - 1;
        const int b0 = lab_batch_find(L.vox_off, L.B, s / per);
        w.b0 = b0;
        w.count = lab_batch_find(L.vox_off, L.B, e / per) - b0 + 1;
    }
    __syncthreads();
    for (int i = threadIdx.x; i <= w.count; i += LAB_BLOCK) w.vox[i] = L.vox_off[w.b0 + i];
    for (int i = threadIdx.x; i < w.count; i += LAB_BLOCK)
        for (int d = 0; d < 4; ++d) w.dim[i][d] = L.dim[4 * (w.b0 + i) + d];
    __syncthreads();
}

// lab_pair_items for item idx of the batch: the same rule inside the item's image, `dup_first` on each image's first
// voxel; p and q come back as positions in the concatenation
__device__ __forceinline__ unsigned lab_batch_pair_items(const LabBatch& L, const LabWindow& w, const int* __restrict__ labels,
                                                         long long idx, long long total, int dup_first, long long* p_out,
                                                         long long* q_out)
{
    if (idx >= total) return 0u;
    const int i = lab_batch_find(w.vox, w.count, idx / L.nd);
    const long long v0 = w.vox[i], n = w.vox[i + 1] - v0;
    const long long li = idx - (long long)L.nd * v0;
    const int d = (int)(li / n);
    const long long p = li - (long long)d * n;
    long long stride = 1;
    for (int a = L.nd - 1; a > d; --a) stride *= w.dim[i][a];
    const long long dd = w.dim[i][d];
    if ((p / stride) % dd >= dd - 1) return 0u;
    const long long q = p + stride;
    if (labels[v0 + p] == labels[v0 + q]) return 0u;
    *p_out = v0 + p;
    *q_out = v0 + q;
    return (dup_first && p == 0) ? 2u : 1u;
}

__global__ void __launch_bounds__(LAB_BLOCK) k_lab_batch_pair_count(LabBatch L, long long total, const int* __restrict__ labels,
                                                                     int dup_first, unsigned* __restrict__ block_count)
{
    __shared__ LabWindow w;
    lab_batch_window(L, L.nd, total, w);
    const long long idx = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    long long p, q;
    const unsigned c = lab_batch_pair_items(L, w, labels, idx, total, dup_first, &p, &q);
    unsigned sum;
    lab_block_scan(c, &sum);
    if (threadIdx.x == 0) block_count[blockIdx.x] = sum;
}

// k_lab_pair_emit over the batch: keys are (global lo << 32) | global hi, so every key's records come from one image,
// in that image's order
template <typename E, int MODE>
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_batch_pair_emit(LabBatch L, long long total, const int* __restrict__ labels,
                                                                    const E* __restrict__ grad, double beta, int dark_to_light,
                                                                    const unsigned long long* __restrict__ block_off,
                                                                    unsigned long long* __restrict__ keys,
                                                                    double* __restrict__ wf, double* __restrict__ wr)
{
    __shared__ LabWindow w;
    lab_batch_window(L, L.nd, total, w);
    const long long idx = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    long long p = 0, q = 0;
    const unsigned c = lab_batch_pair_items(L, w, labels, idx, total, MODE == 2, &p, &q);
    unsigned sum;
    const unsigned ex = lab_block_scan(c, &sum);
    if (!c) return;
    lab_pair_write<E, MODE>(labels, grad, beta, dark_to_light, p, q, c, block_off, ex, keys, wf, wr);
}

// __check_label_image per image, first pass: min and max label of every image (mm[2b], mm[2b+1]); one block reduces
// its share of an image in shared memory before one atomic per image
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_batch_minmax(LabBatch L, const int* __restrict__ labels, long long n,
                                                                int* __restrict__ mm)
{
    __shared__ LabWindow w;
    __shared__ int lo[LAB_BLOCK], hi[LAB_BLOCK];
    lab_batch_window(L, 1, n, w);
    for (int i = threadIdx.x; i < w.count; i += LAB_BLOCK) { lo[i] = INT32_MAX; hi[i] = INT32_MIN; }
    __syncthreads();
    const long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (p < n) {
        const int i = lab_batch_find(w.vox, w.count, p), l = labels[p];
        atomicMin(&lo[i], l);
        atomicMax(&hi[i], l);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < w.count; i += LAB_BLOCK) {
        atomicMin(&mm[2 * (w.b0 + i)], lo[i]);
        atomicMax(&mm[2 * (w.b0 + i) + 1], hi[i]);
    }
}

// second pass, once every image holds labels in 1..K_b: labels[p] += node_off[b] and present[global id] = 1
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_batch_offset(LabBatch L, int* __restrict__ labels, long long n,
                                                                const long long* __restrict__ node_off,
                                                                uint8_t* __restrict__ present)
{
    __shared__ LabWindow w;
    lab_batch_window(L, 1, n, w);
    const long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (p >= n) return;
    const int g = labels[p] + (int)node_off[w.b0 + lab_batch_find(w.vox, w.count, p)];
    labels[p] = g;
    present[g - 1] = 1;
}

__global__ void __launch_bounds__(LAB_BLOCK) k_lab_iota(unsigned* __restrict__ a, long long m)
{
    const long long i = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (i < m) a[i] = (unsigned)i;
}

__global__ void __launch_bounds__(LAB_BLOCK) k_lab_permute(const double* __restrict__ src, const unsigned* __restrict__ perm, long long m,
                                                           double* __restrict__ dst)
{
    const long long i = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (i < m) dst[i] = src[perm[i]];
}

// runs of equal keys in the sorted key array: heads per block (-> exclusive scan -> output slot of every run, so the
// region pairs come out ordered by key without any further sort)
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_seg_head_count(const unsigned long long* __restrict__ keys, long long m,
                                                                  unsigned* __restrict__ block_count)
{
    const long long i = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    const unsigned head = (i < m && (i == 0 || keys[i - 1] != keys[i])) ? 1u : 0u;
    unsigned total;
    lab_block_scan(head, &total);
    if (threadIdx.x == 0) block_count[blockIdx.x] = total;
}

// one thread per run of equal keys: front-to-back float64 sum (the order `r_cap += w` sees in the reference)
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_seg_reduce(const unsigned long long* __restrict__ keys, const double* __restrict__ wf,
                                                              const double* __restrict__ wr, long long m,
                                                              const unsigned long long* __restrict__ block_off,
                                                              unsigned long long* __restrict__ out_key, double* __restrict__ out_f,
                                                              double* __restrict__ out_r)
{
    const long long i = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    const unsigned head = (i < m && (i == 0 || keys[i - 1] != keys[i])) ? 1u : 0u;
    unsigned total;
    const unsigned ex = lab_block_scan(head, &total);
    if (!head) return;
    const unsigned long long key = keys[i];
    double a = 0.0, b = 0.0;
    for (long long j = i; j < m && keys[j] == key; ++j) {
        if (wf) a = __dadd_rn(a, wf[j]);
        if (wr) b = __dadd_rn(b, wr[j]);
    }
    const unsigned long long pos = block_off[blockIdx.x] + ex;
    out_key[pos] = key;
    out_f[pos] = a;
    out_r[pos] = wr ? b : a;
}

// ---------------------------------------------------------------------------------------------------------------
// per-region sums (numpy.bincount(labels.ravel(), weights=image.ravel()) inside scipy.ndimage.mean; regional_atlas)
// ---------------------------------------------------------------------------------------------------------------
template <typename E, typename V>
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_region_items(const int* __restrict__ labels, const E* __restrict__ values, long long n,
                                                                unsigned* __restrict__ keys, V* __restrict__ vals)
{
    const long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (p >= n) return;
    keys[p] = (unsigned)(labels[p] - 1);
    vals[p] = (V)values[p];
}

// numpy.bincount(labels, weights): float64, front to back
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_region_reduce(const unsigned* __restrict__ keys, const double* __restrict__ vals, long long n,
                                                                 double* __restrict__ sums, long long* __restrict__ counts)
{
    const long long i = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (i >= n) return;
    const unsigned key = keys[i];
    if (i > 0 && keys[i - 1] == key) return;
    double a = 0.0;
    long long j = i;
    for (; j < n && keys[j] == key; ++j) a = __dadd_rn(a, vals[j]);
    sums[key] = a;
    counts[key] = j - i;
}

template <typename V>
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_region_reduce_pairwise(const unsigned* __restrict__ keys, const V* __restrict__ vals, long long n,
                                                                          double* __restrict__ sums, long long* __restrict__ counts)
{
    const long long i = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x;
    if (i >= n) return;
    const unsigned key = keys[i];
    if (i > 0 && keys[i - 1] == key) return;
    long long j = i;
    while (j < n && keys[j] == key) ++j;
    sums[key] = (double)lab_pairwise_sum<V>(vals + i, j - i);
    counts[key] = j - i;
}

// flags[l-1] = 1 for every region with a marked voxel (numpy.unique(label_image[markers] - 1), generate.py:334-337)
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_region_flags(const int* __restrict__ labels, const uint8_t* __restrict__ markers, long long n,
                                                                uint8_t* __restrict__ flags)
{
    for (long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x; p < n; p += (long long)gridDim.x * LAB_BLOCK)
        if (markers[p]) flags[labels[p] - 1] = 1;
}

// the same flags from a list of marked voxels: one thread per id, flags[label[id] - 1] = 1
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_voxel_flags(const int* __restrict__ labels, const long long* __restrict__ ids, long long m,
                                                               uint8_t* __restrict__ flags)
{
    for (long long t = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x; t < m; t += (long long)gridDim.x * LAB_BLOCK)
        flags[labels[ids[t]] - 1] = 1;
}

// out[p] = per_region[label[p] - 1]: the relabel_map step of bin/medpy_graphcut_label.py:139-148
__global__ void __launch_bounds__(LAB_BLOCK) k_lab_apply(const int* __restrict__ labels, const uint8_t* __restrict__ per_region, long long n,
                                                         uint8_t* __restrict__ out)
{
    for (long long p = (long long)blockIdx.x * LAB_BLOCK + threadIdx.x; p < n; p += (long long)gridDim.x * LAB_BLOCK)
        out[p] = per_region[labels[p] - 1];
}
