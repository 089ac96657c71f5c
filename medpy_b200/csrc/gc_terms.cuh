// gc_terms.cuh -- energy-term kernels: K0 (min/max), K1 (n-link stencils), K2 (t-links / markers).
//
// They replace the reference's per-edge / per-node Python loops
//   energy_voxel.py:611-664 (__skeleton_base) -> GCGraph.set_nweight -> Graph::sum_edge (graph.h:456-480)
//   graph.py:532-552 (set_tweights_all), :310-380 (set_source_nodes/set_sink_nodes)
//     -> Graph::add_tweights (graph.h:415-425)
// All arithmetic is float64 with explicitly rounded operations (no FMA contraction) so the weights
// equal numpy's bit for bit wherever numpy's own operations are correctly rounded (+,-,*,/); exp and
// pow are within an ulp or two of numpy's libm.
#pragma once
#include "gc_common.cuh"
#include "gc_exprange.cuh"
#include "gc_expneg.cuh"
#include <cfloat>

// ---------------------------------------------------------------------------------------------------
// input element access
// ---------------------------------------------------------------------------------------------------
template <typename E> struct Elem;
template <> struct Elem<float> {
    static __device__ __forceinline__ double val(float x) { return (double)x; }
    static __device__ __forceinline__ float absv(float x) { return fabsf(x); }
};
template <> struct Elem<double> {
    static __device__ __forceinline__ double val(double x) { return x; }
    static __device__ __forceinline__ double absv(double x) { return fabs(x); }
};
template <> struct Elem<uint8_t> {
    static __device__ __forceinline__ double val(uint8_t x) { return (double)x; }
    static __device__ __forceinline__ uint8_t absv(uint8_t x) { return x; }
};
template <> struct Elem<int16_t> {
    static __device__ __forceinline__ double val(int16_t x) { return (double)x; }
    // numpy.abs on int16 wraps for -32768 (energy_voxel.py:558 works in the input dtype)
    static __device__ __forceinline__ int16_t absv(int16_t x) { return (int16_t)(x < 0 ? -x : x); }
};
template <> struct Elem<int32_t> {
    static __device__ __forceinline__ double val(int32_t x) { return (double)x; }
    static __device__ __forceinline__ int32_t absv(int32_t x) { return (int32_t)(x < 0 ? (int32_t)(0u - (unsigned)x) : x); }
};

// ---------------------------------------------------------------------------------------------------
// strided gather: arbitrary positive byte strides -> C-contiguous (used for Fortran-ordered inputs
// such as medpy.io.load returns, io/load.py:125-127)
// ---------------------------------------------------------------------------------------------------
struct Strides4 { long long s[4]; };

template <typename E, int ND>
__global__ void k_gather(Lattice L, const char* __restrict__ src, Strides4 st, E* __restrict__ dst)
{
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= L.n) return;
    int c[ND];
    decode<ND>(L, v, c);
    long long off = 0;
#pragma unroll
    for (int d = 0; d < ND; ++d) off += (long long)c[d] * st.s[d];
    dst[v] = *reinterpret_cast<const E*>(src + off);
}

// Fortran-ordered 3-D input (what medpy.io.load returns, io/load.py:125-127): logical axis 0 is the FASTEST in memory,
// so the plain gather above reads one element per 128-byte line.  Tiled transpose instead: for a fixed logical y, a
// 32 x 32 tile of the (z, x) plane is read with z fastest (coalesced in the source) into shared memory and written with x
// fastest (coalesced in the destination).  src element (z, y, x) sits at z + Z * (y + Y * x); dst is C order.
template <typename E>
__global__ void __launch_bounds__(256) k_gather_fortran3(int Z, int Y, int X, const E* __restrict__ src, E* __restrict__ dst)
{
    __shared__ E tile[32][33];
    const int y = blockIdx.y;
    const int z0 = blockIdx.z * 32, x0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8 threads
#pragma unroll
    for (int r = 0; r < 32; r += 8) {
        const int x = x0 + ty + r, z = z0 + tx;
        if (x < X && z < Z) tile[ty + r][tx] = src[(size_t)z + (size_t)Z * ((size_t)y + (size_t)Y * (size_t)x)];
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 32; r += 8) {
        const int z = z0 + ty + r, x = x0 + tx;
        if (x < X && z < Z) dst[((size_t)z * Y + y) * (size_t)X + x] = tile[tx][ty + r];
    }
}

// ---------------------------------------------------------------------------------------------------
// K0: global min / max (difference_linear: |max - min| in the input dtype, energy_voxel.py:174;
//     maximum_linear: max |x| in the input dtype, energy_voxel.py:99)
// A NaN anywhere makes min, max and max |x| NaN, as numpy's min / max do, whatever cell, thread or block it falls in: the
// folds below keep a NaN once they have met one (x < NaN is false) and take the other operand when it is NaN.  For the
// integer types x != x is false and the folds are the plain ones.
// ---------------------------------------------------------------------------------------------------
template <typename E> __device__ __forceinline__ E min_nan(E acc, E x) { return (x < acc || x != x) ? x : acc; }
template <typename E> __device__ __forceinline__ E max_nan(E acc, E x) { return (x > acc || x != x) ? x : acc; }

template <typename E>
__global__ void k_minmax_partial(const E* __restrict__ img, unsigned n, E* __restrict__ pmin, E* __restrict__ pmax,
                                 E* __restrict__ pabs)
{
    __shared__ E smin[256], smax[256], sabs[256];
    unsigned tid = threadIdx.x;
    unsigned i = blockIdx.x * blockDim.x + tid;
    unsigned step = gridDim.x * blockDim.x;
    E lo = img[0], hi = img[0], ab = Elem<E>::absv(img[0]);
    for (; i < n; i += step) {
        E x = img[i];
        E a = Elem<E>::absv(x);
        lo = min_nan(lo, x);
        hi = max_nan(hi, x);
        ab = max_nan(ab, a);
    }
    smin[tid] = lo; smax[tid] = hi; sabs[tid] = ab;
    __syncthreads();
    for (unsigned s = 128; s > 0; s >>= 1) {
        if (tid < s) {
            smin[tid] = min_nan(smin[tid], smin[tid + s]);
            smax[tid] = max_nan(smax[tid], smax[tid + s]);
            sabs[tid] = max_nan(sabs[tid], sabs[tid + s]);
        }
        __syncthreads();
    }
    if (tid == 0) { pmin[blockIdx.x] = smin[0]; pmax[blockIdx.x] = smax[0]; pabs[blockIdx.x] = sabs[0]; }
}

// out[0] = float(abs(max - min)) computed in E; out[1] = float(max |x|)
template <typename E>
__global__ void k_minmax_final(const E* pmin, const E* pmax, const E* pabs, unsigned nb, double* out)
{
    if (threadIdx.x || blockIdx.x) return;
    E lo = pmin[0], hi = pmax[0], ab = pabs[0];
    for (unsigned i = 1; i < nb; ++i) {
        lo = min_nan(lo, pmin[i]);
        hi = max_nan(hi, pmax[i]);
        ab = max_nan(ab, pabs[i]);
    }
    E diff = (E)(hi - lo);            // in the input dtype, like numpy (wraps for narrow ints)
    diff = Elem<E>::absv(diff);
    out[0] = Elem<E>::val(diff);
    out[1] = Elem<E>::val(ab);
}

// ---------------------------------------------------------------------------------------------------
// K1: boundary (n-link) stencil
// ---------------------------------------------------------------------------------------------------
struct BoundaryParams {
    int fn;            // 0 linear, 1 exponential, 2 division, 3 power
    int use_max;       // 1: g(max(|a|,|b|)) (energy_voxel.py:519-558), 0: g(|a-b|) (:561-608)
    double norm;       // linear: M
    double sigma;      // division / power: sigma ; exponential: pow(sigma, 2)
    double inv_sigma2; // exponential: 1 / pow(sigma, 2) (see g_weight)
    double inv_spacing_on; // 0: no spacing
    double spacing[4]; // canonical axes
    // batch lattice (Lattice::zper > 0): per image the one constant its term reads -- M (linear), sigma (division, power)
    // or pow(sigma, 2) (exponential) -- replacing norm / sigma above (device array, one entry per image); else nullptr
    const double* ktab;
};

// The term's constants for a voxel in plane gz: P itself on a lattice of one image, else P with the constant of the
// plane's image (inv_sigma2 formed from it exactly as the host forms it from pow(sigma, 2)).  A pair never spans two images
// (z_pairs), so either end of a pair gives the same constants.
__device__ __forceinline__ BoundaryParams params_at(const BoundaryParams& P, const Lattice& L, int gz)
{
    BoundaryParams Q = P;
    if (L.zper) {
        const double k = P.ktab[image_of(L, gz < L.dim[0] ? gz : L.dim[0] - 1)];
        Q.norm = k;
        Q.sigma = k;
        Q.inv_sigma2 = (P.fn == 1 && k != 0.0) ? __ddiv_rn(1.0, k) : 0.0;
    }
    return Q;
}

// The exponential constant of the range test of a block whose staged box covers planes z_lo .. z_hi (clamped to the
// lattice): on a batch lattice the largest of the images' constants (exp_table_inv_max, gc_exprange.cuh)
__device__ __forceinline__ double range_inv_sigma2(const BoundaryParams& P, const Lattice& L, int z_lo, int z_hi)
{
    if (!L.zper) return P.inv_sigma2;
    z_lo = z_lo < 0 ? 0 : z_lo;
    z_hi = z_hi < L.dim[0] ? z_hi : L.dim[0] - 1;
    return exp_table_inv_max(P.ktab, image_of(L, z_lo), image_of(L, z_hi));
}

// exp_neg / exp_neg_inrange: gc_expneg.cuh

// argument of the exponential term, exactly as g_weight<1> forms it (gc_exprange.cuh)
__device__ __forceinline__ double exp_term_arg(const BoundaryParams& P, double x)
{
    return exp_arg(x, P.inv_sigma2, P.sigma);
}

// FN >= 0 fixes the term at compile time (the specialised kernels of the common cases), FN < 0 reads it from P
template <int FN>
__device__ __forceinline__ double g_weight(const BoundaryParams& P, double x)
{
    const int fn = FN >= 0 ? FN : P.fn;
    double w;
    if (fn == 0) {                       // energy_voxel.py:101-114,176-189
        w = __dsub_rn(1.0, __ddiv_rn(x, P.norm));
        if (w == 0.0) w = DBL_MIN;
    } else if (fn == 1) {                  // :226-236,290-300
        // x^2 / sigma^2 as a multiplication by the pre-computed reciprocal: K1 is instruction-issue bound (fp64 exp
        // + IEEE division), and exp() is not bit-identical to numpy's libm anyway; the argument moves
        // by <= 1 ulp, i.e. the weight by <= |arg| * 1.1e-16 relative (tests allow 2e-13; the north star 1e-5).
        // sigma == 0 keeps the exact division so x = 0 still gives NaN and x > 0 gives DBL_MIN like the reference.
        double t = (P.inv_sigma2 > 0.0 && P.inv_sigma2 < 1e300) ? __dmul_rn(__dmul_rn(x, x), P.inv_sigma2)
                                                                : __ddiv_rn(__dmul_rn(x, x), P.sigma);
        w = exp_neg(t);
        if (w <= 0.0) w = DBL_MIN;
    } else if (fn == 2) {                  // :337-345,399-407
        w = __ddiv_rn(1.0, __dadd_rn(__ddiv_rn(x, P.sigma), 1.0));
        if (w <= 0.0) w = DBL_MIN;
    } else {                               // :444-452,506-514
        w = pow(__ddiv_rn(1.0, __dadd_rn(x, 1.0)), P.sigma);
        if (w <= 0.0) w = DBL_MIN;
    }
    return w;
}

// One thread per voxel p: for every axis d with p_d < D_d-1 computes the weight of the pair (p, q=p+e_d) once
// and adds it to cap(p->q) [array 2d+1, index p] and cap(q->p) [array 2d, index q]; both stores are
// coalesced because q = p + stride_d is contiguous in p.  `bad` is set if a weight <= 0 appears
// (GCGraph.set_nweight raises ValueError there, graph.py:436-437; NaN passes, like the reference).
// FRESH = the capacity arrays hold garbage (first n-link term after create/reset): every entry is then written
// exactly once with plain stores -- arcs that would leave the lattice get 0 -- which saves the memset and the
// read-modify-write (48 + 48 B/voxel in 3-D).
// FN / USE_MAX / SPACING: -1 = decided at run time from P (generic kernel); 0/1/... = compile-time constant, which
// strips the per-arc branch chain from this instruction-issue-bound kernel (the exponential term without spacing,
// i.e. every BASELINE config, runs specialised).
template <typename E, int ND, typename T, bool FRESH, int FN = -1, int USE_MAX = -1, int SPACING = -1>
__global__ void __launch_bounds__(256)
k_boundary(Lattice L, State<T> S, const E* __restrict__ img, BoundaryParams P, int* __restrict__ bad)
{
    unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= L.n) return;
    int c[ND];
    decode<ND>(L, p, c);
    const bool use_max = USE_MAX >= 0 ? (USE_MAX != 0) : (P.use_max != 0);
    const bool spacing = SPACING >= 0 ? (SPACING != 0) : (P.inv_spacing_on != 0.0);
    E ip = img[p];
    double a = use_max ? Elem<E>::val(Elem<E>::absv(ip)) : Elem<E>::val(ip);
    int isbad = 0;
#pragma unroll
    for (int d = 0; d < ND; ++d) {
        if (c[d] + 1 < L.dim[d]) {
            unsigned q = p + L.stride[d];
            E iq = img[q];
            double b = use_max ? Elem<E>::val(Elem<E>::absv(iq)) : Elem<E>::val(iq);
            double x = use_max ? fmax(a, b) : fabs(__dsub_rn(a, b));
            double w = g_weight<FN>(P, x);
            if (spacing) w = __ddiv_rn(w, P.spacing[d]);
            if (w <= 0.0) isbad = 1;
            if (FRESH) {
                S.cap[2 * d + 1][p] = (T)w;
                S.cap[2 * d][q] = (T)w;
            } else {
                S.cap[2 * d + 1][p] += (T)w;
                S.cap[2 * d][q] += (T)w;
            }
        } else if (FRESH) {
            S.cap[2 * d + 1][p] = (T)0;      // no neighbour in +d
        }
        if (FRESH && c[d] == 0) S.cap[2 * d][p] = (T)0;   // no neighbour in -d
    }
    if (isbad) *bad = 1;
}

// dense user-supplied n-links along one axis (sum_edge semantics)
template <int ND, typename T>
__global__ void k_nweights_dense(Lattice L, State<T> S, int axis, const double* __restrict__ fwd,
                                 const double* __restrict__ bwd, int* __restrict__ bad)
{
    unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= L.n) return;
    int c[ND];
    decode<ND>(L, p, c);
    if (c[axis] + 1 >= L.dim[axis]) return;
    double f = fwd[p], b = bwd[p];
    if (f < 0.0 || b < 0.0) *bad = 1;   // Graph::sum_edge asserts cap >= 0 (graph.h:462-463); 0 = pair not set
    S.cap[2 * axis + 1][p] += (T)f;
    S.cap[2 * axis][p + L.stride[axis]] += (T)b;
}

// ---------------------------------------------------------------------------------------------------
// K2: t-links.  add_tweights (graph.h:415-425):
//     delta = tr; if (delta > 0) s += delta; else t -= delta; flow += min(s,t); tr = s - t
// The flow constant is reduced deterministically: per-block tree -> partials -> k_sum_partials.
// ---------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ double add_tweights_dev(T& tr, double s, double t)
{
    double delta = (double)tr;
    if (delta > 0) s = __dadd_rn(s, delta); else t = __dsub_rn(t, delta);
    tr = (T)__dsub_rn(s, t);
    return (s < t) ? s : t;
}

// Deterministic reduction: every thread accumulates its own grid-stride share in a fixed order, then warp
// shuffles + one shared-memory step give the block's partial; k_sum_partials adds the (<= REDUCE_BLOCKS) partials
// in a fixed order.  The result depends only on the launch shape, which is fixed per lattice size.
#define REDUCE_BLOCKS 1056   // 8 x 132 SMs (H100 SXM)
__device__ __forceinline__ void block_sum_store(double x, double* __restrict__ partials)
{
    __shared__ double sh[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = __dadd_rn(x, __shfl_down_sync(0xffffffffu, x, o));
    const unsigned tid = threadIdx.x;
    if ((tid & 31) == 0) sh[tid >> 5] = x;
    __syncthreads();
    if (tid == 0) {
        double t = sh[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) t = __dadd_rn(t, sh[w]);
        partials[blockIdx.x] = t;
    }
}

// regional_probability_map (energy_voxel.py:62-65): products formed in the map's dtype when F32 != 0
template <typename E, typename T>
__global__ void __launch_bounds__(256)
k_regional(Lattice L, State<T> S, const E* __restrict__ prob, double alpha, int compute_f32, int fresh, double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        double s, t;
        if (compute_f32) {
            float p = (float)prob[v];
            float a = (float)alpha;
            s = (double)__fmul_rn(p, a);
            t = (double)__fmul_rn(__fsub_rn(1.0f, p), a);
        } else {
            double p = (double)prob[v];
            s = __dmul_rn(p, alpha);
            t = __dmul_rn(__dsub_rn(1.0, p), alpha);
        }
        T tr = fresh ? (T)0 : S.tr[v];      // fresh: tr[] holds garbage (first t-link term after create/reset)
        double mm = add_tweights_dev(tr, s, t);
        S.tr[v] = tr;
        if (owned(L, v)) m = __dadd_rn(m, mm);
    }
    block_sum_store(m, partials);
}

// float32 probability map, four voxels per thread: one 16-byte load of the map and two 16-byte stores of tr per
// iteration keep enough bytes in flight to run the pass at HBM rate (the scalar form above has one 4-byte load per
// thread outstanding and is bound by load latency).  Requires n % 4 == 0 and a 16-byte aligned map; same arithmetic.
template <typename T>
__global__ void __launch_bounds__(256)
k_regional_f32x4(Lattice L, State<T> S, const float4* __restrict__ prob, double alpha, int compute_f32, int fresh,
                 double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned groups = L.n >> 2;
    const unsigned step = gridDim.x * blockDim.x;
    const float af = (float)alpha;
    for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += step) {
        const float4 p4 = __ldg(prob + q);
        const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
        double2 t01 = make_double2(0.0, 0.0), t23 = make_double2(0.0, 0.0);
        if (!fresh) {
            t01 = reinterpret_cast<const double2*>(S.tr)[2 * q];
            t23 = reinterpret_cast<const double2*>(S.tr)[2 * q + 1];
        }
        double trv[4] = {t01.x, t01.y, t23.x, t23.y};
        const unsigned v = q << 2;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            double s, t;
            if (compute_f32) {
                s = (double)__fmul_rn(pv[k], af);
                t = (double)__fmul_rn(__fsub_rn(1.0f, pv[k]), af);
            } else {
                const double p = (double)pv[k];
                s = __dmul_rn(p, alpha);
                t = __dmul_rn(__dsub_rn(1.0, p), alpha);
            }
            const double mm = add_tweights_dev(trv[k], s, t);
            if (owned(L, v + k)) m = __dadd_rn(m, mm);
        }
        reinterpret_cast<double2*>(S.tr)[2 * q] = make_double2(trv[0], trv[1]);
        reinterpret_cast<double2*>(S.tr)[2 * q + 1] = make_double2(trv[2], trv[3]);
    }
    block_sum_store(m, partials);
}

template <typename T>
__global__ void __launch_bounds__(256)
k_tweights_dense(Lattice L, State<T> S, const double* __restrict__ src, const double* __restrict__ snk,
                 int fresh, double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        T tr = fresh ? (T)0 : S.tr[v];
        double mm = add_tweights_dev(tr, src[v], snk[v]);
        S.tr[v] = tr;
        if (owned(L, v)) m = __dadd_rn(m, mm);
    }
    block_sum_store(m, partials);
}

// set_source_nodes then set_sink_nodes (generate.py:169-172; MAX = 65535, graph.py:286-291)
template <typename T>
__global__ void __launch_bounds__(256)
k_markers(Lattice L, State<T> S, const uint8_t* __restrict__ fg, const uint8_t* __restrict__ bg,
          int fresh, double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        bool f = fg && fg[v], b = bg && bg[v];
        if (f || b || fresh) {
            T tr = fresh ? (T)0 : S.tr[v];
            double mm = 0.0;
            if (f) mm = add_tweights_dev(tr, 65535.0, 0.0);
            if (b) mm = __dadd_rn(mm, add_tweights_dev(tr, 0.0, 65535.0));
            S.tr[v] = tr;
            if (owned(L, v)) m = __dadd_rn(m, mm);
        }
    }
    block_sum_store(m, partials);
}

// Same pass for a graph whose tr[] is already valid (a regional term ran first), 16 voxels per thread: the marker
// volumes are read as 16-byte vectors and the float64 t-link is touched only where a marker is set, so the pass
// costs the 2 B/voxel it has to read (the byte-per-thread form above is load-latency bound).
// Requires n % 16 == 0 and 16-byte aligned marker arrays; the host falls back to k_markers otherwise.
template <typename T>
__global__ void __launch_bounds__(256)
k_markers16(Lattice L, State<T> S, const uint4* __restrict__ fg, const uint4* __restrict__ bg, double* __restrict__ partials)
{
    double m = 0.0;
    const unsigned groups = L.n >> 4;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += step) {
        const uint4 f4 = fg ? __ldg(fg + q) : make_uint4(0u, 0u, 0u, 0u);
        const uint4 b4 = bg ? __ldg(bg + q) : make_uint4(0u, 0u, 0u, 0u);
        if (!(f4.x | f4.y | f4.z | f4.w | b4.x | b4.y | b4.z | b4.w)) continue;
        const unsigned fw[4] = {f4.x, f4.y, f4.z, f4.w};
        const unsigned bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            if (!(fw[w] | bw[w])) continue;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const bool f = ((fw[w] >> (8 * k)) & 0xffu) != 0u;
                const bool b = ((bw[w] >> (8 * k)) & 0xffu) != 0u;
                if (f || b) {
                    const unsigned v = (q << 4) + (unsigned)(w * 4 + k);
                    T tr = S.tr[v];
                    double mm = 0.0;
                    if (f) mm = add_tweights_dev(tr, 65535.0, 0.0);
                    if (b) mm = __dadd_rn(mm, add_tweights_dev(tr, 0.0, 65535.0));
                    S.tr[v] = tr;
                    if (owned(L, v)) m = __dadd_rn(m, mm);
                }
            }
        }
    }
    block_sum_store(m, partials);
}
