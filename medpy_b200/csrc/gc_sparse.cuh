// gc_sparse.cuh -- push-relabel max-flow on an arbitrary sparse graph in CSR form (SURVEY.md §8 rows f3/f4).
//
// Serves the graphs that are NOT voxel lattices: the region adjacency graph `graph_from_labels` builds
// (generate.py:177-338) and graphs a user assembles edge by edge through GCGraph / GraphDouble
// (graph.py:382-440, wrapper.cpp:63-83, e.g. tests/graphcut_/graph.py:47).  Same contract as the lattice solver
// (gc_solver.cuh, DESIGN.md §4): maximum PREFLOW by lock-free push-relabel (one thread per node, neighbour state
// updated with atomics), exact backward BFS from the sink between rounds, stop test only right after such a BFS;
// `height >= SP_HINF` is then exactly the reference's "not SINK" set (graph.h:560-571) and the energy is the
// add_tweights constants plus the flow the sink links absorbed.
//
// The per-node bodies are plain inline functions so that tests/emu/sparse_emu.cpp can compile and run the SAME
// code sequentially on the host (a logic check that needs no GPU); the __global__ wrappers below are the product.
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define SP_HD __host__ __device__ __forceinline__
#else
#define SP_HD inline
#endif

#define SP_HINF 0x3fffffff
#define SP_CLAMP_SLACK 1.0000001   // same head-room as SOURCE_CLAMP_SLACK (gc_common.cuh): no one-ulp residuals

struct SparseState {
    int n;               // nodes
    int m2;              // arcs: two per connected node pair
    const int* row;      // [n+1] first arc of every node
    const int* head;     // [m2]  node the arc points to
    const int* sis;      // [m2]  index of the reverse arc
    double* cap;         // [m2]  residual capacity
    const double* tr;    // [n]   net terminal capacity after the add_tweights replay (graph.h:415-425): >0 source, <0 sink
    double* excess;      // [n]
    double* sunk;        // [n]   flow absorbed by the node's sink link so far (capacity max(-tr, 0))
    int* height;         // [n]
};

SP_HD void sp_atomic_add(double* p, double v)
{
#if defined(__CUDA_ARCH__)
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

// a + b rounded towards +inf (the host emulation may return one ulp more: still an upper bound)
SP_HD double sp_add_up(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dadd_ru(a, b);
#else
    return std::nextafter(a + b, INFINITY);
#endif
}

// excess = min(max(tr,0), roundup(sum of out-capacities) * slack): what cannot leave the node can never be part of a
// flow, so clamping the source link changes neither the cut value nor the sink-reachable set (DESIGN.md §4.2)
SP_HD void sp_init_node(const SparseState& G, int u)
{
    const double tr = G.tr[u];
    double e = 0.0;
    if (tr > 0) {
        double out = 0.0;
        for (int a = G.row[u]; a < G.row[u + 1]; ++a) out = sp_add_up(out, G.cap[a]);
        const double lim = out * SP_CLAMP_SLACK;
        e = tr < lim ? tr : lim;
        if (!(out == out)) e = tr;   // NaN capacities: leave the link alone
    }
    G.excess[u] = e;
    G.sunk[u] = 0.0;
}

// Up to `max_steps` push steps of node u, then a relabel if it is stuck (Hong & He's lock-free formulation: push to
// the lowest residual neighbour while it is strictly lower, otherwise lift to one above it).  Only u lowers
// cap[a] of its own arcs and its own excess is corrected by an atomic subtraction, so concurrent pushes INTO u are
// never lost.  Returns true when u was active.
SP_HD bool sp_push_node(const SparseState& G, int u, int max_steps)
{
    double e = G.excess[u];
    if (!(e > 0)) return false;
    const int h = G.height[u];
    if (h >= SP_HINF) return false;
    double pushed = 0.0;
    const double scap = -G.tr[u];
    if (scap > 0) {                       // the sink sits at height 0: always admissible
        double sf = G.sunk[u];
        const double r = scap - sf;
        if (r > 0) {
            double d;
            if (e < r) { d = e; sf += d; } else { d = r; sf = scap; }   // saturation is exact
            G.sunk[u] = sf;
            e -= d;
            pushed += d;
        }
    }
    int newh = h;
    for (int step = 0; step < max_steps && e > 0; ++step) {
        int ab = -1, hb = SP_HINF;
        for (int a = G.row[u]; a < G.row[u + 1]; ++a) {
            if (G.cap[a] > 0) {
                const int hv = G.height[G.head[a]];
                if (hv < hb) { hb = hv; ab = a; }
            }
        }
        if (ab < 0) { newh = SP_HINF; break; }     // no residual arc and no sink residual: can never reach the sink
        if (hb >= h) { newh = hb + 1; break; }      // relabel
        const double c = G.cap[ab];
        const double d = e < c ? e : c;
        sp_atomic_add(&G.cap[ab], -d);
        sp_atomic_add(&G.cap[G.sis[ab]], d);
        sp_atomic_add(&G.excess[G.head[ab]], d);
        e -= d;
        pushed += d;
    }
    if (newh != h) G.height[u] = newh;    // (e > 0 here implies the sink link, if any, is saturated)
    if (pushed > 0) sp_atomic_add(&G.excess[u], -pushed);
    return true;
}

// exact distances to the sink in the residual graph: start ...
SP_HD void sp_relabel_init_node(const SparseState& G, int u)
{
    G.height[u] = ((-G.tr[u]) - G.sunk[u] > 0) ? 1 : SP_HINF;
}

// ... and relax in place until nothing changes (labels only ever decrease towards the true distance)
SP_HD bool sp_relax_node(const SparseState& G, int u)
{
    const int h = G.height[u];
    if (h <= 1) return false;
    int best = h;
    for (int a = G.row[u]; a < G.row[u + 1]; ++a) {
        if (G.cap[a] > 0) {
            const int hv = G.height[G.head[a]] + 1;
            best = hv < best ? hv : best;
        }
    }
    if (best < h) { G.height[u] = best; return true; }
    return false;
}

SP_HD bool sp_is_active(const SparseState& G, int u)
{
    return G.excess[u] > 0 && G.height[u] < SP_HINF;
}

#if defined(__CUDACC__)
// ---------------------------------------------------------------------------------------------------------------
// kernels: one thread per node (grid-stride)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sp_init(SparseState G)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < G.n; u += gridDim.x * blockDim.x) sp_init_node(G, u);
}

__global__ void __launch_bounds__(256) k_sp_push(SparseState G, int max_steps, int* __restrict__ work)
{
    bool any = false;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < G.n; u += gridDim.x * blockDim.x)
        any |= sp_push_node(G, u, max_steps);
    if (any) *work = 1;
}

__global__ void __launch_bounds__(256) k_sp_relabel_init(SparseState G)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < G.n; u += gridDim.x * blockDim.x) sp_relabel_init_node(G, u);
}

__global__ void __launch_bounds__(256) k_sp_relax(SparseState G, int* __restrict__ changed)
{
    bool any = false;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < G.n; u += gridDim.x * blockDim.x) any |= sp_relax_node(G, u);
    if (any) *changed = 1;
}

__global__ void __launch_bounds__(256) k_sp_count_active(SparseState G, unsigned long long* __restrict__ count)
{
    unsigned long long c = 0;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < G.n; u += gridDim.x * blockDim.x) c += sp_is_active(G, u) ? 1u : 0u;
    if (c) atomicAdd(count, c);
}

// mask[u] = 1 unless u can reach the sink (graph.h:560-571); energy part = sum of absorbed flow in a FIXED order
// (256 interleaved chains + tree, one block): deterministic for a given graph
__global__ void __launch_bounds__(256) k_sp_readout(SparseState G, uint8_t* __restrict__ mask, double* __restrict__ absorbed)
{
    __shared__ double sh[256];
    const int tid = threadIdx.x;
    double s = 0.0;
    for (int u = tid; u < G.n; u += 256) {
        mask[u] = G.height[u] >= SP_HINF ? 1 : 0;
        s = __dadd_rn(s, G.sunk[u]);
    }
    sh[tid] = s;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (tid < k) sh[tid] = __dadd_rn(sh[tid], sh[tid + k]);
        __syncthreads();
    }
    if (tid == 0) absorbed[0] = sh[0];
}

// absorbed[s] = flow absorbed by the nodes [off[s], off[s+1]), summed as k_sp_readout sums a whole graph's (256 chains
// interleaved from the range's first node, then the same tree): one block per range, no atomics, the same bits every run
__global__ void __launch_bounds__(256) k_sp_segment_absorbed(const double* __restrict__ sunk, const long long* __restrict__ off,
                                                             long long segs, double* __restrict__ absorbed)
{
    __shared__ double sh[256];
    const int tid = threadIdx.x;
    for (long long s = blockIdx.x; s < segs; s += gridDim.x) {
        const long long a = off[s], b = off[s + 1];
        double acc = 0.0;
        for (long long u = a + tid; u < b; u += 256) acc = __dadd_rn(acc, sunk[u]);
        sh[tid] = acc;
        __syncthreads();
        for (int k = 128; k > 0; k >>= 1) {
            if (tid < k) sh[tid] = __dadd_rn(sh[tid], sh[tid + k]);
            __syncthreads();
        }
        if (tid == 0) absorbed[s] = sh[0];
        __syncthreads();
    }
}
#endif  // __CUDACC__
