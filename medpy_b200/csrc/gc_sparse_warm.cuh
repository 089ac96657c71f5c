// gc_sparse_warm.cuh -- folding add_tweights / sum_edge calls into the solved state of a general sparse graph
// (mgc_sparse_* with MGC_OPT_WARM; DESIGN.md §8 "Warm re-solve of sparse graphs").
//
// BK's add_tweights and sum_edge act on the residual tr_cap / r_cap (graph.h:415-480), so maxflow(), more calls,
// maxflow() continues from the residual graph.  A warm handle keeps the push-relabel state of its last solve resident
// (gc_sparse.cuh's SparseState plus `sent`, the source flow each node has pushed into the network) and these per-node
// bodies restate the lattice fold arithmetic of DESIGN.md §4.6 on CSR arcs:
//   * spw_read: the residual terminal capacity r(v); absorbed sink flow moves into the constant;
//   * spw_add_tweights: BK's add_tweights on r, the minimum into the constant;
//   * spw_write: r' back: a sink link drains the node's excess at once, a source residual pushes the clamp of the
//     residual out-capacity;
//   * spw_pair_dec / spw_excess_change: n-link decrements, flow beyond the new capacity cancelled, a node left short
//     covered by the Kohli-Torr step.
// Like gc_sparse.cuh the bodies are plain inline functions, so tests/emu/sparse_warm_emu.cpp runs them on the host.
#pragma once
#include "gc_sparse.cuh"

#define SPW_TOL 5.684341886080802e-14   // 2^-44: the pair rule of the decrement fold (DESIGN.md §4.6, "Tolerance")

struct SparseWarm {
    int n;
    const int* row;      // [n+1]
    const int* head;     // [m2]
    double* cap;         // [m2] residual capacity
    double* tr;          // [n]  residual terminal representation: >0 source capacity (of which `sent` was pushed), <0 sink
    double* excess;      // [n]
    double* sunk;        // [n]  flow absorbed by the sink link since it was last written
    double* sent;        // [n]  source flow pushed since the source link was last written
};

// the clamp of a source link: the sum of the residual out-capacities rounded up, times the clamp slack, and from 1 on
// rounded up to an integer (NaN stays NaN).  Whatever a node is sent beyond its out-capacity can never leave it, so any
// bound above that sum keeps the cut; an integer one keeps integer graphs integer, so `tr - sent` reads back exactly.
// Below 1 the bound stays at the scale of the capacities: an excess far above them would lose the small pushes to
// rounding (e - d == e).
SP_HD double spw_clamp_limit(const SparseWarm& W, int v)
{
    double out = 0.0;
    for (int a = W.row[v]; a < W.row[v + 1]; ++a) out = sp_add_up(out, W.cap[a]);
    const double lim = out * SP_CLAMP_SLACK;
    return lim >= 1.0 ? ceil(lim) : lim;
}

// r(v): tr > 0: the un-pushed source residual; tr < 0: the remaining sink capacity, negated, with the absorbed flow
// moved into *dk (energy = constant + absorbed flow, so it stays counted once); else 0
SP_HD double spw_read(const SparseWarm& W, int v, double* dk)
{
    const double tr = W.tr[v];
    if (tr > 0) return tr - W.sent[v];
    if (tr < 0) {
        const double a = W.sunk[v];
        *dk += a;
        W.sunk[v] = 0.0;
        return tr + a;
    }
    return 0.0;
}

// graph.h:418-424 on the residual terminal capacity
SP_HD double spw_add_tweights(double r, double s, double t, double* dk)
{
    if (r > 0) s += r; else t -= r;
    *dk += (s < t) ? s : t;
    return s - t;
}

// r' back into a node that carries no terminal flow once spw_read ran
SP_HD void spw_write(const SparseWarm& W, int v, double r)
{
    if (r < 0) {
        W.tr[v] = r;
        W.sent[v] = 0.0;
        const double e = W.excess[v], c = -r;
        if (e < c) { W.sunk[v] = e; W.excess[v] = 0.0; } else { W.sunk[v] = c; W.excess[v] = e - c; }   // saturation exact
    } else if (r > 0) {
        W.tr[v] = r;
        const double lim = spw_clamp_limit(W, v);
        double p = r < lim ? r : lim;
        if (!(lim == lim)) p = r;
        W.sent[v] = p;
        W.excess[v] += p;
    } else {
        W.tr[v] = 0.0;
        W.sent[v] = 0.0;
    }
}

// the first solve's init on a warm handle: the source link pushes the clamp and records it as `sent`
SP_HD void spw_init_node(const SparseWarm& W, int v)
{
    W.excess[v] = 0.0;
    W.sunk[v] = 0.0;
    W.sent[v] = 0.0;
    const double tr = W.tr[v];
    if (tr > 0) spw_write(W, v, tr);
}

// one node's add_tweights calls, in call order (`order` lists them)
SP_HD double spw_tlink_node(const SparseWarm& W, int v, const unsigned* order, long long first, long long count,
                            const double* src, const double* snk)
{
    double dk = 0.0;
    double r = spw_read(W, v, &dk);
    for (long long k = 0; k < count; ++k) {
        const unsigned c = order[first + k];
        r = spw_add_tweights(r, src[c], snk[c], &dk);
    }
    spw_write(W, v, r);
    return dk;
}

// a node whose residual out-capacity rose: release more of its un-pushed source residual under the same clamp
SP_HD void spw_reclamp_node(const SparseWarm& W, int v)
{
    if (!(W.tr[v] > 0)) return;
    const double r = W.tr[v] - W.sent[v];
    if (r > 0) spw_write(W, v, r);
}

// sum_edge increments of one pair in call order, as BK's sequence of residual += (graph.h:472-476)
SP_HD void spw_pair_inc(double* cap, int a, int b, const unsigned* order, long long first, long long count,
                        const double* c_lh, const double* c_hl)
{
    double x = cap[a], y = cap[b];
    for (long long k = 0; k < count; ++k) {
        const unsigned c = order[first + k];
        x += c_lh[c];
        y += c_hl[c];
    }
    cap[a] = x;
    cap[b] = y;
}

// decrements of one pair: true when the pair cannot give them (δ + δ' beyond r_ab + r_ba by more than the tolerance)
SP_HD bool spw_pair_refused(double ra, double rb, double dl, double dh)
{
    const double have = ra + rb, take = dl + dh;
    const double big = have > take ? have : take;
    return take - have > SPW_TOL * big;
}

// a = r_ab − δ, b = r_ba − δ'; flow beyond the new capacity is cancelled, the ends' excess changes go to dx_*
SP_HD void spw_pair_dec(double* cap, int a, int b, double dl, double dh, double* dx_lo, double* dx_hi)
{
    double x = cap[a] - dl, y = cap[b] - dh, el = 0.0, eh = 0.0;
    if (x < 0) { const double d = -x; x = 0.0; y -= d; el = d; eh = -d; }
    else if (y < 0) { const double d = -y; y = 0.0; x -= d; eh = d; el = -d; }
    cap[a] = x < 0 ? 0.0 : x;      // what the tolerance lets come out negative
    cap[b] = y < 0 ? 0.0 : y;
    *dx_lo = el;
    *dx_hi = eh;
}

// e' = e + Δe; a node left short takes s = −e' from its un-pushed source residual, and the rest raises both terminal
// links by the same amount (Kohli-Torr), lowering the constant
SP_HD double spw_excess_change(const SparseWarm& W, int v, double de)
{
    const double e = W.excess[v] + de;
    if (e >= 0) { W.excess[v] = e; return 0.0; }
    W.excess[v] = 0.0;
    const double s = -e;
    double dk = 0.0;
    double r = spw_read(W, v, &dk);
    const double take = r > 0 ? (r < s ? r : s) : 0.0;
    dk += take - s;
    r -= s;
    spw_write(W, v, r);
    return dk;
}

// CSR re-assembly: node u's old arcs move to the front of its new range, the reverse-arc ids follow their node
SP_HD void spw_move_node(int u, const int* row_old, const int* head_old, const int* sis_old, const double* cap_old,
                         const int* row_new, int* head_new, int* sis_new, double* cap_new)
{
    const int a0 = row_old[u], deg = row_old[u + 1] - a0, b0 = row_new[u];
    for (int k = 0; k < deg; ++k) {
        const int a = a0 + k, v = head_old[a];
        head_new[b0 + k] = v;
        cap_new[b0 + k] = cap_old[a];
        sis_new[b0 + k] = row_new[v] + (sis_old[a] - row_old[v]);
    }
}

// a new pair's two arcs at their node-local offsets, capacity 0 (the increments then add the calls' capacities)
SP_HD void spw_new_pair(int lo, int hi, int olo, int ohi, const int* row_new, int* head_new, int* sis_new, double* cap_new)
{
    const int a = row_new[lo] + olo, b = row_new[hi] + ohi;
    head_new[a] = hi; head_new[b] = lo;
    sis_new[a] = b; sis_new[b] = a;
    cap_new[a] = 0.0; cap_new[b] = 0.0;
}

#if defined(__CUDACC__)
// ---------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_spw_init(SparseWarm W)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < W.n; u += gridDim.x * blockDim.x) spw_init_node(W, u);
}

// fixed-order block sum of one value per thread into partials[blockIdx.x]
__device__ __forceinline__ void spw_block_sum(double v, double* __restrict__ partials)
{
    __shared__ double sh[256];
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + k]);
        __syncthreads();
    }
    if (threadIdx.x == 0) partials[blockIdx.x] = sh[0];
}

__global__ void __launch_bounds__(256) k_spw_sum_partials(const double* __restrict__ partials, long long nb, double* __restrict__ out)
{
    __shared__ double sh[256];
    double s = 0.0;
    for (long long b = threadIdx.x; b < nb; b += 256) s = __dadd_rn(s, partials[b]);
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + k]);
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = sh[0];
}

__device__ __forceinline__ bool spw_is_head(const unsigned* keys, long long i, long long m)
{
    return i < m && keys[i] != 0xffffffffu && (i == 0 || keys[i - 1] != keys[i]);
}

__device__ __forceinline__ long long spw_run_end(const unsigned* keys, long long i, long long m)
{
    long long k = i + 1;
    while (k < m && keys[k] == keys[i]) ++k;
    return k;
}

// one thread per node with calls (the first of its run of sorted keys)
__global__ void __launch_bounds__(256) k_spw_tlink_fold(SparseWarm W, const unsigned* __restrict__ keys, const unsigned* __restrict__ order,
                                                        long long m, const double* __restrict__ src, const double* __restrict__ snk,
                                                        double* __restrict__ partials)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    double dk = 0.0;
    if (spw_is_head(keys, i, m)) dk = spw_tlink_node(W, (int)keys[i], order, i, spw_run_end(keys, i, m) - i, src, snk);
    spw_block_sum(dk, partials);
}

// CSR re-assembly: new degree per node, the exclusive scan as int row offsets, old arcs, new pairs
__global__ void __launch_bounds__(256) k_spw_count_new(const int* __restrict__ lo, const int* __restrict__ hi, long long q,
                                                       unsigned* __restrict__ added)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i < q) { atomicAdd(&added[lo[i]], 1u); atomicAdd(&added[hi[i]], 1u); }
}

__global__ void __launch_bounds__(256) k_spw_degree(const int* __restrict__ row_old, int n, unsigned* __restrict__ cnt)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x)
        cnt[u] += (unsigned)(row_old[u + 1] - row_old[u]);
}

__global__ void __launch_bounds__(256) k_spw_row(const unsigned long long* __restrict__ off, int n, int* __restrict__ row_new)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u <= n; u += gridDim.x * blockDim.x) row_new[u] = (int)off[u];
}

__global__ void __launch_bounds__(256) k_spw_move(int n, const int* __restrict__ row_old, const int* __restrict__ head_old,
                                                  const int* __restrict__ sis_old, const double* __restrict__ cap_old,
                                                  const int* __restrict__ row_new, int* __restrict__ head_new, int* __restrict__ sis_new,
                                                  double* __restrict__ cap_new)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x)
        spw_move_node(u, row_old, head_old, sis_old, cap_old, row_new, head_new, sis_new, cap_new);
}

__global__ void __launch_bounds__(256) k_spw_new_pairs(const int* __restrict__ lo, const int* __restrict__ hi, const int* __restrict__ olo,
                                                       const int* __restrict__ ohi, long long q, const int* __restrict__ row_new,
                                                       int* __restrict__ head_new, int* __restrict__ sis_new, double* __restrict__ cap_new)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i < q) spw_new_pair(lo[i], hi[i], olo[i], ohi[i], row_new, head_new, sis_new, cap_new);
}

// one thread per pair with increments; flags the tails whose out-capacity rose
__global__ void __launch_bounds__(256) k_spw_pair_inc(SparseWarm W, const unsigned* __restrict__ keys, const unsigned* __restrict__ order,
                                                      long long m, const int* __restrict__ lo, const int* __restrict__ hi,
                                                      const int* __restrict__ olo, const int* __restrict__ ohi,
                                                      const double* __restrict__ c_lh, const double* __restrict__ c_hl,
                                                      uint8_t* __restrict__ tail)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (!spw_is_head(keys, i, m)) return;
    const long long end = spw_run_end(keys, i, m);
    const unsigned c0 = order[i];
    const int u = lo[c0], v = hi[c0];
    const int a = W.row[u] + olo[c0], b = W.row[v] + ohi[c0];
    spw_pair_inc(W.cap, a, b, order, i, end - i, c_lh, c_hl);
    bool up_lh = false, up_hl = false;
    for (long long k = i; k < end; ++k) { up_lh |= c_lh[order[k]] > 0; up_hl |= c_hl[order[k]] > 0; }
    if (up_lh) tail[u] = 1;
    if (up_hl) tail[v] = 1;
}

__global__ void __launch_bounds__(256) k_spw_reclamp(SparseWarm W, uint8_t* __restrict__ tail)
{
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < W.n; u += gridDim.x * blockDim.x) {
        if (!tail[u]) continue;
        tail[u] = 0;
        spw_reclamp_node(W, u);
    }
}

// decrements: per pair the sums in call order, the pair rule (flag), then the arcs and the ends' excess changes
__device__ __forceinline__ double2 spw_pair_dec_sums(const unsigned* order, long long i, long long end, const double* d_lh,
                                                     const double* d_hl)
{
    double x = 0.0, y = 0.0;
    for (long long k = i; k < end; ++k) { x += d_lh[order[k]]; y += d_hl[order[k]]; }
    return make_double2(x, y);
}

__global__ void __launch_bounds__(256) k_spw_pair_check(SparseWarm W, const unsigned* __restrict__ keys, const unsigned* __restrict__ order,
                                                        long long m, const int* __restrict__ lo, const int* __restrict__ hi,
                                                        const int* __restrict__ olo, const int* __restrict__ ohi,
                                                        const double* __restrict__ d_lh, const double* __restrict__ d_hl,
                                                        int* __restrict__ refused)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (!spw_is_head(keys, i, m)) return;
    const unsigned c0 = order[i];
    const double2 d = spw_pair_dec_sums(order, i, spw_run_end(keys, i, m), d_lh, d_hl);
    const int a = W.row[lo[c0]] + olo[c0], b = W.row[hi[c0]] + ohi[c0];
    if (spw_pair_refused(W.cap[a], W.cap[b], d.x, d.y)) *refused = 1;
}

// writes two end entries per call slot: node key (0xffffffff for slots that are no pair's first) and excess change
__global__ void __launch_bounds__(256) k_spw_pair_dec(SparseWarm W, const unsigned* __restrict__ keys, const unsigned* __restrict__ order,
                                                      long long m, const int* __restrict__ lo, const int* __restrict__ hi,
                                                      const int* __restrict__ olo, const int* __restrict__ ohi,
                                                      const double* __restrict__ d_lh, const double* __restrict__ d_hl,
                                                      unsigned* __restrict__ end_key, double* __restrict__ end_dx)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= m) return;
    unsigned ku = 0xffffffffu, kv = 0xffffffffu;
    double el = 0.0, eh = 0.0;
    if (spw_is_head(keys, i, m)) {
        const unsigned c0 = order[i];
        const int u = lo[c0], v = hi[c0];
        const double2 d = spw_pair_dec_sums(order, i, spw_run_end(keys, i, m), d_lh, d_hl);
        spw_pair_dec(W.cap, W.row[u] + olo[c0], W.row[v] + ohi[c0], d.x, d.y, &el, &eh);
        ku = (unsigned)u;
        kv = (unsigned)v;
    }
    end_key[2 * i] = ku;
    end_key[2 * i + 1] = kv;
    end_dx[2 * i] = el;
    end_dx[2 * i + 1] = eh;
}

// each end once, in ascending node order; its changes summed in the order of the (stable) sorted entries
__global__ void __launch_bounds__(256) k_spw_ends(SparseWarm W, const unsigned* __restrict__ keys, const unsigned* __restrict__ order,
                                                  long long m, const double* __restrict__ dx, double* __restrict__ partials)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    double dk = 0.0;
    if (spw_is_head(keys, i, m)) {
        const long long end = spw_run_end(keys, i, m);
        double de = 0.0;
        for (long long k = i; k < end; ++k) de += dx[order[k]];
        dk = spw_excess_change(W, (int)keys[i], de);
    }
    spw_block_sum(dk, partials);
}
#endif  // __CUDACC__
