// gc_solver.cuh -- lattice push-relabel max-flow kernels (replace Graph::maxflow, maxflow.cpp:471-604).
//
// Algorithm (DESIGN.md §4): maximum PREFLOW by lock-free push-relabel on the implicit lattice, with an
// exact backward BFS from the sink (global relabel) every few sweeps.  The min cut the reference reports
// is solver independent: what_segment(v) == SINK  <=>  v can still reach the sink in the residual graph
// (SURVEY.md §3.3), which is exactly "height[v] finite after an exact global relabel" of a maximum
// preflow.  The stop test is only ever made right after such a relabel: no voxel with excess > 0 has a
// finite label.
#pragma once
#include "gc_common.cuh"

// ---------------------------------------------------------------------------------------------------
// init: excess = min(max(tr,0), roundup(sum of out-capacities)), sink = max(-tr,0)
// Clamping the source link to what can leave the voxel changes neither the cut value nor the minimal
// sink set (DESIGN.md §4.2), and keeps the 65535 hard-marker links from flooding the lattice.
// ---------------------------------------------------------------------------------------------------
template <int ND, typename T>
__global__ void __launch_bounds__(256) k_init_state(Lattice L, State<T> S)
{
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= L.n) return;
    double tr = (double)S.tr[v];
    double e = 0.0;
    if (tr > 0) {
        double out = 0.0;
#pragma unroll
        for (int k = 0; k < 2 * ND; ++k) out = __dadd_ru(out, (double)S.cap[k][v]);
        const double lim = out * SOURCE_CLAMP_SLACK;
        e = tr < lim ? tr : lim;
        if (!(out == out)) e = tr;  // NaN capacities (zero-image linear terms): leave the link alone
    }
    if (!owned(L, v)) e = 0.0;      // ghost planes of a z-slab start with an empty outbox
    S.excess[v] = (T)e;
    S.sink[v] = (T)0;               // flow absorbed so far; the link's capacity is max(-tr, 0)
}

// ---------------------------------------------------------------------------------------------------
// push / relabel sweep: one thread per voxel, lock-free (Hong & He style): an active voxel pushes to its
// lowest residual neighbours while they are strictly lower, then relabels to 1 + the lowest remaining
// residual neighbour.  Neighbour state is updated with atomics; own excess is corrected by an atomic
// subtraction because neighbours add to it concurrently.  `work` is set when anything was active.
// ---------------------------------------------------------------------------------------------------
template <int ND, typename T>
__global__ void __launch_bounds__(256) k_push(Lattice L, State<T> S, int* __restrict__ work)
{
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= L.n) return;
    T e = S.excess[v];
    if (!(e > 0)) return;
    int h = S.height[v];
    if (h >= MGC_HINF) return;
    if (!owned(L, v)) return;
    *work = 1;
    T pushed = 0;
    T scap = -S.tr[v];                // capacity of the sink link (if any)
    if (scap > 0) {                   // the sink sits at height 0: always admissible
        T sf = S.sink[v];             // absorbed so far (kept as a sum of pushes: summing these gives the flow
        T r = scap - sf;              //  without the 65535 - (65535 - tiny) cancellation a residual would have)
        if (r > 0) {
            T d;
            if (e < r) { d = e; sf += d; } else { d = r; sf = scap; }   // saturation is exact
            S.sink[v] = sf;
            e -= d;
            pushed += d;
        }
    }
    if (e > 0) {
        T c[2 * ND];
        int hn[2 * ND];
#pragma unroll
        for (int k = 0; k < 2 * ND; ++k) {
            c[k] = S.cap[k][v];
            hn[k] = MGC_HINF;
            if (c[k] > 0) hn[k] = S.height[(int)v + dir_offset(L, k)];
        }
        int newh = h;
#pragma unroll 1
        for (int it = 0; it < 2 * ND; ++it) {
            int kb = -1, hb = MGC_HINF;
#pragma unroll
            for (int k = 0; k < 2 * ND; ++k)
                if (c[k] > 0 && hn[k] < hb) { hb = hn[k]; kb = k; }
            if (kb < 0) { newh = MGC_HINF; break; }          // no residual arc left: can never reach the sink
            if (hb >= h) { newh = hb + 1; break; }            // relabel
            T d = e < c[kb] ? e : c[kb];
            unsigned w = (unsigned)((int)v + dir_offset(L, kb));
            atomicAdd(&S.cap[kb][v], -d);
            atomicAdd(&S.cap[kb ^ 1][w], d);
            atomicAdd(&S.excess[w], d);
            e -= d;
            pushed += d;
            c[kb] = 0;                                        // saturated, or e is exhausted
            if (!(e > 0)) break;
        }
        if (newh != h) S.height[v] = newh;
    }
    if (pushed > 0) atomicAdd(&S.excess[v], -pushed);
}

// ---------------------------------------------------------------------------------------------------
// global relabel: exact distances to the sink in the residual graph by in-place relaxation
// ---------------------------------------------------------------------------------------------------
template <int ND, typename T>
__global__ void __launch_bounds__(256) k_relabel_init(Lattice L, State<T> S)
{
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= L.n) return;
    unsigned m = 0;
#pragma unroll
    for (int k = 0; k < 2 * ND; ++k)
        if (S.cap[k][v] > 0) m |= 1u << k;
    S.rmask[v] = (uint8_t)m;
    // ghost planes restart at HINF: a from-scratch BFS must only ever see upper bounds, otherwise two slabs
    // can keep each other's stale finite labels alive (count-to-infinity) and the stop test never fires
    S.height[v] = (owned(L, v) && (-S.tr[v]) - S.sink[v] > 0) ? 1 : MGC_HINF;
}

template <int ND>
__global__ void __launch_bounds__(256) k_relabel_relax(Lattice L, const uint8_t* __restrict__ rmask,
                                                        int* __restrict__ height, int* __restrict__ changed)
{
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= L.n) return;
    unsigned m = rmask[v];
    if (!m) return;
    if (!owned(L, v)) return;
    int h = height[v];
    if (h <= 1) return;
    int best = h;
#pragma unroll
    for (int k = 0; k < 2 * ND; ++k) {
        if (m & (1u << k)) {
            int hw = height[(int)v + dir_offset(L, k)] + 1;
            best = hw < best ? hw : best;
        }
    }
    if (best < h) {
        height[v] = best;
        *changed = 1;
    }
}

template <typename T>
__global__ void __launch_bounds__(256) k_count_active(Lattice L, State<T> S, unsigned long long* __restrict__ count)
{
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    bool act = false;
    if (v < L.n) act = (S.excess[v] > 0) && (S.height[v] < MGC_HINF) && owned(L, v);
    unsigned b = __ballot_sync(0xffffffffu, act);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, (unsigned long long)__popc(b));
}

// ---------------------------------------------------------------------------------------------------
// read-out: mask (K5) and energy (K6)
// ---------------------------------------------------------------------------------------------------
// mask[v] = 1 unless v can reach the sink (bin/medpy_graphcut_voxel.py:177-181 with graph.h:560-571), fused with the
// energy reduction: flow absorbed by the sink links of the owned voxels (fixed-order fp64 sums, deterministic)
// LAZY: sink[v] holds a value only where rmask bit 7 (RM_SINKV, gc_tiles.cuh) is set -- the 3-D tile solver never
// zero-fills the array, and only the voxels that absorbed flow are read here (4 + 1 B/voxel instead of 4 + 8).
// CLEAN (3-D tile solver, X % 4 == 0, dirty-tile tracking over the whole solve): a tile that is not flagged in
// `dflag` still holds the reset labels (1 where the sink link is residual and the voxel owned, HINF elsewhere), so its
// mask comes from rmask alone and its labels are not read (1 B read per voxel there instead of 5).
template <typename T, bool LAZY, bool CLEAN = false>
__global__ void __launch_bounds__(256) k_readout(Lattice L, State<T> S, uint8_t* __restrict__ mask, double* __restrict__ partials,
                                                 const int* __restrict__ dflag = nullptr, int nty = 0, int ntx = 0)
{
    __shared__ double sh[8];
    double a = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    // four voxels per thread and iteration (16 B label load, 32 B of sink flow, 4 B mask store); tail handled scalar
    const unsigned n4 = L.n >> 2;
    for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += step) {
        const unsigned v = q << 2;
        uchar4 m;
        unsigned rm = 0;
        bool clean = false;
        if (CLEAN) {      // the four voxels lie in one row of one tile
            rm = reinterpret_cast<const unsigned*>(S.rmask)[q];
            const unsigned gz = div_stride(L, v, 0), r = v - gz * L.stride[0];
            const unsigned gy = div_stride(L, r, 1), gx = r - gy * L.stride[1];
            clean = dflag[((int)(gz >> 3) * nty + (int)(gy >> 3)) * ntx + (int)(gx >> 3)] == 0;
        }
        if (clean) {
            const bool own = owned(L, v);          // bit 6 of rmask: RM_SINK (gc_tiles.cuh)
            m.x = (own && (rm & 0x40u)) ? 0 : 1; m.y = (own && ((rm >> 8) & 0x40u)) ? 0 : 1;
            m.z = (own && ((rm >> 16) & 0x40u)) ? 0 : 1; m.w = (own && ((rm >> 24) & 0x40u)) ? 0 : 1;
        } else {
            const int4 h = reinterpret_cast<const int4*>(S.height)[q];
            m.x = h.x >= MGC_HINF ? 1 : 0; m.y = h.y >= MGC_HINF ? 1 : 0;
            m.z = h.z >= MGC_HINF ? 1 : 0; m.w = h.w >= MGC_HINF ? 1 : 0;
        }
        reinterpret_cast<uchar4*>(mask)[q] = m;
        if (LAZY) {
            const unsigned r4 = (CLEAN ? rm : reinterpret_cast<const unsigned*>(S.rmask)[q]) & 0x80808080u;
            if (r4) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if ((r4 >> (8 * i + 7)) & 1u) { if (owned(L, v + i)) a = __dadd_rn(a, (double)S.sink[v + i]); }
            }
        } else if (sizeof(T) == 8) {
            const double2 s0 = reinterpret_cast<const double2*>(S.sink)[2 * q];
            const double2 s1 = reinterpret_cast<const double2*>(S.sink)[2 * q + 1];
            if (owned(L, v)) a = __dadd_rn(a, s0.x);
            if (owned(L, v + 1)) a = __dadd_rn(a, s0.y);
            if (owned(L, v + 2)) a = __dadd_rn(a, s1.x);
            if (owned(L, v + 3)) a = __dadd_rn(a, s1.y);
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) if (owned(L, v + i)) a = __dadd_rn(a, (double)S.sink[v + i]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (L.n & 3u)) {
        const unsigned v = (n4 << 2) + threadIdx.x;
        mask[v] = S.height[v] >= MGC_HINF ? 1 : 0;
        if (owned(L, v) && (!LAZY || (S.rmask[v] & 0x80u))) a = __dadd_rn(a, (double)S.sink[v]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a = __dadd_rn(a, __shfl_down_sync(0xffffffffu, a, o));
    const unsigned tid = threadIdx.x;
    if ((tid & 31) == 0) sh[tid >> 5] = a;
    __syncthreads();
    if (tid == 0) {
        double t = sh[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) t = __dadd_rn(t, sh[w]);
        partials[blockIdx.x] = t;
    }
}

// ---------------------------------------------------------------------------------------------------
// z-slab border messages
// ---------------------------------------------------------------------------------------------------
// pack: heights of my border plane + the flow parked in the ghost plane's excess (my outbox), which is cleared
template <typename T>
__global__ void k_slab_pack(unsigned plane, const int* __restrict__ height_border, T* __restrict__ excess_ghost,
                            int* __restrict__ h_out, double* __restrict__ f_out)
{
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= plane) return;
    h_out[i] = height_border[i];
    if (f_out) {                    // labels-only messages (relabel rounds: nothing was pushed since the last exchange) leave the outbox alone
        f_out[i] = (double)excess_ghost[i];
        excess_ghost[i] = 0;
    }
}

// unpack: ghost heights <- neighbour's border heights; received flow joins the excess of my border voxel
// and the residual of my arc towards the ghost (it is the reverse of the arc the flow arrived on)
template <typename T>
__global__ void k_slab_unpack(unsigned plane, int* __restrict__ height_ghost, T* __restrict__ excess_border,
                              T* __restrict__ cap_border_to_ghost, const int* __restrict__ h_in,
                              const double* __restrict__ f_in, int* __restrict__ changed)
{
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= plane) return;
    int hn = h_in[i];
    if (height_ghost[i] != hn) { height_ghost[i] = hn; if (changed) *changed = 1; }
    double f = f_in ? f_in[i] : 0.0;
    if (f > 0) {
        excess_border[i] += (T)f;
        cap_border_to_ghost[i] += (T)f;
    }
}

// ---------------------------------------------------------------------------------------------------
// debug-mode invariants (MEDPY_GC_DEBUG=1; SURVEY.md §5.2): out[0] += excess, out[1] += flow absorbed by the sink links,
// out[2] += violations of: excess >= 0, every residual capacity >= 0, absorbed flow within [0, sink capacity], and (tile
// solver, CHECK_RMASK) every residual-mask bit equal to "capacity > 0".  Flow conservation is checked by the host:
// sum(excess) + sum(absorbed) must equal the clamped source excess the solve started from.
// ---------------------------------------------------------------------------------------------------
template <int ND, typename T, bool CHECK_RMASK>
__global__ void __launch_bounds__(256) k_debug_invariants(Lattice L, State<T> S, double* __restrict__ out)
{
    const unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0, a = 0.0;
    unsigned long long bad = 0;
    if (v < L.n && owned(L, v)) {
        e = (double)S.excess[v];
        if (!(e >= 0.0)) bad++;
        const double tr = (double)S.tr[v];
        const unsigned m = S.rmask[v];
        const bool lazy = CHECK_RMASK;      // 3-D tile solver: sink[] valid only where bit 7 of rmask is set
        if (tr < 0) {
            a = (!lazy || (m & 0x80u)) ? (double)S.sink[v] : 0.0;
            if (!(a >= 0.0) || a > -tr) bad++;
            if (CHECK_RMASK && (((m & 0x40u) != 0) != ((-tr) - a > 0))) bad++;
        }
#pragma unroll
        for (int k = 0; k < 2 * ND; ++k) {
            const double c = (double)S.cap[k][v];
            if (c < 0.0) bad++;
            if (CHECK_RMASK && (((m >> k) & 1u) != (c > 0 ? 1u : 0u))) bad++;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        e += __shfl_down_sync(0xffffffffu, e, o);
        a += __shfl_down_sync(0xffffffffu, a, o);
        bad += __shfl_down_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (e != 0.0) atomicAdd(out, e);
        if (a != 0.0) atomicAdd(out + 1, a);
        if (bad) atomicAdd(out + 2, (double)bad);
    }
}
