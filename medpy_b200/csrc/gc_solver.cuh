// gc_solver.cuh -- per-voxel kernels around the lattice tile solver (gc_tiles.cuh, gc_tiles4.cuh): the read-out of
// mask and energy, the pack half of the z-slab border messages, and the debug-mode invariant checks.
//
// The solver (DESIGN.md §4) computes a maximum PREFLOW by push-relabel on the implicit lattice, with an exact backward
// BFS from the sink (global relabel) between rounds.  The min cut the reference reports is solver independent:
// what_segment(v) == SINK  <=>  v can still reach the sink in the residual graph (SURVEY.md §3.3), which is exactly
// "height[v] finite after an exact global relabel" of a maximum preflow -- the mask the read-out writes.  The stop
// test is only ever made right after such a relabel: no voxel with excess > 0 has a finite label.
#pragma once
#include "gc_common.cuh"

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
