// gc_tma.cuh -- TMA (cp.async.bulk.tensor) staging for the tile discharge kernel.
//
// The seven float64 planes a push visit needs per tile (six residual capacities + excess: 7 x 8^3 x 8 B = 28 KB)
// are described to the hardware once per graph as rank-3 tensor maps with an 8x8x8 box; one elected thread per CTA
// then issues seven `cp.async.bulk.tensor.3d` copies per tile and the bytes land in shared memory while the
// mbarrier counts them (SASS: UTMALDG + SYNCS).  Because the persistent CTAs know their NEXT tile before they
// start working on the current one, the copy of tile i+1 is in flight while tile i iterates (two stages), which
// takes the global-load latency off the critical path of this latency-bound kernel.  Out-of-lattice parts of a
// border tile are zero-filled by the TMA unit, which is exactly "no arc" / "no excess".
// Requirements (checked on the host, else the plain-load kernel is used): extents along x even (global strides
// must be multiples of 16 B) and 16 B-aligned base pointers.
#pragma once
#include <cuda.h>
#include "gc_tiles.cuh"

#define TMA_PLANES 7
#define TMA_STAGE_BYTES (TMA_PLANES * TILE_VOX * 8)

struct PushMaps {
    CUtensorMap m[TMA_PLANES];   // [0..5] cap[k], [6] excess
};

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, unsigned long long* bar, int x, int y, int z)
{
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(dst)), "l"((unsigned long long)map), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar)) : "memory");
}

// issue the seven box copies of tile t into `stage` (called by ONE thread)
__device__ __forceinline__ void tma_issue_tile(const PushMaps& maps, const Tiles& TL, int t, double* stage, unsigned long long* bar)
{
    const int tx = t % TL.nt[2];
    const int r = t / TL.nt[2];
    const int ty = r % TL.nt[1], tz = r / TL.nt[1];
    mbar_expect_tx(bar, TMA_STAGE_BYTES);
#pragma unroll
    for (int p = 0; p < TMA_PLANES; ++p)
        tma_load_3d(stage + p * TILE_VOX, &maps.m[p], bar, tx * TILE, ty * TILE, tz * TILE);
}

// Same discharge as k_push_tile (gc_tiles.cuh) with the capacity/excess planes staged by TMA, double buffered.
// dynamic shared memory: 2 stages x 28 KB | s_out 24 KB | s_h 4 KB | 2 mbarriers | 2 slots
template <typename T>
__global__ void __launch_bounds__(TILE_VOX, 2)
k_push_tile_tma(Lattice L, Tiles TL, State<T> S, const __grid_constant__ PushMaps maps, int iters, int* __restrict__ pflag,
                WorkList cur, int* __restrict__ cursor, WorkList self_next, WorkList other_next, int labels_capped)
{
    extern __shared__ __align__(128) unsigned char smem[];
    double* stage0 = reinterpret_cast<double*>(smem);
    double* stage1 = stage0 + TMA_PLANES * TILE_VOX;
    T* s_out = reinterpret_cast<T*>(stage1 + TMA_PLANES * TILE_VOX);
    int* s_h = reinterpret_cast<int*>(s_out + 6 * TILE_VOX);
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(s_h + 1024);
    int* s_next = reinterpret_cast<int*>(bars + 2);

    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // first tile of this CTA
        const int i = atomicAdd(cursor, 1);
        const int t0 = (i < *(volatile int*)cur.count) ? cur.items[i] : -1;
        s_next[0] = t0;
        if (t0 >= 0) tma_issue_tile(maps, TL, t0, stage0, &bars[0]);
    }
    __syncthreads();
    int t = s_next[0];
    unsigned phase[2] = {0u, 0u};
    int buf = 0;
    while (t >= 0) {
        // claim the next tile and start its copy into the other stage before touching the current one
        if (tid == 0) {
            const int i = atomicAdd(cursor, 1);
            const int tn = (i < *(volatile int*)cur.count) ? cur.items[i] : -1;
            s_next[1] = tn;
            if (tn >= 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic reads of that stage are done
                tma_issue_tile(maps, TL, tn, buf ? stage0 : stage1, &bars[buf ^ 1]);
            }
        }
        mbar_wait(&bars[buf], phase[buf]);
        phase[buf] ^= 1u;
        const double* stg = buf ? stage1 : stage0;
        push_visit_staged<T>(L, TL, S, iters, pflag, self_next, other_next, t, s_out, s_h, stg, labels_capped != 0);
        __syncthreads();                 // stage `buf` and s_out/s_h are free again; s_next[1] is visible
        t = s_next[1];
        buf ^= 1;
        __syncthreads();
    }
}
