// gc_common.cuh -- shared device-side types for the H100 voxel graph-cut path.
//
// Data layout in HBM (structure of arrays over the C-order flat voxel index v, see DESIGN.md §3):
//   cap[k][v]   residual capacity of the arc leaving v in direction k = 2*axis + (0: -1, 1: +1)
//               (the implicit lattice replaces the reference's 48 B node / 32 B arc objects,
//               lib/maxflow/src/graph.h:283-318); arcs that would leave the lattice hold 0 forever
//   tr[v]       net terminal capacity exactly as Graph::add_tweights leaves it (graph.h:415-425)
//   excess[v]   preflow excess;  sink[v] residual capacity v -> sink
//   height[v]   push-relabel label (int32), HINF = cannot reach the sink
//   rmask[v]    bit k set iff cap[k][v] > 0 (snapshot used by the global relabel)
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#define MGC_HINF 0x3fffffff
#define MGC_MAXDIR 8
// The source link of a voxel is clamped to what can leave it: sum of its out-capacities (rounded up) times this slack.
// The slack matters: the excess is consumed by a SEQUENCE of rounded subtractions (one per saturated arc, in whatever
// order the solver visits them), and without head-room the last arc can be left with a one-ulp residual that keeps
// the voxel "connected to the sink" although every arc is saturated in exact arithmetic (found by the full-size 512^3
// comparison against BK: 1 voxel of 134 M, tools/compare_fullsize.py).  Any factor > 1 + a few ulp is correct.
#define SOURCE_CLAMP_SLACK 1.0000001

struct Lattice {
    int nd;                 // canonical number of axes: 3 or 4
    int dim[4];             // extents, axis 0 slowest
    unsigned stride[4];     // element strides (C order)
    unsigned long long magic[4];  // ceil(2^64 / stride[d]) (0 when stride[d] == 1): exact u32 division by multiply-high
    unsigned n;             // voxels in the local lattice (< 2^31)
    unsigned plane;         // voxels per axis-0 plane
    int own0, own1;         // owned axis-0 planes [own0, own1): all of them unless this is a z-slab
    int zper;               // batch of images stacked along axis 0: planes per image (0: one image, DESIGN.md §3.1)
    unsigned long long zmagic;    // ceil(2^64 / zper) (0 when zper <= 1), as magic[]
};

template <typename T>
struct State {
    T* cap[MGC_MAXDIR];
    T* excess;
    T* sink;
    T* tr;
    int* height;
    uint8_t* rmask;
};

// floor(v / stride[d]) for v < 2^32 without a hardware divide: v * ceil(2^64/d) >> 64 is exact for 32-bit v
__device__ __forceinline__ unsigned div_stride(const Lattice& L, unsigned v, int d)
{
    const unsigned long long m = L.magic[d];
    return m ? (unsigned)__umul64hi((unsigned long long)v, m) : v;
}

template <int ND>
__device__ __forceinline__ void decode(const Lattice& L, unsigned v, int (&c)[ND])
{
    unsigned r = v;
#pragma unroll
    for (int d = 0; d < ND - 1; ++d) {
        unsigned q = div_stride(L, r, d);
        c[d] = (int)q;
        r -= q * L.stride[d];
    }
    c[ND - 1] = (int)r;
}

// signed element offset of direction k
__device__ __forceinline__ int dir_offset(const Lattice& L, int k)
{
    int s = (int)L.stride[k >> 1];
    return (k & 1) ? s : -s;
}

// the image of plane gz >= 0 of a batch lattice (0 on a lattice of one image)
__device__ __forceinline__ int image_of(const Lattice& L, int gz)
{
    if (!L.zper) return 0;
    return L.zmagic ? (int)__umul64hi((unsigned long long)(unsigned)gz, L.zmagic) : gz;
}

// The axis-0 pairs of a voxel in plane gz >= 0 (bit 0: the pair with plane gz - 1, bit 1: with plane gz + 1): inside the
// lattice and, in a batch, not across the seam between two images.  Every place that forms axis-0 validity calls this;
// on a lattice of one image it is the extent test alone.
__device__ __forceinline__ unsigned z_pairs(const Lattice& L, int gz)
{
    unsigned b = (gz > 0 ? 1u : 0u) | (gz + 1 < L.dim[0] ? 2u : 0u);
    if (L.zper) {
        const int r = gz - image_of(L, gz) * L.zper;
        if (r == 0) b &= ~1u;
        if (r == L.zper - 1) b &= ~2u;
    }
    return b;
}

__device__ __forceinline__ bool owned(const Lattice& L, unsigned v)
{
    int p = (int)div_stride(L, v, 0);   // plane == stride[0]
    return p >= L.own0 && p < L.own1;
}
