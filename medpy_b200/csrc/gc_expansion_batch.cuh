// gc_expansion_batch.cuh -- kernels of the batched alpha-expansion / alpha-beta swap unit (gc_expansion_batch.cu,
// DESIGN.md §11 "Batches", "Swap moves"): B images of one shape stacked along axis 0 of a batch lattice (B * Z, Y, X)
// with Lattice::zper = Z, every move one cut of the whole batch.  Launched by gc_expansion_batch.cu only; the initial
// labels and the range checks are the single unit's kernels (gc_expansion.cuh, through its host launchers), which run
// unchanged over the B * N voxels.
//
// A per-image flag active[b] freezes image b once a cycle of it switched nothing: its move graph is empty (every capacity
// and tr 0, no constant) and its labels stay as they are.
#pragma once
#include "gc_expansion_cost.cuh"

// k_exp_move over the batch lattice, for the images whose flag is set: the same exp_move_voxel, with the axis-0 pairs
// those inside the image (none across a seam, as z_pairs), so a voxel's t-link has the bits of the single image's run.
// The pair weights W.w[d] are 0 across the seams and on the last plane of every axis.
template <typename P, typename C>
__global__ void __launch_bounds__(256)
k_bexp_move(Lattice L, State<double> S, const C* __restrict__ costs, const uint8_t* __restrict__ markers,
            const uint8_t* __restrict__ labels, ExpWeights W, const uint8_t* __restrict__ active, int alpha,
            double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[3];
        decode<3>(L, v, c);
        const int img = image_of(L, c[0]);
        double tr = 0.0;
        if (active[img]) {
            c[0] -= img * L.zper;                   // the plane within the image: its axis-0 pairs stop at the seams
            m = __dadd_rn(m, exp_move_voxel<3>(L, S, costs, markers, labels, W, pair, alpha, v, c, L.zper, tr));
        } else {                                    // frozen: the empty graph
#pragma unroll
            for (int k = 0; k < 6; ++k) S.cap[k][v] = 0.0;
        }
        S.tr[v] = tr;
    }
    block_sum_store(m, partials);
}

// k_bexp_move's swap counterpart: swap_move_voxel of (alpha, beta) in the images whose flag is set, the empty graph in the
// frozen ones
template <typename P, typename C>
__global__ void __launch_bounds__(256)
k_bswap_move(Lattice L, State<double> S, const C* __restrict__ costs, const uint8_t* __restrict__ markers,
             const uint8_t* __restrict__ labels, ExpWeights W, const uint8_t* __restrict__ active, int alpha, int beta,
             double* __restrict__ partials, P pair)
{
    double m = 0.0;
    const unsigned step = gridDim.x * blockDim.x;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < L.n; v += step) {
        int c[3];
        decode<3>(L, v, c);
        const int img = image_of(L, c[0]);
        double tr = 0.0;
        if (active[img]) {
            c[0] -= img * L.zper;
            m = __dadd_rn(m, swap_move_voxel<3>(L, S, costs, markers, labels, W, pair, alpha, beta, v, c, L.zper, tr));
        } else {
#pragma unroll
            for (int k = 0; k < 6; ++k) S.cap[k][v] = 0.0;
        }
        S.tr[v] = tr;
    }
    block_sum_store(m, partials);
}

// The label update of a batch move, in active images only: relabel(v) updates voxel v by the move's rule and says whether
// its label changed; switched[b] += the voxels of image b that changed.  Each warp walks one contiguous range 32 voxels at
// a time and keeps the count of the image it is in; a step that spans two or more images (images of fewer than 32
// voxels, or a seam) adds per image with one atomic per image (integer atomics: the counts are exact).
template <typename F>
__device__ __forceinline__ void bexp_apply_body(const Lattice& L, const uint8_t* __restrict__ active,
                                                unsigned long long* __restrict__ switched, F relabel)
{
    const unsigned lane = threadIdx.x & 31u;
    const unsigned warps = (gridDim.x * blockDim.x) >> 5;
    const unsigned warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned per = ((L.n + warps - 1) / warps + 31u) & ~31u;
    const unsigned begin = warp * per;
    const unsigned end = begin + per < L.n ? begin + per : L.n;
    int cur = -1;                   // warp-uniform: the image `cnt` belongs to
    unsigned cnt = 0;
    for (unsigned base = begin; base < end; base += 32u) {
        const unsigned v = base + lane;
        int img = -1;
        bool did = false;
        if (v < end) {
            img = image_of(L, (int)div_stride(L, v, 0));
            did = active[img] && relabel(v);
        }
        const unsigned sw = __ballot_sync(0xffffffffu, did);
        if (!sw) continue;
        const int first = __shfl_sync(0xffffffffu, img, 0);
        const int last = __shfl_sync(0xffffffffu, img, 31);
        if (first == last) {            // one image (a full step: v < end in every lane)
            if (first != cur) {
                if (lane == 0 && cnt) atomicAdd(switched + cur, (unsigned long long)cnt);
                cur = first;
                cnt = 0;
            }
            cnt += __popc(sw);
        } else {
            if (lane == 0 && cnt) atomicAdd(switched + cur, (unsigned long long)cnt);
            cur = -1;
            cnt = 0;
            const unsigned peers = __match_any_sync(0xffffffffu, img);
            const unsigned c = __popc(sw & peers);
            if (img >= 0 && c && lane == (unsigned)(__ffs(peers) - 1)) atomicAdd(switched + img, (unsigned long long)c);
        }
    }
    if (lane == 0 && cnt) atomicAdd(switched + cur, (unsigned long long)cnt);
}

// labels <- alpha where the cut put the voxel on the SINK side (mask 0)
__global__ void __launch_bounds__(256)
k_bexp_apply(Lattice L, const uint8_t* __restrict__ mask, uint8_t* __restrict__ labels, const uint8_t* __restrict__ active,
             int alpha, unsigned long long* __restrict__ switched)
{
    bexp_apply_body(L, active, switched, [&](unsigned v) {
        if (mask[v] || labels[v] == alpha) return false;
        labels[v] = (uint8_t)alpha;
        return true;
    });
}

// labels of alpha or beta <- beta where the cut put the voxel on the SINK side (mask 0), alpha elsewhere
__global__ void __launch_bounds__(256)
k_bswap_apply(Lattice L, const uint8_t* __restrict__ mask, uint8_t* __restrict__ labels, const uint8_t* __restrict__ active,
              int alpha, int beta, unsigned long long* __restrict__ switched)
{
    bexp_apply_body(L, active, switched, [&](unsigned v) {
        const int l = labels[v];
        if (l != alpha && l != beta) return false;
        const int to = mask[v] ? alpha : beta;
        if (l == to) return false;
        labels[v] = (uint8_t)to;
        return true;
    });
}

// E(l) of every image in a fixed order: block b * chunks + c sums exp_energy_voxel (its axis-0 pairs none across a seam)
// over the voxels c * 256 + t of image b, stepping by chunks * 256, into partials[b * chunks + c]; batch_sum then adds
// each image's partials in a fixed tree.  The same labels give the same bits.
template <typename P, typename C>
__global__ void __launch_bounds__(256)
k_bexp_energy(Lattice L, const C* __restrict__ costs, const uint8_t* __restrict__ markers, const uint8_t* __restrict__ labels,
              ExpWeights W, unsigned chunks, double* __restrict__ partials, P pair)
{
    const unsigned per = (unsigned)L.zper * L.plane, base = (blockIdx.x / chunks) * per, ch = blockIdx.x % chunks;
    double m = 0.0;
    for (unsigned i = ch * blockDim.x + threadIdx.x; i < per; i += chunks * blockDim.x) {
        const unsigned v = base + i;
        int c[3];
        decode<3>(L, v, c);
        m = __dadd_rn(m, exp_energy_voxel<3>(L, costs, markers, labels, W, pair, v, c));
    }
    block_sum_store(m, partials);
}
