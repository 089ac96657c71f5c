// gc_host.hpp -- host helpers shared by the lattice units (gc_handle.cuh), the sparse unit (gc_sparse_api.cu) and the
// label-image unit (gc_labels_api.cu).
#pragma once
#include "../../include/medpy_b200_graphcut.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

// Error returns of an entry point on a handle `g` with an `err` string.  CK clears the runtime's last error after a failed
// call, so that a later CK(cudaGetLastError()) does not report it against an unrelated launch.
#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            g->err = std::string(#call) + ": " + cudaGetErrorString(_e);                           \
            cudaGetLastError();                                                                    \
            return MGC_E_CUDA;                                                                     \
        }                                                                                          \
    } while (0)

#define FAIL(code, msg)                                                                            \
    do {                                                                                           \
        g->err = (msg);                                                                            \
        return (code);                                                                             \
    } while (0)

// pass on the nonzero status of a call that returns one
#define RC(call)                                                                                   \
    do {                                                                                           \
        int rc0 = (call);                                                                          \
        if (rc0) return rc0;                                                                       \
    } while (0)

// SMs of device `dev`, cached per device (132, an H100 SXM, when the runtime cannot tell)
inline int cached_sm_count(int dev)
{
    static std::mutex mu;
    static std::map<int, int> cache;
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(dev);
    if (it != cache.end()) return it->second;
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); n = 132; }
    cache[dev] = n;
    return n;
}

// number of bits needed to represent values in [0, v] (at least 1)
inline int bits_for(unsigned long long v)
{
    int b = 0;
    while (v) { ++b; v >>= 1; }
    return b ? b : 1;
}

// ---- the sparse and label units: synchronous calls on the legacy default stream, temporaries per call -----------------

// device allocations of one call, released together
struct DevScope {
    std::vector<void*> ptrs;
    ~DevScope() { for (void* p : ptrs) cudaFree(p); }
    template <typename T>
    cudaError_t alloc(T** out, size_t count)
    {
        void* p = nullptr;
        cudaError_t e = cudaMalloc(&p, (count ? count : 1) * sizeof(T));
        if (e == cudaSuccess) ptrs.push_back(p);
        *out = (T*)p;
        return e;
    }
    // `p`, allocated here, outlives the scope
    void keep(const void* p) { ptrs.erase(std::find(ptrs.begin(), ptrs.end(), p)); }
    // `p`, allocated here, and `held`, owned by the caller, trade places: the scope frees the old `held`
    template <typename T>
    void trade(T*& p, T*& held)
    {
        *std::find(ptrs.begin(), ptrs.end(), (void*)p) = held;
        std::swap(p, held);
    }
};

// grid of the grid-stride kernels (blocks of 256 threads): one block per 256 items, at most 32 blocks per SM of the
// current device
inline unsigned grid_for(long long n)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
    const long long cap = 32LL * cached_sm_count(dev);
    long long b = (n + 255) / 256;
    if (b < 1) b = 1;
    return (unsigned)(b < cap ? b : cap);
}

// kernels of gc_labels.cuh the sparse unit launches too, compiled into gc_labels_api.cu only
void lab_iota(unsigned* a, long long m);                                              // a[i] = i
void lab_scan_blocks(const unsigned* cnt, long long nb, unsigned long long* out);     // exclusive scan, out[nb] = total

// k_sum_partials, compiled into gc_api.cu only, on stream `s`: *out += the fixed-order sum of partials[0..n)
void sum_partials_on(cudaStream_t s, const double* partials, unsigned n, double* out);
