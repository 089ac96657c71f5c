// gc_host.hpp -- host helpers shared by the lattice units (gc_handle.cuh) and the sparse unit (gc_sparse_api.cu).
#pragma once
#include "../../include/medpy_b200_graphcut.h"

#include <cuda_runtime.h>

#include <map>
#include <mutex>
#include <string>

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
