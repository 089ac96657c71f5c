// gc_sort.cuh -- the stable radix sort of the sparse and label units (cub::DeviceRadixSort, CUDA toolkit): scratch from
// the call's DevScope, the legacy default stream.
#pragma once
#include <type_traits>

#include <cub/device/device_radix_sort.cuh>

#include "gc_host.hpp"

// bits [0, end_bit) of `keys` sorted into `keys_sorted`, stably, carrying `vals` along into `vals_sorted` (V = void:
// the keys alone)
template <typename V = void, typename K, typename N>
cudaError_t radix_sort(DevScope& dev, K* keys, K* keys_sorted, N m, int end_bit, V* vals = nullptr, V* vals_sorted = nullptr)
{
    auto sort = [&](void* tmp, size_t& bytes) {
        if constexpr (std::is_void_v<V>)
            return cub::DeviceRadixSort::SortKeys(tmp, bytes, keys, keys_sorted, m, 0, end_bit, 0);
        else
            return cub::DeviceRadixSort::SortPairs(tmp, bytes, keys, keys_sorted, vals, vals_sorted, m, 0, end_bit, 0);
    };
    size_t bytes = 0;
    cudaError_t e = sort(nullptr, bytes);
    char* tmp = nullptr;
    if (e == cudaSuccess) e = dev.alloc(&tmp, bytes);
    return e == cudaSuccess ? sort(tmp, bytes) : e;
}
