// gc_sparse_held.hpp -- an internal interface of the sparse unit (gc_sparse_api.cu) for callers that write a graph's
// capacities and t-links on the device themselves (gc_region_expansion.cu).  Not part of the C ABI.
//
// sparse_hold allocates the handle's device arrays once for a CSR topology (row[n+1], head and sis per arc, n = the
// handle's node count) and keeps them until the next sparse_hold, mgc_sparse_reset or mgc_sparse_destroy.  The caller
// writes cap (per arc) and tr (per node, the net terminal capacity after add_tweights) through the returned pointers;
// sparse_solve_held then runs a cold solve of whatever they hold (k_sp_init, the push-relabel loop, the read-out) and
// returns the device mask (1 = not SINK).  `base` is the add_tweights constant of that state.  Both return an MGC_*
// status with the message in mgc_sparse_last_error.  Nothing else of the handle is meant to be used alongside.
#pragma once
#include <cstdint>
#include <vector>

#include "../../include/medpy_b200_graphcut.h"

struct SparseHeld {
    int n = 0, m2 = 0;
    const int* row = nullptr;
    const int* head = nullptr;
    double* cap = nullptr;
    double* tr = nullptr;
};

int sparse_hold(mgc_sparse* g, const std::vector<int>& row, const std::vector<int>& head, const std::vector<int>& sis,
                SparseHeld* out);
int sparse_solve_held(mgc_sparse* g, double base, double* energy, const uint8_t** mask);
