// tests/emu/sparse_emu.cpp -- TEST INFRASTRUCTURE.
// Builds the graph of a raw call sequence through the host state of the C ABI (medpy_b200/csrc/gc_sparse_host.hpp, the
// very code gc_sparse_api.cu runs), then compiles the per-node bodies of medpy_b200/csrc/gc_sparse.cuh (the very
// functions the CUDA kernels wrap) as plain host C++ and drives them with the same round structure as the device loop in
// gc_sparse_api.cu (sparse_loop), one node after the other.  It checks the LOGIC of the sparse push-relabel where no GPU
// is available; races and launch code are only exercised by the `-m gpu` tests.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../medpy_b200/csrc/gc_sparse.cuh"
#include "../../medpy_b200/csrc/gc_sparse_host.hpp"

static int solve(int n, int m2, const int* row, const int* head, const int* sis, const double* cap_in, const double* tr,
                 int push_steps, int sweeps_per_round, uint8_t* mask_out, double* absorbed_out)
{
    std::vector<double> cap(cap_in, cap_in + m2), excess(n), sunk(n);
    std::vector<int> height(n);
    SparseState S{};
    S.n = n; S.m2 = m2; S.row = row; S.head = head; S.sis = sis; S.cap = cap.data(); S.tr = tr;
    S.excess = excess.data(); S.sunk = sunk.data(); S.height = height.data();
    for (int u = 0; u < n; ++u) sp_init_node(S, u);
    long long rounds = 0;
    for (;;) {
        for (int u = 0; u < n; ++u) sp_relabel_init_node(S, u);
        for (;;) {
            bool changed = false;
            for (int u = 0; u < n; ++u) changed |= sp_relax_node(S, u);
            if (!changed) break;
        }
        long long active = 0;
        for (int u = 0; u < n; ++u) active += sp_is_active(S, u) ? 1 : 0;
        if (!active) break;
        if (++rounds > 1000000) return -1;
        for (int s = 0; s < sweeps_per_round; ++s)
            for (int u = 0; u < n; ++u) sp_push_node(S, u, push_steps);
    }
    double a = 0.0;
    for (int u = 0; u < n; ++u) { mask_out[u] = height[u] >= SP_HINF ? 1 : 0; a += sunk[u]; }
    *absorbed_out = a;
    return 0;
}

// m sum_edge calls, then t add_tweights calls, as mgc_sparse_sum_edges / mgc_sparse_add_tweights take them, and the
// solve of the CSR the first maxflow() lays out.  Out: the pairs in insertion order (lo, hi, c_lh, c_hl, sized for m
// pairs), tr[n], the flow constant, mask[n] and the energy.  Returns the number of pairs, -1 when the loop stalls.
extern "C" long long emu_sparse_calls(int n, long long m, const int* i, const int* j, const double* cap, const double* rev,
                                      long long t, const int* nodes, const double* src, const double* snk, int push_steps,
                                      int sweeps_per_round, int* lo, int* hi, double* c_lh, double* c_hl, double* tr,
                                      double* flow_const, uint8_t* mask, double* energy)
{
    SparseHost h(n);
    h.sum_edges(m, i, j, cap, rev);
    h.add_tweights(t, nodes, src, snk);
    std::vector<int> row, head, sis;
    std::vector<double> c;
    h.csr(row, head, sis, c);
    double absorbed = 0.0;
    if (solve(n, (int)c.size(), row.data(), head.data(), sis.data(), c.data(), h.tr.data(), push_steps, sweeps_per_round,
              mask, &absorbed))
        return -1;
    std::copy(h.plo.begin(), h.plo.end(), lo);
    std::copy(h.phi.begin(), h.phi.end(), hi);
    std::copy(h.cap_lh.begin(), h.cap_lh.end(), c_lh);
    std::copy(h.cap_hl.begin(), h.cap_hl.end(), c_hl);
    std::copy(h.tr.begin(), h.tr.end(), tr);
    *flow_const = h.flow_const;
    *energy = h.flow_const + absorbed;
    return (long long)h.plo.size();
}
