// tests/emu/sparse_warm_emu.cpp -- TEST INFRASTRUCTURE.
// A warm sparse handle on the host.  The calls go through the host state of the C ABI (medpy_b200/csrc/gc_sparse_host.hpp,
// the very code gc_sparse_api.cu runs: pair resolution, accumulation, add_tweights, the CSR of the first solve, arc
// offsets); the device steps run the per-node fold bodies of gc_sparse_warm.cuh (the functions the warm CUDA kernels
// wrap) and the solver bodies of gc_sparse.cuh one node after the other, with the grouping by a stable sort and the
// CSR re-assembly restated sequentially.  It checks the LOGIC of solve -> fold -> continue where no GPU is available;
// races and launch code are only exercised by the `-m gpu` tests.
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

#include "../../medpy_b200/csrc/gc_sparse_host.hpp"
#include "../../medpy_b200/csrc/gc_sparse_warm.cuh"

namespace {

struct Emu {
    SparseHost h;
    bool resident = false;                             // solved: the device state below is live and calls fold into it
    std::vector<int> row, head, sis, height;
    std::vector<double> cap, tr, excess, sunk, sent;
    double wconst = 0.0;

    SparseState state()
    {
        return SparseState{(int)h.n, (int)cap.size(), row.data(), head.data(), sis.data(), cap.data(), tr.data(),
                           excess.data(), sunk.data(), height.data()};
    }
    SparseWarm view()
    {
        return SparseWarm{(int)h.n, row.data(), head.data(), cap.data(), tr.data(), excess.data(), sunk.data(), sent.data()};
    }
    int arc(int v, int offset) const { return row[(size_t)v] + offset; }
};

// stable grouping: indices of `keys` in ascending key order, equal keys in call order
std::vector<unsigned> group(const std::vector<unsigned>& keys)
{
    std::vector<unsigned> order(keys.size());
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(), [&](unsigned a, unsigned b) { return keys[a] < keys[b]; });
    return order;
}

}  // namespace

extern "C" {

void* emu_warm_create(int n)
{
    Emu* e = new Emu();
    e->h = SparseHost(n);
    return e;
}

void emu_warm_destroy(void* h) { delete (Emu*)h; }

// the loop of sparse_loop: exact relabel, stop test, push sweeps; energy = constant + absorbed flow.  The first solve
// lays out the CSR and runs k_spw_init as sparse_first_solve does.
int emu_warm_solve(void* h, int push_steps, int sweeps, uint8_t* mask, double* energy)
{
    Emu* e = (Emu*)h;
    const int n = (int)e->h.n;
    if (!e->resident) {
        e->h.csr(e->row, e->head, e->sis, e->cap);
        e->tr = e->h.tr;
        e->excess.assign((size_t)n, 0.0); e->sunk.assign((size_t)n, 0.0); e->sent.assign((size_t)n, 0.0);
        e->height.assign((size_t)n, 0);
        SparseWarm W = e->view();
        for (int u = 0; u < n; ++u) spw_init_node(W, u);   // k_spw_init
        e->wconst = e->h.flow_const;
        e->h.record_offsets();
        e->resident = true;
    }
    SparseState S = e->state();
    for (long long rounds = 0;; ++rounds) {
        for (int u = 0; u < n; ++u) sp_relabel_init_node(S, u);
        for (;;) {
            bool changed = false;
            for (int u = 0; u < n; ++u) changed |= sp_relax_node(S, u);
            if (!changed) break;
        }
        long long active = 0;
        for (int u = 0; u < n; ++u) active += sp_is_active(S, u) ? 1 : 0;
        if (!active) break;
        if (rounds > 1000000) return -1;
        for (int s = 0; s < sweeps; ++s)
            for (int u = 0; u < n; ++u) sp_push_node(S, u, push_steps);
    }
    double a = 0.0;
    for (int u = 0; u < n; ++u) { mask[u] = S.height[u] >= SP_HINF ? 1 : 0; a += S.sunk[u]; }
    *energy = e->wconst + a;
    return 0;
}

// mgc_sparse_add_tweights: folded into a solved state, and always into the host state
void emu_warm_tweights(void* h, long long m, const int* nodes, const double* src, const double* snk)
{
    Emu* e = (Emu*)h;
    if (e->resident) {
        std::vector<unsigned> keys((size_t)m);
        for (long long k = 0; k < m; ++k) keys[(size_t)k] = (unsigned)nodes[k];
        const std::vector<unsigned> order = group(keys);
        SparseWarm W = e->view();
        double dk = 0.0;
        for (long long k = 0; k < m;) {
            const unsigned v = keys[order[(size_t)k]];
            long long end = k + 1;
            while (end < m && keys[order[(size_t)end]] == v) ++end;
            dk += spw_tlink_node(W, (int)v, order.data(), k, end - k, src, snk);
            k = end;
        }
        e->wconst += dk;
    }
    e->h.add_tweights(m, nodes, src, snk);
}

// mgc_sparse_sum_edges: accumulated on the host before the first solve; after it nonnegative calls on any pairs fold
void emu_warm_edges(void* h, long long m, const int* i, const int* j, const double* cap, const double* rev)
{
    Emu* e = (Emu*)h;
    if (!e->resident) {
        e->h.sum_edges(m, i, j, cap, rev);
        return;
    }
    const int n = (int)e->h.n;
    const size_t first_fresh = e->h.plo.size();
    SparseCalls c;
    e->h.resolve(m, i, j, cap, rev, true, c);
    e->h.add(c);
    const SparseHost& hs = e->h;
    if (hs.plo.size() > first_fresh) {
        std::vector<int> row((size_t)n + 1, 0), head(2 * hs.plo.size()), sis(2 * hs.plo.size());
        std::vector<double> capn(2 * hs.plo.size());
        for (int v = 0; v < n; ++v) row[(size_t)v + 1] = row[(size_t)v] + hs.deg[(size_t)v];
        for (int u = 0; u < n; ++u)
            spw_move_node(u, e->row.data(), e->head.data(), e->sis.data(), e->cap.data(), row.data(), head.data(), sis.data(), capn.data());
        for (size_t p = first_fresh; p < hs.plo.size(); ++p)
            spw_new_pair(hs.plo[p], hs.phi[p], hs.olo[p], hs.ohi[p], row.data(), head.data(), sis.data(), capn.data());
        e->row.swap(row); e->head.swap(head); e->sis.swap(sis); e->cap.swap(capn);
    }
    const std::vector<unsigned> order = group(c.pk);
    std::vector<uint8_t> tail((size_t)n, 0);
    for (long long k = 0; k < m;) {
        const size_t c0 = order[(size_t)k];
        long long end = k + 1;
        while (end < m && c.pk[order[(size_t)end]] == c.pk[c0]) ++end;
        spw_pair_inc(e->cap.data(), e->arc(c.lo[c0], c.olo[c0]), e->arc(c.hi[c0], c.ohi[c0]), order.data(), k, end - k,
                     c.c_lh.data(), c.c_hl.data());
        for (long long q = k; q < end; ++q) {
            if (c.c_lh[order[(size_t)q]] > 0) tail[(size_t)c.lo[c0]] = 1;
            if (c.c_hl[order[(size_t)q]] > 0) tail[(size_t)c.hi[c0]] = 1;
        }
        k = end;
    }
    SparseWarm W = e->view();
    for (int u = 0; u < n; ++u)
        if (tail[(size_t)u]) spw_reclamp_node(W, u);
}

// mgc_sparse_remove_edges_warm on a solved handle, nonnegative decrements on existing pairs: 0 done, 1 refused
// (nothing changed), -1 a pair without an edge
int emu_warm_remove(void* h, long long m, const int* i, const int* j, const double* cap, const double* rev)
{
    Emu* e = (Emu*)h;
    SparseCalls c;
    if (e->h.resolve(m, i, j, cap, rev, false, c) >= 0) return -1;
    const std::vector<unsigned> order = group(c.pk);
    struct Item { size_t c0; double dl, dh; };
    std::vector<Item> items;
    for (long long k = 0; k < m;) {
        const size_t c0 = order[(size_t)k];
        long long end = k;
        double dl = 0.0, dh = 0.0;
        for (; end < m && c.pk[order[(size_t)end]] == c.pk[c0]; ++end) { dl += c.c_lh[order[(size_t)end]]; dh += c.c_hl[order[(size_t)end]]; }
        items.push_back({c0, dl, dh});
        k = end;
    }
    for (const Item& it : items)
        if (spw_pair_refused(e->cap[(size_t)e->arc(c.lo[it.c0], c.olo[it.c0])], e->cap[(size_t)e->arc(c.hi[it.c0], c.ohi[it.c0])],
                             it.dl, it.dh))
            return 1;
    std::vector<unsigned> end_key;
    std::vector<double> end_dx;
    for (const Item& it : items) {
        double el, eh;
        spw_pair_dec(e->cap.data(), e->arc(c.lo[it.c0], c.olo[it.c0]), e->arc(c.hi[it.c0], c.ohi[it.c0]), it.dl, it.dh, &el, &eh);
        end_key.push_back((unsigned)c.lo[it.c0]); end_dx.push_back(el);
        end_key.push_back((unsigned)c.hi[it.c0]); end_dx.push_back(eh);
    }
    const std::vector<unsigned> eo = group(end_key);
    SparseWarm W = e->view();
    double dk = 0.0;
    for (size_t k = 0; k < eo.size();) {
        const unsigned v = end_key[eo[k]];
        double de = 0.0;
        size_t end = k;
        for (; end < eo.size() && end_key[eo[end]] == v; ++end) de += end_dx[eo[end]];
        dk += spw_excess_change(W, (int)v, de);
        k = end;
    }
    e->wconst += dk;
    std::vector<unsigned> pairs;
    std::vector<double> sl, sh;
    SparseHost::pair_sums(c, pairs, sl, sh);
    e->h.lower(pairs, sl, sh);
    return 0;
}

// the host state: returns the number of pairs; with arrays (sized for that many pairs, and n nodes) it fills the pairs
// in insertion order, tr and the flow constant
long long emu_warm_host(void* h, int* lo, int* hi, double* c_lh, double* c_hl, double* tr, double* flow_const)
{
    const SparseHost& s = ((Emu*)h)->h;
    if (lo) {
        std::copy(s.plo.begin(), s.plo.end(), lo);
        std::copy(s.phi.begin(), s.phi.end(), hi);
        std::copy(s.cap_lh.begin(), s.cap_lh.end(), c_lh);
        std::copy(s.cap_hl.begin(), s.cap_hl.end(), c_hl);
        std::copy(s.tr.begin(), s.tr.end(), tr);
        *flow_const = s.flow_const;
    }
    return (long long)s.plo.size();
}

}  // extern "C"
