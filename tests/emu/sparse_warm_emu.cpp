// tests/emu/sparse_warm_emu.cpp -- TEST INFRASTRUCTURE.
// Runs the per-node fold bodies of medpy_b200/csrc/gc_sparse_warm.cuh (the functions the warm CUDA kernels wrap) and
// the solver bodies of gc_sparse.cuh on the host, one node after the other, with the host steps of gc_sparse_api.cu
// (pair resolution, grouping by a stable sort, CSR re-assembly, fixed-order visits) restated sequentially.  It checks
// the LOGIC of solve -> fold -> continue where no GPU is available; races and launch code are only exercised by the
// `-m gpu` tests.
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <unordered_map>
#include <vector>

#include "../../medpy_b200/csrc/gc_sparse_warm.cuh"

namespace {

struct Emu {
    int n = 0;
    std::vector<int> row, head, sis, height, deg;
    std::vector<double> cap, tr, excess, sunk, sent;
    std::vector<int> plo, phi, olo, ohi;
    std::unordered_map<uint64_t, int> pair_of;
    double wconst = 0.0;

    SparseState state()
    {
        SparseState S{};
        S.n = n; S.m2 = (int)cap.size(); S.row = row.data(); S.head = head.data(); S.sis = sis.data(); S.cap = cap.data();
        S.tr = tr.data(); S.excess = excess.data(); S.sunk = sunk.data(); S.height = height.data();
        return S;
    }
    SparseWarm view()
    {
        SparseWarm W{};
        W.n = n; W.row = row.data(); W.head = head.data(); W.cap = cap.data(); W.tr = tr.data(); W.excess = excess.data();
        W.sunk = sunk.data(); W.sent = sent.data();
        return W;
    }
    static uint64_t key(int a, int b) { return ((uint64_t)(uint32_t)a << 32) | (uint32_t)b; }
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

// unique pairs lo < hi in insertion order with their capacities, net terminal capacities and the add_tweights constant
void* emu_warm_create(int n, long long np, const int* lo, const int* hi, const double* c_lh, const double* c_hl,
                      const double* tr, double flow_const)
{
    Emu* e = new Emu();
    e->n = n;
    e->row.assign((size_t)n + 1, 0);
    e->deg.assign((size_t)n, 0);
    for (long long p = 0; p < np; ++p) {
        e->plo.push_back(lo[p]); e->phi.push_back(hi[p]);
        e->pair_of[Emu::key(lo[p], hi[p])] = (int)p;
        e->olo.push_back(e->deg[(size_t)lo[p]]++);
        e->ohi.push_back(e->deg[(size_t)hi[p]]++);
    }
    for (int v = 0; v < n; ++v) e->row[(size_t)v + 1] = e->row[(size_t)v] + e->deg[(size_t)v];
    e->head.assign(2 * (size_t)np, 0); e->sis.assign(2 * (size_t)np, 0); e->cap.assign(2 * (size_t)np, 0.0);
    for (long long p = 0; p < np; ++p) {
        const int a = e->row[(size_t)lo[p]] + e->olo[(size_t)p], b = e->row[(size_t)hi[p]] + e->ohi[(size_t)p];
        e->head[(size_t)a] = hi[p]; e->head[(size_t)b] = lo[p];
        e->sis[(size_t)a] = b; e->sis[(size_t)b] = a;
        e->cap[(size_t)a] = c_lh[p]; e->cap[(size_t)b] = c_hl[p];
    }
    e->tr.assign(tr, tr + n);
    e->excess.assign((size_t)n, 0.0); e->sunk.assign((size_t)n, 0.0); e->sent.assign((size_t)n, 0.0);
    e->height.assign((size_t)n, 0);
    SparseWarm W = e->view();
    for (int u = 0; u < n; ++u) spw_init_node(W, u);   // k_spw_init
    e->wconst = flow_const;
    return e;
}

void emu_warm_destroy(void* h) { delete (Emu*)h; }

// the loop of sparse_loop: exact relabel, stop test, push sweeps; energy = constant + absorbed flow
int emu_warm_solve(void* h, int push_steps, int sweeps, uint8_t* mask, double* energy)
{
    Emu* e = (Emu*)h;
    SparseState S = e->state();
    const int n = e->n;
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

// add_tweights calls (mgc_sparse_add_tweights on a resident warm handle)
void emu_warm_tweights(void* h, long long m, const int* nodes, const double* src, const double* snk)
{
    Emu* e = (Emu*)h;
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

// nonnegative sum_edge calls on any pairs (mgc_sparse_sum_edges on a resident warm handle)
void emu_warm_edges(void* h, long long m, const int* i, const int* j, const double* cap, const double* rev)
{
    Emu* e = (Emu*)h;
    const int n = e->n;
    const size_t first_fresh = e->plo.size();
    std::vector<unsigned> pk((size_t)m);
    std::vector<double> c_lh((size_t)m), c_hl((size_t)m);
    for (long long k = 0; k < m; ++k) {
        const bool fwd = i[k] < j[k];
        const int a = fwd ? i[k] : j[k], b = fwd ? j[k] : i[k];
        auto it = e->pair_of.find(Emu::key(a, b));
        int p;
        if (it == e->pair_of.end()) {
            p = (int)e->plo.size();
            e->pair_of[Emu::key(a, b)] = p;
            e->plo.push_back(a); e->phi.push_back(b);
            e->olo.push_back(e->deg[(size_t)a]++); e->ohi.push_back(e->deg[(size_t)b]++);
        } else {
            p = it->second;
        }
        pk[(size_t)k] = (unsigned)p;
        c_lh[(size_t)k] = fwd ? cap[k] : rev[k];
        c_hl[(size_t)k] = fwd ? rev[k] : cap[k];
    }
    if (e->plo.size() > first_fresh) {
        std::vector<int> row((size_t)n + 1, 0), head(2 * e->plo.size()), sis(2 * e->plo.size());
        std::vector<double> capn(2 * e->plo.size());
        for (int v = 0; v < n; ++v) row[(size_t)v + 1] = row[(size_t)v] + e->deg[(size_t)v];
        for (int u = 0; u < n; ++u)
            spw_move_node(u, e->row.data(), e->head.data(), e->sis.data(), e->cap.data(), row.data(), head.data(), sis.data(), capn.data());
        for (size_t p = first_fresh; p < e->plo.size(); ++p)
            spw_new_pair(e->plo[p], e->phi[p], e->olo[p], e->ohi[p], row.data(), head.data(), sis.data(), capn.data());
        e->row.swap(row); e->head.swap(head); e->sis.swap(sis); e->cap.swap(capn);
    }
    const std::vector<unsigned> order = group(pk);
    std::vector<uint8_t> tail((size_t)n, 0);
    for (long long k = 0; k < m;) {
        const unsigned p = pk[order[(size_t)k]];
        long long end = k + 1;
        while (end < m && pk[order[(size_t)end]] == p) ++end;
        const int u = e->plo[p], v = e->phi[p];
        spw_pair_inc(e->cap.data(), e->row[(size_t)u] + e->olo[p], e->row[(size_t)v] + e->ohi[p], order.data(), k, end - k,
                     c_lh.data(), c_hl.data());
        for (long long q = k; q < end; ++q) {
            if (c_lh[order[(size_t)q]] > 0) tail[(size_t)u] = 1;
            if (c_hl[order[(size_t)q]] > 0) tail[(size_t)v] = 1;
        }
        k = end;
    }
    SparseWarm W = e->view();
    for (int u = 0; u < n; ++u)
        if (tail[(size_t)u]) spw_reclamp_node(W, u);
}

// nonnegative decrements on existing pairs (mgc_sparse_remove_edges_warm on a resident handle): 0 done, 1 refused
// (nothing changed), -1 a pair without an edge
int emu_warm_remove(void* h, long long m, const int* i, const int* j, const double* cap, const double* rev)
{
    Emu* e = (Emu*)h;
    std::vector<unsigned> pk((size_t)m);
    std::vector<double> d_lh((size_t)m), d_hl((size_t)m);
    for (long long k = 0; k < m; ++k) {
        const bool fwd = i[k] < j[k];
        const int a = fwd ? i[k] : j[k], b = fwd ? j[k] : i[k];
        auto it = e->pair_of.find(Emu::key(a, b));
        if (it == e->pair_of.end()) return -1;
        pk[(size_t)k] = (unsigned)it->second;
        d_lh[(size_t)k] = fwd ? cap[k] : rev[k];
        d_hl[(size_t)k] = fwd ? rev[k] : cap[k];
    }
    const std::vector<unsigned> order = group(pk);
    struct Item { unsigned p; double dl, dh; };
    std::vector<Item> items;
    for (long long k = 0; k < m;) {
        const unsigned p = pk[order[(size_t)k]];
        long long end = k + 1;
        double dl = 0.0, dh = 0.0;
        for (long long q = k; q < m && pk[order[(size_t)q]] == p; ++q, end = q) { dl += d_lh[order[(size_t)q]]; dh += d_hl[order[(size_t)q]]; }
        items.push_back({p, dl, dh});
        k = end;
    }
    for (const Item& it : items) {
        const int a = e->row[(size_t)e->plo[it.p]] + e->olo[it.p], b = e->row[(size_t)e->phi[it.p]] + e->ohi[it.p];
        if (spw_pair_refused(e->cap[(size_t)a], e->cap[(size_t)b], it.dl, it.dh)) return 1;
    }
    std::vector<unsigned> end_key;
    std::vector<double> end_dx;
    for (const Item& it : items) {
        const int u = e->plo[it.p], v = e->phi[it.p];
        double el, eh;
        spw_pair_dec(e->cap.data(), e->row[(size_t)u] + e->olo[it.p], e->row[(size_t)v] + e->ohi[it.p], it.dl, it.dh, &el, &eh);
        end_key.push_back((unsigned)u); end_dx.push_back(el);
        end_key.push_back((unsigned)v); end_dx.push_back(eh);
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
    return 0;
}

}  // extern "C"
