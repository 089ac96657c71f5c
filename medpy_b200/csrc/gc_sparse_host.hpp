// gc_sparse_host.hpp -- what a general sparse graph (mgc_sparse, gc_sparse_api.cu) keeps on the host, and the rules
// that decide it: the arc pairs in insertion order with accumulated capacities (graph.h:427-480), tr_cap and the flow
// constant of add_tweights (graph.h:415-425), the CSR the device solves, and for a warm handle each pair's node-local arc
// offsets.  These are O(1) updates per call exactly like the reference's.  Plain C++17 with no CUDA: the emulators in
// tests/emu/ compile it with g++ and so run the very host steps of the C ABI.
#pragma once
#include <cstdint>
#include <unordered_map>
#include <vector>

// calls resolved to pairs: pair index, ends lo < hi, capacities oriented lo->hi / hi->lo and, once the arc offsets are
// recorded, the pair's offsets
struct SparseCalls {
    std::vector<unsigned> pk;
    std::vector<int32_t> lo, hi, olo, ohi;
    std::vector<double> c_lh, c_hl;
};

struct SparseHost {
    int64_t n = 0;
    std::vector<double> tr;                            // net terminal capacity per node
    double flow_const = 0.0;                           // sum of the add_tweights minima (graph.h:423)
    std::vector<int32_t> plo, phi;                     // node pairs in insertion order, lo < hi
    std::vector<double> cap_lh, cap_hl;                // capacity lo->hi, hi->lo
    std::unordered_map<uint64_t, int64_t> pair_of;     // key() -> index into the pair arrays (built on demand)
    bool indexed = true;                               // pair_of covers every pair
    std::vector<int32_t> olo, ohi;                     // per pair: node-local offsets of its arcs lo->hi and hi->lo
    std::vector<int32_t> deg;                          // arcs per node; empty while no offsets are recorded
    bool log_const = false;                            // keep every add_tweights call's node and constant (segment energies)
    std::vector<int32_t> const_node;
    std::vector<double> const_part;

    explicit SparseHost(int64_t nodes = 0) : n(nodes), tr((size_t)nodes, 0.0) {}

    static uint64_t key(int32_t lo, int32_t hi) { return ((uint64_t)(uint32_t)lo << 32) | (uint32_t)hi; }

    void ensure_index()
    {
        if (indexed) return;
        pair_of.clear();
        pair_of.reserve(plo.size() * 2);
        for (size_t p = 0; p < plo.size(); ++p) pair_of.emplace(key(plo[p], phi[p]), (int64_t)p);
        indexed = true;
    }

    // index of the pair (lo, hi), or -1; the index must be built
    int64_t find(int32_t lo, int32_t hi) const
    {
        auto it = pair_of.find(key(lo, hi));
        return it == pair_of.end() ? -1 : it->second;
    }

    // a new pair (lo, hi) with capacities (a, b); its arcs come last in both nodes' lists
    int64_t append(int32_t lo, int32_t hi, double a, double b)
    {
        const int64_t p = (int64_t)plo.size();
        pair_of.emplace(key(lo, hi), p);
        plo.push_back(lo); phi.push_back(hi);
        cap_lh.push_back(a); cap_hl.push_back(b);
        if (!deg.empty()) { olo.push_back(deg[(size_t)lo]++); ohi.push_back(deg[(size_t)hi]++); }
        return p;
    }

    // sum_edge calls on a graph that is not resident on the device
    void sum_edges(int64_t count, const int32_t* i, const int32_t* j, const double* cap, const double* rev)
    {
        // A batch of distinct pairs in strictly increasing (i, j) order with i < j -- what the region adjacency
        // reduction delivers (mgc_labels_fetch_edges) -- landing in an empty graph needs no look-ups: append, index
        // later if ever needed.
        if (plo.empty() && count > 0) {
            bool sorted_unique = true;
            uint64_t prev = 0;
            for (int64_t k = 0; k < count && sorted_unique; ++k) {
                const uint64_t kk = key(i[k], j[k]);
                sorted_unique = i[k] < j[k] && (k == 0 || kk > prev);
                prev = kk;
            }
            if (sorted_unique) {
                plo.assign(i, i + count);
                phi.assign(j, j + count);
                cap_lh.assign(cap, cap + count);
                cap_hl.assign(rev, rev + count);
                pair_of.clear();
                indexed = false;
                return;
            }
        }
        ensure_index();
        for (int64_t k = 0; k < count; ++k) {
            const bool fwd = i[k] < j[k];
            const int32_t lo = fwd ? i[k] : j[k], hi = fwd ? j[k] : i[k];
            const double a = fwd ? cap[k] : rev[k], b = fwd ? rev[k] : cap[k];
            const int64_t p = find(lo, hi);
            if (p < 0) {
                append(lo, hi, a, b);                    // add_edge: r_cap = cap (graph.h:449-450)
            } else {
                cap_lh[(size_t)p] += a;                  // sum_edge: r_cap += cap (graph.h:472-476)
                cap_hl[(size_t)p] += b;
            }
        }
    }

    // Resolves the calls to pairs into `c`.  A missing pair is created at capacity 0 when `create` (the caller adds the
    // calls' capacities); otherwise it is refused and the index of its call returned.  -1: every call resolved.
    int64_t resolve(int64_t count, const int32_t* i, const int32_t* j, const double* cap, const double* rev, bool create,
                    SparseCalls& c)
    {
        ensure_index();
        const size_t m = (size_t)count;
        c.pk.resize(m); c.lo.resize(m); c.hi.resize(m); c.c_lh.resize(m); c.c_hl.resize(m);
        c.olo.resize(deg.empty() ? 0 : m); c.ohi.resize(deg.empty() ? 0 : m);
        for (int64_t k = 0; k < count; ++k) {
            const bool fwd = i[k] < j[k];
            const int32_t a = fwd ? i[k] : j[k], b = fwd ? j[k] : i[k];
            int64_t p = find(a, b);
            if (p < 0) {
                if (!create) return k;
                p = append(a, b, 0.0, 0.0);
            }
            c.pk[(size_t)k] = (unsigned)p;
            c.lo[(size_t)k] = a; c.hi[(size_t)k] = b;
            c.c_lh[(size_t)k] = fwd ? cap[k] : rev[k];
            c.c_hl[(size_t)k] = fwd ? rev[k] : cap[k];
            if (!deg.empty()) { c.olo[(size_t)k] = olo[(size_t)p]; c.ohi[(size_t)k] = ohi[(size_t)p]; }
        }
        return -1;
    }

    // the resolved calls' capacities added to their pairs in call order (a new pair starts at 0: add_edge's r_cap = cap)
    void add(const SparseCalls& c)
    {
        for (size_t k = 0; k < c.pk.size(); ++k) {
            cap_lh[c.pk[k]] += c.c_lh[k];
            cap_hl[c.pk[k]] += c.c_hl[k];
        }
    }

    // per pair of the resolved calls: their capacities summed in call order, pairs in order of their first call
    static void pair_sums(const SparseCalls& c, std::vector<unsigned>& pairs, std::vector<double>& sl, std::vector<double>& sh)
    {
        std::unordered_map<unsigned, size_t> slot;
        for (size_t k = 0; k < c.pk.size(); ++k) {
            auto ins = slot.emplace(c.pk[k], pairs.size());
            if (ins.second) { pairs.push_back(c.pk[k]); sl.push_back(0.0); sh.push_back(0.0); }
            sl[ins.first->second] += c.c_lh[k];
            sh[ins.first->second] += c.c_hl[k];
        }
    }

    // the pairs lowered by the sums of pair_sums(), clamped at 0
    void lower(const std::vector<unsigned>& pairs, const std::vector<double>& sl, const std::vector<double>& sh)
    {
        for (size_t q = 0; q < pairs.size(); ++q) {
            const size_t p = pairs[q];
            const double a = cap_lh[p] - sl[q], b = cap_hl[p] - sh[q];
            cap_lh[p] = a < 0 ? 0.0 : a;
            cap_hl[p] = b < 0 ? 0.0 : b;
        }
    }

    // BK's add_tweights (graph.h:415-424), call by call; nodes null: call k is node k
    void add_tweights(int64_t count, const int32_t* nodes, const double* src, const double* snk)
    {
        for (int64_t k = 0; k < count; ++k) {
            const size_t v = (size_t)(nodes ? nodes[k] : k);
            double s = src[k], t = snk[k];
            const double delta = tr[v];
            if (delta > 0) s += delta; else t -= delta;
            const double part = (s < t) ? s : t;
            flow_const += part;
            tr[v] = s - t;
            if (log_const) { const_node.push_back((int32_t)v); const_part.push_back(part); }
        }
    }

    // CSR in insertion order of the pairs (the order add_edge appends arcs to a node's list, graph.h:443-452)
    void csr(std::vector<int>& row, std::vector<int>& head, std::vector<int>& sis, std::vector<double>& cap) const
    {
        const size_t np = plo.size();
        row.assign((size_t)n + 1, 0);
        head.resize(2 * np); sis.resize(2 * np); cap.resize(2 * np);
        for (size_t p = 0; p < np; ++p) { row[(size_t)plo[p] + 1]++; row[(size_t)phi[p] + 1]++; }
        for (int64_t v = 0; v < n; ++v) row[(size_t)v + 1] += row[(size_t)v];
        std::vector<int> fill(row.begin(), row.end() - 1);
        for (size_t p = 0; p < np; ++p) {
            const int a = fill[(size_t)plo[p]]++, b = fill[(size_t)phi[p]]++;
            head[(size_t)a] = phi[p]; head[(size_t)b] = plo[p];
            sis[(size_t)a] = b; sis[(size_t)b] = a;
            cap[(size_t)a] = cap_lh[p]; cap[(size_t)b] = cap_hl[p];
        }
    }

    // each pair's arc offsets in the CSR of csr(); from here on new pairs get theirs as they are appended
    void record_offsets()
    {
        deg.assign((size_t)n, 0);
        olo.resize(plo.size());
        ohi.resize(plo.size());
        for (size_t p = 0; p < plo.size(); ++p) {
            olo[p] = deg[(size_t)plo[p]]++;
            ohi[p] = deg[(size_t)phi[p]]++;
        }
    }
};
