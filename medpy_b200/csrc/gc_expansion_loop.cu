// gc_expansion_loop.cu -- the alpha-expansion loop of gc_expansion_loop.hpp.  Host code only: every kernel it launches
// is compiled into gc_expansion.cu or the unit that supplies the hook.
#include "gc_expansion_loop.hpp"

#include <algorithm>
#include <cmath>

namespace {
float elapsed(cudaEvent_t a, cudaEvent_t b)
{
    float ms = 0.0f;
    return cudaEventElapsedTime(&ms, a, b) == cudaSuccess ? ms : 0.0f;
}
}  // namespace

int expansion_check_labels(int K, std::string& err)
{
    if (K >= 2 && K <= 255) return MGC_OK;
    err = "the number of labels must be 2..255";
    return MGC_E_ARG;
}

int expansion_check_distance(const double* V, int K, std::string& err, bool semi_metric)
{
    const auto at = [&](int a, int b) { return V[(size_t)a * K + b]; };
    const auto pair = [](int a, int b) { return "V[" + std::to_string(a) + "][" + std::to_string(b) + "]"; };
    for (int a = 0; a < K; ++a)
        for (int b = 0; b < K; ++b)
            if (!std::isfinite(at(a, b)) || !(at(a, b) >= 0.0)) {
                err = "label_distance must be finite and >= 0, " + pair(a, b) + " is not";
                return MGC_E_ARG;
            }
    for (int a = 0; a < K; ++a)
        if (at(a, a) != 0.0) {
            err = "label_distance must have a zero diagonal, " + pair(a, a) + " is not 0";
            return MGC_E_ARG;
        }
    for (int a = 0; a < K; ++a)
        for (int b = a + 1; b < K; ++b)
            if (at(a, b) != at(b, a)) {
                err = "label_distance must be symmetric, " + pair(a, b) + " != " + pair(b, a);
                return MGC_E_ARG;
            }
    if (semi_metric) return MGC_OK;
    for (int a = 0; a < K; ++a)
        for (int b = 0; b < K; ++b)
            for (int c = 0; c < K; ++c)
                if (at(a, c) > at(a, b) + at(b, c)) {
                    err = "label_distance must satisfy the triangle inequality V[a][c] <= V[a][b] + V[b][c], (a, b, c) = (" +
                          std::to_string(a) + ", " + std::to_string(b) + ", " + std::to_string(c) +
                          ") breaks it; a semi-metric such as truncated quadratic needs alpha-beta swap moves";
                    return MGC_E_ARG;
                }
    return MGC_OK;
}

// In the members below `g` is the handle itself: the CK and FAIL macros of gc_host.hpp report into g->err.

Expansion::~Expansion()
{
    for (auto& e : ev) if (e) cudaEventDestroy(e);
}

void Expansion::apply(const uint8_t* mask, const ExpMove& m)
{
    if (m.beta < 0) exp_apply_launch(stream, blocks, n, mask, labels, m.alpha, d_switched);
    else            swap_apply_launch(stream, blocks, n, mask, labels, m.alpha, m.beta, d_switched);
}

int Expansion::setup()
{
    Expansion* const g = this;
    CK(cudaSetDevice(device));
    RC(alloc(n, (void**)&labels));
    RC(alloc((size_t)B * sizeof(unsigned long long), (void**)&d_switched));
    RC(alloc((size_t)B * sizeof(double), (void**)&d_energy));
    RC(alloc(sizeof(int), (void**)&d_bad));
    for (auto& e : ev) CK(cudaEventCreate(&e));
    return MGC_OK;
}

int Expansion::read_bad(int* bad)
{
    Expansion* const g = this;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    return MGC_OK;
}

int Expansion::set_cost(int label, const mgc_array* cost)
{
    Expansion* const g = this;
    if (!cost) return MGC_E_ARG;
    if (label < 0 || label >= K) FAIL(MGC_E_ARG, "label out of range");
    if (cost->dtype != MGC_F32 && cost->dtype != MGC_F64) FAIL(MGC_E_ARG, "costs must be float32 or float64");
    if (cost_dtype >= 0 && cost->dtype != cost_dtype) FAIL(MGC_E_ARG, "every cost plane must have the same dtype");
    cost_set[(size_t)label] = 0;
    ran = false;
    CK(cudaSetDevice(device));
    const size_t es = cost->dtype == MGC_F32 ? 4 : 8, bytes = (size_t)n * es;
    const void* p = nullptr;
    RC(stage(cost, es, "costs", &p));
    if (!costs) {
        const int rc = alloc((size_t)K * bytes, &costs);
        if (rc) { release(); return rc; }
        cost_dtype = cost->dtype;
    }
    void* dst = (char*)costs + (size_t)label * bytes;
    CK(cudaMemcpyAsync(dst, p, bytes, cudaMemcpyDefault, stream));
    release();
    CK(cudaMemsetAsync(d_bad, 0, sizeof(int), stream));
    exp_check_costs_launch(stream, blocks, n, cost_dtype, dst, d_bad);
    int bad = 0;
    RC(read_bad(&bad));
    if (bad) FAIL(MGC_E_ARG, "costs must be finite and >= 0");
    cost_set[(size_t)label] = 1;
    return MGC_OK;
}

// a uint8 label input staged into *dst (allocated on first use), refused (MGC_E_ARG) when an entry exceeds `limit`
int Expansion::set_u8(const mgc_array* a, uint8_t** dst, bool* have, int limit, const char* what)
{
    Expansion* const g = this;
    if (!a) return MGC_E_ARG;
    if (a->dtype != MGC_U8) FAIL(MGC_E_ARG, std::string(what) + " must be uint8");
    *have = false;
    ran = false;
    CK(cudaSetDevice(device));
    if (!*dst) RC(alloc(n, (void**)dst));
    const void* p = nullptr;
    RC(stage(a, 1, what, &p));
    CK(cudaMemcpyAsync(*dst, p, n, cudaMemcpyDefault, stream));
    release();
    CK(cudaMemsetAsync(d_bad, 0, sizeof(int), stream));
    exp_check_u8_launch(stream, blocks, n, *dst, limit, d_bad);
    int bad = 0;
    RC(read_bad(&bad));
    if (bad) FAIL(MGC_E_ARG, std::string(what) + " holds a value above " + std::to_string(limit));
    *have = true;
    return MGC_OK;
}

int Expansion::set_markers(const mgc_array* a) { return set_u8(a, &markers, &have_markers, K, "markers"); }

int Expansion::set_init(const mgc_array* a) { return set_u8(a, &init, &have_init, K - 1, "init"); }

int Expansion::set_moves(int kind)
{
    Expansion* const g = this;
    if (kind != MGC_MOVES_EXPANSION && kind != MGC_MOVES_SWAP)
        FAIL(MGC_E_ARG, "moves must be MGC_MOVES_EXPANSION (0) or MGC_MOVES_SWAP (1)");
    moves = kind;
    have_dist = false;
    ran = false;
    return MGC_OK;
}

int Expansion::set_label_distance(const double* host_V)
{
    Expansion* const g = this;
    have_dist = false;
    ran = false;
    if (!host_V) return MGC_OK;
    RC(expansion_check_distance(host_V, K, err, moves == MGC_MOVES_SWAP));
    CK(cudaSetDevice(device));
    const size_t bytes = (size_t)K * K * sizeof(double);
    if (!dist) RC(alloc(bytes, (void**)&dist));
    CK(cudaMemcpyAsync(dist, host_V, bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));      // the caller's matrix is borrowed for the call only
    have_dist = true;
    return MGC_OK;
}

int Expansion::run(int max_cycles)
{
    Expansion* const g = this;
    if (max_cycles < 1) FAIL(MGC_E_ARG, "max_cycles must be >= 1");
    for (int k = 0; k < K; ++k)
        if (!cost_set[(size_t)k]) FAIL(MGC_E_STATE, "the costs of label " + std::to_string(k) + " are not set");
    CK(cudaSetDevice(device));
    ran = false;
    st = mgc_expansion_stats{};
    per.assign((size_t)B, mgc_expansion_stats{});
    switched.clear();
    const bool check_init = have_init && have_markers;
    CK(cudaEventRecord(ev[4], stream));
    if (check_init) CK(cudaMemsetAsync(d_bad, 0, sizeof(int), stream));
    exp_init_launch(stream, blocks, n, K, cost_dtype, costs, have_markers ? markers : nullptr, have_init ? init : nullptr,
                    labels, d_bad);
    CK(cudaGetLastError());
    if (check_init) {
        int bad = 0;
        RC(read_bad(&bad));
        if (bad) FAIL(MGC_E_ARG, "init gives a marked voxel another label than its marker");
    }
    // the moves of one cycle: alpha = 0..K-1, or the pairs alpha < beta in lexicographic order
    std::vector<ExpMove> cycle_moves;
    for (int a = 0; a < K; ++a) {
        if (moves == MGC_MOVES_EXPANSION) cycle_moves.push_back({a, -1});
        else for (int b = a + 1; b < K; ++b) cycle_moves.push_back({a, b});
    }
    std::vector<uint8_t> active((size_t)B, 1);
    std::vector<unsigned long long> sw((size_t)B);
    std::vector<int64_t> changed((size_t)B);
    RC(freeze(active));
    int live = B;
    for (int cycle = 0; cycle < max_cycles && live; ++cycle) {
        std::fill(changed.begin(), changed.end(), 0);
        for (const ExpMove& m : cycle_moves) {
            RC(reset());
            CK(cudaEventRecord(ev[0], stream));
            RC(build(m));
            CK(cudaEventRecord(ev[1], stream));
            const uint8_t* mask = nullptr;
            RC(solve(&mask));
            CK(cudaEventRecord(ev[2], stream));
            CK(cudaMemsetAsync(d_switched, 0, (size_t)B * sizeof(unsigned long long), stream));
            apply(mask, m);
            CK(cudaGetLastError());
            CK(cudaEventRecord(ev[3], stream));
            CK(cudaMemcpyAsync(sw.data(), d_switched, (size_t)B * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                               stream));
            CK(cudaStreamSynchronize(stream));
            st.ms_build += elapsed(ev[0], ev[1]);
            st.ms_solve += elapsed(ev[1], ev[2]);
            st.ms_apply += elapsed(ev[2], ev[3]);
            for (int b = 0; b < B; ++b) {
                switched.push_back((int64_t)sw[(size_t)b]);
                changed[(size_t)b] += (int64_t)sw[(size_t)b];
            }
            st.moves++;
        }
        st.cycles++;
        // an image whose cycle switched nothing is at a fixed point: its own run stops here
        bool froze = false;
        for (int b = 0; b < B; ++b) {
            if (!active[(size_t)b]) continue;
            mgc_expansion_stats& s = per[(size_t)b];
            s.cycles++;
            s.moves += (int64_t)cycle_moves.size();
            if (!changed[(size_t)b]) { s.converged = 1; active[(size_t)b] = 0; --live; froze = true; }
        }
        if (froze && live) RC(freeze(active));
    }
    st.converged = live ? 0 : 1;
    RC(energy());
    CK(cudaGetLastError());
    CK(cudaEventRecord(ev[5], stream));
    std::vector<double> e((size_t)B);
    CK(cudaMemcpyAsync(e.data(), d_energy, (size_t)B * sizeof(double), cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    st.ms_total = elapsed(ev[4], ev[5]);
    for (int b = 0; b < B; ++b) {
        per[(size_t)b].energy = e[(size_t)b];
        st.energy += e[(size_t)b];          // in image order
    }
    ran = true;
    return MGC_OK;
}

int Expansion::get_labels(uint8_t* out, int mem)
{
    Expansion* const g = this;
    if (!out) return MGC_E_ARG;
    if (!ran) FAIL(MGC_E_STATE, std::string("call ") + abi + "_run first");
    CK(cudaSetDevice(device));
    CK(cudaMemcpyAsync(out, labels, n, mem == MGC_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    return MGC_OK;
}

int Expansion::get_stats(mgc_expansion_stats* out) const
{
    if (!out) return MGC_E_ARG;
    if (!ran) { err = std::string("call ") + abi + "_run first"; return MGC_E_STATE; }
    *out = st;
    return MGC_OK;
}

int Expansion::get_image_stats(mgc_expansion_stats* out) const
{
    if (!out) return MGC_E_ARG;
    if (!ran) { err = std::string("call ") + abi + "_run first"; return MGC_E_STATE; }
    std::copy(per.begin(), per.end(), out);
    return MGC_OK;
}

int Expansion::get_switched(int64_t* out) const
{
    if (!out) return MGC_E_ARG;
    if (!ran) { err = std::string("call ") + abi + "_run first"; return MGC_E_STATE; }
    std::copy(switched.begin(), switched.end(), out);
    return MGC_OK;
}
