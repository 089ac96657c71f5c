// gc_slab.cu -- z-slab handles (gc_handle.cuh): stepping from the host (mgc_slab_*) and the whole distributed solve
// inside the library over NCCL point-to-point on the handle's stream.
#include "gc_handle.cuh"
#include "gc_slab_kernels.cuh"

#include <dlfcn.h>

#include <chrono>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>

namespace {
// ---- NCCL, bound at run time ------------------------------------------------------------------------------
// The library does not link libnccl: the first mgc_slab_comm_* call binds the copy that is already loaded in the
// process (torch's, when the host side is Python) or opens libnccl.so.2 itself.
struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*CommAbort)(ncclComm_t) = nullptr;
    ncclResult_t (*CommGetAsyncError)(ncclComm_t, ncclResult_t*) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    bool ok = false;
};

NcclApi& nccl_api()
{
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        bool all = true;
        auto bind = [&](auto& fn, const char* name) { fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name)); if (!fn) all = false; };
        bind(api.GetUniqueId, "ncclGetUniqueId"); bind(api.CommInitRank, "ncclCommInitRank"); bind(api.CommDestroy, "ncclCommDestroy");
        bind(api.CommAbort, "ncclCommAbort"); bind(api.CommGetAsyncError, "ncclCommGetAsyncError"); bind(api.GetErrorString, "ncclGetErrorString");
        bind(api.AllReduce, "ncclAllReduce"); bind(api.Send, "ncclSend"); bind(api.Recv, "ncclRecv");
        bind(api.GroupStart, "ncclGroupStart"); bind(api.GroupEnd, "ncclGroupEnd");
        api.ok = all;
    });
    return api;
}

#define NK(call)                                                                                   \
    do {                                                                                           \
        ncclResult_t _r = (call);                                                                  \
        if (_r != ncclSuccess) {                                                                   \
            g->err = std::string(#call) + ": " + nccl_api().GetErrorString(_r);                    \
            return MGC_E_CUDA;                                                                     \
        }                                                                                          \
    } while (0)
}  // namespace

void slab_comm_release(mgc_graph* g)
{
    if (g->comm && nccl_api().ok) nccl_api().CommDestroy(g->comm);
    g->comm = nullptr;
}

namespace {
// asynchronous NCCL errors (a peer that died, a network fault) surface here instead of as a hang: polled at every
// host-visible decision of the slab solve (SURVEY.md §5.3)
int slab_comm_poll(mgc_graph* g)
{
    if (!g->comm) return MGC_OK;
    ncclResult_t async = ncclSuccess;
    NK(nccl_api().CommGetAsyncError(g->comm, &async));
    if (async != ncclSuccess && async != ncclInProgress) {
        g->err = std::string("NCCL asynchronous error: ") + nccl_api().GetErrorString(async);
        nccl_api().CommAbort(g->comm);
        g->comm = nullptr;
        return MGC_E_CUDA;
    }
    return MGC_OK;
}

// phase spans of the slab solve: begin / end record an event pair on the stream; resolved once the solve is over
void phase_begin(mgc_graph* g, int kind)
{
    if (g->ph_used + 2 > g->ph_events.size()) { g->ph_events.resize(g->ph_used + 2, nullptr); }
    for (int i = 0; i < 2; ++i) if (!g->ph_events[g->ph_used + i]) cudaEventCreate(&g->ph_events[g->ph_used + i]);
    cudaEventRecord(g->ph_events[g->ph_used], g->stream);
    g->ph_kind.push_back(kind);
}
void phase_end(mgc_graph* g)
{
    cudaEventRecord(g->ph_events[g->ph_used + 1], g->stream);
    g->ph_used += 2;
}
void phase_resolve(mgc_graph* g)
{
    for (size_t i = 0; i + 1 < g->ph_used; i += 2) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, g->ph_events[i], g->ph_events[i + 1]) == cudaSuccess) g->slab_phase_ms[g->ph_kind[i / 2]] += ms;
    }
    g->ph_used = 0;
    g->ph_kind.clear();
}

// one border exchange: pack -> grouped send/recv with both neighbours -> unpack, all enqueued on the handle's stream
int slab_exchange(mgc_graph* g, long long* changed_dev, bool labels_only)
{
    Nvtx range("mgc:slab_exchange");
    phase_begin(g, 1);
    NcclApi& N = nccl_api();
    const unsigned P = g->L.plane;
    const unsigned nb = (P + 255u) / 256u;
    int32_t* h_send[2] = {(int32_t*)g->msg[0], (int32_t*)g->msg[1]};
    double* f_send[2] = {(double*)(g->msg[0] + g->msg_h_bytes), (double*)(g->msg[1] + g->msg_h_bytes)};
    const bool have[2] = {g->ghost_lo, g->ghost_hi};
    for (int side = 0; side < 2; ++side) {
        if (!have[side]) continue;
        const size_t border = side == 0 ? (size_t)g->L.own0 * P : (size_t)(g->L.own1 - 1) * P;
        const size_t ghost = side == 0 ? border - P : border + P;
        k_slab_pack<double><<<nb, 256, 0, g->stream>>>(P, g->S.height + border, g->S.excess + ghost, h_send[side], labels_only ? nullptr : f_send[side]);
        g->st.kernel_launches++;
    }
    CK(cudaGetLastError());
    // relabel rounds exchange labels only (4 B per border voxel); push exchanges add the parked flow (12 B per border voxel)
    const size_t bytes = labels_only ? g->msg_h_bytes : g->msg_bytes;
    if (g->comm_world > 1) {
        NK(N.GroupStart());
        if (have[0]) { NK(N.Send(g->msg[0], bytes, ncclUint8, g->comm_rank - 1, g->comm, g->stream)); NK(N.Recv(g->msg[2], bytes, ncclUint8, g->comm_rank - 1, g->comm, g->stream)); }
        if (have[1]) { NK(N.Send(g->msg[1], bytes, ncclUint8, g->comm_rank + 1, g->comm, g->stream)); NK(N.Recv(g->msg[3], bytes, ncclUint8, g->comm_rank + 1, g->comm, g->stream)); }
        NK(N.GroupEnd());
    }
    const int32_t* h_lo = have[0] ? (const int32_t*)g->msg[2] : nullptr;
    const double* f_lo = (have[0] && !labels_only) ? (const double*)(g->msg[2] + g->msg_h_bytes) : nullptr;
    const int32_t* h_hi = have[1] ? (const int32_t*)g->msg[3] : nullptr;
    const double* f_hi = (have[1] && !labels_only) ? (const double*)(g->msg[3] + g->msg_h_bytes) : nullptr;
    g->slab_exchanges++;
    const int rc_unpack = mgc_slab_unpack(g, h_lo, f_lo, h_hi, f_hi, (int32_t*)changed_dev);
    phase_end(g);
    return rc_unpack;
}
}  // namespace

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

// ---- z-slab stepping --------------------------------------------------------------------------------

int mgc_slab_plane_elems(const mgc_graph* g, int64_t* n)
{
    if (!g || !n) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    *n = (int64_t)g->L.plane;
    return MGC_OK;
}

int mgc_slab_begin(mgc_graph* g)
{
    if (!g) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    CK(cudaSetDevice(g->device));
    { int rc0 = check_pending(g); if (rc0) return rc0; }
    resolve_term_span(g);
    // MGC_OPT_WARM: the first solve records the residual source capacities before any push (the init of the per-term
    // builds, k_warm_convert after the fused build); a no-op once recorded, so a re-solve after a fold continues from
    // the state the fold left
    int rc = warm_prepare(g);
    if (rc) return rc;
    rc = materialise_zeros(g);
    if (rc) return rc;
    return g->state_init ? MGC_OK : init_tiles(g);
}

int mgc_slab_push(mgc_graph* g, int32_t n)
{
    if (!g || n < 0) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (!g->state_init) FAIL(MGC_E_STATE, "call mgc_slab_begin first");
    CK(cudaSetDevice(g->device));
    g->iters_now = g->tile_iters;
    return push_tiles(g, n);
}

int mgc_slab_pack(mgc_graph* g, int32_t* h_lo, double* f_lo, int32_t* h_hi, double* f_hi)
{
    if (!g) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    CK(cudaSetDevice(g->device));
    const unsigned P = g->L.plane;
    const unsigned nb = (P + 255u) / 256u;
    if (g->ghost_lo && h_lo) {
        const size_t border = (size_t)g->L.own0 * P, ghost = border - P;
        k_slab_pack<double><<<nb, 256, 0, g->stream>>>(P, g->S.height + border, g->S.excess + ghost, h_lo, f_lo);
        g->st.kernel_launches++;
    }
    if (g->ghost_hi && h_hi) {
        const size_t border = (size_t)(g->L.own1 - 1) * P, ghost = border + P;
        k_slab_pack<double><<<nb, 256, 0, g->stream>>>(P, g->S.height + border, g->S.excess + ghost, h_hi, f_hi);
        g->st.kernel_launches++;
    }
    CK(cudaGetLastError());
    return MGC_OK;
}

int mgc_slab_unpack(mgc_graph* g, const int32_t* h_lo, const double* f_lo, const int32_t* h_hi, const double* f_hi,
                    int32_t* changed_dev)
{
    if (!g) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    CK(cudaSetDevice(g->device));
    const unsigned P = g->L.plane;
    const unsigned nb = (P + 255u) / 256u;
    for (int side = 0; side < 2; ++side) {
        const bool have = side == 0 ? (g->ghost_lo && h_lo) : (g->ghost_hi && h_hi);
        if (!have) continue;
        const int zb = side == 0 ? g->L.own0 : g->L.own1 - 1;
        const int zg = side == 0 ? zb - 1 : zb + 1;
        const int k = side == 0 ? 0 : 1;     // my arc border -> ghost: axis 0, -1 (lo) or +1 (hi)
        const int32_t* hin = side == 0 ? h_lo : h_hi;
        const double* fin = side == 0 ? f_lo : f_hi;
        if (g->nd == 4)
            k_slab_unpack_tiles4<double><<<nb, 256, 0, g->stream>>>(g->L, g->TL4, g->S, zg, zb, k, hin, fin, g->rflag, rl(g, 0), rl(g, 1),
                                                                   g->d_tcount + CTL_RLCUR, g->pflag, pl(g, 0, g->pl_sel[0]),
                                                                   pl(g, 1, g->pl_sel[1]), changed_dev);
        else
            k_slab_unpack_tiles<double><<<nb, 256, 0, g->stream>>>(g->L, g->TL, g->S, zg, zb, k, hin, fin, g->rflag, rl(g, 0), rl(g, 1),
                                                                  g->d_tcount + CTL_RLCUR, g->pflag, pl(g, 0, g->pl_sel[0]),
                                                                  pl(g, 1, g->pl_sel[1]), changed_dev);
        g->st.kernel_launches++;
    }
    CK(cudaGetLastError());
    return MGC_OK;
}

int mgc_slab_relabel_begin(mgc_graph* g)
{
    if (!g) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (!g->state_init) FAIL(MGC_E_STATE, "call mgc_slab_begin first");
    CK(cudaSetDevice(g->device));
    g->st.global_relabels++;
    const int rc = relabel_tiles_begin(g);
    if (rc) return rc;
    // a neighbour may have pushed (with a stale ghost label) into a voxel this slab had labelled HINF, which can reach the
    // sink now: every tile with excess goes back on the push lists, the only tiles the stop test counts
    const int ntiles = g->nd == 4 ? g->TL4.ntiles : g->TL.ntiles;
    unsigned grid = (unsigned)g->n_ctas * 4u;
    if (grid > (unsigned)ntiles) grid = (unsigned)ntiles;
    if (g->nd == 4)
        k_slab_relist4<double><<<grid, T4_VOX, 0, g->stream>>>(g->L, g->TL4, g->S, g->pflag, pl(g, 0, g->pl_sel[0]), pl(g, 1, g->pl_sel[1]));
    else
        k_slab_relist<double><<<grid, TILE_VOX, 0, g->stream>>>(g->L, g->TL, g->S, g->pflag, pl(g, 0, g->pl_sel[0]), pl(g, 1, g->pl_sel[1]));
    g->st.kernel_launches++;
    CK(cudaGetLastError());
    return MGC_OK;
}

int mgc_slab_relabel_relax(mgc_graph* g, int32_t* changed_out)
{
    if (!g) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    CK(cudaSetDevice(g->device));
    int any = 0;
    const int rc = relabel_tiles_run(g, &any, changed_out != nullptr);
    if (rc) return rc;
    if (changed_out) *changed_out = any ? 1 : 0;
    return MGC_OK;
}

int mgc_slab_count_active(mgc_graph* g, int64_t* active_out)
{
    if (!g || !active_out) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    CK(cudaSetDevice(g->device));
    return count_active_tiles(g, active_out);
}

int mgc_slab_count_active_dev(mgc_graph* g, unsigned long long* count_dev)
{
    if (!g || !count_dev) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    CK(cudaSetDevice(g->device));
    return count_active_tiles_enqueue(g, count_dev);
}

int mgc_slab_finish(mgc_graph* g, double* energy_part)
{
    if (!g || !energy_part) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    CK(cudaSetDevice(g->device));
    int rc = readout(g, energy_part);
    if (rc) return rc;
    g->energy = *energy_part;
    g->st.energy = g->energy;
    g->solved = true;
    return MGC_OK;
}

// ---- z-slab solve inside the library: NCCL point-to-point on the handle's stream, one host decision per relabel round --

int mgc_slab_comm_unique_id(void* out128)
{
    if (!out128) return MGC_E_ARG;
    NcclApi& N = nccl_api();
    if (!N.ok) { g_create_error = "libnccl.so.2 could not be loaded"; return MGC_E_CUDA; }
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    if (N.GetUniqueId(&id) != ncclSuccess) { g_create_error = "ncclGetUniqueId failed"; return MGC_E_CUDA; }
    memcpy(out128, &id, sizeof(id));
    return MGC_OK;
}

int mgc_slab_comm_init(mgc_graph* g, int32_t rank, int32_t world, const void* unique_id128)
{
    if (!g || !unique_id128 || world < 1 || rank < 0 || rank >= world) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (!g->slab) FAIL(MGC_E_STATE, "not a z-slab handle");
    NcclApi& N = nccl_api();
    if (!N.ok) FAIL(MGC_E_CUDA, "libnccl.so.2 could not be loaded");
    CK(cudaSetDevice(g->device));
    if ((rank > 0) != g->ghost_lo || (rank < world - 1) != g->ghost_hi) FAIL(MGC_E_ARG, "rank / world do not match the slab's position");
    slab_comm_release(g);
    ncclUniqueId id;
    memcpy(&id, unique_id128, sizeof(id));
    NK(N.CommInitRank(&g->comm, world, id, rank));
    g->comm_rank = rank; g->comm_world = world;
    const size_t P = g->L.plane;
    g->msg_h_bytes = (P * 4 + 7) / 8 * 8;
    g->msg_bytes = g->msg_h_bytes + P * 8;
    void* p = nullptr;
    for (int i = 0; i < 4; ++i) if (!g->msg[i]) { int rc = alloc_buf(g, g->msg_bytes, &p); if (rc) return rc; g->msg[i] = (char*)p; CK(cudaMemsetAsync(p, 0, g->msg_bytes, g->stream)); }
    if (!g->d_stat) { int rc = alloc_buf(g, 64, &p); if (rc) return rc; g->d_stat = (long long*)p; }
    if (!g->d_esum) { int rc = alloc_buf(g, 64, &p); if (rc) return rc; g->d_esum = (double*)p; }
    if (!g->h_stat) { void* hp = nullptr; if (mgc_host_alloc(64, &hp) != MGC_OK) FAIL(MGC_E_NOMEM, "pinned host allocation failed"); g->h_stat = (long long*)hp; }
    return MGC_OK;
}

// The whole distributed solve (what medpy_b200/distributed.py sequenced from Python in round 1).  Distributed global
// relabel = local BFS to a fixed point <-> border-label exchange; two rounds + the active count are enqueued
// speculatively and checked with ONE all-reduce and ONE host synchronisation (valid iff round B changed nothing anywhere).
// Returns the TOTAL energy (all-reduced) in *energy_total.
int mgc_slab_solve(mgc_graph* g, double* energy_total)
{
    if (!g || !energy_total) return MGC_E_ARG;
    if (batch_refused(g)) return MGC_E_STATE;
    if (!g->slab || !g->comm) FAIL(MGC_E_STATE, "call mgc_slab_comm_init first");
    NcclApi& N = nccl_api();
    CK(cudaSetDevice(g->device));
    int rc = mgc_slab_begin(g);
    if (rc) return rc;
    g->slab_exchanges = g->slab_relabel_rounds = g->slab_push_passes = g->slab_global_relabels = 0;
    for (double& x : g->slab_phase_ms) x = 0.0;
    g->ph_used = 0; g->ph_kind.clear();
    auto timed_sync = [&]() -> cudaError_t {
        const auto t0 = std::chrono::steady_clock::now();
        const cudaError_t e = cudaStreamSynchronize(g->stream);
        g->slab_phase_ms[5] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        return e;
    };
    int passes = g->passes0 > 0 ? g->passes0 : 1;
    const int passes_cap = g->passes_max < 8 ? g->passes_max : 8;
    int64_t rounds = 0;
    for (;;) {
        phase_begin(g, 0);
        rc = mgc_slab_relabel_begin(g);
        phase_end(g);
        if (rc) return rc;
        for (;;) {
            CK(cudaMemsetAsync(g->d_stat, 0, 3 * sizeof(long long), g->stream));
            for (int k = 0; k < 2; ++k) {
                phase_begin(g, 0);
                rc = mgc_slab_relabel_relax(g, nullptr);
                phase_end(g);
                if (rc) return rc;
                rc = slab_exchange(g, g->d_stat + k, true);
                if (rc) return rc;
                g->slab_relabel_rounds++;
            }
            phase_begin(g, 2);
            rc = mgc_slab_count_active_dev(g, (unsigned long long*)(g->d_stat + 2));
            if (rc) return rc;
            if (g->comm_world > 1) NK(N.AllReduce(g->d_stat, g->d_stat, 3, ncclInt64, ncclSum, g->comm, g->stream));
            CK(cudaMemcpyAsync(g->h_stat, g->d_stat, 3 * sizeof(long long), cudaMemcpyDeviceToHost, g->stream));
            phase_end(g);
            CK(timed_sync());                                          // the one host decision of this round
            rc = slab_comm_poll(g);
            if (rc) return rc;
            if (g->h_stat[1] == 0) break;
        }
        g->slab_global_relabels++;
        if (g->h_stat[2] == 0) break;
        if (++rounds > g->max_rounds) FAIL(MGC_E_NOCONV, "push-relabel did not converge within the round cap");
        for (int p = 0; p < passes; ++p) {
            phase_begin(g, 3);
            rc = mgc_slab_push(g, 1);
            phase_end(g);
            if (rc) return rc;
            rc = slab_exchange(g, nullptr, false);
            if (rc) return rc;
            g->slab_push_passes++;
        }
        passes = passes * 2 > passes_cap ? passes_cap : passes * 2;
    }
    double part = 0.0;
    phase_begin(g, 4);
    rc = mgc_slab_finish(g, &part);
    if (rc) return rc;
    CK(cudaMemcpyAsync(g->d_esum, &part, sizeof(double), cudaMemcpyHostToDevice, g->stream));
    if (g->comm_world > 1) NK(N.AllReduce(g->d_esum, g->d_esum, 1, ncclFloat64, ncclSum, g->comm, g->stream));
    CK(cudaMemcpyAsync(energy_total, g->d_esum, sizeof(double), cudaMemcpyDeviceToHost, g->stream));
    phase_end(g);
    CK(timed_sync());
    phase_resolve(g);
    return slab_comm_poll(g);
}

int mgc_slab_solve_phase_ms(const mgc_graph* g, double* out6)
{
    if (!g || !out6) return MGC_E_ARG;
    for (int i = 0; i < 6; ++i) out6[i] = g->slab_phase_ms[i];
    return MGC_OK;
}

int mgc_slab_solve_stats(const mgc_graph* g, int64_t* exchanges, int64_t* relabel_rounds, int64_t* push_passes, int64_t* global_relabels)
{
    if (!g) return MGC_E_ARG;
    if (exchanges) *exchanges = g->slab_exchanges;
    if (relabel_rounds) *relabel_rounds = g->slab_relabel_rounds;
    if (push_passes) *push_passes = g->slab_push_passes;
    if (global_relabels) *global_relabels = g->slab_global_relabels;
    return MGC_OK;
}

}  // extern "C"
