// gc_expansion_loop.hpp -- the K-label move loop the three expansion units share (DESIGN.md §11): the cost planes,
// markers and initial labels with their checks, the cycles of moves over B images with freezing (alpha-expansions
// alpha = 0, 1, ..., K-1, or alpha-beta swaps (0, 1), (0, 2), ..., (K-2, K-1)), the statistics and the energy read-back.  A unit's handle derives from Expansion and supplies the hooks: where its
// buffers come from, how an input is staged, and how a move is built, cut and applied.  The single-image units run the
// loop with B = 1.  The loop is gc_expansion_loop.cu; the element-wise kernels it launches are compiled into
// gc_expansion.cu only, behind the launchers at the end of this file.
//
// A refused input leaves nothing behind: set_cost, set_markers, set_init and set_label_distance clear the input's flag and
// `ran` before they stage it, and set the flag only once the input passed its check, so run never sees a refused input.
#pragma once
#include "gc_host.hpp"

#include <cstdint>
#include <string>
#include <vector>

// One move of the loop: the alpha-expansion of `alpha` (beta < 0), or the alpha-beta swap of (alpha, beta), alpha < beta
struct ExpMove {
    int alpha, beta;
};

struct Expansion {
    Expansion(std::string& err, const char* abi, int device, cudaStream_t stream, unsigned n, unsigned blocks, int K, int B)
        : err(err), abi(abi), device(device), stream(stream), n(n), blocks(blocks), K(K), B(B), cost_set((size_t)K, 0)
    {
    }
    virtual ~Expansion();       // the events (the caller made `device` current); a unit frees its own buffers

    // ---- the hooks a unit supplies
    // a device buffer that lives as long as the handle
    virtual int alloc(size_t bytes, void** out) = 0;
    // `a` as n contiguous elements of `es` bytes (device or host: it is read by one cudaMemcpyDefault on `stream`);
    // `what` names it in errors.  release() follows once the copy is queued.
    virtual int stage(const mgc_array* a, size_t es, const char* what, const void** out) = 0;
    virtual void release() {}
    // before a move's first event (outside its timing)
    virtual int reset() { return MGC_OK; }
    // the graph of move `m` over the current labels, between the build and solve events
    virtual int build(const ExpMove& m) = 0;
    // its cut, between the solve and apply events: *mask = 0 (SINK) where a voxel takes alpha (expansion) or beta (swap)
    virtual int solve(const uint8_t** mask) = 0;
    // the labels the mask gives, d_switched[b] += the switches of image b (k_exp_apply / k_swap_apply unless overridden)
    virtual void apply(const uint8_t* mask, const ExpMove& m);
    // the images still in the loop, uploaded before the first cycle and after a cycle that froze some but not all
    // images; only a unit whose move kernel freezes images needs them
    virtual int freeze(const std::vector<uint8_t>& active) { (void)active; return MGC_OK; }
    // the energies of the B images into d_energy
    virtual int energy() = 0;

    // ---- the entry points, with the unit's error string (the C ABI of each unit forwards to these)
    int setup();                                        // the buffers and events below; once, after the constructor
    int set_cost(int label, const mgc_array* cost);
    int set_markers(const mgc_array* markers);
    int set_init(const mgc_array* init);
    // MGC_MOVES_EXPANSION or MGC_MOVES_SWAP; clears `ran` and the label distance (back to Potts)
    int set_moves(int kind);
    // the K x K host matrix of a label distance (checked here, uploaded to `dist`): a metric for expansion moves, a
    // semi-metric for swap moves; nullptr: back to Potts
    int set_label_distance(const double* host_V);
    int run(int max_cycles);
    int get_labels(uint8_t* out, int mem);
    int get_stats(mgc_expansion_stats* out) const;
    int get_image_stats(mgc_expansion_stats* out) const;
    int get_switched(int64_t* out) const;

    std::string& err;                   // CK and FAIL report here: the unit's own error string
    const char* const abi;              // the unit's ABI prefix, for "call <abi>_run first"
    const int device;
    const cudaStream_t stream;
    const unsigned n;                   // elements of one plane: voxels of the B images, or regions
    const unsigned blocks;              // grid of the element-wise kernels (at most REDUCE_BLOCKS)
    const int K, B;
    int cost_dtype = -1;                // MGC_F32 / MGC_F64 of the cost planes (fixed by the first plane staged)
    void* costs = nullptr;              // K planes of n elements
    std::vector<uint8_t> cost_set;
    uint8_t* labels = nullptr;
    uint8_t* markers = nullptr;         // 0 none, m > 0: label m - 1
    uint8_t* init = nullptr;
    bool have_markers = false, have_init = false;
    int moves = MGC_MOVES_EXPANSION;    // the move kind of run; a unit's build and apply hooks launch its kernels
    double* dist = nullptr;             // K x K label distance, row-major; a unit's build and energy hooks launch the
    bool have_dist = false;             // MetricPair kernels while it is set, the PottsPair ones otherwise (with_pair_rule)
    unsigned long long* d_switched = nullptr;   // [B] elements the current move switched per image
    double* d_energy = nullptr;                 // [B]
    int* d_bad = nullptr;
    cudaEvent_t ev[6] = {};             // [0..3] one move: build | solve | apply; [4..5] the whole run
    bool ran = false;
    mgc_expansion_stats st{};           // the loop
    std::vector<mgc_expansion_stats> per;       // per image
    std::vector<int64_t> switched;              // moves x B, row-major

private:
    int set_u8(const mgc_array* a, uint8_t** dst, bool* have, int limit, const char* what);
    int read_bad(int* bad);
};

// the create() check of every unit: MGC_E_ARG with the message in `err` unless 2 <= K <= 255
int expansion_check_labels(int K, std::string& err);
// MGC_E_ARG with the message in `err` unless the K x K row-major V is a metric: finite entries >= 0, a zero diagonal,
// symmetric, and V[a][c] <= V[a][b] + V[b][c] in float64 (DESIGN.md §11, "Label distances"); the message names the rule
// and the first (a, b) or (a, b, c) that breaks it.  semi_metric skips the triangle rule only (swap moves).
int expansion_check_distance(const double* V, int K, std::string& err, bool semi_metric = false);

// the element-wise kernels of gc_expansion.cuh the loop launches, compiled into gc_expansion.cu only; `dtype` (MGC_F32 /
// MGC_F64) selects the cost type, and markers / init may be nullptr
void exp_init_launch(cudaStream_t s, unsigned blocks, unsigned n, int K, int dtype, const void* costs, const uint8_t* markers,
                     const uint8_t* init, uint8_t* labels, int* bad);
void exp_apply_launch(cudaStream_t s, unsigned blocks, unsigned n, const uint8_t* mask, uint8_t* labels, int alpha,
                      unsigned long long* switched);
void swap_apply_launch(cudaStream_t s, unsigned blocks, unsigned n, const uint8_t* mask, uint8_t* labels, int alpha, int beta,
                       unsigned long long* switched);
void exp_check_costs_launch(cudaStream_t s, unsigned blocks, unsigned n, int dtype, const void* cost, int* bad);
void exp_check_u8_launch(cudaStream_t s, unsigned blocks, unsigned n, const uint8_t* a, int limit, int* bad);
