/* medpy_b200_graphcut.h -- the drop-in boundary of the H100 voxel graph-cut path.
 *
 * C ABI (plain pointers and sizes, no torch / numpy / C++ types) of libmedpy_b200_gc.so.  It replaces,
 * for the voxel path only, what the reference reaches through its Boost.Python extension
 * `medpy.graphcut.maxflow` (lib/maxflow/src/wrapper.cpp:59-89,125-134; class GraphDouble =
 * Pythongraph<double,double,double>, pythongraph.h:15-22) plus the per-edge / per-node Python loops that
 * feed it (medpy/graphcut/energy_voxel.py:611-664, graph.py:310-380,532-552).  Instead of one FFI call per
 * edge, a whole energy term crosses the boundary in one call and is evaluated by a CUDA kernel on the
 * implicit 2*ndim-connected lattice; no edge list is ever materialised.
 *
 * Conventions
 *   - every function returns an int status: MGC_OK (0) or a negative MGC_E_* code; the message for the
 *     last failure on a handle is available from mgc_last_error() (never exit(), unlike graph.cpp:22);
 *   - node id == C-order flat index over the logical shape (generate.py:170-172, energy_voxel.py:650-677);
 *   - arrays are described by (pointer, dtype, byte strides over the logical shape); host pointers are only
 *     borrowed for the duration of the call (copied to the device inside); MGC_MEM_DEVICE pointers must be
 *     valid on the handle's device and are read on the handle's stream; they too are borrowed for the call only,
 *     except the image and probability map of mgc_build_voxel_graph under MGC_OPT_KEEP_DEVICE_INPUTS (see there);
 *   - all device memory is owned by the library; a handle is not thread-safe, distinct handles are
 *     independent; the GIL can be released around every call;
 *   - there is NO CPU solver behind this ABI: with no usable CUDA device mgc_create fails with
 *     MGC_E_CUDA and nothing else works.
 */
#ifndef MEDPY_B200_GRAPHCUT_H
#define MEDPY_B200_GRAPHCUT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MGC_ABI_VERSION 3
#define MGC_MAX_NDIM 4

/* status codes */
#define MGC_OK 0
#define MGC_E_ARG (-1)     /* malformed argument (mirrors the reference's ValueError cases)     */
#define MGC_E_CUDA (-2)    /* CUDA runtime failure / no device                                  */
#define MGC_E_NOMEM (-3)   /* device allocation failed                                          */
#define MGC_E_STATE (-4)   /* call not valid in the handle's current state                      */
#define MGC_E_WEIGHT (-5)  /* an n-link weight <= 0 was produced (GCGraph.set_nweight, graph.py:436-437) */
#define MGC_E_NOCONV (-6)  /* solver hit its iteration cap without converging                   */
#define MGC_E_LABELS (-7)  /* label image is not numbered 1..K (energy_label.py:444-456 raises AttributeError) */

/* element types of input arrays */
#define MGC_F32 0
#define MGC_F64 1
#define MGC_U8 2
#define MGC_I16 3
#define MGC_I32 4

/* memory space of an input / output pointer */
#define MGC_MEM_HOST 0
#define MGC_MEM_DEVICE 1

/* boundary terms: the eight energy_voxel.boundary_* functions (energy_voxel.py:68-516) */
#define MGC_BOUNDARY_DIFFERENCE_LINEAR 0       /* energy_voxel.py:145-191 */
#define MGC_BOUNDARY_DIFFERENCE_EXPONENTIAL 1  /* :241-302 */
#define MGC_BOUNDARY_DIFFERENCE_DIVISION 2     /* :352-409 */
#define MGC_BOUNDARY_DIFFERENCE_POWER 3        /* :457-516 */
#define MGC_BOUNDARY_MAXIMUM_LINEAR 4          /* :68-116  */
#define MGC_BOUNDARY_MAXIMUM_EXPONENTIAL 5     /* :194-238 */
#define MGC_BOUNDARY_MAXIMUM_DIVISION 6        /* :305-349 (computes the *difference* variant, :347) */
#define MGC_BOUNDARY_MAXIMUM_POWER 7           /* :412-454 */

/* termtype (graph.h:57-61, wrapper.cpp:85-88) */
#define MGC_SOURCE 0
#define MGC_SINK 1

typedef struct mgc_graph mgc_graph; /* opaque; replaces GraphDouble + GCGraph storage */

typedef struct mgc_array {
    const void* data;                    /* first element (logical index 0,...,0) */
    int32_t dtype;                       /* MGC_F32 ... */
    int32_t mem;                         /* MGC_MEM_HOST | MGC_MEM_DEVICE */
    int64_t strides[MGC_MAX_NDIM];       /* BYTE strides over the logical shape (numpy .strides) */
} mgc_array;

typedef struct mgc_stats {
    int64_t n_voxels;
    int64_t push_sweeps;        /* push/relabel sweeps executed                     */
    int64_t global_relabels;    /* exact backward BFS passes                        */
    int64_t relabel_sweeps;     /* relaxation sweeps inside those                   */
    int64_t kernel_launches;    /* every kernel this handle launched                */
    int64_t active_last;        /* active voxels at the last check (0 = converged)  */
    double ms_terms;            /* device ms: boundary + regional + marker kernels  */
    double ms_solve;            /* device ms: init + push-relabel + global relabels */
    double ms_readout;          /* device ms: mask + energy kernels                 */
    double flow_const;          /* sum of the add_tweights minima (graph.h:423)     */
    double energy;              /* value maxflow() returned                         */
    int64_t device_bytes;       /* device memory held by the handle                 */
    double ms_push;             /* device ms inside push/relabel sweeps (CUDA events around each batch)  */
    double ms_relabel;          /* device ms inside global-relabel kernels (init + relaxation sweeps)    */
    double ms_boundary;         /* device ms of the last boundary (n-link) kernel alone                  */
    double ms_init;             /* device ms of the solver-state initialisation kernel (k_init_tile); 0 after a fused build */
    int64_t tiles_materialised; /* lazy build: 8^3 tiles whose capacities, tr and excess k_caps_tiles computed (0 eager) */
    double ms_caps;             /* device ms of the materialiser launches (k_caps_claim + k_caps_tiles; not in ms_push)  */
    int64_t seed_folds;         /* mgc_add_seeds, mgc_remove_seeds, mgc_add_tweights_warm and the two n-link warm     */
                                /* calls (mgc_add_nweights_warm / _dense_warm) folded into this handle since its      */
                                /* build (reset by the build; erase, t-link and n-link calls count like add calls in  */
                                /* all three fields; a call of only zero weights folds nothing, counts not)           */
    double ms_seeds;            /* device ms of those calls: id / weight upload, grouping (sort or compaction,        */
                                /* run-length), tile claim + materialisation, fold, push-list fix-up; not the one     */
                                /* read-back of the item count                                                         */
    double ms_seeds_host;       /* host ms of those calls before anything is enqueued: scratch growth, launch count   */
    int64_t tiles_deferred;     /* 3-D tile solver, easy instance: listed tiles the label window held back, summed over the push launches of each solve */
    int64_t tiles_dropped;      /* ... listed tiles that left the push lists without a visit (no active voxel at a finite label) */
    int64_t relabel_passes;     /* tile solver: BFS passes (worklist generations) of all global relabels; relabel_sweeps counts launches */
    double ms_relabel_first;    /* device ms of the first global relabel of each solve (tile solver), summed */
    int64_t relabel_passes_first; /* ... its BFS passes, summed */
    int64_t build_blocks_refused; /* lazy exponential build staged by TMA: 8 x 8 x 32 build blocks whose range test failed */
                                  /* (built by the per-warp fallback launch instead of the lean one); read at the solve  */
} mgc_stats;

/* ---- lifetime ------------------------------------------------------------------------------------- */

/* Replaces GraphDouble(nodes, edges) + add_node(nodes) (graph.py:305-306; graph.cpp:11-31) for a lattice
 * of logical shape `shape[ndim]`, 1 <= ndim <= 4.  `device` = CUDA ordinal (or -1 for the current one). */
int mgc_create(int32_t ndim, const int64_t* shape, int32_t device, mgc_graph** out);
/* Slab variant for the z-slab multi-GPU path: this handle owns planes [z0, z1) of axis 0 of the global
 * lattice `shape` and keeps one ghost plane on each interior side. */
int mgc_create_slab(int32_t ndim, const int64_t* shape, int64_t z0, int64_t z1, int32_t device, mgc_graph** out);
void mgc_destroy(mgc_graph* g); /* ~Graph (graph.cpp:34-43) */
/* Graph::reset (graph.h:133): forget all weights, keep the allocation. */
int mgc_reset(mgc_graph* g);
const char* mgc_last_error(const mgc_graph* g); /* g may be NULL: last create() failure */
int mgc_abi_version(void);
/* Page-locked host buffers from a process-wide pool (the bindings hand the mask back in one: a device->host copy
 * into pinned memory runs at PCIe rate, into fresh pageable memory at a fraction of it).  mgc_host_free returns
 * the block to the pool. */
int mgc_host_alloc(size_t bytes, void** out);
void mgc_host_free(void* p);
/* Device and pinned-host blocks are cached process-wide (a 1024^3 handle holds 84 GB; its blocks stay cached for the next
 * graph after mgc_destroy).  mgc_trim_pools returns every cached block to the driver; live handles keep theirs. */
int mgc_trim_pools(void);
/* Options.  MGC_OPT_DEFER_WEIGHT_CHECK (default 0): mgc_add_boundary on a HOST image does not wait for its kernel to
 * report non-positive weights; the verdict (MGC_E_WEIGHT) is delivered by the next call on the handle instead (terms,
 * markers, maxflow, mgc_check).  graph_from_voxels switches it on because it always adds the markers right after the
 * boundary term, which lets the marker upload overlap the stencil kernel. */
#define MGC_OPT_DEFER_WEIGHT_CHECK 1
/* MGC_OPT_WARM (default 0; 1 switches it on): warm re-solves (mgc_add_seeds / mgc_remove_seeds / mgc_add_tweights_warm /
 * mgc_add_nweights_warm / mgc_add_nweights_dense_warm) on handles the lazy fused build did not build -- see mgc_add_seeds. */
#define MGC_OPT_WARM 2
/* MGC_OPT_KEEP_DEVICE_INPUTS (default 0; 1 switches it on): a lifetime promise, not a speed knob.  The lazy fused build
 * (mgc_build_voxel_graph) keeps reading its image and probability map after the call: the materialiser, the solve and
 * the warm folds recompute capacities and t-links from them.  By default the build keeps a copy of each, and device inputs
 * are borrowed for the call only.  With the option set, a contiguous MGC_MEM_DEVICE image or map is not copied: the
 * handle records the caller's pointer and reads it on its stream until the next build, mgc_reset or mgc_destroy.  The
 * caller then keeps the array alive and unchanged until then, and until the handle's stream has finished the work queued
 * before (mgc_synchronize).  mgc_destroy never frees it.  Host and strided inputs are staged into buffers the handle
 * owns as before.  The option applies to builds that start after it is set.  Adding it left MGC_ABI_VERSION at 3. */
#define MGC_OPT_KEEP_DEVICE_INPUTS 3
int mgc_set_option(mgc_graph* g, int32_t option, int64_t value);
/* Deliver a deferred verdict now (MGC_OK / MGC_E_WEIGHT). */
int mgc_check(mgc_graph* g);
/* Use an externally owned cudaStream_t (e.g. torch's current stream) for all work of this handle. */
int mgc_set_stream(mgc_graph* g, void* cuda_stream);
int mgc_synchronize(mgc_graph* g);

/* ---- t-links -------------------------------------------------------------------------------------- */

/* regional_probability_map (energy_voxel.py:33-65) -> set_tweights_all (graph.py:532-552) ->
 * add_tweights(v, p*alpha, (1-p)*alpha) for every voxel (graph.h:415-425).  The products are formed in
 * `compute_dtype` (MGC_F32 or MGC_F64) -- the dtype numpy's promotion gives `probability_map * alpha`
 * (f32 map * Python float stays f32) -- and only then widened to double (graph.py:496-498). */
int mgc_add_regional_probability(mgc_graph* g, const mgc_array* prob, double alpha, int32_t compute_dtype);
/* Generic set_tweights_all: add_tweights(v, src[v], snk[v]); src/snk are arrays of doubles over the
 * logical shape. */
int mgc_add_tweights_dense(mgc_graph* g, const mgc_array* src, const mgc_array* snk);
/* set_source_nodes / set_sink_nodes (graph.py:310-380) as called by graph_from_voxels
 * (generate.py:169-172): add_tweights(v, 65535, 0) where fg != 0, THEN add_tweights(v, 0, 65535) where
 * bg != 0.  Either array may be NULL.  dtype MGC_U8 (numpy bool_). */
int mgc_add_markers(mgc_graph* g, const mgc_array* fg, const mgc_array* bg);

/* ---- n-links -------------------------------------------------------------------------------------- */

/* One of the eight boundary terms evaluated over the whole lattice (replaces the per-edge loop
 * energy_voxel.py:660-664 -> GCGraph.set_nweight -> Graph::sum_edge graph.h:456-480): for every axis d and
 * voxel pair (p, p+e_d):  w = g(|I_p - I_q|) or g(max(|I_p|,|I_q|)), w /= spacing[d] when spacing != NULL,
 * cap(p->q) += w, cap(q->p) += w, all in float64.
 *   sigma : ignored by the two linear terms.
 *   norm  : linear terms only -- the normaliser max|grad| / |max-min| the host computed in the image's own
 *           dtype (energy_voxel.py:99,174); pass NaN to have the device compute it (f32/f64 images).
 * Returns MGC_E_WEIGHT if any produced weight is <= 0 (the reference raises ValueError there). */
int mgc_add_boundary(mgc_graph* g, int32_t kind, const mgc_array* image, double sigma,
                     const double* spacing, double norm);
/* Dense n-links along one axis for user-written boundary terms: fwd/bwd are double arrays over the logical
 * shape; entry p holds cap(p -> p+e_axis) / cap(p+e_axis -> p); entries on the last plane of `axis` are
 * ignored.  Accumulates like sum_edge (graph.h:456-480); 0 leaves a pair untouched, negative values ->
 * MGC_E_WEIGHT (the `<= 0` ValueError of GCGraph.set_nweight is raised by the host layer, graph.py:436-437). */
int mgc_add_nweights_dense(mgc_graph* g, int32_t axis, const mgc_array* fwd, const mgc_array* bwd);

/* ---- the whole graph of graph_from_voxels in one call -------------------------------------------------- */

/* Everything graph_from_voxels puts into the graph (generate.py:159-172: regional term, boundary term, foreground
 * markers, background markers) handed over at once.  On a fresh handle (create / mgc_reset, nothing added yet) of a
 * 1-D..3-D lattice the terms are evaluated by ONE kernel pass (csrc/gc_build.cuh: n-link stencil + t-link replay +
 * solver-state initialisation; the image block of every CTA is staged by a TMA box copy) instead of four passes
 * over the lattice, and for contiguous host arrays the upload of z-chunk c+1 overlaps the build of chunk c.  The
 * result is the graph mgc_add_regional_probability + mgc_add_boundary + mgc_add_markers would leave (same
 * arithmetic per weight; the add_tweights constant is summed in a different, still fixed, order).  Anything else
 * (4-D lattice, no boundary term, terms already present) runs those three calls in that order.
 *   prob / fg / bg may be NULL; boundary_kind -1 = no boundary term; markers either as uint8 arrays (fg, bg) or
 *   bit-packed over the C-order flat voxel index v: bit (v & 31) of word (v >> 5) (fg_bits, bg_bits, bits_mem).
 * Weight verdict: MGC_E_WEIGHT from this call, or -- with MGC_OPT_DEFER_WEIGHT_CHECK -- from the next
 * mgc_check / mgc_maxflow.  Host pointers are borrowed for the duration of the call only. */
typedef struct mgc_voxel_terms {
    const mgc_array* prob;   /* regional_probability_map input (energy_voxel.py:33-65) or NULL */
    double alpha;
    int32_t compute_dtype;   /* MGC_F32 / MGC_F64, see mgc_add_regional_probability */
    int32_t boundary_kind;   /* MGC_BOUNDARY_* or -1 */
    const mgc_array* image;
    double sigma;
    const double* spacing;   /* NULL: no distance weighting */
    double norm;             /* linear terms: normaliser or NaN, see mgc_add_boundary */
    const mgc_array* fg;     /* uint8 marker volumes or NULL */
    const mgc_array* bg;
    const uint32_t* fg_bits; /* bit-packed marker volumes or NULL */
    const uint32_t* bg_bits;
    int32_t bits_mem;        /* MGC_MEM_HOST / MGC_MEM_DEVICE of fg_bits / bg_bits */
    /* Optional (host bit planes only): the number of leading 32-bit WORDS of BOTH planes that have been written so far,
     * advanced by a producer thread while this call runs (the binding packs the marker bytes on worker threads while the
     * image is already on its way to the device).  The call waits for it before it enqueues the upload of a chunk.
     * NULL: the planes are complete. */
    const volatile int64_t* bits_ready_words;
} mgc_voxel_terms;
int mgc_build_voxel_graph(mgc_graph* g, const mgc_voxel_terms* terms);
/* 1 if mgc_build_voxel_graph would take the single-pass path on a fresh state of this handle. */
int mgc_can_fuse(const mgc_graph* g);

/* ---- batches of independent images ------------------------------------------------------------------- */

/* A handle for `batch` independent images of shape image_shape[0..ndim) (1 <= ndim <= 3), cut in one build and one
 * solve.  The images are stacked along axis 0 of one (batch * Z, Y, X) lattice (canonical image shape (Z, Y, X) with
 * leading 1s) whose pairs across the seams between images do not exist, so each image is cut as if it were alone.
 * MGC_E_ARG when batch * (voxels per image) would reach 2^31, checked before anything is allocated.
 * On a batch handle the per-term calls, mgc_build_voxel_graph and the z-slab calls return MGC_E_STATE with one message.
 * The warm calls (mgc_add_seeds ... mgc_remove_nweights_dense_warm) return it too unless MGC_OPT_WARM is set and the
 * state comes from mgc_build_voxel_batch (not after mgc_reset).  The option follows the rule of a single handle: on an
 * eagerly built batch (MEDPY_GC_LAZY_CAPS=0) it must be set before the first solve, whose start records the residual
 * source capacities the folds read; a lazily built batch (the default) needs no record, so there it is also accepted
 * after a solve and admits the folds from then on.  With the option
 * they fold as on a single lattice handle, before or after a solve: node ids are C-order over (batch, ...image); a listed
 * pair across the seam between two images is no lattice pair (MGC_E_ARG, the handle unchanged); the dense n-link forms
 * take the lattice's canonical axis (0 = the image's Z axis of 3-D images) and ignore the last plane of every image along
 * axis 0; each fold's change of the add_tweights constants goes to the images it touched, so mgc_get_batch_energies
 * stays per image and the images a fold does not touch keep their energies bit for bit.
 * Adding these three entry points left MGC_ABI_VERSION at 3 and mgc_stats unchanged. */
int mgc_create_batch(int32_t ndim, const int64_t* image_shape, int64_t batch, int32_t device, mgc_graph** out);
/* The terms of every image in one fused build.  The arrays of `terms` are over the logical (batch, ...image) shape
 * (strided arrays are gathered); alpha, compute_dtype, the probability-map dtype and the spacing are shared by the batch.
 * A boundary term is required (MGC_E_ARG), markers are uint8 arrays (no bit planes).  sigmas / norms: host arrays of
 * `batch` entries, or NULL for terms->sigma / terms->norm on every image; a NaN norm of a linear term means the image's
 * normaliser is reduced on the device over that image alone.  MGC_E_STATE on a handle that is not fresh (reset() it),
 * or when the fused build is switched off (MEDPY_GC_FUSE=0).  mgc_maxflow then returns the energy of the whole lattice
 * (the sum over the images) and mgc_get_mask the whole (batch, ...image) mask. */
int mgc_build_voxel_batch(mgc_graph* g, const mgc_voxel_terms* terms, const double* sigmas, const double* norms);
/* After mgc_maxflow: out[b] (batch host doubles) = the energy of image b, its add_tweights constant plus the flow its
 * sink links absorbed -- what graph_from_voxels + maxflow return for that image alone, up to the order of the sums. */
int mgc_get_batch_energies(mgc_graph* g, double* out);

/* ---- solve / read-out ----------------------------------------------------------------------------- */

/* Graph::maxflow() (maxflow.cpp:471-604; wrapper.cpp:68): runs the lattice push-relabel to a maximum
 * preflow and returns the min-cut energy INCLUDING the add_tweights constants, like the reference's `flow`.
 * Idempotent after convergence. */
int mgc_maxflow(mgc_graph* g, double* energy);
/* Seeds added to a graph and solved warm (the interactive refinement loop of the reference: maxflow(), then
 * add_tweights(v, 65535, 0) on new foreground seeds and add_tweights(v, 0, 65535) on new background seeds, then
 * maxflow() again, which continues from BK's residual graph; graph.py:310-380, graph.h:415-425).  The meaning is exactly
 * add_tweights(v, 65535, 0) for every id of fg_ids in list order, THEN add_tweights(v, 0, 65535) for every id of bg_ids;
 * duplicate ids count once per occurrence, an id in both lists cancels like fg and bg markers do.  The seeds are folded
 * into the handle's current state (solved or not; before the first solve the build's pending source excess is
 * materialised first) and the next mgc_maxflow / mgc_get_mask / mgc_what_segment returns
 * the result for the enlarged graph, starting from the flow already routed instead of from zero.
 *   fg_ids / bg_ids : C-order node ids, int64, in host or device memory (`mem`); either may be NULL when its count is 0.
 * MGC_E_ARG for an id out of range.  MGC_E_STATE unless the handle's last build was the lazy fused build
 * (mgc_build_voxel_graph on a 1-D..3-D lattice with a boundary term, tile solver, not a z-slab, lazy capacities on): the
 * fold recomputes capacities from the copies that build keeps.  Elsewhere reset() and a rebuild with the seeds is the way.
 * mgc_add_tweights_dense / mgc_add_markers and the other term entry points still refuse a solved graph.  Adding this
 * entry point left MGC_ABI_VERSION at 3: nothing that existed changed.
 * MGC_OPT_WARM = 1 (mgc_set_option) extends these folds to every other tile-solver handle: 4-D lattices, 1-D..3-D graphs
 * built term by term, the eager fused build (lazy capacities off), and z-slab handles.  Such a handle keeps no copy of its
 * inputs, so its first solve records the residual source capacity of every voxel in place of the net t-link, before the
 * first push (a pass over tr and the capacities after the eager fused build; nothing extra on the per-term path).
 *   - Set it before the first solve: while no flow has started (a handle fresh from create / mgc_reset / a build).  Later
 *     it returns MGC_E_STATE, except on a lazily built handle, where it changes nothing.
 *   - It persists across mgc_reset, like MGC_OPT_DEFER_WEIGHT_CHECK, and changes neither results nor the first solve's
 *     mask and energy.
 *   - A fold on such a handle before its first solve initialises the solver state and takes the record first.
 *   - z-slab handles (mgc_create_slab): set the option before the first mgc_slab_begin / mgc_slab_solve; the first one
 *     takes the record, and the next mgc_slab_solve (or the stepped sequence) re-solves from the state the folds left.
 *     Node ids are the slab's local lattice ids (owned planes plus ghost planes, C order, as mgc_get_edge /
 *     mgc_what_segment / mgc_get_trcap take them), and the dense forms take the arrays the slab's cold
 *     mgc_add_tweights_dense / mgc_add_nweights_dense take, ghost planes included.  Each slab applies only what it owns:
 *     a t-link call on a ghost voxel is skipped (the neighbour owns it), and an n-link call on (u, v) adds cap to
 *     r(u->v) only if u is owned and rev_cap to r(v->u) only if v is owned, so an axis-0 pair across a border is applied
 *     half on each slab with no communication, and a pair inside a ghost plane is skipped.  Range, neighbour, finiteness
 *     and sign checks run over every entry, skipped ones included.  Each slab adds the constant change of its owned
 *     voxels to its own share of the energy, so the all-reduced total is the energy of the edited global graph.
 * MGC_ABI_VERSION stays 3 and mgc_stats keeps its layout. */
int mgc_add_seeds(mgc_graph* g, const int64_t* fg_ids, int64_t n_fg, const int64_t* bg_ids, int64_t n_bg, int32_t mem);
/* Seeds erased from a graph and solved warm: the inverse call of mgc_add_seeds, as the reference erases a seed
 * (add_tweights accepts negative capacities, graph.h:415-425).  The meaning is exactly add_tweights(v, -65535, 0) for
 * every id of fg_ids in list order, THEN add_tweights(v, 0, -65535) for every id of bg_ids; duplicate ids count once per
 * occurrence.  The call does not check that a seed was ever added: erasing a seed that is not there applies the call
 * anyway, as the reference does, and leaves the graph with that t-link lowered by 65535.  The markers of
 * mgc_build_voxel_graph are the same add_tweights calls, so this also erases them.  Same arguments, preconditions and
 * errors as mgc_add_seeds (MGC_E_ARG for an id out of range, with the handle unchanged; MGC_E_STATE unless the last build
 * was the lazy fused build), solved or not.  Adding this entry point left MGC_ABI_VERSION at 3. */
int mgc_remove_seeds(mgc_graph* g, const int64_t* fg_ids, int64_t n_fg, const int64_t* bg_ids, int64_t n_bg, int32_t mem);
/* Any add_tweights calls folded into a graph and solved warm (soft strokes, a GrabCut-style re-estimation of the
 * regional term, a change of the regional / boundary weight on a solved graph; graph.h:415-425: BK applies the call to
 * the residual terminal capacity and the next maxflow() continues from the residual graph).
 *   ids != NULL : the list form, add_tweights(ids[k], src[k], snk[k]) for k = 0 .. count-1 in array order; duplicate ids
 *                 are applied in order, once per occurrence.
 *   ids == NULL : the dense form, add_tweights(v, src[v], snk[v]) for every voxel in C order (set_tweights_all on a solved
 *                 graph); count must be the voxel count.  add_tweights(v, 0, 0) changes nothing, so only the voxels with
 *                 a nonzero weight are touched.
 * src / snk are contiguous doubles of any sign, `count` of each; ids are C-order int64 node ids.  All three live in `mem`
 * (host memory is borrowed for the call, device memory is read in place on the handle's stream).  count == 0 does
 * nothing.  MGC_E_ARG, with the handle unchanged, for an id out of range, a NaN or infinite weight (the reference would
 * carry it into BK) or bad counts and pointers.  Same preconditions, MGC_E_STATE message and behaviour on solved and
 * unsolved handles as mgc_add_seeds.  Adding this entry point left MGC_ABI_VERSION at 3. */
int mgc_add_tweights_warm(mgc_graph* g, const int64_t* ids, const double* src, const double* snk, int64_t count, int32_t mem);
/* sum_edge calls folded into a graph and solved warm (a boundary brush, a larger boundary weight, a second boundary term on
 * a solved graph; graph.h:456-480: BK adds cap to the residual capacity of i -> j and rev_cap to that of j -> i, and the
 * next maxflow() continues from the residual graph).  The meaning is exactly sum_edge(i[k], j[k], cap[k], rev_cap[k]) for
 * k = 0 .. count-1 in array order, applied to the residual capacities: a repeated pair is applied once per occurrence, in
 * call order.  The add_tweights constant does not change.
 *   i / j          : C-order int64 ids of lattice neighbours (i != j); cap / rev_cap: contiguous doubles; all four in `mem`
 *                    (host memory is borrowed for the call, device memory is read in place on the handle's stream).
 *   increments     : nonnegative and finite, as the reference's sum_edge asserts.  A zero increment changes nothing and is
 *                    skipped; a call of only zero increments keeps the solved state, mask and energy.  Capacities are
 *                    lowered by mgc_remove_nweights_warm / mgc_remove_nweights_dense_warm.
 * count == 0 does nothing.  MGC_E_ARG, with the handle unchanged, for an id out of range, a pair that is not a lattice
 * neighbour, a NaN or infinite weight, or bad counts and pointers; MGC_E_WEIGHT, with the handle unchanged, for a negative
 * weight.  Same preconditions, MGC_E_STATE message and behaviour on solved and unsolved handles as mgc_add_tweights_warm.
 * mgc_add_nweights_dense, mgc_add_boundary and the other term entry points still refuse a solved graph.  Adding this entry
 * point left MGC_ABI_VERSION at 3. */
int mgc_add_nweights_warm(mgc_graph* g, const int64_t* i, const int64_t* j, const double* cap, const double* rev_cap,
                          int64_t count, int32_t mem);
/* The dense form of mgc_add_nweights_warm, in the layout of mgc_add_nweights_dense: fwd / bwd are float64 arrays over the
 * logical shape (any positive strides, host or device); entry p holds the increments of cap(p -> p+e_axis) and
 * cap(p+e_axis -> p), and the last plane of `axis` is ignored.  Only the pairs with a nonzero entry are touched, so an
 * update of a box only materialises that box's tiles on a lazily built handle.  Same errors, preconditions and behaviour
 * as mgc_add_nweights_warm.  Adding this entry point left MGC_ABI_VERSION at 3. */
int mgc_add_nweights_dense_warm(mgc_graph* g, int32_t axis, const mgc_array* fwd, const mgc_array* bwd);
/* The inverse of mgc_add_nweights_warm: n-link capacity taken off a graph and solved warm (a boundary brush undone, a lower
 * boundary weight, a relaxed boundary along a cut).  The meaning is exactly sum_edge(i[k], j[k], -cap[k], -rev_cap[k]) for
 * k = 0 .. count-1 in array order: the next maxflow() returns the min cut and the energy of a graph built from scratch
 * with every call so far replayed and the decrements subtracted from the capacities.  On an unsolved graph that is what
 * the reference's sum_edge with negated values does.  On a solved one the reference has no defined meaning for a
 * decrease below the flow an arc carries (BK would run on negative residuals); this definition is an extension of the
 * library: the excess flow is cancelled and a voxel left short takes the shortfall from its terminal link (Kohli and
 * Torr's reparametrisation, which lowers the add_tweights constant and keeps the cut of the decreased graph).
 *   i / j, cap / rev_cap, mem : as in mgc_add_nweights_warm; cap / rev_cap are the DECREMENTS, nonnegative and finite.
 *   caller's promise          : every arc's capacity stays >= 0.  The handle keeps no per-arc capacity, so it checks the
 *                               pair: r(i->j) + r(j->i) = c(i->j) + c(j->i) under any flow, and a pair whose total
 *                               decrement exceeds its residual sum by more than 2^-44 x max(sum, decrement) -- a few
 *                               hundred roundings of the push updates -- is refused.  Within that tolerance a residual
 *                               that comes out negative is clamped to 0, so removing exactly the weight that was there is
 *                               accepted.
 * count == 0 does nothing.  MGC_E_ARG for an id out of range, a pair that is not a lattice neighbour, a NaN or infinite
 * decrement, or bad counts and pointers; MGC_E_WEIGHT for a negative decrement or a pair whose decrement exceeds its
 * residual sum.  Every check finishes before anything is written, and the handle is left unchanged when one fails (an
 * MGC_OPT_WARM handle that was never solved may have run the init its first solve would run).  Same preconditions,
 * memory spaces, statistics and MGC_E_STATE message as mgc_add_nweights_warm; sparse graphs refuse.  z-slab handles return
 * MGC_E_STATE for every call, whatever the pairs: a decrement of a pair across a border needs the neighbour's residual, and
 * a refusal on every slab alike would need a two-phase collective, so the answer does not depend on the partition.
 * Adding this entry point left MGC_ABI_VERSION at 3. */
int mgc_remove_nweights_warm(mgc_graph* g, const int64_t* i, const int64_t* j, const double* cap, const double* rev_cap,
                             int64_t count, int32_t mem);
/* The dense form of mgc_remove_nweights_warm, in the layout of mgc_add_nweights_dense_warm: entry p of fwd / bwd holds the
 * decrements of cap(p -> p+e_axis) and cap(p+e_axis -> p); the last plane of `axis` is ignored and only the pairs with a
 * nonzero entry are touched.  Same meaning, checks and errors as mgc_remove_nweights_warm.  Adding this entry point left
 * MGC_ABI_VERSION at 3. */
int mgc_remove_nweights_dense_warm(mgc_graph* g, int32_t axis, const mgc_array* fwd, const mgc_array* bwd);
/* Bulk form of the what_segment loop (bin/medpy_graphcut_voxel.py:177-181): out[v] = 0 if the voxel is in
 * the SINK set else 1, C-order over the logical shape.  `mem` selects host or device destination. */
int mgc_get_mask(mgc_graph* g, uint8_t* out, int32_t mem);
/* Graph::what_segment(i) (graph.h:560-571): MGC_SINK or MGC_SOURCE (free nodes -> SOURCE). */
int mgc_what_segment(mgc_graph* g, int64_t node, int32_t* segment);
/* Graph::get_edge(i, j) (graph.h:482-497): current residual capacity of arc i->j, 0 if not lattice neighbours. */
int mgc_get_edge(mgc_graph* g, int64_t i, int64_t j, double* cap);
/* Graph::get_trcap(i) (graph.h:535-540): current residual terminal capacity (>0 source, <0 sink). */
int mgc_get_trcap(mgc_graph* g, int64_t node, double* trcap);
int mgc_get_node_num(const mgc_graph* g, int64_t* n);
int mgc_get_arc_num(const mgc_graph* g, int64_t* n);
int mgc_get_stats(const mgc_graph* g, mgc_stats* out);

/* ---- pre-step of the boundary_maximum_* terms (SURVEY.md §8 row f1) ----------------------------------- */

/* bin/medpy_gradient.py:79-85: scipy.ndimage.generic_gradient_magnitude(image, prewitt, output=float32), mode 'reflect',
 * reproduced bit for bit.  `image`: f32/f64/u8/i16/i32 array over `shape[ndim]` (1 <= ndim <= 4, any positive strides);
 * `out`: C-contiguous float32 array of the same shape in host (MGC_MEM_HOST) or device memory. */
int mgc_gradient_magnitude_prewitt(int32_t ndim, const int64_t* shape, const mgc_array* image, float* out,
                                   int32_t out_mem, int32_t device);

/* ---- z-slab multi-GPU stepping (driven by the host over NCCL; see INTEGRATION.md) ------------------- */

/* Number of elements of one border-plane message: the product of the extents of axes 1..ndim-1. */
int mgc_slab_plane_elems(const mgc_graph* g, int64_t* n);
/* Initialise the solver state (source-excess clamp, sink capacities) once all terms are in. */
int mgc_slab_begin(mgc_graph* g);
/* `n` local push/relabel passes of the tile solver, each one over both tile colours. */
int mgc_slab_push(mgc_graph* g, int32_t n);
/* Pack the messages for the lower / upper neighbour into device buffers of plane_elems elements each:
 * heights (int32) of my border plane and the flow (double) pushed across the border since the last pack.
 * Pass NULL for a side without neighbour. */
int mgc_slab_pack(mgc_graph* g, int32_t* h_lo, double* f_lo, int32_t* h_hi, double* f_hi);
/* Apply the neighbours' messages: ghost-plane heights, and received flow added to excess and to the reverse
 * residual of my border plane.  `changed_dev` (DEVICE pointer or NULL) is set to 1 by the kernel if any ghost label
 * differs from before; the caller zeroes it and typically all-reduces it over the ranks.  No host synchronisation. */
int mgc_slab_unpack(mgc_graph* g, const int32_t* h_lo, const double* f_lo, const int32_t* h_hi, const double* f_hi,
                    int32_t* changed_dev);
/* Global relabel, distributed: (re)start a backward BFS from the sink ... */
int mgc_slab_relabel_begin(mgc_graph* g);
/* ... relax locally until nothing changes (given the current ghost labels).  changed_out may be NULL (then the call
 * does not synchronise with the host); otherwise *changed_out = 1 if any tile was visited in this call. */
int mgc_slab_relabel_relax(mgc_graph* g, int32_t* changed_out);
/* Voxels with excess > 0 and a finite label (owned planes only). */
int mgc_slab_count_active(mgc_graph* g, int64_t* active_out);
/* Same, written to a DEVICE counter (uint64) without synchronising with the host. */
int mgc_slab_count_active_dev(mgc_graph* g, unsigned long long* count_dev);
/* Finish: build the mask of the owned planes and this slab's share of the energy
 * (flow absorbed by the owned sink links + owned add_tweights constants). */
int mgc_slab_finish(mgc_graph* g, double* energy_part);

/* ---- z-slab solve inside the library (NCCL over NVLink on the handle's stream) ------------------------------ */

/* The stepping calls above let a host drive the slabs; these three run the WHOLE distributed solve natively: border
 * messages go out with ncclSend / ncclRecv (grouped, on the handle's stream), the stop test is one ncclAllReduce and
 * one host synchronisation per relabel round, the energy is all-reduced (float64).  libnccl.so.2 is bound at run time
 * (the copy already loaded in the process, e.g. torch's); asynchronous NCCL errors are polled at every host decision
 * and returned as MGC_E_CUDA instead of hanging.
 *   mgc_slab_comm_unique_id : 128-byte ncclUniqueId made by ONE rank; the host distributes it (any transport);
 *   mgc_slab_comm_init      : collective over the `world` slab ranks (rank r owns the r-th slab);
 *   mgc_slab_solve          : collective; *energy_total = the global min-cut energy on every rank.  mgc_get_mask then
 *                             returns the rank's owned planes. */
int mgc_slab_comm_unique_id(void* out128);
int mgc_slab_comm_init(mgc_graph* g, int32_t rank, int32_t world, const void* unique_id128);
int mgc_slab_solve(mgc_graph* g, double* energy_total);
int mgc_slab_solve_stats(const mgc_graph* g, int64_t* exchanges, int64_t* relabel_rounds, int64_t* push_passes,
                         int64_t* global_relabels);
/* Device milliseconds of the last mgc_slab_solve per phase (CUDA events on the handle's stream): out6[0] local BFS,
 * [1] border exchanges (pack + ncclSend/ncclRecv + unpack), [2] stop test (count + all-reduce), [3] push passes,
 * [4] read-out + energy all-reduce, and out6[5] = HOST milliseconds spent blocked in the per-round synchronisations. */
int mgc_slab_solve_phase_ms(const mgc_graph* g, double* out6);

/* ---- general sparse graphs (SURVEY.md §8 rows f3/f4) ----------------------------------------------------- */

/* The graphs of the reference that are NOT voxel lattices: the region adjacency graph graph_from_labels builds
 * (generate.py:177-338) and graphs assembled call by call through GCGraph / GraphDouble (graph.py:382-498,
 * wrapper.cpp:63-83; e.g. tests/graphcut_/graph.py:47).  The handle replaces GraphDouble(nodes, edges) + add_node:
 * edges and terminal weights arrive in bulk (arrays of what would have been one call each, applied in array order with
 * the reference's accumulation semantics), the max-flow runs on the device as a CSR push-relabel (gc_sparse.cuh). */
typedef struct mgc_sparse mgc_sparse;
int mgc_sparse_create(int64_t n_nodes, int32_t device, mgc_sparse** out);
void mgc_sparse_destroy(mgc_sparse* g);
int mgc_sparse_reset(mgc_sparse* g);                           /* Graph::reset (graph.h:133) */
const char* mgc_sparse_last_error(const mgc_sparse* g);        /* g may be NULL: last create() failure */
/* count x Graph::sum_edge(i[k], j[k], cap[k], rev_cap[k]) (graph.h:456-480) in order: the first call for a node pair
 * creates its arc pair, later calls -- in either orientation -- accumulate with +=.  Host arrays.  MGC_E_ARG for ids
 * outside [0, n) or i == j (the ValueErrors of GCGraph.set_nweight, graph.py:418-435). */
int mgc_sparse_sum_edges(mgc_sparse* g, int64_t count, const int32_t* i, const int32_t* j, const double* cap,
                         const double* rev_cap);
/* count x Graph::add_tweights(nodes[k], src[k], snk[k]) (graph.h:415-425) in order; nodes == NULL means 0..count-1. */
int mgc_sparse_add_tweights(mgc_sparse* g, int64_t count, const int32_t* nodes, const double* src, const double* snk);
/* Graph::maxflow(): min-cut energy including the add_tweights constants.  Idempotent until the graph changes. */
int mgc_sparse_maxflow(mgc_sparse* g, double* energy);
/* out[v] = 0 if what_segment(v) == SINK else 1, for all n nodes (host buffer). */
int mgc_sparse_get_mask(mgc_sparse* g, uint8_t* out);
int mgc_sparse_what_segment(mgc_sparse* g, int64_t node, int32_t* segment);
/* Capacity of arc i->j / net terminal capacity as assembled so far (the values the reference's getters return before
 * maxflow(); 0 for unconnected pairs). */
int mgc_sparse_get_edge(const mgc_sparse* g, int64_t i, int64_t j, double* cap);
int mgc_sparse_get_trcap(const mgc_sparse* g, int64_t node, double* trcap);
int mgc_sparse_get_node_num(const mgc_sparse* g, int64_t* n);
int mgc_sparse_get_arc_num(const mgc_sparse* g, int64_t* n);    /* 2 per connected node pair */
int mgc_sparse_get_stats(const mgc_sparse* g, mgc_stats* out);
/* Warm re-solves of a general sparse graph (DESIGN.md §8, "Warm re-solve of sparse graphs").
 * mgc_sparse_set_option(g, MGC_OPT_WARM, 1): only on a handle that was not solved since create or mgc_sparse_reset
 * (MGC_E_STATE otherwise); the option survives mgc_sparse_reset.  The first solve of a warm handle keeps its device
 * state (about 16 B per arc and 41 B per node) until reset or destroy.  From then on mgc_sparse_sum_edges and
 * mgc_sparse_add_tweights fold into that residual state as the reference's calls act on its residual graph
 * (graph.h:415-480), and the next maxflow continues from it; MGC_E_ARG, with the handle unchanged, for bad ids, NaN or
 * infinite values, or a negative edge capacity.  The getters keep returning the values accumulated from scratch.  If
 * the first solve's graph held a NaN or infinite capacity or t-link, every fold returns MGC_E_STATE.
 * Without the option nothing changes: a call after a solve invalidates it and the next maxflow solves from scratch.
 * Adding these entry points left MGC_ABI_VERSION at 3 and mgc_stats unchanged (seed_folds / ms_seeds count the folds). */
int mgc_sparse_set_option(mgc_sparse* g, int32_t option, int64_t value);
/* count x sum_edge(i[k], j[k], -cap[k], -rev_cap[k]) on existing pairs, with nonnegative finite decrements, on a warm
 * handle (MGC_E_STATE without the option).  Per pair the decrements are summed in call order; the pair is refused with
 * MGC_E_WEIGHT, the handle unchanged, when δ + δ' − (r_ij + r_ji) > 2^-44 · max(r_ij + r_ji, δ + δ') (residual
 * capacities after a solve, accumulated ones before).  After a solve, flow beyond a lowered capacity is cancelled and a
 * node left short is covered by its terminal links (Kohli-Torr).  MGC_E_ARG for bad ids, a pair without an edge or NaN
 * / infinite values. */
int mgc_sparse_remove_edges_warm(mgc_sparse* g, int64_t count, const int32_t* i, const int32_t* j, const double* cap,
                                 const double* rev_cap);
/* Energies of a graph made of independent parts (DESIGN.md §8, "A batch of label images").
 * mgc_sparse_set_option(g, MGC_OPT_SEGMENT_ENERGIES, 1): before the first mgc_sparse_add_tweights and the first solve
 * since create or reset (MGC_E_STATE otherwise); it survives mgc_sparse_reset and may be combined with MGC_OPT_WARM.  The
 * handle then keeps the contribution to the constant of every add_tweights call made before the first solve (12 B per
 * call) and, after a solve, the flow each node's sink link absorbed (8 B per node on the device).  On a warm handle the
 * folds after the first solve also add each node's change of the constant into a per-node account (8 B per node more,
 * counted in device_bytes; cleared by mgc_sparse_reset).
 * mgc_sparse_get_segment_energies(g, B, node_off, out): node_off[0..B] ascending from 0 to n splits the nodes into B
 * ranges; out[b] = the constant of the logged calls on nodes of range b, summed in call order, + on a warm handle the
 * range's accounts, + the flow absorbed by those nodes in the current (resident) state; both device sums run in a fixed
 * order with no atomics, so two reads give the same bits (solves first if needed).  When no arc joins two ranges, out[b]
 * is the energy the range alone would have, and a range whose nodes no fold touched keeps its value bit for bit across
 * warm re-solves; mgc_sparse_maxflow keeps returning the total. */
#define MGC_OPT_SEGMENT_ENERGIES 4
int mgc_sparse_get_segment_energies(mgc_sparse* g, int64_t B, const int64_t* node_off, double* out);

/* ---- label images: the region adjacency graph built on the device (row f3) ------------------------------------ */

/* A label image resident in device memory.  Replaces what every energy_label term recomputes from the numpy array
 * (energy_label.py:78-86,181-189): mgc_labels_create stages `labels` (MGC_I32, any positive strides, logical shape
 * `shape[ndim]`, 1 <= ndim <= 4) once and runs __check_label_image (:444-456): MGC_E_LABELS unless the ids are
 * exactly 1..K.  Region r of the image is node r-1 of the graph (generate.py:334-337). */
typedef struct mgc_labels mgc_labels;
int mgc_labels_create(int32_t ndim, const int64_t* shape, const mgc_array* labels, int32_t device, mgc_labels** out);
void mgc_labels_destroy(mgc_labels* l);
const char* mgc_labels_last_error(const mgc_labels* l);       /* l may be NULL: last create() failure */
int mgc_labels_region_count(const mgc_labels* l, int64_t* k);
/* Boundary terms over all border voxel pairs (2*ndim-connectivity), reduced per region pair in the reference's own
 * accumulation order (axis by axis, C order inside an axis), so the sums equal what the chain of set_nweight ->
 * sum_edge calls leaves in the reference's arcs:
 *   MGC_LABELS_ADJACENCY  : __compute_edges_nd (energy_label.py:411-441): the pairs only (`values` ignored);
 *   MGC_LABELS_STAWIASKI  : boundary_stawiaski (:123-214): w = (1/(1+max(|g_p|,|g_q|)))^2, both directions;
 *   MGC_LABELS_STAWIASKI_DIRECTED : boundary_stawiaski_directed (:217-342) with `directedness` (incl. the double
 *                                   count of every axis' first pair that numpy.vectorize causes there).
 * `values` = gradient image (f32/f64/u8/i16/i32) over the same shape.  The result stays in the handle:
 * *n_edges region pairs, fetched with mgc_labels_fetch_edges into host arrays of that length, sorted by (i, j), i < j:
 * w_ij = capacity i->j, w_ji = capacity j->i. */
#define MGC_LABELS_ADJACENCY 0
#define MGC_LABELS_STAWIASKI 1
#define MGC_LABELS_STAWIASKI_DIRECTED 2
int mgc_labels_boundary(mgc_labels* l, int32_t kind, const mgc_array* values, double directedness, int64_t* n_edges);
int mgc_labels_fetch_edges(const mgc_labels* l, int32_t* i, int32_t* j, double* w_ij, double* w_ji);
/* Per-region sums of `values` and voxel counts (host arrays of K entries).
 *   MGC_SUM_BINCOUNT : numpy.bincount(labels, weights) as used by scipy.ndimage.mean (energy_label.py:92): float64,
 *                      front to back in C order;
 *   MGC_SUM_PAIRWISE : numpy.sum over the region's voxels in the array's own float type (regional_atlas,
 *                      energy_label.py:384-386): numpy's pairwise summation, reproduced exactly (integer arrays are
 *                      summed exactly either way). */
#define MGC_SUM_BINCOUNT 0
#define MGC_SUM_PAIRWISE 1
int mgc_labels_region_sums(mgc_labels* l, const mgc_array* values, int32_t mode, double* sums, int64_t* counts);
/* flags[r] = 1 if any voxel of region r+1 is marked (numpy.unique(label_image[markers] - 1), generate.py:334-337);
 * `markers` MGC_U8 over the same shape, flags = host array of K bytes. */
int mgc_labels_region_flags(mgc_labels* l, const mgc_array* markers, uint8_t* flags);
/* The flags of mgc_labels_region_flags from a list of marked voxels instead of a full marker image: flags[label[ids[t]]
 * - 1] = 1 for t < count, ids = host int64 voxel indices in [0, voxels) (C order; on a batch handle indices into the
 * concatenation), flags = host array of K bytes.  MGC_E_ARG for an id out of range, before any device work.  A stroke on
 * one image of a large batch then moves its own voxel ids instead of a marker image of the whole batch. */
int mgc_labels_voxel_flags(mgc_labels* l, int64_t count, const int64_t* ids, uint8_t* flags);
/* out[p] = per_region[label[p] - 1]: maps the cut back onto the voxels (bin/medpy_graphcut_label.py:139-148).
 * per_region = host array of K bytes; out = C-contiguous uint8 over the shape in host or device memory. */
int mgc_labels_apply(mgc_labels* l, const uint8_t* per_region, uint8_t* out, int32_t out_mem);
/* A batch of `batch` label images of `ndim` axes each, cut as one disjoint union of their region graphs (DESIGN.md §8,
 * "A batch of label images").  Image b has the extents shapes[b*ndim .. b*ndim+ndim-1]; the images may differ in shape.
 * `labels` (MGC_I32) is the images' C-ordered voxels concatenated image after image, passed as one 1-D array of
 * sum(voxels) elements.  Each image must hold exactly 1..K_b: MGC_E_LABELS otherwise, with last_error naming the image.
 * Label l of image b is node node_off[b] + l - 1, node_off the exclusive prefix of the K_b.  Refused before any
 * allocation (MGC_E_ARG): an image of 2^31 voxels or more, 2^31 voxels or more in all; then 2^31 regions or more in all
 * (node ids are int32), and from mgc_labels_boundary 2^32 border pairs or more in all.
 * On a batch handle every call above works on the concatenation: `values`, `markers` and `out` are 1-D arrays of
 * sum(voxels) elements laid out like `labels`, per-region arrays have sum(K_b) entries in node order, and
 * mgc_labels_region_count returns sum(K_b).  mgc_labels_boundary gives every image's own edge list (bit for bit what
 * mgc_labels_create + mgc_labels_boundary on that image gives, its ids shifted by node_off[b]), image after image; a
 * pair never crosses images.  The per-region sums are each image's own too. */
int mgc_labels_create_batch(int32_t batch, int32_t ndim, const int64_t* shapes, const mgc_array* labels, int32_t device,
                            mgc_labels** out);
/* node_off[0 .. batch]: the first node id of every image and the total (a handle of one image: {0, K}). */
int mgc_labels_batch_offsets(const mgc_labels* l, int64_t* node_off);

/* ---- K-label segmentation by alpha-expansion (DESIGN.md §11) ------------------------------------------------------ */

/* Labels 0..K-1 (2 <= K <= 255) over a lattice of shape[ndim] (1 <= ndim <= 4), minimising the Potts energy
 *   E(l) = sum_p D_p(l_p) + sum_{lattice pairs} w_pq [l_p != l_q]
 * by alpha-expansion (Boykov, Veksler & Zabih 2001): cycles of moves alpha = 0, 1, ..., K-1, each move one binary s-t cut
 * of the lattice on the eager handle and mgc_maxflow, until a full cycle switches no voxel or max_cycles cycles ran.
 *   D_p(k)  cost plane k at p widened to double; + 65535.0 (GCGraph.MAX) for every k != m-1 where the marker image holds
 *           m > 0 (the soft-hard seed of graph_from_voxels: with K = 2, marker 1 = background, 2 = foreground, the
 *           result is graph_from_voxels' cut)
 *   w_pq    the float64 weight mgc_add_boundary puts on both arcs of the pair; 0 without a boundary term
 * The move graph for alpha, its case table and the exactness argument are in DESIGN.md §11.  A voxel switches to alpha
 * only where its move's minimal sink set puts it, so a move that switches nothing shows that no expansion on alpha lowers
 * E.  Labels start from the init image, or argmin_k D_p(k) with ties to the lowest k.
 * Arrays are mgc_array over the lattice shape (host or device, any positive strides), borrowed for the call.  Adding
 * these entry points left MGC_ABI_VERSION at 3.
 * A refused input leaves nothing behind, here and in mgc_expansion_batch_* and mgc_region_expansion_*: set_cost,
 * set_markers and set_init unset that input (the label's costs, the markers, the init) and the last run's results before
 * they read it, and set it only once it passed its checks.  So after a refused cost plane the run returns MGC_E_STATE
 * until the label's costs are set again, and after refused markers or init it runs without them. */
typedef struct mgc_expansion mgc_expansion;
typedef struct mgc_expansion_stats {
    int64_t moves;          /* moves cut by the last run                                               */
    int64_t cycles;         /* cycles started (the last may be the one that switched nothing)          */
    int64_t converged;      /* 1: the last cycle switched no voxel; 0: max_cycles stopped the run       */
    double energy;          /* E of the final labels, fixed-order device sum (same labels, same bits)   */
    double ms_build;        /* device ms of the move kernels, summed over the moves                     */
    double ms_solve;        /* ... of mgc_maxflow (solve and read-out)                                  */
    double ms_apply;        /* ... of the label updates                                                 */
    double ms_total;        /* device ms of the whole run: initial labels to the energy                 */
} mgc_expansion_stats;
/* MGC_E_ARG for K outside 2..255 or a bad shape (as mgc_create). */
int mgc_expansion_create(int32_t ndim, const int64_t* shape, int32_t labels, int32_t device, mgc_expansion** out);
void mgc_expansion_destroy(mgc_expansion* e);
const char* mgc_expansion_last_error(const mgc_expansion* e);   /* e may be NULL: last create() failure */
/* Cost plane of one label: MGC_F32 or MGC_F64 (the same for every plane), finite and >= 0, else MGC_E_ARG. */
int mgc_expansion_set_cost(mgc_expansion* e, int32_t label, const mgc_array* cost);
/* The pair weights of one of the eight boundary terms, arguments as mgc_add_boundary (MGC_E_WEIGHT where it refuses);
 * replaces the weights of an earlier call. */
int mgc_expansion_set_boundary(mgc_expansion* e, int32_t kind, const mgc_array* image, double sigma, const double* spacing,
                               double norm);
/* MGC_U8 marker image, 0 = none, m = label m-1; MGC_E_ARG for a value above K. */
int mgc_expansion_set_markers(mgc_expansion* e, const mgc_array* markers);
/* MGC_U8 initial labels, each below K (MGC_E_ARG otherwise); mgc_expansion_run refuses (MGC_E_ARG) an init that gives a
 * marked voxel another label than its marker. */
int mgc_expansion_set_init(mgc_expansion* e, const mgc_array* init);
/* The move kind of mgc_expansion_run (and of the batch and region units' set_moves):
 *   MGC_MOVES_EXPANSION  (the default) cycles of alpha-expansions alpha = 0, 1, ..., K-1; the label distance must be a
 *                        metric
 *   MGC_MOVES_SWAP       cycles of alpha-beta swaps (0, 1), (0, 2), ..., (K-2, K-1), K(K-1)/2 moves per cycle; each
 *                        move is one binary cut in which only the voxels labelled alpha or beta take part, and the label
 *                        distance may be any semi-metric (the triangle rule is not needed), e.g. truncated quadratic
 *                        min((i - j)^2, T).  The move graph and the stop argument are in DESIGN.md §11, "Swap moves".
 * Any other kind is refused (MGC_E_ARG) and leaves the handle as it was.  set_moves clears the last run's results and
 * drops a label distance the handle holds, leaving it on Potts: call it before set_label_distance.  Adding it,
 * mgc_expansion_batch_set_moves and mgc_region_expansion_set_moves left MGC_ABI_VERSION at 3. */
#define MGC_MOVES_EXPANSION 0
#define MGC_MOVES_SWAP 1
int mgc_expansion_set_moves(mgc_expansion* e, int32_t kind);
/* A label distance: the pair term becomes w_pq V(l_p, l_q) in place of w_pq [l_p != l_q].  dist holds K x K host
 * doubles, row-major, borrowed for the call; every entry finite and >= 0, V[a][a] == 0, V[a][b] == V[b][a], and, under
 * expansion moves, V[a][c] <= V[a][b] + V[b][c] in float64 (zero off the diagonal is allowed).  A matrix that breaks a
 * rule is refused (MGC_E_ARG, the message names the rule and the first (a, b) or (a, b, c)) and leaves the handle on
 * Potts, as NULL does.  Semi-metrics such as truncated quadratic break the triangle inequality: alpha-expansion cannot
 * cut them exactly, so they need MGC_MOVES_SWAP, set before this call.  The move graphs with a distance are in DESIGN.md
 * §11, "Label distances" and "Swap moves"; V = 1 - I gives the Potts move graphs bit for bit.  Adding it,
 * mgc_expansion_batch_set_label_distance and mgc_region_expansion_set_label_distance left MGC_ABI_VERSION at 3. */
int mgc_expansion_set_label_distance(mgc_expansion* e, const double* dist);
/* MGC_E_STATE until every cost plane is set; max_cycles >= 1. */
int mgc_expansion_run(mgc_expansion* e, int32_t max_cycles);
/* After a run: the labels (uint8, C order, host or device), the statistics, and moves int64 switch counts, one per move. */
int mgc_expansion_get_labels(mgc_expansion* e, uint8_t* out, int32_t mem);
int mgc_expansion_get_stats(const mgc_expansion* e, mgc_expansion_stats* out);
int mgc_expansion_get_switched(const mgc_expansion* e, int64_t* out);

/* The same segmentation for B images of one shape image_shape[ndim] (1 <= ndim <= 3, B * voxels per image < 2^31), all
 * cut together: the images are stacked along axis 0 of one batch lattice (as mgc_create_batch stacks them), and every
 * move alpha is one move kernel, one mgc_maxflow and one label update over the whole batch.  Each image's move graphs are
 * bit for bit those mgc_expansion_* builds for it alone, and where the tile solver returns the minimal minimum cut of
 * every move (BK's), the image gets exactly the single run's labels, per-move switch counts, moves, cycles and converged
 * flag, and its energy up to the order of the sums.  The tile solver's floating-point residuals can, on some graphs,
 * leave an ulp on a saturated arc and so move voxels off the minimal cut; which graphs depends on the tile colour parity
 * of the image's position in the lattice, so on such a graph the batch and the single run can differ (DESIGN.md §11,
 * "Batches").  An image whose cycle switched no voxel is frozen from then on (its move
 * graphs are empty and its labels stay): its own run would have stopped there, and its labels are a fixed point of every
 * later move.  The batch loop stops after a cycle in which no image switched a voxel, or after max_cycles cycles.
 * Arrays are mgc_array of shape (B, *image_shape) (host or device, any positive strides), borrowed for the call; D_p(k),
 * markers and init have the meaning of mgc_expansion_*, image by image.  Adding these entry points left MGC_ABI_VERSION
 * at 3. */
typedef struct mgc_expansion_batch mgc_expansion_batch;
/* MGC_E_ARG for K outside 2..255, a batch < 1 or a bad shape (as mgc_create_batch). */
int mgc_expansion_batch_create(int32_t ndim, const int64_t* image_shape, int64_t batch, int32_t labels, int32_t device,
                               mgc_expansion_batch** out);
void mgc_expansion_batch_destroy(mgc_expansion_batch* e);
const char* mgc_expansion_batch_last_error(const mgc_expansion_batch* e);   /* e may be NULL: last create() failure */
/* Cost of one label for every image, (B, *image): MGC_F32 or MGC_F64 (the same for every label), finite and >= 0, else
 * MGC_E_ARG.  costs[:, k] of a (B, K, *image) device array goes in as it is (gathered on the device). */
int mgc_expansion_batch_set_cost(mgc_expansion_batch* e, int32_t label, const mgc_array* cost);
/* The pair weights of one of the eight boundary terms on the (B, *image) image, with one sigma and one linear normaliser
 * per image (NaN: reduced on the device over that image), as mgc_build_voxel_batch takes them; spacing has ndim entries
 * or is NULL.  The weights of image b are bit for bit those mgc_expansion_set_boundary gives that image alone (what
 * mgc_add_boundary writes on a fresh handle), 0 across the seams; MGC_E_WEIGHT where the build refuses.  Without this
 * call every weight is 0.  Replaces the weights of an earlier call. */
int mgc_expansion_batch_set_boundary(mgc_expansion_batch* e, int32_t kind, const mgc_array* image, const double* sigmas,
                                     const double* spacing, const double* norms);
/* MGC_U8 (B, *image) marker images, 0 = none, m = label m-1; MGC_E_ARG for a value above K. */
int mgc_expansion_batch_set_markers(mgc_expansion_batch* e, const mgc_array* markers);
/* MGC_U8 (B, *image) initial labels, each below K (MGC_E_ARG otherwise); mgc_expansion_batch_run refuses (MGC_E_ARG) an
 * init that gives a marked voxel another label than its marker. */
int mgc_expansion_batch_set_init(mgc_expansion_batch* e, const mgc_array* init);
/* The move kind of every image, as mgc_expansion_set_moves: a swap cycle gives each image K(K-1)/2 moves. */
int mgc_expansion_batch_set_moves(mgc_expansion_batch* e, int32_t kind);
/* The label distance of every image, as mgc_expansion_set_label_distance (NULL: Potts). */
int mgc_expansion_batch_set_label_distance(mgc_expansion_batch* e, const double* dist);
/* MGC_E_STATE until every cost plane is set; max_cycles >= 1 (per image, as mgc_expansion_run). */
int mgc_expansion_batch_run(mgc_expansion_batch* e, int32_t max_cycles);
/* After a run: the (B, *image) labels (uint8, C order, host or device). */
int mgc_expansion_batch_get_labels(mgc_expansion_batch* e, uint8_t* out, int32_t mem);
/* The batch loop: moves and cycles it ran, converged = 1 when every image converged, energy = the sum of the B image
 * energies in image order, and the device ms of its phases. */
int mgc_expansion_batch_get_stats(const mgc_expansion_batch* e, mgc_expansion_stats* out);
/* out[B]: per image its moves (K x cycles, or K(K-1)/2 x cycles under swap moves), cycles (the first cycle that switched none of its voxels, or max_cycles),
 * converged and energy (fixed-order device sum: same labels, same bits); the ms fields are 0. */
int mgc_expansion_batch_get_image_stats(const mgc_expansion_batch* e, mgc_expansion_stats* out);
/* out[moves x B], row-major: the voxels of image b the move switched (0 once b is frozen); image b's own switch counts
 * are the first moves_b rows of column b. */
int mgc_expansion_batch_get_switched(const mgc_expansion_batch* e, int64_t* out);
/* The pair weights along image axis `axis` (0..ndim-1) as a (B, *image) float64 array, host or device: entry p holds the
 * weight of the pair (p, p + e_axis), 0 on the last plane of the axis in every image. */
int mgc_expansion_batch_get_weights(mgc_expansion_batch* e, int32_t axis, double* out, int32_t mem);

/* Region labels 0..K-1 (2 <= K <= 255) over the R regions of a region adjacency graph (the nodes of graph_from_labels:
 * region r of a label image is node r-1), minimising the Potts energy
 *   E(l) = sum_r D_r(l_r) + sum_{region pairs r<s} w_rs [l_r != l_s]
 * by alpha-expansion: cycles of moves alpha = 0, 1, ..., K-1, each move one binary s-t cut of the region graph by the
 * sparse push-relabel, until a full cycle switches no region or max_cycles cycles ran.
 *   D_r(k)  entry r of the cost row of label k widened to double (marker seeds, if any, are the caller's additions)
 *   w_rs    the weight of the pair (r, s) given to mgc_region_expansion_set_pairs; 0 (no pair) otherwise
 * The handle keeps the CSR of the pairs on the device; a move writes only its capacities and t-links there (the per-arc
 * rules and the exactness argument are in DESIGN.md §11, "Region graphs") and a region switches to alpha only where the
 * move's minimal sink set puts it.  Labels start from the init labels, or argmin_k D_r(k) with ties to the lowest k.
 * Per-region arrays are 1-D mgc_array of R entries with unit stride (host or device), borrowed for the call.  The
 * statistics are those of mgc_expansion_*, with regions in place of voxels.  Adding these entry points left
 * MGC_ABI_VERSION at 3. */
typedef struct mgc_region_expansion mgc_region_expansion;
/* MGC_E_ARG for K outside 2..255 or R outside [1, 2^31-2]; device < 0: the current device. */
int mgc_region_expansion_create(int64_t regions, int32_t labels, int32_t device, mgc_region_expansion** out);
void mgc_region_expansion_destroy(mgc_region_expansion* e);
const char* mgc_region_expansion_last_error(const mgc_region_expansion* e);   /* e may be NULL: last create() failure */
/* Cost row of one label: R entries, MGC_F32 or MGC_F64 (the same for every row), finite and >= 0, else MGC_E_ARG. */
int mgc_region_expansion_set_cost(mgc_region_expansion* e, int32_t label, const mgc_array* cost);
/* The pairs: host arrays of `count` entries, 0 <= i[k] < j[k] < R, (i, j) strictly ascending, w finite and >= 0, else
 * MGC_E_ARG.  A second call replaces the pairs. */
int mgc_region_expansion_set_pairs(mgc_region_expansion* e, int64_t count, const int32_t* i, const int32_t* j,
                                   const double* w);
/* MGC_U8 initial region labels, each below K (MGC_E_ARG otherwise). */
int mgc_region_expansion_set_init(mgc_region_expansion* e, const mgc_array* init);
/* The move kind, as mgc_expansion_set_moves. */
int mgc_region_expansion_set_moves(mgc_region_expansion* e, int32_t kind);
/* The label distance, as mgc_expansion_set_label_distance (NULL: Potts): the pair term becomes w_rs V(l_r, l_s). */
int mgc_region_expansion_set_label_distance(mgc_region_expansion* e, const double* dist);
/* MGC_E_STATE until every cost row is set; max_cycles >= 1. */
int mgc_region_expansion_run(mgc_region_expansion* e, int32_t max_cycles);
/* After a run: the R region labels (uint8, host or device), the statistics, and moves int64 switch counts. */
int mgc_region_expansion_get_labels(mgc_region_expansion* e, uint8_t* out, int32_t mem);
int mgc_region_expansion_get_stats(const mgc_region_expansion* e, mgc_expansion_stats* out);
int mgc_region_expansion_get_switched(const mgc_region_expansion* e, int64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* MEDPY_B200_GRAPHCUT_H */
