"""``medpy_b200.graphcut.maxflow`` -- the object ``graph_from_voxels`` returns.

Mirror of the reference's compiled module ``medpy.graphcut.maxflow`` (Boost.Python,
lib/maxflow/src/wrapper.cpp:59-89): class ``GraphDouble`` with ``add_tweights / sum_edge / add_edge /
maxflow / what_segment / get_edge / get_trcap / get_node_num / get_arc_num / reset`` and the nested enum
``termtype`` (wrapper.cpp:85-88).  Storage is NOT the reference's node/arc lists: the graph is a dense
2*ndim-connected lattice living in device memory behind the C ABI (include/medpy_b200_graphcut.h); whole energy
terms are handed to CUDA kernels, element-wise calls are staged in dense host arrays and uploaded in bulk.

There is no CPU solver here: the first operation that needs the device creates the native graph and
raises ``RuntimeError`` when no CUDA device / built extension is available.
"""
import enum

import numpy

from . import _warm_args

__all__ = ["GraphDouble", "GraphFloat", "GraphInt"]


class _termtype(enum.IntEnum):
    """graph.h:57-61: terminals."""
    SOURCE = 0
    SINK = 1


def _strides_of(shape):
    st = []
    acc = 1
    for s in reversed(shape):
        st.append(acc)
        acc *= int(s)
    return tuple(reversed(st))


def _cannot_fold(rebuild):
    """The refusal of a warm call that a solved general sparse graph, created without warm=True, cannot fold."""
    return RuntimeError("a warm re-solve needs a lattice graph built by graph_from_voxels; reset() the graph and rebuild "
                        "it {} instead".format(rebuild))


class GraphDouble:
    """Lattice max-flow graph with the reference's ``GraphDouble`` method names.

    ``GraphDouble(node_num_max, edge_num_max, shape=None)``: ``shape`` is the logical lattice shape (C-order
    node ids, generate.py:170-172); without it the graph is a 1-D chain of ``node_num_max`` nodes.
    """

    termtype = _termtype

    def __init__(self, node_num_max, edge_num_max=0, shape=None, device=-1, sparse=None, warm=False):
        # Without a lattice shape the graph starts as a 1-D chain (what element-wise users of the voxel path build) and
        # keeps a journal of its calls; the first edge that does not join chain neighbours -- or sparse=True -- moves
        # it, journal and all, onto the general sparse backend (sparse.py, SURVEY.md §8 row f4).  warm=True (with
        # sparse=True only) makes the sparse graph fold calls made after a solve into its residual state.
        if warm and not sparse:
            raise ValueError("warm=True needs sparse=True; lattice graphs call enable_warm() instead")
        self._sp = None
        self._sp_warm = bool(warm)
        self._journal = [] if shape is None else None
        if shape is None:
            shape = (int(node_num_max),)
        shape = tuple(int(s) for s in shape)
        if len(shape) < 1 or len(shape) > 4:
            raise ValueError("the lattice path supports 1 to 4 dimensions, got shape {}".format(shape))
        n = 1
        for s in shape:
            n *= s
        if n != int(node_num_max):
            raise ValueError("shape {} does not hold {} nodes".format(shape, node_num_max))
        self._shape = shape
        self._n = n
        self._strides = _strides_of(shape)
        self._edges = int(edge_num_max)
        self._device = device
        self._native = None
        # element-wise staging (dense host arrays, flushed in bulk)
        self._st_src = None
        self._st_snk = None
        self._st_touched = None
        self._st_nw = {}  # axis -> [fwd, bwd] dense arrays
        self._mask = None
        self._offlattice = None
        self._pending = []
        self._defer_weight_check = False
        self._warm = False       # enable_warm(): MGC_OPT_WARM, set on the native handle when it is created
        # whole-lattice terms collected while graph_from_voxels runs (regional, boundary, markers): handed to the device
        # in ONE native call (mgc_build_voxel_graph: single-pass fused build) when the markers arrive or anything else
        # needs the graph.  Only while nothing has reached the device yet (_fresh).
        self._lazy = None
        self._fresh = True
        self._solved = False     # maxflow() ran since the last reset: add_seeds folds into the residual state
        # a removal folded into the handle before the first maxflow(): the terms are fixed from then on, and the warm
        # calls fold natively as on a solved graph
        self._folded = False
        if sparse:
            if self._journal is None:
                raise ValueError("a lattice shape and sparse=True exclude each other")
            self._to_sparse()

    def _to_sparse(self):
        from .sparse import SparseGraphDouble
        sp = SparseGraphDouble(self._n, self._edges, device=self._device, warm=getattr(self, "_sp_warm", False))
        for op in self._journal or []:
            if op[0] == "e":
                sp.sum_edge(op[1], op[2], op[3], op[4])
            elif op[0] == "t":
                sp.add_tweights(op[1], op[2], op[3])
            else:
                sp.add_tweights_bulk(op[1], op[2], op[3])
        self._journal = None
        self._sp = sp
        # drop the chain-lattice staging and device state
        self._st_src = self._st_snk = self._st_touched = None
        self._st_nw = {}
        self._pending = []
        self._native = None
        self._mask = None

    @property
    def is_sparse(self):
        return self._sp is not None

    def _warm_sparse(self):
        """A sparse graph created with warm=True: its warm calls are the sparse backend's (sparse.py)."""
        return self._sp is not None and self._sp.warm

    # ------------------------------------------------------------------ native handle
    @property
    def shape(self):
        return self._shape

    def _nat(self):
        if self._sp is not None:
            raise TypeError("this graph is a general sparse graph: lattice terms (energy_voxel.*) need a graph created "
                            "with a lattice shape")
        if self._native is None:
            from .. import _lib  # raises ImportError loudly when the extension is not built
            self._native = _lib.Graph(list(self._shape), self._device)
            if self._defer_weight_check:
                self._native.set_option(_lib._mgc.OPT_DEFER_WEIGHT_CHECK, 1)
            if self._warm:
                self._native.set_option(_lib._mgc.OPT_WARM, 1)
        return self._native

    def enable_warm(self):
        """Let ``add_seeds``, ``remove_seeds`` and ``add_tweights_warm`` fold into this graph after ``maxflow()`` although
        the lazy fused build did not make it: a 4-D graph, a graph built term by term (element-wise calls,
        ``add_nweights_dense``, ``add_regional_probability`` / ``add_boundary`` / ``add_markers``) or by the eager fused
        build (``MEDPY_GC_LAZY_CAPS=0``).

        Call it before the first ``maxflow()`` -- the graph ``graph_from_voxels`` returns is built but not solved yet, so
        ``g = graph_from_voxels(...); g.enable_warm(); g.maxflow()`` is the order.  The first solve then records the residual
        source capacities the folds read (``mgc_set_option(MGC_OPT_WARM)``); its mask and energy are those without the
        call.  The setting survives ``reset()``.  On a graph the lazy fused build made it changes nothing.  A solved graph
        that cannot fold raises ``RuntimeError``, a sparse graph ``TypeError``."""
        if self._sp is not None:
            if self._sp.warm:
                return                      # created with warm=True: already warm
            raise TypeError("enable_warm() needs a lattice graph: a general sparse graph has no warm re-solve unless it "
                            "is created with warm=True")
        if self._native is not None:
            from .. import _lib
            try:
                self._native.set_option(_lib._mgc.OPT_WARM, 1)
            except RuntimeError:
                raise RuntimeError("this graph was solved without a warm path: call enable_warm() before the first "
                                   "maxflow(); reset() the graph and rebuild it to re-solve it warm") from None
        self._warm = True

    def defer_weight_check(self, on=True):
        """Let a boundary term return before its kernel has reported non-positive weights; the ValueError is then
        raised by the next call on the graph (graph_from_voxels adds the markers right after the boundary term, so the
        marker upload overlaps the stencil kernel).  ``check_deferred()`` forces the verdict."""
        if not on:
            self._commit()
        self._defer_weight_check = bool(on)
        if self._native is not None:
            from .. import _lib
            self._native.set_option(_lib._mgc.OPT_DEFER_WEIGHT_CHECK, 1 if on else 0)

    def check_deferred(self):
        self._commit()
        if self._native is not None:
            self._native.check_deferred()

    # ------------------------------------------------------------------ collected whole-lattice terms
    def _collect(self, key, value):
        """Record a whole-lattice term instead of launching it; False if it has to run right away (the graph already
        holds terms, element-wise calls are staged, the same kind of term was collected before, or collection is off)."""
        if not self._defer_weight_check or not self._fresh or self._sp is not None:
            return False
        if self._st_src is not None or self._st_nw or self._pending:
            return False
        if self._lazy is not None and key in self._lazy:
            return False
        if self._lazy is None:
            self._lazy = {}
        self._lazy[key] = value
        return True

    def _commit(self):
        """Hand the collected terms to the device: regional term, boundary term, fg / bg markers in the reference's
        order (generate.py:159-172), as one fused pass where the native side can (mgc_build_voxel_graph)."""
        lazy, self._lazy = self._lazy, None
        if not lazy:
            return
        self._fresh = False
        prob, alpha, f32 = lazy.get("reg", (None, 0.0, False))
        kind, image, sigma, spacing, norm = lazy.get("bnd", (-1, None, 0.0, None, float("nan")))
        fg, bg = lazy.get("mark", (None, None))
        self._nat().build_voxel_graph(prob, float(alpha), bool(f32), int(kind), image, float(sigma), spacing, float(norm), fg, bg)

    def _dirty(self):
        self._mask = None

    # ------------------------------------------------------------------ staging of element-wise calls
    # Element-wise calls (add_tweights / sum_edge, i.e. GCGraph.set_tweight / set_nweight / set_source_nodes)
    # never touch the device: they fill dense host batches that are uploaded in call order by _flush().
    def _close_tweight_batch(self):
        if self._st_src is not None:
            self._pending.append(("tw", self._st_src, self._st_snk))
            self._st_src = self._st_snk = self._st_touched = None

    def _open_tweight_batch(self):
        if self._st_src is None:
            self._st_src = numpy.zeros(self._n, dtype=numpy.float64)
            self._st_snk = numpy.zeros(self._n, dtype=numpy.float64)
            self._st_touched = numpy.zeros(self._n, dtype=numpy.bool_)

    def stage_tweights_many(self, ids, cap_source, cap_sink):
        """add_tweights(v, cap_source, cap_sink) for every v in ids, in order (ids already range-checked)."""
        self._terms_open()
        ids = numpy.asarray(ids, dtype=numpy.int64)
        if self._sp is not None:
            return self._sp.stage_tweights_many(ids, cap_source, cap_sink)
        if self._journal is not None:
            self._journal.append(("T", ids.copy(), numpy.full(ids.size, float(cap_source)), numpy.full(ids.size, float(cap_sink))))
        self._dirty()
        self._open_tweight_batch()
        if numpy.unique(ids).size == ids.size:
            if self._st_touched[ids].any():
                self._close_tweight_batch()
                self._open_tweight_batch()
            self._st_src[ids] = float(cap_source)
            self._st_snk[ids] = float(cap_sink)
            self._st_touched[ids] = True
        else:
            for v in ids:
                self._add_tweights_staged(int(v), cap_source, cap_sink)

    def _flush(self):
        self._commit()
        self._close_tweight_batch()
        if self._st_nw:
            for axis in sorted(self._st_nw):
                fwd, bwd = self._st_nw[axis]
                self._pending.append(("nw", axis, fwd, bwd))
            self._st_nw = {}
        pending, self._pending = self._pending, []
        if pending:
            self._fresh = False
        for op in pending:
            if op[0] == "tw":
                self._nat().add_tweights_dense(op[1].reshape(self._shape), op[2].reshape(self._shape))
            else:
                # pairs never set stay 0, which sum_edge semantics allow (graph.h:456-463 asserts cap >= 0)
                self._nat().add_nweights_dense(op[1], op[2].reshape(self._shape), op[3].reshape(self._shape))

    # ------------------------------------------------------------------ bulk term entry points (used by energy_voxel)
    def _lattice_term(self):
        """A whole-lattice term is about to be applied: a shape-less graph that takes one stays the 1-D chain it was
        created as (its journal cannot describe device-side terms, so it can no longer move to the sparse backend)."""
        if self._sp is None:
            self._journal = None

    def add_regional_probability(self, prob, alpha, compute_f32):
        self._terms_open()
        self._lattice_term()
        self._dirty()
        if self._collect("reg", (self._positive_strides(prob), float(alpha), bool(compute_f32))):
            return
        self._flush()
        self._fresh = False
        self._nat().add_regional_probability(self._positive_strides(prob), float(alpha), bool(compute_f32))

    def add_tweights_dense(self, src, snk):
        """add_tweights(v, src[v], snk[v]) for every node (GCGraph.set_tweights_all, graph.py:532-552)."""
        self._terms_open()
        if self._sp is not None:
            return self._sp.add_tweights_bulk(None, numpy.ravel(src), numpy.ravel(snk))
        src = numpy.ascontiguousarray(src, dtype=numpy.float64).reshape(self._shape)
        snk = numpy.ascontiguousarray(snk, dtype=numpy.float64).reshape(self._shape)
        if self._journal is not None:
            # shape-less graph: staged like the element-wise calls (no device needed yet) and journaled node-wise, so a
            # later move to the sparse backend can replay it
            self._journal.append(("T", numpy.arange(self._n), src.ravel().copy(), snk.ravel().copy()))
            self._close_tweight_batch()
            self._pending.append(("tw", src.ravel().copy(), snk.ravel().copy()))
            self._dirty()
            return
        self._flush()
        self._dirty()
        self._fresh = False
        self._nat().add_tweights_dense(src, snk)

    @staticmethod
    def _positive_strides(a):
        """Host arrays with zero / negative strides (broadcast views, reversed slices) are copied once; everything
        else -- including Fortran-ordered arrays as medpy.io.load returns them -- is handed over as is."""
        if a is None or not isinstance(a, numpy.ndarray):
            return a
        if any(st <= 0 and n > 1 for st, n in zip(a.strides, a.shape)):
            return numpy.ascontiguousarray(a)
        return a

    def add_markers(self, fg, bg):
        self._terms_open()
        self._lattice_term()
        self._dirty()
        if self._lazy and "mark" not in self._lazy and self._collect("mark", (self._positive_strides(fg), self._positive_strides(bg))):
            return self._commit()        # the markers are graph_from_voxels' last step: build now
        self._flush()
        self._fresh = False
        self._nat().add_markers(self._positive_strides(fg), self._positive_strides(bg))

    def add_boundary(self, kind, image, sigma, spacing, norm):
        self._terms_open()
        self._lattice_term()
        self._dirty()
        if self._collect("bnd", (int(kind), self._positive_strides(image), float(sigma), spacing, float(norm))):
            return
        self._flush()
        self._fresh = False
        self._nat().add_boundary(int(kind), self._positive_strides(image), float(sigma), spacing, float(norm))

    def add_nweights_dense(self, axis, fwd, bwd):
        self._terms_open()
        self._lattice_term()
        self._flush()
        self._dirty()
        self._fresh = False
        self._nat().add_nweights_dense(int(axis), fwd, bwd)

    # ------------------------------------------------------------------ reference GraphDouble API
    def add_node(self, num=1):
        """graph.h:388-413.  Nodes are implied by the lattice; returns the id the reference would."""
        return 0

    def add_tweights(self, i, cap_source, cap_sink):
        """graph.h:415-425, staged: calls on distinct nodes are batched into one dense device pass.  A solved graph
        refuses it; ``add_tweights_warm`` is the warm form, which folds the calls into the solved state."""
        self._terms_open()
        i = int(i)
        if i < 0 or i >= self._n:
            raise ValueError("Invalid node id of {}. Valid values are 0 to {}.".format(i, self._n - 1))
        if self._sp is not None:
            return self._sp.add_tweights(i, cap_source, cap_sink)
        if self._journal is not None:
            self._journal.append(("t", i, float(cap_source), float(cap_sink)))
        self._add_tweights_staged(i, cap_source, cap_sink)

    def _add_tweights_staged(self, i, cap_source, cap_sink):
        self._open_tweight_batch()
        if self._st_touched[i]:
            self._close_tweight_batch()  # add_tweights is order dependent per node: start a new batch
            self._open_tweight_batch()
        self._st_src[i] = float(cap_source)
        self._st_snk[i] = float(cap_sink)
        self._st_touched[i] = True
        self._dirty()

    def _axis_of(self, i, j):
        d = j - i
        for axis, st in enumerate(self._strides):
            if abs(d) == st and self._shape[axis] > 1:
                lo = min(i, j)
                if (lo // st) % self._shape[axis] < self._shape[axis] - 1:
                    return axis
        return None

    def sum_edge(self, i, j, cap, rev_cap):
        """graph.h:456-480 for lattice neighbours (accumulating)."""
        self._terms_open()
        i, j = int(i), int(j)
        if i < 0 or j < 0 or i >= self._n or j >= self._n or i == j:
            raise ValueError("invalid node ids ({}, {})".format(i, j))
        if self._sp is not None:
            return self._sp.sum_edge(i, j, cap, rev_cap)
        axis = self._axis_of(i, j)
        if axis is None:
            if self._journal is not None:
                # not a chain neighbour: this is a general graph (tests/graphcut_/graph.py:47) -> sparse backend
                self._to_sparse()
                return self._sp.sum_edge(i, j, cap, rev_cap)
            # a lattice graph (graph_from_voxels) accepts the call like the reference would, but an edge between
            # non-neighbours can never be solved on the lattice; maxflow() refuses.
            self._offlattice = (i, j)
            return
        if self._journal is not None:
            self._journal.append(("e", i, j, float(cap), float(rev_cap)))
        if axis not in self._st_nw:
            self._st_nw[axis] = [numpy.zeros(self._n, dtype=numpy.float64), numpy.zeros(self._n, dtype=numpy.float64)]
        fwd, bwd = self._st_nw[axis]
        if i < j:
            fwd[i] += float(cap)
            bwd[i] += float(rev_cap)
        else:
            fwd[j] += float(rev_cap)
            bwd[j] += float(cap)
        self._dirty()

    add_edge = sum_edge  # graph.h:427-454: parallel arcs act as summed capacities

    def sum_edges_bulk(self, i, j, cap, rev_cap):
        """One sum_edge call per array entry, in order (general graphs: moves the graph to the sparse backend)."""
        if self._sp is None:
            if self._journal is None:
                raise ValueError("bulk edges between arbitrary nodes need a graph without lattice shape")
            self._to_sparse()
        self._sp.sum_edges_bulk(i, j, cap, rev_cap)

    def add_tweights_bulk(self, nodes, src, snk):
        """One add_tweights call per array entry, in order."""
        if self._sp is not None:
            return self._sp.add_tweights_bulk(nodes, src, snk)
        nodes = numpy.arange(len(src)) if nodes is None else numpy.asarray(nodes)
        for v, a, b in zip(nodes.tolist(), numpy.asarray(src, dtype=float).tolist(), numpy.asarray(snk, dtype=float).tolist()):
            self.add_tweights(v, a, b)

    def maxflow(self):
        """Graph::maxflow (maxflow.cpp:471-604): min-cut energy including the add_tweights constants."""
        if self._sp is not None:
            return self._sp.maxflow()
        if self._offlattice is not None:
            raise NotImplementedError(
                "edge {} does not join lattice neighbours of shape {}: build general graphs with "
                "GraphDouble(nodes, edges) (no shape), which uses the sparse backend".format(self._offlattice, self._shape))
        self._flush()
        flow = self._nat().maxflow()
        self._solved = True
        return flow

    def add_seeds(self, fg=None, bg=None):
        """Add foreground / background seeds and let the next ``maxflow()`` return the cut of the enlarged graph.

        Exactly ``add_tweights(v, 65535, 0)`` for every foreground id in order, then ``add_tweights(v, 0, 65535)`` for
        every background id (GCGraph.set_source_nodes / set_sink_nodes, graph.py:310-380).  ``fg`` / ``bg``: a boolean
        mask of the lattice shape, a 1-D integer id array (repeated ids count once per occurrence), or None.

        Before the first ``maxflow()`` the calls are staged like ``add_tweights``.  After it, on a graph that
        ``graph_from_voxels`` built in one fused pass (1-D..3-D lattice on one GPU), the seeds are folded into the solved
        state and the next solve continues from the flow already routed (mgc_add_seeds); so on any lattice graph that called
        ``enable_warm()`` before its first solve.  Any other solved graph raises ``RuntimeError``: ``reset()`` it and
        build the graph again with the seeds."""
        if self._warm_sparse():
            return self._sp.add_seeds(fg, bg)
        self._fold_seeds(fg, bg, 65535.0, "add_seeds", "with the seeds")

    def remove_seeds(self, fg=None, bg=None):
        """Erase foreground / background seeds and let the next ``maxflow()`` return the cut of the reduced graph.

        The inverse of ``add_seeds``, as the reference erases a seed: exactly ``add_tweights(v, -65535, 0)`` for every
        foreground id in order, then ``add_tweights(v, 0, -65535)`` for every background id.  ``fg`` / ``bg`` take the
        same forms as in ``add_seeds``; repeated ids count once per occurrence.  The markers ``graph_from_voxels`` put
        into the graph are the same ``add_tweights`` calls, so this erases them as well as seeds added later.  Nothing
        checks that a seed was there: erasing one that was never added applies the call anyway, as the reference does.

        Before the first ``maxflow()`` the calls are staged like ``add_tweights``.  After it the seeds are folded into
        the solved state on the same graphs as ``add_seeds`` (``enable_warm()`` included, mgc_remove_seeds); any other
        solved graph raises
        ``RuntimeError``: ``reset()`` it and build the graph again without the seeds."""
        if self._warm_sparse():
            return self._sp.remove_seeds(fg, bg)
        self._fold_seeds(fg, bg, -65535.0, "remove_seeds", "without the seeds")

    def _fold_seeds(self, fg, bg, cap, native, rebuild):
        ids = _warm_args.seed_args(fg, bg, self._shape, self._n, mixed=True)
        self._warm_call(native, ids, lambda f, b: self._stage_seeds(f, b, cap), rebuild)

    def _stage_seeds(self, fg, bg, cap):
        for ids, src, snk in ((fg, cap, 0.0), (bg, 0.0, cap)):
            if ids is not None and len(ids):
                self.stage_tweights_many(ids, src, snk)

    def _warm_call(self, native, args, stage, rebuild):
        """One warm call on parsed arguments: before the first solve (and before a removal folded) ``stage`` takes host
        copies of them; after it the native fold ``native`` reads them where they are.  ``rebuild`` completes the refusal
        of a graph that cannot fold."""
        if not self._solved and not self._folded:
            return stage(*(a.cpu().numpy() if _warm_args.on_device(a) else a for a in args))
        if self._sp is not None:
            raise _cannot_fold(rebuild)
        self._dirty()
        getattr(self._nat(), native)(*args)

    def add_tweights_warm(self, nodes, cap_source, cap_sink):
        """``add_tweights`` calls on a solved graph, re-solved warm by the next ``maxflow()``: soft strokes, a GrabCut-style
        update of the regional term, a new weight between the regional and the boundary term.

        ``nodes``: a 1-D integer id array (or a boolean mask of the lattice shape, ids in logical C order), one call
        ``add_tweights(nodes[k], cap_source[k], cap_sink[k])`` per entry in order, repeated ids once per occurrence; or
        None for the dense form, ``add_tweights(v, cap_source[v], cap_sink[v])`` for every node in C order
        (``GCGraph.set_tweights_all`` on a solved graph), where ``cap_source`` / ``cap_sink`` have the lattice shape (any
        strides, read in logical C order) or one entry per node.  Scalars broadcast.  Weights are finite reals of either
        sign, widened to float64.  numpy arrays or CUDA tensors, all in one memory space.  Bad ids, lengths, shapes or NaN
        / infinite weights raise ``ValueError``.

        Before the first ``maxflow()`` the calls are staged like ``add_tweights``.  After it, on a graph that
        ``graph_from_voxels`` built in one fused pass (1-D..3-D lattice on one GPU), they are folded into the solved state
        and the next solve continues from the flow already routed (mgc_add_tweights_warm); so on any lattice graph that
        called ``enable_warm()`` before its first solve.  Any other solved graph raises ``RuntimeError``: ``reset()`` it and
        build the graph again with the calls."""
        if self._warm_sparse():
            return self._sp.add_tweights_warm(nodes, cap_source, cap_sink)
        ids, src, snk = _warm_args.tlink_args(nodes, cap_source, cap_sink, self._shape, self._n,
                                              ("nodes", "cap_source", "cap_sink"))
        self._warm_call("add_tweights_warm", (ids, src, snk), self._stage_tweights_calls, "with the t-link calls")

    def add_nweights_warm(self, i, j, cap, rev_cap):
        """``sum_edge`` calls on a solved graph, re-solved warm by the next ``maxflow()``: a boundary brush ("do not cut
        here"), a larger boundary weight, a second boundary term.

        One call ``sum_edge(i[k], j[k], cap[k], rev_cap[k])`` per entry, in order, applied to the residual capacities as
        the reference applies it to a solved graph (graph.h:456-480); repeated pairs count once per occurrence.  ``i`` /
        ``j``: 1-D integer arrays of lattice-neighbour node ids in logical C order; ``cap`` / ``rev_cap``: nonnegative
        finite reals, widened to float64.  Scalars broadcast.  numpy arrays or CUDA tensors, all in one memory space.  Bad
        ids, pairs that are not lattice neighbours, lengths, negative, NaN or infinite weights raise ``ValueError``.

        Before the first ``maxflow()`` the calls are staged exactly like ``sum_edge``.  After it they are folded into the
        solved state on the graphs ``add_tweights_warm`` folds into (mgc_add_nweights_warm); any other solved graph raises
        ``RuntimeError``: ``reset()`` it and build the graph again with the calls."""
        if self._warm_sparse():
            return self._sp.add_nweights_warm(i, j, cap, rev_cap)
        ii, jj, c, r, _ = _warm_args.nlink_args(i, j, cap, rev_cap, self._n)
        self._warm_call("add_nweights_warm", (ii, jj, c, r), self._stage_nweights_calls, "with the n-link calls")

    def add_nweights_dense_warm(self, axis, fwd, bwd):
        """The dense form of ``add_nweights_warm``, in the layout of ``add_nweights_dense``: ``fwd`` / ``bwd`` have the
        lattice shape (any strides, read in logical C order) and entry p holds the increments of the arcs p -> p + e_axis
        and back; the last plane of ``axis`` is ignored.  Entries are nonnegative finite reals, widened to float64; only the
        pairs with a nonzero entry are touched.  numpy arrays or CUDA tensors, both in one memory space.  A bad axis or
        shape, negative, NaN or infinite weights raise ``ValueError``.

        Before the first ``maxflow()`` the call is staged exactly like ``add_nweights_dense``.  After it, the same graphs
        as ``add_nweights_warm`` fold it into the solved state (mgc_add_nweights_dense_warm)."""
        if self._warm_sparse():
            return self._sp.add_nweights_dense_warm(axis, fwd, bwd)
        axis, fwd, bwd, _ = _warm_args.nlink_dense_args(axis, fwd, bwd, self._shape)
        self._warm_call("add_nweights_dense_warm", (axis, fwd, bwd), self._stage_nweights_dense, "with the n-link calls")

    def _stage_nweights_dense(self, axis, fwd, bwd):
        """add_nweights_dense_warm before the first solve: checked like the warm fold checks it, then staged exactly like
        ``add_nweights_dense``."""
        cut = _warm_args.pair_entries(self._shape, axis)
        _warm_args.check_amounts(((fwd[cut], "fwd"), (bwd[cut], "bwd")), _warm_args.ONLY_RAISES)
        staged = [numpy.zeros(self._shape), numpy.zeros(self._shape)]
        staged[0][cut], staged[1][cut] = fwd[cut], bwd[cut]
        self.add_nweights_dense(axis, *staged)

    def remove_nweights_warm(self, i, j, cap, rev_cap):
        """The inverse of ``add_nweights_warm``: n-link capacity taken off the graph, re-solved warm by the next
        ``maxflow()`` -- a boundary brush undone, a lower boundary weight, a boundary relaxed along a cut.

        Exactly ``sum_edge(i[k], j[k], -cap[k], -rev_cap[k])`` per entry, in order: the next ``maxflow()`` returns the cut
        and the energy of the graph built from scratch with every call so far and these decrements subtracted.  ``cap`` /
        ``rev_cap`` are the decrements, nonnegative finite reals; the arguments take the forms of ``add_nweights_warm``.
        The caller promises that every capacity stays >= 0; a pair whose residual capacities r(i->j) + r(j->i) (which
        equal c(i->j) + c(j->i)) fall short of its total decrement beyond a few hundred roundings raises ``ValueError``,
        and the graph is left as it was.  On a solved graph an arc may carry more flow than its lowered capacity: that
        flow is cancelled and the terminal links make up the difference (a documented extension of the reference, whose
        BK has no meaning for it; see mgc_remove_nweights_warm).

        Before the first ``maxflow()`` the pending build is flushed and the calls are folded into it natively (staging
        cannot lower a capacity).  The graph's terms are fixed from then on: a later term call (``add_tweights``,
        ``sum_edge``, the whole-lattice terms) raises ``RuntimeError``, and the warm calls fold natively as on a solved
        graph.  So make every term call before the first removal.  The graphs ``add_nweights_warm`` folds into take the calls; any other graph raises
        ``RuntimeError``: ``reset()`` it and build the graph again without the weight."""
        if self._warm_sparse():
            return self._sp.remove_nweights_warm(i, j, cap, rev_cap)
        ii, jj, c, r, cuda = _warm_args.nlink_args(i, j, cap, rev_cap, self._n)
        if not cuda:        # the native grouping checks device decrements in the same pass
            _warm_args.check_amounts(((c, "cap"), (r, "rev_cap")), _warm_args.DECREMENTS)
        self._fold_decrements("remove_nweights_warm", ii, jj, c, r)

    def remove_nweights_dense_warm(self, axis, fwd, bwd):
        """The dense form of ``remove_nweights_warm``, in the layout of ``add_nweights_dense_warm``: entry p of ``fwd`` /
        ``bwd`` holds the decrements of the arcs p -> p + e_axis and back; the last plane of ``axis`` is ignored and only
        the pairs with a nonzero entry are touched.  Same meaning, checks and errors as ``remove_nweights_warm``."""
        if self._warm_sparse():
            return self._sp.remove_nweights_dense_warm(axis, fwd, bwd)
        axis, fwd, bwd, cuda = _warm_args.nlink_dense_args(axis, fwd, bwd, self._shape)
        if not cuda:
            cut = _warm_args.pair_entries(self._shape, axis)
            _warm_args.check_amounts(((fwd[cut], "fwd"), (bwd[cut], "bwd")), _warm_args.DECREMENTS)
        self._fold_decrements("remove_nweights_dense_warm", axis, fwd, bwd)

    def _terms_open(self):
        """Term calls are refused once a removal has folded into the graph before its first solve: the handle then holds
        a residual state, which staged terms cannot be added to."""
        if self._folded:
            raise RuntimeError("an n-link removal was folded into this graph before its first maxflow(), so its terms are "
                               "fixed: make the term calls before remove_nweights_warm / remove_nweights_dense_warm, or "
                               "reset() the graph and rebuild it")

    def _fold_decrements(self, native, *args):
        """A removal folds natively on solved and unsolved graphs alike: the pending build is flushed first.  Folded into
        an unsolved graph, it fixes the terms (``_terms_open``); so does a refused pair check there, which runs after the
        init that the first solve would run on an ``enable_warm()`` graph."""
        self._lattice_term()
        if self._sp is not None:
            raise _cannot_fold("without the n-link weight")
        if self._offlattice is not None:
            raise RuntimeError("edge {} does not join lattice neighbours: reset() the graph and rebuild it without the "
                               "n-link weight instead".format(self._offlattice))
        unsolved = not self._solved
        if unsolved:
            self._flush()
        self._dirty()
        try:
            getattr(self._nat(), native)(*args)
        except ValueError:
            self._folded = self._folded or unsolved
            raise
        self._folded = self._folded or unsolved

    def _stage_nweights_calls(self, i, j, cap, rev):
        """sum_edge(i[k], j[k], cap[k], rev[k]) in order, staged before the first solve: checked like the warm fold checks
        them, then added into the dense per-axis batches exactly as ``sum_edge`` adds (repeated pairs in call order)."""
        for a in (i, j):
            _warm_args.check_ids(a, self._n)          # numpy.add.at would wrap a negative id
        _warm_args.check_amounts(((cap, "cap"), (rev, "rev_cap")), _warm_args.ONLY_RAISES)
        if self._sp is not None:
            for a, b, c, r in zip(i.tolist(), j.tolist(), cap.tolist(), rev.tolist()):
                self._sp.sum_edge(a, b, c, r)
            return
        axes = _warm_args.lattice_axes(i, j, self._shape)
        if (axes < 0).any():
            k = int(numpy.flatnonzero(axes < 0)[0])
            raise ValueError("node ids ({}, {}) are not lattice neighbours".format(int(i[k]), int(j[k])))
        if self._journal is not None:
            for a, b, c, r in zip(i.tolist(), j.tolist(), cap.tolist(), rev.tolist()):
                self.sum_edge(a, b, c, r)
            return
        lo, up = numpy.minimum(i, j), i < j
        f, b = numpy.where(up, cap, rev), numpy.where(up, rev, cap)
        for axis in numpy.unique(axes).tolist():
            sel = axes == axis
            if axis not in self._st_nw:
                self._st_nw[axis] = [numpy.zeros(self._n, dtype=numpy.float64), numpy.zeros(self._n, dtype=numpy.float64)]
            fw, bw = self._st_nw[axis]
            numpy.add.at(fw, lo[sel], f[sel])        # unbuffered, in index order: a repeated pair adds in call order
            numpy.add.at(bw, lo[sel], b[sel])
        self._dirty()

    def _stage_tweights_calls(self, ids, src, snk):
        """add_tweights(ids[k], src[k], snk[k]) in order (ids None: one call per node), staged before the first solve.
        The k-th call on a node goes into dense batch k: a node's calls keep their order, and no Python loop runs per
        call."""
        _warm_args.check_finite(src, "cap_source")
        _warm_args.check_finite(snk, "cap_sink")
        if self._sp is not None:
            return self._sp.add_tweights_bulk(ids, src, snk)
        if self._journal is not None:
            self._journal.append(("T", numpy.arange(self._n) if ids is None else ids.copy(), src.copy(), snk.copy()))
        self._dirty()
        if ids is None:
            self._close_tweight_batch()          # one dense pass of its own
            self._pending.append(("tw", src.copy(), snk.copy()))
            return
        if ids.size == 0:
            return
        order = numpy.argsort(ids, kind="stable")
        sids = ids[order]
        starts = numpy.flatnonzero(numpy.r_[True, sids[1:] != sids[:-1]])
        rank = numpy.empty(ids.size, numpy.int64)
        rank[order] = numpy.arange(ids.size) - numpy.repeat(starts, numpy.diff(numpy.r_[starts, ids.size]))
        for r in range(int(rank.max()) + 1):
            sel = rank == r
            v = ids[sel]
            self._open_tweight_batch()
            if self._st_touched[v].any():
                self._close_tweight_batch()      # add_tweights is order dependent per node: start a new batch
                self._open_tweight_batch()
            self._st_src[v] = src[sel]
            self._st_snk[v] = snk[sel]
            self._st_touched[v] = True

    def get_mask(self):
        """Bulk read-out: uint8 array of the lattice shape, 0 where what_segment == SINK else 1
        (what bin/medpy_graphcut_voxel.py:177-181 builds voxel by voxel)."""
        if self._sp is not None:
            return self._sp.get_mask()
        if self._mask is None:
            self.maxflow()
            self._mask = self._nat().get_mask()
        return self._mask

    def what_segment(self, i, default_segm=None):
        """graph.h:560-571."""
        if self._sp is not None:
            return self._sp.what_segment(i)
        m = self.get_mask()
        i = int(i)
        if i < 0 or i >= self._n:
            raise ValueError("Invalid node id of {}. Valid values are 0 to {}.".format(i, self._n - 1))
        return _termtype.SOURCE if m.flat[i] else _termtype.SINK

    def reset(self):
        if self._sp is not None:
            return self._sp.reset()
        if self._journal is not None:
            self._journal = []
        self._st_src = self._st_snk = self._st_touched = None
        self._st_nw = {}
        self._mask = None
        self._offlattice = None
        self._pending = []
        self._lazy = None
        self._fresh = True
        self._solved = False
        self._folded = False
        if self._native is not None:
            self._native.reset()

    def get_edge(self, i, j):
        if self._sp is not None:
            return self._sp.get_edge(i, j)
        self._flush()
        return self._nat().get_edge(int(i), int(j))

    def get_trcap(self, i):
        if self._sp is not None:
            return self._sp.get_trcap(i)
        self._flush()
        return self._nat().get_trcap(int(i))

    def get_node_num(self):
        return self._n

    def get_arc_num(self):
        if self._sp is not None:
            return self._sp.get_arc_num()
        self._flush()
        return self._nat().get_arc_num()

    def stats(self):
        if self._sp is not None:
            return self._sp.stats()
        return self._nat().stats()


# The reference module exports three instantiations (wrapper.cpp:8-10); only GraphDouble is used by the
# Python layer (graph.py:26,305).  The other names resolve to the same lattice graph.
GraphFloat = GraphDouble
GraphInt = GraphDouble
