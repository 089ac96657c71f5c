"""General sparse graphs behind the ``GraphDouble`` API (SURVEY.md §8 rows f3/f4).

The reference's ``GraphDouble`` (lib/maxflow/src/wrapper.cpp:63-83) is a general graph; the voxel path only ever fills it
with lattice edges, which is why ``medpy_b200.graphcut.maxflow.GraphDouble`` stores a dense lattice.  Graphs that are
not lattices -- the region adjacency graph of ``graph_from_labels`` (generate.py:177-338) and graphs users assemble
edge by edge (tests/graphcut_/graph.py:47) -- are held by ``SparseGraphDouble``: calls are staged in host lists and
cross the C ABI in bulk (``mgc_sparse_sum_edges`` / ``mgc_sparse_add_tweights``, which apply them in order with the
reference's accumulation semantics); ``maxflow()`` runs a CSR push-relabel on the device (csrc/gc_sparse.cuh).

A graph created with ``warm=True`` keeps the device state of its first solve.  Calls made after a solve are staged the
same way and fold into that residual state at the next ``maxflow()`` (or getter), as the reference's ``add_tweights`` /
``sum_edge`` act on its residual graph (graph.h:415-480); ``remove_nweights_warm`` lowers capacities
(csrc/gc_sparse_warm.cuh).

No CPU solver: the first call that needs a result creates the native graph and raises ``RuntimeError`` without a CUDA
device or built extension.
"""
import numpy

from . import _warm_args
from .maxflow import _termtype

__all__ = ["SparseGraphDouble"]


def _host(x):
    """Sparse handles take host arrays: a tensor argument (CUDA or CPU) is copied to numpy before it is parsed."""
    if hasattr(x, "__cuda_array_interface__") or type(x).__module__.startswith("torch"):
        return x.detach().cpu().numpy()
    return x


# why a sum_edge call on a solved warm graph may not be negative
_LOWER = "a solved graph lowers capacities only through remove_nweights_warm"


def warm_ids(x, n, what):
    """Node ids of one warm-call argument on a graph of n nodes, as host int32: a boolean mask of shape (n,), a 1-D
    integer id array or a single id."""
    a = numpy.asarray(_host(x))
    if a.ndim == 0 and a.dtype != numpy.bool_:
        a = a.reshape(1)
    return _warm_args.node_ids(a, (n,), n, what).astype(numpy.int32)


def warm_weights(w, m, what):
    """One weight argument of a warm call as m finite host float64 values."""
    w = _warm_args.weights(_host(w), m, what)
    _warm_args.check_finite(w, what)
    return w


def warm_pairs(i, j, cap, rev_cap, n, why):
    """The sum_edge calls of an n-link edit on a graph of n nodes as host arrays.  Unlike on the lattice, a one-element
    id array broadcasts to the length of the longest argument."""
    ii, jj = warm_ids(i, n, "i"), warm_ids(j, n, "j")
    cap, rev_cap = _host(cap), _host(rev_cap)
    m = max(ii.size, jj.size, *(numpy.size(w) for w in (cap, rev_cap) if numpy.ndim(w)))
    ii, jj = (numpy.repeat(x, m) if x.size == 1 else x for x in (ii, jj))
    ii, jj, c, r = _warm_args.nlink_calls(ii, jj, cap, rev_cap)
    _warm_args.check_amounts(((c, "cap"), (r, "rev_cap")), why)
    if (ii == jj).any():
        raise ValueError("invalid node ids in the edge arrays")
    return ii, jj, c, r


def warm_seeds(fg, bg, cap, n):
    """The add_tweights calls of add_seeds (``cap`` 65535) or remove_seeds (-65535) on a graph of n nodes, as
    ``[(ids, src, snk), ...]`` host arrays: the foreground call, then the background call, each only where it has ids."""
    ids = [None if x is None else warm_ids(x, n, what) for x, what in ((fg, "fg"), (bg, "bg"))]
    return [(v, numpy.full(v.size, src), numpy.full(v.size, snk))
            for v, src, snk in ((ids[0], cap, 0.0), (ids[1], 0.0, cap)) if v is not None and v.size]


def warm_tweights(nodes, cap_source, cap_sink, n):
    """The add_tweights calls of add_tweights_warm on a graph of n nodes as host arrays: node ids (None: one call per
    node) and finite weights of one entry per call."""
    ids = None if nodes is None else warm_ids(nodes, n, "nodes")
    m = n if ids is None else ids.size
    return ids, warm_weights(cap_source, m, "cap_source"), warm_weights(cap_sink, m, "cap_sink")


class SparseGraphDouble:
    """``GraphDouble(node_num_max, edge_num_max)`` for arbitrary node pairs."""

    termtype = _termtype

    def __init__(self, node_num_max, edge_num_max=0, device=-1, warm=False):
        self._n = int(node_num_max)
        if self._n < 1:
            raise ValueError("a graph needs at least one node")
        self._edges = int(edge_num_max)
        self._device = device
        self._native = None
        self._ops = []            # staged calls in order: ("e", i, j, cap, rev) / ("t", nodes|None, src, snk) arrays
        self._e = ([], [], [], [])
        self._t = ([], [], [])
        self._mask = None
        self._warm = bool(warm)   # MGC_OPT_WARM on the handle: calls after a solve fold into its residual state
        self._solved = False      # a warm graph was solved since the last reset

    @property
    def warm(self):
        return self._warm

    # ------------------------------------------------------------------ staging
    def _nat(self):
        if self._native is None:
            from .. import _lib  # raises ImportError loudly when the extension is not built
            self._native = _lib._mgc.SparseGraph(self._n, self._device)
            if self._warm:
                self._native.set_option(_lib._mgc.OPT_WARM, 1)
        return self._native

    def _close_edges(self):
        if self._e[0]:
            self._ops.append(("e", numpy.asarray(self._e[0], dtype=numpy.int32), numpy.asarray(self._e[1], dtype=numpy.int32),
                              numpy.asarray(self._e[2], dtype=numpy.float64), numpy.asarray(self._e[3], dtype=numpy.float64)))
            self._e = ([], [], [], [])

    def _close_tweights(self):
        if self._t[0]:
            self._ops.append(("t", numpy.asarray(self._t[0], dtype=numpy.int32), numpy.asarray(self._t[1], dtype=numpy.float64),
                              numpy.asarray(self._t[2], dtype=numpy.float64)))
            self._t = ([], [], [])

    def _flush(self):
        # edges and t-links are independent state in the reference (graph.h:415-480), so the two staged groups may be
        # applied one after the other; inside a group the call order is kept
        self._close_edges()
        self._close_tweights()
        ops, self._ops = self._ops, []
        for op in ops:
            if op[0] == "e":
                self._nat().sum_edges(op[1], op[2], op[3], op[4])
            else:
                self._nat().add_tweights(op[1], op[2], op[3])

    def _check_node(self, i):
        if i < 0 or i >= self._n:
            raise ValueError("Invalid node id of {}. Valid values are 0 to {}.".format(i, self._n - 1))

    # ------------------------------------------------------------------ reference GraphDouble API
    def add_node(self, num=1):
        """graph.h:388-413: nodes exist from construction; returns the id of the first one."""
        return 0

    def add_tweights(self, i, cap_source, cap_sink):
        """graph.h:415-425."""
        i = int(i)
        self._check_node(i)
        if self._solved:                    # the call folds into the residual state: finite weights only
            _warm_args.check_finite(cap_source, "cap_source")
            _warm_args.check_finite(cap_sink, "cap_sink")
        self._t[0].append(i)
        self._t[1].append(float(cap_source))
        self._t[2].append(float(cap_sink))
        self._mask = None

    def stage_tweights_many(self, ids, cap_source, cap_sink):
        """add_tweights(v, cap_source, cap_sink) for every v in ids, in order (ids already range-checked)."""
        ids = numpy.asarray(ids, dtype=numpy.int32).ravel()
        self.add_tweights_bulk(ids, numpy.full(ids.size, float(cap_source)), numpy.full(ids.size, float(cap_sink)))

    def add_tweights_bulk(self, nodes, src, snk):
        """One add_tweights call per entry, in array order; ``nodes`` None means 0..len-1."""
        src = numpy.ascontiguousarray(src, dtype=numpy.float64).ravel()
        snk = numpy.ascontiguousarray(snk, dtype=numpy.float64).ravel()
        if nodes is not None:
            nodes = _warm_args.check_ids(numpy.ascontiguousarray(nodes, dtype=numpy.int32).ravel(), self._n)
        elif src.size > self._n:
            raise ValueError("Invalid node id of {}. Valid values are 0 to {}.".format(src.size - 1, self._n - 1))
        if self._solved:
            _warm_args.check_finite(src, "cap_source")
            _warm_args.check_finite(snk, "cap_sink")
        self._close_tweights()
        self._ops.append(("t", nodes, src, snk))
        self._mask = None

    def sum_edge(self, i, j, cap, rev_cap):
        """graph.h:456-480: creates the arc pair on the first call for (i, j), accumulates afterwards."""
        i, j = int(i), int(j)
        if i < 0 or j < 0 or i >= self._n or j >= self._n or i == j:
            raise ValueError("invalid node ids ({}, {})".format(i, j))
        if self._solved:                    # the call folds as an increment
            _warm_args.check_amounts(((cap, "cap"), (rev_cap, "rev_cap")), _LOWER)
        self._e[0].append(i)
        self._e[1].append(j)
        self._e[2].append(float(cap))
        self._e[3].append(float(rev_cap))
        self._mask = None

    add_edge = sum_edge  # graph.h:427-454: parallel arcs carry the summed capacity

    def sum_edges_bulk(self, i, j, cap, rev_cap):
        """One sum_edge call per entry, in array order."""
        i = numpy.ascontiguousarray(i, dtype=numpy.int32).ravel()
        j = numpy.ascontiguousarray(j, dtype=numpy.int32).ravel()
        cap = numpy.ascontiguousarray(cap, dtype=numpy.float64).ravel()
        rev_cap = numpy.ascontiguousarray(rev_cap, dtype=numpy.float64).ravel()
        if not (i.size == j.size == cap.size == rev_cap.size):
            raise ValueError("edge arrays differ in length")
        if i.size and (min(i.min(), j.min()) < 0 or max(i.max(), j.max()) >= self._n or (i == j).any()):
            raise ValueError("invalid node ids in the edge arrays")
        if self._solved:
            _warm_args.check_amounts(((cap, "cap"), (rev_cap, "rev_cap")), _LOWER)
        self._close_edges()
        self._ops.append(("e", i, j, cap, rev_cap))
        self._mask = None

    def maxflow(self):
        """Graph::maxflow (maxflow.cpp:471-604): min-cut energy including the add_tweights constants."""
        self._flush()
        flow = self._nat().maxflow()
        self._solved = self._warm
        return flow

    def get_mask(self):
        """uint8[n]: 0 where what_segment == SINK else 1 (the loop of bin/medpy_graphcut_label.py:139-145 in bulk)."""
        if self._mask is None:
            self.maxflow()
            self._mask = self._nat().get_mask()
        return self._mask

    def what_segment(self, i, default_segm=None):
        """graph.h:560-571."""
        i = int(i)
        self._check_node(i)
        return _termtype.SOURCE if self.get_mask()[i] else _termtype.SINK

    def reset(self):
        self._ops = []
        self._e = ([], [], [], [])
        self._t = ([], [], [])
        self._mask = None
        self._solved = False
        if self._native is not None:
            self._native.reset()            # the warm option stays set on the handle

    def get_edge(self, i, j):
        self._flush()
        return self._nat().get_edge(int(i), int(j))

    def get_trcap(self, i):
        self._flush()
        return self._nat().get_trcap(int(i))

    def get_node_num(self):
        return self._n

    def get_arc_num(self):
        self._flush()
        return self._nat().get_arc_num()

    def stats(self):
        return self._nat().stats()

    # ------------------------------------------------------------------ warm calls (graphs created with warm=True)
    def _require_warm(self, what):
        if not self._warm:
            raise RuntimeError("{} needs a sparse graph created with warm=True; reset() the graph and rebuild it "
                               "instead".format(what))

    def add_seeds(self, fg=None, bg=None):
        """add_tweights(v, 65535, 0) per foreground id in order, then add_tweights(v, 0, 65535) per background id."""
        self._require_warm("add_seeds")
        for call in warm_seeds(fg, bg, 65535.0, self._n):
            self.add_tweights_bulk(*call)

    def remove_seeds(self, fg=None, bg=None):
        """The inverse of add_seeds: add_tweights(v, -65535, 0) / add_tweights(v, 0, -65535)."""
        self._require_warm("remove_seeds")
        for call in warm_seeds(fg, bg, -65535.0, self._n):
            self.add_tweights_bulk(*call)

    def add_tweights_warm(self, nodes, cap_source, cap_sink):
        """add_tweights(nodes[k], cap_source[k], cap_sink[k]) per entry in order; nodes None: one call per node."""
        self._require_warm("add_tweights_warm")
        self.add_tweights_bulk(*warm_tweights(nodes, cap_source, cap_sink, self._n))

    def add_nweights_warm(self, i, j, cap, rev_cap):
        """sum_edge(i[k], j[k], cap[k], rev_cap[k]) per entry in order, on any node pairs (new ones included)."""
        self._require_warm("add_nweights_warm")
        ii, jj, c, r = warm_pairs(i, j, cap, rev_cap, self._n, _warm_args.ONLY_RAISES)
        if ii.size:
            self.sum_edges_bulk(ii, jj, c, r)

    def remove_nweights_warm(self, i, j, cap, rev_cap):
        """sum_edge(i[k], j[k], -cap[k], -rev_cap[k]) per entry in order on existing pairs: the only way to lower a
        capacity.  What is staged is folded first, so the call order is kept.  A pair whose decrements exceed what it
        holds (beyond a few hundred roundings) raises ValueError with the graph unchanged."""
        self._require_warm("remove_nweights_warm")
        ii, jj, c, r = warm_pairs(i, j, cap, rev_cap, self._n, _warm_args.DECREMENTS)
        self._flush()
        self._mask = None
        if ii.size:
            self._nat().remove_edges_warm(ii, jj, c, r)

    def add_nweights_dense_warm(self, *args, **kwargs):
        raise ValueError("a general sparse graph has no lattice axes: use add_nweights_warm")

    def remove_nweights_dense_warm(self, *args, **kwargs):
        raise ValueError("a general sparse graph has no lattice axes: use remove_nweights_warm")
