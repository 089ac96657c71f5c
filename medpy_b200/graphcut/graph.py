"""Host-side mirror of ``medpy.graphcut.graph.GCGraph`` (reference: medpy/graphcut/graph.py:267-596).

Same method names, argument meaning and error behaviour (``ValueError`` for bad node ids, self loops and
n-weights <= 0; t-weights may be <= 0); the storage underneath is the dense device lattice of
``medpy_b200.graphcut.maxflow.GraphDouble`` instead of BK's node/arc lists.  Extra, optional entry points
(``set_nweights_dense``, ``set_tweights_dense``) let user-written 2-argument energy terms hand whole arrays
over instead of looping per edge.
"""
import numpy

from .maxflow import GraphDouble


class Graph(object):
    """The reference's plain-Python graph description (medpy/graphcut/graph.py:29-265): a record of node count,
    source / sink node lists and weight dictionaries with node ids starting at 1, consumed by ``graph_to_dimacs``.
    It holds no solver; use ``GCGraph`` to cut a graph."""

    MAX = 65535
    """The maximum value a weight can take (graph.py:45-50)."""

    def __init__(self):
        self._node_count = 0
        self._source_nodes = []
        self._sink_nodes = []
        self._nweights = {}
        self._tweights = {}

    def set_nodes(self, nodes):
        """Number of nodes, terminals excluded (graph.py:58-66)."""
        self._node_count = int(nodes)

    def set_source_nodes(self, source_nodes):
        """Tie nodes to the source: t-weight (MAX, 0) each (graph.py:68-85)."""
        self._source_nodes = list(source_nodes)
        self._tweights.update((v, (self.MAX, 0)) for v in self._source_nodes)

    def set_sink_nodes(self, sink_nodes):
        """Tie nodes to the sink: t-weight (0, MAX) each (graph.py:87-104)."""
        self._sink_nodes = list(sink_nodes)
        self._tweights.update((v, (0, self.MAX)) for v in self._sink_nodes)

    def set_nweights(self, nweights):
        """{(node, node): (weight, reverse weight)}; replaces what was set before (graph.py:106-113)."""
        self._nweights = nweights

    def add_tweights(self, tweights):
        """{node: (weight to source, weight to sink)}; overrides entries set before, markers included (graph.py:115-128)."""
        self._tweights.update(tweights)

    def get_node_count(self):
        return self._node_count

    def get_nodes(self):
        return list(range(1, self._node_count + 1))

    def get_source_nodes(self):
        return self._source_nodes

    def get_sink_nodes(self):
        return self._sink_nodes

    def get_edges(self):
        return list(self._nweights.keys())

    def get_nweights(self):
        return self._nweights

    def get_tweights(self):
        """Only the t-weights set so far (graph.py:210-222)."""
        return self._tweights

    def inconsistent(self):
        """False, or the list of problems: ids above the node count, edges stored in both directions (graph.py:224-265)."""
        found = []
        found += ["Node {} in t-weights but not in nodes.".format(v) for v in self._tweights if not v <= self._node_count]
        found += ["Node {} in s-nodes but not in nodes.".format(v) for v in self._source_nodes if not v <= self._node_count]
        found += ["Node {} in t-nodes but not in nodes.".format(v) for v in self._sink_nodes if not v <= self._node_count]
        for e in self._nweights:
            found += ["Node {} in edge {} but not in nodes.".format(v, e) for v in e[:2] if not v <= self._node_count]
            if (e[1], e[0]) in self._nweights:
                found.append("The reversed edges of {} is also in the n-weights.".format(e))
        return found if found else False


class GCGraph:
    """Validated wrapper over the lattice graph, API-compatible with the reference's GCGraph."""

    # graph.py:286-291
    __INT_16_BIT = 32767
    __UINT_16_BIT = 65535
    MAX = __UINT_16_BIT
    """The maximum value a terminal weight can take."""

    def __init__(self, nodes, edges, shape=None, device=-1, sparse=None, warm=False):
        """``GCGraph(nodes, edges)`` as in the reference (graph.py:294-308); ``shape`` (given by
        ``graph_from_voxels``) is the logical lattice shape whose C-order flat index is the node id.  Without a shape
        the graph is general: it moves to the sparse backend with the first edge between arbitrary nodes, or at once
        with ``sparse=True`` (``graph_from_labels``).  ``warm=True`` (with ``sparse=True``): calls made after a solve
        fold into its residual state and the next solve continues from there."""
        self.__graph = GraphDouble(int(nodes), int(edges), shape=shape, device=device, sparse=sparse, warm=warm)
        self.__graph.add_node(int(nodes))
        self.__nodes = int(nodes)
        self.__edges = int(edges)

    # ------------------------------------------------------------------ t-links
    def __check_nodes(self, ids):
        ids = numpy.asarray(list(ids) if not isinstance(ids, numpy.ndarray) else ids)
        if ids.size == 0:
            raise ValueError("max() arg is an empty sequence")  # what the reference's max([]) raises
        hi, lo = ids.max(), ids.min()
        if hi >= self.__nodes or lo < 0:
            raise ValueError("Invalid node id of {} or {}. Valid values are 0 to {}.".format(hi, lo, self.__nodes - 1))
        return ids.astype(numpy.int64)

    def __set_terminal_nodes(self, ids, as_source):
        ids = self.__check_nodes(ids)
        # add_tweights(v, MAX, 0) resp. (v, 0, MAX) per node, in order (graph.py:341-344, 377-380)
        self.__graph.stage_tweights_many(ids, self.MAX if as_source else 0, 0 if as_source else self.MAX)

    def set_source_nodes(self, source_nodes):
        """graph.py:310-344: hard-wire nodes to the source (foreground) with weight MAX = 65535."""
        self.__set_terminal_nodes(source_nodes, True)

    def set_sink_nodes(self, sink_nodes):
        """graph.py:346-380: hard-wire nodes to the sink (background) with weight MAX = 65535."""
        self.__set_terminal_nodes(sink_nodes, False)

    def set_tweight(self, node, weight_source, weight_sink):
        """graph.py:462-498: add_tweights(node, weight_source, weight_sink); weights may be <= 0.  On a solved graph use
        ``get_graph().add_tweights_warm``, the warm form of the same calls."""
        if node >= self.__nodes or node < 0:
            raise ValueError("Invalid node id of {}. Valid values are 0 to {}.".format(node, self.__nodes - 1))
        self.__graph.add_tweights(int(node), float(weight_source), float(weight_sink))

    def set_tweights(self, tweights):
        """graph.py:500-530."""
        for node, weight in list(tweights.items()):
            self.set_tweight(node, weight[0], weight[1])

    def set_tweights_all(self, tweights):
        """graph.py:532-552: one (source, sink) pair per node, in node order -- done as ONE dense device pass.  On a
        solved graph use ``get_graph().add_tweights_warm(None, source, sink)``, the warm form of the same calls."""
        tw = numpy.asarray(tweights if isinstance(tweights, numpy.ndarray) else list(tweights), dtype=numpy.float64)
        if tw.ndim != 2 or tw.shape[1] != 2:
            raise ValueError("tweights must hold one (source, sink) pair per node")
        if tw.shape[0] > self.__nodes:
            raise ValueError("Invalid node id of {}. Valid values are 0 to {}.".format(tw.shape[0] - 1, self.__nodes - 1))
        if tw.shape[0] < self.__nodes:  # the reference's loop simply stops early
            pad = numpy.zeros((self.__nodes - tw.shape[0], 2))
            tw = numpy.vstack([tw, pad])
        self.set_tweights_dense(tw[:, 0], tw[:, 1])

    def set_tweights_dense(self, weight_source, weight_sink):
        """Array form of ``set_tweights_all``: add_tweights(v, weight_source[v], weight_sink[v]) for all v."""
        self.__graph.add_tweights_dense(numpy.asarray(weight_source, dtype=numpy.float64),
                                        numpy.asarray(weight_sink, dtype=numpy.float64))

    # ------------------------------------------------------------------ n-links
    def set_nweight(self, node_from, node_to, weight_there, weight_back):
        """graph.py:382-440 (validation order preserved) -> sum_edge."""
        if node_from >= self.__nodes or node_from < 0:
            raise ValueError("Invalid node id (node_from) of {}. Valid values are 0 to {}.".format(node_from, self.__nodes - 1))
        elif node_to >= self.__nodes or node_to < 0:
            raise ValueError("Invalid node id (node_to) of {}. Valid values are 0 to {}.".format(node_to, self.__nodes - 1))
        elif node_from == node_to:
            raise ValueError("The node_from ({}) can not be equal to the node_to ({}) (self-connections are forbidden in graph cuts).".format(node_from, node_to))
        elif weight_there <= 0 or weight_back <= 0:
            raise ValueError("Negative or zero weights are not allowed.")
        self.__graph.sum_edge(int(node_from), int(node_to), float(weight_there), float(weight_back))

    def set_nweights_bulk(self, nodes_from, nodes_to, weights_there, weights_back):
        """Array form of ``set_nweight``: one call per entry, in order, with the same checks (graph.py:418-437)."""
        i = numpy.asarray(nodes_from).ravel()
        j = numpy.asarray(nodes_to).ravel()
        wt = numpy.asarray(weights_there, dtype=numpy.float64).ravel()
        wb = numpy.asarray(weights_back, dtype=numpy.float64).ravel()
        if not (i.size == j.size == wt.size == wb.size):
            raise ValueError("edge arrays differ in length")
        if i.size == 0:
            return
        if i.max() >= self.__nodes or i.min() < 0:
            raise ValueError("Invalid node id (node_from) of {} or {}. Valid values are 0 to {}.".format(i.max(), i.min(), self.__nodes - 1))
        if j.max() >= self.__nodes or j.min() < 0:
            raise ValueError("Invalid node id (node_to) of {} or {}. Valid values are 0 to {}.".format(j.max(), j.min(), self.__nodes - 1))
        if (i == j).any():
            raise ValueError("The node_from can not be equal to the node_to (self-connections are forbidden in graph cuts).")
        if (wt <= 0).any() or (wb <= 0).any():
            raise ValueError("Negative or zero weights are not allowed.")
        self.__graph.sum_edges_bulk(i, j, wt, wb)

    def set_tweights_bulk(self, nodes, weights_source, weights_sink):
        """Array form of ``set_tweight`` (graph.py:462-498): one add_tweights call per entry, in order."""
        nodes = numpy.asarray(nodes).ravel()
        if nodes.size and (nodes.max() >= self.__nodes or nodes.min() < 0):
            raise ValueError("Invalid node id of {} or {}. Valid values are 0 to {}.".format(nodes.max(), nodes.min(), self.__nodes - 1))
        self.__graph.add_tweights_bulk(nodes, numpy.asarray(weights_source, dtype=numpy.float64),
                                       numpy.asarray(weights_sink, dtype=numpy.float64))

    def set_nweights(self, nweights):
        """graph.py:442-460."""
        for edge, weight in list(nweights.items()):
            self.set_nweight(edge[0], edge[1], weight[0], weight[1])

    def set_nweights_dense(self, axis, weight_there, weight_back):
        """Array form of the per-edge loop energy_voxel.py:660-664 for one lattice axis: arrays of the lattice
        shape with extent D_axis-1 (or D_axis, last plane ignored) along ``axis``; entry p is the weight of
        p -> p+e_axis (there) and p+e_axis -> p (back).  Raises ValueError on weights <= 0 like set_nweight."""
        shape = self.__graph.shape
        there = numpy.asarray(weight_there, dtype=numpy.float64)
        back = numpy.asarray(weight_back, dtype=numpy.float64)
        short = list(shape)
        short[axis] -= 1
        if there.shape == tuple(short):
            if (there <= 0).any() or (back <= 0).any():
                raise ValueError("Negative or zero weights are not allowed.")
            pad = [(0, 0)] * len(shape)
            pad[axis] = (0, 1)
            there = numpy.pad(there, pad)
            back = numpy.pad(back, pad)
        elif there.shape == tuple(shape):
            sl = [slice(None)] * len(shape)
            sl[axis] = slice(0, shape[axis] - 1)
            if (there[tuple(sl)] <= 0).any() or (back[tuple(sl)] <= 0).any():
                raise ValueError("Negative or zero weights are not allowed.")
        else:
            raise ValueError("weights must have the lattice shape (optionally one shorter along the axis)")
        self.__graph.add_nweights_dense(axis, numpy.ascontiguousarray(there), numpy.ascontiguousarray(back))

    # ------------------------------------------------------------------ bulk energy terms (used by energy_voxel)
    def _add_boundary(self, kind, image, sigma, spacing, norm):
        self.__graph.add_boundary(kind, image, sigma, spacing, norm)

    def _add_regional_probability(self, prob, alpha, compute_f32):
        self.__graph.add_regional_probability(prob, alpha, compute_f32)

    def _add_markers(self, fg, bg):
        self.__graph.add_markers(fg, bg)

    # ------------------------------------------------------------------ getters (graph.py:554-596)
    def get_graph(self):
        """The underlying lattice graph (the reference returns its maxflow.GraphDouble, graph.py:554-563)."""
        return self.__graph

    def get_node_count(self):
        return self.__nodes

    def get_nodes(self):
        return list(range(0, self.__nodes))

    def get_edge_count(self):
        return self.__edges
