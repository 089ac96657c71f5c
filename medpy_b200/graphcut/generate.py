"""Host-side mirror of ``medpy.graphcut.generate`` (reference: medpy/graphcut/generate.py): ``graph_from_voxels``
(:33-174) and ``graph_from_labels`` (:177-338).

Same signature, same validation and the same order of operations -- regional term, boundary term, foreground
markers, background markers (generate.py:159-172) -- but no edge list is built: the GCGraph handed to the
term functions is a dense lattice in device memory and each term is one CUDA kernel launch.
"""
import inspect
import logging

import numpy

from .graph import GCGraph

_logger = logging.getLogger("medpy_b200.graphcut")


def voxel_edge_count(shape):
    """Number of edges of the 2*ndim-connected lattice, size-1 axes dropped
    (what the reference's ``__voxel_4conectedness`` computes, generate.py:363-383)."""
    dims = [int(s) for s in shape if int(s) != 1]
    total = 1
    for s in dims:
        total *= s
    return sum((total // s) * (s - 1) for s in dims)


def _noop_term(graph, term_args):
    """Default for a missing term: same 2-parameter signature the reference's dummies have (generate.py:341-355)."""
    return {}


def _takes_two_parameters(fn):
    return hasattr(fn, "__call__") and 2 == len(inspect.getfullargspec(fn)[0])


def graph_from_voxels(fg_markers, bg_markers, regional_term=False, boundary_term=False,
                      regional_term_args=False, boundary_term_args=False):
    """Create a graph-cut ready graph from a voxel image.

    Parameters and behaviour follow the reference (generate.py:33-110): ``fg_markers`` / ``bg_markers`` are
    array-likes of one shape (converted to bool); ``regional_term`` / ``boundary_term`` are callables taking
    exactly two positional parameters ``(graph, term_args)`` (``AttributeError`` otherwise); they receive a
    ``GCGraph`` whose node ids are the C-order flat voxel indices.  Returns the solver-side graph object
    (``graph.get_graph()``) offering ``maxflow()``, ``what_segment(i)`` and ``termtype``.

    A voxel marked as both foreground and background receives both hard links, which cancel
    (SURVEY.md App. A.5), exactly as in the reference.
    """
    fg_in = numpy.asarray(fg_markers)
    _logger.debug("Assuming %d nodes and %d edges for image of shape %s", fg_in.size, voxel_edge_count(fg_in.shape), fg_in.shape)
    graph = GCGraph(fg_in.size, voxel_edge_count(fg_in.shape), shape=fg_in.shape)
    # the markers follow the boundary term immediately: a non-positive-weight ValueError may be delivered by that next
    # call (still inside this function) so that the marker upload overlaps the stencil kernel
    graph.get_graph().defer_weight_check(True)

    fg = numpy.asarray(fg_markers, dtype=numpy.bool_)
    bg = numpy.asarray(bg_markers, dtype=numpy.bool_)

    if not regional_term:
        regional_term = _noop_term
    if not boundary_term:
        boundary_term = _noop_term

    if not _takes_two_parameters(regional_term):
        raise AttributeError("regional_term has to be a callable object which takes two parameter.")
    if not _takes_two_parameters(boundary_term):
        raise AttributeError("boundary_term has to be a callable object which takes two parameters.")

    _logger.info("Computing and adding terminal edge weights...")
    regional_term(graph, regional_term_args)

    _logger.info("Computing and adding inter-node edge weights...")
    boundary_term(graph, boundary_term_args)

    _logger.info("Setting terminal weights for the markers...")
    if bg.shape != fg.shape:
        raise ValueError("fg_markers and bg_markers must have the same shape")
    # set_source_nodes(fg ids) THEN set_sink_nodes(bg ids) (generate.py:169-172) as one fused device pass.  The
    # reference skips an empty marker set; an all-False array does the same thing here, so no host-side scan.
    graph._add_markers(fg, bg)
    gc_graph = graph.get_graph()
    gc_graph.check_deferred()
    gc_graph.defer_weight_check(False)
    return gc_graph


def _noop_label_term(graph, label_image, term_args):
    """Default for a missing term of graph_from_labels (generate.py:346-360)."""
    return {}


def _takes_three_parameters(fn):
    return hasattr(fn, "__call__") and 3 == len(inspect.getfullargspec(fn)[0])


def graph_from_labels(label_image, fg_markers, bg_markers, regional_term=False, boundary_term=False,
                      regional_term_args=False, boundary_term_args=False, *, warm=False):
    """Create a graph-cut ready graph from a label (region) image -- generate.py:177-338.

    Every region of ``label_image`` (ids exactly 1..K, ``AttributeError`` otherwise) is a node (id = label - 1);
    ``regional_term`` / ``boundary_term`` are callables ``(graph, label_image, term_args)`` (see ``energy_label``;
    ``AttributeError`` for any other arity) that add t- and n-weights; regions touched by a foreground / background
    marker are then tied to the source / sink with ``GCGraph.MAX`` (set_source_nodes before set_sink_nodes,
    generate.py:334-337).  Returns the solver-side graph object offering ``maxflow()``, ``what_segment(i)``,
    ``get_mask()`` and ``termtype``.

    The label image is staged on the device once and shared by the terms and the marker step; the resulting region
    graph is solved by the sparse push-relabel (csrc/gc_sparse.cuh).  (The reference itself cannot run this function on
    Python >= 3.11: it calls ``inspect.getargspec``, generate.py:280.)

    ``warm=True`` (an addition to the reference's parameters) keeps the solved state: seeds added or erased on regions
    (``add_seeds`` / ``remove_seeds`` with region ids or a boolean mask over the regions), t-link and edge calls made
    after ``maxflow()`` fold into it, and the next ``maxflow()`` continues from the flow already routed.
    """
    from .energy_label import LabelContext
    label_image = numpy.asarray(label_image)
    fg = numpy.asarray(fg_markers, dtype=numpy.bool_)
    bg = numpy.asarray(bg_markers, dtype=numpy.bool_)
    if not regional_term:
        regional_term = _noop_label_term
    if not boundary_term:
        boundary_term = _noop_label_term
    # (both this and a malformed label image are AttributeErrors in the reference, generate.py:272-289)
    if not _takes_three_parameters(regional_term):
        raise AttributeError("regional_term has to be a callable object which takes three parameters.")
    if not _takes_three_parameters(boundary_term):
        raise AttributeError("boundary_term has to be a callable object which takes three parameters.")
    context = LabelContext(label_image)                      # stages the image; __check_label_image (generate.py:272)

    nodes = context.regions
    edges = 10 * nodes                                       # the reference's guess (generate.py:296)
    _logger.debug("guessed: #nodes=%d nodes / #edges=%d", nodes, edges)
    graph = GCGraph(nodes, edges, sparse=True, warm=warm)
    graph._label_context = context

    _logger.info("Computing and adding terminal edge weights...")
    regional_term(graph, label_image, regional_term_args)
    _logger.info("Computing and adding inter-node edge weights...")
    boundary_term(graph, label_image, boundary_term_args)

    _logger.info("Setting terminal weights for the markers...")
    # numpy.unique(label_image[markers] - 1) (generate.py:334-337): one flag per region, set on the device
    graph.set_source_nodes(numpy.nonzero(context.region_flags(fg))[0])
    graph.set_sink_nodes(numpy.nonzero(context.region_flags(bg))[0])
    gc_graph = graph.get_graph()
    gc_graph.label_context = context                         # lets callers map the cut back: see label_cut_mask
    return gc_graph


def label_cut_mask(gc_graph, label_image=None):
    """Voxel mask of a region cut: 1 where the voxel's region is not in the SINK set -- the mapping + relabel_map step
    of bin/medpy_graphcut_label.py:139-148 as one device gather.  ``gc_graph`` is what ``graph_from_labels`` returned."""
    from .energy_label import LabelContext
    context = getattr(gc_graph, "label_context", None)
    if label_image is not None and (context is None or context.source is not label_image):
        context = LabelContext(label_image)
    if context is None:
        raise ValueError("pass the label image the graph was built from")
    return context.apply(gc_graph.get_mask())
