"""Host-side mirror of ``medpy/graphcut/wrapper.py``: ``split_marker`` (:39-69), ``graphcut_stawiaski`` (:271-329),
``graphcut_split`` (:72-225) and ``graphcut_subprocesses`` (:228-268).

The reference speeds a region cut up by cutting overlapping sub-volumes in a pool of CPU processes.  Here every cut
runs on the GPU (milliseconds each), and CUDA contexts do not survive ``fork``, so ``graphcut_subprocesses`` runs its
jobs back to back in this process; ``processes`` is validated like the reference does and otherwise ignored.  With
``batch=True`` the ``graphcut_stawiaski`` jobs of ``graphcut_subprocesses`` / ``graphcut_split`` are cut together as one
region graph (``graphcut_stawiaski_batch``), with the same results.  The splitting and re-assembly rules of
``graphcut_split`` are the reference's, so its results are too.
"""
import itertools
import logging
import math

import numpy

from ..errors import ArgumentError
from ..relabel import relabel

__all__ = ["split_marker", "graphcut_split", "graphcut_subprocesses", "graphcut_stawiaski", "graphcut_stawiaski_batch"]

_logger = logging.getLogger("medpy_b200.graphcut")


def split_marker(marker, fg_id=1, bg_id=2):
    """Marker image -> (foreground, background) boolean arrays; by default label 1 marks foreground and
    label 2 background (same contract as the reference's medpy/graphcut/wrapper.py:39-69)."""
    labels = numpy.asarray(marker)
    return numpy.equal(labels, fg_id), numpy.equal(labels, bg_id)


def graphcut_stawiaski(regions, gradient=False, foreground=False, background=False):
    """Region graph cut with the Stawiaski boundary term (wrapper.py:271-329): relabel, ``graph_from_labels``,
    ``maxflow``, map the regions' sides back onto the voxels.  Takes the four images, or one 4-tuple of them (the form
    ``graphcut_subprocesses`` passes).  Returns a boolean array, True where the voxel's region is not on the sink side."""
    from . import energy_label
    from .generate import graph_from_labels, label_cut_mask
    if gradient is False and foreground is False and background is False:
        regions, gradient, foreground, background = regions
    img_region = numpy.asarray(regions)
    img_gradient = numpy.ascontiguousarray(gradient)           # sub-volume views of graphcut_split become dense copies
    img_fg = numpy.ascontiguousarray(foreground, dtype=numpy.bool_)
    img_bg = numpy.ascontiguousarray(background, dtype=numpy.bool_)
    if not (img_region.shape == img_gradient.shape == img_fg.shape == img_bg.shape):
        raise ArgumentError("All supplied images must be of the same shape.")
    img_region = relabel(img_region)
    gcgraph = graph_from_labels(img_region, img_fg, img_bg, boundary_term=energy_label.boundary_stawiaski,
                                boundary_term_args=img_gradient)
    maxflow = gcgraph.maxflow()
    _logger.debug("Graph-cut terminated successfully with maxflow of %s.", maxflow)
    return label_cut_mask(gcgraph).astype(numpy.bool_)


def _stawiaski_job(job):
    """graphcut_stawiaski's argument checks and relabelling of one job -> (regions, gradient, fg, bg)."""
    regions, gradient, foreground, background = job
    img_region = numpy.asarray(regions)
    img_gradient = numpy.ascontiguousarray(gradient)
    img_fg = numpy.ascontiguousarray(foreground, dtype=numpy.bool_)
    img_bg = numpy.ascontiguousarray(background, dtype=numpy.bool_)
    if not (img_region.shape == img_gradient.shape == img_fg.shape == img_bg.shape):
        raise ArgumentError("All supplied images must be of the same shape.")
    return relabel(img_region), img_gradient, img_fg, img_bg


def graphcut_stawiaski_batch(jobs):
    """``[graphcut_stawiaski(j) for j in jobs]`` as one batch: every job is a 4-tuple (regions, gradient, foreground,
    background), checked and relabelled as ``graphcut_stawiaski`` does, and all jobs are cut together by
    ``graph_from_labels_batch``.  The jobs' shapes may differ (``graphcut_split``'s last sub-volumes along an axis are
    clipped)."""
    from . import energy_label
    from .labels_batch import graph_from_labels_batch
    jobs = [_stawiaski_job(j) for j in jobs]
    if not jobs:
        return []
    regions, gradients, fg, bg = (list(x) for x in zip(*jobs))
    graph = graph_from_labels_batch(regions, fg, bg, boundary_term=energy_label.boundary_stawiaski,
                                    boundary_term_args=gradients)
    _logger.debug("Batched graph-cut of %d jobs terminated successfully with maxflows of %s.", len(jobs), graph.maxflow())
    return [m.astype(numpy.bool_) for m in graph.label_cut_masks()]


def graphcut_subprocesses(graphcut_function, graphcut_arguments, processes=None, *, batch=False):
    """``[graphcut_function(a) for a in graphcut_arguments]`` (wrapper.py:228-268), one after the other on the GPU.
    ``batch=True`` cuts the jobs of ``graphcut_stawiaski`` as one batch (``graphcut_stawiaski_batch``); any other
    function raises ArgumentError then."""
    # the reference treats every falsy value as "use cpu_count" (`if not processes`, wrapper.py:252) and validates the rest
    if processes and (type(processes) is not int or processes < 0):
        raise ArgumentError("The number processes can not be zero or negative.")
    if batch:
        if graphcut_function is not graphcut_stawiaski:
            raise ArgumentError("batch=True cuts graphcut_stawiaski jobs only; run other functions with batch=False.")
        return graphcut_stawiaski_batch(list(graphcut_arguments))
    return [graphcut_function(a) for a in graphcut_arguments]


def graphcut_split(graphcut_function, regions, gradient, foreground, background, minimal_edge_length=100, overlap=10,
                   processes=None, *, batch=False):
    """Cut overlapping sub-volumes of at least ``minimal_edge_length`` voxels per edge separately and stitch the results
    (wrapper.py:72-225): inside an overlap the voxels of the earlier sub-volume are AND-ed with the later one's, the
    rest of a sub-volume is copied.  Faster on the CPU, not exact; on the GPU the whole volume is usually the better
    call.  Same argument checks (ArgumentError) as the reference.  ``batch=True`` cuts the sub-volumes as one batch
    (see ``graphcut_subprocesses``), with the same result."""
    img_region = numpy.asarray(regions)
    img_gradient = numpy.asarray(gradient)
    img_fg = numpy.asarray(foreground, dtype=numpy.bool_)
    img_bg = numpy.asarray(background, dtype=numpy.bool_)
    if not (img_region.shape == img_gradient.shape == img_fg.shape == img_bg.shape):
        raise ArgumentError("All supplied images must be of the same shape.")
    if minimal_edge_length < 10:
        raise ArgumentError("A minimal edge length smaller than 10 is not supported.")
    if overlap < 0:
        raise ArgumentError("A negative overlap is not supported.")
    if overlap >= minimal_edge_length:
        raise ArgumentError("The overlap is not allowed to exceed the minimal edge length.")
    shape = list(img_region.shape)
    steps = [max(1, extent // minimal_edge_length) for extent in shape]
    stepsizes = [math.ceil(extent / count) for extent, count in zip(shape, steps)]
    _logger.debug("minimal edge length %s -> sub-volume size %s for shape %s", minimal_edge_length, stepsizes, shape)
    starts = [range(0, int(count * size), int(size)) for count, size in zip(steps, stepsizes)]
    slicers = [tuple(slice(begin, begin + size + overlap) for begin, size in zip(corner, stepsizes))
               for corner in itertools.product(*starts)]
    jobs = [(img_region[s], img_gradient[s], img_fg[s], img_bg[s]) for s in slicers]
    parts = graphcut_subprocesses(graphcut_function, jobs, processes, batch=batch)
    result = numpy.zeros(img_region.shape, dtype=numpy.bool_)
    for slicer, part in zip(slicers, parts):
        target = result[slicer]                        # a view: writes land in `result`
        keep = [slice(None)] * result.ndim
        for dim in range(result.ndim):
            if 0 == slicer[dim].start:
                continue
            keep[dim] = slice(overlap, None)
            seam = [slice(None)] * result.ndim
            seam[dim] = slice(0, overlap)
            seam = tuple(seam)
            target[seam] = numpy.logical_and(target[seam], part[seam])
        target[tuple(keep)] = part[tuple(keep)]
    return result
