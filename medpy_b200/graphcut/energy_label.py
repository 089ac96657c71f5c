"""Host-side mirror of ``medpy.graphcut.energy_label`` (reference: medpy/graphcut/energy_label.py).

The four energy terms for region (label) graphs keep the reference's names and their three-parameter signature
``(graph, label_image, term_args)`` (``graph_from_labels`` checks the arity, generate.py:278-289).  Where the
reference walks every border voxel pair in Python and calls ``graph.set_nweight`` once per pair
(energy_label.py:203-214, 325-342), the label image is staged once in device memory and the region adjacency graph is
reduced there (csrc/gc_labels.cuh): border pairs are written in the reference's accumulation order, stably sorted by
region pair and summed front to back, so every edge weight equals what the reference's chain of ``+=`` leaves behind.
Only the per-region-pair results come back; they enter the graph through one bulk call (or, for a user-supplied graph
object that is not ours, one ``set_nweight`` per region pair).

    boundary_stawiaski            w_ij = sum over border pairs of (1 / (1 + max(|g_p|, |g_q|)))^2       (:123-214)
    boundary_stawiaski_directed   same, +beta on one direction depending on the gradient's sign of change (:217-342)
    boundary_difference_of_means  w_ij = max(1 - |mean_i - mean_j| / max difference of means, DBL_MIN)    (:33-120)
    regional_atlas                t-links (alpha * sum of the atlas under the region, -alpha * sum)       (:345-396)

Reference behaviour that is kept on purpose (pinned by tests/golden/golden_labels_v1.npz): float32 gradients are
evaluated in float32 by ``boundary_stawiaski`` (numpy-2 scalar promotion) but in float64 by the directed variant
(numpy.vectorize hands Python floats to its function), which also counts the first voxel pair of every axis twice
(the probing call numpy.vectorize makes); ``regional_atlas`` sums with numpy's pairwise summation in the atlas' own
dtype.  One deliberate difference: for ``directedness >= 0`` the reference raises TypeError (its light-to-dark closure
takes a parameter nobody passes, energy_label.py:281); here that case works as its docstring describes.
"""
import sys

import numpy

__all__ = ["boundary_difference_of_means", "boundary_stawiaski", "boundary_stawiaski_directed", "regional_atlas"]

_DEVICE_DTYPES = (numpy.float32, numpy.float64, numpy.uint8, numpy.int16, numpy.int32)
_DBL_MIN = sys.float_info.min


def device_labels(label_image):
    """The host-side checks of a label image and its int32 form the kernels read (the ids' consecutiveness is checked
    on the device)."""
    if label_image.ndim < 1 or label_image.ndim > 4:
        raise ValueError("label images with 1 to 4 dimensions are supported, got {}".format(label_image.ndim))
    if label_image.size == 0:
        raise AttributeError("The supplied label image does either not contain any regions or they are not labeled "
                             "consecutively starting from 1.")
    dev = label_image
    if dev.dtype != numpy.int32:
        # the kernels read int32; anything else is converted once (ids that do not fit cannot be consecutive)
        lo, hi = dev.min(), dev.max()
        if lo < 1 or hi > numpy.iinfo(numpy.int32).max or (dev.dtype.kind == "f" and not (dev == numpy.floor(dev)).all()):
            raise AttributeError("The supplied label image does either not contain any regions or they are not labeled "
                                 "consecutively starting from 1.")
        dev = dev.astype(numpy.int32)
    elif any(s <= 0 and n > 1 for s, n in zip(dev.strides, dev.shape)):
        dev = numpy.ascontiguousarray(dev)
    return dev


def device_values(array, shape, what):
    """``array`` as an image of ``shape`` in a dtype the kernels read: the rule of ``LabelContext.values``."""
    a = numpy.asarray(array)
    if a.shape != shape:
        raise ValueError("{} of shape {} does not match the label image of shape {}".format(what, a.shape, shape))
    if not a.dtype.isnative:                       # '>f4', '>i2' (FITS / NIfTI readers): the kernels read native values
        a = a.astype(a.dtype.newbyteorder("="))
    if a.dtype == numpy.bool_:
        a = a.view(numpy.uint8)
    if a.dtype.type not in _DEVICE_DTYPES:
        a = a.astype(numpy.float64)
    if any(s <= 0 and n > 1 for s, n in zip(a.strides, a.shape)):
        a = numpy.ascontiguousarray(a)
    return a


class LabelContext:
    """A label image resident on the device (``mgc_labels``): created once by ``graph_from_labels`` and shared by the
    terms and the marker step, or created on the fly when a term is called on its own."""

    def __init__(self, label_image, device=-1):
        label_image = numpy.asarray(label_image)
        self.source = label_image
        dev = device_labels(label_image)
        from .. import _lib  # raises ImportError loudly when the extension is not built
        self._mgc = _lib._mgc
        self.native = _lib._mgc.LabelImage(dev, device)     # AttributeError unless the ids are exactly 1..K
        self.shape = label_image.shape
        self.regions = int(self.native.region_count())

    def values(self, array, what):
        """An image over the label image's shape in a dtype the kernels read (others are widened to float64, which is
        what the reference's arithmetic does to them anyway)."""
        return device_values(array, self.shape, what)

    def region_flags(self, markers):
        m = numpy.asarray(markers, dtype=numpy.bool_)
        if m.shape != self.shape:
            raise IndexError("boolean index did not match the label image: marker shape {} vs {}".format(m.shape, self.shape))
        if any(s <= 0 and n > 1 for s, n in zip(m.strides, m.shape)):
            m = numpy.ascontiguousarray(m)
        return self.native.region_flags(m.view(numpy.uint8))

    def apply(self, per_region):
        """Voxel image with ``per_region[label - 1]`` (uint8): maps a cut back onto the voxels."""
        return self.native.apply(numpy.ascontiguousarray(per_region, dtype=numpy.uint8))


def _context(graph, label_image):
    ctx = getattr(graph, "_label_context", None)
    if ctx is not None and ctx.source is label_image:
        return ctx
    return LabelContext(label_image)


def _refuse_size_one_axes(shape):
    # numpy.vectorize cannot run on the empty slices a size-1 axis produces (energy_label.py:325-328, 430-439)
    if any(int(s) == 1 for s in shape):
        raise ValueError("cannot call `vectorize` on size 0 inputs unless `otypes` is set")


def _add_edges(graph, i, j, w_there, w_back):
    from .graph import GCGraph
    from .multilabel import _PairRecorder
    if isinstance(graph, _PairRecorder) or (isinstance(graph, GCGraph) and type(graph).set_nweight is GCGraph.set_nweight):
        graph.set_nweights_bulk(i, j, w_there, w_back)
    else:   # someone else's graph object (e.g. the recording double of tests/graphcut_/energy_label.py:189-210)
        for a, b, x, y in zip(i.tolist(), j.tolist(), w_there.tolist(), w_back.tolist()):
            graph.set_nweight(a, b, x, y)


def boundary_difference_of_means(graph, label_image, original_image):
    """energy_label.py:33-120: weights from the difference of the regions' mean intensities."""
    ctx = _context(graph, label_image)
    sums, counts = ctx.native.region_sums(ctx.values(original_image, "original_image"), ctx._mgc.SUM_BINCOUNT)
    means = sums / counts.astype(numpy.float64)          # scipy.ndimage.mean: bincount sums / counts
    max_difference = float(abs(means.min() - means.max()))
    _refuse_size_one_axes(ctx.shape)
    i, j, _, _ = ctx.native.boundary(ctx._mgc.LABELS_ADJACENCY)
    if 0.0 == max_difference:
        w = numpy.full(i.size, _DBL_MIN)
    else:
        w = 1.0 - numpy.abs(means[i] - means[j]) / max_difference
        w = numpy.where(_DBL_MIN > w, _DBL_MIN, w)       # max(value, sys.float_info.min)
    _add_edges(graph, i, j, w, w.copy())


def boundary_stawiaski(graph, label_image, gradient_image):
    """energy_label.py:123-214: sum over the border voxel pairs of g(max(|grad_p|, |grad_q|)), g(x) = (1/(1+x))^2."""
    ctx = _context(graph, label_image)
    i, j, w, w_back = ctx.native.boundary(ctx._mgc.LABELS_STAWIASKI, ctx.values(gradient_image, "gradient_image"), 0.0)
    _add_edges(graph, i, j, w, w_back)


def boundary_stawiaski_directed(graph, label_image, term_args):
    """energy_label.py:217-342: as ``boundary_stawiaski`` with ``min(1, g + |directedness|)`` on the direction the
    sign of ``directedness`` favours."""
    (gradient_image, directedness) = term_args
    ctx = _context(graph, label_image)
    values = ctx.values(gradient_image, "gradient_image")
    _refuse_size_one_axes(ctx.shape)
    i, j, w, w_back = ctx.native.boundary(ctx._mgc.LABELS_STAWIASKI_DIRECTED, values, float(directedness))
    _add_edges(graph, i, j, w, w_back)


def regional_atlas(graph, label_image, term_args):
    """energy_label.py:345-396: set_tweight(region, alpha * S, -alpha * S), S = sum of the atlas under the region."""
    (probability_map, alpha) = term_args
    ctx = _context(graph, label_image)
    prob = numpy.asarray(probability_map)
    sums, _ = ctx.native.region_sums(ctx.values(prob, "probability_map"), ctx._mgc.SUM_PAIRWISE)
    weight = sums.astype(numpy.float32) if prob.dtype == numpy.float32 else sums
    src = numpy.asarray(alpha * weight, dtype=numpy.float64)          # numpy-2: float32 sums keep the product in float32
    snk = numpy.asarray(-1.0 * alpha * weight, dtype=numpy.float64)
    nodes = numpy.arange(ctx.regions)
    from .graph import GCGraph
    if isinstance(graph, GCGraph) and type(graph).set_tweight is GCGraph.set_tweight:
        graph.set_tweights_bulk(nodes, src, snk)
    else:
        for r, a, b in zip(nodes.tolist(), src.tolist(), snk.tolist()):
            graph.set_tweight(r, a, b)
