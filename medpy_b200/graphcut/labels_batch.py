"""A batch of label images cut as one region graph: ``graph_from_labels_batch`` (DESIGN.md §8, "A batch of label
images").

B label images -- ragged, or stacked along a first axis -- are staged once as one concatenation (``mgc_labels_create_batch``)
and their region graphs are built and cut as one disjoint union: one border-pair reduction per boundary term, one
region-sum pass per term that needs one, one sparse solve and one voxel gather.  Region r of image b is node
``node_offsets[b] + r - 1``.  No arc joins two images, so every image is cut as its own ``graph_from_labels`` call would
cut it: the same edge weights (bit for bit), the same t-links, the same mask; its energy is split off the union's by the
solver (``mgc_sparse_get_segment_energies``).

A batch built with ``warm=True`` keeps the solved state: seeds, t-links and edges added or lowered on the regions of one
or more images fold into it, and the next ``maxflow()`` continues from the flow already routed.  Each image keeps its
own energy through the folds, and an image that no edit touched keeps its mask and energy bit for bit.
"""
import numpy

from . import _warm_args, energy_label
from .energy_label import _DBL_MIN, device_labels, device_values
from .graph import GCGraph
from .maxflow import _termtype
from .sparse import warm_pairs, warm_seeds, warm_tweights

__all__ = ["graph_from_labels_batch", "LabelBatchGraph"]

_TERMS = (energy_label.boundary_stawiaski, energy_label.boundary_stawiaski_directed,
          energy_label.boundary_difference_of_means, energy_label.regional_atlas)


def _per_image(x, count, what):
    """A list / tuple of per-image arrays, or an array stacked along its first axis -> list of arrays."""
    if isinstance(x, (list, tuple)):
        items = [numpy.asarray(a) for a in x]
    else:
        a = numpy.asarray(x)
        if a.ndim < 1:
            raise ValueError("{}: one array per image expected, as a list or stacked along a first axis".format(what))
        items = list(a)
    if count is not None and len(items) != count:
        raise ValueError("{}: {} arrays for a batch of {} label images".format(what, len(items), count))
    return items


def _at(b, fn, *args):
    """fn(*args); an error is re-raised with the same type, naming image b."""
    try:
        return fn(*args)
    except (ValueError, AttributeError, IndexError) as e:
        raise type(e)("label image {}: {}".format(b, e)) from None


def _concat(arrays):
    """One C-ordered 1-D concatenation; images of different dtypes meet in their common dtype (numpy.result_type)."""
    return numpy.concatenate([numpy.ravel(a) for a in arrays])


class _Term:
    """One of the four energy_label terms with its per-image inputs, checked as that term checks them."""

    def __init__(self, fn, args, shapes):
        self.fn = fn
        if fn is energy_label.boundary_stawiaski_directed:
            images, self.directedness = args
        elif fn is energy_label.regional_atlas:
            images, self.alpha = args
        else:
            images = args
        what = {energy_label.boundary_difference_of_means: "original_image",
                energy_label.regional_atlas: "probability_map"}.get(fn, "gradient_image")
        self.images = _per_image(images, len(shapes), what)
        self.what = what
        self.values = [None] * len(shapes)

    def check(self, b, shape):
        self.values[b] = _at(b, device_values, self.images[b], shape, self.what)
        if self.fn in (energy_label.boundary_stawiaski_directed, energy_label.boundary_difference_of_means):
            _at(b, energy_label._refuse_size_one_axes, shape)

    def apply(self, mgc, native, graph, off):
        vals = _concat(self.values)
        if self.fn is energy_label.regional_atlas:
            sums, _ = native.region_sums(vals, mgc.SUM_PAIRWISE)
            # regional_atlas keeps float32 sums of a float32 atlas (numpy-2 promotion), per image
            f32 = numpy.repeat([vals.dtype == numpy.float32 and a.dtype == numpy.float32 for a in self.images], numpy.diff(off))
            alpha, w32 = self.alpha, sums.astype(numpy.float32)
            src = numpy.where(f32, numpy.asarray(alpha * w32, dtype=numpy.float64), numpy.asarray(alpha * sums, dtype=numpy.float64))
            snk = numpy.where(f32, numpy.asarray(-1.0 * alpha * w32, dtype=numpy.float64),
                              numpy.asarray(-1.0 * alpha * sums, dtype=numpy.float64))
            graph.add_tweights(numpy.arange(int(off[-1]), dtype=numpy.int32), src, snk)
            return
        if self.fn is energy_label.boundary_difference_of_means:
            sums, counts = native.region_sums(vals, mgc.SUM_BINCOUNT)
            means = sums / counts.astype(numpy.float64)          # scipy.ndimage.mean, per image
            starts = off[:-1]
            max_difference = numpy.abs(numpy.minimum.reduceat(means, starts) - numpy.maximum.reduceat(means, starts))
            i, j, _, _ = native.boundary(mgc.LABELS_ADJACENCY)
            md = max_difference[numpy.searchsorted(off, i, side="right") - 1]
            flat = md == 0.0
            w = 1.0 - numpy.abs(means[i] - means[j]) / numpy.where(flat, 1.0, md)
            w = numpy.where(_DBL_MIN > w, _DBL_MIN, w)           # max(value, sys.float_info.min)
            w = numpy.where(flat, _DBL_MIN, w)
            w_back = w.copy()
        elif self.fn is energy_label.boundary_stawiaski:
            i, j, w, w_back = native.boundary(mgc.LABELS_STAWIASKI, vals, 0.0)
        else:
            i, j, w, w_back = native.boundary(mgc.LABELS_STAWIASKI_DIRECTED, vals, float(self.directedness))
        bad = (w <= 0) | (w_back <= 0)
        if bad.any():                                            # GCGraph.set_nweights_bulk's check
            b = int(numpy.searchsorted(off, i[numpy.argmax(bad)], side="right") - 1)
            raise ValueError("label image {}: Negative or zero weights are not allowed.".format(b))
        graph.sum_edges(i, j, w, w_back)


def graph_from_labels_batch(label_images, fg_markers, bg_markers, regional_term=False, boundary_term=False,
                            regional_term_args=False, boundary_term_args=False, *, warm=False):
    """``graph_from_labels`` for B label images at once, cut as one graph.

    ``label_images``, ``fg_markers`` and ``bg_markers`` are lists of B arrays (the images may differ in shape, not in
    their number of dimensions) or arrays stacked along a first axis of length B.  The terms are the four
    ``energy_label`` callables (any other callable raises ``TypeError``); their per-image inputs come the same way: a
    gradient (or original image) per image, ``(gradients, directedness)`` for ``boundary_stawiaski_directed`` and
    ``(probability_maps, alpha)`` for ``regional_atlas``, with one ``directedness`` / ``alpha`` for the batch.  Each
    image's inputs follow the dtype rules of a single call; images of different dtypes are converted once to their
    common dtype and computed in it.

    Each image raises what its own ``graph_from_labels`` call would raise, naming its index; when several images fail,
    the host-side checks (label images, term inputs, marker shapes) come first, image by image, then the label ids, then
    the markers' region sets.  Returns a ``LabelBatchGraph``.

    ``warm=True`` keeps the solved state for the warm edits of ``LabelBatchGraph`` (``add_seeds``, ``remove_seeds``,
    ``add_tweights_warm``, ``add_nweights_warm``, ``remove_nweights_warm``), as ``graph_from_labels(..., warm=True)``
    does for one image.
    """
    stacked = not isinstance(label_images, (list, tuple))
    labels = _per_image(label_images, None, "label_images")
    if not labels:
        raise ValueError("an empty batch: graph_from_labels_batch needs at least one label image")
    B = len(labels)
    terms = []
    for fn, args, what in ((regional_term, regional_term_args, "regional_term"),
                           (boundary_term, boundary_term_args, "boundary_term")):
        if not fn:
            continue
        if not any(fn is t for t in _TERMS):
            raise TypeError("{}: graph_from_labels_batch takes the energy_label terms boundary_stawiaski, "
                            "boundary_stawiaski_directed, boundary_difference_of_means and regional_atlas only; "
                            "cut with graph_from_labels for other terms".format(what))
        terms.append((fn, args))
    fg = _per_image(fg_markers, B, "fg_markers")
    bg = _per_image(bg_markers, B, "bg_markers")
    shapes = [lab.shape for lab in labels]
    terms = [_Term(fn, args, shapes) for fn, args in terms]
    dev, fgs, bgs = [], [], []
    for b, lab in enumerate(labels):
        dev.append(_at(b, device_labels, lab))
        if lab.ndim != labels[0].ndim:
            raise ValueError("label image {}: the images of a batch must have one number of dimensions ({} here, {} for "
                             "image 0)".format(b, lab.ndim, labels[0].ndim))
        for t in terms:
            t.check(b, lab.shape)
        for m, out in ((fg[b], fgs), (bg[b], bgs)):
            m = numpy.asarray(m, dtype=numpy.bool_)
            if m.shape != lab.shape:
                raise IndexError("label image {}: boolean index did not match the label image: marker shape {} vs "
                                 "{}".format(b, m.shape, lab.shape))
            out.append(m)

    from .. import _lib  # raises ImportError loudly when the extension is not built
    mgc = _lib._mgc
    native = mgc.LabelImage.batch([list(s) for s in shapes], _concat(dev))   # AttributeError naming the image
    off = numpy.asarray(native.batch_offsets(), dtype=numpy.int64)
    graph = mgc.SparseGraph(int(off[-1]))
    if warm:
        graph.set_option(mgc.OPT_WARM, 1)
    graph.set_option(mgc.OPT_SEGMENT_ENERGIES, 1)
    for t in terms:                                               # regional term, then boundary term
        t.apply(mgc, native, graph, off)
    # set_source_nodes then set_sink_nodes (generate.py:334-337); each image needs both, like GCGraph's max([])
    flags = [native.region_flags(_concat(ms).view(numpy.uint8)) for ms in (fgs, bgs)]
    has = [numpy.add.reduceat(f.astype(numpy.int64), off[:-1]) for f in flags]      # every image has a region
    for b in range(B):
        if not has[0][b] or not has[1][b]:
            raise ValueError("label image {}: max() arg is an empty sequence".format(b))
    for f, src, snk in ((flags[0], GCGraph.MAX, 0.0), (flags[1], 0.0, GCGraph.MAX)):
        ids = numpy.nonzero(f)[0].astype(numpy.int32)
        graph.add_tweights(ids, numpy.full(ids.size, float(src)), numpy.full(ids.size, float(snk)))
    return LabelBatchGraph(native, graph, off, shapes, stacked, warm)


class LabelBatchGraph:
    """The solved union of a batch's region graphs (what ``graph_from_labels_batch`` returns).

    On a batch built with ``warm=True`` the warm methods take node ids over the union (region r of image b is node
    ``node_offsets[b] + r - 1``) or a boolean mask over all ``node_offsets[-1]`` regions, with the arguments, checks and
    errors of ``SparseGraphDouble``'s warm calls; ``region_flags`` turns strokes drawn on the images into such a mask.
    A pair whose ends lie in two images raises ``ValueError``.  Every refusal comes before any native call, so the
    batch is unchanged."""

    termtype = _termtype

    def __init__(self, native_labels, graph, node_offsets, shapes, stacked, warm=False):
        self._labels = native_labels
        self._graph = graph
        self._off = node_offsets
        self._shapes = [tuple(s) for s in shapes]
        self._stacked = stacked
        self._warm = bool(warm)
        self._vox_off = numpy.concatenate([[0], numpy.cumsum([int(numpy.prod(s)) for s in self._shapes])]).astype(numpy.int64)

    @property
    def warm(self):
        """Whether the batch keeps its solved state for warm edits (``graph_from_labels_batch(..., warm=True)``)."""
        return self._warm

    @property
    def node_offsets(self):
        """int64[B+1]: region r of image b is node node_offsets[b] + r - 1; node_offsets[B] = all regions."""
        return self._off.copy()

    def __len__(self):
        return len(self._shapes)

    def maxflow(self):
        """float64[B]: each image's min-cut energy, including its add_tweights constants."""
        return self._graph.segment_energies(self._off)

    def get_mask(self):
        """Per image, uint8[K_b]: 0 where the region is on the SINK side, else 1."""
        m = self._graph.get_mask()
        return [m[a:b] for a, b in zip(self._off[:-1], self._off[1:])]

    def label_cut_masks(self):
        """Per image, what ``label_cut_mask`` gives: the voxel mask, 1 where the voxel's region is not on the SINK side;
        one (B, ...) array for stacked input."""
        vox = self._labels.apply(self._graph.get_mask())
        if self._stacked:
            return vox.reshape((len(self._shapes),) + self._shapes[0])
        ends = numpy.cumsum([int(numpy.prod(s)) for s in self._shapes])
        return [part.reshape(s) for part, s in zip(numpy.split(vox, ends[:-1]), self._shapes)]

    def stats(self):
        """The sparse solve's statistics, with the batch size."""
        d = dict(self._graph.stats())
        d["images"] = len(self._shapes)
        return d

    def region_flags(self, strokes):
        """bool[node_offsets[-1]]: True for every region of the union that holds a marked voxel.  ``strokes`` has one
        entry per image, ``None`` or a mask of that image's shape (a numpy array or a CUDA tensor), as a list or stacked
        along a first axis.  Only the marked voxels of the given images go to the device, as ids."""
        items = list(strokes)
        if len(items) != len(self._shapes):
            raise ValueError("strokes: {} entries for a batch of {} label images".format(len(items), len(self._shapes)))
        ids = [numpy.zeros(0, numpy.int64)]
        for b, m in enumerate(items):
            if m is None:
                continue
            if _warm_args.on_device(m):
                import torch
                m = torch.as_tensor(m)
                shape = tuple(m.shape)
            else:
                m = numpy.asarray(m, dtype=numpy.bool_)
                shape = m.shape
            if shape != self._shapes[b]:
                raise IndexError("label image {}: boolean index did not match the label image: stroke shape {} vs "
                                 "{}".format(b, shape, self._shapes[b]))
            v = numpy.flatnonzero(m) if isinstance(m, numpy.ndarray) else m.reshape(-1).nonzero().reshape(-1).cpu().numpy()
            ids.append(v.astype(numpy.int64) + self._vox_off[b])
        return self._labels.voxel_flags(numpy.concatenate(ids)).view(numpy.bool_)

    # ------------------------------------------------------------------ warm edits (batches built with warm=True)
    def _require_warm(self, what):
        if not self._warm:
            raise RuntimeError("{} needs a label batch built with warm=True; rebuild it with "
                               "graph_from_labels_batch(..., warm=True) instead".format(what))

    def add_seeds(self, fg=None, bg=None):
        """add_tweights(v, 65535, 0) per foreground id in order, then add_tweights(v, 0, 65535) per background id."""
        self._require_warm("add_seeds")
        for call in warm_seeds(fg, bg, 65535.0, int(self._off[-1])):
            self._graph.add_tweights(*call)

    def remove_seeds(self, fg=None, bg=None):
        """The inverse of add_seeds: add_tweights(v, -65535, 0) / add_tweights(v, 0, -65535)."""
        self._require_warm("remove_seeds")
        for call in warm_seeds(fg, bg, -65535.0, int(self._off[-1])):
            self._graph.add_tweights(*call)

    def add_tweights_warm(self, nodes, cap_source, cap_sink):
        """add_tweights(nodes[k], cap_source[k], cap_sink[k]) per entry in order; nodes None: one call per node."""
        self._require_warm("add_tweights_warm")
        ids, src, snk = warm_tweights(nodes, cap_source, cap_sink, int(self._off[-1]))
        if src.size:
            self._graph.add_tweights(ids, src, snk)

    def _pairs(self, i, j, cap, rev_cap, why):
        """warm_pairs over the union; a pair across two images is refused (no arc may join them, or the energy split
        would be meaningless)."""
        ii, jj, c, r = warm_pairs(i, j, cap, rev_cap, int(self._off[-1]), why)
        bi = numpy.searchsorted(self._off, ii, side="right") - 1
        bj = numpy.searchsorted(self._off, jj, side="right") - 1
        cross = numpy.flatnonzero(bi != bj)
        if cross.size:
            k = cross[0]
            raise ValueError("the pair ({}, {}) joins label image {} and label image {}: an edge must stay inside one "
                             "image".format(ii[k], jj[k], bi[k], bj[k]))
        return ii, jj, c, r

    def add_nweights_warm(self, i, j, cap, rev_cap):
        """sum_edge(i[k], j[k], cap[k], rev_cap[k]) per entry in order, on any pairs inside one image (new ones
        included)."""
        self._require_warm("add_nweights_warm")
        ii, jj, c, r = self._pairs(i, j, cap, rev_cap, _warm_args.ONLY_RAISES)
        if ii.size:
            self._graph.sum_edges(ii, jj, c, r)

    def remove_nweights_warm(self, i, j, cap, rev_cap):
        """sum_edge(i[k], j[k], -cap[k], -rev_cap[k]) per entry in order on existing pairs.  A pair whose decrements
        exceed what it holds (beyond a few hundred roundings) raises ValueError with the batch unchanged."""
        self._require_warm("remove_nweights_warm")
        ii, jj, c, r = self._pairs(i, j, cap, rev_cap, _warm_args.DECREMENTS)
        if ii.size:
            self._graph.remove_edges_warm(ii, jj, c, r)
