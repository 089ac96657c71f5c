"""K-label segmentation of a voxel image, or of a label image's regions, by alpha-expansion (Boykov, Veksler & Zabih
2001; DESIGN.md §11).

MedPy's cut is binary: one structure against the rest.  ``expansion_from_voxels`` labels every voxel with one of K
labels (organs, tumour sub-regions) by minimising the Potts energy whose terms ``graph_from_voxels`` already defines:

    E(l) = sum_p D_p(l_p) + sum_{lattice pairs} w_pq [l_p != l_q]

``D_p(k)`` is the caller's cost of label k at p, ``w_pq`` the weight the boundary term puts on the pair.  Each move is one
binary cut of the lattice on the GPU; the loop, the move graphs, the label updates and the energy never leave the device.
``expansion_from_labels`` does the same over the region adjacency graph ``graph_from_labels`` builds, with the region
sums of the caller's costs as the data term and the ``energy_label`` boundary term's weight as the pair term; each move is
one cut of the region graph by the sparse push-relabel.  ``expansion_from_voxels_batch`` segments B images of one shape
together, every move one cut of the whole batch lattice, each image exactly as ``expansion_from_voxels`` segments it alone.
"""
import math

import numpy

from .energy_voxel import _native_order
from .generate import _takes_three_parameters, _takes_two_parameters
from .graph import GCGraph

_MAX = float(GCGraph.MAX)       # the soft-hard seed of a marker


class _BoundaryRecorder:
    """What a boundary term of ``energy_voxel`` receives in place of a GCGraph: it keeps the one bulk call the term makes
    (``GCGraph._add_boundary``), whose arguments become the pair weights of every move."""

    def __init__(self):
        self.call = None

    def _add_boundary(self, kind, image, sigma, spacing, norm):
        if self.call is not None:
            raise ValueError("the boundary term added more than one set of pair weights")
        self.call = (kind, image, sigma, spacing, norm)


class _PairRecorder:
    """What a boundary term of ``energy_label`` receives in place of a GCGraph: it keeps the term's one bulk edge call
    (``energy_label._add_edges``), whose pairs and weights become the pair term of every move.  The Potts energy has one
    weight per region pair, so the two directions must carry the same bits."""

    def __init__(self, context):
        self._label_context = context       # the terms reuse the staged label image
        self.pairs = None

    def set_nweights_bulk(self, i, j, w_there, w_back):
        if self.pairs is not None:
            raise ValueError("the boundary term added more than one set of pair weights")
        w = numpy.ascontiguousarray(w_there, dtype=numpy.float64)
        w_back = numpy.ascontiguousarray(w_back, dtype=numpy.float64)
        if w.shape != w_back.shape or not numpy.array_equal(w.view(numpy.uint64), w_back.view(numpy.uint64)):
            raise ValueError("the boundary term's weights differ between the two directions of a pair (w_ij != w_ji); "
                             "the Potts energy takes one weight per region pair")
        if w.size and not bool((numpy.isfinite(w) & (w >= 0)).all()):
            raise ValueError("the boundary term's weights must be finite and >= 0")
        self.pairs = (numpy.ascontiguousarray(i, dtype=numpy.int32), numpy.ascontiguousarray(j, dtype=numpy.int32), w)


def _on_device(a):
    return hasattr(a, "__cuda_array_interface__")


def _float_costs(a, what):
    """``a`` as a float32 / float64 CUDA tensor or numpy array in native byte order."""
    if _on_device(a):
        if str(a.dtype) not in ("torch.float32", "torch.float64"):
            raise ValueError("{} must be float32 or float64, got {}".format(what, a.dtype))
        return a
    a = _native_order(numpy.asarray(a))
    if a.dtype not in (numpy.float32, numpy.float64):
        raise ValueError("{} must be float32 or float64, got {}".format(what, a.dtype))
    return a


def _check_range(a, what):
    if _on_device(a):
        bad = a.numel() and not bool((a.isfinite() & (a >= 0)).all())
    else:
        bad = a.size and not bool((numpy.isfinite(a) & (a >= 0)).all())
    if bad:
        raise ValueError("{} must be finite and >= 0".format(what))


def _label_image(a, shape, what, limit):
    """An integer image of `shape` with values in 0..limit, as uint8 on its own side (host or device)."""
    if _on_device(a):
        if tuple(a.shape) != tuple(shape):
            raise ValueError("{} must have the image shape {}, got {}".format(what, tuple(shape), tuple(a.shape)))
        if a.dtype.is_floating_point or a.dtype.is_complex:
            raise ValueError("{} must hold integers".format(what))
        if a.numel() and (bool((a < 0).any()) or bool((a > limit).any())):
            raise ValueError("{} must hold values in 0..{}".format(what, limit))
        import torch
        return a.to(torch.uint8).contiguous()
    a = numpy.asarray(a)
    if a.shape != tuple(shape):
        raise ValueError("{} must have the image shape {}, got {}".format(what, tuple(shape), a.shape))
    if a.dtype.kind not in "biu":
        raise ValueError("{} must hold integers".format(what))
    if a.size and (int(a.min()) < 0 or int(a.max()) > limit):
        raise ValueError("{} must hold values in 0..{}".format(what, limit))
    return numpy.ascontiguousarray(a, dtype=numpy.uint8)


def _check_labels_and_cycles(K, where, max_cycles):
    """K (the labels, from the costs' axis `where`) in 2..255 and max_cycles an integer >= 1."""
    if not 2 <= K <= 255:
        raise ValueError("the number of labels K = {} must be 2..255, got {}".format(where, K))
    if isinstance(max_cycles, bool) or not isinstance(max_cycles, (int, numpy.integer)) or max_cycles < 1:
        raise ValueError("max_cycles must be an integer >= 1")


def _check_init_markers(markers, init):
    """Refuse an init that gives a marked voxel another label than its marker (either may be None)."""
    if markers is None or init is None:
        return
    if _on_device(markers) and _on_device(init):
        m, i = markers.long(), init.long()
    else:       # one side on the host: compare there
        m, i = (numpy.asarray(a.cpu() if _on_device(a) else a, dtype=numpy.int64) for a in (markers, init))
    if bool(((m > 0) & (i != m - 1)).any()):
        raise ValueError("init gives a marked voxel another label than its marker")


def _check_moves(moves):
    """The move kind, "expansion" or "swap"; True for swap moves."""
    if not isinstance(moves, str) or moves not in ("expansion", "swap"):
        raise ValueError("moves must be \"expansion\" or \"swap\", got {!r}".format(moves))
    return moves == "swap"


def _label_distance(V, K, swap=False):
    """A label distance as a C-contiguous float64 (K, K) numpy array, refused (ValueError) unless it is a metric: finite
    entries >= 0, a zero diagonal, symmetric, and V[a][c] <= V[a][b] + V[b][c] in float64 for every a, b, c.  With
    ``swap`` the triangle rule is skipped: swap moves take any semi-metric.  The message names the rule and the first
    (a, b) or (a, b, c), in C order, that breaks it: the native check's words.  A CUDA tensor is copied to the host (K^2
    numbers)."""
    if _on_device(V):
        V = V.detach().cpu().numpy()
    V = numpy.asarray(V)
    if V.dtype.kind not in "iuf":
        raise ValueError("label_distance must hold real numbers, got {}".format(V.dtype))
    V = numpy.ascontiguousarray(V, dtype=numpy.float64)
    if V.shape != (K, K):
        raise ValueError("label_distance must be a (K, K) = ({}, {}) matrix, got shape {}".format(K, K, V.shape))
    bad = numpy.argwhere(~(numpy.isfinite(V) & (V >= 0)))
    if bad.size:
        raise ValueError("label_distance must be finite and >= 0, V[{}][{}] is not".format(*bad[0]))
    bad = numpy.flatnonzero(numpy.diagonal(V) != 0)
    if bad.size:
        raise ValueError("label_distance must have a zero diagonal, V[{0}][{0}] is not 0".format(bad[0]))
    bad = numpy.argwhere(V != V.T)
    if bad.size:
        a, b = bad[0]
        raise ValueError("label_distance must be symmetric, V[{0}][{1}] != V[{1}][{0}]".format(a, b))
    if swap:
        return V
    for a in range(K):
        bad = numpy.argwhere(V[a][None, :] > V[a][:, None] + V)        # [b, c]: V[a][c] > V[a][b] + V[b][c]
        if bad.size:
            b, c = bad[0]
            raise ValueError("label_distance must satisfy the triangle inequality V[a][c] <= V[a][b] + V[b][c], "
                             "(a, b, c) = ({}, {}, {}) breaks it; a semi-metric such as truncated quadratic needs "
                             "alpha-beta swap moves".format(a, b, c))
    return V


def expansion_from_voxels(costs, boundary_term=False, boundary_term_args=False, markers=None, init=None, max_cycles=20,
                          stats=False, *, label_distance=None, moves="expansion"):
    """Segment a voxel image into K labels by alpha-expansion.

    costs              (K, *shape) float32 or float64, a numpy array or a CUDA tensor; ``costs[k]`` is the cost of label k
                       per voxel (finite, >= 0).  2 <= K <= 255, the image has 1 to 4 dimensions.
    boundary_term      one of the eight ``energy_voxel.boundary_*`` functions with its ``boundary_term_args``, as
                       ``graph_from_voxels`` takes them; its weight on a pair is the price of a label change across it.
                       False: no pair term.
    markers            integer image, 0 = free, m > 0 = the voxel belongs to label m-1: every other label costs 65535
                       (GCGraph.MAX) more there, MedPy's soft-hard seed.  With K = 2 and markers 1 = background,
                       2 = foreground, the result is graph_from_voxels' cut.
    init               initial labels (0..K-1, agreeing with the markers); default argmin_k costs[k], ties to the lowest k.
    max_cycles         cycles at most, of the moves 0, 1, ..., K-1 (expansion) or of the K(K-1)/2 pairs (swap); the loop
                       stops earlier after a cycle that switches no voxel.
    stats              also return a dict: moves, cycles, converged, switched (voxels per move), energy and device ms.
    label_distance     (K, K) label distance V (numpy array, nested sequence or CUDA tensor; keyword only): the pair term
                       becomes w_pq V(l_p, l_q), so a change between distant labels costs more than one between
                       neighbours, e.g. ``numpy.minimum(abs(i - j), 2)`` for ordered labels.  Finite, >= 0, zero on the
                       diagonal and symmetric; under expansion moves it must also satisfy the triangle inequality
                       (DESIGN.md §11, "Label distances"), under swap moves it need not (truncated quadratic
                       ``numpy.minimum((i - j) ** 2, 4)``).  None: Potts.
    moves              (keyword only) "expansion": cycles of alpha-expansions alpha = 0, 1, ..., K-1; "swap": cycles of
                       alpha-beta swaps (0, 1), (0, 2), ..., (K-2, K-1), each a cut over the voxels labelled alpha or beta
                       only, exact for any semi-metric label distance (DESIGN.md §11, "Swap moves").

    Returns ``(labels, energy)`` (``(labels, energy, stats)`` with ``stats=True``): uint8 labels of the image shape, a
    numpy array or, for CUDA costs, a CUDA tensor; ``energy`` the energy of those labels (Potts, or with the label
    distance).  Raises ``ValueError`` for
    malformed arguments and ``AttributeError`` for a boundary term that is not a two-parameter callable, before anything
    reaches the device.
    """
    device = -1
    swap = _check_moves(moves)
    costs = _float_costs(costs, "costs")
    if costs.ndim < 2 or costs.ndim > 5:
        raise ValueError("costs must have shape (K, *image shape) with a 1- to 4-D image")
    _check_range(costs, "costs")
    if _on_device(costs):
        device = costs.device.index
    K = int(costs.shape[0])
    shape = tuple(int(s) for s in costs.shape[1:])
    _check_labels_and_cycles(K, "costs.shape[0]", max_cycles)
    if min(shape) < 1:
        raise ValueError("the image must not be empty")

    rec = _BoundaryRecorder()
    if boundary_term:
        if not _takes_two_parameters(boundary_term):
            raise AttributeError("boundary_term has to be a callable object which takes two parameters.")
        boundary_term(rec, boundary_term_args)
        if rec.call is not None and numpy.shape(rec.call[1]) != shape:
            raise ValueError("the boundary term's image must have the image shape {}".format(shape))

    if markers is not None:
        markers = _label_image(markers, shape, "markers", K)
    if init is not None:
        init = _label_image(init, shape, "init", K - 1)
    _check_init_markers(markers, init)
    if label_distance is not None:
        label_distance = _label_distance(label_distance, K, swap)

    from .. import _lib  # raises ImportError loudly when the extension is not built
    on_dev = _on_device(costs)
    if on_dev or _on_device(markers) or _on_device(init):
        import torch
        torch.cuda.current_stream(device if device is not None and device >= 0 else None).synchronize()
    nat = _lib._mgc.Expansion(list(shape), K, -1 if device is None else device)
    for k in range(K):
        nat.set_cost(k, costs[k])
    if rec.call is not None:
        nat.set_boundary(*rec.call)
    if markers is not None:
        nat.set_markers(markers)
    if init is not None:
        nat.set_init(init)
    if swap:
        nat.set_moves(_lib._mgc.MOVES_SWAP)
    if label_distance is not None:
        nat.set_label_distance(label_distance)
    nat.run(int(max_cycles))
    st = nat.stats()
    if on_dev:
        import torch
        labels = torch.empty(shape, dtype=torch.uint8, device=costs.device)
        nat.labels_into(labels)
    else:
        labels = nat.labels()
    if stats:
        return labels, st["energy"], st
    return labels, st["energy"]


def expansion_from_voxels_batch(costs, image=None, boundary=None, sigma=None, spacing=False, markers=None, init=None,
                                max_cycles=20, stats=False, *, label_distance=None, moves="expansion"):
    """Segment B images of one shape into K labels by alpha-expansion, all in one loop (DESIGN.md §11, "Batches").

    Image b is segmented as ``expansion_from_voxels`` segments it alone: the same energy, bit for bit the same move
    graphs, the same stopping rule and ``max_cycles``.  Where the lattice solver returns each move's minimal minimum cut
    (as BK does), the labels, per-move switch counts, moves, cycles and converged flag are the single call's, and the
    energy is its energy up to the order of the sums.  The solver's floating-point residuals can move voxels off that
    cut on some graphs, depending on the image's tile position, so there the two calls can differ (DESIGN.md §11,
    "Batches").  Every move alpha is one cut of the whole batch; an image whose cycle switched nothing is frozen from
    then on, and the loop stops when every image is frozen or ``max_cycles`` cycles ran.

    costs              (B, K, *image) float32 or float64, a numpy array or a CUDA tensor, finite and >= 0; ``costs[b, k]``
                       is the cost of label k in image b.  2 <= K <= 255, images 1- to 3-D, B x voxels per image < 2^31.
    image, boundary    the (B, *image) image (numpy or CUDA) and one of the eight ``energy_voxel`` boundary terms by name
                       without the ``boundary_`` prefix (``"difference_exponential"`` ...), as ``graph_from_voxels_batch``
                       takes them.  None: no pair term.
    sigma              the term's sigma: one float for every image, or one per image.
    spacing            voxel spacing of the images (one entry per image axis), or False.
    markers, init      (B, *image) integer images with the meaning ``expansion_from_voxels`` gives them per image.
    max_cycles         cycles at most per image, of the moves 0, 1, ..., K-1 (expansion) or of the K(K-1)/2 pairs (swap).
    stats              also return a dict: the batch loop's ``batch_moves``, ``batch_cycles``, ``batch_converged``, per-image
                       lists ``moves``, ``cycles``, ``converged``, ``switched`` (voxels per move) and ``energy``, and the
                       device ms (``ms_build``, ``ms_solve``, ``ms_apply`` summed over the moves, ``ms_total``).
    label_distance     (K, K) label distance of every image, as ``expansion_from_voxels`` takes it; None: Potts.
    moves              "expansion" or "swap", as ``expansion_from_voxels`` takes it; a swap cycle is K(K-1)/2 moves of
                       every image.

    Returns ``(labels, energies)`` (``+ (stats,)`` with ``stats=True``): uint8 labels of shape (B, *image), a numpy array
    or, for CUDA costs, a CUDA tensor; ``energies`` a float64 numpy array of the B energies (Potts, or with the label
    distance).  Raises ``ValueError``
    for malformed arguments before anything reaches the device.
    """
    from .batch import INDEX_LIMIT, _host_image, _is_cuda, _sigmas
    from .device import _KINDS
    swap = _check_moves(moves)
    costs = _float_costs(costs, "costs")
    if costs.ndim < 3 or costs.ndim > 5:
        raise ValueError("costs must have shape (B, K, *image shape) with a 1- to 3-D image")
    _check_range(costs, "costs")
    B, K = int(costs.shape[0]), int(costs.shape[1])
    shape = tuple(int(s) for s in costs.shape[2:])
    _check_labels_and_cycles(K, "costs.shape[1]", max_cycles)
    if B < 1 or min(shape) < 1:
        raise ValueError("the batch and its images must not be empty")
    if B * math.prod(shape) >= INDEX_LIMIT:
        raise ValueError("{} images of {} voxels reach the 2^31 voxel index limit of one batch".format(B, math.prod(shape)))
    bshape = (B,) + shape
    if (image is None) != (boundary is None):
        raise ValueError("give both image and boundary for a pair term, or neither")
    if boundary is not None:
        if boundary not in _KINDS:
            raise ValueError("boundary must be one of {}, got {!r}".format(sorted(_KINDS), boundary))
        if tuple(int(s) for s in image.shape) != bshape:
            raise ValueError("image has shape {}, the costs need {}".format(tuple(image.shape), bshape))
        sigmas = _sigmas(sigma, B)
        sp = None
        if spacing:
            sp = [float(s) for s in spacing]
            if len(sp) < len(shape):
                raise ValueError("spacing has fewer entries than the images have dimensions")
        if _is_cuda(image):
            norms = [math.nan] * B
        else:
            image, norms = _host_image(image, boundary)

    if markers is not None:
        markers = _label_image(markers, bshape, "markers", K)
    if init is not None:
        init = _label_image(init, bshape, "init", K - 1)
    _check_init_markers(markers, init)
    if label_distance is not None:
        label_distance = _label_distance(label_distance, K, swap)

    from .. import _lib  # raises ImportError loudly when the extension is not built
    on_dev = _on_device(costs)
    device = costs.device.index if on_dev else -1
    if on_dev or _on_device(markers) or _on_device(init) or (boundary is not None and _on_device(image)):
        import torch
        torch.cuda.current_stream(device if device >= 0 else None).synchronize()
    nat = _lib._mgc.ExpansionBatch(list(shape), B, K, device)
    for k in range(K):
        # a host plane goes contiguous (a strided host array would upload its whole span); a CUDA plane is gathered there
        nat.set_cost(k, costs[:, k] if on_dev else numpy.ascontiguousarray(costs[:, k]))
    if boundary is not None:
        nat.set_boundary(_KINDS[boundary], image, sigmas, sp, norms)
    if markers is not None:
        nat.set_markers(markers)
    if init is not None:
        nat.set_init(init)
    if swap:
        nat.set_moves(_lib._mgc.MOVES_SWAP)
    if label_distance is not None:
        nat.set_label_distance(label_distance)
    nat.run(int(max_cycles))
    per = nat.image_stats()
    energies = numpy.asarray(per["energy"], dtype=numpy.float64)
    if on_dev:
        import torch
        labels = torch.empty(bshape, dtype=torch.uint8, device=costs.device)
        nat.labels_into(labels)
    else:
        labels = nat.labels()
    if not stats:
        return labels, energies
    return labels, energies, _batch_stats(nat.stats(), per, nat.switched())


def _batch_stats(total, per, switched):
    """The stats dict of ``expansion_from_voxels_batch`` from the native batch totals, the per-image statistics and the
    (moves, B) switch matrix: image b's switch counts are the first ``moves[b]`` rows of column b."""
    switched = numpy.asarray(switched, dtype=numpy.int64)
    moves = [int(m) for m in per["moves"]]
    return dict(batch_moves=int(total["moves"]), batch_cycles=int(total["cycles"]), batch_converged=bool(total["converged"]),
                moves=moves, cycles=[int(c) for c in per["cycles"]], converged=[bool(c) for c in per["converged"]],
                switched=[switched[:m, b].tolist() for b, m in enumerate(moves)],
                energy=[float(e) for e in per["energy"]],
                ms_build=total["ms_build"], ms_solve=total["ms_solve"], ms_apply=total["ms_apply"],
                ms_total=total["ms_total"])


def _region_values(a, regions, what, limit):
    """Integer region values of shape (regions,) in 0..limit, as a uint8 numpy array."""
    if _on_device(a):
        a = a.cpu()
    a = numpy.asarray(a)
    if a.shape != (regions,):
        raise ValueError("{} must have one entry per region, shape ({},), got {}".format(what, regions, a.shape))
    if a.dtype.kind not in "biu":
        raise ValueError("{} must hold integers".format(what))
    if a.size and (int(a.min()) < 0 or int(a.max()) > limit):
        raise ValueError("{} must hold values in 0..{}".format(what, limit))
    return numpy.ascontiguousarray(a, dtype=numpy.uint8)


def expansion_from_labels(label_image, costs=None, boundary_term=False, boundary_term_args=False, markers=None, init=None,
                          max_cycles=20, stats=False, *, region_costs=None, label_distance=None, moves="expansion"):
    """Segment the regions of a label image into K labels by alpha-expansion (DESIGN.md §11, "Region graphs").

    Minimises E(l) = sum_r D_r(l_r) + sum_{region pairs r<s} w_rs [l_r != l_s] over region labels 0..K-1
    (2 <= K <= 255) of a 1- to 4-D label image whose ids are exactly 1..R (``AttributeError`` otherwise, as
    ``graph_from_labels``); region r is node r-1.

    label_image        the regions, e.g. supervoxels.
    costs              (K, *label_image.shape) float32 or float64, a numpy array or a CUDA tensor, finite and >= 0:
                       D_r(k) is the sum of ``costs[k]`` over the voxels of region r+1 (numpy.bincount's float64 sum).
    region_costs       (K, R) float32 or float64, finite and >= 0: D_r(k) directly.  Give exactly one of the two.
    boundary_term      an ``energy_label`` boundary term with its ``boundary_term_args``, as ``graph_from_labels`` takes
                       them (a three-parameter callable); w_rs is the weight it puts on the pair, which must be the same
                       in both directions.  False: no pair term.
    markers            integer voxel image, 0 = free, m > 0 = label m-1: for every marker value in a region, every other
                       label costs 65535 (GCGraph.MAX) more there, so a region holding two marker values pays it for
                       every label.  With K = 2, region_costs (src, snk) of graph_from_labels' t-links and markers
                       1 = background, 2 = foreground, the result is graph_from_labels' cut.
    init               initial region labels, shape (R,), 0..K-1; a marked region must start at one of its markers'
                       labels.  Default argmin_k D_r(k), ties to the lowest k.
    max_cycles         cycles at most, of the moves 0, 1, ..., K-1 (expansion) or of the K(K-1)/2 pairs (swap); the loop
                       stops earlier after a cycle that switches no region.
    stats              also return a dict: moves, cycles, converged, switched (regions per move), energy and device ms.
    label_distance     (K, K) label distance, as ``expansion_from_voxels`` takes it: the pair term becomes
                       w_rs V(l_r, l_s).  None: Potts.
    moves              "expansion" or "swap", as ``expansion_from_voxels`` takes it.

    Returns ``(labels, region_labels, energy)`` (``+ (stats,)`` with ``stats=True``): ``labels`` the uint8 voxel image
    ``region_labels[label_image - 1]`` (a CUDA tensor when the costs are one, numpy otherwise), ``region_labels`` uint8
    of shape (R,), ``energy`` the energy of those labels (Potts, or with the label distance).
    """
    swap = _check_moves(moves)
    if (costs is None) == (region_costs is None):
        raise ValueError("give exactly one of costs and region_costs")
    label_image = numpy.asarray(label_image)
    shape = label_image.shape
    what = "costs" if region_costs is None else "region_costs"
    data = _float_costs(costs if region_costs is None else region_costs, what)
    if region_costs is None and (data.ndim != label_image.ndim + 1 or tuple(data.shape[1:]) != shape):
        raise ValueError("costs must have shape (K, *label_image.shape) = (K, {}), got {}".format(
            ", ".join(str(s) for s in shape), tuple(data.shape)))
    if region_costs is not None and data.ndim != 2:
        raise ValueError("region_costs must have shape (K, R), got {}".format(tuple(data.shape)))
    _check_range(data, what)
    K = int(data.shape[0])
    _check_labels_and_cycles(K, what + ".shape[0]", max_cycles)
    if label_distance is not None:
        label_distance = _label_distance(label_distance, K, swap)
    if boundary_term and not _takes_three_parameters(boundary_term):
        raise AttributeError("boundary_term has to be a callable object which takes three parameters.")
    if markers is not None:
        markers = _label_image(markers, shape, "markers", K)
        if _on_device(markers):
            markers = markers.cpu().numpy()

    from .energy_label import LabelContext
    on_dev = _on_device(data)
    device = data.device.index if on_dev else -1
    if on_dev:
        import torch
        torch.cuda.current_stream(device).synchronize()
    ctx = LabelContext(label_image, device)          # stages the image; AttributeError unless the ids are 1..R
    R = ctx.regions
    if region_costs is not None and int(data.shape[1]) != R:
        raise ValueError("region_costs must have shape (K, R) = ({}, {}), got {}".format(K, R, tuple(data.shape)))
    if init is not None:
        init = _region_values(init, R, "init", K - 1)

    if region_costs is None:
        D = numpy.empty((K, R))
        for k in range(K):
            D[k] = ctx.native.region_sums(data[k], ctx._mgc.SUM_BINCOUNT)[0]
    else:
        D = numpy.array(data.cpu().numpy() if on_dev else data, dtype=numpy.float64)
    if markers is not None:
        marked = numpy.zeros(R, bool)
        agrees = numpy.zeros(R, bool)
        for m in numpy.unique(markers):                 # ascending: the additions' order
            if m == 0:
                continue
            inside = ctx.native.region_flags(numpy.ascontiguousarray(markers == m).view(numpy.uint8)).astype(bool)
            D[numpy.ix_(numpy.arange(K) != m - 1, inside)] += _MAX
            marked |= inside
            if init is not None:
                agrees |= inside & (init == m - 1)
        if init is not None and bool((marked & ~agrees).any()):
            raise ValueError("init gives a marked region a label none of its markers gives it")

    rec = _PairRecorder(ctx)
    if boundary_term:
        boundary_term(rec, label_image, boundary_term_args)

    nat = ctx._mgc.RegionExpansion(R, K, device)
    for k in range(K):
        nat.set_cost(k, D[k])
    if rec.pairs is not None:
        nat.set_pairs(*rec.pairs)
    if init is not None:
        nat.set_init(init)
    if swap:
        nat.set_moves(ctx._mgc.MOVES_SWAP)
    if label_distance is not None:
        nat.set_label_distance(label_distance)
    nat.run(int(max_cycles))
    st = nat.stats()
    region_labels = nat.labels()
    if on_dev:
        import torch
        labels = torch.empty(shape, dtype=torch.uint8, device=data.device)
        ctx.native.apply_into(region_labels, labels)
    else:
        labels = ctx.apply(region_labels)
    if stats:
        return labels, region_labels, st["energy"], st
    return labels, region_labels, st["energy"]
