"""K-label segmentation of a voxel image by alpha-expansion (Boykov, Veksler & Zabih 2001; DESIGN.md §11).

MedPy's cut is binary: one structure against the rest.  ``expansion_from_voxels`` labels every voxel with one of K
labels (organs, tumour sub-regions) by minimising the Potts energy whose terms ``graph_from_voxels`` already defines:

    E(l) = sum_p D_p(l_p) + sum_{lattice pairs} w_pq [l_p != l_q]

``D_p(k)`` is the caller's cost of label k at p, ``w_pq`` the weight the boundary term puts on the pair.  Each move is one
binary cut of the lattice on the GPU; the loop, the move graphs, the label updates and the energy never leave the device.
"""
import numpy

from .energy_voxel import _native_order
from .generate import _takes_two_parameters


class _BoundaryRecorder:
    """What a boundary term of ``energy_voxel`` receives in place of a GCGraph: it keeps the one bulk call the term makes
    (``GCGraph._add_boundary``), whose arguments become the pair weights of every move."""

    def __init__(self):
        self.call = None

    def _add_boundary(self, kind, image, sigma, spacing, norm):
        if self.call is not None:
            raise ValueError("the boundary term added more than one set of pair weights")
        self.call = (kind, image, sigma, spacing, norm)


def _on_device(a):
    return hasattr(a, "__cuda_array_interface__")


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


def expansion_from_voxels(costs, boundary_term=False, boundary_term_args=False, markers=None, init=None, max_cycles=20,
                          stats=False):
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
    max_cycles         cycles of the moves 0, 1, ..., K-1 at most; the loop stops earlier after a cycle that switches no
                       voxel.
    stats              also return a dict: moves, cycles, converged, switched (voxels per move), energy and device ms.

    Returns ``(labels, energy)`` (``(labels, energy, stats)`` with ``stats=True``): uint8 labels of the image shape, a
    numpy array or, for CUDA costs, a CUDA tensor; ``energy`` the Potts energy of those labels.  Raises ``ValueError`` for
    malformed arguments and ``AttributeError`` for a boundary term that is not a two-parameter callable, before anything
    reaches the device.
    """
    device = -1
    if _on_device(costs):
        if str(costs.dtype) not in ("torch.float32", "torch.float64"):
            raise ValueError("costs must be float32 or float64, got {}".format(costs.dtype))
        if costs.dim() < 2 or costs.dim() > 5:
            raise ValueError("costs must have shape (K, *image shape) with a 1- to 4-D image")
        if costs.numel() and not bool((costs.isfinite() & (costs >= 0)).all()):
            raise ValueError("costs must be finite and >= 0")
        device = costs.device.index
    else:
        costs = _native_order(numpy.asarray(costs))
        if costs.dtype not in (numpy.float32, numpy.float64):
            raise ValueError("costs must be float32 or float64, got {}".format(costs.dtype))
        if costs.ndim < 2 or costs.ndim > 5:
            raise ValueError("costs must have shape (K, *image shape) with a 1- to 4-D image")
        if costs.size and not bool((numpy.isfinite(costs) & (costs >= 0)).all()):
            raise ValueError("costs must be finite and >= 0")
    K = int(costs.shape[0])
    shape = tuple(int(s) for s in costs.shape[1:])
    if not 2 <= K <= 255:
        raise ValueError("the number of labels K = costs.shape[0] must be 2..255, got {}".format(K))
    if min(shape) < 1:
        raise ValueError("the image must not be empty")
    if isinstance(max_cycles, bool) or not isinstance(max_cycles, (int, numpy.integer)) or max_cycles < 1:
        raise ValueError("max_cycles must be an integer >= 1")

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
        if markers is not None:
            if _on_device(markers) and _on_device(init):
                m, i = markers.long(), init.long()
            else:       # one side on the host: compare there
                m, i = (numpy.asarray(a.cpu() if _on_device(a) else a, dtype=numpy.int64) for a in (markers, init))
            if bool(((m > 0) & (i != m - 1)).any()):
                raise ValueError("init gives a marked voxel another label than its marker")

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
