"""Many small, independent cuts in one build and one solve: the slices of a stack segmented slice by slice, a cohort of
volumes, the patches of a tiled image (DESIGN.md §3.1).

``graph_from_voxels_batch`` takes B images of the same shape (1-D to 3-D) stacked along a leading batch axis, with one
set of markers and (optionally) one probability map per image, and returns a ``BatchGraph`` whose ``maxflow()`` gives
the B energies and whose ``get_mask()`` gives the B masks.  Each image is cut as if it were alone: its mask and energy
are those of ``graph_from_voxels`` on that image (the energy up to the order of the sums).  The images share one
lattice on the device, so a batch of small images fills the GPU where one of them would not.
"""
import math
import numbers

import numpy

from . import _warm_args
from .device import _KINDS, _as_u8
from .energy_voxel import _device_image, _device_products, _exact_as_float64, _native_order, _regional_products

# the lattice index of one handle is 32-bit: batch x voxels per image must stay below this
INDEX_LIMIT = 1 << 31

_LINEAR = {"difference_linear": False, "maximum_linear": True}     # name -> the normaliser is max |x|
_MAX_TERMS = ("maximum_linear", "maximum_exponential", "maximum_power")


def _is_cuda(a):
    return hasattr(a, "__cuda_array_interface__")


def _shape(a):
    return tuple(int(s) for s in a.shape)


def _markers(m):
    if m is None or _is_cuda(m):
        return _as_u8(m)
    m = numpy.asarray(m)
    return m.view(numpy.uint8) if m.dtype in (numpy.bool_, numpy.uint8) else (m != 0).view(numpy.uint8)


def _sigmas(sigma, batch):
    if sigma is None:
        return [0.0] * batch
    if isinstance(sigma, numbers.Real):
        return [float(sigma)] * batch
    s = [float(x) for x in sigma]
    if len(s) != batch:
        raise ValueError(f"sigma has {len(s)} entries for a batch of {batch} images")
    return s


def _host_image(image, boundary):
    """A host image as the native build reads it, and the linear normaliser of every image (NaN: reduced on the device).
    Integer images are normalised with numpy per image, in their own dtype, as ``energy_voxel`` does for one image."""
    image = _native_order(numpy.asarray(image))
    batch = image.shape[0]
    norms = [math.nan] * batch
    if boundary in _LINEAR and image.dtype.type not in (numpy.float32, numpy.float64):
        for b in range(batch):
            if _LINEAR[boundary]:
                norms[b] = float(numpy.abs(image[b]).max())
            else:
                norms[b] = float(abs(image[b].max() - image[b].min()))
    dev = _device_image(image)
    if boundary in _MAX_TERMS and dev.dtype != image.dtype:
        dev = numpy.abs(image).astype(numpy.float64)     # numpy.abs in the input dtype first (energy_voxel.py:558)
    return dev, norms


def _prob_arg(prob, alpha):
    """The probability map as the fused build reads it, and whether its products are float32, decided as
    ``energy_voxel.regional_probability_map`` decides them for one image: the map in native byte order, float32 products
    where numpy forms them in float32 (a float32 map times a Python float), float64 products where numpy forms them in
    float64 from a float64 map.  An integer or bool map whose products numpy forms exactly in float64 goes as a float64
    copy.
    Every other map has products the build cannot form, and is refused: float16 maps, a float32 map with a
    ``numpy.float64`` alpha (numpy rounds ``1 - p`` in float32, then multiplies in float64), and integer maps where
    ``1 - p`` wraps around in the map's dtype (an unsigned map holding 2 or more, a signed map within 1 of its minimum)."""
    if _is_cuda(prob):
        return prob, _device_products(prob, alpha, "a batch's")
    prob = _native_order(numpy.asarray(prob))
    mode = _regional_products(prob.dtype, alpha)
    if mode is not None:
        return prob, mode == "f32"
    if _exact_as_float64(prob, alpha):
        return prob.astype(numpy.float64), False
    raise ValueError(f"the products of a {prob.dtype} probability map with a {type(alpha).__name__} alpha cannot be "
                     f"formed exactly by a batch build: pass a float32 or float64 map (integer maps must keep 1 - p "
                     f"within their dtype)")


class BatchGraph:
    """The graph of a batch of images (``graph_from_voxels_batch``).

    Built with ``warm=True``, it takes the warm edits of ``GraphDouble`` (``add_seeds``, ``remove_seeds``,
    ``add_tweights_warm``, ``add_nweights_warm``, ``remove_nweights_warm`` and their dense forms), before or after a
    ``maxflow()``: the next ``maxflow()`` re-solves the batch from its residual state and returns the B energies of the
    edited images.  Node ids are flat C-order indices over the ``(B, ...image)`` shape, so image b's voxel p is
    ``b * N + p`` (N voxels per image); masks and dense arrays have the batch shape.  An n-link pair never joins two
    images: a listed pair across two images is refused like any pair of non-neighbours.  Without ``warm=True`` every
    warm edit raises ``RuntimeError``."""

    def __init__(self, native, batch, shape=None, warm=False):
        self._native = native
        self.batch = batch
        self.shape = tuple(shape) if shape is not None else None
        self._warm = warm

    def maxflow(self):
        """Solve every image; returns a float64 array of the B energies."""
        self._native.maxflow()
        return self._native.get_batch_energies()

    def get_mask(self):
        """uint8 array of shape (B, ...image): 1 where the voxel is not on the SINK side, as ``GraphDouble.get_mask``."""
        return self._native.get_mask()

    def stats(self):
        return self._native.stats()

    # The warm edits take the arguments of GraphDouble's (see there for their meaning), over the batch shape.  Without
    # warm=True the arguments go to the native handle as given, which refuses the call.
    def add_seeds(self, fg_ids=None, bg_ids=None):
        """``add_tweights(v, 65535, 0)`` for every foreground id, then ``add_tweights(v, 0, 65535)`` for every
        background id; ``fg_ids`` / ``bg_ids``: a boolean mask of the batch shape, a 1-D integer id array, or None."""
        self._seeds("add_seeds", fg_ids, bg_ids)

    def remove_seeds(self, fg_ids=None, bg_ids=None):
        """The inverse of ``add_seeds``: ``add_tweights(v, -65535, 0)`` / ``add_tweights(v, 0, -65535)``."""
        self._seeds("remove_seeds", fg_ids, bg_ids)

    def _seeds(self, native, fg, bg):
        if self._warm:
            fg, bg = _warm_args.seed_args(fg, bg, self.shape, self._n, ("fg_ids", "bg_ids"))
        getattr(self._native, native)(fg, bg)

    def add_tweights_warm(self, ids, src, snk):
        """``add_tweights(ids[k], src[k], snk[k])`` per entry in order; ``ids`` None is the dense form, one call per
        voxel with ``src`` / ``snk`` of the batch shape (or one entry per voxel).  Scalars broadcast."""
        if self._warm:
            ids, src, snk = _warm_args.tlink_args(ids, src, snk, self.shape, self._n)
        self._native.add_tweights_warm(ids, src, snk)

    def add_nweights_warm(self, i, j, cap, rev_cap):
        """``sum_edge(i[k], j[k], cap[k], rev_cap[k])`` per entry in order, on pairs of neighbours inside one image."""
        if self._warm:
            i, j, cap, rev_cap, _ = _warm_args.nlink_args(i, j, cap, rev_cap, self._n)
        self._native.add_nweights_warm(i, j, cap, rev_cap)

    def remove_nweights_warm(self, i, j, cap, rev_cap):
        """``sum_edge(i[k], j[k], -cap[k], -rev_cap[k])`` per entry in order (nonnegative decrements)."""
        if self._warm:
            i, j, cap, rev_cap, cuda = _warm_args.nlink_args(i, j, cap, rev_cap, self._n)
            if not cuda:        # the native grouping checks device decrements in the same pass
                _warm_args.check_amounts(((cap, "cap"), (rev_cap, "rev_cap")), _warm_args.DECREMENTS)
        self._native.remove_nweights_warm(i, j, cap, rev_cap)

    def add_nweights_dense_warm(self, axis, fwd, bwd):
        """The dense form of ``add_nweights_warm``: ``fwd`` / ``bwd`` have the batch shape and entry p holds the
        increments of p -> p + e_axis and back.  ``axis`` counts the axes of the batch shape: axis 0, the batch axis,
        joins no voxels and raises ``ValueError``; axis a >= 1 is the images' axis a - 1, whose last plane in every image
        is ignored."""
        if self._warm:
            axis, fwd, bwd, _ = self._dense_args(axis, fwd, bwd)
        self._native.add_nweights_dense_warm(axis, fwd, bwd)

    def remove_nweights_dense_warm(self, axis, fwd, bwd):
        """The dense form of ``remove_nweights_warm``, in the layout of ``add_nweights_dense_warm``."""
        if self._warm:
            lattice_axis, fwd, bwd, cuda = self._dense_args(axis, fwd, bwd)
            if not cuda:        # the entries that name a pair: all but the last plane of `axis` in every image
                cut = _warm_args.pair_entries(self.shape, int(axis))
                _warm_args.check_amounts(((fwd[cut], "fwd"), (bwd[cut], "bwd")), _warm_args.DECREMENTS)
            axis = lattice_axis
        self._native.remove_nweights_dense_warm(axis, fwd, bwd)

    @property
    def _n(self):
        return math.prod(self.shape)

    def _dense_args(self, axis, fwd, bwd):
        """The dense n-link arguments with the lattice axis of batch axis ``axis`` (the images' axes are the last of the
        lattice's three)."""
        if int(axis) == 0:
            raise ValueError("axis 0 is the batch axis: no n-link joins two images")
        axis, fwd, bwd, cuda = _warm_args.nlink_dense_args(axis, fwd, bwd, self.shape, "batch")
        return 3 - len(self.shape) + axis, fwd, bwd, cuda


def graph_from_voxels_batch(fg_markers, bg_markers, image, boundary, sigma=None, spacing=False, prob=None, alpha=None,
                            warm=False):
    """Build the graphs of B independent images in one fused build.

    The leading axis of every array is the batch; numpy arrays and CUDA arrays (``__cuda_array_interface__``, e.g. torch
    tensors) are both accepted, as in ``graph_from_device_arrays``.
    boundary : one of the eight ``energy_voxel.boundary_*`` names without the prefix (required)
    sigma : a float for every image, or one per image
    spacing, prob, alpha : as in ``graph_from_device_arrays``; shared by the whole batch
    warm : let the graph take warm edits (``BatchGraph.add_seeds`` ...) and re-solve from its residual state, so that a
        correction to a few images does not rebuild the batch.  Off by default, where the warm edits raise.
    """
    if boundary not in _KINDS:
        raise ValueError(f"a batch needs one of the boundary terms {sorted(_KINDS)}, got {boundary!r}")
    shape = _shape(image)
    if len(shape) < 2:
        raise ValueError("the leading axis of the arrays is the batch: image needs at least two axes")
    batch, image_shape = shape[0], shape[1:]
    if len(image_shape) > 3:
        raise ValueError("batch images are 1-D to 3-D")
    for name, a in (("fg_markers", fg_markers), ("bg_markers", bg_markers), ("prob", prob)):
        if a is not None and _shape(a) != shape:
            raise ValueError(f"{name} has shape {_shape(a)}, image has {shape}")
    if batch * math.prod(image_shape) >= INDEX_LIMIT:
        raise ValueError(f"{batch} images of {math.prod(image_shape)} voxels reach the 2^31 voxel index limit of one batch")
    sigmas = _sigmas(sigma, batch)
    sp = None
    if spacing:
        sp = [float(s) for s in spacing]
        if len(sp) < len(image_shape):
            raise ValueError("spacing has fewer entries than the images have dimensions")
    if _is_cuda(image):
        norms = [math.nan] * batch
    else:
        image, norms = _host_image(image, boundary)

    alpha = 0.0 if alpha is None else alpha
    compute_f32 = False
    if prob is not None:
        prob, compute_f32 = _prob_arg(prob, alpha)     # on alpha as given: its type decides the products' dtype
    alpha = float(alpha)

    from .. import _lib   # raises ImportError loudly when the extension is not built
    native = _lib.Graph.batch(list(image_shape), batch, -1)
    if warm:        # before the build: an eagerly built batch records its residual source capacities at the first solve
        native.set_option(_lib._mgc.OPT_WARM, 1)
    native.build_voxel_batch(prob, alpha, compute_f32, _KINDS[boundary], image, sigmas, sp, norms, _markers(fg_markers),
                             _markers(bg_markers))
    return BatchGraph(native, batch, shape, warm)
