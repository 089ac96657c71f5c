"""Host-side mirror of ``medpy.graphcut.energy_voxel`` (reference: medpy/graphcut/energy_voxel.py).

The nine energy-term functions keep the reference's names, their ``(graph, term_args)`` two-parameter
signature (``graph_from_voxels`` checks it with ``inspect.getfullargspec``, generate.py:135-146) and the
tuple layouts of ``term_args``; they stay pure Python so that check passes.  Instead of producing one weight
array per axis and calling ``graph.set_nweight`` per edge (energy_voxel.py:637-664), each hands the image
and its parameters to the graph, which evaluates the stencil on the GPU in float64:

    w(p, q) = g(|I_p - I_q|)            difference terms   (energy_voxel.py:561-608)
    w(p, q) = g(max(|I_p|, |I_q|))      maximum terms      (energy_voxel.py:519-558)

    linear       g(x) = 1 - x / M, exact zeros -> DBL_MIN                      (:101-114, :176-189)
    exponential  g(x) = exp(-(x^2) / sigma^2), <= 0 -> DBL_MIN                 (:226-236, :290-300)
    division     g(x) = 1 / (x / sigma + 1), <= 0 -> DBL_MIN                   (:337-345, :399-407)
    power        g(x) = (1 / (x + 1))^sigma, <= 0 -> DBL_MIN                   (:444-452, :506-514)

followed by ``/ spacing[axis]`` when a spacing is given (:657-658).  Reference quirks are kept:
``boundary_maximum_division`` evaluates the *difference* form (:347), the linear normaliser M is formed in the
image's own dtype (:99, :174), and the two linear terms take a 2-tuple, the others a 3-tuple.
"""
import math

import numpy

__all__ = [
    "regional_probability_map",
    "boundary_maximum_linear", "boundary_difference_linear",
    "boundary_maximum_exponential", "boundary_difference_exponential",
    "boundary_maximum_division", "boundary_difference_division",
    "boundary_maximum_power", "boundary_difference_power",
]

# codes of include/medpy_b200_graphcut.h (MGC_BOUNDARY_*)
_DIFF_LINEAR, _DIFF_EXP, _DIFF_DIV, _DIFF_POW, _MAX_LINEAR, _MAX_EXP, _MAX_DIV, _MAX_POW = range(8)

_DEVICE_DTYPES = (numpy.float32, numpy.float64, numpy.uint8, numpy.int16, numpy.int32)


def _native_order(a):
    """Arrays in non-native byte order ('>f4', '>i2': FITS / NIfTI readers) are converted once; the kernels read native
    values only (the reference goes through numpy, which handles the byte order)."""
    if not a.dtype.isnative:
        return a.astype(a.dtype.newbyteorder("="))
    return a


def _device_image(image):
    """Images whose dtype the kernels read natively pass through untouched (any strides); the rest are widened
    to float64 on the host, which is what the reference does to every image anyway (energy_voxel.py:634)."""
    image = _native_order(numpy.asarray(image))
    if image.dtype == numpy.bool_:
        return image.view(numpy.uint8)
    if image.dtype.type in _DEVICE_DTYPES and all(s > 0 for s in image.strides):
        return image
    if image.dtype.type in _DEVICE_DTYPES:
        return numpy.ascontiguousarray(image)
    return image.astype(numpy.float64)


def _spacing_arg(spacing, ndim):
    if not spacing:  # False / None / empty: no distance weighting (energy_voxel.py:657)
        return None
    sp = [float(s) for s in spacing]
    if len(sp) < ndim:
        raise IndexError("spacing has fewer entries than the image has dimensions")
    return sp


def _boundary(graph, kind, image, sigma, spacing):
    image = _native_order(numpy.asarray(image))
    # linear normaliser M, formed in the image's own dtype (energy_voxel.py:99, :174).  float32/float64 images:
    # NaN asks the device to do the min/max reduction (kernel K0, same dtype arithmetic); integer images:
    # numpy on the host so narrow-integer wrap-around matches the reference exactly.
    norm = float("nan")
    if image.dtype.type not in (numpy.float32, numpy.float64):
        if kind == _MAX_LINEAR:
            norm = float(numpy.abs(image).max())
        elif kind == _DIFF_LINEAR:
            norm = float(abs(image.max() - image.min()))
    if kind in (_DIFF_EXP, _MAX_EXP) and sigma is not None:
        math.pow(sigma, 2)      # the reference's sigma^2 (energy_voxel.py:232, :296): OverflowError for |sigma| > ~1.3e154
    dev = _device_image(image)
    if kind in (_MAX_LINEAR, _MAX_EXP, _MAX_POW) and dev.dtype != image.dtype:
        dev = numpy.abs(image).astype(numpy.float64)  # numpy.abs in the input dtype first (energy_voxel.py:558)
    graph._add_boundary(kind, dev, 0.0 if sigma is None else float(sigma), _spacing_arg(spacing, image.ndim), norm)


def _regional_products(dtype, alpha):
    """How numpy forms the two products ``p * alpha`` and ``(1 - p) * alpha`` of a map of this dtype: ``"f32"`` (a
    float32 map, both in float32, as a float32 map times a Python float), ``"f64"`` (a float64 map, both in float64), or
    None for every other mix, whose products only numpy itself forms exactly (a float32 map times a ``numpy.float64``
    rounds ``1 - p`` in float32 and multiplies in float64; integer maps form ``1 - p`` in their own dtype)."""
    if dtype is None:
        return None
    z = numpy.zeros(0, dtype)
    src, snk = (z * alpha).dtype, ((1 - z) * alpha).dtype      # numpy-2 weak scalars
    if z.dtype == numpy.float32 and src == numpy.float32 and snk == numpy.float32:
        return "f32"
    if z.dtype == numpy.float64 and src == numpy.float64 and snk == numpy.float64:
        return "f64"
    return None


def _device_products(prob, alpha, whose="the"):
    """Whether the products of a device probability map (torch tensor, or any array with a numpy-like ``dtype``) are
    float32, decided as ``_regional_products`` decides them for the host map of the same dtype; ``ValueError`` where
    they are neither pure float32 nor pure float64, since a device map has no dense fallback."""
    try:
        dtype = numpy.dtype(str(prob.dtype).rsplit(".", 1)[-1])      # torch.float32 -> float32
    except TypeError:
        dtype = None
    mode = _regional_products(dtype, 0.0 if alpha is None else alpha)
    if mode is None:
        raise ValueError(f"{whose} probability map must be float32 or float64 and give products of its own dtype with "
                         f"alpha, got a {prob.dtype} map with a {type(alpha).__name__} alpha")
    return mode == "f32"


def _exact_as_float64(prob, alpha):
    """True when an integer or bool map's products are the float64 products of its float64 copy: numpy forms both in
    float64, ``1 - p`` does not wrap around in the map's dtype, and every p and 1 - p is an integer a double holds
    exactly.  A bool map always qualifies when numpy's products are float64: ``1 - p`` is formed in int64 and is 0 or 1."""
    if prob.dtype.kind not in "biu" or (prob[:0] * alpha).dtype != numpy.float64 or ((1 - prob[:0]) * alpha).dtype != numpy.float64:
        return False
    if prob.size == 0 or prob.dtype.kind == "b":
        return True
    lo, hi = int(prob.min()), int(prob.max())
    info = numpy.iinfo(prob.dtype)
    return 1 - hi >= info.min and 1 - lo <= info.max and -2 ** 53 < lo and hi <= 2 ** 53


def regional_probability_map(graph, term_args):
    """Regional term based on a probability atlas (reference: energy_voxel.py:33-65).

    ``term_args = (probability_map, alpha)``; every voxel gets the t-weights
    ``(p * alpha, (1 - p) * alpha)`` (source = foreground, sink = background) through
    ``graph.set_tweights_all`` semantics, i.e. ``add_tweights`` per voxel in node order."""
    (probability_map, alpha) = term_args
    probability_map = _native_order(numpy.asarray(probability_map))
    mode = _regional_products(probability_map.dtype, alpha)
    if mode is not None:
        graph._add_regional_probability(probability_map, float(alpha), mode == "f32")
    else:
        # unusual dtype mixes: form the products with numpy exactly as the reference does, upload densely
        graph.set_tweights_dense((probability_map * alpha).astype(numpy.float64).ravel(),
                                 ((1 - probability_map) * alpha).astype(numpy.float64).ravel())


def boundary_maximum_linear(graph, term_args):
    """Boundary term on the gradient image, linear (reference: energy_voxel.py:68-116).
    ``term_args = (gradient_image, spacing)``."""
    (gradient_image, spacing) = term_args
    _boundary(graph, _MAX_LINEAR, gradient_image, None, spacing)


def boundary_difference_linear(graph, term_args):
    """Boundary term on intensity differences, linear (reference: energy_voxel.py:119-191).
    ``term_args = (original_image, spacing)``."""
    (original_image, spacing) = term_args
    _boundary(graph, _DIFF_LINEAR, original_image, None, spacing)


def boundary_maximum_exponential(graph, term_args):
    """Boundary term on the gradient image, exponential (reference: energy_voxel.py:194-238).
    ``term_args = (gradient_image, sigma, spacing)``."""
    (gradient_image, sigma, spacing) = term_args
    _boundary(graph, _MAX_EXP, gradient_image, sigma, spacing)


def boundary_difference_exponential(graph, term_args):
    """Boundary term on intensity differences, exponential (reference: energy_voxel.py:241-302).
    ``term_args = (original_image, sigma, spacing)``."""
    (original_image, sigma, spacing) = term_args
    _boundary(graph, _DIFF_EXP, original_image, sigma, spacing)


def boundary_maximum_division(graph, term_args):
    """Boundary term on the gradient image, division (reference: energy_voxel.py:305-349; the reference
    evaluates the *difference* skeleton here, :347, and so do we).  ``term_args = (gradient_image, sigma, spacing)``."""
    (gradient_image, sigma, spacing) = term_args
    _boundary(graph, _MAX_DIV, gradient_image, sigma, spacing)


def boundary_difference_division(graph, term_args):
    """Boundary term on intensity differences, division (reference: energy_voxel.py:352-409).
    ``term_args = (original_image, sigma, spacing)``."""
    (original_image, sigma, spacing) = term_args
    _boundary(graph, _DIFF_DIV, original_image, sigma, spacing)


def boundary_maximum_power(graph, term_args):
    """Boundary term on the gradient image, power (reference: energy_voxel.py:412-454).
    ``term_args = (gradient_image, sigma, spacing)``."""
    (gradient_image, sigma, spacing) = term_args
    _boundary(graph, _MAX_POW, gradient_image, sigma, spacing)


def boundary_difference_power(graph, term_args):
    """Boundary term on intensity differences, power (reference: energy_voxel.py:457-516).
    ``term_args = (original_image, sigma, spacing)``."""
    (original_image, sigma, spacing) = term_args
    _boundary(graph, _DIFF_POW, original_image, sigma, spacing)
