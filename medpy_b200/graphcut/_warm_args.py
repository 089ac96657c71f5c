"""Argument parsing of the warm edit calls, shared by the lattice graph (maxflow.py) and the general sparse graph
(sparse.py).  A result stays in the memory space of its argument: a CUDA tensor gives a CUDA tensor, which the lattice's
native folds read in place, anything else (numpy arrays, lists, scalars, CPU tensors) a numpy array.  Broadcasts go to
the device when the caller asks for it; which memory spaces one call may mix is the caller's decision."""
import math

import numpy


def on_device(x):
    return hasattr(x, "__cuda_array_interface__")


def one_space(message, *args):
    """Whether the arguments of one warm call are on the device, for native folds that take their arrays all on the host
    or all on the device: a mix raises ``ValueError(message)``; host scalars (and None) go with either."""
    cuda = any(on_device(x) for x in args)
    if cuda and any(not on_device(x) and numpy.ndim(x) for x in args):
        raise ValueError(message)
    return cuda


def _array(x):
    """``x`` as a torch tensor if it is a CUDA array, else as a numpy array; and numpy's kind of its dtype: "b" bool,
    "i" / "u" integer, "f" float, "c" complex, ..."""
    if not on_device(x):
        a = numpy.asarray(x)
        return a, a.dtype.kind
    import torch
    t = torch.as_tensor(x)
    return t, "b" if t.dtype == torch.bool else "c" if t.dtype.is_complex else "f" if t.dtype.is_floating_point else "i"


def _cast(a, dtype, contiguous):
    """``a`` as ``dtype`` ("int64" or "float64") in its memory space; C-contiguous when asked, else with its strides
    where no copy is needed."""
    if isinstance(a, numpy.ndarray):
        return a.astype(dtype, order="C" if contiguous else "K", copy=False)
    import torch
    a = a.to(getattr(torch, dtype))
    return a.contiguous() if contiguous else a


def _broadcast(a, m, device):
    """A 0-d or m-entry 1-D array as m C-contiguous entries, on the device when ``device``."""
    if device and isinstance(a, numpy.ndarray):
        import torch
        a = torch.as_tensor(a, device="cuda")
    if isinstance(a, numpy.ndarray):
        return numpy.ascontiguousarray(numpy.broadcast_to(a, (m,)))
    return a.expand(m).contiguous()


def check_ids(ids, n):
    """Node ids within 0..n-1, as GCGraph.set_source_nodes checks them (graph.py:334-339); returns ``ids``."""
    if math.prod(ids.shape):
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= n:
            raise ValueError("Invalid node id of {} or {}. Valid values are 0 to {}.".format(hi, lo, n - 1))
    return ids


def node_ids(x, shape, n, what):
    """The node ids of one argument, int64 and range-checked: a boolean mask of ``shape`` (any strides; ids in logical C
    order, like generate.py:169-172) or a 1-D integer id array."""
    a, kind = _array(x)
    if kind == "b":
        if tuple(a.shape) != tuple(shape):
            raise ValueError("{} mask of shape {} does not match the graph's shape {}".format(
                what, tuple(a.shape), tuple(shape)))
        ids = a.reshape(-1).nonzero()
        return ids[0] if isinstance(a, numpy.ndarray) else ids.reshape(-1)
    if a.ndim != 1 or not (kind in "iu" or a.shape[0] == 0):
        raise ValueError("{} must be a boolean mask of the graph's shape or a 1-D integer id array".format(what))
    return check_ids(_cast(a, "int64", True), n)


def pair_ids(x, n, what):
    """One id argument of an n-link call, int64 and range-checked: an integer (a 0-d array) or a 1-D integer array."""
    a, kind = _array(x)
    if a.ndim > 1 or not (kind in "iu" or a.shape == (0,)):
        raise ValueError("{} must be a 1-D integer node id array or an integer".format(what))
    return check_ids(_cast(a, "int64", True), n)


def real(w, what):
    """One weight argument as float64, shape and strides kept; bool, complex and non-numeric dtypes are refused."""
    a, kind = _array(w)
    if kind not in "iuf":
        raise ValueError("{} must hold real numbers".format(what))
    return _cast(a, "float64", False)


def weights(w, m, what, shape=None, device=False):
    """One weight argument as m C-contiguous float64 values: a scalar broadcasts (on the device when ``device``); an array
    has m entries or, for a dense form, ``shape`` (read in logical C order)."""
    a = real(w, what)
    if a.ndim == 0:
        return _broadcast(a, m, device)
    if tuple(a.shape) != (m,) and tuple(a.shape) != shape:
        if shape is not None:
            raise ValueError("{} of shape {} does not match the graph's shape {} or its {} nodes".format(
                what, tuple(a.shape), shape, m))
        raise ValueError("{} has shape {}, expected {} entries like the node ids".format(what, tuple(a.shape), m))
    return _cast(a.reshape(-1), "float64", True)


def nlink_calls(i, j, cap, rev_cap, device=False):
    """The sum_edge calls ``(i[k], j[k], cap[k], rev_cap[k])`` of an n-link edit as four C-contiguous 1-D arrays of one
    length m (on the device when ``device``), from parsed ids ``i`` / ``j`` (0-d or 1-D) and the weight arguments.  1-D
    ids must agree in length, which is m; a 0-d id repeats.  A 0-d pair takes the length of the 1-D weights, so
    (5, 6, [1.0, 2.0], 0.0) is two calls on one pair."""
    sizes = {x.shape[0] for x in (i, j) if x.ndim}
    if len(sizes) > 1:
        raise ValueError("i and j differ in length")
    wsizes = {numpy.shape(w)[0] for w in (cap, rev_cap) if numpy.ndim(w) == 1}
    m = sizes.pop() if sizes else (wsizes.pop() if len(wsizes) == 1 else 1)
    return (_broadcast(i, m, device), _broadcast(j, m, device),
            weights(cap, m, "cap", device=device), weights(rev_cap, m, "rev_cap", device=device))


def check_finite(w, what):
    """Host weights: no NaN or infinite value."""
    if not numpy.isfinite(w).all():
        raise ValueError("{} holds NaN or infinite values".format(what))


# what check_amounts says about a negative amount: raised by an added n-link, or by a removed one
ONLY_RAISES = "a warm n-link edit only raises capacities"
DECREMENTS = "n-link decrements are nonnegative amounts"


def check_amounts(named, why):
    """Host n-link amounts ``[(weights, name), ...]``: finite and nonnegative, argument by argument; ``why`` ends the
    message about a negative value."""
    for w, what in named:
        check_finite(w, what)
        if (numpy.asarray(w) < 0).any():
            raise ValueError("{} holds negative values: {}".format(what, why))
