"""Argument parsing of the warm edit calls (``add_seeds``, ``remove_seeds``, ``add_tweights_warm``, the list and dense
n-link edits), shared by every front-end that takes them.

The lattice front-ends -- a lattice graph (maxflow.GraphDouble), a batch of images (batch.BatchGraph) and one rank's
z-slab (distributed.SlabSolver) -- parse each kind of edit with one function here: ``seed_args``,
``tlink_args``, ``nlink_args`` and ``nlink_dense_args``.  They keep only what is their own: staging before a solve,
the batch axis, the slab's ownership.  The sparse-id front-ends (sparse.SparseGraphDouble,
labels_batch.LabelBatchGraph) parse through the sparse-id functions of sparse.py, which build on ``node_ids``,
``weights`` and ``nlink_calls`` here.

A result stays in the memory space of its argument: a CUDA tensor gives a CUDA tensor, which the native folds read in
place, anything else (numpy arrays, lists, scalars, CPU tensors) a numpy array.  The checks of parsed weights
(``check_finite``, ``check_amounts``) take both; on a CUDA tensor each verdict is one read-back."""
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


def seed_args(fg, bg, shape, n, names=("fg", "bg"), mixed=False):
    """The node ids of an add_seeds / remove_seeds call (``node_ids``; None stays None).  fg and bg must share one
    memory space unless ``mixed``: a graph that stages the seeds on the host takes either."""
    if not mixed:
        one_space("{} and {} must both be host or both be device arrays".format(*names), fg, bg)
    return tuple(None if x is None else node_ids(x, shape, n, what) for x, what in zip((fg, bg), names))


def tlink_args(ids, src, snk, shape, n, names=("ids", "src", "snk")):
    """The calls of an add_tweights_warm edit: the node ids (``node_ids``; None for the dense form, one call per node in
    C order) and the weights as C-contiguous float64 arrays of one entry per call.  Scalars broadcast; a dense form's
    weights have ``shape`` or one entry per node.  All three arguments share one memory space."""
    cuda = one_space("{}, {} and {} must all be host or all be device arrays".format(*names), ids, src, snk)
    ids = None if ids is None else node_ids(ids, shape, n, names[0])
    m, dense = (n, tuple(shape)) if ids is None else (ids.shape[0], None)
    return ids, weights(src, m, names[1], dense, cuda), weights(snk, m, names[2], dense, cuda)


def nlink_args(i, j, cap, rev_cap, n):
    """The calls of a list-form n-link edit on a graph of n nodes as ``nlink_calls`` gives them, from id arguments that
    ``pair_ids`` parses; and whether they are on the device.  All four arguments share one memory space."""
    cuda = one_space("i, j, cap and rev_cap must all be host or all be device arrays", i, j, cap, rev_cap)
    return nlink_calls(pair_ids(i, n, "i"), pair_ids(j, n, "j"), cap, rev_cap, cuda) + (cuda,)


def nlink_dense_args(axis, fwd, bwd, shape, what="graph"):
    """The arguments of a dense n-link edit: the axis, checked against ``shape`` (that of a ``what``), and fwd / bwd as
    float64 arrays of ``shape``, strides kept; and whether they are on the device.  Both arrays share one memory space."""
    axis, shape = int(axis), tuple(shape)
    if not 0 <= axis < len(shape):
        raise ValueError("axis {} is out of range for a {} of shape {}".format(axis, what, shape))
    cuda = one_space("fwd and bwd must both be host or both be device arrays", fwd, bwd)
    fwd, bwd = real(fwd, "fwd"), real(bwd, "bwd")
    for a, name in ((fwd, "fwd"), (bwd, "bwd")):
        if tuple(a.shape) != shape:
            raise ValueError("{} of shape {} does not match the {} shape {}".format(name, tuple(a.shape), what, shape))
    return axis, fwd, bwd, cuda


def pair_entries(shape, axis):
    """The entries of a dense n-link array of ``shape`` that name a pair: the last plane of ``axis`` names none."""
    return tuple(slice(0, s - 1) if d == axis else slice(None) for d, s in enumerate(shape))


def lattice_axes(i, j, shape):
    """The axis that joins each pair (i[k], j[k]) of C-order node ids on a lattice of ``shape``, or -1 where the two are
    not lattice neighbours; int64 numpy arrays or CUDA tensors, with no read-back."""
    lo, d = (numpy.minimum(i, j) if isinstance(i, numpy.ndarray) else i.minimum(j)), abs(i - j)
    axes = d * 0 - 1
    for axis in range(len(shape)):
        stride = math.prod(shape[axis + 1:])
        # at most one axis joins a pair: of two axes with one stride the later has size 1, and a size-1 axis joins none
        axes = axes + ((d == stride) & ((lo // stride) % shape[axis] < shape[axis] - 1)) * (axis + 1)
    return axes


def check_finite(w, what):
    """Weights on the host or the device: no NaN or infinite value."""
    if not bool((w.isfinite() if on_device(w) else numpy.isfinite(w)).all()):
        raise ValueError("{} holds NaN or infinite values".format(what))


# what check_amounts says about a negative amount: raised by an added n-link, or by a removed one
ONLY_RAISES = "a warm n-link edit only raises capacities"
DECREMENTS = "n-link decrements are nonnegative amounts"


def check_amounts(named, why):
    """N-link amounts ``[(weights, name), ...]`` on the host or the device: finite and nonnegative, argument by argument;
    ``why`` ends the message about a negative value."""
    for w, what in named:
        check_finite(w, what)
        if bool(((w if on_device(w) else numpy.asarray(w)) < 0).any()):
            raise ValueError("{} holds negative values: {}".format(what, why))
