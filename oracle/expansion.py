"""oracle/expansion.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the alpha-expansion segmentation (``medpy_b200.graphcut.expansion_from_voxels``, DESIGN.md §11):
every move graph is built in numpy following the case table of DESIGN.md §11 in its stated summation order, laid out
as ``energy_terms.build_problem`` lays out a graph (flat ``tr`` / ``flow_const`` / per-axis ``wf`` / ``wb``), and cut
by ``solvers.solve_port`` (the BK restatement).  BK's sink set is the minimal one, as the device solver's is, so a
chain of moves is reproducible voxel for voxel.

Only tests/ and tools/ may import this module; the product package never does.
"""
import math

import numpy

from . import energy_terms, solvers

MAX = float(energy_terms.MAX_TWEIGHT)   # GCGraph.MAX: the soft-hard seed


def data_costs(costs, markers=None):
    """D[k, p]: cost plane k widened to float64, + 65535.0 for every k != m-1 where markers[p] = m > 0 (flat over p)."""
    costs = numpy.asarray(costs)
    K = costs.shape[0]
    D = costs.reshape(K, -1).astype(numpy.float64)
    if markers is not None:
        m = numpy.asarray(markers).ravel().astype(numpy.int64)
        for k in range(K):
            D[k, (m > 0) & (m - 1 != k)] += MAX
    return D


def pair_weights(shape, boundary=None):
    """Per-axis pair weights of extent D_d - 1 along axis d: ``energy_terms.boundary_weights`` for a boundary term given
    as (kind, image, sigma, spacing), zeros without one."""
    if boundary is None:
        out = []
        for d in range(len(shape)):
            s = list(shape)
            s[d] -= 1
            out.append(numpy.zeros(s))
        return out
    kind, image, sigma, spacing = boundary
    return energy_terms.boundary_weights(kind, image, sigma, spacing)


def _axis_slices(ndim, d):
    lo = [slice(None)] * ndim
    hi = [slice(None)] * ndim
    lo[d] = slice(0, -1)
    hi[d] = slice(1, None)
    return tuple(lo), tuple(hi)


def energy(D, w, labels):
    """E(l) = sum_p D_p(l_p) + sum_pairs w_pq [l_p != l_q], summed exactly (math.fsum) then rounded once."""
    lab = numpy.asarray(labels)
    flat = lab.ravel().astype(numpy.int64)
    terms = [D[flat, numpy.arange(flat.size)]]
    for d, wd in enumerate(w):
        lo, hi = _axis_slices(lab.ndim, d)
        terms.append(wd[lab[lo] != lab[hi]])
    return math.fsum(numpy.concatenate([t.ravel() for t in terms]))


def move_problem(D, w, labels, alpha):
    """The graph of the move for ``alpha`` over ``labels`` as a ``build_problem`` dict (SINK = switch to alpha):
    src_p = D_p(alpha); snk_p = D_p(l_p) + the t-link contributions, added axis by axis, within an axis first the pair
    where p is the lower end; then add_tweights(p, src_p, snk_p) on tr = 0 in node order."""
    lab = numpy.asarray(labels).astype(numpy.int64)
    shape = lab.shape
    n = lab.size
    flat = lab.ravel()
    idx = numpy.arange(n)
    src = D[alpha, idx].copy()
    snk = D[flat, idx].copy()
    wf, wb = [], []
    for d, wd in enumerate(w):
        lo, hi = _axis_slices(lab.ndim, d)
        lp, lq = lab[lo], lab[hi]
        cl = numpy.zeros(shape)
        cu = numpy.zeros(shape)
        f = numpy.zeros(shape)
        b = numpy.zeros(shape)
        cl[lo] = numpy.where((lp != alpha) & (lq != lp), wd, 0.0)    # p non-alpha and the pair split: p pays
        cu[hi] = numpy.where((lq != alpha) & (lp == alpha), wd, 0.0)  # only q non-alpha: q pays
        f[lo] = numpy.where((lp == lq) & (lp != alpha), wd, 0.0)      # arc p -> q
        b[lo] = numpy.where((lp != alpha) & (lq != alpha), wd, 0.0)   # arc q -> p (entry p, as build_problem's wb)
        snk = snk + cl.ravel()
        snk = snk + cu.ravel()
        wf.append(f.ravel())
        wb.append(b.ravel())
    tr = numpy.zeros(n)
    flow = energy_terms.add_tweights_pass(tr, 0.0, src, snk)
    return dict(shape=shape, wf=wf, wb=wb, tr=tr, flow_const=flow)


def move(D, w, labels, alpha):
    """One move: (new labels, switched voxels, cut value = flow_const + max-flow)."""
    lab = numpy.asarray(labels)
    prob = move_problem(D, w, lab, alpha)
    cut, mask, _ = solvers.solve_port(prob)
    switch = (mask == 0) & (lab != alpha)
    out = lab.copy()
    out[switch] = alpha
    return out, int(switch.sum()), cut


def initial_labels(D, shape, init=None):
    """``init`` where given, else argmin_k D_p(k) with ties to the lowest k."""
    if init is not None:
        return numpy.asarray(init).astype(numpy.uint8).reshape(shape)
    return numpy.argmin(D, axis=0).astype(numpy.uint8).reshape(shape)


def expansion(costs, boundary=None, markers=None, init=None, max_cycles=20):
    """The whole loop: cycles alpha = 0 .. K-1 until a cycle switches nothing or ``max_cycles`` cycles ran.
    Returns dict(labels uint8, energy, switched per move, cuts per move, moves, cycles, converged)."""
    costs = numpy.asarray(costs)
    K = costs.shape[0]
    shape = costs.shape[1:]
    D = data_costs(costs, markers)
    w = pair_weights(shape, boundary)
    lab = initial_labels(D, shape, init)
    switched, cuts = [], []
    cycles = 0
    converged = False
    for _ in range(max_cycles):
        changed = 0
        for alpha in range(K):
            lab, s, cut = move(D, w, lab, alpha)
            switched.append(s)
            cuts.append(cut)
            changed += s
        cycles += 1
        if changed == 0:
            converged = True
            break
    return dict(labels=lab, energy=energy(D, w, lab), switched=switched, cuts=cuts, moves=len(switched), cycles=cycles,
                converged=converged)
