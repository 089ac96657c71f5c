"""oracle/region_expansion.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the region alpha-expansion (``medpy_b200.graphcut.expansion_from_labels``, DESIGN.md §11 "Region
graphs"): the data costs (bincount sums and marker seeds), every move problem by the per-arc rules of §11 in their
stated summation order, the loop, and the energy.  Each move is cut by ``solvers.solve_sparse_port`` (the BK
restatement for general graphs), whose sink set is BK's minimal one, as the device solver's is, so a chain of moves is
reproducible region for region.

A region graph is given as its pairs: int arrays ``i < j`` in strictly ascending (i, j) order and one float64 weight
``w`` per pair.  Only tests/ and tools/ may import this module; the product package never does.
"""
import math

import numpy

from . import solvers
from .expansion import MAX


def data_costs(label_image, costs=None, region_costs=None, markers=None):
    """D[k, r]: numpy.bincount of costs[k] over the regions (float64), or region_costs widened to float64; then for every
    marker value m > 0 in ascending order, + MAX for every k != m-1 on the regions holding a voxel marked m."""
    lab = numpy.asarray(label_image).ravel().astype(numpy.int64) - 1
    R = int(lab.max()) + 1
    if region_costs is not None:
        D = numpy.array(region_costs, dtype=numpy.float64)
    else:
        costs = numpy.asarray(costs)
        D = numpy.stack([numpy.bincount(lab, weights=costs[k].ravel().astype(numpy.float64), minlength=R)
                         for k in range(costs.shape[0])])
    if markers is not None:
        m = numpy.asarray(markers).ravel().astype(numpy.int64)
        K = D.shape[0]
        for v in numpy.unique(m):
            if v == 0:
                continue
            inside = numpy.zeros(R, bool)
            inside[numpy.unique(lab[m == v])] = True
            for k in range(K):
                if k != v - 1:
                    D[k, inside] += MAX
    return D


def _arcs(i, j):
    """Both arcs of every pair, sorted by (tail, head): the CSR order of the device, each row in ascending neighbour id.
    Returns (tail, head, pair index)."""
    i = numpy.asarray(i, numpy.int64)
    j = numpy.asarray(j, numpy.int64)
    tail = numpy.concatenate([i, j])
    head = numpy.concatenate([j, i])
    pair = numpy.concatenate([numpy.arange(i.size), numpy.arange(i.size)])
    order = numpy.lexsort((head, tail))
    return tail[order], head[order], pair[order]


def arc_rules(a, b, u, v, alpha):
    """The per-arc rules of §11 for node u with label a and its arc to v with label b: (u's sink link gains w,
    cap(u->v) = w), as booleans (numpy arrays or scalars)."""
    free = a != alpha
    return (free & ((b == alpha) | ((b != a) & (u < v))),
            free & (b != alpha) & ((a == b) | (u > v)))


def move_problem(D, i, j, w, labels, alpha):
    """The move for ``alpha`` over region ``labels`` (SINK = switch to alpha): (sum_edge calls i, j, cap i->j,
    cap j->i; the add_tweights call (nodes, src, snk)).  src_u = D_u(alpha); snk_u = D_u(l_u) + w of every arc whose rule
    says so, added in the row's order (ascending neighbour id)."""
    lab = numpy.asarray(labels).astype(numpy.int64)
    R = lab.size
    idx = numpy.arange(R)
    w = numpy.asarray(w, numpy.float64)
    src = D[alpha, idx].copy()
    snk = D[lab, idx].copy()
    tail, head, pair = _arcs(i, j)
    to_snk, arc = arc_rules(lab[tail], lab[head], tail, head, alpha)
    numpy.add.at(snk, tail[to_snk], w[pair[to_snk]])      # unbuffered, in index order: per node in row order
    cap = numpy.where(arc, w[pair], 0.0)
    fwd = numpy.zeros(len(w))
    bwd = numpy.zeros(len(w))
    lo = tail < head
    fwd[pair[lo]] = cap[lo]
    bwd[pair[~lo]] = cap[~lo]
    return (numpy.asarray(i), numpy.asarray(j), fwd, bwd), (idx, src, snk)


def move(D, i, j, w, labels, alpha):
    """One move: (new labels, switched regions, cut value = add_tweights constant + max-flow)."""
    lab = numpy.asarray(labels)
    edges, tw = move_problem(D, i, j, w, lab, alpha)
    cut, mask, _ = solvers.solve_sparse_port(lab.size, *edges, [tw])
    switch = (mask == 0) & (lab != alpha)
    out = lab.copy()
    out[switch] = alpha
    return out, int(switch.sum()), cut


def energy(D, i, j, w, labels):
    """E(l) = sum_r D_r(l_r) + sum_pairs w_rs [l_r != l_s], summed exactly (math.fsum) then rounded once."""
    lab = numpy.asarray(labels).astype(numpy.int64)
    w = numpy.asarray(w, numpy.float64)
    cut = lab[numpy.asarray(i, numpy.int64)] != lab[numpy.asarray(j, numpy.int64)]
    return math.fsum(numpy.concatenate([D[lab, numpy.arange(lab.size)], w[cut]]))


def expansion(D, i, j, w, init=None, max_cycles=20):
    """The whole loop from ``init`` or argmin_k D (ties to the lowest k): cycles alpha = 0 .. K-1 until a cycle switches
    nothing or ``max_cycles`` cycles ran.  Returns dict(labels uint8, energy, switched per move, cuts per move, moves,
    cycles, converged)."""
    K = D.shape[0]
    lab = (numpy.argmin(D, axis=0) if init is None else numpy.asarray(init)).astype(numpy.uint8)
    switched, cuts = [], []
    cycles = 0
    converged = False
    for _ in range(max_cycles):
        changed = 0
        for alpha in range(K):
            lab, s, cut = move(D, i, j, w, lab, alpha)
            switched.append(s)
            cuts.append(cut)
            changed += s
        cycles += 1
        if changed == 0:
            converged = True
            break
    return dict(labels=lab, energy=energy(D, i, j, w, lab), switched=switched, cuts=cuts, moves=len(switched),
                cycles=cycles, converged=converged)
