"""tests/metric_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the alpha-expansion with a metric label distance V (DESIGN.md §11, "Label distances"): the pair term
w_pq V(l_p, l_q) in place of Potts' w_pq [l_p != l_q], for the voxel, region and batch units.  ``pair_terms`` is the one
case table (the numpy mirror of ``exp_metric_pair`` in gc_expansion_pair.cuh); the voxel and region move problems lay
it out as oracle/expansion.py and oracle/region_expansion.py lay out theirs, in the same summation order, and are cut by
the same BK restatements.  Everything else (data costs, pair weights, initial labels, the pairs' arc order) is those
oracles' own code.  Every entry point takes ``V=None``, which runs the Potts oracle unchanged.
"""
import math

import numpy

from oracle import expansion as ox
from oracle import expansion_batch as oxb
from oracle import region_expansion as orx
from oracle import solvers


def pair_terms(w, V, a, b, alpha):
    """What the pairs (p, q), p the lower end, a = l_p, b = l_q, add to the move graph of ``alpha``: (lo to p's sink link,
    up to q's, fwd on arc p -> q, bwd on arc q -> p), element-wise over numpy arrays, with e(x, y) = w * V[x, y]:
      a = b = alpha           nothing
      a = alpha != b          up = e(alpha, b)
      a != alpha = b          lo = e(a, alpha)
      a = b != alpha          fwd = e(a, alpha), bwd = e(alpha, b)
      a != b, neither alpha   lo = min(e00, e01), up = e00 - lo, fwd = e01 - lo, bwd = max(e10 - up, 0)
    with e00 = e(a, b), e01 = e(a, alpha), e10 = e(alpha, b)."""
    w = numpy.asarray(w, numpy.float64)
    a = numpy.asarray(a, numpy.int64)
    b = numpy.asarray(b, numpy.int64)
    e00, e01, e10 = w * V[a, b], w * V[a, alpha], w * V[alpha, b]
    one_a = (a == alpha) & (b != alpha)
    one_b = (a != alpha) & (b == alpha)
    same = (a == b) & (a != alpha)
    split = (a != b) & (a != alpha) & (b != alpha)
    lo5 = numpy.minimum(e00, e01)
    up5 = e00 - lo5
    lo = numpy.where(one_b, e01, numpy.where(split, lo5, 0.0))
    up = numpy.where(one_a, e10, numpy.where(split, up5, 0.0))
    fwd = numpy.where(same, e01, numpy.where(split, e01 - lo5, 0.0))
    bwd = numpy.where(same, e10, numpy.where(split, numpy.maximum(e10 - up5, 0.0), 0.0))
    return lo, up, fwd, bwd


# ------------------------------------------------------------------------------------------------------------- voxels
def energy(D, w, labels, V=None):
    """E(l) = sum_p D_p(l_p) + sum_pairs w_pq V(l_p, l_q), summed exactly (math.fsum) then rounded once."""
    if V is None:
        return ox.energy(D, w, labels)
    lab = numpy.asarray(labels).astype(numpy.int64)
    flat = lab.ravel()
    terms = [D[flat, numpy.arange(flat.size)]]
    for d, wd in enumerate(w):
        lo, hi = ox._axis_slices(lab.ndim, d)
        cut = lab[lo] != lab[hi]
        terms.append(wd[cut] * V[lab[lo][cut], lab[hi][cut]])
    return math.fsum(numpy.concatenate([t.ravel() for t in terms]))


def move_problem(D, w, labels, alpha, V=None):
    """``ox.move_problem`` with the pair terms of ``pair_terms``: src_p = D_p(alpha); snk_p = D_p(l_p) + lo and up
    contributions axis by axis, within an axis first the pair where p is the lower end; then add_tweights on tr = 0."""
    if V is None:
        return ox.move_problem(D, w, labels, alpha)
    lab = numpy.asarray(labels).astype(numpy.int64)
    shape = lab.shape
    n = lab.size
    flat = lab.ravel()
    idx = numpy.arange(n)
    src = D[alpha, idx].copy()
    snk = D[flat, idx].copy()
    wf, wb = [], []
    for d, wd in enumerate(w):
        lo, hi = ox._axis_slices(lab.ndim, d)
        t_lo, t_up, t_f, t_b = pair_terms(wd, V, lab[lo], lab[hi], alpha)
        cl = numpy.zeros(shape)
        cu = numpy.zeros(shape)
        f = numpy.zeros(shape)
        b = numpy.zeros(shape)
        cl[lo] = t_lo
        cu[hi] = t_up
        f[lo] = t_f                     # arc p -> q
        b[lo] = t_b                     # arc q -> p (entry p, as build_problem's wb)
        snk = snk + cl.ravel()
        snk = snk + cu.ravel()
        wf.append(f.ravel())
        wb.append(b.ravel())
    tr = numpy.zeros(n)
    flow = ox.energy_terms.add_tweights_pass(tr, 0.0, src, snk)
    return dict(shape=shape, wf=wf, wb=wb, tr=tr, flow_const=flow)


def move(D, w, labels, alpha, V=None):
    """One move: (new labels, switched voxels, cut value = flow_const + max-flow)."""
    lab = numpy.asarray(labels)
    cut, mask, _ = solvers.solve_port(move_problem(D, w, lab, alpha, V))
    switch = (mask == 0) & (lab != alpha)
    out = lab.copy()
    out[switch] = alpha
    return out, int(switch.sum()), cut


def expansion(costs, boundary=None, markers=None, init=None, max_cycles=20, V=None):
    """``ox.expansion`` with the label distance V (None: ``ox.expansion`` itself)."""
    if V is None:
        return ox.expansion(costs, boundary, markers, init, max_cycles)
    V = numpy.asarray(V, numpy.float64)
    costs = numpy.asarray(costs)
    K = costs.shape[0]
    shape = costs.shape[1:]
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    lab = ox.initial_labels(D, shape, init)
    switched, cuts = [], []
    cycles = 0
    converged = False
    for _ in range(max_cycles):
        changed = 0
        for alpha in range(K):
            lab, s, cut = move(D, w, lab, alpha, V)
            switched.append(s)
            cuts.append(cut)
            changed += s
        cycles += 1
        if changed == 0:
            converged = True
            break
    return dict(labels=lab, energy=energy(D, w, lab, V), switched=switched, cuts=cuts, moves=len(switched),
                cycles=cycles, converged=converged)


# ------------------------------------------------------------------------------------------------------------ regions
def region_energy(D, i, j, w, labels, V=None):
    """E(l) = sum_r D_r(l_r) + sum_pairs w_rs V(l_r, l_s), summed exactly (math.fsum) then rounded once."""
    if V is None:
        return orx.energy(D, i, j, w, labels)
    lab = numpy.asarray(labels).astype(numpy.int64)
    w = numpy.asarray(w, numpy.float64)
    li, lj = lab[numpy.asarray(i, numpy.int64)], lab[numpy.asarray(j, numpy.int64)]
    cut = li != lj
    return math.fsum(numpy.concatenate([D[lab, numpy.arange(lab.size)], w[cut] * V[li[cut], lj[cut]]]))


def region_move_problem(D, i, j, w, labels, alpha, V=None):
    """``orx.move_problem`` with the pair terms of ``pair_terms``.  Node u with a = l_u != alpha, arc u -> v in the row's
    order: u < v adds lo of the pair (u, v) to snk_u and puts its fwd on the arc; u > v adds up of the pair (v, u) and
    puts its bwd on the arc.  A node labelled alpha adds nothing and has no arcs."""
    if V is None:
        return orx.move_problem(D, i, j, w, labels, alpha)
    lab = numpy.asarray(labels).astype(numpy.int64)
    R = lab.size
    idx = numpy.arange(R)
    w = numpy.asarray(w, numpy.float64)
    src = D[alpha, idx].copy()
    snk = D[lab, idx].copy()
    tail, head, pair = orx._arcs(i, j)
    a, b = lab[tail], lab[head]
    lower = tail < head
    lo_t, _, fwd_t, _ = pair_terms(w[pair], V, a, b, alpha)          # the arc's tail is the pair's lower end
    _, up_t, _, bwd_t = pair_terms(w[pair], V, b, a, alpha)          # ... its upper end
    t = numpy.where(lower, lo_t, up_t)
    cap = numpy.where(lower, fwd_t, bwd_t)
    free = a != alpha
    numpy.add.at(snk, tail[free], t[free])              # unbuffered, in index order: per node in row order
    cap = numpy.where(free, cap, 0.0)
    fwd = numpy.zeros(len(w))
    bwd = numpy.zeros(len(w))
    fwd[pair[lower]] = cap[lower]
    bwd[pair[~lower]] = cap[~lower]
    return (numpy.asarray(i), numpy.asarray(j), fwd, bwd), (idx, src, snk)


def region_move(D, i, j, w, labels, alpha, V=None):
    """One move: (new labels, switched regions, cut value = add_tweights constant + max-flow)."""
    lab = numpy.asarray(labels)
    edges, tw = region_move_problem(D, i, j, w, lab, alpha, V)
    cut, mask, _ = solvers.solve_sparse_port(lab.size, *edges, [tw])
    switch = (mask == 0) & (lab != alpha)
    out = lab.copy()
    out[switch] = alpha
    return out, int(switch.sum()), cut


def region_expansion(D, i, j, w, init=None, max_cycles=20, V=None):
    """``orx.expansion`` with the label distance V (None: ``orx.expansion`` itself)."""
    if V is None:
        return orx.expansion(D, i, j, w, init=init, max_cycles=max_cycles)
    V = numpy.asarray(V, numpy.float64)
    K = D.shape[0]
    lab = (numpy.argmin(D, axis=0) if init is None else numpy.asarray(init)).astype(numpy.uint8)
    switched, cuts = [], []
    cycles = 0
    converged = False
    for _ in range(max_cycles):
        changed = 0
        for alpha in range(K):
            lab, s, cut = region_move(D, i, j, w, lab, alpha, V)
            switched.append(s)
            cuts.append(cut)
            changed += s
        cycles += 1
        if changed == 0:
            converged = True
            break
    return dict(labels=lab, energy=region_energy(D, i, j, w, lab, V), switched=switched, cuts=cuts,
                moves=len(switched), cycles=cycles, converged=converged)


# ------------------------------------------------------------------------------------------------------------ batches
def expansion_batch(costs, boundaries=None, markers=None, init=None, max_cycles=20, V=None):
    """``oxb.expansion_batch`` with the label distance V (None: ``oxb.expansion_batch`` itself): the same loop, freezing
    and results, each image's moves built and cut by ``move`` on that image alone."""
    if V is None:
        return oxb.expansion_batch(costs, boundaries, markers, init, max_cycles)
    V = numpy.asarray(V, numpy.float64)
    costs = numpy.asarray(costs)
    B, K = costs.shape[:2]
    shape = costs.shape[2:]
    D, w, lab = [], [], []
    for b in range(B):
        D.append(ox.data_costs(costs[b], None if markers is None else markers[b]))
        w.append(ox.pair_weights(shape, None if boundaries is None else boundaries[b]))
        lab.append(ox.initial_labels(D[b], shape, None if init is None else init[b]))
    active = [True] * B
    cycles = [0] * B
    converged = [False] * B
    rows = []
    batch_cycles = 0
    for _ in range(max_cycles):
        if not any(active):
            break
        changed = [0] * B
        for alpha in range(K):
            row = [0] * B
            for b in range(B):
                if active[b]:
                    lab[b], row[b], _ = move(D[b], w[b], lab[b], alpha, V)
                    changed[b] += row[b]
            rows.append(row)
        batch_cycles += 1
        for b in range(B):
            if active[b]:
                cycles[b] += 1
                if changed[b] == 0:
                    converged[b] = True
                    active[b] = False
    matrix = numpy.asarray(rows, dtype=numpy.int64).reshape(len(rows), B)
    moves = [K * c for c in cycles]
    return dict(labels=numpy.stack(lab).astype(numpy.uint8),
                energies=numpy.asarray([energy(D[b], w[b], lab[b], V) for b in range(B)]),
                matrix=matrix, batch_moves=len(rows), batch_cycles=batch_cycles, batch_converged=not any(active),
                moves=moves, cycles=cycles, converged=converged,
                switched=[matrix[:moves[b], b].tolist() for b in range(B)])


# ----------------------------------------------------------------------------------------------------------- matrices
def truncated_linear(K, T=2.0):
    i = numpy.arange(K)
    return numpy.minimum(numpy.abs(i[:, None] - i[None, :]), T).astype(numpy.float64)


def scaled_potts(K, s=0.7):
    return s * (1.0 - numpy.eye(K))


def random_metric(K, seed):
    """The shortest-path (Floyd-Warshall) closure of a random symmetric matrix, repeated until no entry changes so that the
    triangle inequality holds in float64: a metric."""
    rng = numpy.random.default_rng(seed)
    A = rng.random((K, K)) * 2.0 + 0.1
    V = numpy.minimum(A, A.T)
    numpy.fill_diagonal(V, 0.0)
    while True:
        old = V.copy()
        for k in range(K):
            V = numpy.minimum(V, V[:, k:k + 1] + V[k:k + 1, :])
        if numpy.array_equal(V, old):
            return V


def pseudo_metric(K):
    """|c(a) - c(b)| over label classes c where labels 0 and 1 share a class: V(0, 1) = 0."""
    c = numpy.maximum(numpy.arange(K) - 1, 0).astype(numpy.float64) * 0.75      # exact: the triangle holds in float64
    return numpy.abs(c[:, None] - c[None, :])


def is_metric(V):
    """The rules DESIGN.md §11 states, in float64."""
    return bool(numpy.isfinite(V).all() and (V >= 0).all() and not numpy.diagonal(V).any() and (V == V.T).all()
                and (V[:, None, :] <= V[:, :, None] + V[None, :, :]).all())
