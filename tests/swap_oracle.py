"""tests/swap_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the alpha-beta swap moves (DESIGN.md §11, "Swap moves") for the voxel, region and batch units: every
move graph of the pair (alpha, beta) in numpy, in the kernels' summation order, laid out as oracle/expansion.py and
oracle/region_expansion.py lay out theirs and cut by the same BK restatements (oracle/solvers.py).  The data costs, pair
weights, initial labels and the region arcs' order are those oracles' own code; the energy is tests/metric_oracle.py's.
Every entry point takes ``V=None`` for Potts, which is V = 1 - I: w * 1.0 has the bits of w, so the Potts kernels and
this mirror agree bit for bit.
"""
import math

import numpy

from oracle import expansion as ox
from oracle import region_expansion as orx
from oracle import solvers

import metric_oracle as mo


def pairs(K):
    """The moves of one cycle: (alpha, beta), alpha < beta, in lexicographic order."""
    return [(a, b) for a in range(K) for b in range(a + 1, K)]


def _dist(V, K):
    return 1.0 - numpy.eye(K) if V is None else numpy.asarray(V, numpy.float64)


def _apply(lab, mask, alpha, beta):
    """Participants take beta where the mask says SINK (0), alpha elsewhere; (new labels, elements that changed)."""
    part = (lab == alpha) | (lab == beta)
    out = numpy.where(part, numpy.where(mask == 0, beta, alpha), lab).astype(lab.dtype)
    return out, int((out != lab).sum())


# ------------------------------------------------------------------------------------------------------------- voxels
def move_problem(D, w, labels, alpha, beta, V=None):
    """The swap move of (alpha, beta) over ``labels`` as a ``build_problem`` dict (SINK = beta).  A participant p has
    src_p = D_p(beta), snk_p = D_p(alpha); per axis, first the pair where p is the lower end, then the one where it is the
    upper end, a neighbour labelled c that is no participant adds w V(beta, c) to src_p and w V(alpha, c) to snk_p; two
    participants get w V(alpha, beta) on both arcs.  Then add_tweights on tr = 0 in node order."""
    lab = numpy.asarray(labels).astype(numpy.int64)
    K = D.shape[0]
    V = _dist(V, K)
    shape = lab.shape
    n = lab.size
    idx = numpy.arange(n)
    part = (lab == alpha) | (lab == beta)
    src = numpy.where(part.ravel(), D[beta, idx], 0.0)
    snk = numpy.where(part.ravel(), D[alpha, idx], 0.0)
    wf, wb = [], []
    for d, wd in enumerate(w):
        lo, hi = ox._axis_slices(lab.ndim, d)
        lp, lq, pp, pq = lab[lo], lab[hi], part[lo], part[hi]
        seen_p = pp & ~pq                       # p a participant, q fixed at lq
        seen_q = pq & ~pp
        both = pp & pq
        ls, lk, us, uk = (numpy.zeros(shape) for _ in range(4))
        ls[lo] = numpy.where(seen_p, wd * V[beta, lq], 0.0)
        lk[lo] = numpy.where(seen_p, wd * V[alpha, lq], 0.0)
        us[hi] = numpy.where(seen_q, wd * V[beta, lp], 0.0)
        uk[hi] = numpy.where(seen_q, wd * V[alpha, lp], 0.0)
        f = numpy.zeros(shape)
        b = numpy.zeros(shape)
        f[lo] = numpy.where(both, wd * V[alpha, beta], 0.0)      # arc p -> q
        b[lo] = numpy.where(both, wd * V[beta, alpha], 0.0)      # arc q -> p (entry p, as build_problem's wb)
        src = src + ls.ravel()
        src = src + us.ravel()
        snk = snk + lk.ravel()
        snk = snk + uk.ravel()
        wf.append(f.ravel())
        wb.append(b.ravel())
    tr = numpy.zeros(n)
    flow = ox.energy_terms.add_tweights_pass(tr, 0.0, src, snk)
    return dict(shape=shape, wf=wf, wb=wb, tr=tr, flow_const=flow)


def move(D, w, labels, alpha, beta, V=None):
    """One swap move: (new labels, switched voxels, cut value = flow_const + max-flow)."""
    lab = numpy.asarray(labels)
    cut, mask, _ = solvers.solve_port(move_problem(D, w, lab, alpha, beta, V))
    out, switched = _apply(lab, mask, alpha, beta)
    return out, switched, cut


def fixed_energy(D, w, labels, alpha, beta, V=None):
    """F: the energy the swap move of (alpha, beta) cannot change -- the data of the non-participants and the pairs with
    no participant.  A move's cut value is E(result) - F."""
    lab = numpy.asarray(labels).astype(numpy.int64)
    V = _dist(V, D.shape[0])
    part = (lab == alpha) | (lab == beta)
    flat = lab.ravel()
    keep = ~part.ravel()
    terms = [D[flat[keep], numpy.flatnonzero(keep)]]
    for d, wd in enumerate(w):
        lo, hi = ox._axis_slices(lab.ndim, d)
        none = ~part[lo] & ~part[hi]
        terms.append(wd[none] * V[lab[lo][none], lab[hi][none]])
    return math.fsum(numpy.concatenate([t.ravel() for t in terms]))


def swap(costs, boundary=None, markers=None, init=None, max_cycles=20, V=None):
    """The whole loop: cycles of the pairs until a cycle switches nothing or ``max_cycles`` cycles ran.  Returns
    dict(labels uint8, energy, switched per move, cuts per move, moves, cycles, converged)."""
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
        for alpha, beta in pairs(K):
            lab, s, cut = move(D, w, lab, alpha, beta, V)
            switched.append(s)
            cuts.append(cut)
            changed += s
        cycles += 1
        if changed == 0:
            converged = True
            break
    return dict(labels=lab, energy=mo.energy(D, w, lab, V), switched=switched, cuts=cuts, moves=len(switched),
                cycles=cycles, converged=converged)


# ------------------------------------------------------------------------------------------------------------ regions
def region_move_problem(D, i, j, w, labels, alpha, beta, V=None):
    """The swap move of (alpha, beta) over region ``labels`` (SINK = beta): (sum_edge calls i, j, cap i->j, cap j->i;
    the add_tweights call (nodes, src, snk)).  A participant u has src_u = D_u(beta), snk_u = D_u(alpha); every arc u -> v
    in the row's order adds w V(beta, l_v) to src_u and w V(alpha, l_v) to snk_u when v is no participant (+0.0 when it
    is), and carries w V(alpha, beta) when both are participants."""
    lab = numpy.asarray(labels).astype(numpy.int64)
    K = D.shape[0]
    V = _dist(V, K)
    R = lab.size
    idx = numpy.arange(R)
    w = numpy.asarray(w, numpy.float64)
    part = (lab == alpha) | (lab == beta)
    src = numpy.where(part, D[beta, idx], 0.0)
    snk = numpy.where(part, D[alpha, idx], 0.0)
    tail, head, pair = orx._arcs(i, j)
    wa = w[pair]
    pt, ph = part[tail], part[head]
    b = lab[head]
    fixed = pt & ~ph
    ts = numpy.where(fixed, wa * V[beta, b], 0.0)
    tk = numpy.where(fixed, wa * V[alpha, b], 0.0)
    numpy.add.at(src, tail[pt], ts[pt])                 # unbuffered, in index order: per node in row order
    numpy.add.at(snk, tail[pt], tk[pt])
    cap = numpy.where(pt & ph, wa * V[alpha, beta], 0.0)
    fwd = numpy.zeros(len(w))
    bwd = numpy.zeros(len(w))
    lo = tail < head
    fwd[pair[lo]] = cap[lo]
    bwd[pair[~lo]] = cap[~lo]
    return (numpy.asarray(i), numpy.asarray(j), fwd, bwd), (idx, src, snk)


def region_move(D, i, j, w, labels, alpha, beta, V=None):
    """One swap move: (new labels, switched regions, cut value = add_tweights constant + max-flow)."""
    lab = numpy.asarray(labels)
    edges, tw = region_move_problem(D, i, j, w, lab, alpha, beta, V)
    cut, mask, _ = solvers.solve_sparse_port(lab.size, *edges, [tw])
    out, switched = _apply(lab, numpy.asarray(mask), alpha, beta)
    return out, switched, cut


def region_fixed_energy(D, i, j, w, labels, alpha, beta, V=None):
    """F of a region move: the data of the non-participants and the pairs with no participant."""
    lab = numpy.asarray(labels).astype(numpy.int64)
    V = _dist(V, D.shape[0])
    part = (lab == alpha) | (lab == beta)
    i, j = numpy.asarray(i, numpy.int64), numpy.asarray(j, numpy.int64)
    none = ~part[i] & ~part[j]
    keep = numpy.flatnonzero(~part)
    return math.fsum(numpy.concatenate([D[lab[keep], keep],
                                           numpy.asarray(w, numpy.float64)[none] * V[lab[i][none], lab[j][none]]]))


def region_swap(D, i, j, w, init=None, max_cycles=20, V=None):
    """The region loop from ``init`` or argmin_k D (ties to the lowest k), as ``swap``."""
    K = D.shape[0]
    lab = (numpy.argmin(D, axis=0) if init is None else numpy.asarray(init)).astype(numpy.uint8)
    switched, cuts = [], []
    cycles = 0
    converged = False
    for _ in range(max_cycles):
        changed = 0
        for alpha, beta in pairs(K):
            lab, s, cut = region_move(D, i, j, w, lab, alpha, beta, V)
            switched.append(s)
            cuts.append(cut)
            changed += s
        cycles += 1
        if changed == 0:
            converged = True
            break
    return dict(labels=lab, energy=mo.region_energy(D, i, j, w, lab, V), switched=switched, cuts=cuts,
                moves=len(switched), cycles=cycles, converged=converged)


# ------------------------------------------------------------------------------------------------------------ batches
def swap_batch(costs, boundaries=None, markers=None, init=None, max_cycles=20, V=None):
    """The batch loop of oracle/expansion_batch.py with swap moves: each image's moves built and cut by ``move`` on that
    image alone; an image whose cycle switched nothing is frozen (its column holds 0 from then on), and image b has
    K(K-1)/2 x cycles_b moves."""
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
        for alpha, beta in pairs(K):
            row = [0] * B
            for b in range(B):
                if active[b]:
                    lab[b], row[b], _ = move(D[b], w[b], lab[b], alpha, beta, V)
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
    moves = [len(pairs(K)) * c for c in cycles]
    return dict(labels=numpy.stack(lab).astype(numpy.uint8),
                energies=numpy.asarray([mo.energy(D[b], w[b], lab[b], V) for b in range(B)]),
                matrix=matrix, batch_moves=len(rows), batch_cycles=batch_cycles, batch_converged=not any(active),
                moves=moves, cycles=cycles, converged=converged,
                switched=[matrix[:moves[b], b].tolist() for b in range(B)])


# ----------------------------------------------------------------------------------------------------------- matrices
def truncated_quadratic(K, T=4.0):
    i = numpy.arange(K)
    return numpy.minimum((i[:, None] - i[None, :]) ** 2, T).astype(numpy.float64)


def random_semi_metric(K, seed):
    """A random symmetric V >= 0 with a zero diagonal that breaks the triangle inequality (for K >= 3)."""
    rng = numpy.random.default_rng(seed)
    A = rng.random((K, K)) * 2.0 + 0.1
    V = numpy.minimum(A, A.T)
    numpy.fill_diagonal(V, 0.0)
    if K >= 3:
        V[0, 2] = V[2, 0] = V[0, 1] + V[1, 2] + 0.5
    return V


def is_semi_metric(V):
    V = numpy.asarray(V)
    return bool(numpy.isfinite(V).all() and (V >= 0).all() and not numpy.diagonal(V).any() and (V == V.T).all())
