"""GraphDouble.remove_nweights_warm / remove_nweights_dense_warm on the host: argument handling (id arrays, scalars,
lattice-shaped dense decrements, dtypes), the errors, the flush-then-fold path before the first solve, the graphs that
cannot fold -- and, with the real reference BK, the claim the decrement fold rests on: solve, lower capacities (cancelling
the flow an arc carries beyond its new capacity and making up the terminal links), solve again == a fresh solve of the
decreased graph."""
import os
import sys

import numpy
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_native  # noqa: E402
from test_host_seeds import _reference_bk  # noqa: E402
from test_host_warm_tweights import _DeviceArray  # noqa: E402

_SHAPE = (6, 7, 8)
_N = 6 * 7 * 8


class _RemoveGraph(fake_native.FakeGraph):
    """FakeGraph plus the n-link decrement calls: records every call in order and subtracts the decrements from the
    from-scratch n-links (the meaning of the calls)."""

    def __init__(self, shape, device=-1):
        super().__init__(shape, device)
        self.calls = []

    def add_nweights_dense(self, axis, fwd, bwd):
        self.calls.append(("stage", axis))
        super().add_nweights_dense(axis, fwd, bwd)

    def remove_nweights_warm(self, i, j, cap, rev):
        for a in (i, j):
            assert a.dtype == numpy.int64 and a.ndim == 1 and a.flags.c_contiguous
        assert cap.dtype == numpy.float64 and rev.dtype == numpy.float64 and cap.shape == rev.shape == i.shape == j.shape
        self.calls.append(("n", i.copy(), j.copy(), cap.copy(), rev.copy()))
        for a, b, c, r in zip(i.tolist(), j.tolist(), cap.tolist(), rev.tolist()):
            axis, lo = self._axis(a, b)
            self.wf[axis][lo] -= c if a < b else r
            self.wb[axis][lo] -= r if a < b else c
        self.result = None

    def remove_nweights_dense_warm(self, axis, fwd, bwd):
        assert fwd.dtype == numpy.float64 and tuple(fwd.shape) == tuple(self.shape)
        self.calls.append(("d", axis, numpy.array(fwd), numpy.array(bwd)))
        stride = int(numpy.prod(self.shape[axis + 1:]))
        last = (numpy.arange(self.n) // stride) % self.shape[axis] == self.shape[axis] - 1
        self.wf[axis] -= numpy.where(last, 0.0, numpy.ravel(fwd))
        self.wb[axis] -= numpy.where(last, 0.0, numpy.ravel(bwd))
        self.result = None


@pytest.fixture()
def made(monkeypatch):
    from medpy_b200 import _lib
    out = []

    def factory(shape, device=-1):
        g = _RemoveGraph(shape, device)
        out.append(g)
        return g
    monkeypatch.setattr(_lib, "Graph", factory)
    return out


def _chain(shape=_SHAPE, w=4.0):
    """A lattice graph built term by term: every pair with capacity w both ways, a source and a sink voxel."""
    from medpy_b200.graphcut import GraphDouble
    n = int(numpy.prod(shape))
    g = GraphDouble(n, 3 * n, shape=shape)
    for axis in range(len(shape)):
        g.add_nweights_dense(axis, numpy.full(shape, w), numpy.full(shape, w))
    g.add_tweights(0, 100.0, 0.0)
    g.add_tweights(n - 1, 0.0, 100.0)
    return g


def test_list_form_broadcasts_and_widens(made):
    g = _chain()
    g.maxflow()
    g.remove_nweights_warm(numpy.array([5, 6, 5], numpy.int32), numpy.array([6, 5, 13], numpy.int16),
                           numpy.array([1.5, 2.0, 0.25], numpy.float32), 0)
    op = made[0].calls[-1]
    assert op[0] == "n" and op[1].tolist() == [5, 6, 5] and op[2].tolist() == [6, 5, 13]
    assert op[3].tolist() == [1.5, 2.0, 0.25] and op[4].tolist() == [0.0] * 3
    g.remove_nweights_warm(7, [15, 6, 63], 1.0, [1.0, 0.0, 2])
    op = made[0].calls[-1]
    assert op[1].tolist() == [7] * 3 and op[2].tolist() == [15, 6, 63] and op[3].tolist() == [1.0] * 3
    assert op[4].tolist() == [1.0, 0.0, 2.0]
    g.remove_nweights_warm(torch.tensor([5, 21]), torch.tensor(13, dtype=torch.int16), torch.tensor([0.5, 1.0]), torch.tensor(0))
    op = made[0].calls[-1]
    assert op[1].tolist() == [5, 21] and op[2].tolist() == [13, 13] and op[3].tolist() == [0.5, 1.0] and op[4].tolist() == [0.0] * 2


def test_dense_form_takes_any_strides(made):
    g = _chain()
    g.maxflow()
    rng = numpy.random.default_rng(0)
    a = rng.random(_SHAPE)
    b = rng.random(_SHAPE).astype(numpy.float32)
    g.remove_nweights_dense_warm(1, numpy.asfortranarray(a), b[::-1][::-1])
    op = made[0].calls[-1]
    assert op[0] == "d" and op[1] == 1 and numpy.array_equal(op[2], a)
    assert numpy.array_equal(op[3], b.astype(numpy.float64))


def test_bad_arguments_touch_nothing(made):
    g = _chain()
    g.maxflow()
    n_calls = len(made[0].calls)
    for args, what in ((([0, _N - 1], [1, _N], 1.0, 0.0), "Invalid node id"), (([-1], [0], 1.0, 0.0), "Invalid node id"),
                       (([1, 2], [2, 3, 4], 1.0, 0.0), "differ in length"), (([1.5], [2], 1.0, 0.0), "integer"),
                       (([5], [6, 7], 1.0, 0.0), "differ in length"),
                       (([1], [2], _DeviceArray(), 0.0), "must all be host or all be device arrays"),
                       (([1, 2], [2, 3], [1.0, 2.0, 3.0], 0.0), "entries"), (([1], [2], numpy.array([True]), 0.0), "real"),
                       (([1], [2], -1.0, 0.0), "negative"), (([1], [2], 0.0, -1e-300), "negative"),
                       (([1], [2], numpy.nan, 0.0), "NaN"), (([1], [2], 0.0, numpy.inf), "NaN")):
        with pytest.raises(ValueError, match=what):
            g.remove_nweights_warm(*args)
    with pytest.raises(ValueError, match="axis"):
        g.remove_nweights_dense_warm(3, numpy.zeros(_SHAPE), numpy.zeros(_SHAPE))
    with pytest.raises(ValueError, match="shape"):
        g.remove_nweights_dense_warm(0, numpy.zeros((6, 7)), numpy.zeros(_SHAPE))
    bad = numpy.zeros(_SHAPE)
    bad[2, 3, 4] = -1.0
    with pytest.raises(ValueError, match="negative"):
        g.remove_nweights_dense_warm(2, bad, numpy.zeros(_SHAPE))
    bad[2, 3, 4] = numpy.nan
    with pytest.raises(ValueError, match="NaN"):
        g.remove_nweights_dense_warm(2, numpy.zeros(_SHAPE), bad)
    assert len(made[0].calls) == n_calls
    # the last plane of the axis names no pair: whatever it holds is ignored
    last = numpy.zeros(_SHAPE)
    last[:, :, -1] = -numpy.inf
    g.remove_nweights_dense_warm(2, last, numpy.zeros(_SHAPE))
    assert made[0].calls[-1][0] == "d"


def test_unsolved_graph_flushes_then_folds(made):
    """Before the first maxflow() the staged build reaches the handle first, then the decrement folds natively; the
    result is that of the decreased graph."""
    g, ref = _chain(w=4.0), _chain(w=4.0)
    g.sum_edge(3, 4, 2.0, 1.0)                  # staged, not flushed yet
    ref.sum_edge(3, 4, 2.0, 1.0)
    g.remove_nweights_warm([3, 9], [4, 10], [5.0, 1.0], [0.5, 2.0])
    kinds = [c[0] for c in made[0].calls]
    assert kinds.index("n") > max(k for k, c in enumerate(kinds) if c == "stage")
    ref.sum_edge(3, 4, 0.0, 0.0)
    ref._flush()
    r = made[1]
    r.wf[2][3] -= 5.0
    r.wb[2][3] -= 0.5
    r.wf[2][9] -= 1.0
    r.wb[2][9] -= 2.0
    assert g.maxflow() == r.maxflow()
    assert numpy.array_equal(g.get_mask(), r.get_mask())


def test_removal_before_the_first_solve_fixes_the_terms(made):
    """A removal folded into an unsolved graph leaves it holding a residual state: later term calls are refused with a
    clear error instead of failing at the next flush, the graph still solves, and reset() opens it again."""
    g = _chain()
    g.remove_nweights_warm([3], [4], 1.0, 0.0)
    for call in (lambda: g.add_tweights(5, 1.0, 0.0), lambda: g.sum_edge(5, 6, 1.0, 1.0),
                 lambda: g.add_nweights_dense(0, numpy.ones(_SHAPE), numpy.ones(_SHAPE)),
                 lambda: g.add_tweights_dense(numpy.ones(_SHAPE), numpy.zeros(_SHAPE))):
        with pytest.raises(RuntimeError, match="fixed"):
            call()
    g.remove_nweights_warm([9], [10], 0.5, 0.5)          # further removals fold natively
    assert [c[0] for c in made[0].calls].count("n") == 2
    g.maxflow()
    g.reset()
    g.add_tweights(5, 1.0, 0.0)


def test_graphs_that_cannot_fold_raise_runtime_error():
    from medpy_b200.graphcut import GraphDouble
    g = GraphDouble(4, 4)                       # no lattice shape: a general graph
    g.add_tweights(0, 5.0, 0.0)
    g.sum_edge(0, 2, 1.0, 1.0)                  # not a chain neighbour: the sparse backend
    with pytest.raises(RuntimeError, match="reset"):
        g.remove_nweights_warm([0], [1], 1.0, 0.0)
    with pytest.raises(RuntimeError, match="reset"):
        g.remove_nweights_dense_warm(0, numpy.zeros(4), numpy.zeros(4))


# ---- the claim, on the unmodified reference BK ------------------------------------------------------------------------
def _bk_remove(bk, h, pairs):
    """The decrement fold's step 1 on a solved BK graph: per pair (i < j, axis pair) with decrements (df, db), the negated
    decrements; where a residual went negative by d, the cancelling sum_edge(i, j, d, -d) (or its mirror) and the
    terminal links of both ends raised by d: add_tweights(i, d, 0) / add_tweights(j, 0, d) (for the lo -> hi case),
    whose constant d is taken off the energy.  Returns the total taken off."""
    off = 0.0
    for i, j, df, db in pairs:
        a = bk.bkref_get_edge(h, i, j) - df
        b = bk.bkref_get_edge(h, j, i) - db
        bk.bkref_sum_edge(h, i, j, -df, -db)
        if a < 0:
            d = -a
            bk.bkref_sum_edge(h, i, j, d, -d)
            bk.bkref_add_tweights(h, i, d, 0.0)
            bk.bkref_add_tweights(h, j, 0.0, d)
            off += d
        elif b < 0:
            d = -b
            bk.bkref_sum_edge(h, i, j, -d, d)
            bk.bkref_add_tweights(h, j, d, 0.0)
            bk.bkref_add_tweights(h, i, 0.0, d)
            off += d
    return off


def _bk_graph(bk, n, edges, tw):
    h = bk.bkref_new(n, len(edges))
    for i, j, a, b in edges:
        bk.bkref_sum_edge(h, i, j, a, b)
    for v, a, b in tw:
        bk.bkref_add_tweights(h, v, a, b)
    return h


def _bk():
    """_reference_bk plus the residual read-back (bkref_get_edge returns the residual r_cap of the arc i -> j)."""
    import ctypes
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    bk.bkref_get_edge.restype = ctypes.c_double
    bk.bkref_get_edge.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    return bk


def _cut_value(n, edges, tw, seg):
    """Capacity of the cut `seg` (BK's what_segment: 0 source side, 1 sink side) in the graph of `edges` and `tw`: an
    arc i -> j counts when i is on the source side and j on the sink side; a voxel on the sink side pays its source
    links, one on the source side its sink links."""
    v = 0.0
    for i, j, a, b in edges:
        if seg[i] == 0 and seg[j] == 1:
            v += a
        elif seg[j] == 0 and seg[i] == 1:
            v += b
    for x, a, b in tw:
        v += a if seg[x] == 1 else b
    return v


def _check_claim(bk, n, edges, tw, pairs):
    """Warm energy == the fresh solve's, and the warm partition is a minimum cut of the decreased graph (its capacity
    equals the fresh min-cut value; with integer weights the min cut need not be unique, so the partitions themselves
    may differ only between cuts of equal capacity)."""
    warm = _bk_graph(bk, n, edges, tw)
    try:
        bk.bkref_maxflow(warm)
        off = _bk_remove(bk, warm, pairs)
        e = bk.bkref_maxflow(warm) - off
        dec = {(i, j): (df, db) for i, j, df, db in pairs}
        decreased = [(i, j, a - dec.get((i, j), (0, 0))[0], b - dec.get((i, j), (0, 0))[1]) for i, j, a, b in edges]
        cold = _bk_graph(bk, n, decreased, tw)
        try:
            ce = bk.bkref_maxflow(cold)
            assert abs(e - ce) <= 1e-9 * max(1.0, abs(ce)), (e, ce)
            ws = [bk.bkref_what_segment(warm, v) for v in range(n)]
            cs = [bk.bkref_what_segment(cold, v) for v in range(n)]
            assert abs(_cut_value(n, decreased, tw, ws) - ce) <= 1e-9 * max(1.0, abs(ce)), "warm partition is no min cut"
            assert abs(_cut_value(n, decreased, tw, cs) - ce) <= 1e-9 * max(1.0, abs(ce))
            return e, ws, cs
        finally:
            bk.bkref_delete(cold)
    finally:
        bk.bkref_delete(warm)


def test_reference_bk_two_voxel_chain():
    """s -5-> i -5-> j -5-> t: lowering c(i->j) by 3 gives energy 2, by 5 energy 0."""
    bk = _bk()
    edges = [(0, 1, 5.0, 0.0)]
    tw = [(0, 5.0, 0.0), (1, 0.0, 5.0)]
    e, ws, cs = _check_claim(bk, 2, edges, tw, [(0, 1, 3.0, 0.0)])
    assert e == 2.0 and ws == cs
    assert _check_claim(bk, 2, edges, tw, [(0, 1, 5.0, 0.0)])[0] == 0.0


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4, 5])
def test_reference_bk_resolve_after_decrements_equals_from_scratch(seed):
    """Random small lattices, integer weights (exact): decrements of random arcs, of every arc across the solved cut
    (saturated: the cancel branch runs), and of whole pairs; the warm re-solve gives the min-cut energy of the decreased
    graph, and its partition is a minimum cut of that graph."""
    bk = _bk()
    rng = numpy.random.default_rng(seed)
    shape = (4, 5, 6)
    n = int(numpy.prod(shape))
    strides = (30, 6, 1)
    edges = []
    for v in range(n):
        c = numpy.unravel_index(v, shape)
        for d in range(3):
            if c[d] + 1 < shape[d]:
                edges.append((v, v + strides[d], float(rng.integers(1, 20)), float(rng.integers(1, 20))))
    tw = [(int(v), float(rng.integers(0, 40)), float(rng.integers(0, 40))) for v in rng.choice(n, n // 2, replace=False)]
    first = _bk_graph(bk, n, edges, tw)
    try:
        bk.bkref_maxflow(first)
        seg = [bk.bkref_what_segment(first, v) for v in range(n)]
    finally:
        bk.bkref_delete(first)
    cut = [(i, j, a, b) for i, j, a, b in edges if seg[i] != seg[j]]
    picks = [edges[k] for k in rng.choice(len(edges), 25, replace=False)]
    for choose in (lambda e: (e[0], e[1], float(rng.integers(0, int(e[2]) + 1)), float(rng.integers(0, int(e[3]) + 1))),
                   lambda e: (e[0], e[1], e[2] // 2, e[3] // 2),
                   lambda e: (e[0], e[1], e[2], e[3])):
        pairs = [choose(e) for e in (cut + picks)]
        pairs = list({(p[0], p[1]): p for p in pairs}.values())
        _check_claim(bk, n, edges, tw, pairs)
