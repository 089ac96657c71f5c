"""GraphDouble.add_nweights_warm / add_nweights_dense_warm on the host: argument handling (id arrays, scalars, lattice-shaped
dense weights, dtypes), the errors, the staged path before the first solve -- and, with the real reference BK, the claim the
warm n-link fold rests on: solve, sum_edge with nonnegative increments, solve again == a fresh solve of all calls."""
import os
import sys

import numpy
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_native  # noqa: E402
from test_host_erase_seeds import _fresh, _lattice, _mask  # noqa: E402
from test_host_seeds import _reference_bk  # noqa: E402
from test_host_warm_eager import _lattice4  # noqa: E402
from test_host_warm_tweights import _DeviceArray  # noqa: E402

_SHAPE = (6, 7, 8)
_N = 6 * 7 * 8


class _WarmGraph(fake_native.FakeGraph):
    """FakeGraph plus the warm n-link calls: records the arguments and adds the increments to the from-scratch n-links."""

    def __init__(self, shape, device=-1):
        super().__init__(shape, device)
        self.warm_calls = []

    def add_nweights_warm(self, i, j, cap, rev):
        for a in (i, j):
            assert a.dtype == numpy.int64 and a.ndim == 1 and a.flags.c_contiguous
        assert cap.dtype == numpy.float64 and rev.dtype == numpy.float64 and cap.shape == rev.shape == i.shape == j.shape
        self.warm_calls.append(("n", i.copy(), j.copy(), cap.copy(), rev.copy()))
        for a, b, c, r in zip(i.tolist(), j.tolist(), cap.tolist(), rev.tolist()):
            axis, lo = self._axis(a, b)
            self.wf[axis][lo] += c if a < b else r
            self.wb[axis][lo] += r if a < b else c
        self.result = None

    def add_nweights_dense_warm(self, axis, fwd, bwd):
        assert fwd.dtype == numpy.float64 and tuple(fwd.shape) == tuple(self.shape)
        self.warm_calls.append(("d", axis, numpy.array(fwd), numpy.array(bwd)))
        self.add_nweights_dense(axis, numpy.array(fwd), numpy.array(bwd))
        self.result = None


@pytest.fixture()
def made(monkeypatch):
    from medpy_b200 import _lib
    out = []

    def factory(shape, device=-1):
        g = _WarmGraph(shape, device)
        out.append(g)
        return g
    monkeypatch.setattr(_lib, "Graph", factory)
    return out


def _graph(seed=0):
    import medpy_b200.graphcut as gc
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(_SHAPE, seed=seed)
    return gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                                regional_term_args=(vol["prob"], vol["alpha"]),
                                boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                boundary_term_args=(vol["image"], vol["sigma"], False))


def test_list_form_keeps_order_broadcasts_and_widens(made):
    g = _graph()
    g.maxflow()
    g.add_nweights_warm(numpy.array([5, 6, 5], numpy.int32), numpy.array([6, 5, 13], numpy.int16),
                        numpy.array([1.5, 2.0, 3.25], numpy.float32), 0)
    op = made[0].warm_calls[-1]
    assert op[1].tolist() == [5, 6, 5] and op[2].tolist() == [6, 5, 13]
    assert op[3].tolist() == [1.5, 2.0, 3.25] and op[4].tolist() == [0.0] * 3
    g.add_nweights_warm(7, [15, 6, 63], 2.0, [1.0, 0.0, 4.0])
    op = made[0].warm_calls[-1]
    assert op[1].tolist() == [7] * 3 and op[2].tolist() == [15, 6, 63] and op[3].tolist() == [2.0] * 3
    g.add_nweights_warm(torch.tensor([5, 21], dtype=torch.int32), torch.tensor(13), torch.tensor([1.5, 2.0], dtype=torch.float32),
                        torch.tensor(0.5))
    op = made[0].warm_calls[-1]
    assert op[1].tolist() == [5, 21] and op[2].tolist() == [13, 13] and op[3].tolist() == [1.5, 2.0] and op[4].tolist() == [0.5] * 2
    g.add_nweights_warm([3], [4], numpy.nan, 0.0)   # folded calls leave the finite check to the native fold
    assert numpy.isnan(made[0].warm_calls[-1][3]).all()


def test_dense_form_takes_any_strides(made):
    g = _graph()
    g.maxflow()
    rng = numpy.random.default_rng(0)
    a = rng.random(_SHAPE)
    b = rng.random(_SHAPE).astype(numpy.float32)
    g.add_nweights_dense_warm(1, numpy.asfortranarray(a), b[::-1][::-1])
    op = made[0].warm_calls[-1]
    assert op[1] == 1 and numpy.array_equal(op[2], a) and numpy.array_equal(op[3], b.astype(numpy.float64))
    g.add_nweights_dense_warm(0, torch.from_numpy(a), torch.from_numpy(b))
    op = made[0].warm_calls[-1]
    assert op[1] == 0 and numpy.array_equal(op[2], a) and numpy.array_equal(op[3], b.astype(numpy.float64))


def test_bad_arguments(made):
    g = _graph()
    g.maxflow()
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_nweights_warm([0, _N - 1], [1, _N], 1.0, 0.0)
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_nweights_warm([-1], [0], 1.0, 0.0)
    with pytest.raises(ValueError, match="differ in length"):
        g.add_nweights_warm([1, 2], [2, 3, 4], 1.0, 0.0)
    with pytest.raises(ValueError, match="differ in length"):
        g.add_nweights_warm([5], [6, 7], 1.0, 0.0)      # a one-element id array does not broadcast on the lattice
    with pytest.raises(ValueError, match="must all be host or all be device arrays"):
        g.add_nweights_warm([1], [2], _DeviceArray(), 0.0)
    with pytest.raises(ValueError, match="must both be host or both be device arrays"):
        g.add_nweights_dense_warm(0, numpy.zeros(_SHAPE), _DeviceArray())
    with pytest.raises(ValueError, match="integer"):
        g.add_nweights_warm([1.5], [2], 1.0, 0.0)
    with pytest.raises(ValueError, match="integer"):
        g.add_nweights_warm(numpy.zeros((2, 2), numpy.int64), 1, 1.0, 0.0)
    with pytest.raises(ValueError, match="entries"):
        g.add_nweights_warm([1, 2], [2, 3], [1.0, 2.0, 3.0], 0.0)
    with pytest.raises(ValueError, match="real"):
        g.add_nweights_warm([1], [2], numpy.array([True]), 0.0)
    with pytest.raises(ValueError, match="axis"):
        g.add_nweights_dense_warm(3, numpy.zeros(_SHAPE), numpy.zeros(_SHAPE))
    with pytest.raises(ValueError, match="shape"):
        g.add_nweights_dense_warm(0, numpy.zeros((6, 7)), numpy.zeros(_SHAPE))
    with pytest.raises(ValueError, match="shape"):
        g.add_nweights_dense_warm(0, numpy.zeros(_SHAPE), numpy.zeros(_N))
    assert made[0].warm_calls == []


def test_staging_checks_pairs_and_weights(made):
    g = _graph()
    for i, j, c, r, what in ((0, 2, 1.0, 1.0, "neighbours"), (7, 8, 1.0, 1.0, "neighbours"), (3, 3, 1.0, 1.0, "neighbours"),
                             (0, 1, -1.0, 1.0, "negative"), (0, 1, 1.0, numpy.nan, "NaN"), (0, 8, numpy.inf, 0.0, "NaN")):
        with pytest.raises(ValueError, match=what):
            g.add_nweights_warm([i], [j], c, r)
    bad = numpy.ones(_SHAPE)
    bad[2, 3, 4] = -1.0
    with pytest.raises(ValueError, match="negative"):
        g.add_nweights_dense_warm(2, bad, numpy.ones(_SHAPE))
    bad[2, 3, 4] = numpy.nan
    with pytest.raises(ValueError, match="NaN"):
        g.add_nweights_dense_warm(2, numpy.ones(_SHAPE), bad)
    assert not g._st_nw
    last = numpy.ones(_SHAPE)
    last[:, :, -1] = -numpy.inf                 # the last plane names no pair: ignored
    g.add_nweights_dense_warm(2, last, numpy.ones(_SHAPE))
    g._flush()
    assert not made[0].wf[2].reshape(_SHAPE)[:, :, -1].any() and made[0].wf[2].reshape(_SHAPE)[:, :, :-1].all()


def test_unsolved_graph_stages_the_same_sum_edge_calls(made):
    """Before the first maxflow() the calls are staged; the result equals the explicit sum_edge calls (repeated pairs in
    order, pairs named from either end, a dense pass in between)."""
    g, ref = _graph(), _graph()
    rng = numpy.random.default_rng(2)
    i = numpy.array([3, 4, 3, 10, 66, 10, 100])
    j = numpy.array([4, 3, 4, 66, 10, 11, 44])
    cap, rev = rng.random(7) * 10, rng.random(7) * 10
    dense = rng.random(_SHAPE)
    g.add_nweights_warm(i, j, cap, rev)
    g.add_nweights_dense_warm(0, dense, 0.5 * dense)
    g.add_nweights_warm([3], [4], 1.0, 2.0)
    for a, b, c, r in zip(i.tolist(), j.tolist(), cap.tolist(), rev.tolist()):
        ref.sum_edge(a, b, c, r)
    ref.add_nweights_dense(0, dense, 0.5 * dense)
    ref.sum_edge(3, 4, 1.0, 2.0)
    assert made[0].warm_calls == [] and g.maxflow() == ref.maxflow()
    assert numpy.array_equal(g.get_mask(), ref.get_mask())
    for d in range(3):
        assert numpy.array_equal(made[0].wf[d], made[1].wf[d]) and numpy.array_equal(made[0].wb[d], made[1].wb[d])


def test_warm_calls_equal_from_scratch(made):
    from oracle import solvers
    g = _graph()
    g.maxflow()
    g.add_nweights_warm([3, 4, 100], [4, 3, 44], [5.0, 1.0, 2.0], [0.0, 3.0, 7.0])
    g.maxflow()
    rng = numpy.random.default_rng(3)
    g.add_nweights_dense_warm(2, rng.random(_SHAPE), rng.random(_SHAPE))
    e, m = g.maxflow(), g.get_mask()
    f = made[0]
    oe, om, _ = solvers.solve_port(dict(shape=_SHAPE, wf=f.wf, wb=f.wb, tr=f.tr.copy(), flow_const=f.flow))
    assert numpy.array_equal(m, om) and e == oe and len(f.warm_calls) == 2


def test_scalar_and_array_arguments_give_one_native_call(made):
    """A list form always reaches the native side as four 1-D arrays of one length, whatever mix of scalars came in; a
    scalar id pair takes the length of the weights."""
    g = _graph()
    g.maxflow()
    g.add_nweights_warm(numpy.int64(9), 10, 1.0, 2.0)
    g.add_nweights_warm([9], [10], [1.0], [2.0])
    a, b = made[0].warm_calls
    assert all(numpy.array_equal(x, y) and x.dtype == y.dtype for x, y in zip(a[1:], b[1:]))
    g.add_nweights_warm(5, 6, [1.0, 2.0], 0.0)
    op = made[0].warm_calls[-1]
    assert op[1].tolist() == [5, 5] and op[2].tolist() == [6, 6] and op[3].tolist() == [1.0, 2.0] and op[4].tolist() == [0.0] * 2
    with pytest.raises(ValueError, match="entries"):
        g.add_nweights_warm(5, 6, [1.0, 2.0], [0.0, 1.0, 2.0])


def test_staging_refuses_ids_out_of_range(made):
    """Before the first solve no native check runs: ids out of range raise ValueError in the staging itself, and a
    negative id is never wrapped onto another arc."""
    g = _graph()
    for i, j in (([-2], [-1]), ([_N - 1], [_N]), ([0, -8], [1, 0]), ([_N + 55], [_N + 56])):
        with pytest.raises(ValueError, match="Invalid node id"):
            g.add_nweights_warm(i, j, 5.0, 0.0)
        with pytest.raises(ValueError, match="Invalid node id"):
            g._stage_nweights_calls(numpy.array(i, numpy.int64), numpy.array(j, numpy.int64), numpy.full(len(i), 5.0),
                                    numpy.zeros(len(i)))
    assert not g._st_nw


def test_sparse_graph_refusal_says_rebuild():
    from medpy_b200.graphcut import GCGraph
    g = GCGraph(4, 4, sparse=True).get_graph()
    g._solved = True
    with pytest.raises(RuntimeError, match="reset.*rebuild"):
        g.add_nweights_warm([1], [2], 1.0, 0.0)
    with pytest.raises(RuntimeError, match="reset.*rebuild"):
        g.add_nweights_dense_warm(0, numpy.ones(4), numpy.ones(4))


def _nlink_steps(rng, edges):
    """Nonnegative sum_edge increments: repeated pairs, pairs named from their upper end, zero capacities, arcs at voxels
    with a large source link (fg-seeded), interleaved with add_tweights."""
    pick = [edges[k] for k in rng.integers(0, len(edges), 12)]
    fg = sorted({e[0] for e in pick[:3]})
    zero = [(i, j, 0.0, 0.0) for i, j, _, _ in pick[6:8]]
    return [
        [("t", v, 65535.0, 0.0) for v in fg],
        [("e", i, j, float(rng.uniform(0, 5)), float(rng.uniform(0, 5))) for i, j, _, _ in pick[:6]]
        + [("e", j, i, float(rng.uniform(0, 5)), 0.0) for i, j, _, _ in pick[:3]] + [("e",) + z for z in zero],
        [("e", i, j, 50.0, 0.0) for i, j, _, _ in pick[:3]] + [("t", pick[0][1], 0.0, 3.0)],
        [("e", i, j, float(rng.uniform(0, 2)), float(rng.uniform(0, 2))) for i, j, _, _ in edges[::5]],
    ]


def _ops(bk, h, ops):
    for op in ops:
        if op[0] == "t":
            bk.bkref_add_tweights(h, op[1], op[2], op[3])
        else:
            bk.bkref_sum_edge(h, op[1], op[2], op[3], op[4])


@pytest.mark.parametrize("dims,seed", [(3, 0), (3, 1), (3, 2), (4, 0), (4, 1), (2, 0), (1, 0)])
def test_reference_bk_resolve_after_sum_edge_equals_from_scratch(dims, seed):
    """Pinned on the unmodified reference BK: after maxflow(), nonnegative sum_edge increments (and add_tweights between
    them) followed by maxflow() again give the min cut of the graph with the whole call sequence."""
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    if dims == 4:
        rng, n, edges, tw = _lattice4(seed)
    elif dims == 3:
        rng, n, edges, tw = _lattice(bk, seed)
    else:
        rng = numpy.random.default_rng(seed)
        shape = (9, 11) if dims == 2 else (40,)
        n = int(numpy.prod(shape))
        st = (11, 1) if dims == 2 else (1,)
        edges = [(v, v + st[d], float(rng.uniform(0.01, 2.0)), float(rng.uniform(0.01, 2.0)))
                 for v in range(n) for d in range(dims) if numpy.unravel_index(v, shape)[d] + 1 < shape[d]]
        tw = [(v, float(rng.uniform(0, 3)), float(rng.uniform(0, 3))) for v in range(n)]
    steps = _nlink_steps(rng, edges)
    warm = _fresh(bk, n, edges, tw, [])
    try:
        bk.bkref_maxflow(warm)
        done = []
        for ops in steps:
            _ops(bk, warm, ops)
            done += ops
            e = bk.bkref_maxflow(warm)
            cold = _fresh(bk, n, edges, tw, [])
            try:
                _ops(bk, cold, done)
                ce = bk.bkref_maxflow(cold)
                assert _mask(bk, warm, n) == _mask(bk, cold, n)
                assert abs(e - ce) <= 1e-9 * max(abs(ce), 1.0)
            finally:
                bk.bkref_delete(cold)
    finally:
        bk.bkref_delete(warm)

