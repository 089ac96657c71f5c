"""GraphDouble.add_tweights_warm on the host: argument handling (id arrays, masks, scalars, lattice-shaped and flat dense
weights in logical C order, dtypes), the errors, the staged path before the first solve -- and, with the real reference BK,
the claim the warm fold rests on: solve, add_tweights with any real values, solve again == a fresh solve of all calls."""
import os
import sys

import numpy
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_native  # noqa: E402
from test_host_erase_seeds import _calls, _fresh, _lattice, _mask  # noqa: E402
from test_host_seeds import _reference_bk  # noqa: E402

_SHAPE = (6, 7, 8)
_N = 6 * 7 * 8


class _DeviceArray:
    """Stands for an array in device memory: a lattice warm call refuses it next to a host array before reading it."""
    __cuda_array_interface__ = {}


class _WarmGraph(fake_native.FakeGraph):
    """FakeGraph plus add_tweights_warm: records the arguments and replays the calls on the from-scratch t-links."""

    def __init__(self, shape, device=-1):
        super().__init__(shape, device)
        self.warm_calls = []

    def add_tweights_warm(self, ids, src, snk):
        from oracle import energy_terms as et
        assert src.dtype == numpy.float64 and snk.dtype == numpy.float64 and src.flags.c_contiguous
        assert src.ndim == 1 and src.shape == snk.shape
        if ids is not None:
            assert ids.dtype == numpy.int64 and ids.shape == src.shape
        if not (numpy.isfinite(src).all() and numpy.isfinite(snk).all()):
            raise ValueError("a t-link weight is NaN or infinite")      # the native check
        self.warm_calls.append((None if ids is None else ids.copy(), src.copy(), snk.copy()))
        if ids is None:
            self.flow = et.add_tweights_pass(self.tr, self.flow, src, snk)
        else:
            for v, s, t in zip(ids.tolist(), src.tolist(), snk.tolist()):
                self.flow = et.add_tweights_pass(self.tr, self.flow, s, t, where=numpy.arange(self.n) == v)
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
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(vol["prob"], vol["alpha"]),
                             boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    return g, vol


def test_list_form_keeps_order_duplicates_and_widens(made):
    g, _ = _graph()
    g.maxflow()
    g.add_tweights_warm(numpy.array([5, 3, 5], numpy.int32), numpy.array([1.5, -2.0, 3.25], numpy.float32), [0.0, 4.0, -1.0])
    ids, src, snk = made[0].warm_calls[-1]
    assert ids.tolist() == [5, 3, 5] and src.tolist() == [1.5, -2.0, 3.25] and snk.tolist() == [0.0, 4.0, -1.0]
    g.add_tweights_warm(torch.tensor([4, 2], dtype=torch.int32), torch.tensor([0.5, -1.0], dtype=torch.float32), torch.tensor(2))
    ids, src, snk = made[0].warm_calls[-1]
    assert ids.tolist() == [4, 2] and src.tolist() == [0.5, -1.0] and snk.tolist() == [2.0, 2.0]


def test_scalars_broadcast_and_masks_give_c_order_ids(made):
    g, _ = _graph()
    g.maxflow()
    m = numpy.zeros(_SHAPE, bool)
    m[1, 2, 3] = m[4, 0, 7] = m[0, 6, 0] = True
    g.add_tweights_warm(numpy.asfortranarray(m), 50, 0.0)
    ids, src, snk = made[0].warm_calls[-1]
    assert ids.tolist() == [0 * 56 + 6 * 8 + 0, 1 * 56 + 2 * 8 + 3, 4 * 56 + 0 * 8 + 7]
    assert src.tolist() == [50.0] * 3 and snk.tolist() == [0.0] * 3


def test_dense_form_reads_logical_c_order(made):
    g, _ = _graph()
    g.maxflow()
    rng = numpy.random.default_rng(0)
    a = rng.normal(size=_SHAPE)
    b = rng.normal(size=_SHAPE).astype(numpy.float32)
    g.add_tweights_warm(None, numpy.asfortranarray(a), b[::-1][::-1])
    ids, src, snk = made[0].warm_calls[-1]
    assert ids is None
    assert numpy.array_equal(src, a.ravel()) and numpy.array_equal(snk, b.astype(numpy.float64).ravel())
    g.add_tweights_warm(None, a.ravel(), 0.0)
    ids, src, snk = made[0].warm_calls[-1]
    assert ids is None and numpy.array_equal(src, a.ravel()) and not snk.any() and snk.size == _N
    g.add_tweights_warm(None, torch.from_numpy(a), torch.from_numpy(b.ravel()))
    ids, src, snk = made[0].warm_calls[-1]
    assert ids is None and numpy.array_equal(src, a.ravel()) and numpy.array_equal(snk, b.astype(numpy.float64).ravel())


def test_bad_arguments(made):
    g, _ = _graph()
    g.maxflow()
    with pytest.raises(ValueError, match="Invalid node id of {} or 0. Valid values are 0 to {}.".format(_N, _N - 1)):
        g.add_tweights_warm([0, _N], 1.0, 0.0)
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_tweights_warm([-1], 1.0, 0.0)
    with pytest.raises(ValueError):
        g.add_tweights_warm(numpy.zeros((2, 2), numpy.int64), 1.0, 0.0)
    with pytest.raises(ValueError):
        g.add_tweights_warm([1.5], 1.0, 0.0)
    with pytest.raises(ValueError, match="entries"):
        g.add_tweights_warm([1, 2], [1.0, 2.0, 3.0], 0.0)
    with pytest.raises(ValueError, match="shape"):
        g.add_tweights_warm(None, numpy.zeros((6, 7)), 0.0)
    with pytest.raises(ValueError, match="shape"):
        g.add_tweights_warm(None, numpy.zeros(_N + 1), 0.0)
    with pytest.raises(ValueError, match="NaN"):
        g.add_tweights_warm([1, 2], [1.0, numpy.nan], 0.0)
    with pytest.raises(ValueError, match="NaN"):
        g.add_tweights_warm([1], 0.0, numpy.inf)
    with pytest.raises(ValueError, match="NaN"):
        g.add_tweights_warm(None, numpy.full(_SHAPE, -numpy.inf), 0.0)
    with pytest.raises(ValueError, match="real"):
        g.add_tweights_warm([1], numpy.array([True]), 0.0)
    with pytest.raises(ValueError):
        g.add_tweights_warm(3, 1.0, 0.0)                # a single id is not an id array on the lattice
    with pytest.raises(ValueError, match="must all be host or all be device arrays"):
        g.add_tweights_warm([1, 2], _DeviceArray(), 0.0)
    with pytest.raises(ValueError, match="a t-link weight is NaN"):
        g.add_tweights_warm([1], numpy.nan, 0.0)        # folded calls are checked by the native fold, not twice
    assert made[0].warm_calls == []


def test_staging_refuses_non_finite_weights(made):
    g, _ = _graph()
    with pytest.raises(ValueError, match="NaN"):
        g.add_tweights_warm([1, 2], [1.0, numpy.nan], 0.0)
    with pytest.raises(ValueError, match="NaN"):
        g.add_tweights_warm(None, 0.0, numpy.full(_SHAPE, numpy.inf))
    assert g._st_src is None and not g._pending


def test_warm_calls_equal_from_scratch(made):
    """Soft stroke, dense regional delta, negative and mixed values on one voxel: the fake's from-scratch replay of the same
    add_tweights sequence is what the warm path must give."""
    from oracle import energy_terms as et, solvers
    g, vol = _graph()
    g.maxflow()
    rng = numpy.random.default_rng(1)
    ids = numpy.array([100, 101, 5, 100, 9])
    src, snk = numpy.array([50.0, -3.0, 0.0, 2.5, -7.0]), numpy.array([0.0, 4.0, 12.0, -1.5, 7.0])
    g.add_tweights_warm(ids, src, snk)
    g.maxflow()
    dense = (rng.normal(size=_SHAPE) * (rng.random(_SHAPE) < 0.3), rng.normal(size=_SHAPE))
    g.add_tweights_warm(None, *dense)
    e, m = g.maxflow(), g.get_mask()
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    for v, s, t in zip(ids, src, snk):
        prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], s, t, where=numpy.arange(_N) == v)
    prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], dense[0].ravel(), dense[1].ravel())
    oe, om, _ = solvers.solve_port(prob)
    assert numpy.array_equal(m, om) and abs(e - oe) <= 1e-9 * abs(oe)


def test_unsolved_graph_stages_the_same_add_tweights_calls(made):
    """Before the first maxflow() the calls are staged; the result equals the explicit add_tweights calls (repeated ids
    kept in order, a dense pass in between)."""
    g, _ = _graph()
    ref, _ = _graph()
    rng = numpy.random.default_rng(2)
    ids = numpy.array([3, 7, 3, 3, 9, 7])
    src, snk = rng.normal(size=6) * 10, rng.normal(size=6) * 10
    dense = rng.normal(size=_SHAPE)
    g.add_tweights_warm(ids, src, snk)
    g.add_tweights_warm(None, dense, 0.5)
    g.add_tweights_warm([3], -1.0, 2.0)
    for v, s, t in zip(ids.tolist(), src.tolist(), snk.tolist()):
        ref.add_tweights(v, s, t)
    for v in range(_N):
        ref.add_tweights(v, float(dense.flat[v]), 0.5)
    ref.add_tweights(3, -1.0, 2.0)
    assert made[0].warm_calls == [] and g.maxflow() == ref.maxflow()
    assert numpy.array_equal(g.get_mask(), ref.get_mask())
    assert numpy.array_equal(made[0].tr, made[1].tr) and made[0].flow == made[1].flow


def test_sparse_graph_refusal_says_rebuild():
    from medpy_b200.graphcut import GCGraph
    g = GCGraph(4, 4, sparse=True).get_graph()
    g._solved = True            # stands for a solved graph: the sparse solve itself needs the device
    with pytest.raises(RuntimeError, match="reset.*rebuild"):
        g.add_tweights_warm([1], 1.0, 0.0)
    with pytest.raises(RuntimeError, match="reset.*rebuild"):
        g.add_tweights_warm(None, numpy.ones(4), 0.0)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_reference_bk_resolve_after_real_tweights_equals_from_scratch(seed):
    """Pinned on the unmodified reference BK: after maxflow(), add_tweights with random reals of both signs (soft strokes,
    repeated ids, mixed signs on one voxel, dense passes with zero entries) and maxflow() again give the min cut of the
    graph with the whole call sequence (same mask, same energy as a fresh solve)."""
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    rng, n, edges, tw = _lattice(bk, seed)
    v = int(rng.integers(0, n))
    ids = rng.integers(0, n, 8).tolist()
    dense = rng.normal(0, 2, n) * (rng.random(n) < 0.5)
    steps = [[(i, float(rng.uniform(0, 5)), 0.0) for i in ids],                        # soft fg stroke
             [(i, float(rng.uniform(-4, 4)), float(rng.uniform(-4, 4))) for i in ids + [v, v, v]],
             [(i, float(dense[i]), float(-dense[i] / 2)) for i in range(n)],           # dense pass
             [(v, -3.0, 2.0), (v, 1.0, -5.0)] + [(i, 0.0, float(rng.uniform(0, 3))) for i in ids[:4]]]
    warm = _fresh(bk, n, edges, tw, [])
    try:
        bk.bkref_maxflow(warm)
        done = []
        for calls in steps:
            _calls(bk, warm, calls)
            done += calls
            e = bk.bkref_maxflow(warm)
            cold = _fresh(bk, n, edges, tw, done)
            try:
                ce = bk.bkref_maxflow(cold)
                assert _mask(bk, warm, n) == _mask(bk, cold, n)
                assert abs(e - ce) <= 1e-9 * max(abs(ce), 1.0)
            finally:
                bk.bkref_delete(cold)
    finally:
        bk.bkref_delete(warm)
