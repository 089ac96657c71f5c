"""GraphDouble.remove_seeds on the host: argument handling (masks to ids in logical C order, order and duplicates kept, id
range, shapes), the staged path before the first solve -- and, with the real reference BK, the semantic claim the warm
erase rests on: solve, add_tweights with negative capacities, solve again == from scratch."""
import os
import sys

import numpy
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_native  # noqa: E402
from test_host_seeds import _reference_bk  # noqa: E402


class _EraseGraph(fake_native.FakeGraph):
    """FakeGraph plus add_seeds / remove_seeds: replays the calls on the from-scratch t-links."""

    def __init__(self, shape, device=-1):
        super().__init__(shape, device)
        self.seed_calls = []

    def _fold(self, kind, fg_ids, bg_ids, cap):
        from oracle import energy_terms as et
        self.seed_calls.append((kind, fg_ids, bg_ids))
        for ids, s, t in ((fg_ids, cap, 0.0), (bg_ids, 0.0, cap)):
            if ids is None:
                continue
            ids = numpy.asarray(ids)
            assert ids.dtype == numpy.int64 and ids.ndim == 1
            for v in ids.tolist():
                self.flow = et.add_tweights_pass(self.tr, self.flow, s, t, where=numpy.arange(self.n) == v)
        self.result = None

    def add_seeds(self, fg_ids, bg_ids):
        self._fold("add", fg_ids, bg_ids, 65535.0)

    def remove_seeds(self, fg_ids, bg_ids):
        self._fold("remove", fg_ids, bg_ids, -65535.0)


@pytest.fixture()
def made(monkeypatch):
    from medpy_b200 import _lib
    out = []

    def factory(shape, device=-1):
        g = _EraseGraph(shape, device)
        out.append(g)
        return g
    monkeypatch.setattr(_lib, "Graph", factory)
    return out


def _graph(shape=(6, 7, 8), seed=0):
    import medpy_b200.graphcut as gc
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=seed)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(vol["prob"], vol["alpha"]),
                             boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    return g, vol


def test_fortran_mask_gives_c_order_ids(made):
    g, _ = _graph()
    g.maxflow()
    m = numpy.zeros((6, 7, 8), bool)
    m[1, 2, 3] = m[4, 0, 7] = m[0, 6, 0] = True
    g.remove_seeds(fg=numpy.asfortranarray(m), bg=m[::-1][::-1])
    kind, fg, bg = made[0].seed_calls[-1]
    assert kind == "remove"
    assert fg.tolist() == [0 * 56 + 6 * 8 + 0, 1 * 56 + 2 * 8 + 3, 4 * 56 + 0 * 8 + 7]
    assert bg.tolist() == fg.tolist()


def test_ids_keep_order_and_duplicates(made):
    g, _ = _graph()
    g.maxflow()
    g.remove_seeds(fg=[5, 3, 5], bg=numpy.array([7, 7], numpy.int32))
    kind, fg, bg = made[0].seed_calls[-1]
    assert kind == "remove" and fg.tolist() == [5, 3, 5] and bg.tolist() == [7, 7]
    g.remove_seeds(fg=torch.tensor([9, 9]), bg=torch.zeros((6, 7, 8), dtype=torch.bool))
    kind, fg, bg = made[0].seed_calls[-1]
    assert kind == "remove" and fg.tolist() == [9, 9] and bg.tolist() == []


def test_bad_arguments(made):
    g, _ = _graph()
    g.maxflow()
    n = 6 * 7 * 8
    with pytest.raises(ValueError, match="Invalid node id of {} or 0. Valid values are 0 to {}.".format(n, n - 1)):
        g.remove_seeds(fg=[0, n])
    with pytest.raises(ValueError, match="Invalid node id"):
        g.remove_seeds(bg=[-1])
    with pytest.raises(ValueError, match="shape"):
        g.remove_seeds(fg=numpy.zeros((6, 7), bool))
    with pytest.raises(ValueError):
        g.remove_seeds(fg=numpy.zeros((2, 2), numpy.int64))
    with pytest.raises(ValueError):
        g.remove_seeds(bg=[1.5])
    assert made[0].seed_calls == []
    g.remove_seeds()
    assert made[0].seed_calls[-1] == ("remove", None, None)


def test_sparse_graph_refusal_says_rebuild_without_the_seeds():
    from medpy_b200.graphcut import GCGraph
    g = GCGraph(4, 4, sparse=True).get_graph()
    g._solved = True            # stands for a solved graph: the sparse solve itself needs the device
    with pytest.raises(RuntimeError, match="reset.*without the seeds"):
        g.remove_seeds(fg=[1])
    with pytest.raises(RuntimeError, match="reset.*with the seeds"):
        g.add_seeds(fg=[1])


def test_warm_erase_equals_from_scratch(made):
    """Add a stroke, solve, erase it (and a marker, and a seed never added), solve: the fake's from-scratch replay of the
    same add_tweights sequence is what the warm path must give."""
    from oracle import energy_terms as et, solvers
    g, vol = _graph()
    g.maxflow()
    marker = int(numpy.flatnonzero(vol["fg"])[0])
    g.add_seeds(fg=[100, 101], bg=[5])
    g.maxflow()
    g.remove_seeds(fg=[100, 101, marker], bg=[5, 9])
    e, m = g.maxflow(), g.get_mask()
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    for ids, s, t in (([100, 101], 65535.0, 0.0), ([5], 0.0, 65535.0), ([100, 101, marker], -65535.0, 0.0),
                      ([5, 9], 0.0, -65535.0)):
        for v in ids:
            prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], s, t,
                                                      where=numpy.arange(prob["tr"].size) == v)
    oe, om, _ = solvers.solve_port(prob)
    assert numpy.array_equal(m, om) and abs(e - oe) <= 1e-9 * abs(oe)


def test_unsolved_graph_stages_negative_add_tweights(made):
    """Before the first maxflow() remove_seeds is add_tweights with -65535: the staged dense pass carries it."""
    g, _ = _graph()
    ref, _ = _graph()
    g.add_seeds(fg=[3], bg=[4])
    g.remove_seeds(fg=[3, 3], bg=[4])
    ref.add_tweights(3, 65535.0, 0.0)
    ref.add_tweights(4, 0.0, 65535.0)
    for v in (3, 3):
        ref.add_tweights(v, -65535.0, 0.0)
    ref.add_tweights(4, 0.0, -65535.0)
    assert made[0].seed_calls == [] and g.maxflow() == ref.maxflow()
    assert numpy.array_equal(g.get_mask(), ref.get_mask())
    assert numpy.array_equal(made[0].tr, made[1].tr) and made[0].flow == made[1].flow


def _lattice(bk, seed):
    rng = numpy.random.default_rng(seed)
    shape = (5, 6, 7)
    n = int(numpy.prod(shape))
    strides = (42, 7, 1)
    edges = []
    for v in range(n):
        c = numpy.unravel_index(v, shape)
        for d in range(3):
            if c[d] + 1 < shape[d]:
                edges.append((v, v + strides[d], float(rng.uniform(0.01, 2.0)), float(rng.uniform(0.01, 2.0))))
    tw = [(v, float(rng.uniform(0, 3)), float(rng.uniform(0, 3))) for v in range(n)]
    return rng, n, edges, tw


def _calls(bk, h, calls):
    for v, s, t in calls:
        bk.bkref_add_tweights(h, v, s, t)


def _fresh(bk, n, edges, tw, calls):
    h = bk.bkref_new(n, len(edges))
    for i, j, a, b in edges:
        bk.bkref_sum_edge(h, i, j, a, b)
    _calls(bk, h, [(v, a, b) for v, a, b in tw])
    _calls(bk, h, calls)
    return h


def _mask(bk, h, n):
    return [bk.bkref_what_segment(h, v) for v in range(n)]


def _seed_calls(fg, bg, cap):
    return [(v, cap, 0.0) for v in fg] + [(v, 0.0, cap) for v in bg]


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_reference_bk_resolve_after_erase_equals_from_scratch(seed):
    """The claim the warm erase rests on, pinned on the unmodified reference BK: after maxflow(), add_tweights with
    -65535 on seeds (added before, never added, repeated, in both lists) and maxflow() again give the min cut of the
    graph with that call sequence (same mask, same energy as a fresh solve)."""
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    rng, n, edges, tw = _lattice(bk, seed)
    added = (rng.integers(0, n, 6).tolist(), rng.integers(0, n, 6).tolist())
    v = int(rng.integers(0, n))
    steps = [_seed_calls(added[0], added[1], 65535.0),
             _seed_calls(added[0][:3], added[1][:2], -65535.0),
             _seed_calls(rng.integers(0, n, 3).tolist() + [v, v, v], [v] + rng.integers(0, n, 2).tolist(), -65535.0),
             _seed_calls(added[0][3:], added[1][2:], -65535.0) + _seed_calls([v], [], 65535.0)]
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


@pytest.mark.parametrize("seed", [4, 5, 6])
def test_reference_bk_erasing_every_added_seed_restores_the_graph(seed):
    """Erasing every seed that was added gives back the original graph's mask and energy."""
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    rng, n, edges, tw = _lattice(bk, seed)
    fg, bg = rng.integers(0, n, 8).tolist(), rng.integers(0, n, 8).tolist()
    h = _fresh(bk, n, edges, tw, [])
    try:
        e0 = bk.bkref_maxflow(h)
        m0 = _mask(bk, h, n)
        _calls(bk, h, _seed_calls(fg, bg, 65535.0))
        bk.bkref_maxflow(h)
        _calls(bk, h, _seed_calls(fg[::-1], bg[::-1], -65535.0))
        e = bk.bkref_maxflow(h)
        assert _mask(bk, h, n) == m0
        assert abs(e - e0) <= 1e-9 * abs(e0)
    finally:
        bk.bkref_delete(h)
