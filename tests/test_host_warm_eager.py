"""GraphDouble.enable_warm() on the host: the opt-in that lets eager, per-term and 4-D lattice graphs fold seeds and t-link
calls into their solved state (MGC_OPT_WARM) -- when it reaches the native handle, the order against build and solve, the
errors, staging before the first solve and persistence across reset() -- and, with the real reference BK, the claim the
warm fold rests on extended to 4-D lattices: solve, add_tweights, solve again == a fresh solve of all calls."""
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_native  # noqa: E402
from test_host_erase_seeds import _calls, _fresh, _mask  # noqa: E402
from test_host_seeds import _reference_bk  # noqa: E402


class _OptGraph(fake_native.FakeGraph):
    """FakeGraph that keeps its options and refuses MGC_OPT_WARM changes once a solve has started, like the native handle
    (which accepts them on a lazily built handle: `lazy`)."""

    lazy = False

    def __init__(self, shape, device=-1):
        self.options = {}
        self.option_calls = []
        self.flow_started = False
        self.folds = []
        super().__init__(shape, device)

    def reset(self):
        super().reset()
        self.flow_started = False          # the options stay, as MGC_OPT_DEFER_WEIGHT_CHECK and MGC_OPT_WARM do

    def set_option(self, option, value):
        from medpy_b200 import _lib
        if option == _lib._mgc.OPT_WARM and bool(value) != bool(self.options.get(option, 0)) and self.flow_started \
                and not self.lazy:
            raise RuntimeError("MGC_OPT_WARM is set before the first solve")
        self.option_calls.append((option, value))
        self.options[option] = value

    def maxflow(self):
        self.flow_started = True
        return super().maxflow()

    def add_seeds(self, fg_ids, bg_ids):
        self.folds.append(("add_seeds", fg_ids, bg_ids))
        self.result = None

    def add_tweights_warm(self, ids, src, snk):
        self.folds.append(("add_tweights_warm", ids, src, snk))
        self.result = None


@pytest.fixture()
def made(monkeypatch):
    from medpy_b200 import _lib
    out = []

    def factory(shape, device=-1):
        g = _OptGraph(shape, device)
        out.append(g)
        return g
    monkeypatch.setattr(_lib, "Graph", factory)
    return out


def _warm_opt():
    from medpy_b200 import _lib
    return _lib._mgc.OPT_WARM


def _voxel_graph(shape=(6, 7, 8), seed=0):
    import medpy_b200.graphcut as gc
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=seed)
    return gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                                regional_term_args=(vol["prob"], vol["alpha"]),
                                boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                boundary_term_args=(vol["image"], vol["sigma"], False))


def test_option_id():
    from medpy_b200 import _lib
    assert _lib._mgc.OPT_WARM == 2 and _lib._mgc.OPT_DEFER_WEIGHT_CHECK == 1


@pytest.mark.parametrize("shape", [(6, 7, 8), (4, 5, 6, 3)])
def test_built_unsolved_graph_sets_the_option(made, shape):
    """graph_from_voxels returns a built, unsolved graph: enable_warm() reaches its handle at once."""
    g = _voxel_graph(shape)
    assert (_warm_opt(), 1) not in made[0].option_calls
    g.enable_warm()
    assert made[0].options[_warm_opt()] == 1
    g.maxflow()
    g.enable_warm()                        # no change: accepted after the solve too
    assert len(made) == 1


def test_option_waits_for_the_handle(made):
    """Before anything needs the device there is no handle: the option is set when _nat() creates it, before any term."""
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(12, 11)
    g.enable_warm()
    assert made == []
    g.add_tweights(0, 5.0, 0.0)
    g.add_tweights(11, 0.0, 5.0)
    g.sum_edge(0, 1, 1.0, 1.0)
    assert made == []
    g.maxflow()
    assert made[0].option_calls[0] == (_warm_opt(), 1)


def test_after_the_first_solve_raises_naming_the_order(made):
    g = _voxel_graph()
    g.maxflow()
    with pytest.raises(RuntimeError, match=r"enable_warm\(\) before the first maxflow\(\); reset\(\)"):
        g.enable_warm()
    assert not g._warm and _warm_opt() not in made[0].options


def test_lazily_built_solved_graph_accepts_it(made):
    """A graph the lazy fused build made folds without the option: setting it late changes nothing and raises nothing."""
    _OptGraph.lazy = True
    try:
        g = _voxel_graph()
        g.maxflow()
        g.enable_warm()
        assert made[0].options[_warm_opt()] == 1
    finally:
        _OptGraph.lazy = False


def test_survives_reset(made):
    g = _voxel_graph()
    g.enable_warm()
    g.maxflow()
    g.reset()
    assert g._warm and made[0].options[_warm_opt()] == 1
    g.add_tweights(3, 2.0, 0.0)
    g.maxflow()
    g.add_seeds([3], None)
    assert made[0].folds and made[0].folds[-1][0] == "add_seeds"
    assert len(made) == 1


def test_calls_before_the_first_solve_are_staged(made):
    """With the option on, seeds and t-link calls before the first maxflow() are staged as before: nothing folds."""
    g = _voxel_graph()
    ref = _voxel_graph()
    g.enable_warm()
    g.add_seeds([3, 4], [9])
    g.add_tweights_warm(numpy.array([3, 7, 3]), numpy.array([1.0, -2.0, 0.5]), 1.0)
    ref.add_seeds([3, 4], [9])
    ref.add_tweights_warm(numpy.array([3, 7, 3]), numpy.array([1.0, -2.0, 0.5]), 1.0)
    assert g.maxflow() == ref.maxflow()
    assert made[0].folds == [] and numpy.array_equal(made[0].tr, made[1].tr)
    g.add_tweights_warm([5], 1.0, 0.0)
    assert made[0].folds[-1][0] == "add_tweights_warm"


def test_sparse_graph_raises_type_error():
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(4, 4, sparse=True)
    with pytest.raises(TypeError):
        g.enable_warm()


def _lattice4(seed):
    """A random 4-D lattice (8-connected, as the reference treats an n-D volume) with t-links of both kinds."""
    rng = numpy.random.default_rng(seed)
    shape = (3, 4, 3, 5)
    n = int(numpy.prod(shape))
    strides = (60, 15, 5, 1)
    edges = []
    for v in range(n):
        c = numpy.unravel_index(v, shape)
        for d in range(4):
            if c[d] + 1 < shape[d]:
                edges.append((v, v + strides[d], float(rng.uniform(0.01, 2.0)), float(rng.uniform(0.01, 2.0))))
    tw = [(v, float(rng.uniform(0, 3)), float(rng.uniform(0, 3))) for v in range(n)]
    return rng, n, edges, tw


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_reference_bk_4d_resolve_after_add_tweights_equals_from_scratch(seed):
    """Pinned on the unmodified reference BK on 4-D lattices: after maxflow(), seeds, erased seeds and add_tweights with
    random reals of both signs (repeated ids, mixed signs on one voxel, a dense pass), then maxflow() again, give the min
    cut of the graph with the whole call sequence."""
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    rng, n, edges, tw = _lattice4(seed)
    ids = rng.integers(0, n, 10).tolist()
    v = int(rng.integers(0, n))
    dense = rng.normal(0, 2, n) * (rng.random(n) < 0.5)
    steps = [[(i, 65535.0, 0.0) for i in ids[:3]] + [(i, 0.0, 65535.0) for i in ids[3:5]],     # seeds
             [(i, -65535.0, 0.0) for i in ids[:2]],                                            # erase
             [(i, float(rng.uniform(-4, 4)), float(rng.uniform(-4, 4))) for i in ids + [v, v]],
             [(i, float(dense[i]), float(-dense[i] / 2)) for i in range(n)]]
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
