"""Differential matrix of the 4-D tile solver (the 4 x 4 x 8 x 4 tiles of gc_tiles4.cuh): every lattice_cases4 instance
under every solver option that changes how a 4-D instance is relabelled (classification, sweeps, sweep rounds) or how
long a tile visit runs.  Each cell must give BK's mask (bit for bit on integer instances; a float mismatch only with an
exact-tie certificate), BK's energy (exactly on integer instances), an energy equal to the exact capacity of its own cut
and an ended solve.

The statistics also show which relabel ran: every relabel adds 1 to `global_relabels` and 1 to `relabel_sweeps` for its
cooperative BFS launch, and each directional sweep round adds 1 more to `relabel_sweeps`.  Sweeps run on instances of at
least 64 tiles that are hard, by default or forced."""
import pytest

import lattice_cases as lc
import lattice_cases4 as l4
from test_gpu_push_window import _env
from test_gpu_solver_matrix import _assert_energy, _assert_mask, _build

pytestmark = pytest.mark.gpu

OPTIONS = {
    "default": {},
    "easy": dict(MEDPY_GC_SWEEP_FRAC=1),
    "hard": dict(MEDPY_GC_SWEEP_FRAC=1000000),
    "sweep_off": dict(MEDPY_GC_SWEEP=0),
    "sweep_rounds": dict(MEDPY_GC_SWEEP_FRAC=1000000, MEDPY_GC_SWEEP_MIN_ROUNDS=3, MEDPY_GC_SWEEP_ROUNDS=4),
    "iters1": dict(MEDPY_GC_ITERS=1, MEDPY_GC_PASSES_MAX=1),
    "debug": dict(MEDPY_GC_DEBUG=1),
}

CELLS = [(name, opt) for name in l4.CASES for opt in OPTIONS]

_case = {}


def _get(name):
    """The instance, kept only while its cells run (instance-major order)."""
    if name not in _case:
        _case.clear()
        _case[name] = l4.make(name)
    return _case[name]


def _sweeps_expected(case, opt):
    """Whether the relabels of this cell run directional sweeps: at least 64 tiles, sweeps on, and a hard instance."""
    if l4.tiles4(case["prob"]["shape"]) < 64 or opt == "sweep_off":
        return False
    if opt in ("hard", "sweep_rounds"):
        return True
    return opt != "easy" and not case["easy"]


@pytest.mark.parametrize("name,opt", CELLS, ids=["%s-%s" % c for c in CELLS])
def test_cell_matches_bk(name, opt):
    case = _get(name)
    with _env(**OPTIONS[opt]):
        g = _build(case)
        e = g.maxflow()
        m = g.get_mask()
        st = g.stats()
    e_bk, m_bk = lc.bk(case)
    _assert_mask(case, m, e_bk, m_bk)
    _assert_energy(case, e, e_bk)
    ref = lc.bk_ref(case)
    if ref is not None:
        _assert_mask(case, m, ref[0], ref[1])
        _assert_energy(case, e, ref[0])
    # the energy is the capacity of the solver's own cut, summed exactly over the oracle's float64 capacities
    _assert_energy(case, e, lc.cut_capacity(case["prob"], m))
    assert st["active_last"] == 0, st

    if not _sweeps_expected(case, opt):
        assert st["relabel_passes"] > 0, st     # where sweeps run they may leave the BFS nothing to do
    if _sweeps_expected(case, opt):
        assert st["relabel_sweeps"] > st["global_relabels"], st
    else:
        assert st["relabel_sweeps"] == st["global_relabels"], st
    if opt == "sweep_rounds" and _sweeps_expected(case, opt):
        # every relabel of a hard instance has tiles to label, and runs 3 rounds before its first fixed-point check
        assert st["relabel_sweeps"] >= 4 * st["global_relabels"], st


def test_iters_sets_the_first_round_too():
    """MEDPY_GC_ITERS sets the iterations of every tile visit, the first round's included.  A chain of 4 voxels along
    axis 3 inside one tile, a source link of 1 at one end and a sink link of 2 at the other: the first relabel labels the
    chain 4, 3, 2, 1, and each iteration moves the unit of excess one arc.  With 1 iteration per visit and 1 pass per
    round, the excess needs 4 rounds, and the fifth relabel's stop test ends the solve; with the first round's default
    of 4 iterations it would be absorbed in round 1 and the second relabel would end it."""
    import numpy
    import medpy_b200.graphcut as gc
    shape = (1, 1, 1, 4)
    t = numpy.array([1.0, 0.0, 0.0, -2.0]).reshape(shape)
    arcs = [numpy.ones(tuple(s - 1 if d == e else s for e, s in enumerate(shape))) for d in range(4)]
    case = l4._dense("chain", "I", shape, t, arcs, arcs, exact=True)
    for env, relabels in ((dict(MEDPY_GC_ITERS=1, MEDPY_GC_PASSES_MAX=1), 5), (dict(MEDPY_GC_ITERS=4, MEDPY_GC_PASSES_MAX=1), 2)):
        with _env(**env):
            graph = gc.GCGraph(4, 16, shape=shape)
            graph.set_tweights_dense(case["src"], case["snk"])
            graph.set_nweights_dense(3, arcs[3], arcs[3])
            g = graph.get_graph()
            e = g.maxflow()
            st = g.stats()
        e_bk, m_bk = lc.bk(case)
        assert e == e_bk == 1.0 and numpy.array_equal(numpy.ravel(g.get_mask()), numpy.ravel(m_bk)), (e, e_bk)
        assert st["global_relabels"] == relabels and st["active_last"] == 0, (env, st)
