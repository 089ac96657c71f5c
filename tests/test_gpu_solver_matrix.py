"""Differential matrix of the 3-D tile solver: every lattice_cases instance under every solver option that changes how an
easy instance is scheduled (label window, capped first relabel, lazy push state, partial relabel reset) or which kernel of
a pair runs.  Each cell must give BK's mask (bit for bit; integer instances also the exact energy), an energy equal to the
exact capacity of its own cut, an ended solve, and -- where the instance is built for it -- show that the targeted code
ran.  Warm re-solves after add_seeds are checked on the ladders and tubes under the options that change their schedule."""
import numpy
import pytest

import lattice_cases as lc
from test_gpu_fullsize import _cut_difference_exact
from test_gpu_push_window import _env
from test_gpu_seeds import _replay

pytestmark = pytest.mark.gpu

OPTIONS = {
    "default": {},
    "first_cap0": dict(MEDPY_GC_FIRST_CAP=0),
    "first_cap2": dict(MEDPY_GC_FIRST_CAP=2),
    "first_cap13": dict(MEDPY_GC_FIRST_CAP=13),
    "first_test": dict(MEDPY_GC_FIRST_TEST=1),
    "full_reset": dict(MEDPY_GC_PARTIAL_RESET=0),
    "eager": dict(MEDPY_GC_LAZY_CAPS=0),
    "no_tma": dict(MEDPY_GC_TMA=0),
    "iters1": dict(MEDPY_GC_ITERS=1, MEDPY_GC_PASSES_MAX=1),
    "easy": dict(MEDPY_GC_SWEEP_FRAC=1),
    "hard": dict(MEDPY_GC_SWEEP_FRAC=1000000),
    "debug": dict(MEDPY_GC_DEBUG=1),
    "easy_cap0": dict(MEDPY_GC_SWEEP_FRAC=1, MEDPY_GC_FIRST_CAP=0),     # only read by the `easy` cells
}


def _applies(name, opt):
    # the dense per-term path builds the push state eagerly whatever MEDPY_GC_LAZY_CAPS says
    return opt != "easy_cap0" and not (opt == "eager" and lc.family(name).startswith("B"))


CELLS = [(name, opt) for name in lc.CASES for opt in OPTIONS if _applies(name, opt)]

_case = {}
_solved = {}


def _get(name):
    """The instance, kept only while its cells run (instance-major order)."""
    if name not in _case:
        _case.clear()
        _case[name] = lc.make(name)
    return _case[name]


def _build(case):
    """The case's graph through graph_from_voxels (fused; difference_exponential unless the case names another boundary
    term) or the dense per-term calls, in as many dimensions as the case has."""
    import medpy_b200.graphcut as gc
    if case["kind"] == "fused":
        vol = case["vol"]
        kw = dict(boundary_term=getattr(gc.energy_voxel, "boundary_" + case.get("boundary", "difference_exponential")),
                  boundary_term_args=(vol["image"], vol["sigma"], False))
        if vol.get("prob") is not None:
            kw.update(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=(vol["prob"], vol["alpha"]))
        return gc.graph_from_voxels(vol["fg"], vol["bg"], **kw)
    shape = tuple(case["prob"]["shape"])
    n = int(numpy.prod(shape))
    graph = gc.GCGraph(n, len(shape) * n, shape=shape)
    graph.set_tweights_dense(case["src"], case["snk"])
    for d in range(len(shape)):
        graph.set_nweights_dense(d, case["there"][d], case["back"][d])
    return graph.get_graph()


def _solve(name, opt):
    """(energy, mask, stats) of one GPU solve, cached per cell (the default cell also reads the cap-off one)."""
    key = (name, opt)
    if key not in _solved:
        with _env(**OPTIONS[opt]):
            g = _build(_get(name))
            e = g.maxflow()
            _solved[key] = (e, g.get_mask().copy(), g.stats())
    return _solved[key]


def _assert_mask(case, m, e_bk, m_bk):
    """The mask must be BK's.  Integer instances have no excuse; a float instance may only differ by an exact tie: the
    two cuts' capacities equal to below half an ulp of the energy, measured in exact arithmetic."""
    differing = int((m != m_bk).sum())
    if differing and not case["exact"]:
        diff = _cut_difference_exact(case["prob"], m, m_bk)
        assert abs(diff) <= 0.5 * numpy.spacing(abs(e_bk)), ("mask differs from BK's by more than a tie", differing, diff)
    else:
        assert differing == 0, ("mask differs from BK's", differing)


def _assert_energy(case, e, e_bk):
    if case["exact"]:
        assert e == e_bk, (e, e_bk)
    else:
        assert abs(e - e_bk) <= 1e-9 * abs(e_bk), (e, e_bk)


@pytest.mark.parametrize("name,opt", CELLS, ids=["%s-%s" % c for c in CELLS])
def test_cell_matches_bk(name, opt):
    case = _get(name)
    e, m, st = _solve(name, opt)
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

    # the targeted code ran: on the instances built to be easy under the default options, and on every instance whose
    # classification is forced easy
    fam = case["family"]
    if (opt == "default" and case["easy"]) or opt == "easy":
        if fam in ("A1", "A2", "B2"):
            assert st["tiles_deferred"] > 0, st
        if fam == "A1":
            assert st["tiles_dropped"] > 0, st
            # every ladder has a rung deeper than the cap: the capped relabel leaves it to a second, exact one, and runs
            # fewer BFS passes than the exact one.  A pass relabels whole 8^3 tiles, so labels 12 and 14 can take the same
            # number of passes: where the deepest rung (13) lies just beyond the cap the counts may be equal, and the
            # first_cap2 cell shows the cap cutting passes on that ladder instead
            assert st["global_relabels"] >= 2, st
            off = _solve(name, "first_cap0" if opt == "default" else "easy_cap0")[2]
            if max(s for s, _ in case["rungs"]) >= 2 * lc.CAP:
                assert st["relabel_passes_first"] < off["relabel_passes_first"], (st, off)
            else:
                assert st["relabel_passes_first"] <= off["relabel_passes_first"], (st, off)
        if fam == "A5":
            assert st["tiles_deferred"] + st["tiles_dropped"] > 0, st
    if opt == "first_cap2" and fam == "A1" and case["easy"]:
        # a cap of 2 stops the first relabel after the labels next to the sinks, well before the exact BFS ends
        off = _solve(name, "first_cap0")[2]
        assert st["relabel_passes_first"] < off["relabel_passes_first"], (st, off)
        assert st["tiles_deferred"] > 0, st
    if opt == "hard":
        assert st["tiles_deferred"] == 0 and st["tiles_dropped"] == 0, st
    if opt == "first_cap0":
        _solved.pop((name, "default"), None)
    if opt != "default":
        for o in (opt, "first_cap0", "easy_cap0"):
            _solved.pop((name, o), None)


# --------------------------------------------------------------------------------------------------------- warm seeds
WARM_CASES = ["a1-ladder-s0", "a1-ladder-s2", "a2-serp-w3"]
WARM_OPTIONS = ["default", "first_cap2", "full_reset", "no_tma", "iters1"]


def _steps(case):
    """Refinement 1: background seeds inside the deepest core, foreground seeds where the excess stays (the tiles the
    window drops).  Refinement 2: foreground seeds on sink-side background, background seeds on half of the first
    foreground seeds."""
    s = case["seeds"]
    return [(s["stuck"], s["deep"]), (s["far"], s["stuck"][::2])]


def _oracle(case, done):
    from oracle import solvers
    prob = dict(case["prob"], tr=case["prob"]["tr"].copy())
    _replay(prob, done)
    return solvers.solve_port(prob)[:2]


def _cold(case, done):
    g = _build(case)
    for fg, bg in done:
        g.add_seeds(numpy.asarray(fg, numpy.int64), numpy.asarray(bg, numpy.int64))
    return g.maxflow(), g.get_mask()


@pytest.mark.parametrize("opt", WARM_OPTIONS)
@pytest.mark.parametrize("name", WARM_CASES)
def test_warm_refinements_match_from_scratch(name, opt):
    case = _get(name)
    with _env(**OPTIONS[opt]):
        g = _build(case)
        g.maxflow()
        done = []
        for fg, bg in _steps(case):
            g.add_seeds(numpy.asarray(fg, numpy.int64), numpy.asarray(bg, numpy.int64))
            done.append((fg, bg))
            e, m = g.maxflow(), g.get_mask()
            oe, om = _oracle(case, done)
            assert numpy.array_equal(m, om), ("warm mask differs from the oracle", len(done), int((m != om).sum()))
            assert abs(e - oe) <= 1e-9 * max(abs(oe), 1.0), (len(done), e, oe)
            ce, cm = _cold(case, done)
            assert numpy.array_equal(m, cm), ("warm mask differs from the cold rebuild", len(done))
            assert abs(e - ce) <= 1e-12 * max(abs(ce), 1.0) + 1e-10, (len(done), e, ce)
            assert g.stats()["active_last"] == 0
        assert g.stats()["seed_folds"] == len(done)
