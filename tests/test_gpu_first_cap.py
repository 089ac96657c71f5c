"""Label cap of the first global relabel of an easy solve: no stop test reads that relabel, only the label window of round
1's push passes, so the BFS stops at FIRST_RELABEL_CAP and tiles whose excess sits deeper wait for the next, exact,
relabel instead of leaving the lists.  The mask must stay the reference BK's under the solver options that change the
schedule around it, the capped relabel must run fewer BFS passes than the exact one, and an instance whose sources all
lie deeper than the cap (round 1 pushes nothing) must still converge to BK's cut."""
import numpy
import pytest

from test_gpu_push_window import _assert_ref, _env, _graph, _need_ref, _ref

pytestmark = pytest.mark.gpu

_ENVS = [{}, dict(MEDPY_GC_FIRST_TEST=1), dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_LAZY_CAPS=0),
         dict(MEDPY_GC_FIRST_CAP=0)]


def _solve(vol, **env):
    with _env(**env):
        g = _graph(vol)
        e = g.maxflow()
        return e, g.get_mask().copy(), g.stats()


@pytest.mark.parametrize("env", _ENVS, ids=["default", "first_test", "full_reset", "eager", "cap_off"])
@pytest.mark.parametrize("size", [128, 192])
def test_config3_capped_first_relabel_matches_reference_bk(size, env):
    _need_ref()
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume((size,) * 3, seed=0)
    e, m, st = _solve(vol, **env)
    assert st["relabel_passes"] >= st["relabel_passes_first"] > 0, st
    assert 0 < st["ms_relabel_first"] <= st["ms_relabel"], st
    oe, om = _ref(vol)
    _assert_ref(e, m, oe, om)


@pytest.mark.parametrize("size", [128, 192])
def test_capped_first_relabel_runs_fewer_passes(size):
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume((size,) * 3, seed=0)
    e_on, m_on, on = _solve(vol)
    e_off, m_off, off = _solve(vol, MEDPY_GC_FIRST_CAP=0)
    _, _, tested = _solve(vol, MEDPY_GC_FIRST_TEST=1)      # a stop test reads the first relabel: it stays exact
    assert on["relabel_passes_first"] < off["relabel_passes_first"], (on, off)
    assert tested["relabel_passes_first"] == off["relabel_passes_first"], (tested, off)
    assert numpy.array_equal(m_on, m_off)
    assert abs(e_on - e_off) <= 1e-9 * abs(e_off), (e_on, e_off)


def _deep_source_volume(shape, core, shell):
    """Sink links everywhere but in a corner block: a core of source links [0, core)^3 inside a shell of voxels without
    t-links (probability 0.5) up to [0, core + shell)^3.  Every source voxel is more than `shell` arcs from a sink link."""
    rng = numpy.random.default_rng(3)
    image = rng.normal(0.0, 10.0, size=shape).astype(numpy.float32)
    prob = numpy.full(shape, 0.2, numpy.float32)
    out = core + shell
    prob[:out, :out, :out] = 0.5
    prob[:core, :core, :core] = 0.9
    image[:out, :out, :out] += 30.0
    from medpy_b200 import synthetic
    return dict(image=image, prob=prob, alpha=0.1, fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool),
                sigma=synthetic.rms_neighbour_difference(image))


@pytest.mark.parametrize("env", [{}, dict(MEDPY_GC_FIRST_CAP=24), dict(MEDPY_GC_LAZY_CAPS=0), dict(MEDPY_GC_FIRST_CAP=0)],
                         ids=["default", "cap24", "eager", "cap_off"])
def test_sources_deeper_than_the_cap_converge(env):
    """The capped first relabel labels no source voxel: round 1 pushes nothing and defers every listed tile, and the exact
    relabel of round 2 takes over."""
    _need_ref()
    vol = _deep_source_volume((128, 128, 128), core=8, shell=32)
    e, m, st = _solve(vol, **env)
    assert st["global_relabels"] >= 2, st
    oe, om = _ref(vol)
    _assert_ref(e, m, oe, om)
