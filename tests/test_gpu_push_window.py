"""Label window of the push passes on easy instances: each colour's push launch takes only the listed tiles whose lowest
active label is within a window of the list's lowest, defers the other active tiles and drops tiles without an active
voxel.  The mask must stay the reference BK's, at sizes where the window really defers tiles (at 64^3 it covers almost
every tile), under the solver options that change the schedule around it, after seeds added to a windowed solve, and
on an instance whose excess has to travel far before it reaches a sink."""
import os

import numpy
import pytest

pytestmark = pytest.mark.gpu


class _env:
    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kw}
        for k, v in self.kw.items():
            os.environ[k] = str(v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _need_ref():
    from oracle import solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")


def _graph(vol):
    import medpy_b200.graphcut as gc
    return gc.graph_from_voxels(vol["fg"], vol["bg"],
                                regional_term=gc.energy_voxel.regional_probability_map,
                                regional_term_args=(vol["prob"], vol["alpha"]),
                                boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                boundary_term_args=(vol["image"], vol["sigma"], False))


def _problem(vol):
    from oracle import energy_terms as et
    return et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))


def _ref(vol):
    from oracle import solvers
    oe, om, _ = solvers.solve_ref(_problem(vol))
    return oe, om


def _assert_ref(e, m, oe, om):
    assert int((m != om).sum()) == 0, ("mask differs from the reference BK", int((m != om).sum()))
    assert abs(e - oe) <= 1e-9 * abs(oe), (e, oe)


@pytest.mark.parametrize("env", [{}, dict(MEDPY_GC_FIRST_TEST=1), dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_LAZY_CAPS=0)],
                         ids=["default", "first_test", "full_reset", "eager"])
@pytest.mark.parametrize("size", [128, 192])
def test_config3_windowed_solve_matches_reference_bk(size, env):
    _need_ref()
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume((size,) * 3, seed=0)
    with _env(**env):
        g = _graph(vol)
        e = g.maxflow()
        m = g.get_mask()
        st = g.stats()
    assert st["tiles_deferred"] > 0 and st["tiles_dropped"] > 0, st
    oe, om = _ref(vol)
    _assert_ref(e, m, oe, om)


def test_background_seed_inside_the_foreground_after_a_windowed_solve():
    """The window drops ball-interior tiles whose source excess was never materialised; a background ball seeded inside
    the foreground must still drain it.  Warm result = cold rebuild = reference BK."""
    _need_ref()
    from medpy_b200 import synthetic
    from oracle import energy_terms as et, solvers
    shape = (128, 128, 128)
    vol = synthetic.two_blob_volume(shape, seed=1)
    carve = numpy.flatnonzero(synthetic._ball_mask(shape, (0.3,), 0.05, min_radius=1.0))
    g = _graph(vol)
    g.maxflow()
    assert g.stats()["tiles_dropped"] > 0
    g.add_seeds(None, carve)
    e, m = g.maxflow(), g.get_mask().copy()

    cold = _graph(vol)
    cold.add_seeds(None, carve)
    ce, cm = cold.maxflow(), cold.get_mask()
    assert numpy.array_equal(m, cm), int((m != cm).sum())
    assert abs(e - ce) <= 1e-12 * abs(ce) + 1e-10, (e, ce)

    # the reference BK on the from-scratch graph: the final t-links as one dense pass, the constant added here
    prob = _problem(vol)
    seeded = numpy.zeros(prob["tr"].size, bool)
    seeded[carve] = True
    prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], 0.0, 65535.0, where=seeded)
    ref = dict(prob, src=numpy.maximum(prob["tr"], 0.0), snk=numpy.maximum(-prob["tr"], 0.0),
               fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool))
    oe, om, _ = solvers.solve_ref(ref)
    _assert_ref(e, m, oe + prob["flow_const"], om)


def test_excess_that_travels_far_converges():
    """A long tube of foreground in a background with sink links everywhere, the tube's only sink links at one end: once
    the weak arcs across the tube wall are saturated, the rest of the tube's excess has to travel along it to that end,
    through many label windows."""
    _need_ref()
    from medpy_b200 import synthetic
    shape = (64, 64, 512)
    rng = numpy.random.default_rng(7)
    image = rng.normal(0.0, 10.0, size=shape).astype(numpy.float32)
    tube = numpy.zeros(shape, bool)
    tube[28:36, 28:36, 8:504] = True
    image[tube] += 100.0
    prob = numpy.full(shape, 0.2, numpy.float32)
    prob[tube] = 0.51                        # a weak source link: most of the tube's excess is needed at the far end
    prob[28:36, 28:36, 8:16] = 0.05          # the tube's sink links: its first 8 voxels
    vol = dict(image=image, prob=prob, alpha=0.1, fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool),
               sigma=synthetic.rms_neighbour_difference(image))
    g = _graph(vol)
    e = g.maxflow()
    m = g.get_mask()
    st = g.stats()
    assert st["tiles_deferred"] > 0, st
    oe, om = _ref(vol)
    _assert_ref(e, m, oe, om)
