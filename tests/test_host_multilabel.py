"""The alpha-expansion oracle (oracle/expansion.py) against brute force on tiny lattices and against the binary path, and
the argument checks of ``graphcut.expansion_from_voxels`` through the Python layer with a recording stand-in for the
native class.  No GPU needed."""
import itertools
import math

import numpy
import pytest

from oracle import energy_terms as et
from oracle import expansion as ox
from oracle import solvers

TINY = [((8,), 0), ((7,), 1), ((2, 4), 2), ((3, 2), 3), ((2, 3), 4)]


def _problem(shape, seed, K=3, with_markers=False):
    rng = numpy.random.default_rng(seed)
    costs = rng.random((K,) + shape) * 2.0
    image = rng.random(shape).astype(numpy.float32) * 3.0
    boundary = ("difference_exponential", image, 0.8, False)
    markers = None
    if with_markers:
        markers = numpy.zeros(shape, numpy.uint8)
        markers.flat[0] = 1 + seed % K
    return costs, boundary, markers


def _naive_energy(D, w, lab):
    """E by loops over voxels and pairs."""
    e = [D[int(lab.flat[p]), p] for p in range(lab.size)]
    for d, wd in enumerate(w):
        for idx in numpy.ndindex(wd.shape):
            q = list(idx)
            q[d] += 1
            if lab[idx] != lab[tuple(q)]:
                e.append(wd[idx])
    return math.fsum(e)


@pytest.mark.parametrize("shape,seed", TINY)
def test_energy_matches_enumeration(shape, seed):
    costs, boundary, markers = _problem(shape, seed, with_markers=True)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    n = int(numpy.prod(shape))
    for flat in itertools.product(range(3), repeat=n):
        lab = numpy.asarray(flat, numpy.uint8).reshape(shape)
        assert ox.energy(D, w, lab) == _naive_energy(D, w, lab)


@pytest.mark.parametrize("shape,seed", TINY)
@pytest.mark.parametrize("with_markers", [False, True])
def test_every_move_is_the_best_switch_set_and_its_cut_is_its_energy(shape, seed, with_markers):
    costs, boundary, markers = _problem(shape, seed, with_markers=with_markers)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    lab = ox.initial_labels(D, shape)
    for _ in range(3):
        for alpha in range(3):
            new, switched, cut = ox.move(D, w, lab, alpha)
            assert switched == int(((new != lab)).sum())
            e_new = ox.energy(D, w, new)
            assert abs(cut - e_new) <= 1e-12 * abs(e_new)
            free = numpy.flatnonzero(lab.ravel() != alpha)
            best = math.inf
            for bits in itertools.product((0, 1), repeat=free.size):
                cand = lab.copy().ravel()
                cand[free[numpy.asarray(bits, bool)]] = alpha
                best = min(best, ox.energy(D, w, cand.reshape(shape)))
            assert abs(e_new - best) <= 1e-12 * abs(best)
            lab = new


@pytest.mark.parametrize("shape,seed", TINY)
def test_two_labels_reach_the_global_minimum_from_any_init(shape, seed):
    costs, boundary, markers = _problem(shape, seed, K=2, with_markers=True)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    n = int(numpy.prod(shape))
    energies = {flat: ox.energy(D, w, numpy.asarray(flat, numpy.uint8).reshape(shape))
                for flat in itertools.product(range(2), repeat=n)}
    best = min(energies.values())
    m = markers.ravel()
    for flat in energies:
        init = numpy.asarray(flat, numpy.uint8).reshape(shape)
        if ((m > 0) & (init.ravel() != m - 1)).any():
            continue
        r = ox.expansion(costs, boundary, markers, init=init)
        assert r["converged"] and r["moves"] <= 4
        assert abs(r["energy"] - best) <= 1e-12 * abs(best)


@pytest.mark.parametrize("kind", et.BOUNDARY_KINDS)
@pytest.mark.parametrize("shape", [(6, 7), (4, 5, 6)])
def test_two_labels_give_the_binary_cut(kind, shape):
    rng = numpy.random.default_rng(len(kind) + len(shape))
    prob = rng.random(shape)
    alpha = 0.7
    image = (rng.random(shape) * 5).astype(numpy.float32)
    fg = numpy.zeros(shape, bool)
    bg = numpy.zeros(shape, bool)
    fg.flat[3] = True
    bg.flat[-2] = True
    sigma = None if kind.endswith("linear") else 1.3
    boundary = (kind, image, sigma, False)
    costs = numpy.stack([prob * alpha, (1 - prob) * alpha])
    markers = numpy.where(fg, 2, numpy.where(bg, 1, 0)).astype(numpy.uint8)
    r = ox.expansion(costs, boundary, markers)
    flow, mask, _ = solvers.solve_port(et.build_problem(fg, bg, regional=(prob, alpha), boundary=boundary))
    assert abs(r["energy"] - flow) <= 1e-9 * abs(flow)
    assert r["converged"]


# ---------------------------------------------------------------------------------------------------- the Python layer
class _Recorder:
    """Stands in for ``_mgc.Expansion``: records every call, and runs the oracle."""
    made = []

    def __init__(self, shape, labels, device=-1):
        self.shape, self.K, self.calls = tuple(shape), labels, []
        self.costs = [None] * labels
        self.boundary = self.markers = self.init = None
        _Recorder.made.append(self)

    def set_cost(self, k, c):
        self.calls.append("set_cost")
        self.costs[k] = numpy.asarray(c)

    def set_boundary(self, kind, image, sigma, spacing, norm):
        self.calls.append("set_boundary")
        self.boundary = (et.BOUNDARY_KINDS[kind], image, sigma, spacing if spacing else False)

    def set_markers(self, m):
        self.calls.append("set_markers")
        self.markers = m

    def set_init(self, i):
        self.calls.append("set_init")
        self.init = i

    def run(self, max_cycles):
        self.calls.append("run")
        self.r = ox.expansion(numpy.stack(self.costs), self.boundary, self.markers, self.init, max_cycles)

    def stats(self):
        return dict(moves=self.r["moves"], cycles=self.r["cycles"], converged=self.r["converged"],
                    switched=self.r["switched"], energy=self.r["energy"])

    def labels(self):
        return self.r["labels"]


@pytest.fixture
def native(monkeypatch):
    from medpy_b200 import _lib
    _Recorder.made = []
    monkeypatch.setattr(_lib._mgc, "Expansion", _Recorder)
    return _Recorder


def _args():
    from medpy_b200.graphcut import energy_voxel as ev
    rng = numpy.random.default_rng(5)
    costs = rng.random((3, 5, 6)).astype(numpy.float32)
    image = rng.random((5, 6)).astype(numpy.float32)
    return costs, ev.boundary_difference_exponential, (image, 0.5, (1.0, 2.0))


def test_python_layer_runs_the_oracle_end_to_end(native):
    from medpy_b200 import graphcut
    costs, term, args = _args()
    markers = numpy.zeros((5, 6), numpy.int32)
    markers[0, 0] = 3
    labels, energy, st = graphcut.expansion_from_voxels(costs, term, args, markers=markers, stats=True)
    ref = ox.expansion(costs, ("difference_exponential", args[0], 0.5, [1.0, 2.0]), markers)
    assert numpy.array_equal(labels, ref["labels"]) and energy == ref["energy"]
    assert st["switched"] == ref["switched"] and labels[0, 0] == 2
    assert native.made[0].calls == ["set_cost"] * 3 + ["set_boundary", "set_markers", "run"]


def _bad(costs, term, args):
    shape = costs.shape[1:]
    return [
        (dict(costs=costs.astype(numpy.int32)), ValueError, "float32 or float64"),
        (dict(costs=costs[:1]), ValueError, "2..255"),
        (dict(costs=numpy.zeros((256, 2, 2), numpy.float32)), ValueError, "2..255"),
        (dict(costs=numpy.zeros((2, 1, 1, 1, 1, 1), numpy.float32)), ValueError, "1- to 4-D"),
        (dict(costs=numpy.where(costs > 0.5, numpy.nan, costs)), ValueError, "finite"),
        (dict(costs=numpy.where(costs > 0.5, numpy.inf, costs)), ValueError, "finite"),
        (dict(costs=costs - 1.0), ValueError, ">= 0"),
        (dict(boundary_term=lambda g: None), AttributeError, "two parameters"),
        (dict(boundary_term=42), AttributeError, "two parameters"),
        (dict(markers=numpy.zeros((5, 5), numpy.uint8)), ValueError, "image shape"),
        (dict(markers=numpy.full(shape, 4, numpy.uint8)), ValueError, "0..3"),
        (dict(markers=numpy.full(shape, -1, numpy.int16)), ValueError, "0..3"),
        (dict(markers=numpy.zeros(shape, numpy.float32)), ValueError, "integers"),
        (dict(init=numpy.full(shape, 3, numpy.uint8)), ValueError, "0..2"),
        (dict(init=numpy.zeros(shape, numpy.uint8), markers=numpy.full(shape, 2, numpy.uint8)), ValueError, "marker"),
        (dict(max_cycles=0), ValueError, "max_cycles"),
        (dict(max_cycles=1.5), ValueError, "max_cycles"),
    ]


@pytest.mark.parametrize("case", range(17))
def test_bad_arguments_are_refused_before_the_native_class(native, case):
    from medpy_b200 import graphcut
    costs, term, args = _args()
    kw, exc, msg = _bad(costs, term, args)[case]
    call = dict(costs=costs, boundary_term=term, boundary_term_args=args)
    call.update(kw)
    with pytest.raises(exc, match=msg):
        graphcut.expansion_from_voxels(**call)
    assert native.made == []


def test_max_cycles_and_init_reach_the_native_class(native):
    from medpy_b200 import graphcut
    costs, term, args = _args()
    init = numpy.zeros((5, 6), numpy.int64)
    labels, energy, st = graphcut.expansion_from_voxels(costs, init=init, max_cycles=1, stats=True)
    ref = ox.expansion(costs, None, None, init, 1)
    assert native.made[0].calls == ["set_cost"] * 3 + ["set_init", "run"]
    assert st["moves"] == 3 and st["cycles"] == 1 and numpy.array_equal(labels, ref["labels"])
