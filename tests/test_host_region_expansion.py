"""The region alpha-expansion oracle (oracle/region_expansion.py) against brute force on region graphs of up to 8
regions, its per-arc rules against the case table of DESIGN.md §11, and the argument checks of
``graphcut.expansion_from_labels`` through the Python layer with stand-ins for the native classes (the label image
double of tests/fake_native.py and a recorder of ``RegionExpansion`` that runs the oracle).  No GPU needed."""
import itertools
import math
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import energy_label_terms as elt  # noqa: E402
from oracle import region_expansion as orx  # noqa: E402
from oracle import solvers  # noqa: E402

import fake_native  # noqa: E402

SIZES = [(2, 0), (4, 1), (5, 2), (6, 3), (7, 4), (8, 5)]


def _graph(R, seed, K=3, integer=False):
    """Random pairs (ascending, distinct), weights and data costs; integer values make ties of the cut exact."""
    rng = numpy.random.default_rng(seed)
    all_pairs = [(a, b) for a in range(R) for b in range(a + 1, R)]
    keep = sorted(rng.choice(len(all_pairs), size=max(1, (2 * len(all_pairs)) // 3), replace=False))
    i = numpy.asarray([all_pairs[k][0] for k in keep], numpy.int32)
    j = numpy.asarray([all_pairs[k][1] for k in keep], numpy.int32)
    if integer:
        w = rng.integers(0, 4, size=i.size).astype(numpy.float64)
        D = rng.integers(0, 6, size=(K, R)).astype(numpy.float64)
    else:
        w = rng.random(i.size) * 1.5
        D = rng.random((K, R)) * 2.0
    return D, i, j, w


def _naive_energy(D, i, j, w, lab):
    e = [D[int(lab[r]), r] for r in range(lab.size)]
    e += [w[k] for k in range(i.size) if lab[i[k]] != lab[j[k]]]
    return math.fsum(e)


@pytest.mark.parametrize("R,seed", SIZES)
def test_energy_matches_enumeration(R, seed):
    D, i, j, w = _graph(R, seed)
    for flat in itertools.product(range(3), repeat=R):
        lab = numpy.asarray(flat, numpy.uint8)
        assert orx.energy(D, i, j, w, lab) == _naive_energy(D, i, j, w, lab)


@pytest.mark.parametrize("R,seed", SIZES)
@pytest.mark.parametrize("integer", [False, True])
def test_every_move_is_the_best_switch_set_and_its_cut_is_its_energy(R, seed, integer):
    D, i, j, w = _graph(R, seed, integer=integer)
    lab = numpy.argmin(D, axis=0).astype(numpy.uint8)
    for _ in range(3):
        for alpha in range(3):
            new, switched, cut = orx.move(D, i, j, w, lab, alpha)
            assert switched == int((new != lab).sum())
            e_new = orx.energy(D, i, j, w, new)
            assert abs(cut - e_new) <= 1e-12 * abs(e_new)
            free = numpy.flatnonzero(lab != alpha)
            best = math.inf
            for bits in itertools.product((0, 1), repeat=free.size):
                cand = lab.copy()
                cand[free[numpy.asarray(bits, bool)]] = alpha
                best = min(best, orx.energy(D, i, j, w, cand))
            assert abs(e_new - best) <= 1e-12 * abs(best)
            lab = new


@pytest.mark.parametrize("R,seed", SIZES)
def test_two_labels_reach_the_global_minimum_from_any_init(R, seed):
    D, i, j, w = _graph(R, seed, K=2)
    energies = {flat: orx.energy(D, i, j, w, numpy.asarray(flat, numpy.uint8))
                for flat in itertools.product(range(2), repeat=R)}
    best = min(energies.values())
    for flat in energies:
        r = orx.expansion(D, i, j, w, init=numpy.asarray(flat, numpy.uint8))
        assert r["converged"] and r["moves"] <= 4
        assert abs(r["energy"] - best) <= 1e-12 * abs(best)


@pytest.mark.parametrize("alpha", [0, 1, 2])
def test_per_arc_rules_are_the_case_table(alpha):
    """For every label pair of a region pair (p < q): the two ends' rules together charge what §11's table charges."""
    for lp, lq in itertools.product(range(3), repeat=2):
        snk_p, cap_pq = orx.arc_rules(lp, lq, 0, 1, alpha)      # p's arc to q
        snk_q, cap_qp = orx.arc_rules(lq, lp, 1, 0, alpha)      # q's arc to p
        if lp == alpha and lq == alpha:
            want = (False, False, False, False)
        elif lp == alpha or lq == alpha:                        # w to the non-alpha end's sink link
            want = (lq == alpha, lp == alpha, False, False)
        elif lp == lq:                                          # arcs p->q and q->p
            want = (False, False, True, True)
        else:                                                   # p's sink link, arc q->p
            want = (True, False, False, True)
        assert (bool(snk_p), bool(snk_q), bool(cap_pq), bool(cap_qp)) == want, (lp, lq, alpha)


def test_data_costs_are_bincount_sums_then_markers_in_ascending_order():
    rng = numpy.random.default_rng(3)
    lab = rng.integers(1, 6, size=(6, 7)).astype(numpy.int32)
    lab.flat[:5] = numpy.arange(1, 6)
    costs = rng.random((3, 6, 7)).astype(numpy.float32)
    markers = numpy.zeros(lab.shape, numpy.uint8)
    r0 = lab.flat[0] - 1
    markers[lab == lab.flat[0]] = 1
    markers.flat[0] = 3                                          # region r0 holds markers 1 and 3
    D = orx.data_costs(lab, costs, markers=markers)
    for k in range(3):
        plain = numpy.bincount(lab.ravel() - 1, weights=costs[k].ravel().astype(numpy.float64))
        seeded = plain.copy()
        if k != 0:
            seeded[r0] += orx.MAX
        if k != 2:
            seeded[r0] += orx.MAX
        assert numpy.array_equal(D[k], seeded)


def test_two_labels_give_graph_from_labels_cut():
    """The oracle at K = 2 against the binary region cut: t-links (D0, D1), bg -> sink, fg -> source, symmetric w."""
    lab = _labels((9, 11), 4, seed=7)
    R = int(lab.max())
    rng = numpy.random.default_rng(8)
    D = rng.random((2, R)) * 3.0
    i, j, w = _stawiaski_pairs(lab, rng.random(lab.shape).astype(numpy.float32) * 4)
    fg = numpy.zeros(lab.shape, bool)
    bg = numpy.zeros(lab.shape, bool)
    fg.flat[0] = True
    bg.flat[-1] = True
    markers = numpy.where(fg, 2, numpy.where(bg, 1, 0))
    Dm = orx.data_costs(lab, region_costs=D, markers=markers)
    r = orx.expansion(Dm, i, j, w)
    fgr, bgr = elt.marker_regions(lab, fg), elt.marker_regions(lab, bg)
    tw = [(numpy.arange(R), D[0], D[1]), (fgr, numpy.full(fgr.size, orx.MAX), numpy.zeros(fgr.size)),
          (bgr, numpy.zeros(bgr.size), numpy.full(bgr.size, orx.MAX))]
    flow, mask, _ = solvers.solve_sparse_port(R, i, j, w, w, tw)
    assert r["converged"] and numpy.array_equal(r["labels"], mask)
    assert abs(r["energy"] - flow) <= 1e-12 * abs(flow)


def _labels(shape, cell, seed):
    """A jittered grid of regions with ids exactly 1..R."""
    rng = numpy.random.default_rng(seed)
    idx = numpy.indices(shape)
    key = numpy.zeros(shape, numpy.int64)
    for g, s in zip(idx, shape):
        key = key * (s // cell + 2) + numpy.clip(g + rng.integers(-1, 2, size=shape), 0, s - 1) // cell
    _, inv = numpy.unique(key, return_inverse=True)
    return (inv + 1).reshape(shape).astype(numpy.int32)


def _stawiaski_pairs(lab, grad):
    lo, hi, a, _ = elt.merge_edges(*elt.stawiaski_calls(lab, grad))
    order = numpy.lexsort((hi, lo))
    return lo[order].astype(numpy.int32), hi[order].astype(numpy.int32), numpy.asarray(a, numpy.float64)[order]


# ---------------------------------------------------------------------------------------------------- the Python layer
class _Recorder:
    """Stands in for ``_mgc.RegionExpansion``: records every call, and runs the oracle."""
    made = []

    def __init__(self, regions, labels, device=-1):
        self.R, self.K, self.calls = regions, labels, []
        self.costs = [None] * labels
        self.pairs = (numpy.zeros(0, numpy.int32), numpy.zeros(0, numpy.int32), numpy.zeros(0))
        self.init = None
        _Recorder.made.append(self)

    def set_cost(self, k, c):
        self.calls.append("set_cost")
        self.costs[k] = numpy.array(c)

    def set_pairs(self, i, j, w):
        self.calls.append("set_pairs")
        self.pairs = (i, j, w)

    def set_init(self, init):
        self.calls.append("set_init")
        self.init = init

    def run(self, max_cycles):
        self.calls.append("run")
        self.r = orx.expansion(numpy.stack(self.costs), *self.pairs, init=self.init, max_cycles=max_cycles)

    def stats(self):
        return dict(moves=self.r["moves"], cycles=self.r["cycles"], converged=self.r["converged"],
                    switched=self.r["switched"], energy=self.r["energy"])

    def labels(self):
        return self.r["labels"]


@pytest.fixture
def native(monkeypatch):
    from medpy_b200 import _lib
    _Recorder.made = []
    monkeypatch.setattr(_lib._mgc, "LabelImage", fake_native.FakeLabelImage)
    monkeypatch.setattr(_lib._mgc, "RegionExpansion", _Recorder)
    return _Recorder


def _args():
    from medpy_b200.graphcut import energy_label
    lab = _labels((8, 9), 3, seed=2)
    rng = numpy.random.default_rng(5)
    costs = rng.random((3,) + lab.shape).astype(numpy.float32)
    grad = rng.random(lab.shape).astype(numpy.float32) * 3
    return lab, costs, energy_label.boundary_stawiaski, grad


def test_python_layer_runs_the_oracle_end_to_end(native):
    from medpy_b200 import graphcut
    lab, costs, term, grad = _args()
    markers = numpy.zeros(lab.shape, numpy.int32)
    markers[0, 0] = 3
    markers[-1, -1] = 1
    markers[-1, -2] = 2                                  # likely the same region as [-1, -1]: two markers
    labels, region_labels, energy, st = graphcut.expansion_from_labels(lab, costs, term, grad, markers=markers,
                                                                       stats=True)
    D = orx.data_costs(lab, costs, markers=markers)
    ref = orx.expansion(D, *_stawiaski_pairs(lab, grad))
    assert numpy.array_equal(region_labels, ref["labels"]) and energy == ref["energy"]
    assert numpy.array_equal(labels, ref["labels"][lab - 1]) and labels.dtype == numpy.uint8
    assert st["switched"] == ref["switched"] and region_labels[lab[0, 0] - 1] == 2
    assert native.made[0].calls == ["set_cost"] * 3 + ["set_pairs", "run"]


def test_region_costs_and_difference_of_means_reach_the_native_class(native):
    from medpy_b200 import graphcut
    from medpy_b200.graphcut import energy_label
    lab, costs, term, grad = _args()
    R = int(lab.max())
    rc = numpy.random.default_rng(9).random((4, R))
    init = numpy.arange(R) % 4
    labels, region_labels, energy = graphcut.expansion_from_labels(
        lab, None, energy_label.boundary_difference_of_means, grad, init=init, max_cycles=1, region_costs=rc)
    lo, hi, a, _ = elt.merge_edges(*elt.difference_of_means_calls(lab, grad))
    order = numpy.lexsort((hi, lo))
    ref = orx.expansion(rc, lo[order], hi[order], numpy.asarray(a, numpy.float64)[order], init=init, max_cycles=1)
    assert numpy.array_equal(region_labels, ref["labels"]) and energy == ref["energy"]
    assert native.made[0].calls == ["set_cost"] * 4 + ["set_pairs", "set_init", "run"]


def test_no_boundary_term_sets_no_pairs(native):
    from medpy_b200 import graphcut
    lab, costs, term, grad = _args()
    labels, region_labels, energy = graphcut.expansion_from_labels(lab, costs)
    D = orx.data_costs(lab, costs)
    assert numpy.array_equal(region_labels, numpy.argmin(D, axis=0))
    assert native.made[0].calls == ["set_cost"] * 3 + ["run"]


def _directed(graph, label_image, args):
    from medpy_b200.graphcut import energy_label
    energy_label.boundary_stawiaski_directed(graph, label_image, args)


def _twice(graph, label_image, grad):
    from medpy_b200.graphcut import energy_label
    energy_label.boundary_stawiaski(graph, label_image, grad)
    energy_label.boundary_stawiaski(graph, label_image, grad)


def _bad(lab, costs, term, grad):
    R = int(lab.max())
    shape = lab.shape
    broken = lab.copy()
    broken[broken == R] = R + 1                          # ids not consecutive
    return [
        (dict(costs=None), ValueError, "exactly one of costs and region_costs"),
        (dict(region_costs=numpy.zeros((3, R))), ValueError, "exactly one of costs and region_costs"),
        (dict(costs=costs.astype(numpy.int32)), ValueError, "float32 or float64"),
        (dict(costs=costs[:, :-1]), ValueError, "label_image.shape"),
        (dict(costs=costs[0]), ValueError, "label_image.shape"),
        (dict(costs=costs[:1]), ValueError, "2..255"),
        (dict(costs=numpy.where(costs > 0.5, numpy.nan, costs)), ValueError, "finite"),
        (dict(costs=numpy.where(costs > 0.5, numpy.inf, costs)), ValueError, "finite"),
        (dict(costs=costs - 1.0), ValueError, ">= 0"),
        (dict(costs=None, region_costs=numpy.zeros((3, R + 1))), ValueError, r"\(K, R\)"),
        (dict(costs=None, region_costs=numpy.zeros((3, R, 1))), ValueError, r"\(K, R\)"),
        (dict(costs=None, region_costs=numpy.full((3, R), -1.0)), ValueError, ">= 0"),
        (dict(costs=None, region_costs=numpy.zeros((3, R), numpy.float16)), ValueError, "float32 or float64"),
        (dict(boundary_term=lambda g, a: None), AttributeError, "three parameters"),
        (dict(boundary_term=42), AttributeError, "three parameters"),
        (dict(boundary_term=_directed, boundary_term_args=(grad, 0.4)), ValueError, "w_ij != w_ji"),
        (dict(boundary_term=_twice), ValueError, "more than one set"),
        (dict(markers=numpy.zeros((5, 5), numpy.uint8)), ValueError, "image shape"),
        (dict(markers=numpy.full(shape, 4, numpy.uint8)), ValueError, "0..3"),
        (dict(markers=numpy.full(shape, -1, numpy.int16)), ValueError, "0..3"),
        (dict(markers=numpy.zeros(shape, numpy.float32)), ValueError, "integers"),
        (dict(init=numpy.full(R, 3, numpy.uint8)), ValueError, "0..2"),
        (dict(init=numpy.zeros(R + 1, numpy.uint8)), ValueError, "one entry per region"),
        (dict(init=numpy.zeros(R, numpy.uint8), markers=numpy.full(shape, 2, numpy.uint8)), ValueError, "marker"),
        (dict(max_cycles=0), ValueError, "max_cycles"),
        (dict(max_cycles=1.5), ValueError, "max_cycles"),
        (dict(label_image=broken), AttributeError, "labeled consecutively"),
        (dict(label_image=lab - 1), AttributeError, "labeled consecutively"),
    ]


BAD_CASES = 28


def test_every_bad_case_is_listed():
    assert len(_bad(*_args())) == BAD_CASES


@pytest.mark.parametrize("case", range(BAD_CASES))
def test_bad_arguments_are_refused_before_the_native_class(native, case):
    from medpy_b200 import graphcut
    lab, costs, term, grad = _args()
    kw, exc, msg = _bad(lab, costs, term, grad)[case]
    call = dict(label_image=lab, costs=costs, boundary_term=term, boundary_term_args=grad)
    call.update(kw)
    with pytest.raises(exc, match=msg):
        graphcut.expansion_from_labels(**call)
    assert native.made == []


def test_a_region_holding_two_markers_accepts_either_init(native):
    from medpy_b200 import graphcut
    lab, costs, term, grad = _args()
    markers = numpy.zeros(lab.shape, numpy.uint8)
    r = lab[0, 0]
    markers[lab == r] = 1
    markers[0, 0] = 3
    for start in (0, 2):
        init = numpy.zeros(int(lab.max()), numpy.uint8)
        init[r - 1] = start
        graphcut.expansion_from_labels(lab, costs, term, grad, markers=markers, init=init)
    init[r - 1] = 1
    with pytest.raises(ValueError, match="marker"):
        graphcut.expansion_from_labels(lab, costs, term, grad, markers=markers, init=init)
