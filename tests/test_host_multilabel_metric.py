"""Alpha-expansion with a metric label distance (DESIGN.md §11, "Label distances"), without a GPU: the metric oracle
(tests/metric_oracle.py) against brute force on tiny lattices and region graphs, its reduction to the Potts oracles at
V = 1 - I bit for bit, K = 2 against enumeration, and ``label_distance`` of the three Python front ends through
recording stand-ins for the native classes."""
import itertools
import math
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import expansion as ox  # noqa: E402
from oracle import expansion_batch as oxb  # noqa: E402
from oracle import region_expansion as orx  # noqa: E402

import fake_native  # noqa: E402
import metric_oracle as mo  # noqa: E402

TINY = [((8,), 0), ((7,), 1), ((2, 4), 2), ((3, 2), 3), ((2, 3), 4)]
REGIONS = [(4, 1), (6, 3), (8, 5)]
KINDS = ["truncated_linear", "random", "scaled_potts", "pseudo"]


def _metric(kind, K, seed=0):
    if kind == "truncated_linear":
        return mo.truncated_linear(K, 1.5)
    if kind == "random":
        return mo.random_metric(K, 100 + seed)
    if kind == "scaled_potts":
        return mo.scaled_potts(K, 0.7)
    return mo.pseudo_metric(K)


def _voxel_problem(shape, seed, K):
    rng = numpy.random.default_rng(seed)
    costs = rng.random((K,) + shape) * 2.0
    image = rng.random(shape).astype(numpy.float32) * 3.0
    markers = numpy.zeros(shape, numpy.uint8)
    markers.flat[0] = 1 + seed % K
    return costs, ("difference_exponential", image, 0.8, False), markers


def _region_graph(R, seed, K):
    rng = numpy.random.default_rng(seed)
    all_pairs = [(a, b) for a in range(R) for b in range(a + 1, R)]
    keep = sorted(rng.choice(len(all_pairs), size=max(1, (2 * len(all_pairs)) // 3), replace=False))
    i = numpy.asarray([all_pairs[k][0] for k in keep], numpy.int32)
    j = numpy.asarray([all_pairs[k][1] for k in keep], numpy.int32)
    return rng.random((K, R)) * 2.0, i, j, rng.random(i.size) * 1.5


@pytest.mark.parametrize("K", [3, 4, 5, 17])
@pytest.mark.parametrize("kind", KINDS)
def test_the_matrices_are_metrics(kind, K):
    assert mo.is_metric(_metric(kind, K))


@pytest.mark.parametrize("kind", KINDS)
def test_pair_table_cuts_w_times_v_of_every_outcome(kind):
    """The 2 x 2 check: keep/keep pays lo + up, keep/switch lo + fwd, switch/keep up + bwd, switch/switch nothing; every
    entry >= 0."""
    K = 5
    V = _metric(kind, K)
    w = 1.37
    for a, b, alpha in itertools.product(range(K), repeat=3):
        lo, up, fwd, bwd = (float(x) for x in mo.pair_terms(w, V, a, b, alpha))
        assert min(lo, up, fwd, bwd) >= 0.0
        for got, want in [(lo + up, w * V[a, b]), (lo + fwd, w * V[a, alpha]), (up + bwd, w * V[alpha, b])]:
            assert abs(got - want) <= 1e-15 * max(1.0, want), (a, b, alpha)


@pytest.mark.parametrize("shape,seed", TINY)
@pytest.mark.parametrize("K", [3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_every_voxel_move_is_the_best_expansion_and_its_cut_is_its_energy(shape, seed, K, kind):
    costs, boundary, markers = _voxel_problem(shape, seed, K)
    V = _metric(kind, K, seed)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    lab = ox.initial_labels(D, shape)
    for _ in range(2):
        for alpha in range(K):
            new, switched, cut = mo.move(D, w, lab, alpha, V)
            assert switched == int((new != lab).sum())
            e_new = mo.energy(D, w, new, V)
            assert abs(cut - e_new) <= 1e-12 * abs(e_new)
            free = numpy.flatnonzero(lab.ravel() != alpha)
            best = math.inf
            for bits in itertools.product((0, 1), repeat=free.size):
                cand = lab.copy().ravel()
                cand[free[numpy.asarray(bits, bool)]] = alpha
                best = min(best, mo.energy(D, w, cand.reshape(shape), V))
            assert abs(e_new - best) <= 1e-12 * abs(best)
            lab = new


@pytest.mark.parametrize("R,seed", REGIONS)
@pytest.mark.parametrize("K", [3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_every_region_move_is_the_best_expansion_and_its_cut_is_its_energy(R, seed, K, kind):
    D, i, j, w = _region_graph(R, seed, K)
    V = _metric(kind, K, seed)
    lab = numpy.argmin(D, axis=0).astype(numpy.uint8)
    for _ in range(2):
        for alpha in range(K):
            new, switched, cut = mo.region_move(D, i, j, w, lab, alpha, V)
            assert switched == int((new != lab).sum())
            e_new = mo.region_energy(D, i, j, w, new, V)
            assert abs(cut - e_new) <= 1e-12 * abs(e_new)
            free = numpy.flatnonzero(lab != alpha)
            best = math.inf
            for bits in itertools.product((0, 1), repeat=free.size):
                cand = lab.copy()
                cand[free[numpy.asarray(bits, bool)]] = alpha
                best = min(best, mo.region_energy(D, i, j, w, cand, V))
            assert abs(e_new - best) <= 1e-12 * abs(best)
            lab = new


@pytest.mark.parametrize("kind", KINDS)
def test_batch_model_runs_each_image_as_the_single_oracle(kind):
    B, K, shape = 3, 4, (3, 4)
    rng = numpy.random.default_rng(11)
    costs = rng.random((B, K) + shape) * 2.0
    for b in range(B):
        costs[b] = costs[b] * (1.0 - 0.3 * b) + 0.3 * b
    images = (rng.random((B,) + shape) * 3.0).astype(numpy.float32)
    boundaries = [("difference_exponential", images[b], 0.4 + 0.3 * b, False) for b in range(B)]
    V = _metric(kind, K)
    r = mo.expansion_batch(costs, boundaries, V=V)
    for b in range(B):
        ref = mo.expansion(costs[b], boundaries[b], V=V)
        assert numpy.array_equal(r["labels"][b], ref["labels"]) and r["energies"][b] == ref["energy"]
        assert r["switched"][b] == ref["switched"] and r["cycles"][b] == ref["cycles"]


# ------------------------------------------------------------------------------------------ V = 1 - I is Potts, bitwise
def _bits(x):
    return numpy.ascontiguousarray(x, numpy.float64).view(numpy.uint64)


@pytest.mark.parametrize("shape,seed", TINY + [((5, 6, 7), 9), ((3, 4, 5, 6), 10)])
@pytest.mark.parametrize("K", [3, 4])
def test_potts_matrix_gives_the_potts_voxel_move_graphs_bit_for_bit(shape, seed, K):
    costs, boundary, markers = _voxel_problem(shape, seed, K)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    rng = numpy.random.default_rng(seed)
    V = 1.0 - numpy.eye(K)
    for _ in range(3):
        lab = rng.integers(0, K, size=shape).astype(numpy.uint8)
        for alpha in range(K):
            p, m = ox.move_problem(D, w, lab, alpha), mo.move_problem(D, w, lab, alpha, V)
            assert numpy.array_equal(_bits(p["tr"]), _bits(m["tr"]))
            assert _bits(p["flow_const"]) == _bits(m["flow_const"])
            for d in range(len(shape)):
                assert numpy.array_equal(_bits(p["wf"][d]), _bits(m["wf"][d]))
                assert numpy.array_equal(_bits(p["wb"][d]), _bits(m["wb"][d]))


@pytest.mark.parametrize("R,seed", REGIONS + [(30, 7)])
@pytest.mark.parametrize("K", [3, 4])
def test_potts_matrix_gives_the_potts_region_move_graphs_bit_for_bit(R, seed, K):
    D, i, j, w = _region_graph(R, seed, K)
    rng = numpy.random.default_rng(seed)
    V = 1.0 - numpy.eye(K)
    for _ in range(3):
        lab = rng.integers(0, K, size=R).astype(numpy.uint8)
        for alpha in range(K):
            (pe, pt), (me, mt) = orx.move_problem(D, i, j, w, lab, alpha), mo.region_move_problem(D, i, j, w, lab, alpha, V)
            for x, y in zip(pe[2:] + pt[1:], me[2:] + mt[1:]):
                assert numpy.array_equal(_bits(x), _bits(y))


def test_potts_matrix_runs_are_the_potts_runs():
    K = 4
    V = 1.0 - numpy.eye(K)
    costs, boundary, markers = _voxel_problem((6, 7), 3, K)
    a, b = ox.expansion(costs, boundary, markers), mo.expansion(costs, boundary, markers, V=V)
    assert numpy.array_equal(a["labels"], b["labels"]) and a["switched"] == b["switched"]
    assert a["energy"] == b["energy"] and a["cuts"] == b["cuts"]
    D, i, j, w = _region_graph(12, 4, K)
    a, b = orx.expansion(D, i, j, w), mo.region_expansion(D, i, j, w, V=V)
    assert numpy.array_equal(a["labels"], b["labels"]) and a["switched"] == b["switched"] and a["energy"] == b["energy"]
    bc = numpy.stack([costs, costs[::-1]])
    a, b = oxb.expansion_batch(bc, [boundary, boundary]), mo.expansion_batch(bc, [boundary, boundary], V=V)
    assert numpy.array_equal(a["labels"], b["labels"]) and numpy.array_equal(a["matrix"], b["matrix"])
    assert numpy.array_equal(a["energies"], b["energies"])


# ----------------------------------------------------------------------------------------------------------------- K = 2
@pytest.mark.parametrize("shape,seed", TINY)
@pytest.mark.parametrize("s", [0.7, 0.0])
def test_two_labels_reach_the_global_minimum_from_any_init(shape, seed, s):
    costs, boundary, markers = _voxel_problem(shape, seed, 2)
    V = mo.scaled_potts(2, s)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    n = int(numpy.prod(shape))
    energies = {flat: mo.energy(D, w, numpy.asarray(flat, numpy.uint8).reshape(shape), V)
                for flat in itertools.product(range(2), repeat=n)}
    best = min(energies.values())
    m = markers.ravel()
    for flat in energies:
        init = numpy.asarray(flat, numpy.uint8).reshape(shape)
        if ((m > 0) & (init.ravel() != m - 1)).any():
            continue
        r = mo.expansion(costs, boundary, markers, init=init, V=V)
        assert r["converged"] and r["moves"] <= 4
        assert abs(r["energy"] - best) <= 1e-12 * abs(best)


@pytest.mark.parametrize("R,seed", REGIONS)
def test_two_labels_reach_the_global_minimum_of_a_region_graph_from_any_init(R, seed):
    D, i, j, w = _region_graph(R, seed, 2)
    V = mo.scaled_potts(2, 1.3)
    energies = {flat: mo.region_energy(D, i, j, w, numpy.asarray(flat, numpy.uint8), V)
                for flat in itertools.product(range(2), repeat=R)}
    best = min(energies.values())
    for flat in energies:
        r = mo.region_expansion(D, i, j, w, init=numpy.asarray(flat, numpy.uint8), V=V)
        assert r["converged"] and r["moves"] <= 4
        assert abs(r["energy"] - best) <= 1e-12 * abs(best)


# ---------------------------------------------------------------------------------------------------- the Python layer
class _Recorder:
    """Stands in for the three native expansion classes: records every call (with the label distance it was given) and
    runs the metric oracle."""
    made = []

    def __init__(self, unit, *args):
        self.unit, self.calls, self.V = unit, [], None
        self.K = args[-2] if unit != "voxel" else args[1]
        self.costs = [None] * self.K
        self.boundary = self.markers = self.init = None
        self.pairs = (numpy.zeros(0, numpy.int32), numpy.zeros(0, numpy.int32), numpy.zeros(0))
        _Recorder.made.append(self)

    def set_cost(self, k, c):
        self.calls.append("set_cost")
        self.costs[k] = numpy.array(c)

    def set_boundary(self, *args):
        self.calls.append("set_boundary")

    def set_pairs(self, i, j, w):
        self.calls.append("set_pairs")
        self.pairs = (i, j, w)

    def set_markers(self, m):
        self.calls.append("set_markers")
        self.markers = m

    def set_init(self, i):
        self.calls.append("set_init")
        self.init = i

    def set_label_distance(self, V):
        self.calls.append("set_label_distance")
        assert V.dtype == numpy.float64 and V.flags.c_contiguous and V.shape == (self.K, self.K)
        self.V = V

    def run(self, max_cycles):
        self.calls.append("run")
        if self.unit == "voxel":
            self.r = mo.expansion(numpy.stack(self.costs), None, self.markers, self.init, max_cycles, V=self.V)
        elif self.unit == "batch":
            self.r = mo.expansion_batch(numpy.stack(self.costs, axis=1), None, self.markers, self.init, max_cycles,
                                        V=self.V)
        else:
            self.r = mo.region_expansion(numpy.stack(self.costs), *self.pairs, init=self.init, max_cycles=max_cycles,
                                         V=self.V)

    def stats(self):
        r = self.r
        if self.unit == "batch":
            return dict(moves=r["batch_moves"], cycles=r["batch_cycles"], converged=r["batch_converged"],
                        energy=float(r["energies"].sum()), ms_build=0.0, ms_solve=0.0, ms_apply=0.0, ms_total=0.0)
        return dict(moves=r["moves"], cycles=r["cycles"], converged=r["converged"], switched=r["switched"],
                    energy=r["energy"])

    def image_stats(self):
        r = self.r
        return dict(moves=numpy.asarray(r["moves"]), cycles=numpy.asarray(r["cycles"]),
                    converged=numpy.asarray(r["converged"]), energy=r["energies"])

    def switched(self):
        return self.r["matrix"]

    def labels(self):
        return self.r["labels"]


@pytest.fixture
def native(monkeypatch):
    from medpy_b200 import _lib
    _Recorder.made = []
    monkeypatch.setattr(_lib._mgc, "Expansion", lambda *a: _Recorder("voxel", *a))
    monkeypatch.setattr(_lib._mgc, "ExpansionBatch", lambda *a: _Recorder("batch", *a))
    monkeypatch.setattr(_lib._mgc, "RegionExpansion", lambda *a: _Recorder("region", *a))
    monkeypatch.setattr(_lib._mgc, "LabelImage", fake_native.FakeLabelImage)
    return _Recorder


K4 = 4


def _call(unit, **kw):
    """One front-end call on a small K = 4 problem: the voxel image, a batch of two, or the regions of a label image."""
    from medpy_b200 import graphcut
    rng = numpy.random.default_rng(21)
    if unit == "voxel":
        return graphcut.expansion_from_voxels(rng.random((K4, 5, 6)).astype(numpy.float32), stats=True, **kw)
    if unit == "batch":
        return graphcut.expansion_from_voxels_batch(rng.random((2, K4, 5, 6)), stats=True, **kw)
    lab = numpy.repeat(numpy.repeat(numpy.arange(1, 7, dtype=numpy.int32).reshape(2, 3), 3, 0), 3, 1)
    return graphcut.expansion_from_labels(lab, rng.random((K4,) + lab.shape), stats=True, **kw)


def _refused():
    V = mo.truncated_linear(K4, 2.0)
    nan, inf, neg, diag, asym = (V.copy() for _ in range(5))
    nan[1, 2] = numpy.nan
    inf[3, 0] = numpy.inf
    neg[2, 1] = -0.5
    diag[2, 2] = 0.25
    asym[0, 3] += 0.125
    i = numpy.arange(K4)
    quad = numpy.minimum((i[:, None] - i[None, :]) ** 2, 9)
    return [
        (numpy.zeros((K4, K4 + 1)), r"\(K, K\) = \(4, 4\)"),
        (numpy.zeros((3, 3)), r"\(K, K\) = \(4, 4\)"),
        (nan, r"finite and >= 0, V\[1\]\[2\] is not"),
        (inf, r"finite and >= 0, V\[3\]\[0\] is not"),
        (neg, r"finite and >= 0, V\[2\]\[1\] is not"),
        (diag, r"zero diagonal, V\[2\]\[2\] is not 0"),
        (asym, r"symmetric, V\[0\]\[3\] != V\[3\]\[0\]"),
        (quad, r"triangle inequality .*\(a, b, c\) = \(0, 1, 2\) breaks it; .*truncated quadratic"),
        (numpy.full((K4, K4), "x"), "real numbers"),
    ]


@pytest.mark.parametrize("case", range(9))
@pytest.mark.parametrize("unit", ["voxel", "batch", "region"])
def test_a_refused_matrix_is_refused_before_the_native_class(native, unit, case):
    V, msg = _refused()[case]
    with pytest.raises(ValueError, match=msg):
        _call(unit, label_distance=V)
    assert native.made == []


@pytest.mark.parametrize("unit", ["voxel", "batch", "region"])
def test_no_matrix_never_calls_set_label_distance(native, unit):
    _call(unit)
    _call(unit, label_distance=None)
    assert len(native.made) == 2
    assert all("set_label_distance" not in r.calls and r.V is None for r in native.made)


@pytest.mark.parametrize("unit", ["voxel", "batch", "region"])
def test_a_matrix_reaches_the_native_class_as_float64_before_the_run(native, unit):
    V = mo.truncated_linear(K4, 2.0)
    out = _call(unit, label_distance=V.astype(numpy.int64).tolist())        # a nested sequence of integers
    rec = native.made[0]
    assert rec.calls[-2:] == ["set_label_distance", "run"]
    assert numpy.array_equal(rec.V, V)
    energy = out[-2]
    if unit == "batch":
        assert numpy.array_equal(energy, rec.r["energies"])
    else:
        assert energy == rec.r["energy"]
