"""Alpha-beta swap moves (DESIGN.md §11, "Swap moves"), without a GPU: the swap oracle (tests/swap_oracle.py) against
enumeration on tiny lattices and region graphs under Potts, truncated linear, truncated quadratic and a random
semi-metric; K = 2 against the global minimum; the batch model against per-image runs; and ``moves`` of the three Python
front ends through recording stand-ins for the native classes."""
import itertools
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import expansion as ox  # noqa: E402

import fake_native  # noqa: E402
import metric_oracle as mo  # noqa: E402
import swap_oracle as so  # noqa: E402

TINY = [((8,), 0), ((7,), 1), ((2, 4), 2), ((3, 2), 3), ((2, 3), 4)]
REGIONS = [(4, 1), (6, 3), (8, 5)]
KINDS = ["potts", "truncated_linear", "truncated_quadratic", "random"]


def _dist(kind, K, seed=0):
    if kind == "potts":
        return None
    if kind == "truncated_linear":
        return mo.truncated_linear(K, 2.0)
    if kind == "truncated_quadratic":
        return so.truncated_quadratic(K, 4.0)
    return so.random_semi_metric(K, 200 + seed)


def _V(kind, K, seed=0):
    V = _dist(kind, K, seed)
    return 1.0 - numpy.eye(K) if V is None else V


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


@pytest.mark.parametrize("K", [3, 4, 5])
def test_the_matrices_are_semi_metrics_and_two_break_the_triangle(K):
    for kind in KINDS:
        assert so.is_semi_metric(_V(kind, K))
    assert not mo.is_metric(so.truncated_quadratic(K, 4.0))
    assert not mo.is_metric(so.random_semi_metric(K, 3))


def _best_swap(lab, alpha, beta, energy):
    """The lowest energy over every relabelling of the participants to alpha or beta."""
    flat = lab.ravel()
    part = numpy.flatnonzero((flat == alpha) | (flat == beta))
    best = numpy.inf
    for bits in itertools.product((alpha, beta), repeat=part.size):
        cand = flat.copy()
        cand[part] = bits
        best = min(best, energy(cand.reshape(lab.shape)))
    return best


@pytest.mark.parametrize("shape,seed", TINY)
@pytest.mark.parametrize("K", [3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_every_voxel_move_is_the_best_swap_and_its_cut_is_its_energy(shape, seed, K, kind):
    costs, boundary, markers = _voxel_problem(shape, seed, K)
    V = _dist(kind, K, seed)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    lab = ox.initial_labels(D, shape)
    energy = lambda l: mo.energy(D, w, l, V)      # noqa: E731
    for _ in range(2):
        for alpha, beta in so.pairs(K):
            new, switched, cut = so.move(D, w, lab, alpha, beta, V)
            assert switched == int((new != lab).sum())
            assert numpy.array_equal(new == lab, ~(((lab == alpha) | (lab == beta)) & (new != lab)))
            e_new = energy(new)
            assert abs(cut + so.fixed_energy(D, w, lab, alpha, beta, V) - e_new) <= 1e-12 * abs(e_new)
            assert abs(e_new - _best_swap(lab, alpha, beta, energy)) <= 1e-12 * abs(e_new)
            lab = new


@pytest.mark.parametrize("R,seed", REGIONS)
@pytest.mark.parametrize("K", [3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_every_region_move_is_the_best_swap_and_its_cut_is_its_energy(R, seed, K, kind):
    D, i, j, w = _region_graph(R, seed, K)
    V = _dist(kind, K, seed)
    lab = numpy.argmin(D, axis=0).astype(numpy.uint8)
    energy = lambda l: mo.region_energy(D, i, j, w, l, V)      # noqa: E731
    for _ in range(2):
        for alpha, beta in so.pairs(K):
            new, switched, cut = so.region_move(D, i, j, w, lab, alpha, beta, V)
            assert switched == int((new != lab).sum())
            e_new = energy(new)
            assert abs(cut + so.region_fixed_energy(D, i, j, w, lab, alpha, beta, V) - e_new) <= 1e-12 * abs(e_new)
            assert abs(e_new - _best_swap(lab, alpha, beta, energy)) <= 1e-12 * abs(e_new)
            lab = new


@pytest.mark.parametrize("shape,seed", TINY)
@pytest.mark.parametrize("K", [3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_a_converged_voxel_run_admits_no_improving_swap(shape, seed, K, kind):
    costs, boundary, markers = _voxel_problem(shape, seed, K)
    V = _dist(kind, K, seed)
    r = so.swap(costs, boundary, markers, V=V)
    assert r["converged"] and r["moves"] == len(so.pairs(K)) * r["cycles"]
    assert r["switched"][-len(so.pairs(K)):] == [0] * len(so.pairs(K))
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights(shape, boundary)
    energy = lambda l: mo.energy(D, w, l, V)      # noqa: E731
    for alpha, beta in so.pairs(K):
        assert _best_swap(r["labels"], alpha, beta, energy) >= r["energy"] * (1 - 1e-12)


@pytest.mark.parametrize("R,seed", REGIONS)
@pytest.mark.parametrize("K", [3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_a_converged_region_run_admits_no_improving_swap(R, seed, K, kind):
    D, i, j, w = _region_graph(R, seed, K)
    V = _dist(kind, K, seed)
    r = so.region_swap(D, i, j, w, V=V)
    assert r["converged"]
    energy = lambda l: mo.region_energy(D, i, j, w, l, V)      # noqa: E731
    for alpha, beta in so.pairs(K):
        assert _best_swap(r["labels"], alpha, beta, energy) >= r["energy"] * (1 - 1e-12)


def test_potts_is_v_equal_one_minus_identity_bit_for_bit():
    K = 4
    costs, boundary, markers = _voxel_problem((3, 5), 7, K)
    D = ox.data_costs(costs, markers)
    w = ox.pair_weights((3, 5), boundary)
    rng = numpy.random.default_rng(1)
    lab = rng.integers(0, K, size=(3, 5)).astype(numpy.uint8)
    for alpha, beta in so.pairs(K):
        p, m = so.move_problem(D, w, lab, alpha, beta), so.move_problem(D, w, lab, alpha, beta, 1.0 - numpy.eye(K))
        for x, y in [(p["tr"], m["tr"])] + list(zip(p["wf"] + p["wb"], m["wf"] + m["wb"])):
            assert x.tobytes() == y.tobytes()


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
        r = so.swap(costs, boundary, markers, init=init, V=V)
        assert r["converged"] and r["moves"] <= 2
        assert abs(r["energy"] - best) <= 1e-12 * abs(best)


@pytest.mark.parametrize("R,seed", REGIONS)
def test_two_labels_reach_the_global_minimum_of_a_region_graph_from_any_init(R, seed):
    D, i, j, w = _region_graph(R, seed, 2)
    energies = {flat: mo.region_energy(D, i, j, w, numpy.asarray(flat, numpy.uint8))
                for flat in itertools.product(range(2), repeat=R)}
    best = min(energies.values())
    for flat in energies:
        r = so.region_swap(D, i, j, w, init=numpy.asarray(flat, numpy.uint8))
        assert r["converged"] and r["moves"] <= 2
        assert abs(r["energy"] - best) <= 1e-12 * abs(best)


# ------------------------------------------------------------------------------------------------------------ batches
@pytest.mark.parametrize("kind", KINDS)
def test_batch_model_runs_each_image_as_the_single_oracle(kind):
    B, K, shape = 3, 4, (3, 4)
    rng = numpy.random.default_rng(11)
    costs = rng.random((B, K) + shape) * 2.0
    for b in range(B):
        costs[b] = costs[b] * (1.0 - 0.3 * b) + 0.3 * b
    images = (rng.random((B,) + shape) * 3.0).astype(numpy.float32)
    boundaries = [("difference_exponential", images[b], 0.4 + 0.3 * b, False) for b in range(B)]
    V = _dist(kind, K)
    r = so.swap_batch(costs, boundaries, V=V)
    for b in range(B):
        ref = so.swap(costs[b], boundaries[b], V=V)
        assert numpy.array_equal(r["labels"][b], ref["labels"]) and r["energies"][b] == ref["energy"]
        assert r["switched"][b] == ref["switched"] and r["cycles"][b] == ref["cycles"]
        assert r["moves"][b] == len(so.pairs(K)) * ref["cycles"]


# ---------------------------------------------------------------------------------------------------- the Python layer
class _Recorder:
    """Stands in for the three native expansion classes: records every call and runs the swap or expansion oracle."""
    made = []

    def __init__(self, unit, *args):
        self.unit, self.calls, self.V, self.swap = unit, [], None, False
        self.K = args[-2] if unit != "voxel" else args[1]
        self.costs = [None] * self.K
        self.markers = self.init = None
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

    def set_moves(self, kind):
        from medpy_b200 import _lib
        self.calls.append("set_moves")
        assert kind == _lib._mgc.MOVES_SWAP
        self.swap, self.V = True, None

    def set_label_distance(self, V):
        self.calls.append("set_label_distance")
        assert V.dtype == numpy.float64 and V.flags.c_contiguous and V.shape == (self.K, self.K)
        self.V = V

    def run(self, max_cycles):
        self.calls.append("run")
        if self.unit == "voxel":
            run = so.swap if self.swap else mo.expansion
            self.r = run(numpy.stack(self.costs), None, self.markers, self.init, max_cycles, V=self.V)
        elif self.unit == "batch":
            run = so.swap_batch if self.swap else mo.expansion_batch
            self.r = run(numpy.stack(self.costs, axis=1), None, self.markers, self.init, max_cycles, V=self.V)
        else:
            run = so.region_swap if self.swap else mo.region_expansion
            self.r = run(numpy.stack(self.costs), *self.pairs, init=self.init, max_cycles=max_cycles, V=self.V)

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
UNITS = ["voxel", "batch", "region"]


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


@pytest.mark.parametrize("moves", ["Swap", "alpha-beta", "", None, 1, ["swap"]])
@pytest.mark.parametrize("unit", UNITS)
def test_a_bad_moves_value_is_refused_before_the_native_class(native, unit, moves):
    with pytest.raises(ValueError, match="moves must be"):
        _call(unit, moves=moves)
    assert native.made == []


@pytest.mark.parametrize("unit", UNITS)
def test_a_semi_metric_is_taken_by_swap_and_refused_by_expansion(native, unit):
    V = so.truncated_quadratic(K4, 4.0)
    with pytest.raises(ValueError, match=r"triangle inequality .*\(a, b, c\) = \(0, 1, 2\) breaks it; .*swap moves"):
        _call(unit, label_distance=V)
    with pytest.raises(ValueError, match=r"triangle inequality"):
        _call(unit, label_distance=V, moves="expansion")
    assert native.made == []
    out = _call(unit, label_distance=V.astype(numpy.int64).tolist(), moves="swap")
    rec = native.made[0]
    assert rec.calls[-3:] == ["set_moves", "set_label_distance", "run"]
    assert numpy.array_equal(rec.V, V)
    energy = out[-2]
    if unit == "batch":
        assert numpy.array_equal(energy, rec.r["energies"])
        assert out[-1]["moves"] == [6 * c for c in out[-1]["cycles"]]
    else:
        assert energy == rec.r["energy"]
        assert out[-1]["moves"] == 6 * out[-1]["cycles"]


@pytest.mark.parametrize("case", range(7))
@pytest.mark.parametrize("unit", UNITS)
def test_swap_keeps_every_other_rule_of_the_label_distance(native, unit, case):
    V = so.truncated_quadratic(K4, 4.0)
    nan, neg, diag, asym = (V.copy() for _ in range(4))
    nan[1, 2] = numpy.nan
    neg[2, 1] = -0.5
    diag[2, 2] = 0.25
    asym[0, 3] += 0.125
    V, msg = [(numpy.zeros((K4, K4 + 1)), r"\(K, K\) = \(4, 4\)"),
              (nan, r"finite and >= 0, V\[1\]\[2\] is not"),
              (neg, r"finite and >= 0, V\[2\]\[1\] is not"),
              (diag, r"zero diagonal, V\[2\]\[2\] is not 0"),
              (asym, r"symmetric, V\[0\]\[3\] != V\[3\]\[0\]"),
              (numpy.full((K4, K4), "x"), "real numbers"),
              (numpy.zeros((3, 3)), r"\(K, K\) = \(4, 4\)")][case]
    with pytest.raises(ValueError, match=msg):
        _call(unit, label_distance=V, moves="swap")
    assert native.made == []


@pytest.mark.parametrize("unit", UNITS)
def test_set_moves_is_called_before_set_label_distance_and_never_by_default(native, unit):
    _call(unit)
    _call(unit, moves="expansion", label_distance=mo.truncated_linear(K4, 2.0))
    _call(unit, moves="swap")
    _call(unit, moves="swap", label_distance=so.truncated_quadratic(K4, 4.0))
    a, b, c, d = native.made
    assert "set_moves" not in a.calls and "set_moves" not in b.calls
    assert c.calls[-2:] == ["set_moves", "run"] and c.V is None
    assert d.calls[-3:] == ["set_moves", "set_label_distance", "run"]
