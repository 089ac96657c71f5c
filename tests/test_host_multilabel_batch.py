"""The batched alpha-expansion model (oracle/expansion_batch.py) against per-image runs of oracle/expansion.py and against a
brute-force expansion loop on tiny images, and ``graphcut.expansion_from_voxels_batch``'s argument checks and stats
assembly through the Python layer with a recording stand-in for the native class.  No GPU needed."""
import itertools
import math

import numpy
import pytest

from oracle import energy_terms as et
from oracle import expansion as ox
from oracle import expansion_batch as oxb


def _batch(B, shape, K, seed, spread=0.0):
    """B tiny images; image b's costs are flattened by `spread * b` so the images need different numbers of cycles."""
    rng = numpy.random.default_rng(seed)
    costs = rng.random((B, K) + shape) * 2.0
    for b in range(B):
        costs[b] = costs[b] * (1.0 - spread * b) + spread * b
    images = (rng.random((B,) + shape) * 3.0).astype(numpy.float32)
    boundaries = [("difference_exponential", images[b], 0.4 + 0.3 * b, False) for b in range(B)]
    return costs, boundaries


def _brute_move(D, w, lab, alpha):
    """The move by enumeration: the smallest of the minimum-energy switch sets (the minimal sink set)."""
    shape = lab.shape
    free = numpy.flatnonzero(lab.ravel() != alpha)
    sets = []
    for bits in itertools.product((0, 1), repeat=free.size):
        cand = lab.copy().ravel()
        chosen = free[numpy.asarray(bits, bool)]
        cand[chosen] = alpha
        sets.append((ox.energy(D, w, cand.reshape(shape)), frozenset(chosen.tolist())))
    best = min(e for e, _ in sets)
    tied = [s for e, s in sets if e <= best + 1e-12 * abs(best)]
    core = frozenset.intersection(*tied)
    assert core in tied
    out = lab.copy().ravel()
    out[list(core)] = alpha
    return out.reshape(shape), len(core)


def _brute_batch(costs, boundaries, max_cycles):
    """The batch loop with every move enumerated, images frozen after a cycle without a switch."""
    B, K = costs.shape[:2]
    shape = costs.shape[2:]
    D = [ox.data_costs(costs[b]) for b in range(B)]
    w = [ox.pair_weights(shape, boundaries[b]) for b in range(B)]
    lab = [ox.initial_labels(D[b], shape) for b in range(B)]
    active, cycles, conv, sw = [True] * B, [0] * B, [False] * B, [[] for _ in range(B)]
    for _ in range(max_cycles):
        if not any(active):
            break
        changed = [0] * B
        for alpha in range(K):
            for b in range(B):
                if active[b]:
                    lab[b], s = _brute_move(D[b], w[b], lab[b], alpha)
                    sw[b].append(s)
                    changed[b] += s
        for b in range(B):
            if active[b]:
                cycles[b] += 1
                if not changed[b]:
                    conv[b], active[b] = True, False
    return lab, [ox.energy(D[b], w[b], lab[b]) for b in range(B)], sw, cycles, conv


TINY = [(1, (8,), 3, 0), (2, (7,), 3, 1), (3, (2, 4), 3, 2), (4, (3, 2), 2, 3), (4, (2, 3), 4, 4), (2, (2, 2, 2), 3, 5)]


@pytest.mark.parametrize("B,shape,K,seed", TINY)
@pytest.mark.parametrize("max_cycles", [1, 2, 20])
def test_model_matches_brute_force(B, shape, K, seed, max_cycles):
    costs, boundaries = _batch(B, shape, K, seed, spread=0.2)
    r = oxb.expansion_batch(costs, boundaries, max_cycles=max_cycles)
    lab, energies, sw, cycles, conv = _brute_batch(costs, boundaries, max_cycles)
    for b in range(B):
        assert numpy.array_equal(r["labels"][b], lab[b])
        assert abs(r["energies"][b] - energies[b]) <= 1e-12 * abs(energies[b])
    assert r["switched"] == sw and r["cycles"] == cycles and r["converged"] == conv
    assert r["moves"] == [K * c for c in cycles]


def _single(costs, boundaries, markers, init, max_cycles):
    return [ox.expansion(costs[b], boundaries[b] if boundaries else None, None if markers is None else markers[b],
                         None if init is None else init[b], max_cycles) for b in range(costs.shape[0])]


@pytest.mark.parametrize("max_cycles", [1, 2, 3, 20])
@pytest.mark.parametrize("with_markers", [False, True])
def test_model_is_the_single_run_of_every_image(max_cycles, with_markers):
    # image 0 has no pair term (its argmin is final: one cycle), the others are more and more pair-dominated (two or more
    # cycles), so the images converge at different cycles
    B, K, shape = 5, 4, (6, 7)
    rng = numpy.random.default_rng(11)
    costs = rng.random((B, K) + shape) * numpy.asarray([1.0, 1.0, 0.3, 0.1, 0.03])[:, None, None, None]
    boundaries = [None]
    for b in range(1, B):
        image = (rng.random(shape) * (0.2 + b)).astype(numpy.float64)
        boundaries.append(("difference_exponential", image, 0.5 + 0.6 * b, False))
    markers = None
    if with_markers:
        markers = numpy.zeros((B,) + shape, numpy.uint8)
        markers[:, 0, 0] = 1 + numpy.arange(B) % K
    r = oxb.expansion_batch(costs, boundaries, markers, max_cycles=max_cycles)
    ref = _single(costs, boundaries, markers, None, max_cycles)
    for b in range(B):
        assert numpy.array_equal(r["labels"][b], ref[b]["labels"])
        assert r["switched"][b] == ref[b]["switched"]
        assert (r["moves"][b], r["cycles"][b], r["converged"][b]) == (ref[b]["moves"], ref[b]["cycles"], ref[b]["converged"])
        assert abs(r["energies"][b] - ref[b]["energy"]) <= 1e-12 * abs(ref[b]["energy"])
    assert r["batch_cycles"] == max(x["cycles"] for x in ref)
    assert r["batch_converged"] == all(x["converged"] for x in ref)
    assert r["matrix"].shape == (K * r["batch_cycles"], B)
    if max_cycles == 20:
        assert len({x["cycles"] for x in ref}) > 1, "the images should converge at different cycles"
    if max_cycles == 1:
        assert not all(x["converged"] for x in ref), "max_cycles = 1 should cut some image off"


def test_frozen_images_have_zero_rows():
    costs, boundaries = _batch(3, (9,), 3, 7, spread=0.3)
    r = oxb.expansion_batch(costs, boundaries)
    for b in range(3):
        assert not r["matrix"][r["moves"][b]:, b].any()


# ---------------------------------------------------------------------------------------------------- the Python layer
class _Recorder:
    """Stands in for ``_mgc.ExpansionBatch``: records every call, and runs the batch model."""
    made = []

    def __init__(self, image_shape, batch, labels, device=-1):
        self.shape, self.B, self.K, self.calls = tuple(image_shape), batch, labels, []
        self.costs = [None] * labels
        self.boundaries = self.markers = self.init = None
        self.sigmas = self.norms = None
        _Recorder.made.append(self)

    def set_cost(self, k, c):
        self.calls.append("set_cost")
        c = numpy.asarray(c)
        assert c.shape == (self.B,) + self.shape and c.flags.c_contiguous
        self.costs[k] = c

    def set_boundary(self, kind, image, sigmas, spacing, norms):
        self.calls.append("set_boundary")
        self.sigmas, self.norms = list(sigmas), list(norms)
        self.boundaries = [(et.BOUNDARY_KINDS[kind], numpy.asarray(image)[b], sigmas[b], spacing if spacing else False)
                           for b in range(self.B)]

    def set_markers(self, m):
        self.calls.append("set_markers")
        self.markers = m

    def set_init(self, i):
        self.calls.append("set_init")
        self.init = i

    def run(self, max_cycles):
        self.calls.append("run")
        self.r = oxb.expansion_batch(numpy.stack(self.costs, axis=1), self.boundaries, self.markers, self.init, max_cycles)

    def image_stats(self):
        r = self.r
        return dict(moves=numpy.asarray(r["moves"]), cycles=numpy.asarray(r["cycles"]),
                    converged=numpy.asarray(r["converged"]), energy=r["energies"])

    def stats(self):
        r = self.r
        return dict(moves=r["batch_moves"], cycles=r["batch_cycles"], converged=r["batch_converged"],
                    energy=float(r["energies"].sum()), ms_build=0.0, ms_solve=0.0, ms_apply=0.0, ms_total=0.0)

    def switched(self):
        return self.r["matrix"]

    def labels(self):
        return self.r["labels"]


@pytest.fixture
def native(monkeypatch):
    from medpy_b200 import _lib
    _Recorder.made = []
    monkeypatch.setattr(_lib._mgc, "ExpansionBatch", _Recorder)
    return _Recorder


def _args(B=3, K=3, shape=(5, 6)):
    rng = numpy.random.default_rng(5)
    costs = rng.random((B, K) + shape).astype(numpy.float32)
    image = rng.random((B,) + shape).astype(numpy.float32)
    return costs, image


def test_python_layer_runs_the_model_end_to_end(native):
    from medpy_b200 import graphcut
    costs, image = _args()
    markers = numpy.zeros(image.shape, numpy.int32)
    markers[1, 0, 0] = 3
    sigma = [0.5, 0.9, 1.4]
    labels, energies, st = graphcut.expansion_from_voxels_batch(costs, image, "difference_exponential", sigma=sigma,
                                                                spacing=(1.0, 2.0), markers=markers, max_cycles=4,
                                                                stats=True)
    assert native.made[0].calls == ["set_cost"] * 3 + ["set_boundary", "set_markers", "run"]
    assert native.made[0].sigmas == sigma
    assert energies.dtype == numpy.float64 and energies.shape == (3,)
    for b in range(3):
        ref = ox.expansion(costs[b], ("difference_exponential", image[b], sigma[b], [1.0, 2.0]),
                           markers[b].astype(numpy.uint8), max_cycles=4)
        assert numpy.array_equal(labels[b], ref["labels"]) and energies[b] == ref["energy"]
        assert st["switched"][b] == ref["switched"]
        assert (st["moves"][b], st["cycles"][b], st["converged"][b]) == (ref["moves"], ref["cycles"], ref["converged"])
        assert st["energy"][b] == ref["energy"]
    assert labels[1, 0, 0] == 2
    assert st["batch_cycles"] == max(st["cycles"]) and st["batch_moves"] == 3 * st["batch_cycles"]
    assert st["batch_converged"] == all(st["converged"])


def test_integer_images_get_their_linear_normaliser_per_image(native):
    from medpy_b200 import graphcut
    costs, _ = _args()
    image = numpy.stack([numpy.full((5, 6), b, numpy.int16) for b in range(3)])
    image[:, 0, 0] = [9, -4, 100]
    graphcut.expansion_from_voxels_batch(costs, image, "difference_linear")
    assert native.made[0].norms == [9.0, 5.0, 98.0]
    graphcut.expansion_from_voxels_batch(costs, image.astype(numpy.float32), "maximum_linear")
    assert all(math.isnan(x) for x in native.made[1].norms)


def test_stats_assembly_cuts_each_column_at_its_moves():
    from medpy_b200.graphcut.multilabel import _batch_stats
    matrix = numpy.arange(12, dtype=numpy.int64).reshape(6, 2)
    per = dict(moves=numpy.asarray([3, 6]), cycles=numpy.asarray([1, 2]), converged=numpy.asarray([True, False]),
               energy=numpy.asarray([1.5, 2.5]))
    total = dict(moves=6, cycles=2, converged=False, energy=4.0, ms_build=1.0, ms_solve=2.0, ms_apply=3.0, ms_total=7.0)
    st = _batch_stats(total, per, matrix)
    assert st["switched"] == [[0, 2, 4], [1, 3, 5, 7, 9, 11]]
    assert st["moves"] == [3, 6] and st["cycles"] == [1, 2] and st["converged"] == [True, False]
    assert st["energy"] == [1.5, 2.5]
    assert (st["batch_moves"], st["batch_cycles"], st["batch_converged"]) == (6, 2, False)
    assert (st["ms_build"], st["ms_solve"], st["ms_apply"], st["ms_total"]) == (1.0, 2.0, 3.0, 7.0)


def _bad(costs, image):
    shape = image.shape
    return [
        (dict(costs=costs.astype(numpy.int32)), "float32 or float64"),
        (dict(costs=costs[:, :1]), "2..255"),
        (dict(costs=numpy.zeros((2, 256, 2, 2), numpy.float32)), "2..255"),
        (dict(costs=numpy.zeros((2, 2, 2, 2, 2, 2), numpy.float32)), "1- to 3-D"),
        (dict(costs=costs[0, 0]), "1- to 3-D"),
        (dict(costs=numpy.where(costs > 0.5, numpy.nan, costs)), "finite"),
        (dict(costs=costs - 1.0), ">= 0"),
        (dict(image=image[:2]), "image has shape"),
        (dict(image=None), "both image and boundary"),
        (dict(boundary="gaussian"), "boundary must be one of"),
        (dict(sigma=[1.0, 2.0]), "sigma has 2 entries"),
        (dict(spacing=(1.0,)), "spacing"),
        (dict(markers=numpy.zeros(shape[1:], numpy.uint8)), "image shape"),
        (dict(markers=numpy.full(shape, 4, numpy.uint8)), "0..3"),
        (dict(markers=numpy.zeros(shape, numpy.float32)), "integers"),
        (dict(init=numpy.full(shape, 3, numpy.uint8)), "0..2"),
        (dict(init=numpy.zeros(shape, numpy.uint8), markers=numpy.full(shape, 2, numpy.uint8)), "marker"),
        (dict(max_cycles=0), "max_cycles"),
        (dict(max_cycles=True), "max_cycles"),
    ]


@pytest.mark.parametrize("case", range(19))
def test_bad_arguments_are_refused_before_the_native_class(native, case):
    from medpy_b200 import graphcut
    costs, image = _args()
    kw, msg = _bad(costs, image)[case]
    call = dict(costs=costs, image=image, boundary="difference_exponential", sigma=1.0)
    call.update(kw)
    with pytest.raises(ValueError, match=msg):
        graphcut.expansion_from_voxels_batch(**call)
    assert native.made == []


def test_the_index_limit_is_refused_before_the_native_class(native):
    from medpy_b200 import graphcut
    big = numpy.lib.stride_tricks.as_strided(numpy.zeros(1, numpy.float32), shape=(2048, 2, 1024, 1024),
                                             strides=(0, 0, 0, 0))
    with pytest.raises(ValueError, match="2\\^31"):
        graphcut.expansion_from_voxels_batch(big)
    assert native.made == []


def test_max_cycles_and_init_reach_the_native_class(native):
    from medpy_b200 import graphcut
    costs, _ = _args()
    init = numpy.zeros((3, 5, 6), numpy.int64)
    labels, energies, st = graphcut.expansion_from_voxels_batch(costs, init=init, max_cycles=1, stats=True)
    assert native.made[0].calls == ["set_cost"] * 3 + ["set_init", "run"]
    assert st["batch_moves"] == 3 and st["batch_cycles"] == 1
    for b in range(3):
        ref = ox.expansion(costs[b], None, None, init[b], 1)
        assert numpy.array_equal(labels[b], ref["labels"])
