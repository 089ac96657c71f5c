"""Alpha-expansion with a metric label distance on the GPU (DESIGN.md §11, "Label distances"): the voxel, batch and region
units against the metric oracle (tests/metric_oracle.py: every move graph in numpy, cut by the BK restatements) --
labels element for element, the switch count of every move, the energy to 1e-12; V = 1 - I against the run without a
matrix bit for bit; two runs give the same bits; and the native classes' refusals and their return to Potts."""
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import energy_label_terms as elt  # noqa: E402
from oracle import region_expansion as orx  # noqa: E402

import metric_oracle as mo  # noqa: E402
import region_cases  # noqa: E402

pytestmark = pytest.mark.gpu

TERMS = ["difference_linear", "difference_exponential", "difference_division", "difference_power",
         "maximum_linear", "maximum_exponential", "maximum_division", "maximum_power"]
SHAPES = [(301,), (19, 37), (9, 17, 33), (5, 9, 6, 10)]
KS = [3, 5, 17]
METRICS = ["truncated_linear", "random", "scaled_potts", "pseudo"]


def _metric(kind, K, seed=0):
    if kind == "truncated_linear":
        return mo.truncated_linear(K, 2.0)
    if kind == "random":
        return mo.random_metric(K, 500 + seed)
    if kind == "scaled_potts":
        return mo.scaled_potts(K, 1.7)
    return mo.pseudo_metric(K)


def _term(kind):
    from medpy_b200.graphcut import energy_voxel
    return getattr(energy_voxel, "boundary_" + kind)


def _term_args(kind, image, sigma, spacing):
    return (image, spacing) if kind.endswith("linear") else (image, sigma, spacing)


def _costs(rng, K, shape, dtype, lead=()):
    coord = numpy.indices(shape).sum(axis=0) / max(1, sum(shape))
    pref = numpy.stack([numpy.abs(coord * K - k) * 0.6 for k in range(K)])
    return (pref + rng.random(lead + (K,) + shape) * 0.8).astype(dtype)


def _markers(rng, shape, K):
    m = numpy.zeros(shape, numpy.uint8)
    idx = rng.choice(m.size, size=max(1, m.size // 20), replace=False)
    m.flat[idx] = rng.integers(1, K + 1, size=idx.size)
    return m


def _init(rng, shape, K, markers):
    init = rng.integers(0, K, size=shape).astype(numpy.uint8)
    return init if markers is None else numpy.where(markers > 0, markers - 1, init).astype(numpy.uint8)


def _cuda(a):
    import torch
    return None if a is None else torch.from_numpy(a).cuda()


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else a


# ------------------------------------------------------------------------------------------------------------- voxels
def _voxel_case(i):
    return dict(kind=TERMS[i % 8], shape=SHAPES[i % 4], K=KS[(i // 4) % 3], metric=METRICS[(i + i // 4) % 4],
                cost_dtype=numpy.float32 if i % 2 else numpy.float64, on_device=i % 3 == 1, markers=i % 3 != 2,
                init=i % 5 == 3)


def _voxel_inputs(i):
    c = _voxel_case(i)
    rng = numpy.random.default_rng(3000 + i)
    shape, K = c["shape"], c["K"]
    image = (rng.random(shape) * 20.0).astype(numpy.float32)
    spacing = tuple([1.0, 2.5, 0.5, 1.5][:len(shape)]) if i % 2 == 0 else False
    costs = _costs(rng, K, shape, c["cost_dtype"])
    markers = _markers(rng, shape, K) if c["markers"] else None
    init = _init(rng, shape, K, markers) if c["init"] else None
    sigma = None if c["kind"].endswith("linear") else 3.0
    return c, (c["kind"], image, sigma, spacing), costs, markers, init, _metric(c["metric"], K, i)


def _voxel_run(costs, boundary, markers, init, V, on_device, max_cycles=20):
    from medpy_b200 import graphcut
    kind, image, sigma, spacing = boundary
    if on_device:
        costs, markers, V = _cuda(costs), _cuda(markers), None if V is None else _cuda(numpy.asarray(V))
    labels, energy, st = graphcut.expansion_from_voxels(costs, _term(kind), _term_args(kind, image, sigma, spacing),
                                                        markers=markers, init=init, max_cycles=max_cycles, stats=True,
                                                        label_distance=V)
    return _host(labels), energy, st


def _check(st, labels, energy, ref):
    assert st["switched"] == ref["switched"]
    assert (st["moves"], st["cycles"], st["converged"]) == (ref["moves"], ref["cycles"], ref["converged"])
    assert numpy.array_equal(labels, ref["labels"])
    assert abs(energy - ref["energy"]) <= 1e-12 * abs(ref["energy"])


@pytest.mark.parametrize("i", range(16))
def test_voxels_match_the_metric_oracle(i):
    c, boundary, costs, markers, init, V = _voxel_inputs(i)
    labels, energy, st = _voxel_run(costs, boundary, markers, init, V, c["on_device"])
    ref = mo.expansion(costs, boundary, markers, init, V=V)
    _check(st, labels, energy, ref)


def test_four_labels_at_96_cubed_with_truncated_linear_match_the_oracle():
    from medpy_b200 import graphcut, synthetic
    vol = synthetic.two_blob_volume((96,) * 3, seed=4)
    image = vol["image"]
    means = numpy.asarray([0.0, 33.0, 66.0, 100.0], numpy.float32)
    costs = ((image[None] - means[:, None, None, None]) / numpy.float32(20.0)) ** 2
    markers = numpy.where(vol["fg"], 4, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)
    V = mo.truncated_linear(4, 2.0)
    labels, energy, st = graphcut.expansion_from_voxels(costs, graphcut.energy_voxel.boundary_difference_exponential,
                                                        (image, vol["sigma"], False), markers=markers, stats=True,
                                                        label_distance=V)
    ref = mo.expansion(costs, ("difference_exponential", image, vol["sigma"], False), markers, V=V)
    _check(st, labels, energy, ref)


# ------------------------------------------------------------------------------------------------------------ batches
BATCH_SHAPES = [(301,), (19, 37), (9, 17, 33), (5, 6)]
BS = [1, 2, 7]


def _batch_inputs(i):
    rng = numpy.random.default_rng(4000 + i)
    shape, B, K = BATCH_SHAPES[i % 4], BS[i % 3], KS[(i // 2) % 3]
    kind = TERMS[(3 * i) % 8]
    bshape = (B,) + shape
    image = (rng.random(bshape) * 20.0).astype(numpy.float32)
    scale = 0.2 + 3.0 * rng.random(B)
    costs = (_costs(rng, K, shape, numpy.float64, (B,)) * scale.reshape((B, 1) + (1,) * len(shape)))
    costs = costs.astype(numpy.float32 if i % 2 else numpy.float64)
    markers = _markers(rng, bshape, K) if i % 3 != 1 else None
    init = _init(rng, bshape, K, markers) if i % 4 == 3 else None
    sigma = None if kind.endswith("linear") else 3.0
    c = dict(kind=kind, K=K, B=B, sigma=sigma, on_device=i % 2 == 1)
    return c, image, costs, markers, init, _metric(METRICS[i % 4], K, i)


def _batch_run(c, image, costs, markers, init, V, max_cycles=20):
    from medpy_b200 import graphcut
    if c["on_device"]:
        costs, markers = _cuda(costs), _cuda(markers)
    labels, energies, st = graphcut.expansion_from_voxels_batch(costs, image, c["kind"], sigma=c["sigma"], markers=markers,
                                                                init=init, max_cycles=max_cycles, stats=True,
                                                                label_distance=V)
    return _host(labels), energies, st


@pytest.mark.parametrize("i", range(12))
def test_batches_match_the_metric_batch_model(i):
    # the reference is the batch model (each image's moves cut by BK, the minimal minimum cut), not expansion_from_voxels
    # on each image: the single call's tile solve can leave an ulp on a saturated arc and move a voxel off the minimal
    # cut on some graphs, depending on the tile colour parity of the image's position (DESIGN.md §11, "Batches", "Where
    # the batch and the single call differ").  Case 11 is one: image 1's batch run is BK's, its single run is not.
    c, image, costs, markers, init, V = _batch_inputs(i)
    labels, energies, st = _batch_run(c, image, costs, markers, init, V)
    assert st["batch_cycles"] == max(st["cycles"]) and st["batch_moves"] == c["K"] * st["batch_cycles"]
    bounds = [(c["kind"], image[b], c["sigma"], False) for b in range(c["B"])]
    ref = mo.expansion_batch(costs, bounds, markers, init, V=V)
    assert numpy.array_equal(labels, ref["labels"])
    assert st["switched"] == ref["switched"] and st["cycles"] == ref["cycles"] and st["converged"] == ref["converged"]
    assert numpy.all(numpy.abs(energies - ref["energies"]) <= 1e-12 * numpy.abs(ref["energies"]))


# ------------------------------------------------------------------------------------------------------------ regions
def _region_inputs(i):
    lab = region_cases.label_volume([4, 1][i % 2])["label"]
    rng = numpy.random.default_rng(5000 + i)
    K = KS[i % 3]
    image = rng.random(lab.shape).astype(numpy.float32) * 10.0
    dtype = numpy.float32 if i % 2 else numpy.float64
    coord = numpy.indices(lab.shape).sum(axis=0) / max(1, sum(lab.shape))
    costs = (numpy.stack([numpy.abs(coord * K - k) for k in range(K)]) + rng.random((K,) + lab.shape)).astype(dtype)
    markers = None
    if i % 2 == 0:
        markers = numpy.zeros(lab.shape, numpy.uint8)
        idx = rng.choice(markers.size, size=max(2, markers.size // 1000), replace=False)
        markers.flat[idx] = rng.integers(1, K + 1, size=idx.size)
    return lab, K, image, costs, markers, _metric(METRICS[i % 4], K, i), i % 3 == 1


def _pairs(lab, image):
    lo, hi, a, _ = elt.merge_edges(*elt.stawiaski_calls(lab, image))
    order = numpy.lexsort((hi, lo))
    return lo[order], hi[order], numpy.asarray(a, numpy.float64)[order]


def _region_run(lab, costs, image, markers, V, on_device, max_cycles=20):
    from medpy_b200 import graphcut
    if on_device:
        costs = _cuda(costs)
    labels, region_labels, energy, st = graphcut.expansion_from_labels(
        lab, costs, graphcut.energy_label.boundary_stawiaski, image, markers=markers, max_cycles=max_cycles, stats=True,
        label_distance=V)
    return _host(labels), region_labels, energy, st


@pytest.mark.parametrize("i", range(6))
def test_regions_match_the_metric_oracle(i):
    lab, K, image, costs, markers, V, on_device = _region_inputs(i)
    labels, region_labels, energy, st = _region_run(lab, costs, image, markers, V, on_device)
    D = orx.data_costs(lab, costs, markers=markers)
    ref = mo.region_expansion(D, *_pairs(lab, image), V=V)
    _check(st, region_labels, energy, ref)
    assert numpy.array_equal(labels, ref["labels"][lab - 1])


# ------------------------------------------------------------------------------------- V = 1 - I and the same bits
def _same_bits(a, b):
    assert numpy.array_equal(a[0], b[0])
    assert numpy.asarray(a[1], numpy.float64).tobytes() == numpy.asarray(b[1], numpy.float64).tobytes()
    assert a[2]["switched"] == b[2]["switched"]


@pytest.mark.parametrize("i", [0, 5, 10, 15])
def test_potts_matrix_is_the_run_without_a_matrix_on_voxels(i):
    c, boundary, costs, markers, init, _ = _voxel_inputs(i)
    potts = 1.0 - numpy.eye(c["K"])
    _same_bits(_voxel_run(costs, boundary, markers, init, None, c["on_device"]),
               _voxel_run(costs, boundary, markers, init, potts, c["on_device"]))


@pytest.mark.parametrize("i", [1, 2, 6])
def test_potts_matrix_is_the_run_without_a_matrix_on_batches(i):
    c, image, costs, markers, init, _ = _batch_inputs(i)
    potts = 1.0 - numpy.eye(c["K"])
    _same_bits(_batch_run(c, image, costs, markers, init, None), _batch_run(c, image, costs, markers, init, potts))


@pytest.mark.parametrize("i", [0, 3, 5])
def test_potts_matrix_is_the_run_without_a_matrix_on_regions(i):
    lab, K, image, costs, markers, _, on_device = _region_inputs(i)
    potts = 1.0 - numpy.eye(K)
    a = _region_run(lab, costs, image, markers, None, on_device)
    b = _region_run(lab, costs, image, markers, potts, on_device)
    _same_bits(a[1:], b[1:])
    assert numpy.array_equal(a[0], b[0])


def test_two_runs_give_the_same_bits():
    c, boundary, costs, markers, init, V = _voxel_inputs(6)
    _same_bits(_voxel_run(costs, boundary, markers, init, V, False), _voxel_run(costs, boundary, markers, init, V, True))
    c, image, costs, markers, init, V = _batch_inputs(7)
    _same_bits(_batch_run(c, image, costs, markers, init, V), _batch_run(c, image, costs, markers, init, V))
    lab, K, image, costs, markers, V, _ = _region_inputs(6)
    a, b = _region_run(lab, costs, image, markers, V, False), _region_run(lab, costs, image, markers, V, True)
    _same_bits(a[1:], b[1:])


# ----------------------------------------------------------------------------------------------- the native classes
def _native(unit, K):
    """A native handle of `unit` with random costs set (no pair term on the lattices, a chain of pairs on the regions)."""
    from medpy_b200 import _lib
    rng = numpy.random.default_rng(len(unit) + K)
    if unit == "voxel":
        nat, shape = _lib._mgc.Expansion([6, 7, 8], K), (6, 7, 8)
    elif unit == "batch":
        nat, shape = _lib._mgc.ExpansionBatch([6, 7], 3, K), (3, 6, 7)
    else:
        nat, shape = _lib._mgc.RegionExpansion(50, K), (50,)
        nat.set_pairs(numpy.arange(49, dtype=numpy.int32), numpy.arange(1, 50, dtype=numpy.int32), rng.random(49) * 2.0)
    for k in range(K):
        nat.set_cost(k, rng.random(shape))
    return nat


def _result(nat):
    st = nat.stats()
    return nat.labels(), st["energy"], st.get("switched", nat.switched().tolist() if hasattr(nat, "switched") else None)


@pytest.mark.parametrize("unit", ["voxel", "batch", "region"])
def test_a_refused_matrix_leaves_the_native_class_on_potts_and_none_restores_it(unit):
    K = 4
    nat = _native(unit, K)
    nat.run(20)
    potts = _result(nat)
    V = mo.truncated_linear(K, 2.0) * 3.0
    nat.set_label_distance(V)
    nat.run(20)
    metric = _result(nat)
    i = numpy.arange(K)
    with pytest.raises(ValueError, match=r"triangle inequality.*\(0, 1, 2\)"):
        nat.set_label_distance(numpy.minimum((i[:, None] - i[None, :]) ** 2, 9).astype(numpy.float64))
    with pytest.raises(RuntimeError, match="first"):
        nat.stats()                                     # the refusal cleared the last run
    nat.run(20)
    again = _result(nat)
    assert numpy.array_equal(again[0], potts[0]) and again[1] == potts[1] and again[2] == potts[2]
    with pytest.raises(ValueError, match=r"\(K, K\)"):
        nat.set_label_distance(numpy.zeros((K, K + 1)))
    nat.set_label_distance(V)
    nat.run(20)
    back = _result(nat)
    assert numpy.array_equal(back[0], metric[0]) and back[1] == metric[1]
    nat.set_label_distance(None)
    nat.run(20)
    none = _result(nat)
    assert numpy.array_equal(none[0], potts[0]) and none[1] == potts[1] and none[2] == potts[2]
