"""``graphcut.expansion_from_labels`` on the GPU against the region alpha-expansion oracle (oracle/region_expansion.py:
every move problem in numpy, cut by the BK restatement for general graphs): region labels, voxel labels, the switch count
of every move, the energy to 1e-12; and K = 2 against ``graph_from_labels``."""
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from medpy_b200 import synthetic  # noqa: E402
from oracle import energy_label_terms as elt  # noqa: E402
from oracle import region_expansion as orx  # noqa: E402

import region_cases  # noqa: E402

pytestmark = pytest.mark.gpu

KS = [2, 3, 5, 17]
TERMS = ["stawiaski", "difference_of_means", None]
COSTS = ["f32", "f64", "f32_cuda", "f64_cuda", "region_f64", "region_f32_cuda"]
VOLUMES = [1, 2, 3, 4, "supervoxels"]


def supervoxels(shape, cell, seed):
    """A jittered grid of regions (cell voxels per axis, borders moved by one voxel at random) with ids exactly 1..R."""
    rng = numpy.random.default_rng(seed)
    key = numpy.zeros(shape, numpy.int64)
    for axis, s in enumerate(shape):
        idx = numpy.arange(s).reshape([-1 if a == axis else 1 for a in range(len(shape))])
        jit = numpy.clip(idx + rng.integers(-1, 2, size=shape) * (rng.random(shape) < 0.15), 0, s - 1) // cell
        key = key * (-(-s // cell)) + jit
    _, inv = numpy.unique(key, return_inverse=True)
    return (inv + 1).reshape(shape).astype(numpy.int32)


def _label_image(vol):
    if vol == "supervoxels":
        return supervoxels((40, 48, 36), 4, seed=11)
    return region_cases.label_volume(vol)["label"]


def _term(name):
    from medpy_b200.graphcut import energy_label
    return None if name is None else getattr(energy_label, "boundary_" + name)


def _pairs(name, lab, image):
    """The pair list of a term as the oracle computes it: ascending (i, j), one weight per pair."""
    if name is None:
        return numpy.zeros(0, numpy.int32), numpy.zeros(0, numpy.int32), numpy.zeros(0)
    calls = elt.stawiaski_calls(lab, image) if name == "stawiaski" else elt.difference_of_means_calls(lab, image)
    lo, hi, a, _ = elt.merge_edges(*calls)
    order = numpy.lexsort((hi, lo))
    return lo[order], hi[order], numpy.asarray(a, numpy.float64)[order]


def _markers(rng, lab, K):
    """0.1 % of the voxels marked at random, and the region of voxel 0 holding two marker values."""
    m = numpy.zeros(lab.shape, numpy.uint8)
    idx = rng.choice(m.size, size=max(2, m.size // 1000), replace=False)
    m.flat[idx] = rng.integers(1, K + 1, size=idx.size)
    where = numpy.flatnonzero(lab.ravel() == lab.flat[0])
    m.flat[where[0]] = 1
    m.flat[where[-1]] = 2
    return m


def _init(rng, lab, K, markers):
    """Random region labels; a marked region starts at the label of its lowest marker value."""
    R = int(lab.max())
    init = rng.integers(0, K, size=R).astype(numpy.uint8)
    if markers is not None:
        done = numpy.zeros(R, bool)
        for m in numpy.unique(markers)[1:]:
            inside = numpy.zeros(R, bool)
            inside[numpy.unique(lab[markers == m]) - 1] = True
            init[inside & ~done] = m - 1
            done |= inside
    return init


def _case(c):
    vol, K, term, cost = VOLUMES[c % 5], KS[(c // 2) % 4], TERMS[c % 3], COSTS[c % 6]
    return dict(vol=vol, K=K, term=term, cost=cost, markers=c % 2 == 0, init=c % 7 == 3)


def _run(lab, K, term, image, cost, markers, init, seed, max_cycles=20):
    """(library result, oracle result, the voxel labels as numpy)."""
    import torch
    from medpy_b200 import graphcut
    rng = numpy.random.default_rng(seed)
    R = int(lab.max())
    dtype = numpy.float32 if "f32" in cost else numpy.float64
    if cost.startswith("region"):
        data = (rng.random((K, R)) * 50.0).astype(dtype)
        D = orx.data_costs(lab, region_costs=data, markers=markers)
        kw = dict(costs=None, region_costs=torch.from_numpy(data).cuda() if cost.endswith("cuda") else data)
    else:
        coord = numpy.indices(lab.shape).sum(axis=0) / max(1, sum(lab.shape))
        data = (numpy.stack([numpy.abs(coord * K - k) for k in range(K)]) + rng.random((K,) + lab.shape)).astype(dtype)
        D = orx.data_costs(lab, data, markers=markers)
        kw = dict(costs=torch.from_numpy(data).cuda() if cost.endswith("cuda") else data)
    labels, region_labels, energy, st = graphcut.expansion_from_labels(
        lab, boundary_term=_term(term) or False, boundary_term_args=image, markers=markers, init=init,
        max_cycles=max_cycles, stats=True, **kw)
    if cost.endswith("cuda"):
        assert labels.is_cuda and labels.dtype == torch.uint8
        labels = labels.cpu().numpy()
    ref = orx.expansion(D, *_pairs(term, lab, image), init=init, max_cycles=max_cycles)
    return (region_labels, labels, energy, st), ref


def _check(got, ref, lab):
    region_labels, labels, energy, st = got
    assert st["switched"] == ref["switched"]
    assert (st["moves"], st["cycles"], st["converged"]) == (ref["moves"], ref["cycles"], ref["converged"])
    assert region_labels.dtype == numpy.uint8 and numpy.array_equal(region_labels, ref["labels"])
    assert numpy.array_equal(labels, ref["labels"][lab - 1])
    assert abs(energy - ref["energy"]) <= 1e-12 * abs(ref["energy"])


@pytest.mark.parametrize("c", range(24))
def test_matches_the_oracle(c):
    k = _case(c)
    lab = _label_image(k["vol"])
    rng = numpy.random.default_rng(100 + c)
    image = region_cases.gradient(lab.shape, "float32", seed=200 + c) if k["term"] == "stawiaski" else \
        rng.random(lab.shape).astype(numpy.float32) * 10.0
    image = numpy.abs(numpy.nan_to_num(image, posinf=0.0, neginf=0.0)).astype(numpy.float32)
    markers = _markers(rng, lab, k["K"]) if k["markers"] else None
    init = _init(rng, lab, k["K"], markers) if k["init"] else None
    got, ref = _run(lab, k["K"], k["term"], image, k["cost"], markers, init, seed=300 + c)
    _check(got, ref, lab)
    assert got[3]["moves"] >= k["K"]


def test_one_region():
    from medpy_b200 import graphcut
    lab = numpy.ones((5, 6), numpy.int32)
    costs = numpy.random.default_rng(1).random((3, 5, 6))
    labels, region_labels, energy = graphcut.expansion_from_labels(
        lab, costs, graphcut.energy_label.boundary_stawiaski, numpy.ones((5, 6), numpy.float32))
    D = orx.data_costs(lab, costs)
    assert region_labels.tolist() == [int(numpy.argmin(D[:, 0]))]
    assert numpy.array_equal(labels, numpy.full((5, 6), region_labels[0], numpy.uint8))
    assert abs(energy - D[:, 0].min()) <= 1e-12 * energy


def test_max_cycles_stops_the_loop():
    lab = _label_image("supervoxels")
    rng = numpy.random.default_rng(5)
    image = rng.random(lab.shape).astype(numpy.float32) * 0.2
    full = _run(lab, 5, "stawiaski", image, "f64", None, None, seed=6)[1]
    assert full["cycles"] >= 2
    got, ref = _run(lab, 5, "stawiaski", image, "f64", None, None, seed=6, max_cycles=1)
    assert not got[3]["converged"] and got[3]["cycles"] == 1 and got[3]["moves"] == 5
    _check(got, ref, lab)


def test_two_runs_give_the_same_bits():
    lab = _label_image(3)
    rng = numpy.random.default_rng(7)
    image = rng.random(lab.shape).astype(numpy.float32)
    markers = _markers(rng, lab, 5)
    a = _run(lab, 5, "stawiaski", image, "f32", markers, None, seed=8)[0]
    b = _run(lab, 5, "stawiaski", image, "f32_cuda", markers, None, seed=8)[0]
    assert numpy.array_equal(a[0], b[0]) and numpy.array_equal(a[1], b[1])
    assert numpy.float64(a[2]).tobytes() == numpy.float64(b[2]).tobytes()
    assert a[3]["switched"] == b[3]["switched"]


def test_native_class_with_float32_costs_matches_the_oracle():
    from medpy_b200 import _lib
    rng = numpy.random.default_rng(9)
    lab = _label_image("supervoxels")
    i, j, w = _pairs("stawiaski", lab, rng.random(lab.shape).astype(numpy.float32))
    R, K = int(lab.max()), 4
    costs = (rng.random((K, R)) * 3.0).astype(numpy.float32)
    nat = _lib._mgc.RegionExpansion(R, K)
    for k in range(K):
        nat.set_cost(k, costs[k])
    nat.set_pairs(i.astype(numpy.int32), j.astype(numpy.int32), w)
    nat.run(20)
    st = nat.stats()
    ref = orx.expansion(costs.astype(numpy.float64), i, j, w)
    assert numpy.array_equal(nat.labels(), ref["labels"]) and st["switched"] == ref["switched"]
    assert abs(st["energy"] - ref["energy"]) <= 1e-12 * abs(ref["energy"])
    with pytest.raises(ValueError, match="ascending"):
        nat.set_pairs(numpy.asarray([0, 0], numpy.int32), numpy.asarray([2, 1], numpy.int32), numpy.ones(2))
    with pytest.raises(ValueError, match="finite"):
        nat.set_pairs(numpy.asarray([0], numpy.int32), numpy.asarray([1], numpy.int32), numpy.asarray([-1.0]))


def _blob_case(size, seed):
    vol = synthetic.two_blob_volume((size,) * 3, seed=seed, with_prob=False)
    return supervoxels((size,) * 3, 4, seed), vol


@pytest.mark.parametrize("size", [128, 256])
def test_two_labels_equal_graph_from_labels(size):
    from medpy_b200 import graphcut
    lab, vol = _blob_case(size, seed=size)
    R = int(lab.max())
    image = vol["image"]
    D = numpy.stack([numpy.bincount(lab.ravel() - 1, weights=(image.ravel() / 100.0) ** 2),
                     numpy.bincount(lab.ravel() - 1, weights=(1.0 - image.ravel() / 100.0) ** 2)])

    def regional(graph, label_image, d):
        graph.set_tweights_bulk(numpy.arange(R), d[0], d[1])

    grad = numpy.abs(numpy.gradient(image)[0]).astype(numpy.float32)
    g = graphcut.graph_from_labels(lab, vol["fg"], vol["bg"], regional_term=regional, regional_term_args=D,
                                   boundary_term=graphcut.energy_label.boundary_stawiaski, boundary_term_args=grad)
    flow = g.maxflow()
    mask = graphcut.label_cut_mask(g)
    markers = numpy.where(vol["fg"], 2, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)
    labels, region_labels, energy, st = graphcut.expansion_from_labels(
        lab, None, graphcut.energy_label.boundary_stawiaski, grad, markers=markers, stats=True, region_costs=D)
    assert st["converged"]
    assert numpy.array_equal(labels, mask)
    assert abs(energy - flow) <= 1e-12 * abs(flow)


def test_four_labels_at_128_cubed_match_the_oracle():
    lab, vol = _blob_case(128, seed=3)
    image = vol["image"]
    means = numpy.asarray([0.0, 33.0, 66.0, 100.0], numpy.float32)
    costs = ((image[None] - means[:, None, None, None]) / numpy.float32(20.0)) ** 2
    markers = numpy.where(vol["fg"], 4, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)
    grad = numpy.abs(numpy.gradient(image)[0]).astype(numpy.float32)
    from medpy_b200 import graphcut
    labels, region_labels, energy, st = graphcut.expansion_from_labels(
        lab, costs, graphcut.energy_label.boundary_stawiaski, grad, markers=markers, stats=True)
    D = orx.data_costs(lab, costs, markers=markers)
    ref = orx.expansion(D, *_pairs("stawiaski", lab, grad))
    _check((region_labels, labels, energy, st), ref, lab)
