"""Alpha-beta swap moves on the GPU (DESIGN.md §11, "Swap moves"): the voxel, batch and region units against the swap
oracle (tests/swap_oracle.py: every move graph in numpy, cut by the BK restatements) -- labels element for element, the
switch count of every move, moves, cycles and the converged flag exactly, the energy to 1e-12; V = 1 - I against the
run without a matrix bit for bit; two runs give the same bits; K = 2 against graph_from_voxels; MEDPY_GC_DEBUG=1; and
the native classes' set_moves."""
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
import swap_oracle as so  # noqa: E402
from test_gpu_region_expansion import supervoxels  # noqa: E402

pytestmark = pytest.mark.gpu

TERMS = ["difference_linear", "difference_exponential", "difference_division", "difference_power",
         "maximum_linear", "maximum_exponential", "maximum_division", "maximum_power"]
SHAPES = [(301,), (19, 37), (9, 17, 33), (5, 9, 6, 10)]
KS = [2, 3, 5, 17]
DISTS = ["potts", "truncated_linear", "truncated_quadratic", "random"]


def _dist(kind, K, seed=0):
    if kind == "potts":
        return None
    if kind == "truncated_linear":
        return mo.truncated_linear(K, 2.0)
    if kind == "truncated_quadratic":
        return so.truncated_quadratic(K, 4.0)
    return so.random_semi_metric(K, 600 + seed)


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


def _check(st, labels, energy, ref):
    assert st["switched"] == ref["switched"]
    assert (st["moves"], st["cycles"], st["converged"]) == (ref["moves"], ref["cycles"], ref["converged"])
    assert numpy.array_equal(labels, ref["labels"])
    assert abs(energy - ref["energy"]) <= 1e-12 * abs(ref["energy"])


# ------------------------------------------------------------------------------------------------------------- voxels
def _voxel_inputs(i):
    rng = numpy.random.default_rng(7000 + i)
    kind, shape, K = TERMS[i % 8], SHAPES[i % 4], KS[(i // 4) % 4]
    image = (rng.random(shape) * 20.0).astype(numpy.float32)
    spacing = tuple([1.0, 2.5, 0.5, 1.5][:len(shape)]) if i % 2 == 0 else False
    costs = _costs(rng, K, shape, numpy.float32 if i % 2 else numpy.float64)
    markers = _markers(rng, shape, K) if i % 3 != 2 else None
    init = _init(rng, shape, K, markers) if i % 5 == 3 else None
    sigma = None if kind.endswith("linear") else 3.0
    return dict(K=K, on_device=i % 3 == 1), (kind, image, sigma, spacing), costs, markers, init, \
        _dist(DISTS[(i + i // 4) % 4], K, i)


def _voxel_run(costs, boundary, markers, init, V, on_device, moves="swap"):
    from medpy_b200 import graphcut
    kind, image, sigma, spacing = boundary
    if on_device:
        costs, markers, V = _cuda(costs), _cuda(markers), None if V is None else _cuda(numpy.asarray(V))
    labels, energy, st = graphcut.expansion_from_voxels(costs, _term(kind), _term_args(kind, image, sigma, spacing),
                                                        markers=markers, init=init, stats=True, label_distance=V,
                                                        moves=moves)
    return _host(labels), energy, st


@pytest.mark.parametrize("i", range(16))
def test_voxels_match_the_swap_oracle(i):
    c, boundary, costs, markers, init, V = _voxel_inputs(i)
    labels, energy, st = _voxel_run(costs, boundary, markers, init, V, c["on_device"])
    _check(st, labels, energy, so.swap(costs, boundary, markers, init, V=V))


# ------------------------------------------------------------------------------------------------------------ batches
BATCH_SHAPES = [(301,), (19, 37), (9, 17, 33), (5, 6)]


def _batch_inputs(i):
    rng = numpy.random.default_rng(8000 + i)
    shape, B, K = BATCH_SHAPES[i % 4], [1, 2, 7][i % 3], KS[(i // 2) % 4]
    kind = TERMS[(3 * i) % 8]
    bshape = (B,) + shape
    image = (rng.random(bshape) * 20.0).astype(numpy.float32)
    scale = 0.2 + 3.0 * rng.random(B)
    costs = _costs(rng, K, shape, numpy.float64, (B,)) * scale.reshape((B, 1) + (1,) * len(shape))
    if B > 1:
        costs[1] = numpy.where(numpy.arange(K).reshape((K,) + (1,) * len(shape)) == 0, 0.0, 5.0)   # frozen after cycle 1
    costs = costs.astype(numpy.float32 if i % 2 else numpy.float64)
    markers = _markers(rng, bshape, K) if i % 3 != 1 else None
    init = _init(rng, bshape, K, markers) if i % 4 == 3 else None
    sigma = None if kind.endswith("linear") else 3.0
    c = dict(kind=kind, K=K, B=B, sigma=sigma, on_device=i % 2 == 1)
    return c, image, costs, markers, init, _dist(DISTS[i % 4], K, i)


def _batch_run(c, image, costs, markers, init, V, moves="swap"):
    from medpy_b200 import graphcut
    if c["on_device"]:
        costs, markers = _cuda(costs), _cuda(markers)
    labels, energies, st = graphcut.expansion_from_voxels_batch(costs, image, c["kind"], sigma=c["sigma"], markers=markers,
                                                                init=init, stats=True, label_distance=V, moves=moves)
    return _host(labels), energies, st


@pytest.mark.parametrize("i", range(12))
def test_batches_match_the_swap_batch_model(i):
    c, image, costs, markers, init, V = _batch_inputs(i)
    labels, energies, st = _batch_run(c, image, costs, markers, init, V)
    P = c["K"] * (c["K"] - 1) // 2
    assert st["batch_cycles"] == max(st["cycles"]) and st["batch_moves"] == P * st["batch_cycles"]
    assert st["moves"] == [P * cyc for cyc in st["cycles"]]
    bounds = [(c["kind"], image[b], c["sigma"], False) for b in range(c["B"])]
    ref = so.swap_batch(costs, bounds, markers, init, V=V)
    assert numpy.array_equal(labels, ref["labels"])
    assert st["switched"] == ref["switched"] and st["cycles"] == ref["cycles"] and st["converged"] == ref["converged"]
    assert (st["batch_moves"], st["batch_cycles"]) == (ref["batch_moves"], ref["batch_cycles"])
    assert numpy.all(numpy.abs(energies - ref["energies"]) <= 1e-12 * numpy.abs(ref["energies"]))


# ------------------------------------------------------------------------------------------------------------ regions
def _region_inputs(i):
    lab = supervoxels((24, 20, 16), 4, seed=30 + i) if i % 3 == 2 else region_cases.label_volume([4, 1][i % 2])["label"]
    rng = numpy.random.default_rng(9000 + i)
    K = KS[i % 4]
    image = rng.random(lab.shape).astype(numpy.float32) * 10.0
    coord = numpy.indices(lab.shape).sum(axis=0) / max(1, sum(lab.shape))
    costs = numpy.stack([numpy.abs(coord * K - k) for k in range(K)]) + rng.random((K,) + lab.shape)
    costs = costs.astype(numpy.float32 if i % 2 else numpy.float64)
    markers = None
    if i % 2 == 0:
        markers = numpy.zeros(lab.shape, numpy.uint8)
        idx = rng.choice(markers.size, size=max(2, markers.size // 1000), replace=False)
        markers.flat[idx] = rng.integers(1, K + 1, size=idx.size)
    return lab, K, image, costs, markers, _dist(DISTS[(i + 1) % 4], K, i), i % 3 == 1


def _pairs(lab, image):
    lo, hi, a, _ = elt.merge_edges(*elt.stawiaski_calls(lab, image))
    order = numpy.lexsort((hi, lo))
    return lo[order], hi[order], numpy.asarray(a, numpy.float64)[order]


def _region_run(lab, costs, image, markers, V, on_device, moves="swap"):
    from medpy_b200 import graphcut
    if on_device:
        costs = _cuda(costs)
    labels, region_labels, energy, st = graphcut.expansion_from_labels(
        lab, costs, graphcut.energy_label.boundary_stawiaski, image, markers=markers, stats=True, label_distance=V,
        moves=moves)
    return _host(labels), region_labels, energy, st


@pytest.mark.parametrize("i", range(8))
def test_regions_match_the_swap_oracle(i):
    lab, K, image, costs, markers, V, on_device = _region_inputs(i)
    labels, region_labels, energy, st = _region_run(lab, costs, image, markers, V, on_device)
    ref = so.region_swap(orx.data_costs(lab, costs, markers=markers), *_pairs(lab, image), V=V)
    _check(st, region_labels, energy, ref)
    assert numpy.array_equal(labels, ref["labels"][lab - 1])


# ------------------------------------------------------------------------------------- V = 1 - I and the same bits
def _same_bits(a, b):
    assert numpy.array_equal(a[0], b[0])
    assert numpy.asarray(a[1], numpy.float64).tobytes() == numpy.asarray(b[1], numpy.float64).tobytes()
    assert a[2]["switched"] == b[2]["switched"]


@pytest.mark.parametrize("i", [1, 6, 11])
def test_potts_matrix_is_the_swap_run_without_a_matrix(i):
    c, boundary, costs, markers, init, _ = _voxel_inputs(i)
    potts = 1.0 - numpy.eye(c["K"])
    _same_bits(_voxel_run(costs, boundary, markers, init, None, c["on_device"]),
               _voxel_run(costs, boundary, markers, init, potts, c["on_device"]))
    c, image, costs, markers, init, _ = _batch_inputs(i)
    potts = 1.0 - numpy.eye(c["K"])
    _same_bits(_batch_run(c, image, costs, markers, init, None), _batch_run(c, image, costs, markers, init, potts))
    lab, K, image, costs, markers, _, on_device = _region_inputs(i % 8)
    a = _region_run(lab, costs, image, markers, None, on_device)
    b = _region_run(lab, costs, image, markers, 1.0 - numpy.eye(K), on_device)
    _same_bits(a[1:], b[1:])


def test_two_runs_give_the_same_bits():
    c, boundary, costs, markers, init, V = _voxel_inputs(7)
    _same_bits(_voxel_run(costs, boundary, markers, init, V, False), _voxel_run(costs, boundary, markers, init, V, True))
    c, image, costs, markers, init, V = _batch_inputs(5)
    _same_bits(_batch_run(c, image, costs, markers, init, V), _batch_run(c, image, costs, markers, init, V))
    lab, K, image, costs, markers, V, _ = _region_inputs(5)
    a, b = _region_run(lab, costs, image, markers, V, False), _region_run(lab, costs, image, markers, V, True)
    _same_bits(a[1:], b[1:])


# ----------------------------------------------------------------------------------------------------------------- K = 2
@pytest.mark.parametrize("kind", ["difference_exponential", "maximum_linear"])
def test_two_labels_equal_graph_from_voxels(kind):
    from medpy_b200 import graphcut, synthetic
    vol = synthetic.two_blob_volume((64,) * 3, seed=64)
    prob, alpha = vol["prob"], vol["alpha"]
    args = _term_args(kind, vol["image"], vol["sigma"], False)
    g = graphcut.graph_from_voxels(vol["fg"], vol["bg"], regional_term=graphcut.energy_voxel.regional_probability_map,
                                   regional_term_args=(prob, alpha), boundary_term=_term(kind), boundary_term_args=args)
    flow = g.maxflow()
    mask = g.get_mask()
    costs = numpy.stack([prob * alpha, (1 - prob) * alpha])
    markers = numpy.where(vol["fg"], 2, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)
    labels, energy, st = graphcut.expansion_from_voxels(costs, _term(kind), args, markers=markers, stats=True,
                                                        moves="swap")
    assert st["converged"] and st["moves"] <= 2
    assert abs(energy - flow) <= 1e-9 * abs(flow)
    assert numpy.array_equal(labels, mask.reshape(labels.shape))


# -------------------------------------------------------------------------------------------------------- debug mode
def test_debug_mode_matches_the_oracle(monkeypatch):
    monkeypatch.setenv("MEDPY_GC_DEBUG", "1")
    c, boundary, costs, markers, init, V = _voxel_inputs(2)
    labels, energy, st = _voxel_run(costs, boundary, markers, init, V, c["on_device"])
    _check(st, labels, energy, so.swap(costs, boundary, markers, init, V=V))
    c, image, costs, markers, init, V = _batch_inputs(4)
    labels, energies, st = _batch_run(c, image, costs, markers, init, V)
    ref = so.swap_batch(costs, [(c["kind"], image[b], c["sigma"], False) for b in range(c["B"])], markers, init, V=V)
    assert numpy.array_equal(labels, ref["labels"]) and st["switched"] == ref["switched"]


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
    return nat.labels(), st["energy"], st.get("switched", nat.switched().tolist() if hasattr(nat, "switched") else None), \
        st["moves"]


@pytest.mark.parametrize("unit", ["voxel", "batch", "region"])
def test_set_moves_refuses_other_kinds_clears_the_run_and_drops_the_distance(unit):
    from medpy_b200 import _lib
    K = 4
    nat = _native(unit, K)
    nat.run(20)
    expansion = _result(nat)
    quad = so.truncated_quadratic(K, 4.0)
    with pytest.raises(ValueError, match=r"triangle inequality.*swap moves"):
        nat.set_label_distance(quad)                    # expansion moves refuse a semi-metric, as before
    for bad in (2, -1):
        with pytest.raises(ValueError, match="moves must be"):
            nat.set_moves(bad)
    nat.set_moves(_lib._mgc.MOVES_SWAP)
    with pytest.raises(RuntimeError, match="first"):
        nat.stats()                                     # set_moves cleared the last run
    nat.run(20)
    swap_potts = _result(nat)
    assert swap_potts[3] % 6 == 0
    nat.set_label_distance(quad)
    nat.run(20)
    swap_quad = _result(nat)
    nat.set_moves(_lib._mgc.MOVES_SWAP)                 # drops the distance: back on Potts
    nat.run(20)
    again = _result(nat)
    assert numpy.array_equal(again[0], swap_potts[0]) and again[1] == swap_potts[1] and again[2] == swap_potts[2]
    nat.set_label_distance(quad)
    nat.run(20)
    back = _result(nat)
    assert numpy.array_equal(back[0], swap_quad[0]) and back[1] == swap_quad[1]
    nat.set_moves(_lib._mgc.MOVES_EXPANSION)
    nat.run(20)
    exp_again = _result(nat)
    assert numpy.array_equal(exp_again[0], expansion[0]) and exp_again[1] == expansion[1]
    assert exp_again[2] == expansion[2] and exp_again[3] == expansion[3]
    with pytest.raises(ValueError, match=r"triangle inequality"):
        nat.set_label_distance(quad)
