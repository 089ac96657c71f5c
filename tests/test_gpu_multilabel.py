"""``graphcut.expansion_from_voxels`` on the GPU against the alpha-expansion oracle (oracle/expansion.py: every move graph
in numpy, cut by the BK restatement): labels voxel for voxel, the switch count of every move, the energy to 1e-12; and
K = 2 against ``graph_from_voxels``."""
import numpy
import pytest

from medpy_b200 import synthetic
from oracle import expansion as ox

pytestmark = pytest.mark.gpu

TERMS = ["difference_linear", "difference_exponential", "difference_division", "difference_power",
         "maximum_linear", "maximum_exponential", "maximum_division", "maximum_power"]
DTYPES = [numpy.float32, numpy.float64, numpy.uint8, numpy.int16, numpy.int32]
# ragged lattices over several tiles: 8^3 tiles in 1-D..3-D (leading axes of extent 1), 4 x 4 x 8 x 4 in 4-D
SHAPES = [(301,), (19, 37), (9, 17, 33), (5, 9, 6, 10)]
KS = [2, 3, 5, 17]


def _term(kind):
    from medpy_b200.graphcut import energy_voxel
    return getattr(energy_voxel, "boundary_" + kind)


def _term_args(kind, image, sigma, spacing):
    if kind.endswith("linear"):
        return (image, spacing)
    return (image, sigma, spacing)


def _image(rng, shape, dtype):
    if numpy.dtype(dtype).kind == "f":
        return (rng.random(shape) * 20.0).astype(dtype)
    return rng.integers(0, 40, size=shape).astype(dtype)


def _costs(rng, K, shape, dtype):
    # a smooth label preference per voxel plus noise, so the pair term decides the borders
    coord = numpy.indices(shape).sum(axis=0) / max(1, sum(shape))
    c = numpy.stack([numpy.abs(coord * K - k) * 0.6 for k in range(K)]) + rng.random((K,) + shape) * 0.8
    return c.astype(dtype)


def _case(i):
    kind = TERMS[i % 8]
    return dict(kind=kind, dtype=DTYPES[i % 5], shape=SHAPES[i % 4], K=KS[(i // 3) % 4], spacing=i % 3 == 0,
                cost_dtype=numpy.float32 if i % 2 else numpy.float64, on_device=i % 4 in (1, 2), markers=i % 3 != 1,
                init=i % 7 == 3)


def _inputs(i):
    c = _case(i)
    rng = numpy.random.default_rng(1000 + i)
    shape, K = c["shape"], c["K"]
    image = _image(rng, shape, c["dtype"])
    sigma = None if c["kind"].endswith("linear") else 3.0
    spacing = tuple([1.0, 2.5, 0.5, 1.5][:len(shape)]) if c["spacing"] else False
    costs = _costs(rng, K, shape, c["cost_dtype"])
    markers = None
    if c["markers"]:
        markers = numpy.zeros(shape, numpy.uint8)
        idx = rng.choice(markers.size, size=max(1, markers.size // 20), replace=False)
        markers.flat[idx] = rng.integers(1, K + 1, size=idx.size)
    init = None
    if c["init"]:
        init = rng.integers(0, K, size=shape).astype(numpy.uint8)
        if markers is not None:
            init = numpy.where(markers > 0, markers - 1, init).astype(numpy.uint8)
    return c, image, sigma, spacing, costs, markers, init


def _run(costs, kind, image, sigma, spacing, markers, init, on_device, max_cycles=20):
    from medpy_b200 import graphcut
    import torch
    if on_device:
        costs = torch.from_numpy(costs).cuda()
        markers = None if markers is None else torch.from_numpy(markers).cuda()
    labels, energy, st = graphcut.expansion_from_voxels(costs, _term(kind), _term_args(kind, image, sigma, spacing),
                                                        markers=markers, init=init, max_cycles=max_cycles, stats=True)
    if on_device:
        assert labels.is_cuda and labels.dtype == torch.uint8
        labels = labels.cpu().numpy()
    return labels, energy, st


def _check(st, labels, energy, ref):
    assert st["switched"] == ref["switched"]
    assert (st["moves"], st["cycles"], st["converged"]) == (ref["moves"], ref["cycles"], ref["converged"])
    assert numpy.array_equal(labels, ref["labels"])
    assert abs(energy - ref["energy"]) <= 1e-12 * abs(ref["energy"])


@pytest.mark.parametrize("i", range(40))
def test_matches_the_oracle(i):
    c, image, sigma, spacing, costs, markers, init = _inputs(i)
    labels, energy, st = _run(costs, c["kind"], image, sigma, spacing, markers, init, c["on_device"])
    ref = ox.expansion(costs, (c["kind"], image, sigma, spacing), markers, init)
    _check(st, labels, energy, ref)
    assert st["moves"] >= c["K"]


@pytest.mark.parametrize("shape", [(40,), (23, 31), (12, 20, 28), (6, 9, 10, 11)])
def test_no_boundary_term_is_the_per_voxel_argmin(shape):
    from medpy_b200 import graphcut
    rng = numpy.random.default_rng(len(shape))
    costs = rng.random((4,) + shape)
    labels, energy, st = graphcut.expansion_from_voxels(costs, stats=True)
    assert numpy.array_equal(labels, numpy.argmin(costs, axis=0))
    assert st["moves"] == 4 and st["converged"]
    assert abs(energy - costs.min(axis=0).sum()) <= 1e-12 * energy


def test_max_cycles_stops_the_loop():
    c, image, sigma, spacing, costs, markers, init = _inputs(5)
    full = ox.expansion(costs, (c["kind"], image, sigma, spacing), markers, init)
    assert full["cycles"] >= 2
    labels, energy, st = _run(costs, c["kind"], image, sigma, spacing, markers, init, False, max_cycles=1)
    ref = ox.expansion(costs, (c["kind"], image, sigma, spacing), markers, init, max_cycles=1)
    assert not st["converged"] and st["cycles"] == 1 and st["moves"] == c["K"]
    _check(st, labels, energy, ref)


def test_two_runs_give_the_same_bits():
    c, image, sigma, spacing, costs, markers, init = _inputs(6)
    a = _run(costs, c["kind"], image, sigma, spacing, markers, init, False)
    b = _run(costs, c["kind"], image, sigma, spacing, markers, init, True)
    assert numpy.array_equal(a[0], b[0])
    assert numpy.float64(a[1]).tobytes() == numpy.float64(b[1]).tobytes()
    assert a[2]["switched"] == b[2]["switched"]


@pytest.mark.parametrize("size", [64, 128])
@pytest.mark.parametrize("kind", TERMS)
def test_two_labels_equal_graph_from_voxels(size, kind):
    from medpy_b200 import graphcut
    vol = synthetic.two_blob_volume((size,) * 3, seed=size)
    prob, alpha = vol["prob"], vol["alpha"]
    args = _term_args(kind, vol["image"], vol["sigma"], False)
    g = graphcut.graph_from_voxels(vol["fg"], vol["bg"], regional_term=graphcut.energy_voxel.regional_probability_map,
                                   regional_term_args=(prob, alpha), boundary_term=_term(kind), boundary_term_args=args)
    flow = g.maxflow()
    mask = g.get_mask()
    costs = numpy.stack([prob * alpha, (1 - prob) * alpha])         # the products graph_from_voxels forms (float32)
    markers = numpy.where(vol["fg"], 2, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)
    labels, energy, st = graphcut.expansion_from_voxels(costs, _term(kind), args, markers=markers, stats=True)
    assert st["converged"]
    assert abs(energy - flow) <= 1e-9 * abs(flow)
    assert numpy.array_equal(labels, mask.reshape(labels.shape))


def test_four_labels_at_256_cubed_match_the_oracle():
    from medpy_b200 import graphcut
    vol = synthetic.two_blob_volume((256,) * 3, seed=3)
    image = vol["image"]
    means = numpy.asarray([0.0, 33.0, 66.0, 100.0], numpy.float32)
    costs = ((image[None] - means[:, None, None, None]) / numpy.float32(20.0)) ** 2
    markers = numpy.where(vol["fg"], 4, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)
    args = (image, vol["sigma"], False)
    labels, energy, st = graphcut.expansion_from_voxels(costs, graphcut.energy_voxel.boundary_difference_exponential, args,
                                                        markers=markers, stats=True)
    ref = ox.expansion(costs, ("difference_exponential", image, vol["sigma"], False), markers)
    _check(st, labels, energy, ref)
