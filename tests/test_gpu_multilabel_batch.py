"""``graphcut.expansion_from_voxels_batch`` on the GPU: every image against ``expansion_from_voxels`` on that image alone
(labels voxel for voxel, the switch count of every move, moves, cycles, converged, the energy to 1e-12) and, on the small
batches, against the batch model (oracle/expansion_batch.py); the pair weights bit for bit against the single path's;
K = 2 against ``graph_from_voxels_batch``."""
import numpy
import pytest

from medpy_b200 import synthetic
from oracle import expansion_batch as oxb

pytestmark = pytest.mark.gpu

TERMS = ["difference_linear", "difference_exponential", "difference_division", "difference_power",
         "maximum_linear", "maximum_exponential", "maximum_division", "maximum_power", None]
DTYPES = [numpy.float32, numpy.float64, numpy.uint8, numpy.int16, numpy.int32]
# ragged images over several 8^3 tiles: 1-D, 2-D (a batch of 2-D images shares tiles eight images at a time), 3-D with
# Z not a multiple of 8, and small 2-D images of a few voxels
SHAPES = [(301,), (19, 37), (9, 17, 33), (5, 6), (11, 8, 9)]
BS = [1, 2, 7, 33]
KS = [2, 3, 5, 17]


def _term(kind):
    from medpy_b200.graphcut import energy_voxel
    return getattr(energy_voxel, "boundary_" + kind)


def _term_args(kind, image, sigma, spacing):
    if kind.endswith("linear"):
        return (image, spacing)
    return (image, sigma, spacing)


def _case(i):
    # shape and image dtype vary independently (cases 0..24 hold every pair); the term, B and K on strides of their own;
    # every sixth case passes the images as a CUDA tensor, whose linear normalisers are reduced on the device
    return dict(kind=TERMS[i % 9], dtype=DTYPES[(i // 5) % 5], shape=SHAPES[i % 5], B=BS[(i // 2) % 4],
                K=KS[(i // 3) % 4], spacing=i % 3 == 0, per_sigma=i % 2 == 0,
                cost_dtype=numpy.float32 if i % 2 else numpy.float64, on_device=i % 4 in (1, 2),
                cuda_image=i % 6 == 5, markers=i % 3 != 1, init=i % 7 == 3)


def _inputs(i):
    c = _case(i)
    rng = numpy.random.default_rng(2000 + i)
    B, K, shape = c["B"], c["K"], c["shape"]
    bshape = (B,) + shape
    if numpy.dtype(c["dtype"]).kind == "f":
        image = (rng.random(bshape) * 20.0).astype(c["dtype"])
    else:
        image = rng.integers(0, 40, size=bshape).astype(c["dtype"])
    sigma = None
    if c["kind"] is not None and not c["kind"].endswith("linear"):
        sigma = [float(s) for s in 2.0 + rng.random(B) * 3.0] if c["per_sigma"] else 3.0
    spacing = tuple([2.5, 0.5, 1.5][:len(shape)]) if c["spacing"] else False
    # a smooth label preference per voxel plus noise, scaled per image so the images need different numbers of cycles
    coord = numpy.indices(shape).sum(axis=0) / max(1, sum(shape))
    pref = numpy.stack([numpy.abs(coord * K - k) * 0.6 for k in range(K)])
    scale = 0.2 + 3.0 * rng.random(B)
    costs = (pref[None] + rng.random((B, K) + shape) * 0.8) * scale.reshape((B, 1) + (1,) * len(shape))
    costs = costs.astype(c["cost_dtype"])
    markers = None
    if c["markers"]:
        markers = numpy.zeros(bshape, numpy.uint8)
        idx = rng.choice(markers.size, size=max(1, markers.size // 20), replace=False)
        markers.flat[idx] = rng.integers(1, K + 1, size=idx.size)
    init = None
    if c["init"]:
        init = rng.integers(0, K, size=bshape).astype(numpy.uint8)
        if markers is not None:
            init = numpy.where(markers > 0, markers - 1, init).astype(numpy.uint8)
    return c, image, sigma, spacing, costs, markers, init


def _sigma_of(sigma, b):
    return sigma[b] if isinstance(sigma, list) else sigma


def _batch(costs, kind, image, sigma, spacing, markers, init, on_device, max_cycles=20, cuda_image=False):
    from medpy_b200 import graphcut
    import torch
    if on_device:
        costs = torch.from_numpy(costs).cuda()
        markers = None if markers is None else torch.from_numpy(markers).cuda()
    if cuda_image:
        image = torch.from_numpy(image).cuda()
    labels, energies, st = graphcut.expansion_from_voxels_batch(
        costs, None if kind is None else image, kind, sigma=sigma, spacing=spacing, markers=markers, init=init,
        max_cycles=max_cycles, stats=True)
    if on_device:
        assert labels.is_cuda and labels.dtype == torch.uint8
        labels = labels.cpu().numpy()
    assert isinstance(energies, numpy.ndarray) and energies.dtype == numpy.float64
    return labels, energies, st


def _single(costs, kind, image, sigma, spacing, markers, init, b, max_cycles=20):
    from medpy_b200 import graphcut
    term = _term(kind) if kind is not None else False
    args = _term_args(kind, image[b], _sigma_of(sigma, b), spacing) if kind is not None else False
    labels, energy, st = graphcut.expansion_from_voxels(costs[b], term, args,
                                                        markers=None if markers is None else markers[b],
                                                        init=None if init is None else init[b], max_cycles=max_cycles,
                                                        stats=True)
    return dict(labels=labels, energy=energy, switched=st["switched"], moves=st["moves"], cycles=st["cycles"],
                converged=st["converged"])


def _check_image(labels, energies, st, b, ref):
    assert st["switched"][b] == ref["switched"], b
    assert (st["moves"][b], st["cycles"][b], st["converged"][b]) == (ref["moves"], ref["cycles"], ref["converged"]), b
    assert numpy.array_equal(labels[b], ref["labels"]), b
    assert abs(energies[b] - ref["energy"]) <= 1e-12 * abs(ref["energy"]), b
    assert st["energy"][b] == energies[b]


def _check_batch(st, K):
    assert st["batch_cycles"] == max(st["cycles"]) and st["batch_moves"] == K * st["batch_cycles"]
    assert st["batch_converged"] == all(st["converged"])


@pytest.mark.parametrize("i", range(36))
def test_every_image_matches_its_single_run(i):
    c, image, sigma, spacing, costs, markers, init = _inputs(i)
    labels, energies, st = _batch(costs, c["kind"], image, sigma, spacing, markers, init, c["on_device"],
                                  cuda_image=c["cuda_image"])
    _check_batch(st, c["K"])
    for b in range(c["B"]):
        _check_image(labels, energies, st, b, _single(costs, c["kind"], image, sigma, spacing, markers, init, b))
    if c["B"] <= 2:     # and the batch model, on the batches small enough for it
        bounds = None if c["kind"] is None else [(c["kind"], image[b], _sigma_of(sigma, b), spacing) for b in range(c["B"])]
        ref = oxb.expansion_batch(costs, bounds, markers, init)
        assert numpy.array_equal(labels, ref["labels"])
        assert st["switched"] == ref["switched"] and st["cycles"] == ref["cycles"]
        assert numpy.all(numpy.abs(energies - ref["energies"]) <= 1e-12 * numpy.abs(ref["energies"]))


def test_a_mixed_batch_freezes_its_easy_images_and_max_cycles_cuts_the_rest():
    # image 0's data term decides every voxel by a margin no pair weight reaches (one cycle); the others are more and
    # more pair-dominated and take longer
    rng = numpy.random.default_rng(7)
    B, K, shape = 6, 4, (23, 29)
    image = (rng.random((B,) + shape) * 20).astype(numpy.float32)
    costs = rng.random((B, K) + shape) * numpy.asarray([1.0, 5.0, 1.0, 0.3, 0.1, 0.03])[:, None, None, None]
    costs[0] = 100.0 * (numpy.arange(K)[:, None, None] != rng.integers(0, K, size=shape)[None])
    bounds = [("difference_exponential", image[b], 3.0, False) for b in range(B)]
    for max_cycles in (20, 1):
        labels, energies, st = _batch(costs, "difference_exponential", image, 3.0, False, None, None, False, max_cycles)
        _check_batch(st, K)
        # against the batch model (BK's minimal cuts): on image 4 the single call's tile solve leaves one voxel off the
        # minimal cut of its first move (DESIGN.md §11 "Batches", "Where the batch and the single call differ"), so
        # the model, not the single call, is the reference here
        ref = oxb.expansion_batch(costs, bounds, max_cycles=max_cycles)
        assert numpy.array_equal(labels, ref["labels"])
        assert st["switched"] == ref["switched"] and st["cycles"] == ref["cycles"]
        assert st["converged"] == ref["converged"]
        assert numpy.all(numpy.abs(energies - ref["energies"]) <= 1e-12 * numpy.abs(ref["energies"]))
        if max_cycles == 20:
            assert len(set(st["cycles"])) > 1 and all(st["converged"])
        else:
            assert st["batch_moves"] == K and not all(st["converged"])


@pytest.mark.parametrize("kind", [k for k in TERMS if k is not None])
@pytest.mark.parametrize("shape", [(13,), (6, 7), (5, 6, 7)])
def test_pair_weights_are_the_single_paths_bit_for_bit(kind, shape):
    from medpy_b200 import _lib
    from medpy_b200.graphcut.batch import _host_image
    from medpy_b200.graphcut.device import _KINDS
    from medpy_b200.graphcut.multilabel import _BoundaryRecorder
    rng = numpy.random.default_rng(len(shape) * 10 + len(kind))
    B = 3
    image = rng.integers(0, 40, size=(B,) + shape).astype(numpy.int16) if kind.endswith("linear") else \
        (rng.random((B,) + shape) * 20).astype(numpy.float32)
    sigmas = [1.5, 3.0, 7.0]
    spacing = [2.5, 0.5, 1.5][:len(shape)]
    nat = _lib._mgc.ExpansionBatch(list(shape), B, 2, -1)
    dev, norms = _host_image(image, kind)
    nat.set_boundary(_KINDS[kind], dev, sigmas, spacing, norms)
    n = int(numpy.prod(shape))
    for a in range(len(shape)):
        w = nat.weights(a)
        stride = int(numpy.prod(shape[a + 1:]))
        for b in range(B):
            rec = _BoundaryRecorder()
            _term(kind)(rec, _term_args(kind, image[b], sigmas[b], spacing))
            g = _lib.Graph(list(shape), -1)
            g.add_boundary(*rec.call)
            ref = numpy.zeros(shape)
            flat = ref.reshape(-1)
            for p in range(n):
                if numpy.unravel_index(p, shape)[a] + 1 < shape[a]:
                    flat[p] = g.get_edge(p, p + stride)
            assert numpy.array_equal(w[b].view(numpy.uint64), ref.view(numpy.uint64)), (a, b)


def test_two_runs_give_the_same_bits_and_identical_images_the_same_results():
    c, image, sigma, spacing, costs, markers, init = _inputs(6)
    one = slice(0, 1)
    costs = numpy.repeat(costs[one], 4, axis=0)
    image = numpy.repeat(image[one], 4, axis=0)
    markers = None if markers is None else numpy.repeat(markers[one], 4, axis=0)
    sigma = None if sigma is None else (_sigma_of(sigma, 0))
    a = _batch(costs, c["kind"], image, sigma, spacing, markers, None, False)
    b = _batch(costs, c["kind"], image, sigma, spacing, markers, None, True)
    assert numpy.array_equal(a[0], b[0])
    assert a[1].tobytes() == b[1].tobytes()
    assert a[2]["switched"] == b[2]["switched"]
    for k in range(1, 4):
        assert numpy.array_equal(a[0][k], a[0][0])
        assert a[1][k].tobytes() == a[1][0].tobytes()
        assert a[2]["switched"][k] == a[2]["switched"][0]


@pytest.mark.parametrize("kind", ["difference_exponential", "maximum_linear", "difference_division"])
def test_two_labels_equal_graph_from_voxels_batch(kind):
    from medpy_b200 import graphcut
    vols = [synthetic.two_blob_volume((24, 20, 28), seed=s) for s in range(3)]
    prob = numpy.stack([v["prob"] for v in vols])
    alpha = vols[0]["alpha"]
    image = numpy.stack([v["image"] for v in vols])
    fg = numpy.stack([v["fg"] for v in vols])
    bg = numpy.stack([v["bg"] for v in vols])
    sigma = None if kind.endswith("linear") else [v["sigma"] for v in vols]
    g = graphcut.graph_from_voxels_batch(fg, bg, image, kind, sigma=sigma, prob=prob, alpha=alpha)
    flows = g.maxflow()
    masks = g.get_mask()
    costs = numpy.stack([prob * alpha, (1 - prob) * alpha], axis=1)      # the products the batch build forms (float32)
    markers = numpy.where(fg, 2, numpy.where(bg, 1, 0)).astype(numpy.uint8)
    labels, energies, st = graphcut.expansion_from_voxels_batch(costs, image, kind, sigma=sigma, markers=markers,
                                                                stats=True)
    assert all(st["converged"])
    assert numpy.array_equal(labels, masks.reshape(labels.shape))
    assert numpy.all(numpy.abs(energies - flows) <= 1e-9 * numpy.abs(flows))


@pytest.mark.parametrize("B,shape", [(64, (256, 256)), (8, (64, 64, 64))])
def test_scale_matches_single_runs(B, shape):
    from medpy_b200 import graphcut
    import torch
    vol = synthetic.two_blob_volume((B,) + shape if len(shape) == 2 else (B * shape[0],) + shape[1:], seed=5)
    image = vol["image"].reshape((B,) + shape)
    means = numpy.asarray([0.0, 33.0, 66.0, 100.0], numpy.float32)
    costs = ((image[:, None] - means.reshape((1, 4) + (1,) * len(shape))) / numpy.float32(20.0)) ** 2
    markers = numpy.where(vol["fg"], 4, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8).reshape((B,) + shape)
    labels, energies, st = graphcut.expansion_from_voxels_batch(torch.from_numpy(costs).cuda(), image,
                                                                "difference_exponential", sigma=vol["sigma"],
                                                                markers=markers, stats=True)
    labels = labels.cpu().numpy()
    _check_batch(st, 4)
    for b in range(B):
        _check_image(labels, energies, st, b, _single(costs, "difference_exponential", image, vol["sigma"], False,
                                                      markers, None, b))


def test_debug_checks_pass(monkeypatch):
    monkeypatch.setenv("MEDPY_GC_DEBUG", "1")
    c, image, sigma, spacing, costs, markers, init = _inputs(2)
    labels, energies, st = _batch(costs, c["kind"], image, sigma, spacing, markers, init, False)
    for b in range(c["B"]):
        _check_image(labels, energies, st, b, _single(costs, c["kind"], image, sigma, spacing, markers, init, b))


def test_native_errors_are_value_errors():
    from medpy_b200 import _lib
    with pytest.raises(ValueError, match="2..255"):
        _lib._mgc.ExpansionBatch([4, 4], 2, 1, -1)
    nat = _lib._mgc.ExpansionBatch([4, 4], 2, 3, -1)
    with pytest.raises(RuntimeError, match="not set"):
        nat.run(3)
    with pytest.raises(ValueError, match="finite"):
        nat.set_cost(0, numpy.full((2, 4, 4), -1.0))
    with pytest.raises(ValueError, match="above 3"):
        nat.set_markers(numpy.full((2, 4, 4), 4, numpy.uint8))
