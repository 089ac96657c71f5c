"""The contract the three native alpha-expansion classes share (``Expansion``, ``ExpansionBatch``, ``RegionExpansion``):
the label-count range, the unset-cost state, the cost, init and marker range checks, ``max_cycles``, and that a refused
input leaves nothing behind -- a refused cost plane unsets its label, so ``run`` refuses instead of cutting it."""
import numpy
import pytest

pytestmark = pytest.mark.gpu

K = 3


def _make(kind, labels=K):
    """The native class `kind` with `labels` labels, and the shape of its per-element arrays."""
    from medpy_b200 import _lib
    if kind == "Expansion":
        return _lib._mgc.Expansion([4, 5], labels), (4, 5)
    if kind == "ExpansionBatch":
        return _lib._mgc.ExpansionBatch([4, 5], 2, labels), (2, 4, 5)
    return _lib._mgc.RegionExpansion(7, labels), (7,)


KINDS = ["Expansion", "ExpansionBatch", "RegionExpansion"]


def _costs(shape, seed=0):
    return numpy.random.default_rng(seed).random((K,) + shape)


@pytest.mark.parametrize("kind", KINDS)
def test_one_label_is_refused(kind):
    with pytest.raises(ValueError, match="2..255"):
        _make(kind, labels=1)


@pytest.mark.parametrize("kind", KINDS)
def test_run_needs_every_cost(kind):
    nat, shape = _make(kind)
    costs = _costs(shape)
    for k in range(K - 1):
        nat.set_cost(k, costs[k])
    with pytest.raises(RuntimeError, match="not set"):
        nat.run(3)
    nat.set_cost(K - 1, costs[K - 1])
    nat.run(3)
    assert nat.labels().shape == shape


@pytest.mark.parametrize("kind", KINDS)
def test_a_negative_cost_is_refused(kind):
    nat, shape = _make(kind)
    with pytest.raises(ValueError, match="finite"):
        nat.set_cost(0, numpy.full(shape, -1.0))


@pytest.mark.parametrize("kind", KINDS)
def test_labels_above_the_range_are_refused(kind):
    nat, shape = _make(kind)
    with pytest.raises(ValueError, match="above {}".format(K - 1)):
        nat.set_init(numpy.full(shape, K, numpy.uint8))
    if kind != "RegionExpansion":           # region markers are in the caller's costs
        with pytest.raises(ValueError, match="above {}".format(K)):
            nat.set_markers(numpy.full(shape, K + 1, numpy.uint8))


@pytest.mark.parametrize("kind", KINDS)
def test_zero_cycles_are_refused(kind):
    nat, shape = _make(kind)
    costs = _costs(shape)
    for k in range(K):
        nat.set_cost(k, costs[k])
    with pytest.raises(ValueError, match="max_cycles"):
        nat.run(0)


@pytest.mark.parametrize("kind", KINDS)
def test_a_refused_plane_unsets_its_label(kind):
    nat, shape = _make(kind)
    costs = _costs(shape)
    for k in range(K):
        nat.set_cost(k, costs[k])
    nat.run(3)
    bad = costs[0].copy()
    bad.flat[0] = numpy.nan
    with pytest.raises(ValueError, match="finite"):
        nat.set_cost(0, bad)
    with pytest.raises(RuntimeError, match="not set"):
        nat.run(3)
    with pytest.raises(RuntimeError, match="run first"):
        nat.labels()
    nat.set_cost(0, costs[0])
    nat.run(3)
    assert nat.stats()["moves"] >= K


@pytest.mark.parametrize("kind", KINDS)
def test_a_refused_init_is_not_used(kind):
    nat, shape = _make(kind)
    costs = _costs(shape, seed=1)
    for k in range(K):
        nat.set_cost(k, costs[k])
    nat.run(1)
    free = nat.labels()
    nat.set_init(numpy.zeros(shape, numpy.uint8))
    with pytest.raises(ValueError, match="above"):
        nat.set_init(numpy.full(shape, K, numpy.uint8))
    nat.run(1)
    assert numpy.array_equal(nat.labels(), free)        # the default start, not the earlier init
