"""The instance generators of lattice_cases.py, checked on the CPU: the geometry is what each family claims (ladder depths
straddle the push window and the first relabel's cap, tubes and corridors are long), every instance is a non-trivial cut,
the BK restatement agrees with the exact capacity of its own cut and with the reference BK, and the integer-tie family
really has ties."""
from collections import deque

import numpy
import pytest
import scipy.ndimage as ndi

import lattice_cases as lc


@pytest.fixture(scope="module", params=sorted(lc.CASES))
def case(request):
    return lc.make(request.param)


def _sink_distance(prob):
    """Taxicab distance of every voxel to the nearest sink-linked voxel (the initial BFS label minus one: every arc of
    these lattices has positive capacity)."""
    shape = tuple(prob["shape"])
    sink = numpy.asarray(prob["tr"]).reshape(shape) < 0
    return ndi.distance_transform_cdt(~sink, metric="taxicab")


def test_at_least_64_tiles(case):
    assert lc._tiles(case["prob"]["shape"]) >= 64


def test_ladder_depths_straddle_the_window_and_the_cap(case):
    if case["family"] not in ("A1", "A4"):
        pytest.skip("not a ladder")
    dist = _sink_distance(case["prob"])
    depths = []
    for shell, core in case["rungs"]:
        d = int(dist[core].min())
        assert d == shell + 1, (case["name"], shell, d)
        depths.append(d - 1)
    # every ladder has a rung beyond the cap; all but the deep-only one also a rung within the window
    assert max(depths) > lc.CAP, depths
    assert min(depths) < lc.WINDOW or case["name"] == "a1-ladder-s1", depths


def test_classification_under_default_options(case):
    """The ladders with shallow rungs, the tubes and the embedded maze leave enough sink-linked tiles to be solved as
    easy instances, so the window and the cap run under the default options; the others need MEDPY_GC_SWEEP_FRAC=1."""
    designed_easy = {"a1-ladder-s0", "a1-ladder-s2", "a2-serp-w2", "a2-serp-w3", "b2-maze-embedded"}
    assert case["easy"] == (case["name"] in designed_easy)


def test_ladders_cover_every_rung_of_the_design():
    shells = set()
    for name in lc.CASES:
        if lc.family(name) == "A1":
            shells |= {s for s, _ in lc.make(name)["rungs"]}
    assert shells == {7, 8, 9, 11, 12, 13, 24, 40}


def _geodesic_length(mask, start):
    """Longest shortest path (in arcs) from `start` inside the 6-connected voxel set `mask`."""
    shape = mask.shape
    flat = mask.ravel()
    dist = numpy.full(flat.size, -1, numpy.int64)
    dist[start] = 0
    strides = [int(numpy.prod(shape[d + 1:])) for d in range(3)]
    q = deque([start])
    while q:
        v = q.popleft()
        c = numpy.unravel_index(v, shape)
        for d in range(3):
            for s in (-1, 1):
                if 0 <= c[d] + s < shape[d]:
                    w = v + s * strides[d]
                    if flat[w] and dist[w] < 0:
                        dist[w] = dist[v] + 1
                        q.append(w)
    return int(dist.max())


def test_tubes_and_corridors_are_long(case):
    if case["family"] not in ("A2", "B2"):
        pytest.skip("no tube or corridor")
    shape = tuple(case["prob"]["shape"])
    path = case["path"]
    if case["family"] == "A2":
        width = int(case["name"][-1])
        mask = lc._tube_mask(shape, [numpy.unravel_index(v, shape) for v in path], width)
        # its source links cover the whole tube, its sink links only the end
        tr = case["prob"]["tr"].reshape(shape)
        assert (tr[mask] != 0).all()
        assert int((tr[mask] < 0).sum()) == (3 + width) * width * width
    else:
        mask = numpy.zeros(shape, bool)
        for d in range(3):
            strong = case["prob"]["wf"][d].reshape(shape) >= 1000
            mask |= strong
            mask[tuple(slice(1, None) if e == d else slice(None) for e in range(3))] |= strong[
                tuple(slice(0, -1) if e == d else slice(None) for e in range(3))]
    assert mask.ravel()[path].all()
    length = _geodesic_length(mask, int(path[-1]))      # from the sink end
    assert length > 3 * lc.CAP, length
    # inside the tube the far end is nearly as far from the sink end as along the path (the turns cut corners): no
    # shortcut between legs
    assert length >= 0.95 * (len(path) - 1), (length, len(path))


def test_every_instance_is_a_non_trivial_cut(case):
    e, m = lc.bk(case)
    if case["no_sink"]:
        assert (numpy.asarray(case["prob"]["tr"]) >= 0).all()
        assert m.all(), "without a sink link every voxel stays on the source side"
    else:
        assert 0 < int(m.sum()) < m.size, int(m.sum())


def test_bk_energy_is_the_exact_capacity_of_its_cut(case):
    e, m = lc.bk(case)
    cap = lc.cut_capacity(case["prob"], m)
    if case["exact"]:
        assert e == cap, (e, cap)
    else:
        assert abs(e - cap) <= 1e-9 * abs(cap), (e, cap)


def test_reference_bk_agrees(case):
    ref = lc.bk_ref(case)
    if ref is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    e, m = lc.bk(case)
    assert numpy.array_equal(ref[1], m)
    assert ref[0] == e if case["exact"] else abs(ref[0] - e) <= 1e-12 * abs(e), (ref[0], e)


def test_integer_ties_are_real(case):
    """BK's source side is the largest source set of a minimum cut; the reversed graph's BK cut gives the smallest.  A
    connected set between the two flips from source to sink side without changing the exact capacity: the instance has
    several minimum cuts, and only the rule "not connected to the sink" picks BK's."""
    if case["family"] != "B1":
        pytest.skip("not an integer-tie instance")
    from oracle import solvers
    e, m = lc.bk(case)
    re, rm, _ = solvers.solve_port(lc.reversed_problem(case["prob"]))
    assert re == e
    smallest = rm == 0
    assert not (smallest & (m == 0)).any(), "the smallest source side lies inside the largest"
    between = (m == 1) & ~smallest
    labels, n = ndi.label(between)
    assert n > 0, "no tie: the minimum cut is unique"
    sizes = numpy.bincount(labels.ravel())[1:]
    comp = labels == 1 + int(numpy.argmax(sizes))
    flipped = m.copy()
    flipped[comp] = 0
    assert lc.cut_capacity(case["prob"], flipped) == lc.cut_capacity(case["prob"], m) == e
    # flipping one sink-side voxel to the source side instead costs capacity: BK's source side is maximal
    sink_voxel = tuple(numpy.argwhere(m == 0)[0])
    grown = m.copy()
    grown[sink_voxel] = 1
    assert lc.cut_capacity(case["prob"], grown) > e
