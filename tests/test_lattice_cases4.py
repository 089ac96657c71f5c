"""The instance generators of lattice_cases4.py, checked on the CPU: together they cover every extent class of the
4 x 4 x 8 x 4 tile, several tiles along the last axis, every kernel of the last axis' row sweep and both sides of the
64-tile threshold; each is classified easy or hard as designed; tubes are long; every instance is a non-trivial cut; the
BK restatement agrees with the exact capacity of its own cut and with the reference BK; the integer family has ties."""
import numpy
import pytest
import scipy.ndimage as ndi

import lattice_cases as lc
import lattice_cases4 as l4


@pytest.fixture(scope="module", params=sorted(l4.CASES))
def case(request):
    return l4.make(request.param)


def _shapes():
    return {name: tuple(l4.make(name)["prob"]["shape"]) for name in l4.CASES}


def test_geometry_table_is_complete():
    shapes = _shapes()
    # every remainder of every axis modulo the tile extent, among the instances of at least 64 tiles
    big = [s for s in shapes.values() if l4.tiles4(s) >= 64]
    for d, ext in enumerate(l4.TILE4):
        assert {s[d] % ext for s in big} == set(range(ext)), (d, sorted({s[d] % ext for s in big}))
    # several tiles along the last axis, and an extent-1 axis in every position
    assert sum(l4.tiles_per_axis(s)[3] > 1 for s in shapes.values()) >= 10
    for d in range(4):
        assert any(s[d] == 1 for s in shapes.values()), d
    # every class of the last axis: no row sweep, short rows (up to and at the limit), warp rows, two segments
    lasts = [s[3] for s in shapes.values()]
    assert 1 in lasts and any(2 <= x <= 4 for x in lasts) and any(5 <= x <= 32 for x in lasts)
    assert l4.SWEEP_SHORT in lasts and any(33 <= x <= 1024 for x in lasts) and any(x > 1024 for x in lasts)
    assert {l4.row_kernel(s) for s in big} == {"none", "short", "warp", "segmented"}


def test_tile_counts_are_on_the_intended_side_of_64():
    for name, shape in _shapes().items():
        assert (l4.tiles4(shape) >= 64) == (name != "g-9x7x11x6"), (name, l4.tiles_per_axis(shape))


def test_classification_under_default_options(case):
    """Two-blob volumes with few tiles per axis hold a blob voxel in more than 1/8 of their tiles, so only the longer or
    flatter ones are easy; the serpentine lies in an easy lattice; boundary-only, far-sink and the dense instances are
    hard.  The matrix's `easy` option solves every instance as an easy one."""
    designed_easy = {"g-7x9x12x33", "g-6x5x9x1030", "g-20x16x1x20", "g-32x24x16x1", "l-serp4"}
    assert case["easy"] == (case["name"] in designed_easy)


def test_tubes_are_long(case):
    if case["family"] != "L":
        pytest.skip("no tube")
    shape = tuple(case["prob"]["shape"])
    path = case["path"]
    mask = lc._tube_mask(shape, [numpy.unravel_index(v, shape) for v in path], 2)
    assert len(path) > 140
    # inside the tube the far end is nearly as far from the sink end as along the path: no shortcut between legs
    length = _geodesic_length4(mask, int(path[-1]))
    assert length >= 0.95 * (len(path) - 1), (length, len(path))
    # every leg direction of the serpentine occurs
    if case["name"] == "l-serp4":
        steps = {tuple(numpy.sign(numpy.subtract(b, a))) for a, b in zip(l4.SERPENTINE4[:-1], l4.SERPENTINE4[1:])}
        assert len(steps) == 8, steps
        for q in l4.SERPENTINE4:
            assert all(c % (8 if d == 2 else 4) == (7 if d == 2 else 3) for d, c in enumerate(q)), q


def _geodesic_length4(mask, start):
    """Longest shortest path (in arcs) from `start` inside the voxel set `mask` of the 4-D lattice."""
    dist = numpy.full(mask.shape, -1, numpy.int64)
    frontier = numpy.zeros(mask.shape, bool)
    frontier.flat[start] = True
    dist.flat[start] = 0
    d = 0
    while frontier.any():
        d += 1
        grown = ndi.binary_dilation(frontier, structure=ndi.generate_binary_structure(4, 1)) & mask & (dist < 0)
        dist[grown] = d
        frontier = grown
    return int(dist.max())


def test_every_instance_is_a_non_trivial_cut(case):
    e, m = lc.bk(case)
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
    connected set between the two flips from source to sink side without changing the exact capacity.  (The far-sink
    variant, whose sink links all lie in the first tile layer, has a unique minimum cut.)"""
    if case["name"] != "i-ties":
        pytest.skip("not the integer-tie instance")
    from oracle import solvers
    e, m = lc.bk(case)
    re, rm, _ = solvers.solve_port(lc.reversed_problem(case["prob"]))
    assert re == e
    assert not numpy.array_equal(rm == 0, m == 1), "no tie: the minimum cut is unique"
    smallest = rm == 0
    assert not (smallest & (m == 0)).any(), "the smallest source side lies inside the largest"
    shape = tuple(case["prob"]["shape"])
    labels, n = ndi.label(((m == 1) & ~smallest).reshape(shape))
    assert n > 0
    sizes = numpy.bincount(labels.ravel())[1:]
    flipped = m.reshape(shape).copy()
    flipped[labels == 1 + int(numpy.argmax(sizes))] = 0
    assert lc.cut_capacity(case["prob"], flipped) == lc.cut_capacity(case["prob"], m) == e
