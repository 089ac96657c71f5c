"""GraphDouble.add_seeds on the host: argument handling (masks to ids in logical C order, id range, shapes), the staged
path before the first solve, the warm path through an oracle-backed double of the native class -- and, with the real
reference BK, the semantic claim the warm path rests on: solve, add_tweights seeds, solve again == from scratch."""
import os
import sys

import numpy
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_native  # noqa: E402


class _SeedGraph(fake_native.FakeGraph):
    """FakeGraph plus add_seeds: replays the seeds on the from-scratch t-links (the oracle of the warm path)."""

    def __init__(self, shape, device=-1):
        super().__init__(shape, device)
        self.seed_calls = []

    def add_seeds(self, fg_ids, bg_ids):
        from oracle import energy_terms as et
        self.seed_calls.append((fg_ids, bg_ids))
        for ids, s, t in ((fg_ids, 65535.0, 0.0), (bg_ids, 0.0, 65535.0)):
            if ids is None:
                continue
            ids = numpy.asarray(ids)
            assert ids.dtype == numpy.int64 and ids.ndim == 1
            for v in ids.tolist():
                self.flow = et.add_tweights_pass(self.tr, self.flow, s, t, where=numpy.arange(self.n) == v)
        self.result = None


@pytest.fixture()
def made(monkeypatch):
    from medpy_b200 import _lib
    out = []

    def factory(shape, device=-1):
        g = _SeedGraph(shape, device)
        out.append(g)
        return g
    monkeypatch.setattr(_lib, "Graph", factory)
    return out


def _graph(shape=(6, 7, 8), seed=0):
    import medpy_b200.graphcut as gc
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=seed)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(vol["prob"], vol["alpha"]),
                             boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    return g, vol


def test_fortran_mask_gives_c_order_ids(made):
    g, _ = _graph()
    g.maxflow()
    m = numpy.zeros((6, 7, 8), bool)
    m[1, 2, 3] = m[4, 0, 7] = m[0, 6, 0] = True
    g.add_seeds(fg=numpy.asfortranarray(m), bg=m[::-1][::-1])
    fg, bg = made[0].seed_calls[-1]
    assert fg.tolist() == [0 * 56 + 6 * 8 + 0, 1 * 56 + 2 * 8 + 3, 4 * 56 + 0 * 8 + 7]
    assert bg.tolist() == fg.tolist()
    g.add_seeds(fg=torch.from_numpy(m), bg=torch.tensor([7, 5], dtype=torch.int32))
    fg, bg = made[0].seed_calls[-1]
    assert fg.tolist() == [0 * 56 + 6 * 8 + 0, 1 * 56 + 2 * 8 + 3, 4 * 56 + 0 * 8 + 7] and bg.tolist() == [7, 5]


def test_ids_keep_order_and_duplicates(made):
    g, _ = _graph()
    g.maxflow()
    g.add_seeds(fg=[5, 3, 5], bg=numpy.array([7], numpy.int32))
    fg, bg = made[0].seed_calls[-1]
    assert fg.tolist() == [5, 3, 5] and bg.tolist() == [7]


def test_bad_arguments(made):
    g, _ = _graph()
    g.maxflow()
    n = 6 * 7 * 8
    with pytest.raises(ValueError, match="Invalid node id of {} or 0. Valid values are 0 to {}.".format(n, n - 1)):
        g.add_seeds(fg=[0, n])
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_seeds(bg=[-1])
    with pytest.raises(ValueError, match="shape"):
        g.add_seeds(fg=numpy.zeros((6, 7), bool))
    with pytest.raises(ValueError):
        g.add_seeds(fg=numpy.zeros((2, 2), numpy.int64))
    with pytest.raises(ValueError):
        g.add_seeds(fg=[1.5])
    with pytest.raises(ValueError):
        g.add_seeds(fg=5)                       # a single id is not an id array on the lattice
    assert made[0].seed_calls == []
    g.add_seeds()
    assert made[0].seed_calls[-1] == (None, None)


def test_warm_path_equals_from_scratch(made):
    from oracle import energy_terms as et, solvers
    g, vol = _graph()
    g.maxflow()
    fg = numpy.array([100, 101, 100])
    bg = numpy.array([5, 100])
    g.add_seeds(fg, bg)
    e, m = g.maxflow(), g.get_mask()
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    for ids, s, t in ((fg, 65535.0, 0.0), (bg, 0.0, 65535.0)):
        for v in ids:
            prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], s, t, where=numpy.arange(prob["tr"].size) == v)
    oe, om, _ = solvers.solve_port(prob)
    assert numpy.array_equal(m, om) and abs(e - oe) <= 1e-9 * abs(oe)


def test_unsolved_graph_stages_add_tweights(made):
    """Before the first maxflow() add_seeds is add_tweights: the staged dense pass carries 65535 on the seeds."""
    g, _ = _graph()
    ref, _ = _graph()
    g.add_seeds(fg=[3, 3], bg=[4])
    g.add_seeds(bg=torch.tensor([6, 4]))
    for v in (3, 3):
        ref.add_tweights(v, 65535.0, 0.0)
    for v in (4, 6, 4):
        ref.add_tweights(v, 0.0, 65535.0)
    assert made[0].seed_calls == [] and g.maxflow() == ref.maxflow()
    assert numpy.array_equal(g.get_mask(), ref.get_mask())
    assert numpy.array_equal(made[0].tr, made[1].tr)


def _reference_bk():
    """The unmodified reference BK as built into oracle/_ref/libbkref.so (its graph-handle entry points)."""
    import ctypes
    from oracle import solvers
    if not solvers.have_ref():
        return None
    lib = ctypes.CDLL(solvers._REF_SO)
    lib.bkref_new.restype = ctypes.c_void_p
    lib.bkref_new.argtypes = [ctypes.c_int, ctypes.c_int]
    lib.bkref_delete.argtypes = [ctypes.c_void_p]
    lib.bkref_add_tweights.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_double]
    lib.bkref_sum_edge.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double]
    lib.bkref_maxflow.restype = ctypes.c_double
    lib.bkref_maxflow.argtypes = [ctypes.c_void_p]
    lib.bkref_what_segment.argtypes = [ctypes.c_void_p, ctypes.c_int]
    return lib


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_reference_bk_resolve_after_add_tweights_equals_from_scratch(seed):
    """The claim the warm path rests on, pinned on the unmodified reference BK: after maxflow(), add_tweights on new
    seeds and maxflow() again give the min cut of the enlarged graph (same mask, same energy as a fresh solve)."""
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    rng = numpy.random.default_rng(seed)
    shape = (5, 6, 7)
    n = int(numpy.prod(shape))
    strides = (42, 7, 1)
    edges = []
    for v in range(n):
        c = numpy.unravel_index(v, shape)
        for d in range(3):
            if c[d] + 1 < shape[d]:
                edges.append((v, v + strides[d], float(rng.uniform(0.01, 2.0)), float(rng.uniform(0.01, 2.0))))
    tw = [(v, float(rng.uniform(0, 3)), float(rng.uniform(0, 3))) for v in range(n)]
    steps = [(rng.integers(0, n, 4).tolist(), rng.integers(0, n, 4).tolist()) for _ in range(3)]

    def seed_calls(h, fg, bg):
        for v in fg:
            bk.bkref_add_tweights(h, v, 65535.0, 0.0)
        for v in bg:
            bk.bkref_add_tweights(h, v, 0.0, 65535.0)

    def fresh(k):
        h = bk.bkref_new(n, len(edges))
        for i, j, a, b in edges:
            bk.bkref_sum_edge(h, i, j, a, b)
        for v, a, b in tw:
            bk.bkref_add_tweights(h, v, a, b)
        for fg, bg in steps[:k]:
            seed_calls(h, fg, bg)
        return h

    warm = fresh(0)
    try:
        bk.bkref_maxflow(warm)
        for k, (fg, bg) in enumerate(steps, 1):
            seed_calls(warm, fg, bg)
            e = bk.bkref_maxflow(warm)
            cold = fresh(k)
            try:
                ce = bk.bkref_maxflow(cold)
                assert [bk.bkref_what_segment(warm, v) for v in range(n)] == [bk.bkref_what_segment(cold, v) for v in range(n)]
                assert abs(e - ce) <= 1e-9 * abs(ce)
            finally:
                bk.bkref_delete(cold)
    finally:
        bk.bkref_delete(warm)
