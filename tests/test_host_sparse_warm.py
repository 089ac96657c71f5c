"""Warm re-solves of general sparse graphs on the host: the claim they rest on, pinned on the unmodified reference BK;
the fold bodies of medpy_b200/csrc/gc_sparse_warm.cuh run on the CPU (tests/emu/sparse_warm_emu.cpp) as
solve -> fold -> continue against BK; and the Python routing of GraphDouble(sparse=True, warm=True), GCGraph and
graph_from_labels(warm=True) with a test double of the native class."""
import ctypes
import os
import subprocess
import sys

import numpy
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import fake_native  # noqa: E402
from oracle import energy_label_terms as elt  # noqa: E402
from oracle import solvers  # noqa: E402
from test_host_seeds import _reference_bk  # noqa: E402


# ---- random call sequences ----------------------------------------------------------------------------------------
def _first_graph(rng, n, m, integer):
    i = rng.integers(0, n, size=m)
    j = rng.integers(0, n, size=m)
    keep = i != j
    i, j = i[keep], j[keep]
    if integer:
        cap, rev = (rng.integers(1, 20, size=i.size).astype(float) for _ in range(2))
        src, snk = (rng.integers(0, 30, size=n).astype(float) for _ in range(2))
    else:
        cap, rev = (rng.uniform(1e-3, 2.0, size=i.size) for _ in range(2))
        src, snk = (rng.uniform(0, 3.0, size=n) for _ in range(2))
    return (i, j, cap, rev), [(numpy.arange(n), src, snk)]


def _round(rng, n, integer, pairs):
    """One round of mixed edits: t-links of both signs, seeds added and erased, sum_edge on existing pairs in both
    orientations and on new pairs.  Returns (t-link calls, edge calls)."""
    k = max(1, n // 8)
    v = rng.integers(0, n, size=k)
    if integer:
        s, t = rng.integers(-10, 20, size=k).astype(float), rng.integers(-10, 20, size=k).astype(float)
    else:
        s, t = rng.uniform(-2, 4, size=k), rng.uniform(-2, 4, size=k)
    fg = rng.choice(n, size=max(1, n // 20), replace=False)
    bg = rng.choice(n, size=max(1, n // 20), replace=False)
    tw = [(v, s, t),
          (fg, numpy.full(fg.size, 65535.0), numpy.zeros(fg.size)),
          (bg, numpy.zeros(bg.size), numpy.full(bg.size, 65535.0)),
          (fg[: fg.size // 2], numpy.full(fg.size // 2, -65535.0), numpy.zeros(fg.size // 2))]   # half the fg erased
    q = max(1, len(pairs) // 6)
    pick = rng.integers(0, len(pairs), size=q)
    ei = numpy.asarray([pairs[p][0] for p in pick])
    ej = numpy.asarray([pairs[p][1] for p in pick])
    flip = rng.random(q) < 0.5
    ei, ej = numpy.where(flip, ej, ei), numpy.where(flip, ei, ej)
    ni = rng.integers(0, n, size=q)
    nj = rng.integers(0, n, size=q)
    keep = ni != nj
    ei, ej = numpy.concatenate([ei, ni[keep]]), numpy.concatenate([ej, nj[keep]])
    if integer:
        c, r = rng.integers(0, 10, size=ei.size).astype(float), rng.integers(0, 10, size=ei.size).astype(float)
    else:
        c, r = rng.uniform(0, 2, size=ei.size), rng.uniform(0, 2, size=ei.size)
    return tw, (ei, ej, c, r)


def _pairs_of(edges):
    seen = {}
    for a, b in zip(*edges[:2]):
        seen.setdefault((min(a, b), max(a, b)), None)
    return list(seen)


def _check(got_e, got_mask, n, edges, tw, integer, rel=1e-12):
    flow, mask, _ = solvers.solve_sparse(n, *edges, tw)
    assert numpy.array_equal(numpy.asarray(got_mask), mask)
    if integer:
        assert got_e == flow
    else:
        assert got_e == pytest.approx(flow, rel=rel, abs=1e-9)


def _cat(e1, e2):
    return tuple(numpy.concatenate([a, b]) for a, b in zip(e1, e2))


# ---- the unmodified reference BK --------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_reference_bk_resolve_after_calls_equals_from_scratch(seed):
    """BK's add_tweights / sum_edge act on the residual graph: solve, add t-links of both signs, sum_edge on existing
    pairs in both orientations and on new pairs, seeds added and erased, solve again == a fresh solve of all calls."""
    bk = _reference_bk()
    if bk is None:
        pytest.skip("oracle/_ref (the reference BK) was not built")
    rng = numpy.random.default_rng(seed)
    integer = seed % 2 == 0
    n = int(rng.integers(8, 200))
    edges, tw = _first_graph(rng, n, int(rng.integers(n, 5 * n)), integer)
    h = bk.bkref_new(n, 4 * edges[0].size + 64)
    try:
        for a, b, c, r in zip(*[x.tolist() for x in edges]):
            bk.bkref_sum_edge(h, a, b, c, r)
        for v, s, t in zip(*[x.tolist() for x in tw[0]]):
            bk.bkref_add_tweights(h, v, s, t)
        bk.bkref_maxflow(h)
        for _ in range(3):
            tw_r, e_r = _round(rng, n, integer, _pairs_of(edges))
            for a, b, c, r in zip(*[x.tolist() for x in e_r]):
                bk.bkref_sum_edge(h, a, b, c, r)
            for op in tw_r:
                for v, s, t in zip(*[numpy.asarray(x).tolist() for x in op]):
                    bk.bkref_add_tweights(h, v, s, t)
            edges, tw = _cat(edges, e_r), tw + tw_r
            e = bk.bkref_maxflow(h)
            mask = numpy.asarray([0 if bk.bkref_what_segment(h, v) == 1 else 1 for v in range(n)], numpy.uint8)
            _check(e, mask, n, edges, tw, integer)
    finally:
        bk.bkref_delete(h)


# ---- the fold bodies on the host --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libsparse_warm_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", so,
                           os.path.join(HERE, "emu", "sparse_warm_emu.cpp")])
    lib = ctypes.CDLL(so)
    ip, dp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)
    lib.emu_warm_create.restype = ctypes.c_void_p
    lib.emu_warm_create.argtypes = [ctypes.c_int]
    lib.emu_warm_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_warm_solve.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_uint8), dp]
    lib.emu_warm_tweights.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ip, dp, dp]
    for f in (lib.emu_warm_edges, lib.emu_warm_remove):
        f.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ip, ip, dp, dp]
    lib.emu_warm_remove.restype = ctypes.c_int
    lib.emu_warm_host.restype = ctypes.c_longlong
    lib.emu_warm_host.argtypes = [ctypes.c_void_p, ip, ip, dp, dp, dp, dp]
    return lib


class _Emu:
    """One warm handle of the emulation: created from the first call sequence, then folded and re-solved."""

    def __init__(self, lib, n, edges, tw, steps=4, sweeps=16):
        self.lib, self.n, self.steps, self.sweeps = lib, n, steps, sweeps
        self.h = lib.emu_warm_create(n)
        self.edges(*edges)
        for op in tw:
            self.tweights(*op)
        # the C ABI's host state of the raw calls against the oracle's replay of them
        np_ = lib.emu_warm_host(self.h, None, None, None, None, None, None)
        lo, hi = numpy.zeros(np_, numpy.int32), numpy.zeros(np_, numpy.int32)
        c_lh, c_hl, tr, const = numpy.zeros(np_), numpy.zeros(np_), numpy.zeros(n), numpy.zeros(1)
        lib.emu_warm_host(self.h, *[self._p(x) for x in (lo, hi, c_lh, c_hl, tr, const)])
        order = numpy.lexsort((hi, lo))
        for got, want in zip((lo, hi, c_lh, c_hl), elt.merge_edges(*edges)):
            assert numpy.array_equal(got[order], want)
        want_tr, want_const = elt.add_tweights_replay(n, tw)
        assert numpy.array_equal(tr, want_tr) and const[0] == want_const

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int if a.dtype == numpy.int32 else ctypes.c_double))

    def solve(self):
        mask = numpy.zeros(self.n, numpy.uint8)
        e = ctypes.c_double(0)
        assert self.lib.emu_warm_solve(self.h, self.steps, self.sweeps, mask.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)),
                                       ctypes.byref(e)) == 0
        return e.value, mask

    def tweights(self, v, s, t):
        a = [numpy.ascontiguousarray(v, dtype=numpy.int32), numpy.ascontiguousarray(s, dtype=float), numpy.ascontiguousarray(t, dtype=float)]
        self.lib.emu_warm_tweights(self.h, a[0].size, *[self._p(x) for x in a])

    def _edges(self, fn, i, j, c, r):
        a = [numpy.ascontiguousarray(i, dtype=numpy.int32), numpy.ascontiguousarray(j, dtype=numpy.int32),
             numpy.ascontiguousarray(c, dtype=float), numpy.ascontiguousarray(r, dtype=float)]
        return fn(self.h, a[0].size, *[self._p(x) for x in a])

    def edges(self, *e):
        self._edges(self.lib.emu_warm_edges, *e)

    def remove(self, *e):
        return self._edges(self.lib.emu_warm_remove, *e)

    def __del__(self):
        self.lib.emu_warm_destroy(self.h)


@pytest.mark.parametrize("seed", range(16))
def test_emulated_folds_continue_to_the_bk_cut(emu, seed):
    """Solve, then three rounds of t-links of both signs, seeds added and erased, increments on existing pairs in both
    orientations and on new pairs, and exact decrements of part of the first weights; each round re-solved from the
    residual state equals BK's fresh solve of the whole call sequence."""
    rng = numpy.random.default_rng(100 + seed)
    integer = seed % 2 == 0
    n = int(rng.integers(4, 160))
    edges, tw = _first_graph(rng, n, int(rng.integers(1, 5 * n)), integer)
    g = _Emu(emu, n, edges, tw, steps=1 + seed % 4, sweeps=1 + 5 * (seed % 3))
    e, mask = g.solve()
    _check(e, mask, n, edges, tw, integer)
    for _ in range(3):
        tw_r, e_r = _round(rng, n, integer, _pairs_of(edges))
        g.edges(*e_r)
        for op in tw_r:
            g.tweights(*op)
        edges, tw = _cat(edges, e_r), tw + tw_r
        # decrements: part of what some pairs hold now, as BK's sum_edge with negated values
        lo, hi, c_lh, c_hl = elt.merge_edges(*edges)
        pick = rng.choice(lo.size, size=max(1, lo.size // 5), replace=False)
        frac = rng.integers(0, 3, size=pick.size) / 2.0 if integer else rng.uniform(0, 1, size=pick.size)
        d_lh, d_hl = numpy.floor(c_lh[pick] * frac) if integer else c_lh[pick] * frac, numpy.zeros(pick.size)
        if not integer:
            d_hl = c_hl[pick] * rng.uniform(0, 1, size=pick.size) * (rng.random(pick.size) < 0.5)
        assert g.remove(lo[pick], hi[pick], d_lh, d_hl) == 0
        edges = _cat(edges, (lo[pick], hi[pick], -d_lh, -d_hl))
        e, mask = g.solve()
        _check(e, mask, n, edges, tw, integer, rel=1e-9)


def test_hand_check_lowered_middle_arc(emu):
    """s ->5-> i ->5-> j ->5-> t solved (energy 5), c(i -> j) lowered by 3: the re-solve gives exactly 2."""
    edges = (numpy.asarray([0]), numpy.asarray([1]), numpy.asarray([5.0]), numpy.asarray([0.0]))
    tw = [(numpy.asarray([0, 1]), numpy.asarray([5.0, 0.0]), numpy.asarray([0.0, 5.0]))]
    g = _Emu(emu, 2, edges, tw)
    assert g.solve()[0] == 5.0
    assert g.remove([0], [1], [3.0], [0.0]) == 0
    e, mask = g.solve()
    assert e == 2.0
    _check(e, mask, 2, _cat(edges, (numpy.asarray([0]), numpy.asarray([1]), numpy.asarray([-3.0]), numpy.asarray([0.0]))), tw, True)


def test_exact_removal_accepted_and_more_refused(emu):
    rng = numpy.random.default_rng(5)
    n = 40
    edges, tw = _first_graph(rng, n, 120, False)
    g = _Emu(emu, n, edges, tw)
    e0, m0 = g.solve()
    lo, hi, c_lh, c_hl = elt.merge_edges(*edges)
    assert g.remove(lo[:3], hi[:3], c_lh[:3] * (1 + 1e-6), c_hl[:3]) == 1          # refused, nothing changed
    e, mask = g.solve()
    assert e == e0 and numpy.array_equal(mask, m0)
    assert g.remove(lo[:3], hi[:3], c_lh[:3], c_hl[:3]) == 0                      # exactly what is there
    e, mask = g.solve()
    _check(e, mask, n, _cat(edges, (lo[:3], hi[:3], -c_lh[:3], -c_hl[:3])), tw, False, rel=1e-9)


def test_tlink_calls_of_a_node_apply_in_order(emu):
    """add_tweights(v, 2^53, 0), (v, 0, 2^53), (v, 1, 0) leaves r = 1 in BK's order; summed first they would leave 0
    (2^53 + 1 rounds to 2^53), and v -- tied to a sink node by an arc of 0.5 -- would fall on the sink side."""
    big = float(2 ** 53)
    edges = (numpy.asarray([0]), numpy.asarray([1]), numpy.asarray([0.5]), numpy.asarray([0.0]))
    tw = [(numpy.asarray([1]), numpy.asarray([0.0]), numpy.asarray([10.0]))]
    g = _Emu(emu, 2, edges, tw)
    g.solve()
    calls = (numpy.asarray([0, 0, 0]), numpy.asarray([big, 0.0, 1.0]), numpy.asarray([0.0, big, 0.0]))
    g.tweights(*calls)
    e, mask = g.solve()
    assert mask.tolist() == [1, 0]
    _check(e, mask, 2, edges, tw + [calls], True)


def test_source_residual_released_through_a_new_arc(emu):
    """An fg seed whose push was clamped at its out-capacity gets a new arc to a sink node: the un-pushed source residual
    must flow through it, otherwise the seed would be cut off on the sink side's terms."""
    edges = (numpy.asarray([0]), numpy.asarray([1]), numpy.asarray([1.0]), numpy.asarray([1.0]))
    tw = [(numpy.asarray([0, 1, 2]), numpy.asarray([65535.0, 0.0, 0.0]), numpy.asarray([0.0, 2.0, 50.0]))]
    g = _Emu(emu, 3, edges, tw)
    g.solve()
    new = (numpy.asarray([0]), numpy.asarray([2]), numpy.asarray([30.0]), numpy.asarray([0.0]))
    g.edges(*new)
    e, mask = g.solve()
    assert e == 31.0
    _check(e, mask, 3, _cat(edges, new), tw, True)


def test_clamp_reads_residual_out_capacity(emu):
    """Node 0 pushes its 4 units into node 1, whose sink link absorbs them: node 1 then has a reverse residual of 4 and
    no original out-capacity.  An fg seed on node 1 must send 2 back through 0 -> 2 (energy 6); a clamp on the original
    capacities would push nothing and leave 4."""
    edges = (numpy.asarray([0, 0]), numpy.asarray([1, 2]), numpy.asarray([4.0, 2.0]), numpy.asarray([0.0, 0.0]))
    tw = [(numpy.asarray([0, 1, 2]), numpy.asarray([4.0, 0.0, 0.0]), numpy.asarray([0.0, 4.0, 10.0]))]
    g = _Emu(emu, 3, edges, tw)
    assert g.solve()[0] == 4.0
    calls = (numpy.asarray([1]), numpy.asarray([65535.0]), numpy.asarray([0.0]))
    g.tweights(*calls)
    e, mask = g.solve()
    assert e == 6.0 and mask.tolist() == [1, 1, 0]
    _check(e, mask, 3, edges, tw + [calls], True)


def test_absorbed_flow_counted_once_after_a_sink_fold(emu):
    rng = numpy.random.default_rng(9)
    n = 30
    edges, tw = _first_graph(rng, n, 90, True)
    g = _Emu(emu, n, edges, tw)
    g.solve()
    calls = (numpy.arange(n), numpy.zeros(n), numpy.full(n, 3.0))     # every sink link grows
    g.tweights(*calls)
    e, mask = g.solve()
    _check(e, mask, n, edges, tw + [calls], True)


# ---- Python routing with a test double of the native class -----------------------------------------------------------
class _WarmSparse(fake_native.FakeSparseGraph):
    """FakeSparseGraph plus the warm option and remove_edges_warm; every call is logged.  Results are fresh solves of
    the calls so far, which is what a warm re-solve must equal."""

    log = []

    def __init__(self, n_nodes, device=-1):
        self.options = {}
        super().__init__(n_nodes, device)
        _WarmSparse.log.append(self)
        self.calls = []

    def set_option(self, option, value):
        self.options[option] = value

    def sum_edges(self, i, j, cap, rev):
        self.calls.append("sum_edges")
        super().sum_edges(i, j, cap, rev)

    def add_tweights(self, nodes, src, snk):
        self.calls.append("add_tweights")
        super().add_tweights(nodes, src, snk)

    def remove_edges_warm(self, i, j, cap, rev):
        assert "OPT" in str(self.options) or self.options, "remove_edges_warm needs the option"
        self.calls.append("remove_edges_warm")
        super().sum_edges(i, j, -numpy.asarray(cap, dtype=float), -numpy.asarray(rev, dtype=float))

    def maxflow(self):
        self.calls.append("maxflow")
        return super().maxflow()


@pytest.fixture()
def fake(monkeypatch):
    from medpy_b200 import _lib
    _WarmSparse.log = []
    monkeypatch.setattr(_lib._mgc, "SparseGraph", _WarmSparse)
    monkeypatch.setattr(_lib._mgc, "LabelImage", fake_native.FakeLabelImage)
    return _WarmSparse.log


def _small(warm=True):
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(6, 8, sparse=True, warm=warm)
    g.add_tweights(0, 10.0, 0.0)
    g.add_tweights(5, 0.0, 10.0)
    for a, b in ((0, 1), (1, 2), (2, 5), (0, 3), (3, 4), (4, 5)):
        g.sum_edge(a, b, 2.0, 1.0)
    return g


def test_option_reaches_the_handle_and_survives_reset(fake):
    from medpy_b200 import _lib
    g = _small()
    g.maxflow()
    assert fake[0].options == {_lib._mgc.OPT_WARM: 1}
    g.reset()
    assert g._sp.warm and fake[0].options == {_lib._mgc.OPT_WARM: 1}
    g.enable_warm()                                  # already warm: nothing to do
    h = _small(warm=False)
    h.maxflow()
    assert fake[1].options == {}


def test_warm_requires_sparse():
    from medpy_b200.graphcut import GCGraph
    from medpy_b200.graphcut.maxflow import GraphDouble
    with pytest.raises(ValueError, match="sparse=True"):
        GraphDouble(4, 4, warm=True)
    with pytest.raises(ValueError, match="sparse=True"):
        GCGraph(4, 4, warm=True)
    assert GCGraph(4, 4, sparse=True, warm=True).get_graph()._sp.warm


def test_plain_calls_after_a_solve_fold(fake):
    g = _small()
    e0 = g.maxflow()
    g.add_tweights(2, 0.0, 7.0)
    g.sum_edge(1, 4, 3.0, 3.0)                       # a new pair
    g.add_tweights_bulk(numpy.asarray([3]), numpy.asarray([1.0]), numpy.asarray([0.0]))
    g.sum_edges_bulk(numpy.asarray([2]), numpy.asarray([1]), numpy.asarray([0.5]), numpy.asarray([0.25]))
    assert fake[0].calls == ["sum_edges", "add_tweights", "maxflow"]        # staged until the next solve
    e1 = g.maxflow()
    assert fake[0].calls[3:] == ["add_tweights", "add_tweights", "sum_edges", "sum_edges", "maxflow"]
    assert g._sp._solved and e1 == fake[0].maxflow()
    assert g.get_edge(1, 4) == 3.0 and g.get_edge(2, 1) == 1.5


def test_warm_calls_route_to_the_sparse_backend(fake):
    g = _small()
    g.maxflow()
    mask = numpy.zeros(6, bool)
    mask[2] = True
    g.add_seeds(fg=mask, bg=numpy.asarray([4]))
    g.remove_seeds(bg=[4])
    g.add_tweights_warm(None, numpy.zeros(6), numpy.full(6, 0.5))
    g.add_tweights_warm([1, 1], 1.0, [0.0, 2.0])
    g.add_nweights_warm([0, 3], [5, 2], 1.0, [0.0, 4.0])
    # CPU tensors, a single id, and one-element id arrays that broadcast to the other arguments' length
    g.add_seeds(fg=torch.tensor([3]), bg=5)
    g.add_tweights_warm(torch.tensor([2, 0], dtype=torch.int32), torch.tensor([1.5, -1.0]), torch.tensor(0.25))
    g.add_nweights_warm([1], torch.tensor([4, 2]), 0.5, [1.0, 0.0])
    g.maxflow()
    nat = fake[0]
    tw_nodes = [None if t[0] is None else numpy.asarray(t[0]).tolist() for t in nat.tw[1:]]
    assert tw_nodes == [[2], [4], [4], list(range(6)), [1, 1], [3], [5], [2, 0]]
    assert nat.tw[3][1].tolist() == [0.0] and nat.tw[3][2].tolist() == [-65535.0]
    assert nat.tw[-1][1].tolist() == [1.5, -1.0] and nat.tw[-1][2].tolist() == [0.25, 0.25]
    assert nat.e[0][-4:].tolist() == [0, 3, 1, 1] and nat.e[1][-4:].tolist() == [5, 2, 4, 2]
    assert nat.e[2][-2:].tolist() == [0.5, 0.5] and nat.e[3][-2:].tolist() == [1.0, 0.0]


def test_remove_flushes_staged_calls_first(fake):
    g = _small()
    g.sum_edge(1, 2, 1.0, 0.0)                       # before the first solve: staged
    g.remove_nweights_warm([1], [2], 2.5, 0.0)       # works unsolved too; the staged call lands first
    assert fake[0].calls == ["sum_edges", "add_tweights", "remove_edges_warm"]
    g.maxflow()
    g.sum_edge(0, 1, 1.0, 1.0)
    g.remove_nweights_warm([0], [1], 0.5, 0.5)
    assert fake[0].calls[-2:] == ["sum_edges", "remove_edges_warm"]


def test_bad_arguments_are_refused(fake):
    g = _small()
    for call in (lambda: g.add_nweights_dense_warm(0, numpy.zeros(6), numpy.zeros(6)),
                 lambda: g.remove_nweights_dense_warm(0, numpy.zeros(6), numpy.zeros(6))):
        with pytest.raises(ValueError, match="axes"):
            call()
    with pytest.raises(ValueError):
        g.add_tweights_warm([1], float("nan"), 0.0)
    with pytest.raises(ValueError):
        g.add_seeds(fg=numpy.zeros(5, bool))
    with pytest.raises(ValueError):
        g.add_seeds(fg=[6])
    with pytest.raises(ValueError):
        g.add_seeds(fg=numpy.zeros((2, 3), bool))      # a sparse mask has shape (n,)
    with pytest.raises(ValueError, match="differ in length"):
        g.add_nweights_warm([], [1], 1.0, 0.0)
    with pytest.raises(ValueError):
        g.remove_nweights_warm([0], [1], -1.0, 0.0)
    with pytest.raises(ValueError):
        g.add_nweights_warm([0], [0], 1.0, 0.0)
    g.maxflow()
    with pytest.raises(ValueError, match="remove_nweights_warm"):
        g.sum_edge(0, 1, -1.0, 0.0)
    with pytest.raises(ValueError):
        g.sum_edge(0, 1, float("inf"), 0.0)
    with pytest.raises(ValueError):
        g.add_tweights(0, float("nan"), 0.0)
    with pytest.raises(ValueError):
        g.add_tweights_bulk(None, numpy.full(6, numpy.inf), numpy.zeros(6))


def test_non_warm_graphs_are_unchanged(fake):
    g = _small(warm=False)
    g.maxflow()
    g.sum_edge(0, 1, -1.0, 0.0)                      # the reference's sum_edge takes it (cold re-solve)
    g.add_tweights(0, float("nan"), 0.0)
    assert not g._sp._solved and not g._sp.warm
    with pytest.raises(TypeError):
        g.enable_warm()
    g._solved = True
    for call in (lambda: g.add_seeds(fg=[1]), lambda: g.add_nweights_warm([1], [2], 1.0, 0.0)):
        with pytest.raises(RuntimeError, match="reset.*rebuild"):
            call()


def test_graph_from_labels_warm_keyword(fake):
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut import energy_label
    lab = numpy.asarray([[1, 1, 2, 2], [3, 3, 4, 4], [3, 5, 5, 4]], numpy.int32)
    fg = numpy.zeros(lab.shape, bool)
    bg = numpy.zeros(lab.shape, bool)
    fg[0, 0] = True
    bg[2, 3] = True
    grad = numpy.arange(lab.size, dtype=float).reshape(lab.shape) / 10
    g = gc.graph_from_labels(lab, fg, bg, boundary_term=energy_label.boundary_stawiaski, boundary_term_args=grad, warm=True)
    assert g._sp.warm
    g.maxflow()
    g.add_seeds(bg=numpy.asarray([1]))
    m = gc.label_cut_mask(g)
    assert m.shape == lab.shape and not m[lab == 2].any()
    assert not gc.graph_from_labels(lab, fg, bg)._sp.warm
