"""Warm re-solves of general sparse graphs on the GPU (GraphDouble(sparse=True, warm=True), graph_from_labels(warm=True);
csrc/gc_sparse_warm.cuh): rounds of t-links of both signs, seeds added and erased, increments on existing and new pairs
and exact decrements, each re-solved from the residual state and checked against BK's fresh solve of the whole call
sequence (oracle.solvers.solve_sparse) under MEDPY_GC_SPARSE_SWEEPS = 1, 16 and 64."""
import os
import sys
from contextlib import contextmanager

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import region_cases as rc  # noqa: E402
from oracle import solvers  # noqa: E402

pytestmark = pytest.mark.gpu


@contextmanager
def _env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


FAMILIES = {
    "random-int": lambda: rc.random_graph(31, 3000, 12000, True),
    "random-float": lambda: rc.random_graph(32, 3000, 12000, False),
    "grid": lambda: rc.grid_graph(33, (24, 24)),
    "bipartite": lambda: rc.bipartite_graph(34, side=60),
    "chain": lambda: rc.chain_graph(35, 150, True),
    "star": lambda: rc.star_graph(36, leaves=2000),
    "ties-zero-reversed": lambda: rc.ties_graph(37, "zero_and_reversed"),
    "ties-isolated-tlinks": lambda: rc.ties_graph(38, "isolated_and_repeated_tlinks"),
    "ties-no-edges": lambda: rc.ties_graph(39, "no_edges"),
}


class _Replay:
    """The call sequence of a graph, for BK's fresh solve."""

    def __init__(self, case):
        self.n = case["n"]
        self.e = [case["i"], case["j"], case["cap"], case["rev"]]
        self.tw = list(case["tw"])
        self.exact = case["exact"]

    def edges(self, i, j, c, r):
        self.e = [numpy.concatenate([a, numpy.asarray(b, a.dtype)]) for a, b in zip(self.e, (i, j, c, r))]

    def check(self, g):
        """Masks equal; on float graphs a differing mask must be another minimum cut (same capacity to 1e-12): the
        warm arithmetic rounds the residual t-links differently from a fresh replay, and where a cut runs through arcs of
        DBL_MIN (the grid family) a node whose terminal capacity is a rounding away from 0 can go either way."""
        e = g.maxflow()
        mask = g.get_mask()
        flow, want, _ = solvers.solve_sparse(self.n, *self.e, self.tw)
        if not numpy.array_equal(mask, want):
            assert not self.exact, int((mask != want).sum())
            case = dict(n=self.n, i=self.e[0], j=self.e[1], cap=self.e[2], rev=self.e[3], tw=self.tw)
            got_cut, want_cut = rc.cut_capacity(case, mask), rc.cut_capacity(case, want)
            assert got_cut == pytest.approx(want_cut, rel=1e-12), (int((mask != want).sum()), got_cut, want_cut)
        if self.exact:
            assert e == flow
        else:
            assert e == pytest.approx(flow, rel=1e-9, abs=1e-9)
        return e, mask


def _build(case, warm):
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(case["n"], case["i"].size, sparse=True, warm=warm)
    for nodes, src, snk in case["tw"]:
        g.add_tweights_bulk(nodes, src, snk)
    if case["i"].size:
        g.sum_edges_bulk(case["i"], case["j"], case["cap"], case["rev"])
    return g


def _round(rng, g, rep, integer):
    n = rep.n
    k = max(1, n // 10)
    v = rng.integers(0, n, size=k)
    if integer:
        s, t = rng.integers(-5, 10, size=k).astype(float), rng.integers(-5, 10, size=k).astype(float)
    else:
        s, t = rng.uniform(-1, 3, size=k), rng.uniform(-1, 3, size=k)
    g.add_tweights_warm(v, s, t)
    rep.tw.append((v, s, t))
    fg = rng.choice(n, size=max(1, n // 50), replace=False)
    bg = rng.choice(n, size=max(1, n // 50), replace=False)
    g.add_seeds(fg=fg, bg=bg)
    rep.tw += [(fg, numpy.full(fg.size, 65535.0), numpy.zeros(fg.size)), (bg, numpy.zeros(bg.size), numpy.full(bg.size, 65535.0))]
    er = fg[: fg.size // 2]
    g.remove_seeds(fg=er)
    rep.tw.append((er, numpy.full(er.size, -65535.0), numpy.zeros(er.size)))
    # increments on existing pairs (either orientation) and on new pairs
    m = rep.e[0].size
    q = max(1, min(m, n) // 10)
    ii = numpy.concatenate([rep.e[1][rng.integers(0, m, size=q)] if m else numpy.zeros(0, numpy.int64), rng.integers(0, n, size=q)])
    jj = numpy.concatenate([rep.e[0][rng.integers(0, m, size=q)] if m else numpy.zeros(0, numpy.int64), rng.integers(0, n, size=q)])
    keep = ii != jj
    ii, jj = ii[keep], jj[keep]
    c = rng.integers(0, 5, size=ii.size).astype(float) if integer else rng.uniform(0, 2, size=ii.size)
    r = rng.integers(0, 5, size=ii.size).astype(float) if integer else rng.uniform(0, 2, size=ii.size)
    g.add_nweights_warm(ii, jj, c, r)
    rep.edges(ii, jj, c, r)
    # exact decrements of what a few pairs hold, and one 1e-6 too large, refused with the graph unchanged
    if rep.e[0].size:
        pick = rng.integers(0, rep.e[0].size, size=max(1, q // 2))
        pairs = sorted({(int(min(a, b)), int(max(a, b))) for a, b in zip(rep.e[0][pick], rep.e[1][pick])})
        di = numpy.asarray([p[0] for p in pairs])
        dj = numpy.asarray([p[1] for p in pairs])
        dc = numpy.asarray([g.get_edge(a, b) for a, b in pairs])
        dr = numpy.asarray([g.get_edge(b, a) for a, b in pairs])
        big = numpy.argmax(dc)
        if dc[big] > 0:
            before = g.maxflow(), g.get_mask().copy()
            with pytest.raises(ValueError):
                g.remove_nweights_warm(di[big:big + 1], dj[big:big + 1], dc[big:big + 1] * (1 + 1e-6), dr[big:big + 1])
            assert g.maxflow() == before[0] and numpy.array_equal(g.get_mask(), before[1])
        g.remove_nweights_warm(di, dj, dc, dr)
        rep.edges(di, dj, -dc, -dr)


@pytest.mark.parametrize("sweeps", [1, 16, 64])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_rounds_of_mixed_edits_match_bk(family, sweeps):
    case = FAMILIES[family]()
    rng = numpy.random.default_rng(100 * sorted(FAMILIES).index(family) + sweeps)
    with _env(MEDPY_GC_SPARSE_SWEEPS=sweeps):
        g = _build(case, True)
        rep = _Replay(case)
        rep.check(g)
        for _ in range(3):
            _round(rng, g, rep, case["exact"])
            rep.check(g)


@pytest.mark.parametrize("family", ["random-int", "random-float", "grid"])
def test_first_solve_equals_cold(family):
    case = FAMILIES[family]()
    cold, warm = _build(case, False), _build(case, True)
    ec, ew = cold.maxflow(), warm.maxflow()
    assert numpy.array_equal(cold.get_mask(), warm.get_mask())
    if case["exact"]:
        assert ec == ew
    else:
        assert ew == pytest.approx(ec, rel=1e-12)
    assert warm.stats()["device_bytes"] > cold.stats()["device_bytes"]


def test_seed_undo_gives_back_the_mask():
    case = FAMILIES["random-float"]()
    g = _build(case, True)
    e0 = g.maxflow()
    m0 = g.get_mask().copy()
    rng = numpy.random.default_rng(3)
    fg, bg = rng.choice(case["n"], 40, replace=False), rng.choice(case["n"], 40, replace=False)
    g.add_seeds(fg=fg, bg=bg)
    g.maxflow()
    assert not numpy.array_equal(g.get_mask(), m0)
    g.remove_seeds(fg=fg, bg=bg)
    assert g.maxflow() == pytest.approx(e0, rel=1e-9)
    assert numpy.array_equal(g.get_mask(), m0)


def test_hand_check_and_refusals_and_reset():
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(2, 1, sparse=True, warm=True)
    g.add_tweights(0, 5.0, 0.0)
    g.add_tweights(1, 0.0, 5.0)
    g.sum_edge(0, 1, 5.0, 0.0)
    assert g.maxflow() == 5.0
    with pytest.raises(ValueError):
        g.remove_nweights_warm([0], [1], 5.0 * (1 + 1e-6), 0.0)
    with pytest.raises(ValueError):
        g.add_tweights_warm([0], float("nan"), 0.0)
    with pytest.raises(ValueError):
        g.sum_edge(0, 1, -1.0, 0.0)
    assert g.maxflow() == 5.0
    g.remove_nweights_warm([0], [1], 3.0, 0.0)
    assert g.maxflow() == 2.0 and g.get_edge(0, 1) == 2.0
    g.reset()
    assert g._sp.warm
    g.add_tweights(0, 1.0, 0.0)
    g.add_tweights(1, 0.0, 1.0)
    g.sum_edge(0, 1, 3.0, 0.0)
    assert g.maxflow() == 1.0
    g.add_tweights(0, 2.0, 0.0)                    # both fold
    g.add_tweights(1, 0.0, 2.0)
    assert g.maxflow() == 3.0 and g.get_trcap(0) == 3.0 and g.get_arc_num() == 2
    with pytest.raises(ValueError):
        g.add_nweights_dense_warm(0, numpy.zeros(2), numpy.zeros(2))
    # host and device arguments mix in one call: a sparse graph copies every argument to the host
    import torch
    g.add_tweights_warm(torch.tensor([0, 1], device="cuda"), numpy.array([1.0, 0.0]), torch.tensor([0.0, 1.0], device="cuda"))
    assert g.maxflow() == 3.0
    g.add_nweights_warm(torch.tensor([0], device="cuda"), [1], numpy.array([1.0]), 0.0)
    assert g.maxflow() == 4.0


def test_nonfinite_first_solve_refuses_folds():
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(3, 2, sparse=True, warm=True)
    g.add_tweights(0, float("inf"), 0.0)
    g.add_tweights(2, 0.0, 1.0)
    g.sum_edge(0, 1, 1.0, 0.0)
    g.sum_edge(1, 2, 1.0, 0.0)
    g.maxflow()
    g.add_tweights(1, 1.0, 0.0)
    with pytest.raises(RuntimeError, match="reset"):
        g.maxflow()


def test_region_graph_strokes_match_the_replay():
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut import energy_label
    vol = rc.label_volume(3)
    lab = vol["label"]
    fg, bg = rc.markers(lab, 5)
    grad = rc.gradient(lab.shape, "float64", 6)
    kw = dict(boundary_term=energy_label.boundary_stawiaski, boundary_term_args=grad)
    warm = gc.graph_from_labels(lab, fg, bg, warm=True, **kw)
    warm.maxflow()
    rng = numpy.random.default_rng(8)
    strokes = []
    for k in range(3):
        ids = rng.choice(vol["regions"], size=20, replace=False)
        strokes.append(("add_seeds", dict(fg=ids[:10], bg=ids[10:])) if k != 1 else ("remove_seeds", dict(fg=ids[:10])))
        getattr(warm, strokes[-1][0])(**strokes[-1][1])
        got = gc.label_cut_mask(warm)
        cold = gc.graph_from_labels(lab, fg, bg, **kw)
        for name, args in strokes:
            cap = 65535.0 if name == "add_seeds" else -65535.0
            for side, ids_ in args.items():
                src, snk = (cap, 0.0) if side == "fg" else (0.0, cap)
                cold.add_tweights_bulk(ids_, numpy.full(ids_.size, src), numpy.full(ids_.size, snk))
        want = gc.label_cut_mask(cold)
        assert numpy.array_equal(got, want)
        assert warm.maxflow() == pytest.approx(cold.maxflow(), rel=1e-9)
