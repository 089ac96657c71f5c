"""The region-graph path on the GPU at scale and on adversarial inputs (SURVEY.md §8 rows f3/f4): the four energy_label
terms and graph_from_labels against the label-term oracle (oracle/energy_label_terms.py), and general graphs built
through GCGraph / GraphDouble(sparse=True) against BK (oracle.solvers.solve_sparse).

The oracle squares with math.pow(r, 2) like the reference; the device forms the correctly rounded r*r.  With the oracle's
_pow2 replaced by numpy.square every contribution is the same float64 and merge_edges adds each region pair's
contributions front to back in the reference's order -- the order the device keeps -- so every device weight must equal
the oracle bit for bit, for every gradient dtype and every term.  test_fuzz_cases_within_tolerance_of_the_pow_oracle
compares once against the unpatched oracle so the substitution cannot hide a real difference.

A. the 150 seeded fuzz cases of tests/golden/fuzz_labels_v1.json (the oracle is pinned to the reference on them);
B. label volumes in 1-D..4-D with tens of thousands to 10^5 regions (region_cases.label_volume), every gradient dtype
   with its extremes, labels / gradients / atlases in every layout;
C. general graphs (region_cases.GRAPHS) under MEDPY_GC_SPARSE_SWEEPS = 1, 16, 64;
D. building, accumulating into and reusing one sparse graph.
"""
import json
import os
import sys
import time
import warnings
from contextlib import contextmanager

import numpy
import pytest

import region_cases as rc
from test_gpu_labels import Recorder

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import energy_label_terms as elt  # noqa: E402
from oracle import solvers  # noqa: E402

pytestmark = pytest.mark.gpu

TIMEOUT = "300"          # seconds per sparse solve: a stuck solve ends on the host instead of spinning


def _gc():
    import medpy_b200.graphcut as gc
    return gc


@pytest.fixture
def timeout(monkeypatch):
    monkeypatch.setenv("MEDPY_GC_SPARSE_TIMEOUT", TIMEOUT)


@contextmanager
def squared_oracle():
    """The oracle with r*r (numpy.square equals the correctly rounded product in float64) instead of math.pow(r, 2)."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(elt, "_pow2", lambda r: numpy.square(numpy.asarray(r, dtype=numpy.float64)))
        yield


@pytest.fixture
def square(timeout):
    with squared_oracle():
        yield


def _merged(calls):
    """Oracle call list (i, j, there, back) -> (lo, hi, cap lo->hi, cap hi->lo) sorted by (lo, hi)."""
    i, j, a, b = calls
    return elt.merge_edges(i, j, a, b)


def _dict(lo, hi, a, b):
    return {(int(x), int(y)): (u, v) for x, y, u, v in zip(lo.tolist(), hi.tolist(), a.tolist(), b.tolist())}


def _assert_bits(got, want, what, equal_nan=False):
    got = numpy.asarray(got, dtype=numpy.float64)
    want = numpy.asarray(want, dtype=numpy.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if equal_nan:
        nan = numpy.isnan(want)
        assert numpy.array_equal(numpy.isnan(got), nan), what
        got, want = got[~nan], want[~nan]
    bad = numpy.flatnonzero(got.view(numpy.uint64) != want.view(numpy.uint64))
    assert bad.size == 0, (what, bad.size, bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())


class ArrayRecorder:
    """A foreign graph object that keeps the calls in arrays: region pairs must arrive once each, in key order."""

    def __init__(self):
        self.n = ([], [], [], [])
        self.t = ([], [], [])

    def set_nweight(self, a, b, w1, w2):
        for lst, v in zip(self.n, (a, b, w1, w2)):
            lst.append(v)

    def set_tweight(self, node, ws, wk):
        for lst, v in zip(self.t, (node, ws, wk)):
            lst.append(v)

    def edges(self):
        lo, hi = numpy.asarray(self.n[0], numpy.int64), numpy.asarray(self.n[1], numpy.int64)
        key = lo * (1 << 32) + hi
        assert (lo < hi).all() and (key[1:] > key[:-1]).all(), "region pairs out of order or repeated"
        return lo, hi, numpy.asarray(self.n[2], numpy.float64), numpy.asarray(self.n[3], numpy.float64)


def _assert_edges(rec, want, what, equal_nan=False):
    lo, hi, a, b = rec.edges()
    assert numpy.array_equal(lo, want[0]) and numpy.array_equal(hi, want[1]), (what, "region pairs differ")
    _assert_bits(a, want[2], what + " there", equal_nan)
    _assert_bits(b, want[3], what + " back", equal_nan)


def _label_problem(lab, fg, bg, boundary, args, atlas=None):
    """(n, i, j, cap, rev, tw) graph_from_labels builds, in the reference's call order: regional, boundary, markers."""
    n = int(numpy.asarray(lab).max())
    tw = []
    if atlas is not None:
        tw.append(elt.regional_atlas_calls(lab, atlas[0], atlas[1]))
    if boundary == "stawiaski":
        e = elt.stawiaski_calls(lab, args)
    elif boundary == "directed":
        e = elt.stawiaski_directed_calls(lab, args[0], args[1])
    else:
        e = elt.difference_of_means_calls(lab, args)
    fgr, bgr = elt.marker_regions(lab, fg), elt.marker_regions(lab, bg)
    tw.append((fgr, numpy.full(fgr.size, rc.MARKER), numpy.zeros(fgr.size)))
    tw.append((bgr, numpy.zeros(bgr.size), numpy.full(bgr.size, rc.MARKER)))
    return n, e[0], e[1], e[2], e[3], tw


def _term(boundary):
    el = _gc().energy_label
    return {"stawiaski": el.boundary_stawiaski, "directed": el.boundary_stawiaski_directed,
            "means": el.boundary_difference_of_means}[boundary]


def _check_cut(g, problem, exact=False):
    flow = g.maxflow()
    rflow, rmask, _ = solvers.solve_sparse(*problem)
    mask = g.get_mask()
    assert numpy.array_equal(mask, rmask), int((mask != rmask).sum())
    if exact:
        assert flow == rflow
    else:
        assert flow == pytest.approx(rflow, rel=1e-9, abs=1e-300)
    return mask


# ---------------------------------------------------------------------------------------------------------------------
# A. the recorded fuzz cases
# ---------------------------------------------------------------------------------------------------------------------
_FUZZ = []


def _fuzz():
    if not _FUZZ:
        sys.path.insert(0, os.path.join(HERE, "golden"))
        import fuzz_labels_against_reference as fz
        with open(fz.GOLDEN) as fh:
            z = json.load(fh)
        rng = numpy.random.default_rng(z["seed"])
        _FUZZ.extend(fz.random_case(rng) for _ in range(z["cases"]))
    return _FUZZ


def _fuzz_markers(lab, c):
    rng = numpy.random.default_rng(5000 + c)
    fg = rng.random(lab.shape) < 0.2
    bg = rng.random(lab.shape) < 0.2
    fg.flat[0] = True
    bg.flat[-1] = True
    return fg, bg


@pytest.mark.parametrize("c", range(150))
def test_fuzz_case_on_the_device(c, square):
    gc = _gc()
    el = gc.energy_label
    lab, img, prob, alpha, directedness = _fuzz()[c]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        staw = _dict(*_merged(elt.stawiaski_calls(lab, img)))
        dire = _dict(*_merged(elt.stawiaski_directed_calls(lab, img, directedness)))
        mi, mj, mw, _ = elt.difference_of_means_calls(lab, img)
        nodes, src, snk = elt.regional_atlas_calls(lab, prob, alpha)
    means = {(int(x), int(y)): (u, u) for x, y, u in zip(mi, mj, mw)}
    for term, args, want, what in ((el.boundary_stawiaski, img, staw, "stawiaski"),
                                   (el.boundary_stawiaski_directed, (img, directedness), dire, "directed"),
                                   (el.boundary_difference_of_means, img, means, "means")):
        r = Recorder()
        term(r, lab, args)
        assert set(r.n) == set(want), what
        for key, (u, v) in want.items():
            gu, gv = r.n[key]
            assert numpy.float64(gu).view(numpy.uint64) == numpy.float64(u).view(numpy.uint64), (what, key, gu, u)
            assert numpy.float64(gv).view(numpy.uint64) == numpy.float64(v).view(numpy.uint64), (what, key, gv, v)
    r = Recorder()
    el.regional_atlas(r, lab, (prob, alpha))
    _assert_bits(numpy.asarray(r.t, dtype=numpy.float64).reshape(-1, 3), numpy.stack([nodes, src, snk], axis=1), "atlas")
    # the same terms through a real GCGraph: every arc pair holds the oracle's capacities, and the cut is BK's
    fg, bg = _fuzz_markers(lab, c)
    for boundary, args, want in (("stawiaski", img, staw), ("directed", (img, directedness), dire), ("means", img, means)):
        g = gc.graph_from_labels(lab, fg, bg, regional_term=el.regional_atlas, regional_term_args=(prob, alpha),
                                 boundary_term=_term(boundary), boundary_term_args=args)
        assert g.is_sparse and g.get_arc_num() == 2 * len(want)
        for (a, b), (u, v) in want.items():
            assert g.get_edge(a, b) == u and g.get_edge(b, a) == v, (boundary, a, b)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            problem = _label_problem(lab, fg, bg, boundary, args, atlas=(prob, alpha))
        tr, _ = elt.add_tweights_replay(problem[0], problem[5])
        assert [g.get_trcap(v) for v in range(problem[0])] == tr.tolist()
        mask = _check_cut(g, problem)
        assert numpy.array_equal(gc.label_cut_mask(g), mask[numpy.asarray(lab) - 1])


def test_fuzz_cases_within_tolerance_of_the_pow_oracle(timeout):
    """The unpatched oracle (math.pow) on every fuzz case: float32-gradient Stawiaski weights bit-exact, the rest within
    1e-14 relative -- the substitution of r*r for pow changes nothing beyond rounding."""
    el = _gc().energy_label
    for c, (lab, img, prob, alpha, directedness) in enumerate(_fuzz()):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            staw = _dict(*_merged(elt.stawiaski_calls(lab, img)))
            dire = _dict(*_merged(elt.stawiaski_directed_calls(lab, img, directedness)))
        for term, args, want, exact in ((el.boundary_stawiaski, img, staw, img.dtype == numpy.float32),
                                        (el.boundary_stawiaski_directed, (img, directedness), dire, False)):
            r = Recorder()
            term(r, lab, args)
            assert set(r.n) == set(want), c
            for key, (u, v) in want.items():
                gu, gv = r.n[key]
                if exact:
                    assert gu == u and gv == v, (c, key)
                else:
                    assert gu == pytest.approx(u, rel=1e-14, abs=1e-320) and gv == pytest.approx(v, rel=1e-14, abs=1e-320), (c, key)


# ---------------------------------------------------------------------------------------------------------------------
# B. label volumes at scale
# ---------------------------------------------------------------------------------------------------------------------
_VOL = {}


def _volume(ndim):
    if ndim not in _VOL:
        _VOL.clear()
        _VOL[ndim] = rc.label_volume(ndim)
    return _VOL[ndim]


VOLUME_CASES = sorted(rc.volume_cases())


@pytest.mark.parametrize("ndim,dtype", VOLUME_CASES)
def test_label_volume_terms_and_cut(ndim, dtype, square):
    """All four terms bit-exact against the oracle, the inputs in the case's layouts; then graph_from_labels with the
    atlas and one boundary term, cut against BK, and label_cut_mask against mask[label - 1]."""
    gc = _gc()
    el = gc.energy_label
    vol = _volume(ndim)
    spec = rc.volume_cases()[(ndim, dtype)]
    lab0, shape = vol["label"], vol["shape"]
    seed = 100 * ndim + rc.DTYPES.index(dtype)
    grad0 = rc.gradient(shape, dtype, seed)
    prob0 = rc.atlas(shape, spec["atlas_dtype"], seed + 50)
    lab = rc.label_layout(lab0, spec["label_layout"])
    grad = rc.value_layout(grad0, spec["grad_layout"])
    prob = rc.value_layout(prob0, spec["atlas_layout"])
    beta, alpha = spec["directedness"], spec["alpha"]

    r = ArrayRecorder()
    el.boundary_stawiaski(r, lab, grad)
    _assert_edges(r, _merged(elt.stawiaski_calls(lab0, grad0)), "stawiaski")
    r = ArrayRecorder()
    el.boundary_stawiaski_directed(r, lab, (grad, beta))
    _assert_edges(r, _merged(elt.stawiaski_directed_calls(lab0, grad0, beta)), "directed")
    r = ArrayRecorder()
    el.boundary_difference_of_means(r, lab, grad)
    mi, mj, mw, _ = elt.difference_of_means_calls(lab0, grad0)
    _assert_edges(r, (mi, mj, mw, mw), "means")
    r = ArrayRecorder()
    el.regional_atlas(r, lab, (prob, alpha))
    nodes, src, snk = elt.regional_atlas_calls(lab0, prob0, alpha)
    assert numpy.array_equal(numpy.asarray(r.t[0]), nodes)
    _assert_bits(r.t[1], src, "atlas source")
    _assert_bits(r.t[2], snk, "atlas sink")

    boundary = ("stawiaski", "directed", "means")[rc.DTYPES.index(dtype) % 3]
    args = (grad, beta) if boundary == "directed" else grad
    fg, bg = rc.markers(lab0, seed)
    g = gc.graph_from_labels(lab, fg, bg, regional_term=el.regional_atlas, regional_term_args=(prob, alpha),
                             boundary_term=_term(boundary), boundary_term_args=args)
    problem = _label_problem(lab0, fg, bg, boundary, (grad0, beta) if boundary == "directed" else grad0, atlas=(prob0, alpha))
    mask = _check_cut(g, problem)
    assert 0 < int(mask.sum()) < mask.size
    assert numpy.array_equal(gc.label_cut_mask(g), mask[lab0 - 1])


@pytest.mark.parametrize("ndim", sorted(rc.VOLUMES))
def test_label_volume_nonfinite_gradient_edges(ndim, square):
    """NaN, +inf and -inf in the gradient: boundary_stawiaski propagates NaN through numpy.maximum, the directed term
    drops a NaN second operand like Python's max; edges only, NaN weights equal NaN."""
    el = _gc().energy_label
    vol = _volume(ndim)
    dtype = "float64" if ndim % 2 else "float32"
    grad = rc.gradient(vol["shape"], dtype, 900 + ndim, nonfinite=True)
    r = ArrayRecorder()
    el.boundary_stawiaski(r, vol["label"], grad)
    want = _merged(elt.stawiaski_calls(vol["label"], grad))
    assert numpy.isnan(want[2]).any()
    _assert_edges(r, want, "stawiaski", equal_nan=True)
    for beta in (-0.01, 0.2):
        r = ArrayRecorder()
        el.boundary_stawiaski_directed(r, vol["label"], (grad, beta))
        _assert_edges(r, _merged(elt.stawiaski_directed_calls(vol["label"], grad, beta)), "directed", equal_nan=True)


# ---------------------------------------------------------------------------------------------------------------------
# C. general graphs
# ---------------------------------------------------------------------------------------------------------------------
_GRAPH = {}
SOLVE_SECONDS = {}


def _graph_case(name):
    """The instance and its BK solution, kept only while its cells run."""
    if name not in _GRAPH:
        _GRAPH.clear()
        case = rc.graph_case(name)
        _GRAPH[name] = (case, rc.bk(case))
    return _GRAPH[name]


def _build(case):
    """The case through the bulk setters: GCGraph's where every capacity is positive, GraphDouble's otherwise (GCGraph
    refuses zero n-weights like the reference)."""
    gc = _gc()
    n, i, j, cap, rev = case["n"], case["i"], case["j"], case["cap"], case["rev"]
    if (cap > 0).all() and (rev > 0).all():
        graph = gc.GCGraph(n, i.size, sparse=True)
        for nodes, src, snk in case["tw"]:
            graph.set_tweights_bulk(nodes, src, snk)
        graph.set_nweights_bulk(i, j, cap, rev)
        return graph.get_graph()
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(n, i.size, sparse=True)
    for nodes, src, snk in case["tw"]:
        g.add_tweights_bulk(nodes, src, snk)
    g.sum_edges_bulk(i, j, cap, rev)
    return g


@pytest.mark.parametrize("sweeps", (1, 16, 64))
@pytest.mark.parametrize("name", sorted(rc.GRAPHS))
def test_general_graph_vs_bk(name, sweeps, timeout, monkeypatch):
    monkeypatch.setenv("MEDPY_GC_SPARSE_SWEEPS", str(sweeps))
    case, (rflow, rmask) = _graph_case(name)
    g = _build(case)
    assert g.is_sparse
    t0 = time.perf_counter()
    flow = g.maxflow()
    SOLVE_SECONDS[(name, sweeps)] = time.perf_counter() - t0
    mask = g.get_mask()
    assert numpy.array_equal(mask, rmask), int((mask != rmask).sum())
    if case["exact"]:
        assert flow == rflow
    else:
        assert flow == pytest.approx(rflow, rel=1e-9)
    print("\n%s sweeps=%d: %.3f s" % (name, sweeps, SOLVE_SECONDS[(name, sweeps)]))


# ---------------------------------------------------------------------------------------------------------------------
# D. building and reusing one sparse graph
# ---------------------------------------------------------------------------------------------------------------------
def _random_calls(rng, n, m):
    i = rng.integers(0, n, size=m)
    j = rng.integers(0, n, size=m)
    keep = i != j
    return i[keep], j[keep], rng.uniform(0.1, 3.0, size=int(keep.sum())), rng.uniform(0.1, 3.0, size=int(keep.sum()))


def _tlinks(rng, n):
    nodes = rng.permutation(n)[: n // 2]
    return nodes, rng.uniform(0.0, 4.0, size=nodes.size), rng.uniform(0.0, 4.0, size=nodes.size)


def _assert_get_edge(g, calls):
    lo, hi, a, b = elt.merge_edges(*[numpy.concatenate(x) for x in zip(*calls)])
    assert g.get_arc_num() == 2 * lo.size
    for x, y, u, v in zip(lo.tolist(), hi.tolist(), a.tolist(), b.tolist()):
        assert g.get_edge(x, y) == u and g.get_edge(y, x) == v, (x, y)


def _solve_and_compare(g, n, calls, tw):
    i, j, cap, rev = [numpy.concatenate(x) for x in zip(*calls)]
    rflow, rmask, _ = solvers.solve_sparse(n, i, j, cap, rev, tw)
    flow = g.maxflow()
    assert numpy.array_equal(g.get_mask(), rmask)
    assert flow == pytest.approx(rflow, rel=1e-9, abs=1e-300)
    return flow


@pytest.mark.parametrize("look_between", (False, True))
def test_edge_batches_accumulate(look_between, timeout):
    """A sorted, unique first batch into an empty graph (the append-only path of mgc_sparse_sum_edges), then batches
    that hit its pairs in both orientations and add new ones, and single sum_edge calls: get_edge returns the
    accumulated capacities before and after maxflow, and the cut is BK's."""
    from medpy_b200.graphcut.maxflow import GraphDouble
    rng = numpy.random.default_rng(31 + look_between)
    n = 6000
    keys = numpy.unique(rng.integers(0, n, size=20000) * n + rng.integers(0, n, size=20000))
    lo, hi = keys // n, keys % n
    keep = lo < hi
    lo, hi = lo[keep], hi[keep]
    first = (lo, hi, rng.uniform(0.1, 3.0, size=lo.size), rng.uniform(0.1, 3.0, size=lo.size))
    tw = [_tlinks(rng, n)]
    g = GraphDouble(n, 0, sparse=True)
    g.add_tweights_bulk(*tw[0])
    g.sum_edges_bulk(*first)
    calls = [first]
    if look_between:
        _assert_get_edge(g, calls)
    k = rng.choice(lo.size, size=lo.size // 3, replace=False)
    again_fwd = (lo[k], hi[k], rng.uniform(0.1, 3.0, size=k.size), rng.uniform(0.1, 3.0, size=k.size))
    k = rng.choice(lo.size, size=lo.size // 3, replace=False)
    again_rev = (hi[k], lo[k], rng.uniform(0.1, 3.0, size=k.size), rng.uniform(0.1, 3.0, size=k.size))
    new = _random_calls(rng, n, 3000)
    for batch in (again_rev, new, again_fwd):
        g.sum_edges_bulk(*batch)
        calls.append(batch)
    for _ in range(50):
        a, b = int(lo[rng.integers(0, lo.size)]), int(hi[rng.integers(0, lo.size)])
        if a != b:
            c1, c2 = float(rng.uniform(0.1, 3.0)), float(rng.uniform(0.1, 3.0))
            g.sum_edge(b, a, c1, c2)
            calls.append((numpy.asarray([b]), numpy.asarray([a]), numpy.asarray([c1]), numpy.asarray([c2])))
    _assert_get_edge(g, calls)
    _solve_and_compare(g, n, calls, tw)
    _assert_get_edge(g, calls)


def test_chain_graph_moves_to_the_sparse_backend(timeout):
    """A shape-less GraphDouble fed chain-neighbour edges and t-links (some nodes twice, both signs) stays a chain until
    an off-chain edge arrives; the journal is then replayed onto the sparse backend and the cut is BK's."""
    from medpy_b200.graphcut.maxflow import GraphDouble
    rng = numpy.random.default_rng(41)
    n = 3000
    g = GraphDouble(n)
    tw_n, tw_s, tw_k, calls = [], [], [], []
    for v in range(n - 1):
        c1, c2 = float(rng.integers(1, 6)), float(rng.integers(1, 6))
        a, b = (v, v + 1) if v % 2 else (v + 1, v)
        g.sum_edge(a, b, c1, c2)
        calls.append((numpy.asarray([a]), numpy.asarray([b]), numpy.asarray([c1]), numpy.asarray([c2])))
    for v in rng.integers(0, n, size=2 * n).tolist():
        s, k = float(rng.integers(-3, 6)), float(rng.integers(-3, 6))
        g.add_tweights(v, s, k)
        tw_n.append(v), tw_s.append(s), tw_k.append(k)
    assert not g.is_sparse
    extra = [(0, n - 1, 4.0, 1.0), (n // 2, 7, 2.0, 3.0), (5, 4, 1.0, 1.0)]
    for a, b, c1, c2 in extra:
        g.sum_edge(a, b, c1, c2)
        calls.append((numpy.asarray([a]), numpy.asarray([b]), numpy.asarray([c1]), numpy.asarray([c2])))
    assert g.is_sparse
    tw = [(numpy.asarray(tw_n), numpy.asarray(tw_s), numpy.asarray(tw_k))]
    flow = _solve_and_compare(g, n, calls, tw)
    tr, _ = elt.add_tweights_replay(n, tw)
    assert [g.get_trcap(v) for v in range(0, n, 97)] == tr[::97].tolist()
    assert flow == float(int(flow))        # integer capacities: exact


def test_solved_graph_grows_and_resets(timeout):
    """After a solve: maxflow() again returns the same, what_segment agrees with get_mask; edges and t-links added to the
    solved graph give BK's cut of the graph as it now stands; reset() and a different graph on the same handle too."""
    gc = _gc()
    rng = numpy.random.default_rng(51)
    n = 5000
    graph = gc.GCGraph(n, 0, sparse=True)
    g = graph.get_graph()
    calls = [_random_calls(rng, n, 15000)]
    tw = [_tlinks(rng, n)]
    graph.set_tweights_bulk(*tw[0])
    graph.set_nweights_bulk(*calls[0])
    flow = _solve_and_compare(g, n, calls, tw)
    assert g.maxflow() == flow
    mask = g.get_mask()
    seg = numpy.asarray([0 if g.what_segment(v) == g.termtype.SINK else 1 for v in range(n)], numpy.uint8)
    assert numpy.array_equal(seg, mask)
    # grow the solved graph: new pairs, existing pairs again, more t-links on nodes that have some
    more = _random_calls(rng, n, 4000)
    k = rng.choice(calls[0][0].size, size=2000, replace=False)
    again = (calls[0][1][k], calls[0][0][k], rng.uniform(0.1, 1.0, size=k.size), rng.uniform(0.1, 1.0, size=k.size))
    graph.set_nweights_bulk(*more)
    graph.set_nweights_bulk(*again)
    calls += [more, again]
    t2 = _tlinks(rng, n)
    graph.set_tweights_bulk(*t2)
    tw.append(t2)
    flow2 = _solve_and_compare(g, n, calls, tw)
    assert g.maxflow() == flow2
    # reset: a different graph on the same handle
    g.reset()
    calls = [_random_calls(rng, n, 8000)]
    tw = [_tlinks(rng, n)]
    g.add_tweights_bulk(*tw[0])
    g.sum_edges_bulk(*calls[0])
    _solve_and_compare(g, n, calls, tw)
    assert g.get_arc_num() == 2 * elt.merge_edges(*calls[0])[0].size
    mask = g.get_mask()
    assert all((g.what_segment(v) == g.termtype.SOURCE) == bool(mask[v]) for v in range(0, n, 7))
