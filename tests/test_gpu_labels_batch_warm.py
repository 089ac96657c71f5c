"""GPU tests (``-m gpu``) of warm edits on a batch of label images (``graph_from_labels_batch(..., warm=True)``;
``MGC_OPT_WARM`` with ``MGC_OPT_SEGMENT_ENERGIES``, ``mgc_labels_voxel_flags``).

Rounds of mixed edits -- stroke seeds through ``region_flags``, erased seeds, t-link updates, increments on existing and
new pairs, exact and partial decrements -- go to one or two images of a batch at a time.  After every round each edited
image must match its own ``graph_from_labels(..., warm=True)`` given the same edits and BK's fresh solve of its whole
call sequence (oracle.solvers; a differing mask must be another minimum cut of equal capacity), and every image no edit
touched keeps its mask and energy bit for bit.  The native sparse handles are wrapped by a recorder that keeps each
handle's call sequence for BK.
"""
import os
import sys
from contextlib import contextmanager

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import region_cases as rc  # noqa: E402
from oracle import solvers  # noqa: E402
from test_gpu_labels_batch import _kw, gradient, markers, ragged_shapes, supervoxels  # noqa: E402

pytestmark = pytest.mark.gpu
os.environ.setdefault("MEDPY_GC_SPARSE_TIMEOUT", "30")


def _gc():
    import medpy_b200.graphcut as gc
    return gc


def _mgc():
    from medpy_b200 import _lib
    return _lib._mgc


def _bits(a):
    return numpy.ascontiguousarray(a, dtype=numpy.float64).view(numpy.uint64)


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


@pytest.fixture(autouse=True)
def recording_sparse(monkeypatch):
    """Every native sparse handle records the calls that reached it (refused ones raise before they are recorded)."""
    from medpy_b200 import _lib
    base = _lib._mgc.SparseGraph

    class Recorder(base):
        def __init__(self, n, device=-1):
            super().__init__(n, device)
            self.n = int(n)
            self.tw = []
            self.e = [[], [], [], []]

        def add_tweights(self, nodes, src, snk):
            super().add_tweights(nodes, src, snk)
            src = numpy.array(src, dtype=numpy.float64).ravel()
            nodes = numpy.arange(src.size) if nodes is None else numpy.array(nodes, dtype=numpy.int64).ravel()
            self.tw.append((nodes, src, numpy.array(snk, dtype=numpy.float64).ravel()))

        def sum_edges(self, i, j, cap, rev):
            super().sum_edges(i, j, cap, rev)
            self._edges(i, j, cap, rev, 1.0)

        def remove_edges_warm(self, i, j, cap, rev):
            super().remove_edges_warm(i, j, cap, rev)
            self._edges(i, j, cap, rev, -1.0)

        def _edges(self, i, j, cap, rev, sign):
            for k, (a, t) in enumerate(((i, numpy.int64), (j, numpy.int64), (cap, numpy.float64), (rev, numpy.float64))):
                a = numpy.array(a, dtype=t).ravel()
                self.e[k].append(a * sign if k >= 2 else a)

        def case(self):
            i, j, c, r = (numpy.concatenate(x) if x else numpy.zeros(0, t)
                          for x, t in zip(self.e, (numpy.int64, numpy.int64, float, float)))
            return dict(n=self.n, i=i, j=j, cap=c, rev=r, tw=list(self.tw))

    monkeypatch.setattr(_lib._mgc, "SparseGraph", Recorder)
    yield


def _bk_check(case, mask, energy, exact):
    """BK's fresh solve of the whole call sequence: the same mask or another minimum cut of equal capacity."""
    flow, want, _ = solvers.solve_sparse(case["n"], case["i"], case["j"], case["cap"], case["rev"], case["tw"])
    _same_cut(case, mask, want, exact)
    if exact:
        assert energy == flow
    else:
        assert energy == pytest.approx(flow, rel=1e-9, abs=1e-9)


def _same_cut(case, got, want, exact):
    if not numpy.array_equal(got, want):
        assert not exact, int((got != want).sum())
        a, b = rc.cut_capacity(case, got), rc.cut_capacity(case, want)
        assert a == pytest.approx(b, rel=1e-12), (int((got != want).sum()), a, b)


class Twin:
    """A warm batch and one graph_from_labels(..., warm=True) per image, edited alike."""

    def __init__(self, labs, fgs, bgs, kw, kws, exact=False):
        """``kw``: the batch's term keywords; ``kws[b]``: image b's own."""
        gc = _gc()
        self.labs, self.exact = labs, exact
        self.g = gc.graph_from_labels_batch(labs, fgs, bgs, warm=True, **kw)
        self.singles = [gc.graph_from_labels(labs[b], fgs[b], bgs[b], warm=True, **kws[b]) for b in range(len(labs))]
        self.off = self.g.node_offsets
        self.seeded = [[] for _ in labs]
        self.last = None

    def native(self, b):
        return self.singles[b]._sp._native

    def check(self, touched):
        """Touched images against their own warm graph and BK, untouched ones against the last round's bits."""
        g = self.g
        energies, masks = g.maxflow(), g.get_mask()
        assert numpy.array_equal(_bits(g.maxflow()), _bits(energies))                  # two reads, the same bits
        assert energies.sum() == pytest.approx(g._graph.maxflow(), rel=1e-9, abs=1e-9)
        for b in range(len(self.labs)):
            if self.last is not None and b not in touched:
                assert _bits(energies[b:b + 1]).tolist() == _bits(self.last[0][b:b + 1]).tolist(), b
                assert numpy.array_equal(masks[b], self.last[1][b]), b
                continue
            s = self.singles[b]
            e1, m1 = s.maxflow(), s.get_mask()
            case = self.native(b).case()
            _same_cut(case, masks[b], m1, self.exact)
            if self.exact:
                assert energies[b] == e1
            else:
                assert energies[b] == pytest.approx(e1, rel=1e-9, abs=1e-9), b
            _bk_check(case, masks[b], energies[b], self.exact)
        vox = g.label_cut_masks()
        for b in range(len(self.labs)):
            assert numpy.array_equal(vox[b], masks[b][self.labs[b] - 1]), b
        self.last = (energies.copy(), [m.copy() for m in masks])

    def edit(self, rng, b):
        """One round of mixed edits on image b."""
        g, s, lab = self.g, self.singles[b], self.labs[b]
        o, k = int(self.off[b]), int(self.off[b + 1] - self.off[b])
        ints = self.exact
        # a stroke of seeds through region_flags, and bg seeds by id
        stroke = numpy.zeros(lab.shape, bool)
        stroke.flat[rng.choice(lab.size, size=max(1, lab.size // 20), replace=False)] = True
        flags = g.region_flags([stroke if c == b else None for c in range(len(self.labs))])
        assert not flags[:o].any() and not flags[o + k:].any()
        assert numpy.array_equal(flags[o:o + k], s.label_context.region_flags(stroke).astype(bool))
        g.add_seeds(fg=flags)
        fg = numpy.flatnonzero(flags[o:o + k])
        s.add_seeds(fg=fg)
        bg = rng.choice(k, size=max(1, k // 8), replace=False)
        g.add_seeds(bg=bg + o)
        s.add_seeds(bg=bg)
        self.seeded[b] += fg.tolist()
        # erased seeds: half of the fg seeds set so far on this image
        er = numpy.asarray(self.seeded[b][: len(self.seeded[b]) // 2], dtype=numpy.int64)
        if er.size:
            g.remove_seeds(fg=er + o)
            s.remove_seeds(fg=er)
            del self.seeded[b][: er.size]
        # t-link updates of both signs
        v = rng.integers(0, k, size=max(1, k // 4))
        if ints:
            src, snk = rng.integers(-3, 6, size=v.size).astype(float), rng.integers(-3, 6, size=v.size).astype(float)
        else:
            src, snk = rng.uniform(-1, 3, size=v.size), rng.uniform(-1, 3, size=v.size)
        g.add_tweights_warm(v + o, src, snk)
        s.add_tweights_warm(v, src, snk)
        if k < 2:
            return
        # increments on existing pairs (either orientation) and on new pairs inside the image
        case = self.native(b).case()
        q = max(1, k // 4)
        if case["i"].size:
            pick = rng.integers(0, case["i"].size, size=q)
            ii, jj = case["j"][pick], case["i"][pick]
        else:
            ii = jj = numpy.zeros(0, numpy.int64)
        ii = numpy.concatenate([ii, rng.integers(0, k, size=q)])
        jj = numpy.concatenate([jj, rng.integers(0, k, size=q)])
        keep = ii != jj
        ii, jj = ii[keep], jj[keep]
        c = rng.integers(0, 4, size=ii.size).astype(float) if ints else rng.uniform(0, 1, size=ii.size)
        r = rng.integers(0, 4, size=ii.size).astype(float) if ints else rng.uniform(0, 1, size=ii.size)
        if ii.size:
            g.add_nweights_warm(ii + o, jj + o, c, r)
            s.add_nweights_warm(ii, jj, c, r)
        # exact decrements of what some pairs hold, partial ones of others
        case = self.native(b).case()
        if case["i"].size:
            pick = rng.integers(0, case["i"].size, size=max(1, q // 2 + 1))
            pairs = sorted({(int(min(x, y)), int(max(x, y))) for x, y in zip(case["i"][pick], case["j"][pick])})
            di = numpy.asarray([p[0] for p in pairs])
            dj = numpy.asarray([p[1] for p in pairs])
            dc = numpy.asarray([s.get_edge(x, y) for x, y in pairs])
            dr = numpy.asarray([s.get_edge(y, x) for x, y in pairs])
            part = numpy.arange(di.size) % 2 == 1
            dc = numpy.where(part, numpy.floor(dc / 2) if ints else dc * 0.5, dc)
            dr = numpy.where(part, numpy.floor(dr / 2) if ints else dr * 0.25, dr)
            g.remove_nweights_warm(di + o, dj + o, dc, dr)
            s.remove_nweights_warm(di, dj, dc, dr)


def _ragged(ndim, count, seed):
    rng = numpy.random.default_rng(seed)
    shapes = ragged_shapes(ndim, count, rng)
    labs = [supervoxels(s, 2, rng) for s in shapes]
    fgs, bgs = (list(x) for x in zip(*[markers(l, rng) for l in labs]))
    grads = [gradient(s, (numpy.float32, numpy.float64)[ndim % 2], rng) for s in shapes]
    probs = [rng.random(s).astype(numpy.float32) for s in shapes]
    return labs, fgs, bgs, grads, probs


def _twin(term, labs, fgs, bgs, grads, probs):
    return Twin(labs, fgs, bgs, _kw(term, grads, probs), [_kw(term, grads[b], probs[b]) for b in range(len(labs))])


def _rounds(t, rng, count, plan):
    t.g.maxflow()
    t.check(range(count))
    for touched in plan:
        for b in touched:
            t.edit(rng, b)
        t.check(touched)


@pytest.mark.parametrize("sweeps", [1, 16, 64])
@pytest.mark.parametrize("ndim", [2, 3])
@pytest.mark.parametrize("term", ["stawiaski", "means", "directed", "atlas"])
def test_rounds_of_mixed_edits(term, ndim, sweeps):
    seed = 10 * ndim + ["stawiaski", "means", "directed", "atlas"].index(term)
    labs, fgs, bgs, grads, probs = _ragged(ndim, 6, seed)
    with _env(MEDPY_GC_SPARSE_SWEEPS=sweeps):
        t = _twin(term, labs, fgs, bgs, grads, probs)
        _rounds(t, numpy.random.default_rng(seed + sweeps), 6, [(1,), (0, 4), (4,)])


def test_integer_capacities_equal_bk_exactly():
    """Atlas t-links of an integer atlas with alpha 1, no boundary term and integer edits: every capacity is an integer."""
    rng = numpy.random.default_rng(21)
    labs = [supervoxels(s, 2, rng) for s in ((9, 7), (5, 11), (8, 8), (6, 6))]
    fgs, bgs = (list(x) for x in zip(*[markers(l, rng) for l in labs]))
    probs = [rng.integers(-3, 4, size=l.shape).astype(numpy.int32) for l in labs]
    atlas = _gc().energy_label.regional_atlas
    t = Twin(labs, fgs, bgs, dict(regional_term=atlas, regional_term_args=(probs, 1.0)),
             [dict(regional_term=atlas, regional_term_args=(p, 1.0)) for p in probs], exact=True)
    _rounds(t, rng, 4, [(0, 2), (2,), (3,)])


def test_batch_of_one():
    labs, fgs, bgs, grads, probs = _ragged(2, 1, 3)
    t = _twin("stawiaski", labs, fgs, bgs, grads, probs)
    _rounds(t, numpy.random.default_rng(4), 1, [(0,), (0,)])


def test_edits_before_the_first_solve_equal_a_cold_batch():
    gc = _gc()
    rng = numpy.random.default_rng(5)
    labs = [supervoxels(s, 2, rng) for s in ((8, 8), (7, 6), (8, 5), (6, 8))]
    fgs, bgs = (list(x) for x in zip(*[markers(l, rng) for l in labs]))
    kw = _kw("stawiaski", [gradient(l.shape, numpy.float64, rng) for l in labs], None)
    warm = gc.graph_from_labels_batch(labs, fgs, bgs, warm=True, **kw)
    cold = gc.graph_from_labels_batch(labs, fgs, bgs, **kw)
    off = warm.node_offsets
    fg = numpy.asarray([off[1] + 1, off[3]])
    ii, jj = numpy.asarray([off[2], off[2] + 1]), numpy.asarray([off[2] + 2, off[2] + 3])
    warm.add_seeds(fg=fg)
    warm.add_tweights_warm([off[0]], 0.5, 2.0)
    warm.add_nweights_warm(ii, jj, 0.75, 0.25)
    warm.remove_nweights_warm(ii[:1], jj[:1], 0.5, 0.125)
    # the same calls on the cold handle: seeds and t-links as add_tweights, the decrement as a negative sum_edge
    cold._graph.add_tweights(fg.astype(numpy.int32), numpy.full(2, 65535.0), numpy.zeros(2))
    cold._graph.add_tweights(numpy.asarray([off[0]], numpy.int32), [0.5], [2.0])
    cold._graph.sum_edges(ii.astype(numpy.int32), jj.astype(numpy.int32), [0.75] * 2, [0.25] * 2)
    cold._graph.sum_edges(ii[:1].astype(numpy.int32), jj[:1].astype(numpy.int32), [-0.5], [-0.125])
    ew, ec = warm.maxflow(), cold.maxflow()
    for b in range(4):
        assert numpy.array_equal(warm.get_mask()[b], cold.get_mask()[b]), b
    numpy.testing.assert_allclose(ew, ec, rtol=1e-12, atol=1e-12)


def test_refusals_leave_every_image_bit_identical():
    labs, fgs, bgs, grads, probs = _ragged(3, 4, 6)
    g = _gc().graph_from_labels_batch(labs, fgs, bgs, warm=True, **_kw("stawiaski", grads, probs))
    e0, m0 = g.maxflow().copy(), [m.copy() for m in g.get_mask()]
    case = g._graph.case()
    a, b = int(case["i"][-1]), int(case["j"][-1])                   # an existing pair of the last image
    have = g._graph.get_edge(a, b) + g._graph.get_edge(b, a)
    with pytest.raises(ValueError, match="exceed"):
        g.remove_nweights_warm([a], [b], have * (1 + 1e-6), 0.0)
    off = g.node_offsets
    with pytest.raises(ValueError, match="label image 0 and label image 1"):
        g.add_nweights_warm([off[1] - 1], [off[1]], 1.0, 1.0)
    with pytest.raises(ValueError, match="NaN"):
        g.add_tweights_warm([0], float("nan"), 0.0)
    assert numpy.array_equal(_bits(g.maxflow()), _bits(e0))
    assert all(numpy.array_equal(x, y) for x, y in zip(g.get_mask(), m0))


def test_512_slices_with_a_stroke_on_slice_300():
    gc = _gc()
    rng = numpy.random.default_rng(7)
    vol = supervoxels((512, 24, 24), 4, rng)
    slices = []
    for z in range(vol.shape[0]):                                   # every slice's labels 1..K
        _, inv = numpy.unique(vol[z], return_inverse=True)
        slices.append((inv + 1).reshape(vol[z].shape).astype(numpy.int32))
    grads = [gradient((24, 24), numpy.float32, rng) for _ in slices]
    fgs, bgs = (list(x) for x in zip(*[markers(s, rng) for s in slices]))
    g = gc.graph_from_labels_batch(slices, fgs, bgs, warm=True, boundary_term=gc.energy_label.boundary_stawiaski,
                                   boundary_term_args=grads)
    e0, m0 = g.maxflow().copy(), [m.copy() for m in g.get_mask()]
    stroke = numpy.zeros((24, 24), bool)
    stroke[8:16, 10] = True
    strokes = [None] * 512
    strokes[300] = stroke
    g.add_seeds(fg=g.region_flags(strokes))
    e1, m1 = g.maxflow(), g.get_mask()
    one = gc.graph_from_labels(slices[300], fgs[300], bgs[300], warm=True, boundary_term=gc.energy_label.boundary_stawiaski,
                               boundary_term_args=grads[300])
    one.maxflow()
    one.add_seeds(fg=numpy.flatnonzero(one.label_context.region_flags(stroke)))
    assert numpy.array_equal(m1[300], one.get_mask())
    assert e1[300] == pytest.approx(one.maxflow(), rel=1e-9)
    keep = numpy.arange(512) != 300
    assert numpy.array_equal(_bits(e1[keep]), _bits(e0[keep]))
    assert all(numpy.array_equal(m1[z], m0[z]) for z in range(512) if z != 300)


def test_cuda_tensor_strokes_equal_numpy_strokes():
    import torch
    gc = _gc()
    rng = numpy.random.default_rng(8)
    labs = numpy.stack([supervoxels((10, 12), 3, rng) for _ in range(3)])
    fgs, bgs = (numpy.stack(x) for x in zip(*[markers(l, rng) for l in labs]))
    g = gc.graph_from_labels_batch(labs, fgs, bgs, warm=True)
    strokes = rng.random(labs.shape) < 0.1
    want = g.region_flags(strokes)
    assert numpy.array_equal(g.region_flags(torch.as_tensor(strokes, device="cuda")), want)
    assert numpy.array_equal(g.region_flags([None, torch.as_tensor(strokes[1], device="cuda"), strokes[2]]),
                             g.region_flags([None, strokes[1], strokes[2]]))
    with pytest.raises(ValueError):                                  # an id outside the concatenation
        g._labels.voxel_flags(numpy.asarray([labs.size], numpy.int64))


def test_reset_clears_the_accounts():
    """A native handle with both options: solve, fold, reset, rebuild and solve give a fresh handle's energies."""
    mgc = _mgc()
    off = numpy.asarray([0, 3, 5], numpy.int64)

    def build(g):
        g.add_tweights(numpy.arange(5, dtype=numpy.int32), [4.0, 0.0, 1.5, 2.0, 0.0], [0.0, 3.0, 0.5, 0.0, 2.5])
        g.sum_edges(numpy.asarray([0, 1, 3], numpy.int32), numpy.asarray([1, 2, 4], numpy.int32), [2.0, 1.25, 3.0],
                    [0.5, 1.0, 0.75])

    def handle():
        g = mgc.SparseGraph(5)
        g.set_option(mgc.OPT_WARM, 1)
        g.set_option(mgc.OPT_SEGMENT_ENERGIES, 1)
        return g

    g = handle()
    build(g)
    g.maxflow()
    g.add_tweights(numpy.asarray([2, 4], numpy.int32), [0.0, 3.0], [5.0, 0.0])
    g.remove_edges_warm(numpy.asarray([0], numpy.int32), numpy.asarray([1], numpy.int32), [1.5], [0.25])
    folded = g.segment_energies(off)
    assert folded.sum() == pytest.approx(g.maxflow(), rel=1e-12)
    g.reset()
    build(g)
    fresh = handle()
    build(fresh)
    assert numpy.array_equal(_bits(g.segment_energies(off)), _bits(fresh.segment_energies(off)))
    assert numpy.array_equal(g.get_mask(), fresh.get_mask())
    assert g.stats()["device_bytes"] == fresh.stats()["device_bytes"]
