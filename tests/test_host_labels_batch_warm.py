"""CPU tests (no GPU) of the warm edits of a label batch (``graph_from_labels_batch(..., warm=True)``): the options and
native calls the batch makes, the mapping of ids, masks and strokes onto the union's nodes, and the refusals that come
before any native call.

The two native classes are replaced by the oracle-backed doubles below: a label batch made of one
``fake_native.FakeLabelImage`` per image, and a sparse graph that records its calls and solves the whole call sequence
(decrements included) with BK.  What this cannot cover: the CUDA kernels, the per-node constant accounts and the warm
re-solve itself (tests/test_gpu_labels_batch_warm.py)."""
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import solvers  # noqa: E402

import fake_native  # noqa: E402


class FakeLabelBatch:
    """``_mgc.LabelImage.batch``: the images' own doubles side by side, node ids shifted by the offsets."""

    def __init__(self, shapes, labels):
        ends = numpy.cumsum([int(numpy.prod(s)) for s in shapes])
        self.starts = numpy.concatenate([[0], ends])
        self.images = [fake_native.FakeLabelImage(part.reshape(s))
                       for s, part in zip(shapes, numpy.split(numpy.asarray(labels), ends[:-1]))]
        self.off = numpy.concatenate([[0], numpy.cumsum([im.k for im in self.images])]).astype(numpy.int64)
        self.nodes = numpy.concatenate([im.lab.ravel() - 1 + o for im, o in zip(self.images, self.off)])

    @staticmethod
    def batch(shapes, label_images, device=-1):
        return FakeLabelBatch([tuple(s) for s in shapes], label_images)

    def _parts(self, values):
        v = numpy.asarray(values)
        return [v[a:b].reshape(im.lab.shape) for a, b, im in zip(self.starts[:-1], self.starts[1:], self.images)]

    def batch_offsets(self):
        return self.off.copy()

    def region_count(self):
        return int(self.off[-1])

    def boundary(self, kind, values=None, directedness=0.0):
        parts = self._parts(values) if values is not None else [None] * len(self.images)
        got = [im.boundary(kind, v, directedness) for im, v in zip(self.images, parts)]
        i = numpy.concatenate([g[0] + o for g, o in zip(got, self.off)]).astype(numpy.int32)
        j = numpy.concatenate([g[1] + o for g, o in zip(got, self.off)]).astype(numpy.int32)
        return i, j, numpy.concatenate([g[2] for g in got]), numpy.concatenate([g[3] for g in got])

    def region_sums(self, values, mode):
        got = [im.region_sums(v, mode) for im, v in zip(self.images, self._parts(values))]
        return numpy.concatenate([g[0] for g in got]), numpy.concatenate([g[1] for g in got])

    def region_flags(self, markers):
        return numpy.concatenate([im.region_flags(m) for im, m in zip(self.images, self._parts(markers))])

    def voxel_flags(self, ids):
        ids = numpy.asarray(ids, dtype=numpy.int64)
        assert ids.ndim == 1
        if ids.size and (ids.min() < 0 or ids.max() >= self.nodes.size):
            raise ValueError("voxel id out of range")
        VOXEL_IDS.append(ids.copy())
        flags = numpy.zeros(int(self.off[-1]), numpy.uint8)
        flags[self.nodes[ids]] = 1
        return flags

    def apply(self, per_region):
        return numpy.asarray(per_region, dtype=numpy.uint8)[self.nodes]


VOXEL_IDS = []


class RecordingSparse(fake_native.FakeSparseGraph):
    """``_mgc.SparseGraph`` that records every call in CALLS and solves the whole call sequence with BK: a decrement
    is a sum_edge of the negated amounts, as on the reference's residual graph."""

    CALLS = []

    def _log(self, name, *args):
        RecordingSparse.CALLS.append((name,) + tuple(None if a is None else numpy.array(a, copy=True) for a in args))

    def set_option(self, option, value):
        RecordingSparse.CALLS.append(("set_option", option, value))

    def sum_edges(self, i, j, cap, rev):
        self._log("sum_edges", i, j, cap, rev)
        super().sum_edges(i, j, cap, rev)

    def add_tweights(self, nodes, src, snk):
        self._log("add_tweights", nodes, src, snk)
        super().add_tweights(nodes, src, snk)

    def remove_edges_warm(self, i, j, cap, rev):
        self._log("remove_edges_warm", i, j, cap, rev)
        super().sum_edges(i, j, -numpy.asarray(cap, dtype=float), -numpy.asarray(rev, dtype=float))

    def segment_energies(self, off):
        i, j, cap, rev = self.e
        out = []
        for a, b in zip(off[:-1], off[1:]):
            keep = (i >= a) & (i < b)
            assert ((j[keep] >= a) & (j[keep] < b)).all(), "an arc joins two images"
            tw = [(nodes[(nodes >= a) & (nodes < b)] - a, src[(nodes >= a) & (nodes < b)], snk[(nodes >= a) & (nodes < b)])
                  for nodes, src, snk in self.tw]
            out.append(solvers.solve_sparse(int(b - a), i[keep] - a, j[keep] - a, cap[keep], rev[keep], tw)[0])
        return numpy.asarray(out)


@pytest.fixture(autouse=True)
def fake_native_classes(monkeypatch):
    from medpy_b200 import _lib
    monkeypatch.setattr(_lib._mgc, "LabelImage", type("LabelImage", (fake_native.FakeLabelImage,),
                                                      {"batch": staticmethod(FakeLabelBatch.batch)}))
    monkeypatch.setattr(_lib._mgc, "SparseGraph", RecordingSparse)
    RecordingSparse.CALLS = []
    VOXEL_IDS.clear()
    yield


def _gc():
    import medpy_b200.graphcut as gc
    return gc


def _mgc():
    from medpy_b200 import _lib
    return _lib._mgc


def _case(shape, k, seed):
    """Labels 1..k (each present), a gradient and markers that hit at least one region each."""
    rng = numpy.random.default_rng(seed)
    n = int(numpy.prod(shape))
    lab = numpy.concatenate([numpy.arange(1, k + 1), rng.integers(1, k + 1, size=n - k)])
    rng.shuffle(lab)
    lab = lab.reshape(shape).astype(numpy.int32)
    grad = rng.random(shape).astype(numpy.float32)
    fg = numpy.zeros(shape, bool)
    bg = numpy.zeros(shape, bool)
    fg.flat[0] = True
    bg.flat[n - 1] = True
    return lab, grad, fg, bg


CASES = [_case((4, 5), 3, 0), _case((6, 3), 5, 1), _case((3, 7), 4, 2)]


def _batch(warm=True, cases=CASES):
    gc = _gc()
    labs, grads, fgs, bgs = (list(x) for x in zip(*cases))
    return gc.graph_from_labels_batch(labs, fgs, bgs, boundary_term=gc.energy_label.boundary_stawiaski,
                                      boundary_term_args=grads, warm=warm)


def _names(calls):
    return [c[0] if c[0] != "set_option" else c for c in calls]


def test_options_come_first_and_cold_calls_are_unchanged():
    mgc = _mgc()
    cold = _batch(False)
    cold_calls = list(RecordingSparse.CALLS)
    assert not cold.warm
    RecordingSparse.CALLS = []
    warm = _batch(True)
    assert warm.warm
    # the cold batch sets the segment option only; the warm one sets the warm option first, then the same calls
    assert _names(cold_calls) == [("set_option", mgc.OPT_SEGMENT_ENERGIES, 1), "sum_edges", "add_tweights", "add_tweights"]
    assert RecordingSparse.CALLS[0] == ("set_option", mgc.OPT_WARM, 1)
    assert len(RecordingSparse.CALLS) == len(cold_calls) + 1
    for a, b in zip(RecordingSparse.CALLS[1:], cold_calls):
        assert a[0] == b[0] and all(x == y if not isinstance(x, numpy.ndarray) else numpy.array_equal(x, y)
                                    for x, y in zip(a[1:], b[1:]))
    numpy.testing.assert_array_equal(warm.maxflow(), cold.maxflow())


def test_ids_and_masks_map_onto_the_union():
    g = _batch()
    off = g.node_offsets
    n = int(off[-1])
    before = len(RecordingSparse.CALLS)
    ids = numpy.asarray([off[1] + 2, off[2] + 0])
    mask = numpy.zeros(n, bool)
    mask[ids] = True
    g.add_seeds(fg=mask, bg=[int(off[0]) + 1])
    g.remove_seeds(fg=ids)
    calls = RecordingSparse.CALLS[before:]
    assert [c[0] for c in calls] == ["add_tweights"] * 3
    numpy.testing.assert_array_equal(calls[0][1], ids)
    numpy.testing.assert_array_equal(calls[0][2], [65535.0] * 2)
    numpy.testing.assert_array_equal(calls[1][1], [1])
    numpy.testing.assert_array_equal(calls[1][3], [65535.0])
    numpy.testing.assert_array_equal(calls[2][1], ids)
    numpy.testing.assert_array_equal(calls[2][2], [-65535.0] * 2)
    g.add_tweights_warm(None, 0.5, 0.25)                     # one call per node of the union
    assert calls[0][1].dtype == numpy.int32 and RecordingSparse.CALLS[-1][1] is None
    assert RecordingSparse.CALLS[-1][2].size == n
    g.add_nweights_warm(off[1] + 0, off[1] + 1, [1.0, 2.0], 0.0)     # two calls on one pair of image 1
    c = RecordingSparse.CALLS[-1]
    assert c[0] == "sum_edges" and c[1].tolist() == [off[1]] * 2 and c[3].tolist() == [1.0, 2.0]


def test_edits_match_each_images_own_warm_graph():
    """Every image of an edited batch has the mask and energy of its own graph_from_labels(warm=True) given the same
    edits (ids shifted by node_offsets)."""
    gc = _gc()
    g = _batch()
    off = g.node_offsets
    g.maxflow()
    singles = [gc.graph_from_labels(lab, fg, bg, boundary_term=gc.energy_label.boundary_stawiaski,
                                    boundary_term_args=grad, warm=True) for lab, grad, fg, bg in CASES]
    for s in singles:
        s.maxflow()
    # image 1: a seed stroke, a t-link update, a new pair and an existing pair lowered; image 2: an erased seed
    g.add_seeds(fg=[off[1] + 3], bg=[off[1] + 4])
    singles[1].add_seeds(fg=[3], bg=[4])
    g.add_tweights_warm([off[1] + 1], 2.0, 1.0)
    singles[1].add_tweights_warm([1], 2.0, 1.0)
    g.add_nweights_warm([off[1] + 0], [off[1] + 4], 0.75, 0.5)
    singles[1].add_nweights_warm([0], [4], 0.75, 0.5)
    _, i, j, w, _ = next(c for c in RecordingSparse.CALLS if c[0] == "sum_edges")     # the batch's edges
    k = int(numpy.flatnonzero(i >= off[1])[0])
    g.remove_nweights_warm([i[k]], [j[k]], w[k] / 2, 0.0)
    singles[1].remove_nweights_warm([i[k] - off[1]], [j[k] - off[1]], w[k] / 2, 0.0)
    g.remove_seeds(bg=[off[2] + 0])
    singles[2].remove_seeds(bg=[0])
    energies, masks = g.maxflow(), g.get_mask()
    for b, s in enumerate(singles):
        assert energies[b] == s.maxflow()
        assert numpy.array_equal(masks[b], s.get_mask())


@pytest.mark.parametrize("stacked", [False, True])
def test_region_flags_equal_each_images_own(stacked):
    gc = _gc()
    from medpy_b200.graphcut.energy_label import LabelContext
    cases = [_case((5, 6), 4, s) for s in range(3)]
    g = _batch(cases=cases) if not stacked else gc.graph_from_labels_batch(
        numpy.stack([c[0] for c in cases]), numpy.stack([c[2] for c in cases]), numpy.stack([c[3] for c in cases]), warm=True)
    rng = numpy.random.default_rng(4)
    strokes = [rng.random((5, 6)) < 0.2 for _ in cases]
    for use in ([0, 1, 2], [1], []):
        given = [s if b in use else None for b, s in enumerate(strokes)]
        VOXEL_IDS.clear()
        got = g.region_flags(numpy.stack(strokes) if stacked and len(use) == 3 else given)
        want = numpy.concatenate([LabelContext(c[0]).region_flags(s) if b in use else numpy.zeros(4, numpy.uint8)
                                  for b, (c, s) in enumerate(zip(cases, strokes))])
        assert got.dtype == numpy.bool_ and numpy.array_equal(got, want.astype(bool))
        # only the given images' marked voxels travel, as ids over the concatenation
        want_ids = numpy.concatenate([numpy.flatnonzero(strokes[b]) + 30 * b for b in use] + [numpy.zeros(0, int)])
        assert numpy.array_equal(VOXEL_IDS[-1], want_ids)
    with pytest.raises(ValueError, match="2 entries for a batch of 3"):
        g.region_flags(strokes[:2])
    with pytest.raises(IndexError, match="label image 1"):
        g.region_flags([None, numpy.zeros((6, 5), bool), None])


def test_refusals_come_before_any_native_call():
    g = _batch()
    off = g.node_offsets
    g.maxflow()
    before = len(RecordingSparse.CALLS)

    def expect(exc, match, fn, *args):
        with pytest.raises(exc, match=match):
            fn(*args)
        assert len(RecordingSparse.CALLS) == before

    a, b = int(off[1]) - 1, int(off[1])                    # the last region of image 0, the first of image 1
    expect(ValueError, "label image 0 and label image 1", g.add_nweights_warm, [a], [b], 1.0, 1.0)
    expect(ValueError, "label image 2 and label image 0", g.remove_nweights_warm, [0, off[2]], [1, 0], 0.5, 0.0)
    expect(ValueError, "NaN", g.add_nweights_warm, [0], [1], float("nan"), 0.0)
    expect(ValueError, "NaN", g.add_tweights_warm, [0], 1.0, float("inf"))
    expect(ValueError, "negative", g.add_nweights_warm, [0], [1], -1.0, 0.0)
    expect(ValueError, "negative", g.remove_nweights_warm, [0], [1], 0.0, -1.0)
    expect(ValueError, "Invalid node id", g.add_seeds, [int(off[-1])])
    expect(ValueError, "does not match", g.add_seeds, numpy.ones(int(off[-1]) + 1, bool))
    expect(ValueError, "differ in length", g.add_nweights_warm, [0, 1, 2], [1, 2], 1.0, 1.0)
    cold = _batch(False)
    before = len(RecordingSparse.CALLS)
    for name, args in (("add_seeds", ([0],)), ("remove_seeds", ([0],)), ("add_tweights_warm", ([0], 1.0, 0.0)),
                       ("add_nweights_warm", ([0], [1], 1.0, 0.0)), ("remove_nweights_warm", ([0], [1], 1.0, 0.0))):
        expect(RuntimeError, "warm=True", getattr(cold, name), *args)
