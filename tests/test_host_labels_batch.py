"""CPU tests (no GPU) of ``graph_from_labels_batch`` and the ``batch=True`` path of the wrapper functions: argument and
error conventions, the node-offset mapping, and that a batch cuts every image as its own ``graph_from_labels`` call does.

The two native classes are replaced by the oracle-backed doubles below: a label batch made of one
``fake_native.FakeLabelImage`` per image, and a sparse graph whose segment energies are the oracle's energies of the
images' own graphs.  What this cannot cover: the CUDA kernels and the C ABI (tests/test_gpu_labels_batch.py)."""
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import solvers  # noqa: E402

import fake_native  # noqa: E402

G = numpy.load(os.path.join(HERE, "golden", "golden_labels_v1.npz"))


class FakeLabelBatch:
    """``_mgc.LabelImage.batch``: the images' own doubles side by side, node ids shifted by the offsets."""

    def __init__(self, shapes, labels):
        ends = numpy.cumsum([int(numpy.prod(s)) for s in shapes])
        self.starts = numpy.concatenate([[0], ends])
        self.images = []
        for b, (s, part) in enumerate(zip(shapes, numpy.split(numpy.asarray(labels), ends[:-1]))):
            try:
                self.images.append(fake_native.FakeLabelImage(part.reshape(s)))
            except AttributeError as e:
                raise AttributeError("label image {}: {}".format(b, e)) from None
        self.off = numpy.concatenate([[0], numpy.cumsum([im.k for im in self.images])]).astype(numpy.int64)

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

    def apply(self, per_region):
        per_region = numpy.asarray(per_region)
        return numpy.concatenate([im.apply(per_region[a:b]).ravel()
                                  for im, a, b in zip(self.images, self.off[:-1], self.off[1:])])


class FakeSegmentSparse(fake_native.FakeSparseGraph):
    """``_mgc.SparseGraph`` with the segment energies: each range's own graph solved by the oracle."""

    OPTIONS = []

    def set_option(self, option, value):
        FakeSegmentSparse.OPTIONS.append((option, value))

    def segment_energies(self, off):
        i, j, cap, rev = self.e
        out = []
        for a, b in zip(off[:-1], off[1:]):
            keep = (i >= a) & (i < b)
            assert ((j[keep] >= a) & (j[keep] < b)).all(), "an arc joins two images"
            tw = []
            for nodes, src, snk in self.tw:
                sel = (nodes >= a) & (nodes < b)
                tw.append((nodes[sel] - a, src[sel], snk[sel]))
            flow, _, _ = solvers.solve_sparse(int(b - a), i[keep] - a, j[keep] - a, cap[keep], rev[keep], tw)
            out.append(flow)
        return numpy.asarray(out)


@pytest.fixture(autouse=True)
def fake_native_classes(monkeypatch):
    from medpy_b200 import _lib
    monkeypatch.setattr(_lib._mgc, "LabelImage", type("LabelImage", (fake_native.FakeLabelImage,),
                                                      {"batch": staticmethod(FakeLabelBatch.batch)}))
    monkeypatch.setattr(_lib._mgc, "SparseGraph", FakeSegmentSparse)
    FakeSegmentSparse.OPTIONS = []
    yield


def _gc():
    import medpy_b200.graphcut as gc
    return gc


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


def test_node_offsets_masks_and_energies_match_single_calls():
    gc = _gc()
    el = gc.energy_label
    cases = [_case((4, 5), 2, 0), _case((6, 3), 5, 1), _case((3, 7), 3, 2)]
    labs, grads, fgs, bgs = (list(x) for x in zip(*cases))
    g = gc.graph_from_labels_batch(labs, fgs, bgs, boundary_term=el.boundary_stawiaski, boundary_term_args=grads)
    assert g.node_offsets.tolist() == [0, 2, 7, 10] and len(g) == 3
    assert (_lib_option(), 1) in FakeSegmentSparse.OPTIONS
    energies = g.maxflow()
    masks, vox = g.get_mask(), g.label_cut_masks()
    for b, (lab, grad, fg, bg) in enumerate(cases):
        one = gc.graph_from_labels(lab, fg, bg, boundary_term=el.boundary_stawiaski, boundary_term_args=grad)
        assert energies[b] == one.maxflow()
        assert numpy.array_equal(masks[b], one.get_mask())
        assert numpy.array_equal(vox[b], gc.label_cut_mask(one))
    assert g.stats()["images"] == 3


def _lib_option():
    from medpy_b200 import _lib
    return _lib._mgc.OPT_SEGMENT_ENERGIES


def test_stacked_input_and_all_terms():
    gc = _gc()
    el = gc.energy_label
    cases = [_case((5, 6), 4, s) for s in range(3)]
    labs, grads, fgs, bgs = (numpy.stack(x) for x in zip(*cases))
    probs = numpy.random.default_rng(9).random(labs.shape)
    for kw in (dict(boundary_term=el.boundary_difference_of_means, boundary_term_args=grads),
               dict(boundary_term=el.boundary_stawiaski_directed, boundary_term_args=(grads, -0.25),
                    regional_term=el.regional_atlas, regional_term_args=(probs, 0.5))):
        g = gc.graph_from_labels_batch(labs, fgs, bgs, **kw)
        vox = g.label_cut_masks()
        assert vox.shape == labs.shape
        for b in range(3):
            one_kw = {k: (v[b] if k.endswith("args") and not isinstance(v, tuple) else
                          (v[0][b], v[1]) if isinstance(v, tuple) else v) for k, v in kw.items()}
            one = gc.graph_from_labels(labs[b], fgs[b], bgs[b], **one_kw)
            assert g.maxflow()[b] == one.maxflow()
            assert numpy.array_equal(vox[b], gc.label_cut_mask(one))


def test_errors_name_the_image():
    gc = _gc()
    el = gc.energy_label
    cases = [_case((4, 4), 3, s) for s in range(3)]
    labs, grads, fgs, bgs = (list(x) for x in zip(*cases))
    kw = dict(boundary_term=el.boundary_stawiaski, boundary_term_args=grads)
    bad = list(labs)
    bad[2] = numpy.asarray([[1, 4], [1, 3]])
    with pytest.raises(AttributeError, match="label image 2"):
        gc.graph_from_labels_batch(bad, fgs[:2] + [numpy.ones((2, 2), bool)], bgs[:2] + [numpy.ones((2, 2), bool)])
    bad[2] = numpy.asarray([[0, 1], [1, 2]], dtype=numpy.int64)             # rejected on the host
    with pytest.raises(AttributeError, match="label image 2"):
        gc.graph_from_labels_batch(bad, fgs[:2] + [numpy.ones((2, 2), bool)], bgs[:2] + [numpy.ones((2, 2), bool)])
    g_bad = list(grads)
    g_bad[1] = numpy.zeros((3, 4))
    with pytest.raises(ValueError, match="label image 1"):
        gc.graph_from_labels_batch(labs, fgs, bgs, boundary_term=el.boundary_stawiaski, boundary_term_args=g_bad)
    m_bad = list(fgs)
    m_bad[0] = numpy.zeros((2, 2), bool)
    with pytest.raises(IndexError, match="label image 0"):
        gc.graph_from_labels_batch(labs, m_bad, bgs, **kw)
    none = list(bgs)
    none[1] = numpy.zeros((4, 4), bool)                                   # no sink marker: max([]) of set_sink_nodes
    with pytest.raises(ValueError, match="label image 1: max"):
        gc.graph_from_labels_batch(labs, fgs, none, **kw)
    one_row = [numpy.asarray([[1, 2, 3]])] * 2
    with pytest.raises(ValueError, match="label image 0: cannot call `vectorize`"):
        gc.graph_from_labels_batch(one_row, [numpy.ones((1, 3), bool)] * 2, [numpy.ones((1, 3), bool)] * 2,
                                   boundary_term=el.boundary_stawiaski_directed,
                                   boundary_term_args=([numpy.zeros((1, 3))] * 2, -0.1))
    with pytest.raises(TypeError, match="energy_label terms"):
        gc.graph_from_labels_batch(labs, fgs, bgs, boundary_term=lambda g, l, a: None)
    with pytest.raises(ValueError, match="empty batch"):
        gc.graph_from_labels_batch([], [], [])
    with pytest.raises(ValueError, match="2 arrays for a batch of 3"):
        gc.graph_from_labels_batch(labs, fgs[:2], bgs, **kw)
    with pytest.raises(ValueError, match="one number of dimensions"):
        gc.graph_from_labels_batch([labs[0], labs[1].ravel()], fgs[:2], bgs[:2])


def test_wrapper_batch_conventions():
    gc = _gc()
    from medpy_b200.errors import ArgumentError
    lab, grad, fg, bg = _case((6, 6), 4, 3)
    with pytest.raises(ArgumentError, match="same shape"):          # a ragged job: its four images disagree
        gc.graphcut_stawiaski_batch([(lab, grad, fg, bg), (lab, grad[1:], fg, bg)])
    with pytest.raises(ArgumentError, match="graphcut_stawiaski jobs only"):
        gc.graphcut_subprocesses(lambda job: None, [(lab, grad, fg, bg)], batch=True)
    with pytest.raises(ArgumentError, match="graphcut_stawiaski jobs only"):
        gc.graphcut_split(lambda job: None, lab, grad, fg, bg, 10, 3, batch=True)
    with pytest.raises(ArgumentError):                                # processes is still validated first
        gc.graphcut_subprocesses(gc.graphcut_stawiaski, [], -1, batch=True)
    assert gc.graphcut_stawiaski_batch([]) == []
    jobs = [(lab, grad, fg, bg), _case((5, 7), 3, 4)]
    got = gc.graphcut_stawiaski_batch(jobs)
    want = [gc.graphcut_stawiaski(j) for j in jobs]
    assert all(a.dtype == numpy.bool_ and numpy.array_equal(a, b) for a, b in zip(got, want))


def test_graphcut_split_batch_equals_back_to_back():
    gc = _gc()
    lab, grad, fg, bg = G["split/label"], G["split/gradient"], G["split/fg"], G["split/bg"]
    one = gc.graphcut_split(gc.graphcut_stawiaski, lab, grad, fg, bg, 10, 3, 2)
    two = gc.graphcut_split(gc.graphcut_stawiaski, lab, grad, fg, bg, 10, 3, 2, batch=True)
    assert numpy.array_equal(one, two) and numpy.array_equal(two, G["split/split_mask"].astype(bool))
