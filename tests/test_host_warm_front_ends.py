"""One table of bad warm-edit arguments fed to the five front-ends that take warm edits: a lattice graph
(``GraphDouble``), a general sparse graph (``SparseGraphDouble``), a batch of images (``BatchGraph``), one rank's z-slab
(``SlabSolver``) and a batch of label images (``LabelBatchGraph``).  Each verdict is pinned per front-end: the exception
type and message with no call reaching the native handle, or the call passed on to the handle, whose own checks decide.
Where the front-ends differ, the table says so on purpose.  Each front-end drives the recording stand-in of its native
handle from its own host tests, so no GPU is needed except for the last test."""
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_host_batch_warm as batch_warm  # noqa: E402
import test_host_labels_batch_warm as labels_warm  # noqa: E402
import test_host_slab_warm as slab_warm  # noqa: E402

SHAPE = (3, 4, 5)       # the lattice front-ends: a batch of 3 images of 4 x 5, a z-slab of 3 planes
N = 60

PASS = "passed on"      # the call reaches the native handle (or, on a sparse graph, its staging)
ABSENT = "absent"       # the front-end has no such method
LATTICE = ("graph", "batch", "slab")
SPARSE = ("sparse", "labels")
FRONT_ENDS = LATTICE + SPARSE


def _all(verdict):
    return {f: verdict for f in FRONT_ENDS}


def _of(**by_front_end):
    """A verdict per front-end; the keys ``lattice`` and ``sparse`` stand for their groups.  A front-end left out takes
    an argument the stand-in device array cannot express: the sparse front-ends copy device arrays to the host, and the
    lattice graph stages seeds on the host before its first solve (test_lattice_seeds_may_mix_memory_spaces_unsolved)."""
    out = {}
    for key, verdict in by_front_end.items():
        out.update({f: verdict for f in {"lattice": LATTICE, "sparse": SPARSE}.get(key, (key,))})
    return out


def _dev(shape=(1,)):
    return batch_warm._DeviceArray(shape)


def _neg():
    f = numpy.zeros(SHAPE)
    f[0, 0, 0] = -1.0
    return f


_Z = numpy.zeros(SHAPE)
_NAN = float("nan")

# (name, method, arguments of a front-end's context, verdicts)
CASES = [
    ("seed_out_of_range", "add_seeds", lambda c: (numpy.array([0, c["n"]]), None),
     _all((ValueError, "Invalid node id"))),
    ("seed_mask_shape", "add_seeds", lambda c: (numpy.zeros(c["mask"][:-1] + (c["mask"][-1] + 1,), bool), None),
     _all((ValueError, "does not match"))),
    ("seed_not_integers", "add_seeds", lambda c: (numpy.array([1.5]), None),
     _all((ValueError, "1-D integer id array"))),
    ("seed_two_memory_spaces", "add_seeds", lambda c: (numpy.array([1]), _dev()),
     _of(batch=(ValueError, "both be host or both be device"), slab=(ValueError, "both be host or both be device"))),
    ("tlink_out_of_range", "add_tweights_warm", lambda c: (numpy.array([c["n"]]), 1.0, 1.0),
     _all((ValueError, "Invalid node id"))),
    ("tlink_length", "add_tweights_warm", lambda c: (numpy.array([0, 1]), numpy.array([1.0, 2.0, 3.0]), 0.0),
     _all((ValueError, "expected 2 entries"))),
    ("tlink_nan", "add_tweights_warm", lambda c: (numpy.array([0]), _NAN, 0.0),
     _of(graph=PASS, batch=PASS, slab=(ValueError, "NaN or infinite"), sparse=(ValueError, "NaN or infinite"))),
    ("tlink_bool", "add_tweights_warm", lambda c: (numpy.array([0]), numpy.array([True]), 0.0),
     _all((ValueError, "real numbers"))),
    ("tlink_dense_shape", "add_tweights_warm", lambda c: (None, numpy.zeros(7), 0.0),
     _all((ValueError, r"shape \(7,\)"))),
    ("tlink_two_memory_spaces", "add_tweights_warm", lambda c: (_dev(), numpy.array([1.0]), 1.0),
     _of(lattice=(ValueError, "all be host or all be device"))),
    ("nlink_out_of_range", "add_nweights_warm", lambda c: ([0], [c["n"]], 1.0, 1.0),
     _all((ValueError, "Invalid node id"))),
    ("nlink_length", "add_nweights_warm", lambda c: ([0, 1, 2], [1, 2], 1.0, 1.0),
     _all((ValueError, "differ in length"))),
    # a one-element id array broadcasts on sparse ids only; on the lattice only a 0-d id repeats
    ("nlink_one_element_ids", "add_nweights_warm", lambda c: (numpy.array([0]), numpy.array([1, 2]), 1.0, 1.0),
     _of(lattice=(ValueError, "differ in length"), sparse=PASS)),
    # the lattice graph and the batch leave the amounts and the pairs of a fold to the native check
    ("nlink_negative", "add_nweights_warm", lambda c: ([0], [1], -1.0, 0.0),
     _of(graph=PASS, batch=PASS, slab=(ValueError, "cap holds negative values"),
         sparse=(ValueError, "cap holds negative values"))),
    ("nlink_nan", "add_nweights_warm", lambda c: ([0], [1], 0.0, _NAN),
     _of(graph=PASS, batch=PASS, slab=(ValueError, "rev_cap holds NaN"), sparse=(ValueError, "rev_cap holds NaN"))),
    ("nlink_not_neighbours", "add_nweights_warm", lambda c: ([0], [2], 1.0, 1.0),
     _of(graph=PASS, batch=PASS, slab=(ValueError, "not lattice neighbours"), sparse=PASS)),
    ("nlink_across_images", "add_nweights_warm", lambda c: ([c["cross"][0]], [c["cross"][1]], 1.0, 1.0),
     _of(graph=PASS, batch=PASS, slab=(ValueError, "not lattice neighbours"), sparse=PASS,
         labels=(ValueError, "joins label image 0 and label image 1"))),
    ("nlink_two_memory_spaces", "add_nweights_warm", lambda c: (numpy.array([0]), _dev(), 1.0, 1.0),
     _of(lattice=(ValueError, "all be host or all be device"))),
    ("decrement_negative", "remove_nweights_warm", lambda c: ([0], [1], -1.0, 0.0),
     _of(graph=(ValueError, "cap holds negative values: n-link decrements"),
         batch=(ValueError, "cap holds negative values: n-link decrements"), slab=ABSENT,
         sparse=(ValueError, "cap holds negative values: n-link decrements"))),
    ("dense_axis", "add_nweights_dense_warm", lambda c: (3, _Z, _Z),
     _of(lattice=(ValueError, "out of range"), sparse=(ValueError, "no lattice axes"), labels=ABSENT)),
    ("dense_axis_0", "add_nweights_dense_warm", lambda c: (0, _Z, _Z),
     _of(graph=PASS, batch=(ValueError, "batch axis"), slab=PASS, sparse=(ValueError, "no lattice axes"),
         labels=ABSENT)),
    ("dense_shape", "add_nweights_dense_warm", lambda c: (1, numpy.zeros(SHAPE[1:]), numpy.zeros(SHAPE[1:])),
     _of(lattice=(ValueError, "does not match"), sparse=(ValueError, "no lattice axes"), labels=ABSENT)),
    ("dense_negative", "add_nweights_dense_warm", lambda c: (1, _neg(), _Z),
     _of(graph=PASS, batch=PASS, slab=(ValueError, "fwd or bwd holds negative, NaN or infinite values"),
         sparse=(ValueError, "no lattice axes"), labels=ABSENT)),
    ("dense_decrement_negative", "remove_nweights_dense_warm", lambda c: (1, _neg(), _Z),
     _of(graph=(ValueError, "fwd holds negative values"), batch=(ValueError, "fwd holds negative values"),
         slab=ABSENT, sparse=(ValueError, "no lattice axes"), labels=ABSENT)),
    ("dense_two_memory_spaces", "add_nweights_dense_warm", lambda c: (1, _Z, _dev(SHAPE)),
     _of(lattice=(ValueError, "both be host or both be device"), sparse=(ValueError, "no lattice axes"),
         labels=ABSENT)),
]


@pytest.fixture()
def front_end(monkeypatch):
    """front_end(name) -> (a warm front-end with a recording native handle, its context, the count of the calls that
    reached the handle).  The lattice graph is solved first, so that its warm edits fold natively."""
    from medpy_b200 import _lib
    mgc = _lib._mgc
    monkeypatch.setattr(mgc, "SparseGraph", labels_warm.RecordingSparse)
    monkeypatch.setattr(mgc, "LabelImage", type("LabelImage", (labels_warm.fake_native.FakeLabelImage,),
                                                 {"batch": staticmethod(labels_warm.FakeLabelBatch.batch)}))
    labels_warm.RecordingSparse.CALLS = []
    batch_warm._Recorder.made.clear()
    lattice = dict(n=N, mask=SHAPE, cross=(19, 20))      # 19 ends image 0 of the batch, 20 starts image 1

    def make(name):
        if name == "graph":
            from medpy_b200.graphcut.maxflow import GraphDouble
            monkeypatch.setattr(_lib, "Graph", lambda shape, device=-1: batch_warm._Recorder(shape, 1, device))
            g = GraphDouble(N, shape=SHAPE)
            g.maxflow()
            return g, lattice, lambda: len(batch_warm._Recorder.made[-1].calls)
        if name == "batch":
            monkeypatch.setattr(_lib, "Graph", type("Graph", (), {"batch": staticmethod(batch_warm._Recorder.factory)}))
            g = batch_warm._graph(batch=SHAPE[0], shape=SHAPE[1:])
            return g, lattice, lambda: len(batch_warm._Recorder.made[-1].calls)
        if name == "slab":
            from medpy_b200.distributed import SlabSolver
            s = SlabSolver(SHAPE, rank=0, world=1, handle_factory=slab_warm.Recorder, warm=True)
            return s, lattice, lambda: len(s.handle.calls)
        if name == "sparse":
            from medpy_b200.graphcut.sparse import SparseGraphDouble
            g = SparseGraphDouble(N, warm=True)

            def count():
                g._flush()                                  # staged calls reach the handle
                return len(labels_warm.RecordingSparse.CALLS)
            return g, dict(lattice, mask=(N,)), count
        g = labels_warm._batch()
        off = g.node_offsets
        ctx = dict(n=int(off[-1]), mask=(int(off[-1]),), cross=(int(off[1]) - 1, int(off[1])))
        return g, ctx, lambda: len(labels_warm.RecordingSparse.CALLS)
    return make


@pytest.mark.parametrize("which,method,args,verdict", [(w, m, a, v[w]) for _, m, a, v in CASES for w in FRONT_ENDS if w in v],
                         ids=["{}-{}".format(c[0], w) for c in CASES for w in FRONT_ENDS if w in c[3]])
def test_front_end_verdicts(front_end, which, method, args, verdict):
    obj, ctx, calls = front_end(which)
    if verdict == ABSENT:
        assert not hasattr(obj, method)
        return
    before = calls()
    if verdict == PASS:
        getattr(obj, method)(*args(ctx))
        assert calls() > before
        return
    exc, match = verdict
    with pytest.raises(exc, match=match):
        getattr(obj, method)(*args(ctx))
    assert calls() == before


def test_without_warm(front_end, monkeypatch):
    """Built without warm=True, a batch of images passes the arguments of a warm edit to its native handle unparsed
    (which refuses the call); a label batch and a sparse graph raise RuntimeError themselves."""
    from medpy_b200 import _lib
    from medpy_b200.graphcut.sparse import SparseGraphDouble
    monkeypatch.setattr(_lib, "Graph", type("Graph", (), {"batch": staticmethod(batch_warm._Recorder.factory)}))
    g = batch_warm._graph(warm=False)
    bad = numpy.array([N])
    g.add_seeds(bad, None)
    assert batch_warm._Recorder.made[-1].calls[-1] == ("add_seeds", bad, None)
    front_end("labels")                                     # installs the sparse stand-ins
    for cold in (labels_warm._batch(warm=False), SparseGraphDouble(N)):
        before = len(labels_warm.RecordingSparse.CALLS)
        with pytest.raises(RuntimeError, match="warm=True"):
            cold.add_seeds(bad)
        assert len(labels_warm.RecordingSparse.CALLS) == before


@pytest.mark.gpu
def test_lattice_seeds_may_mix_memory_spaces_unsolved():
    """Before its first solve a lattice graph stages seeds on the host, so fg and bg may lie in two memory spaces; after
    it the native fold refuses the mix."""
    import torch

    import medpy_b200.graphcut as gc
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume((8, 9, 10), seed=0)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(vol["prob"], vol["alpha"]),
                             boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    g.add_seeds(numpy.array([0]), torch.tensor([5], device="cuda"))
    g.maxflow()
    with pytest.raises(ValueError, match="both be host or both be device"):
        g.add_seeds(numpy.array([1]), torch.tensor([6], device="cuda"))
