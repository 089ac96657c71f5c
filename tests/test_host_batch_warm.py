"""CPU tests of the warm edits of a batch graph (graph_from_voxels_batch(..., warm=True)): the option reaches the native
handle before its build, and the arguments are parsed and checked as GraphDouble's are before any native call.  The
native batch handle is replaced by a stand-in that records its calls, so no GPU is needed."""
import numpy
import pytest


class _Recorder:
    """Stand-in for the native batch handle: records every call in order."""
    made = []

    def __init__(self, image_shape, batch, device):
        self.image_shape, self.batch = list(image_shape), batch
        self.calls = []
        _Recorder.made.append(self)

    @classmethod
    def factory(cls, image_shape, batch, device=-1):
        return cls(image_shape, batch, device)

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *args: self.calls.append((name,) + args)


@pytest.fixture()
def rec(monkeypatch):
    from medpy_b200 import _lib

    class FakeGraph:
        batch = staticmethod(_Recorder.factory)
    monkeypatch.setattr(_lib, "Graph", FakeGraph)
    _Recorder.made.clear()
    return _Recorder.made


class _DeviceArray:
    """A device array as the argument checks see one: a CUDA array interface (never read here)."""

    def __init__(self, shape=(3,)):
        self.shape = shape
        self.__cuda_array_interface__ = {}


def _graph(batch=3, shape=(4, 5), warm=True):
    import medpy_b200.graphcut as gc
    rng = numpy.random.default_rng(0)
    image = rng.random((batch,) + shape).astype(numpy.float32)
    fg = numpy.zeros(image.shape, bool)
    bg = numpy.zeros(image.shape, bool)
    return gc.graph_from_voxels_batch(fg, bg, image, "difference_exponential", sigma=1.0, warm=warm)


def _last(rec):
    return rec[0].calls[-1]


def test_warm_sets_the_option_before_the_build(rec):
    from medpy_b200 import _lib
    _graph(warm=True)
    names = [c[0] for c in rec[0].calls]
    assert names == ["set_option", "build_voxel_batch"]
    assert rec[0].calls[0][1:] == (_lib._mgc.OPT_WARM, 1)


def test_no_warm_adds_no_call(rec):
    _graph(warm=False)
    assert [c[0] for c in rec[0].calls] == ["build_voxel_batch"]


def test_no_warm_passes_the_arguments_through(rec):
    """Without warm=True the native handle gets the arguments as given (and refuses the call)."""
    g = _graph(warm=False)
    ids = numpy.array([1])
    w = numpy.array([1.0])
    g.add_seeds(ids, None)
    assert _last(rec) == ("add_seeds", ids, None)
    g.add_nweights_dense_warm(0, w, w)
    assert _last(rec) == ("add_nweights_dense_warm", 0, w, w)


def test_seed_masks_and_ids(rec):
    g = _graph()
    fg = numpy.zeros((3, 4, 5), bool)
    fg[1, 2, 3] = fg[2, 0, 0] = True
    g.add_seeds(fg, numpy.array([7, 59], numpy.int32))
    name, f, b = _last(rec)
    assert name == "add_seeds"
    assert f.dtype == numpy.int64 and list(f) == [1 * 20 + 2 * 5 + 3, 40]
    assert b.dtype == numpy.int64 and list(b) == [7, 59]
    g.remove_seeds(None, fg)
    assert _last(rec)[0] == "remove_seeds" and _last(rec)[1] is None


def test_wrong_mask_shape_is_refused(rec):
    g = _graph()
    with pytest.raises(ValueError, match="does not match"):
        g.add_seeds(numpy.zeros((4, 5), bool))
    with pytest.raises(ValueError, match="does not match"):
        g.add_tweights_warm(numpy.zeros((3, 4, 6), bool), 1.0, 0.0)
    assert len(rec[0].calls) == 2           # set_option and the build only


@pytest.mark.parametrize("bad", [-1, 60])
def test_ids_out_of_range_are_refused(rec, bad):
    g = _graph()
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_seeds(numpy.array([0, bad]))
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_tweights_warm(numpy.array([bad]), 1.0, 1.0)
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_nweights_warm(numpy.array([0]), numpy.array([bad]), 1.0, 1.0)
    with pytest.raises(ValueError, match="Invalid node id"):
        g.remove_nweights_warm(numpy.array([bad]), numpy.array([0]), 1.0, 1.0)
    assert len(rec[0].calls) == 2           # set_option and the build only


def test_tweights_broadcast_and_dense(rec):
    g = _graph()
    g.add_tweights_warm(numpy.array([3, 4, 3]), 2.0, numpy.array([1, -2, 3]))
    name, ids, src, snk = _last(rec)
    assert list(ids) == [3, 4, 3] and list(src) == [2.0] * 3 and list(snk) == [1.0, -2.0, 3.0]
    dense = numpy.arange(60.0).reshape(3, 4, 5)
    g.add_tweights_warm(None, dense, 0.5)
    name, ids, src, snk = _last(rec)
    assert ids is None and src.shape == (60,) and (src == dense.ravel()).all() and (snk == 0.5).all()


@pytest.mark.parametrize("shape,axis,lattice_axis", [((7,), 1, 2), ((4, 5), 1, 1), ((4, 5), 2, 2), ((2, 4, 5), 1, 0),
                                                     ((2, 4, 5), 3, 2)])
def test_dense_axis_maps_to_the_lattice(rec, shape, axis, lattice_axis):
    g = _graph(shape=shape)
    f = numpy.ones((3,) + shape)
    g.add_nweights_dense_warm(axis, f, f)
    assert _last(rec)[:2] == ("add_nweights_dense_warm", lattice_axis)
    g.remove_nweights_dense_warm(axis, f, f)
    assert _last(rec)[:2] == ("remove_nweights_dense_warm", lattice_axis)


def test_dense_batch_axis_is_refused(rec):
    g = _graph()
    f = numpy.zeros((3, 4, 5))
    for call in (g.add_nweights_dense_warm, g.remove_nweights_dense_warm):
        with pytest.raises(ValueError, match="batch axis"):
            call(0, f, f)
        with pytest.raises(ValueError, match="out of range"):
            call(3, f, f)
    with pytest.raises(ValueError, match="does not match the batch shape"):
        g.add_nweights_dense_warm(1, numpy.zeros((4, 5)), numpy.zeros((4, 5)))
    assert len(rec[0].calls) == 2           # set_option and the build only


def test_negative_host_decrements_are_refused(rec):
    g = _graph()
    with pytest.raises(ValueError, match="cap holds negative values"):
        g.remove_nweights_warm(numpy.array([0]), numpy.array([1]), -1.0, 0.0)
    f = numpy.zeros((3, 4, 5))
    f[1, 0, 0] = -1.0
    with pytest.raises(ValueError, match="fwd holds negative values"):
        g.remove_nweights_dense_warm(1, f, numpy.zeros_like(f))
    assert len(rec[0].calls) == 2           # set_option and the build only
    # the last plane of the axis in every image names no pair: its entries are not checked
    f[:] = 0.0
    f[:, -1, :] = -1.0
    g.remove_nweights_dense_warm(1, f, numpy.zeros_like(f))
    assert _last(rec)[0] == "remove_nweights_dense_warm"


def test_mixed_host_and_device_arguments_are_refused(rec):
    g = _graph()
    dev = _DeviceArray()
    host = numpy.array([1, 2, 3])
    with pytest.raises(ValueError, match="host or both be device"):
        g.add_seeds(host, dev)
    with pytest.raises(ValueError, match="host or all be device"):
        g.add_tweights_warm(dev, host, 1.0)
    with pytest.raises(ValueError, match="host or all be device"):
        g.add_nweights_warm(host, dev, 1.0, 1.0)
    with pytest.raises(ValueError, match="host or all be device"):
        g.remove_nweights_warm(dev, dev, host, 1.0)
    f = numpy.zeros((3, 4, 5))
    with pytest.raises(ValueError, match="host or both be device"):
        g.add_nweights_dense_warm(1, f, _DeviceArray((3, 4, 5)))
    with pytest.raises(ValueError, match="host or both be device"):
        g.remove_nweights_dense_warm(2, _DeviceArray((3, 4, 5)), f)
    assert len(rec[0].calls) == 2           # set_option and the build only
