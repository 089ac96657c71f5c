"""CPU tests of graph_from_voxels_batch's argument checks and per-image parameter plumbing: the native batch handle is
replaced by a stand-in that records its construction and its build call, so no GPU is needed."""
import math

import numpy
import pytest


class _Recorder:
    """Stand-in for the native batch handle: records the factory arguments and the build call."""
    made = []

    def __init__(self, image_shape, batch, device):
        self.image_shape, self.batch, self.device = list(image_shape), batch, device
        self.build = None
        _Recorder.made.append(self)

    @classmethod
    def factory(cls, image_shape, batch, device=-1):
        return cls(image_shape, batch, device)

    def build_voxel_batch(self, *args):
        self.build = args


@pytest.fixture()
def rec(monkeypatch):
    from medpy_b200 import _lib

    class FakeGraph:
        batch = staticmethod(_Recorder.factory)
    monkeypatch.setattr(_lib, "Graph", FakeGraph)
    _Recorder.made.clear()
    return _Recorder.made


def _arrays(batch=4, shape=(5, 6), dtype=numpy.float32, seed=0):
    rng = numpy.random.default_rng(seed)
    image = (rng.random((batch,) + shape) * 200 - 50).astype(dtype)
    fg = numpy.zeros((batch,) + shape, bool)
    bg = numpy.zeros((batch,) + shape, bool)
    fg[:, 1, 1] = True
    bg[:, 0, 0] = True
    return image, fg, bg


def _build(**kw):
    import medpy_b200.graphcut as gc
    image, fg, bg = kw.pop("arrays", _arrays())
    return gc.graph_from_voxels_batch(fg, bg, image, kw.pop("boundary", "difference_exponential"), **kw)


# build_voxel_batch(prob, alpha, compute_f32, kind, image, sigmas, spacing, norms, fg, bg)
def test_sigma_scalar_is_broadcast(rec):
    _build(sigma=3.5)
    (r,) = rec
    assert r.image_shape == [5, 6] and r.batch == 4
    assert r.build[5] == [3.5] * 4


def test_sigma_per_image(rec):
    _build(sigma=[1.0, 2.0, 3.0, 4.0])
    assert rec[0].build[5] == [1.0, 2.0, 3.0, 4.0]


def test_sigma_length_mismatch_is_refused(rec):
    with pytest.raises(ValueError, match="sigma"):
        _build(sigma=[1.0, 2.0])
    assert not rec


@pytest.mark.parametrize("dtype", [numpy.int16, numpy.uint8, numpy.int32])
@pytest.mark.parametrize("boundary", ["difference_linear", "maximum_linear"])
def test_integer_normalisers_per_image(rec, dtype, boundary):
    image, fg, bg = _arrays(dtype=numpy.float64, seed=2)
    image = image.astype(dtype)
    _build(arrays=(image, fg, bg), boundary=boundary)
    norms = rec[0].build[7]
    for b in range(image.shape[0]):
        want = float(numpy.abs(image[b]).max()) if boundary == "maximum_linear" else float(abs(image[b].max() - image[b].min()))
        assert norms[b] == want


def test_float_normalisers_are_left_to_the_device(rec):
    _build(boundary="difference_linear")
    assert all(math.isnan(x) for x in rec[0].build[7])


def test_regional_and_spacing_are_shared(rec):
    image, fg, bg = _arrays()
    prob = numpy.full(image.shape, 0.25, numpy.float32)
    _build(arrays=(image, fg, bg), prob=prob, alpha=0.5, spacing=(2.0, 3.0))
    args = rec[0].build
    assert args[0] is prob and args[1] == 0.5 and args[2] is True
    assert args[6] == [2.0, 3.0]


def test_shape_mismatch_is_refused(rec):
    image, fg, bg = _arrays()
    with pytest.raises(ValueError, match="fg_markers"):
        _build(arrays=(image, fg[:3], bg))
    with pytest.raises(ValueError, match="prob"):
        _build(arrays=(image, fg, bg), prob=numpy.zeros((4, 5, 7), numpy.float32))
    assert not rec


def test_four_d_images_are_refused(rec):
    image, fg, bg = _arrays(batch=2, shape=(2, 3, 4, 5))
    with pytest.raises(ValueError, match="1-D to 3-D"):
        _build(arrays=(image, fg, bg))
    assert not rec


def test_missing_boundary_term_is_refused(rec):
    with pytest.raises(ValueError, match="boundary"):
        _build(boundary=None)
    assert not rec


class _DeviceArray:
    """A device array as the batch path sees one: shape, dtype and a CUDA array interface (never read here)."""

    def __init__(self, shape, dtype="float32"):
        self.shape = shape
        self.dtype = numpy.dtype(dtype)
        self.__cuda_array_interface__ = {}


def test_index_limit_is_refused(rec):
    import medpy_b200.graphcut as gc
    big = _DeviceArray((2, 1024, 1024, 1024))
    with pytest.raises(ValueError, match="2\\^31"):
        gc.graph_from_voxels_batch(big, big, big, "difference_exponential", sigma=1.0)
    assert not rec
    just_below = _DeviceArray((2, 1023, 1024, 1024))
    assert 2 * 1023 * 1024 * 1024 < 2 ** 31
    gc.graph_from_voxels_batch(just_below, just_below, just_below, "difference_exponential", sigma=1.0)
    (r,) = rec
    assert r.batch == 2 and r.image_shape == [1023, 1024, 1024] and r.build is not None


def test_big_endian_probability_map_is_normalised(rec):
    image, fg, bg = _arrays()
    prob = numpy.full(image.shape, 0.25, numpy.float32)
    _build(arrays=(image, fg, bg), prob=prob.astype(">f4"), alpha=0.5)
    args = rec[0].build
    assert args[0].dtype == numpy.dtype("=f4") and (args[0] == prob).all()
    assert args[2] is True


def test_integer_probability_map_gives_float64_products(rec):
    """An integer map goes as a float64 copy only where its float64 products are numpy's: 1 - p must not wrap around in
    the map's dtype (uint8 at p >= 2, int16 at p <= -32767) and alpha must give float64 products."""
    image, fg, bg = _arrays()
    _build(arrays=(image, fg, bg), prob=numpy.ones(image.shape, numpy.int16), alpha=0.5)
    args = rec[0].build
    assert args[0].dtype == numpy.float64 and args[2] is False
    rec.clear()
    for dtype, value, alpha in ((numpy.uint8, 2, 0.5), (numpy.int16, -32767, 0.5), (numpy.int16, 1, numpy.float32(0.5))):
        prob = numpy.ones(image.shape, dtype)
        prob[1, 2, 3] = value
        with pytest.raises(ValueError, match="probability map"):
            _build(arrays=(image, fg, bg), prob=prob, alpha=alpha)
    assert not rec


def test_float16_probability_map_is_refused(rec):
    image, fg, bg = _arrays()
    with pytest.raises(ValueError, match="probability map"):
        _build(arrays=(image, fg, bg), prob=numpy.ones(image.shape, numpy.float16), alpha=0.5)
    assert not rec

