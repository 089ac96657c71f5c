"""CPU tests of which t-link arithmetic each entry point gives a probability map, over the regional term's whole domain.

``regional_probability_map`` gives every voxel ``(p * alpha, (1 - p) * alpha)`` in the dtype numpy forms them in: a
float32 map times a Python float stays float32, a ``numpy.float64`` alpha makes ``p * alpha`` float64 but leaves
``1 - p`` rounded in float32, an integer map forms ``1 - p`` in its own dtype and wraps around.  The native build knows
two arithmetics (float32 products with ``(float)alpha``, float64 products) and a dense fallback that takes the products
as given.  Each entry point decides which one a map and alpha get:

  * ``graph_from_voxels`` with ``energy_voxel.regional_probability_map``;
  * ``graph_from_voxels_batch``;
  * ``graph_from_device_arrays``, with a host stand-in for the device map;
  * ``distributed.graphcut_slab``'s float32 decision for the slab builds.

The native handle is replaced by a recorder; the arithmetic the kernels apply (``tlink_replay``, ``k_regional``,
``k_tweights_dense``) is applied to what reached it and must equal ``oracle.energy_terms.regional_probability_tweights``
bit for bit (-0.0 apart from +0.0, any NaN for NaN), or the entry point must have raised before any native call.  Which
maps are refused is pinned too: only those whose products neither arithmetic forms exactly."""
import warnings

import numpy
import pytest

from oracle import energy_terms as et

# ---- the domain ----------------------------------------------------------------------------------------------------
FLOAT_DTYPES = ("<f2", "<f4", "<f8", ">f4", ">f8")
INT_DTYPES = ("u1", "u2", "i1", "i2", "i4", "i8", "<u8", ">i2")
ALPHA_VALUES = (0.0, -0.0, 5e-324, 1e-30, 0.1, 1.0, -0.1, 3.4e38, 1e39, 1e300)


def _alphas():
    out, seen = [], set()
    for v in ALPHA_VALUES:
        for make in (float, int, numpy.float32, numpy.float64):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                a = make(v)
            key = (type(a).__name__, numpy.asarray(a, dtype=numpy.float64).tobytes())
            if key not in seen:
                seen.add(key)
                out.append(a)
    return out


ALPHAS = _alphas()


def _float_map(dtype):
    """Every special p of the dtype: signed zeros, 1 and 0.5 with their neighbours, subnormal and tiny, +-1e-30, values
    above 1 and below 0, the dtype's extremes, infinities and NaNs (quiet, and a negative payload)."""
    dt = numpy.dtype(dtype)
    ft = dt.newbyteorder("=").type
    fi = numpy.finfo(ft)
    one, half = ft(1), ft(0.5)
    neg_nan = numpy.array(-numpy.nan, ft)
    with numpy.errstate(all="ignore"):
        v = [ft(0), -ft(0), one, numpy.nextafter(one, ft(2)), numpy.nextafter(one, ft(0)), half,
             numpy.nextafter(half, ft(1)), numpy.nextafter(half, ft(0)), fi.smallest_subnormal, fi.tiny,
             -fi.smallest_subnormal, ft(1e-30), ft(-1e-30), ft(1.5), ft(2), ft(-0.5), ft(1e30), fi.max, -fi.max,
             ft(numpy.inf), ft(-numpy.inf), ft(numpy.nan), neg_nan, ft(0.15), ft(0.95)]
    return numpy.array(v, dtype=ft).astype(dt)


def _int_maps(dtype):
    """(all specials: 0, 1, 2, the extremes and one above the minimum) and a map whose ``1 - p`` never wraps."""
    dt = numpy.dtype(dtype)
    ii = numpy.iinfo(dt)
    full = numpy.array(sorted({0, 1, 2, ii.max, ii.min, ii.min + 1}), dtype=dt)
    if ii.min == 0:
        safe = numpy.array([0, 1, 1, 0], dtype=dt)
    else:
        safe = numpy.array([0, 1, 2, ii.min + 2, max(ii.max, 0) if ii.max < 2 ** 53 else 2 ** 53, -5], dtype=dt)
    return full, safe


def _maps():
    out = [(dt, _float_map(dt)) for dt in FLOAT_DTYPES]
    for dt in INT_DTYPES:
        full, safe = _int_maps(dt)
        out += [(dt + "-full", full), (dt + "-safe", safe)]
    out.append(("bool", numpy.array([True, False, True])))
    return out


MAPS = _maps()


# ---- the arithmetic behind the native calls -------------------------------------------------------------------------
def _reference(prob, alpha):
    """regional_probability_tweights, or the exception type numpy raises forming them."""
    with numpy.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return et.regional_probability_tweights(prob, alpha)
        except (OverflowError, TypeError) as e:
            return type(e)


def _kernel(prob, alpha, compute_f32):
    """The products of tlink_replay / k_regional on the map the native call received."""
    prob = numpy.asarray(prob)
    assert prob.dtype.isnative and prob.dtype.type in (numpy.float32, numpy.float64), prob.dtype
    assert isinstance(alpha, float), type(alpha)           # a C double
    with numpy.errstate(all="ignore"):
        if compute_f32:
            assert prob.dtype == numpy.float32         # the kernels read a float32 map as float, exactly
            p, a = prob.ravel(), numpy.float32(alpha)  # (float)alpha, round to nearest
            return (p * a).astype(float), ((numpy.float32(1) - p) * a).astype(float)
        p = prob.ravel().astype(numpy.float64)
        return p * alpha, (1.0 - p) * alpha


def _same(got, want):
    g, w = numpy.asarray(got, dtype=numpy.float64).ravel(), numpy.asarray(want, dtype=numpy.float64).ravel()
    assert g.shape == w.shape
    nan = numpy.isnan(w)
    assert numpy.array_equal(numpy.isnan(g), nan)
    return numpy.array_equal(g[~nan].view(numpy.int64), w[~nan].view(numpy.int64))


def _exact(calls, prob, alpha):
    """The products of every recorded native t-link call equal the reference bit for bit."""
    want = _reference(prob, alpha)
    assert not isinstance(want, type), ("the reference raised", want)
    (call,) = calls
    got = _kernel(*call[1:]) if call[0] == "products" else call[1:]
    for g, w, what in zip(got, want, ("src", "snk")):
        assert _same(g, w), (what, numpy.asarray(g).ravel(), w)


def _pure(prob, alpha):
    """numpy forms both products in the map's own float32 or float64 dtype: every entry point must accept these."""
    z = numpy.asarray(prob)[:0]
    try:
        dtypes = {z.dtype.newbyteorder("="), (z * alpha).dtype, ((1 - z) * alpha).dtype}
    except (OverflowError, TypeError):     # numpy cannot form them at all (a huge Python int with an integer map)
        return False
    return dtypes in ({numpy.dtype(numpy.float32)}, {numpy.dtype(numpy.float64)})


def _float64_products(prob, alpha):
    """numpy forms both products of this map in float64."""
    z = numpy.asarray(prob)[:0]
    try:
        return (z * alpha).dtype == numpy.float64 and ((1 - z) * alpha).dtype == numpy.float64
    except (OverflowError, TypeError):
        return False


def _wraps_or_rounds(prob):
    """An integer map whose 1 - p wraps around in its dtype, or whose p or 1 - p a double does not hold."""
    p = numpy.asarray(prob)
    ii = numpy.iinfo(p.dtype)
    v = [int(x) for x in p.ravel()]
    return any(1 - x < ii.min or 1 - x > ii.max or abs(x) > 2 ** 53 or abs(1 - x) > 2 ** 53 for x in v)


# ---- recorders ------------------------------------------------------------------------------------------------------
class _Lattice:
    """Stand-in for the native lattice handle: keeps the t-link inputs of the build."""

    def __init__(self, shape, device=-1):
        self.shape, self.calls = list(shape), []

    def set_option(self, *a):
        pass

    def check_deferred(self):
        pass

    def set_stream(self, s):
        pass

    def build_voxel_graph(self, prob, alpha, compute_f32, kind, image, sigma, spacing, norm, fg, bg):
        if prob is not None:
            self.calls.append(("products", getattr(prob, "host", prob), alpha, compute_f32))

    def add_regional_probability(self, prob, alpha, compute_f32):
        self.calls.append(("products", prob, alpha, compute_f32))

    def add_tweights_dense(self, src, snk):
        self.calls.append(("dense", numpy.array(src), numpy.array(snk)))

    def add_markers(self, fg, bg):
        pass


class _Batch:
    def __init__(self, image_shape, batch, device=-1):
        self.calls = []

    def set_option(self, *a):
        pass

    def build_voxel_batch(self, prob, alpha, compute_f32, *rest):
        self.calls.append(("products", prob, alpha, compute_f32))


class _DeviceMap:
    """A device array as the entry points see one: shape, dtype and a CUDA array interface; ``host`` holds the values
    the recorders read in its place."""

    def __init__(self, host):
        self.host = host
        self.shape = host.shape
        self.dtype = host.dtype
        self.__cuda_array_interface__ = {}


@pytest.fixture()
def made(monkeypatch):
    from medpy_b200 import _lib
    handles = []

    def lattice(shape, device=-1):
        handles.append(_Lattice(shape, device))
        return handles[-1]

    def batch(image_shape, batch, device=-1):
        handles.append(_Batch(image_shape, batch, device))
        return handles[-1]
    lattice.batch = batch
    monkeypatch.setattr(_lib, "Graph", lattice)
    return handles


# ---- entry points ---------------------------------------------------------------------------------------------------
def _single(prob, alpha):
    import medpy_b200.graphcut as gc
    z = numpy.zeros(prob.shape, bool)
    g = gc.graph_from_voxels(z, z, regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(prob, alpha))
    g.check_deferred()


def _batch(prob, alpha):
    import medpy_b200.graphcut as gc
    stack = numpy.stack([prob, prob[::-1]])
    img = numpy.zeros(stack.shape, numpy.float32)
    gc.graph_from_voxels_batch(numpy.zeros(stack.shape, bool), numpy.zeros(stack.shape, bool), img,
                               "difference_exponential", sigma=1.0, prob=stack, alpha=alpha)
    return stack


def _device(prob, alpha):
    from medpy_b200.graphcut.device import graph_from_device_arrays
    z = _DeviceMap(numpy.zeros(prob.shape, numpy.uint8))
    graph_from_device_arrays(z, z, prob=_DeviceMap(prob), alpha=alpha)


class _Stop(Exception):
    pass


def _slab(monkeypatch, prob, alpha):
    """graphcut_slab up to its slab build, whose arguments it records."""
    from medpy_b200 import distributed
    seen = []

    class Solver:
        def __init__(self, shape, group=None, handle_factory=None):
            pass

        def local_slice(self, a):
            return a

        def build(self, fg, bg, prob_local=None, alpha=None, compute_f32=False, **kw):
            seen.append(("products", prob_local, float(alpha), compute_f32))
            raise _Stop
    monkeypatch.setattr(distributed, "SlabSolver", Solver)
    z = numpy.zeros(prob.shape, bool)
    with pytest.raises(_Stop):
        distributed.graphcut_slab(z, z, prob=prob, alpha=alpha)
    return seen


def _cases():
    return [pytest.param(m, a, id=f"{name}-{type(a).__name__}({float(a)!r})") for name, m in MAPS for a in ALPHAS]


@pytest.mark.parametrize("prob,alpha", _cases())
def test_single_image(made, prob, alpha):
    """graph_from_voxels decides for every map and alpha; it refuses only what the reference refuses."""
    want = _reference(prob, alpha)
    with numpy.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if isinstance(want, type):
            with pytest.raises(want):
                _single(prob, alpha)
            return
        _single(prob, alpha)
    _exact(made[0].calls, prob, alpha)


@pytest.mark.parametrize("prob,alpha", _cases())
def test_batch(made, prob, alpha):
    """graph_from_voxels_batch gives each image the reference's products or raises ValueError before any native call:
    exactly where numpy's products are neither pure float32 nor pure float64 and, for an integer map, not those of its
    float64 copy."""
    with numpy.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = _reference(prob, alpha)
        stack = numpy.stack([prob, prob[::-1]])
        try:
            _batch(prob, alpha)
        except (ValueError, OverflowError, TypeError):
            assert not made, "a refused batch reached the native layer"
            if isinstance(want, type):
                return
            assert not _pure(prob, alpha), "a map of pure float32 or float64 products was refused"
            if prob.dtype.kind == "b" and _float64_products(prob, alpha):
                raise AssertionError("a bool map, whose float64 copy gives numpy's products exactly, was refused")
            if prob.dtype.kind in "iu" and _float64_products(prob, alpha):
                assert _wraps_or_rounds(prob), "an integer map its float64 copy gives exactly was refused"
            return
    assert not isinstance(want, type), ("the batch accepted what the reference refuses", want)
    _exact(made[0].calls, stack, alpha)


@pytest.mark.parametrize("prob,alpha", _cases())
def test_device_arrays(made, prob, alpha):
    """graph_from_device_arrays has no dense fallback: it takes pure float32 and float64 products and refuses every
    other map before any native call."""
    if not prob.dtype.isnative:
        pytest.skip("device arrays are in native byte order")
    with numpy.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if isinstance(_reference(prob, alpha), type):
            with pytest.raises((OverflowError, TypeError)):
                _device(prob, alpha)
            return
        if not _pure(prob, alpha):
            with pytest.raises(ValueError, match="probability map"):
                _device(prob, alpha)
            assert not any(h.calls for h in made)
            return
        _device(prob, alpha)
    _exact(made[0].calls, prob, alpha)


@pytest.mark.parametrize("prob,alpha", _cases())
def test_slab_decision(monkeypatch, prob, alpha):
    """graphcut_slab hands its slabs float32 products exactly where numpy forms them, and refuses the maps neither
    arithmetic forms."""
    pytest.importorskip("torch")
    with numpy.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if isinstance(_reference(prob, alpha), type):
            with pytest.raises((OverflowError, TypeError)):
                _slab(monkeypatch, prob, alpha)
            return
        if not _pure(prob, alpha) or not prob.dtype.isnative:
            with pytest.raises(ValueError, match="probability map"):
                _slab(monkeypatch, prob, alpha)
            return
        seen = _slab(monkeypatch, prob, alpha)
    _exact(seen, prob, alpha)


def test_batch_integer_maps_that_wrap_are_refused(made):
    """The rows the batch used to get wrong: 1 - p wraps in uint8 at p >= 2 and in int16 at p <= -32767, where its
    float64 copy gave (1.0 - p) * alpha."""
    for prob in (numpy.array([0, 2, 200, 255], numpy.uint8), numpy.array([0, -32768], numpy.int16),
                 numpy.array([5, -32767], numpy.int16)):
        with pytest.raises(ValueError, match="cannot be formed exactly"):
            _batch(prob, 0.1)
    assert not made
    ok = numpy.array([0, 1, -32766, 32767], numpy.int16)
    stack = _batch(ok, 0.1)
    _exact(made[0].calls, stack, 0.1)


def test_batch_bool_map_gives_float64_products(made):
    """numpy forms a bool map's products in float64 (1 - p in int64, never wrapping): its float64 copy gives them."""
    prob = numpy.array([True, False, True, True])
    for alpha in (0.1, numpy.float64(-0.1), 1e300):
        stack = _batch(prob, alpha)
        assert made[-1].calls[0][1].dtype == numpy.float64 and made[-1].calls[0][3] is False
        _exact(made[-1].calls, stack, alpha)
    with pytest.raises(ValueError, match="cannot be formed exactly"):
        _batch(prob, numpy.float32(0.1))        # float32 p * alpha next to a float64 1 - p


def test_batch_float32_map_with_numpy_float64_alpha_is_refused(made):
    """numpy rounds 1 - p in float32 and multiplies in float64 here: neither arithmetic of the build forms that."""
    prob = numpy.array([1e-30, 0.3, 0.7], numpy.float32)
    src, snk = et.regional_probability_tweights(prob, numpy.float64(0.1))
    assert snk[0] == 0.1 and src.dtype == numpy.float64          # 1 - 1e-30 rounds to 1 in float32
    with pytest.raises(ValueError, match="cannot be formed exactly"):
        _batch(prob, numpy.float64(0.1))
    assert not made
    _batch(prob, 0.1)                 # a Python float keeps float32 products
    assert made[0].calls[0][3] is True


def test_add_tweights_pass_keeps_the_sign_of_an_untouched_cap():
    """Graph::add_tweights adds delta to one side only: the other keeps its bits, so a -0.0 cap_source stays -0.0 and
    tr = -0.0 - 0.0 is -0.0 (p = -0.0, alpha = 0.0)."""
    tr = numpy.zeros(2)
    et.add_tweights_pass(tr, 0.0, numpy.array([-0.0, 0.0]), numpy.array([0.0, -0.0]))
    assert numpy.signbit(tr[0]) and not numpy.signbit(tr[1])
    prob = et.build_problem(numpy.zeros(1, bool), numpy.zeros(1, bool), regional=(numpy.array([-0.0]), 0.0))
    assert numpy.signbit(prob["tr"][0])
