"""The n-link weights of every build path against high-precision references, over each boundary term's whole domain.

The other weight tests compare the build paths with each other (lean against refused blocks, lazy against eager, fused
against per-term, batch against single image) on smooth volumes whose arguments stay small; a defect all paths share
passes them.  Here every path is read back with get_edge, in both directions, and compared with a reference on images
whose neighbour pairs drive the term's input x = |a - b| (or max(|a|, |b|), in the input dtype, for the maximum terms)
across the whole domain:

  * linear, division: bit for bit with oracle.energy_terms.boundary_weights, NaN where it has NaN -- including the
    linear normaliser M with a NaN anywhere in the image (numpy's max / min propagate it: every weight is NaN);
  * exponential: the device's bits are the host emulation's (tests/emu/expneg_emu.cpp, certified against a 200-bit
    exp by test_expneg_emulation.py) for the argument x^2 * (1 / sigma^2) the kernels form, and within exp_bound() of
    numpy's weights;
  * power: within 2 ulp of the 200-bit pow(b, sigma), b = 1 / (x + 1) as numpy forms it (CUDA documents 2 ulp for
    double pow); special bases and exponents give numpy's value exactly;
  * spacing: the weight with a spacing is the one without it divided by the axis's spacing, correctly rounded; a
    spacing that makes a weight zero or negative is refused with ValueError exactly where build_problem refuses;
  * every path gives the same bits as every other for the same case.
"""
import contextlib
import math
import os
import sys

import numpy
import pytest

import expneg_ref as ref

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
DBL_MIN = sys.float_info.min
KINDS = ("difference_linear", "difference_exponential", "difference_division", "difference_power",
         "maximum_linear", "maximum_exponential", "maximum_division", "maximum_power")
# the 3-D build paths: lazy fused build with lean and refused blocks, every block refused, eager fused, per-term kernels
PATHS_3D = {"lazy": {}, "refuse_all": {"MEDPY_GC_BUILD_REFUSE_ALL": "1"}, "eager": {"MEDPY_GC_LAZY_CAPS": "0"},
            "per_term": {"MEDPY_GC_FUSE": "0"}}
SAMPLE = 400          # pairs read per axis (all of them when there are fewer)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return ref.build_emu(tmp_path_factory.mktemp("expneg"))


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _use_max(kind):
    # boundary_maximum_division evaluates the difference skeleton (energy_voxel.py:347)
    return kind.startswith("maximum") and kind != "maximum_division"


def _fn(kind):
    return kind.split("_")[1]


# ------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------
def _pair_x(kind, image):
    """x of every pair, per axis, as the reference forms it: numpy.abs in the input dtype under the maximum terms, then
    float64, then max(a, b) or |a - b| (energy_voxel.py:551-558, 601-606, 634)."""
    img = numpy.asarray(image)
    if _use_max(kind):
        img = numpy.abs(img)
    img = img.astype(numpy.float64)
    out = []
    for d in range(img.ndim):
        lo = [slice(None)] * img.ndim
        hi = [slice(None)] * img.ndim
        lo[d] = slice(0, -1)
        hi[d] = slice(1, None)
        a, b = img[tuple(lo)], img[tuple(hi)]
        with numpy.errstate(all="ignore"):
            out.append(numpy.maximum(a, b) if _use_max(kind) else numpy.absolute(a - b))
    return out


def exp_bound(w_ref, t):
    """|w - w_ref| allowed between the device's exponential weight w and numpy's w_ref, t = x^2 / sigma^2 (u = 2^-53):

        (4u t + 4u) w_ref + 2^-1074

    The device forms t_d = RN(RN(x^2) * RN(1 / s2)), numpy t_r = RN(RN(x^2) / s2) (s2 = pow(sigma, 2)): three roundings
    of relative size <= u each, so t_d = t_r (1 + e) with |e| <= 3u + O(u^2), and exp(-t_d) = exp(-t_r) (1 + e')
    with |e'| <= 3u t + O((u t)^2) -- 4u t covers the second-order terms for every t where the weight is not subnormal
    (u t < 1e-13).  Each side then evaluates exp within 1 ulp (exp_neg: test_expneg_emulation.py; numpy's libm:
    < 1 ulp), i.e. within 2u relative while the result is normal: 4u.  In the subnormal range an ulp is the absolute
    2^-1074; the device is within 0.84 of it, glibc's exp within 0.5 + a hair, so together below 2^-1074 + the rest."""
    return (4.0 * U * t + 4.0 * U) * w_ref + 2.0 ** -1074


def _exp_unclamp(w, t):
    """The clamp of 0 to DBL_MIN (energy_voxel.py:235) taken back where exp(-t) is far below DBL_MIN (t > 709): there
    the two sides may round the last subnormal differently, to 0 (-> DBL_MIN) on one and 2^-1074 on the other."""
    w = numpy.array(w, dtype=numpy.float64)
    w[(w == DBL_MIN) & (t > 709.0)] = 0.0
    return w


def _pow_special(b, sigma):
    return ~numpy.isfinite(b) | (b <= 0.0) | (b == 1.0) | (not math.isfinite(sigma)) | (sigma == 0.0)


# ------------------------------------------------------------------------------------------------------
# building and reading
# ------------------------------------------------------------------------------------------------------
def _build(kind, image, sigma, spacing=False, path="lazy"):
    import medpy_b200.graphcut as gc
    shape = numpy.shape(image)
    z = numpy.zeros(shape, bool)
    if path == "cuda":
        import torch
        from medpy_b200.graphcut.device import graph_from_device_arrays
        tz = torch.zeros(shape, dtype=torch.bool, device="cuda")
        g = graph_from_device_arrays(tz, tz, image=torch.from_numpy(numpy.ascontiguousarray(image)).cuda(), boundary=kind,
                                     sigma=sigma, spacing=spacing)
        g.check_deferred()
        return g
    img = numpy.asfortranarray(image) if path == "fortran" else image
    fn = getattr(gc.energy_voxel, "boundary_" + kind)
    args = (img, spacing) if _fn(kind) == "linear" else (img, sigma, spacing)
    with _env(**PATHS_3D.get(path, {})):
        return gc.graph_from_voxels(z, z, boundary_term=fn, boundary_term_args=args)


def _marked(image):
    """The cells whose pairs are always read: the head of the ramps (the branch points), non-finite, subnormal and -0
    cells, and the extremes of an integer dtype."""
    img = numpy.asarray(image)
    m = numpy.zeros(img.shape, bool)
    m.reshape(-1)[:160] = True
    if img.dtype.kind == "f":
        m |= ~numpy.isfinite(img) | ((numpy.abs(img) < numpy.finfo(img.dtype).tiny) & (img != 0))
        m |= (img == 0) & numpy.signbit(img)
    elif img.dtype.kind in "iu":
        m |= (img == numpy.iinfo(img.dtype).min) | (img == numpy.iinfo(img.dtype).max)
    return m


def _sample(shape, rng, count=SAMPLE, marked=None):
    """Per axis d: the flat ids p of a sample of the pairs (p, p + stride_d) -- every pair that touches a `marked` cell
    (up to 4 * count) and `count` others -- and their coordinates."""
    strides = [int(numpy.prod(shape[d + 1:])) for d in range(len(shape))]
    out = []
    for d in range(len(shape)):
        short = list(shape)
        short[d] -= 1
        m = int(numpy.prod(short))
        idx = numpy.arange(m) if m <= count else rng.choice(m, count, replace=False)
        if marked is not None and m > count:
            lo = [slice(None)] * len(shape)
            hi = [slice(None)] * len(shape)
            lo[d] = slice(0, -1)
            hi[d] = slice(1, None)
            touch = numpy.flatnonzero(marked[tuple(lo)] | marked[tuple(hi)])[:4 * count]
            idx = numpy.union1d(idx, touch)
        idx = numpy.sort(idx)
        coords = numpy.unravel_index(idx, short)
        p = numpy.ravel_multi_index(coords, shape)
        out.append((p, coords, strides[d]))
    return out


def _read(get_edge, sample, offset=0):
    """(forward, backward) weights of the sampled pairs, per axis; ids shifted by `offset` (image b of a batch)."""
    out = []
    for p, _, st in sample:
        f = numpy.array([get_edge(int(q) + offset, int(q) + st + offset) for q in p])
        b = numpy.array([get_edge(int(q) + st + offset, int(q) + offset) for q in p])
        out.append((f, b))
    return out


def _check(emu, kind, image, sigma, got, sample, spacing=False):
    """The sampled weights of one graph against the references; returns the largest ratio |w - w_ref| / bound of the
    exponential cases (0 otherwise)."""
    from oracle import energy_terms as et
    with numpy.errstate(all="ignore"):
        want = et.boundary_weights(kind, image, sigma, spacing)
    xs = _pair_x(kind, image)
    worst = 0.0
    for d, ((p, coords, _), (f, b)) in enumerate(zip(sample, got)):
        assert numpy.array_equal(f.view(numpy.int64), b.view(numpy.int64)), (kind, d, "asymmetric pair")
        w_ref = want[d][coords]
        x = xs[d][coords]
        fn = _fn(kind)
        if fn in ("linear", "division"):
            bad = ~((f == w_ref) | (numpy.isnan(f) & numpy.isnan(w_ref)))
            assert not bad.any(), (kind, d, x[bad][:4], f[bad][:4], w_ref[bad][:4])
            continue
        if spacing:
            continue                     # spacing: test_spacing divides the weights checked without it
        if fn == "exponential":
            s2 = math.pow(sigma, 2)
            e = emu.term(x, s2)
            e = numpy.where(e <= 0.0, DBL_MIN, e)
            bad = (f.view(numpy.int64) != e.view(numpy.int64)) & ~(numpy.isnan(f) & numpy.isnan(e))
            assert not bad.any(), (kind, d, sigma, x[bad][:4], f[bad][:4], e[bad][:4])
            with numpy.errstate(all="ignore"):
                t = numpy.power(x, 2) / s2
            both_nan = numpy.isnan(f) & numpy.isnan(w_ref)
            assert numpy.array_equal(numpy.isnan(f), numpy.isnan(w_ref)), (kind, d, sigma)
            ok = ~both_nan
            fu, ru = _exp_unclamp(f[ok], t[ok]), _exp_unclamp(w_ref[ok], t[ok])
            with numpy.errstate(all="ignore"):
                bound = exp_bound(ru, t[ok])
                err = numpy.abs(fu - ru)
            good = (fu == ru) | (err <= bound)       # equal values also where t is infinite (inf * 0 bound)
            assert good.all(), (kind, d, sigma, x[ok][~good][:4], fu[~good][:4], ru[~good][:4])
            inexact = fu != ru
            if inexact.any():
                worst = max(worst, float((err[inexact] / bound[inexact]).max()))
        else:
            with numpy.errstate(all="ignore"):
                base = 1.0 / (x + 1)
            special = _pow_special(base, sigma) | ~numpy.isfinite(w_ref) | (w_ref == DBL_MIN) | (f == DBL_MIN)
            bad = special & ~((f == w_ref) | (numpy.isnan(f) & numpy.isnan(w_ref)))
            assert not bad.any(), (kind, d, sigma, x[bad][:4], f[bad][:4], w_ref[bad][:4])
            for g, bb in zip(f[~special], base[~special]):
                e = ref.ulp_error(g, ref.pow_exact(bb, sigma))
                assert e <= 2.0, (kind, sigma, bb, g, e)
    return worst


def _paths(ndim):
    return list(PATHS_3D) + ["cuda", "fortran"] if ndim == 3 else ["lazy", "per_term", "fortran"]


def _run_case(emu, kind, image, sigma, spacing=False, paths=None, seed=0):
    """Every path of the case's dimension against the references and against each other; returns the worst exponential
    bound ratio."""
    from oracle import energy_terms as et
    rng = numpy.random.default_rng(seed)
    shape = numpy.shape(image)
    sample = _sample(shape, rng, marked=_marked(image))
    with numpy.errstate(all="ignore"):
        refused = None              # the exception the reference raises: ValueError for weights <= 0, OverflowError for
        try:                        # math.pow(sigma, 2) of a huge sigma, TypeError for bool - bool
            et.build_problem(numpy.zeros(shape, bool), numpy.zeros(shape, bool), boundary=(kind, image, sigma, spacing))
        except (ValueError, OverflowError, TypeError) as e:
            refused = type(e)
    first, worst = None, 0.0
    cuda_ok = numpy.asarray(image).dtype.type in (numpy.float32, numpy.float64, numpy.uint8, numpy.int16, numpy.int32)
    for path in paths or _paths(len(shape)):
        if path == "cuda" and not cuda_ok:
            continue
        if refused:
            if path == "cuda" and refused is not ValueError:
                continue            # device arrays skip the Python term functions (their sigma is used as given)
            with pytest.raises(refused):
                g = _build(kind, image, sigma, spacing, path)
                g.maxflow()
            continue
        g = _build(kind, image, sigma, spacing, path)
        got = _read(g.get_edge, sample)
        if first is None:            # the reference on one path, the same bits on every other
            worst = _check(emu, kind, image, sigma, got, sample, spacing)
            first = got
        else:
            for (f0, _), (f1, _) in zip(first, got):
                assert numpy.array_equal(f0.view(numpy.int64), f1.view(numpy.int64)), (kind, path, "differs from", paths)
    return refused, worst


# ------------------------------------------------------------------------------------------------------
# images
# ------------------------------------------------------------------------------------------------------
def _branch_t():
    """t at and around every branch point of exp_neg, and the top of exp_neg_inrange's range."""
    pts = [ref.ln2_multiple(k) for k in (1020.5, 1022, 1074, 1075)] + [745.2, 700.0, 708.39]
    return numpy.array([v for x in pts for v in ref.neighbours(x, 6)])


def _exp_image(kind, dtype, shape, sigma, rng, extra_t=()):
    """An image whose pairs cover t = x^2 / sigma^2 over [0, 800] and `extra_t`: the first half of the z planes a
    checkerboard with every pair's t in [600, 700] (the blocks pass the lazy build's range test: lean, exp_neg_inrange
    at the top of its range), the second half a ramp (refused blocks: the full exp_neg)."""
    n = int(numpy.prod(shape))
    t = numpy.concatenate([numpy.asarray(extra_t, float), rng.uniform(0.0, 800.0, n)])[:n]
    x = numpy.sqrt(t) * sigma
    if _use_max(kind):
        ramp = x * numpy.where(numpy.arange(n) % 2 == 0, 1.0, -1.0)
    else:
        ramp = numpy.cumsum(x * numpy.where(numpy.arange(n) % 2 == 0, 1.0, -1.0))
    img = ramp.reshape(shape)
    if len(shape) >= 3:
        h = shape[0] // 2
        grid = numpy.indices(shape).sum(axis=0) % 2 == 1
        ordinary = rng.uniform(numpy.sqrt(600.0), numpy.sqrt(700.0), shape) * sigma
        if _use_max(kind):
            block = ordinary * numpy.where(grid, 1.0, -1.0)
        else:
            block = numpy.where(grid, ordinary, 0.0)
        img[:h] = block[:h]
    return img.astype(dtype)


def _specials(img, rng, subnormal=True):
    """A few non-finite and subnormal cells, away from the lean half."""
    img = img.copy()
    flat = img.reshape(-1)
    n = flat.size
    tiny = numpy.finfo(img.dtype).smallest_subnormal
    vals = [numpy.nan, numpy.inf, -numpy.inf, -0.0] + ([tiny, -tiny * 3] if subnormal else [])
    pos = rng.choice(numpy.arange(n // 2, n), len(vals), replace=False)
    flat[pos] = numpy.array(vals, dtype=img.dtype)
    return img


# ------------------------------------------------------------------------------------------------------
# the exponential term
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["difference_exponential", "maximum_exponential"])
@pytest.mark.parametrize("dtype", [numpy.float64, numpy.float32])
@pytest.mark.parametrize("shape", [(16, 12, 72), (3000,), (40, 60), (6, 5, 8, 7)])
def test_exponential_domain(emu, kind, dtype, shape):
    """t over [0, 800], the branch points (sigma = 1: t = RN(x^2)), lean and refused blocks."""
    rng = numpy.random.default_rng(len(shape))
    img = _exp_image(kind, dtype, shape, 1.0, rng, extra_t=_branch_t())
    _run_case(emu, kind, img, 1.0)
    _run_case(emu, kind, _exp_image(kind, dtype, shape, 3.7, rng), 3.7)


@pytest.mark.parametrize("kind", ["difference_exponential", "maximum_exponential"])
@pytest.mark.parametrize("sigma", [0.0, -2.5, 1e-151, 1e-155, 1e-160, 1e154, 1e200, math.inf, math.nan])
def test_exponential_sigma_extremes(emu, kind, sigma):
    """sigma = 0 (x = 0 gives NaN, x > 0 DBL_MIN), a reciprocal >= 1e300 or infinite (the division form), a subnormal
    or infinite sigma^2, NaN."""
    rng = numpy.random.default_rng(5)
    shape = (10, 9, 40)
    img = rng.normal(0.0, 3.0, shape)
    img[2:4] = 0.0                     # x = 0 pairs
    scale = abs(sigma) if math.isfinite(sigma) and sigma != 0.0 else 1.0
    img[5:] *= scale * 10.0            # t of order 100..1000 for the small sigmas
    _run_case(emu, kind, img, sigma, paths=["lazy", "refuse_all", "per_term"])


@pytest.mark.parametrize("kind", ["difference_exponential", "maximum_exponential"])
def test_exponential_non_finite_and_subnormal_cells(emu, kind, request):
    if kind == "maximum_exponential":
        request.applymarker(pytest.mark.xfail(strict=True, reason=(
            "the kernels form max(|a|, |b|) with fmax, which drops a NaN cell; numpy.maximum gives NaN")))
    rng = numpy.random.default_rng(9)
    for dtype in (numpy.float64, numpy.float32):
        img = _specials(_exp_image(kind, dtype, (16, 12, 40), 2.0, rng), rng)
        _run_case(emu, kind, img, 2.0)


@pytest.mark.parametrize("kind", ["difference_exponential", "maximum_exponential"])
def test_exponential_inf_and_subnormal_cells(emu, kind):
    """The non-finite cells the maximum terms handle like numpy: +-inf (no NaN), and subnormals."""
    rng = numpy.random.default_rng(10)
    for dtype in (numpy.float64, numpy.float32):
        img = _exp_image(kind, dtype, (16, 12, 40), 2.0, rng)
        flat = img.reshape(-1)
        tiny = numpy.finfo(dtype).smallest_subnormal
        flat[-200::7] = numpy.array([numpy.inf, -numpy.inf, tiny, -tiny, -0.0] * 6, dtype=dtype)[:len(flat[-200::7])]
        _run_case(emu, kind, img, 2.0)


@pytest.mark.parametrize("dtype", [numpy.uint8, numpy.int16, numpy.int32, numpy.bool_, numpy.uint16, numpy.int64,
                                   numpy.float16])
@pytest.mark.parametrize("kind", ["difference_exponential", "maximum_exponential"])
def test_exponential_dtypes(emu, kind, dtype):
    rng = numpy.random.default_rng(11)
    shape = (12, 10, 48)
    if dtype == numpy.bool_:
        img = rng.random(shape) < 0.5
        sigma = 0.04                         # t = 625 for every unequal pair
    else:
        info = numpy.iinfo(dtype) if numpy.issubdtype(dtype, numpy.integer) else numpy.finfo(dtype)
        lo, hi = max(float(info.min), -60000.0), min(float(info.max), 60000.0)
        img = rng.uniform(lo, hi, shape).astype(dtype)
        sigma = (hi - lo) / math.sqrt(800.0)
    if dtype == numpy.int16:
        img.reshape(-1)[-50:-40] = -32768     # numpy.abs wraps under the maximum terms
    _run_case(emu, kind, img, sigma)


# ------------------------------------------------------------------------------------------------------
# the power term
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["difference_power", "maximum_power"])
@pytest.mark.parametrize("sigma", [0.5, 2.0, 37.25, 1050.0, 1e6, -0.5, -3.3, 0.0, math.inf, -math.inf, math.nan])
def test_power_domain(emu, kind, sigma):
    """x from 0 (b = 1) over small fractions (b near 1, where pow(b, sigma) spans the subnormals for sigma = 1050) to
    1e300 (b near 0); negative and fractional sigma; sigma large enough to underflow to DBL_MIN."""
    rng = numpy.random.default_rng(13)
    shape = (12, 10, 40)
    n = int(numpy.prod(shape))
    x = numpy.concatenate([10.0 ** rng.uniform(-6, 2, n // 2), rng.uniform(0, 2, n), [0.0, 1e-300, 1e-17, 1.0, 1e300]])[-n:]
    if _use_max(kind):
        img = x * numpy.where(numpy.arange(n) % 2 == 0, 1.0, -1.0)
    else:
        img = numpy.cumsum(x * numpy.where(numpy.arange(n) % 2 == 0, 1.0, -1.0))
    img = img.reshape(shape)
    _run_case(emu, kind, img, sigma, paths=["lazy", "per_term", "cuda"])


@pytest.mark.parametrize("dtype", [numpy.float64, numpy.float32, numpy.uint8, numpy.int16, numpy.int32, numpy.float16])
@pytest.mark.parametrize("kind", ["difference_power", "maximum_power"])
def test_power_dtypes_and_wrap(emu, kind, dtype):
    """int16 -32768 under maximum_power: numpy.abs wraps it, so x + 1 < 0 where two such cells meet (pow of a negative
    base with a fractional sigma: NaN on both sides)."""
    rng = numpy.random.default_rng(17)
    shape = (8, 10, 36)
    img = (rng.normal(0.0, 40.0, shape)).astype(dtype) if dtype != numpy.uint8 else rng.integers(0, 256, shape).astype(dtype)
    if dtype == numpy.int16:
        img[2, 3, 4:9] = -32768
        img[3, 3, 4] = -32768
    _run_case(emu, kind, img, 0.5)


# ------------------------------------------------------------------------------------------------------
# the division term
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["difference_division", "maximum_division"])
@pytest.mark.parametrize("sigma", [0.0, -2.0, -0.3, 1e-300, 3.0, 1e300, math.inf, math.nan])
def test_division_domain(emu, kind, sigma):
    """sigma = 0, sigma < 0 with x / sigma = -1 (weight inf) and < -1 (negative -> DBL_MIN), huge x."""
    rng = numpy.random.default_rng(19)
    shape = (12, 10, 40)
    img = rng.integers(-6, 7, shape).astype(numpy.float64)        # x = 2 = -sigma for sigma = -2
    img[6:] *= 1e300
    img[9:] = rng.normal(0.0, 1.0, img[9:].shape)
    _run_case(emu, kind, img, sigma)


@pytest.mark.parametrize("dtype", [numpy.float32, numpy.uint8, numpy.int16, numpy.int32, numpy.bool_, numpy.uint16,
                                   numpy.int64, numpy.float16])
def test_division_dtypes(emu, dtype):
    rng = numpy.random.default_rng(23)
    shape = (8, 9, 40)
    if dtype == numpy.bool_:
        img = rng.random(shape) < 0.5
    else:
        info = numpy.iinfo(dtype) if numpy.issubdtype(dtype, numpy.integer) else numpy.finfo(dtype)
        img = rng.uniform(max(float(info.min), -60000.0), min(float(info.max), 60000.0), shape).astype(dtype)
    for kind in ("difference_division", "maximum_division"):
        _run_case(emu, kind, img, -17.0)
        _run_case(emu, kind, img, 250.0)


# ------------------------------------------------------------------------------------------------------
# the linear terms and their normaliser
# ------------------------------------------------------------------------------------------------------
LINEAR_SHAPES = [(16, 24, 96), (20000,), (150, 140), (7, 6, 9, 40)]


@pytest.mark.parametrize("kind", ["difference_linear", "maximum_linear"])
@pytest.mark.parametrize("dtype", [numpy.float32, numpy.float64])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("shape", LINEAR_SHAPES)
def test_linear_nan_anywhere_makes_every_weight_nan(emu, kind, dtype, where, shape):
    """numpy's max / min propagate NaN: M is NaN and so is every weight of the term, wherever the NaN cell is (the
    normaliser is reduced over many blocks of the lattice here)."""
    rng = numpy.random.default_rng(29)
    img = rng.normal(0.0, 50.0, shape).astype(dtype)
    n = img.size
    img.reshape(-1)[{"first": 0, "middle": n // 2 + 77, "last": n - 1}[where]] = numpy.nan
    _run_case(emu, kind, img, None, paths=_paths(len(shape)) if len(shape) != 3 else ["lazy", "per_term", "cuda"])


@pytest.mark.parametrize("kind", ["difference_linear", "maximum_linear"])
@pytest.mark.parametrize("dtype", [numpy.float64, numpy.float32, numpy.uint8, numpy.int16, numpy.int32, numpy.bool_,
                                   numpy.uint16, numpy.int64, numpy.float16])
def test_linear_domain(emu, kind, dtype):
    """x from 0 to M (weights from 1 to the DBL_MIN of x = M), a constant image (M = 0: NaN weights), +-inf cells (M =
    inf), the int16 / int32 extremes (M wraps in the input dtype: weights < 0, refused like the reference)."""
    rng = numpy.random.default_rng(31)
    shape = (16, 12, 40)
    if dtype == numpy.bool_:
        img = rng.random(shape) < 0.5
    elif numpy.issubdtype(dtype, numpy.integer):
        info = numpy.iinfo(dtype)
        img = rng.integers(max(info.min, -1000), min(info.max, 1000), shape, endpoint=True).astype(dtype)
    else:
        img = rng.normal(0.0, 100.0, shape).astype(dtype)
    _run_case(emu, kind, img, None)
    _run_case(emu, kind, numpy.full(shape, 3, dtype=dtype), None)               # M = 0
    if numpy.issubdtype(dtype, numpy.floating):
        for vals in ((numpy.inf,), (-numpy.inf,), (numpy.inf, -numpy.inf)):
            sp = img.copy()
            sp.reshape(-1)[100:100 + 13 * len(vals):13] = vals
            _run_case(emu, kind, sp, None)
        sp = img.copy()
        sp.reshape(-1)[::97] = numpy.finfo(dtype).smallest_subnormal
        _run_case(emu, kind, sp, None)
    if dtype in (numpy.int16, numpy.int32):
        info = numpy.iinfo(dtype)
        ext = img.copy()
        ext[0, 0, 0], ext[-1, -1, -1] = info.max, info.min
        _run_case(emu, kind, ext, None)


@pytest.mark.parametrize("kind", ["difference_linear", "maximum_linear"])
def test_linear_nan_and_infinities_together(emu, kind):
    img = numpy.random.default_rng(37).normal(0.0, 10.0, (10, 12, 40))
    img[1, 2, 3], img[4, 5, 6], img[7, 8, 9] = numpy.inf, -numpy.inf, numpy.nan
    _run_case(emu, kind, img, None)


# ------------------------------------------------------------------------------------------------------
# spacing
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_spacing(emu, kind):
    """Each weight with a spacing is RN(the weight without it / spacing[axis]), on every path; spacings that underflow
    a weight to 0, and a negative spacing, are refused exactly where the reference refuses."""
    rng = numpy.random.default_rng(41)
    shape = (12, 10, 40)
    img = _exp_image(kind, numpy.float64, shape, 2.0, rng) if _fn(kind) == "exponential" else rng.normal(0, 30, shape)
    sigma = 2.0 if _fn(kind) != "power" else 0.7
    sample = _sample(shape, rng)
    plain = _read(_build(kind, img, sigma).get_edge, sample)
    for sp in ((1.5, 0.75, 3.0), (1e-300, 7.0, 1e300)):
        refused, _ = _run_case(emu, kind, img, sigma, spacing=sp, seed=0)
        if refused:
            continue
        for path in PATHS_3D:
            got = _read(_build(kind, img, sigma, sp, path).get_edge, sample)
            for d, ((f0, _), (f1, _)) in enumerate(zip(plain, got)):
                with numpy.errstate(all="ignore"):
                    want = f0 / sp[d]
                assert numpy.array_equal(f1, want, equal_nan=True), (kind, sp, path, d)
    for sp in ((1.0, 1.0, math.inf), (1.0, -1.0, 1.0), (1e308, 1e308, 1e308)):
        _run_case(emu, kind, img, sigma, spacing=sp, paths=["lazy", "per_term"])


# ------------------------------------------------------------------------------------------------------
# batches
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("image_shape", [(6, 10, 24), (30, 40), (500,)])
def test_batch_each_image_against_its_own_constants(emu, kind, image_shape):
    """graph_from_voxels_batch with a different sigma (and, for the linear terms, M) per image: image b's pairs at
    flat ids b * N + p against the reference of image b alone.  Linear terms: NaN in the first voxel of image 1 and in
    an interior voxel of image 2 make those images' weights NaN and no other's."""
    import medpy_b200.graphcut as gc
    B = 4
    rng = numpy.random.default_rng(43)
    sigmas = [0.9, 2.5, 7.0, 31.0] if _fn(kind) != "power" else [0.5, 2.0, -0.5, 40.0]
    imgs = []
    for b in range(B):
        if _fn(kind) == "exponential":
            imgs.append(_exp_image(kind, numpy.float32, image_shape, sigmas[b], rng))
        else:
            imgs.append((rng.normal(0.0, 5.0 * (b + 1), image_shape)).astype(numpy.float32))
    image = numpy.stack(imgs)
    if _fn(kind) == "linear":
        image[1].reshape(-1)[0] = numpy.nan
        image[2].reshape(-1)[image[2].size // 2 + 3] = numpy.nan
    z = numpy.zeros(image.shape, bool)
    n = int(numpy.prod(image_shape))
    for src in ("host", "cuda"):
        arr = image
        if src == "cuda":
            import torch
            arr = torch.from_numpy(image).cuda()
        g = gc.graph_from_voxels_batch(z, z, arr, kind, sigma=sigmas)
        for b in range(B):
            sample = _sample(image_shape, numpy.random.default_rng(b), count=120)
            got = _read(g._native.get_edge, sample, offset=b * n)
            _check(emu, kind, image[b], sigmas[b], got, sample)
            if _fn(kind) == "linear":
                assert all(numpy.isnan(f).all() == (b in (1, 2)) for f, _ in got), (kind, b)
