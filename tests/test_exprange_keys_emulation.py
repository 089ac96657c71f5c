"""The lean lazy build's float32 range test without a GPU: k_build_lean reduces order-preserving integer keys of the
staged cells (gc_exprange.cuh: er_f32_key, block_exp_ordinary_keys) where k_build_tile folds the floats with a separate
NaN flag.  Both are compiled as host C++ (tests/emu/exprange_keys_emu.cpp) and must give the same verdict on every block:
random ones, blocks on the threshold (one ulp either side), signed zeros, infinities, NaN of either sign, denormals."""
import ctypes
import os
import subprocess

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libexprange_keys_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-o", so,
                           os.path.join(HERE, "emu", "exprange_keys_emu.cpp")])
    lib = ctypes.CDLL(so)
    for name in ("emu_fold_ok_f32", "emu_keys_ok_f32"):
        f = getattr(lib, name)
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_longlong, ctypes.c_int, ctypes.c_double]
    lib.emu_key_f32.restype = ctypes.c_int
    lib.emu_key_f32.argtypes = [ctypes.POINTER(ctypes.c_float)]
    return lib


def _verdicts(lib, cells, use_max, sigma):
    cells = numpy.ascontiguousarray(cells, dtype=numpy.float32)
    sigma2 = float(sigma) ** 2
    inv = 1.0 / sigma2 if sigma2 != 0.0 else 0.0
    ptr = cells.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    return lib.emu_fold_ok_f32(ptr, cells.size, int(use_max), inv), lib.emu_keys_ok_f32(ptr, cells.size, int(use_max), inv)


def _same(lib, cells, use_max, sigma):
    fold, keys = _verdicts(lib, cells, use_max, sigma)
    assert fold == keys, (cells, use_max, sigma, fold, keys)
    return bool(fold)


def _bits(u):
    return numpy.array([u], dtype=numpy.uint32).view(numpy.float32)[0]


SPECIALS = [0.0, -0.0, numpy.inf, -numpy.inf, _bits(0x7fc00000), _bits(0xffc00000), _bits(0x7f800001), _bits(0xff800001),
            _bits(0x7fffffff), _bits(0xffffffff), _bits(0x00000001), _bits(0x80000001), _bits(0x007fffff),
            _bits(0x807fffff), numpy.finfo(numpy.float32).max, -numpy.finfo(numpy.float32).max, 1.0, -1.0]


def test_keys_order_like_the_floats(emu):
    """Keys sort like the values (-0 just below +0); positive NaN above +inf, negative NaN below -inf."""
    rng = numpy.random.default_rng(3)
    vals = numpy.concatenate([rng.normal(0, 10.0 ** rng.uniform(-40, 38, 2000)).astype(numpy.float32),
                              numpy.array([v for v in SPECIALS if v == v], dtype=numpy.float32)])
    keys = numpy.array([emu.emu_key_f32(ctypes.byref(ctypes.c_float(float(v)))) for v in vals])
    order = numpy.argsort(keys, kind="stable")
    assert numpy.all(numpy.diff(vals[order].astype(numpy.float64)) >= 0)
    k_inf, k_ninf = (emu.emu_key_f32(ctypes.byref(ctypes.c_float(v))) for v in (numpy.inf, -numpy.inf))
    for u in (0x7f800001, 0x7fc00000, 0x7fffffff):
        assert emu.emu_key_f32(ctypes.byref(ctypes.c_float(_bits(u)))) > k_inf
    for u in (0xff800001, 0xffc00000, 0xffffffff):
        assert emu.emu_key_f32(ctypes.byref(ctypes.c_float(_bits(u)))) < k_ninf


@pytest.mark.parametrize("use_max", [0, 1])
def test_random_blocks_same_verdict(emu, use_max):
    rng = numpy.random.default_rng(11 + use_max)
    passed = 0
    for _ in range(600):
        n = int(rng.integers(1, 200))
        scale = 10.0 ** rng.uniform(-3, 4)
        cells = (rng.normal(0.0, scale, size=n) + rng.uniform(-2, 2) * scale).astype(numpy.float32)
        if rng.random() < 0.3:
            cells[rng.integers(0, n)] += numpy.float32(100.0 * scale)
        if rng.random() < 0.2:
            cells[rng.integers(0, n)] = SPECIALS[int(rng.integers(0, len(SPECIALS)))]
        passed += _same(emu, cells, use_max, sigma=scale * rng.uniform(0.02, 2.0))
    assert 50 < passed < 550


@pytest.mark.parametrize("use_max", [0, 1])
def test_threshold_neighbourhood_same_verdict(emu, use_max):
    for sigma in (1.0, 3.0, 14.5, 1e-3, 7.7e5):
        d0 = numpy.float32(numpy.sqrt(700.0) * sigma)
        up = numpy.nextafter(d0, numpy.float32(numpy.inf))
        seen = set()
        for d in (numpy.nextafter(d0, numpy.float32(0)), d0, up, numpy.nextafter(up, numpy.float32(numpy.inf))):
            for base in (numpy.float32(0), numpy.float32(-0.0), numpy.float32(-0.5) * d, numpy.float32(3.0) * d):
                cells = numpy.array([base, base + d, base + d / numpy.float32(2)], dtype=numpy.float32) if use_max == 0 \
                    else numpy.array([-d, d / numpy.float32(3), numpy.float32(-0.0)], dtype=numpy.float32)
                seen.add(_same(emu, cells, use_max, sigma))
        assert seen == {True, False}, (sigma, use_max)


@pytest.mark.parametrize("use_max", [0, 1])
def test_special_values_same_verdict(emu, use_max):
    base = numpy.array([1.0, 2.0, 3.0, -1.5], dtype=numpy.float32)
    for a in SPECIALS:
        for b in SPECIALS:
            cells = base.copy()
            cells[1], cells[3] = a, b
            for sigma in (5.0, 1e-30, 1e30):
                _same(emu, cells, use_max, sigma)
            _same(emu, numpy.array([a, b], dtype=numpy.float32), use_max, 5.0)
    # signed zeros and denormals only: both folds pass
    tiny = numpy.finfo(numpy.float32).smallest_subnormal
    cells = numpy.array([tiny, -tiny, 0.0, -0.0, tiny * 7], dtype=numpy.float32)
    assert _same(emu, cells, use_max, 1e-30) and _same(emu, cells, use_max, 1.0)
    assert _same(emu, numpy.array([-0.0, -0.0], dtype=numpy.float32), use_max, 1.0)
    for sigma in (0.0, 1e-160):           # the division form never passes
        assert not _same(emu, base, use_max, sigma)
