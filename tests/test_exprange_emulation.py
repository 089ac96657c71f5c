"""The lazy graph build's range test without a GPU: medpy_b200/csrc/gc_exprange.cuh is compiled as host C++
(tests/emu/exprange_emu.cpp).  A staged image block that passes block_exp_ordinary skips the per-pair test of the
exponential term, so a block that passes must hold no pair of cells whose argument x^2 / sigma^2 is above 700 or NaN --
on random blocks and on blocks built to sit on the threshold, with infinities, NaN, outliers, denormals and negative
values under maximum_exponential, in float32 and float64."""
import ctypes
import os
import subprocess

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libexprange_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-o", so,
                           os.path.join(HERE, "emu", "exprange_emu.cpp")])
    lib = ctypes.CDLL(so)
    for name, ct in (("f32", ctypes.c_float), ("f64", ctypes.c_double)):
        f = getattr(lib, "emu_block_ok_" + name)
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(ct), ctypes.c_longlong, ctypes.c_int, ctypes.c_double]
        f = getattr(lib, "emu_pairs_ok_" + name)
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(ct), ctypes.c_longlong, ctypes.c_int, ctypes.c_double, ctypes.c_double]
    return lib


def _check(lib, cells, use_max, sigma):
    """Both tests on one block; returns whether the block passed.  sigma2 = pow(sigma, 2) and its reciprocal as the
    build receives them (gc_api.cu)."""
    cells = numpy.ascontiguousarray(cells)
    name, ct = ("f32", ctypes.c_float) if cells.dtype == numpy.float32 else ("f64", ctypes.c_double)
    sigma2 = float(sigma) ** 2
    inv = 1.0 / sigma2 if sigma2 != 0.0 else 0.0
    ptr = cells.ctypes.data_as(ctypes.POINTER(ct))
    block = getattr(lib, "emu_block_ok_" + name)(ptr, cells.size, int(use_max), inv)
    pairs = getattr(lib, "emu_pairs_ok_" + name)(ptr, cells.size, int(use_max), inv, sigma2)
    assert not (block and not pairs), (cells, use_max, sigma)
    return bool(block)


@pytest.mark.parametrize("dtype", [numpy.float32, numpy.float64])
@pytest.mark.parametrize("use_max", [0, 1])
def test_random_blocks(emu, dtype, use_max):
    rng = numpy.random.default_rng(7 + use_max)
    passed = 0
    for k in range(300):
        n = int(rng.integers(1, 160))
        scale = 10.0 ** rng.uniform(-3, 4)
        cells = (rng.normal(0.0, scale, size=n) + rng.uniform(-2, 2) * scale).astype(dtype)
        if use_max == 0 and rng.random() < 0.3:
            cells[rng.integers(0, n)] += dtype(100.0 * scale)          # an edge or an outlier
        passed += _check(emu, cells, use_max, sigma=scale * rng.uniform(0.02, 2.0))
    assert 30 < passed < 290          # both outcomes are exercised


@pytest.mark.parametrize("dtype", [numpy.float32, numpy.float64])
def test_bench_like_block_passes(emu, dtype):
    """A 10 x 10 x 40 block of the two-blob volume (noise 10, contrast 100, zero fill) at its sigma of about 14.5."""
    rng = numpy.random.default_rng(0)
    cells = rng.normal(0.0, 10.0, size=4000).astype(dtype)
    cells[:1500] += dtype(100.0)
    cells[-40:] = 0
    assert _check(emu, cells, 0, sigma=14.5)
    assert _check(emu, cells, 1, sigma=14.5)


@pytest.mark.parametrize("dtype", [numpy.float32, numpy.float64])
@pytest.mark.parametrize("use_max", [0, 1])
def test_threshold_neighbourhood(emu, dtype, use_max):
    """Spans one ulp either side of the largest span that passes; the pair of the two ends decides."""
    for sigma in (1.0, 3.0, 14.5, 1e-3, 7.7e5):
        d0 = dtype(numpy.sqrt(700.0) * sigma)
        seen = set()
        up = numpy.nextafter(d0, dtype(numpy.inf))
        for d in (d0 * dtype(1 - 1e-6), numpy.nextafter(d0, dtype(0)), d0, up, numpy.nextafter(up, dtype(numpy.inf)),
                  d0 * dtype(1 + 1e-6)):
            for base in (dtype(0), dtype(-0.5) * d, dtype(3.0) * d):
                cells = numpy.array([base, base + d, base + d / dtype(2)], dtype=dtype) if use_max == 0 else \
                    numpy.array([-d, d / dtype(3), dtype(0)], dtype=dtype)
                seen.add(_check(emu, cells, use_max, sigma))
        assert seen == {True, False}, (sigma, dtype, use_max)


@pytest.mark.parametrize("dtype", [numpy.float32, numpy.float64])
@pytest.mark.parametrize("use_max", [0, 1])
def test_special_values_refuse(emu, dtype, use_max):
    base = numpy.array([1.0, 2.0, 3.0, -1.5], dtype=dtype)
    assert _check(emu, base, use_max, sigma=5.0)
    for special in (numpy.nan, numpy.inf, -numpy.inf):
        cells = base.copy()
        cells[2] = special
        assert not _check(emu, cells, use_max, sigma=5.0)
    assert not _check(emu, numpy.full(5, numpy.inf, dtype=dtype), use_max, sigma=5.0)
    assert not _check(emu, numpy.full(5, numpy.nan, dtype=dtype), use_max, sigma=5.0)
    # a single outlier
    cells = numpy.concatenate([base, numpy.array([1e4], dtype=dtype)])
    assert not _check(emu, cells, use_max, sigma=5.0)
    # the division form of the argument (sigma == 0, or a reciprocal that is not below 1e300) never passes
    assert not _check(emu, base, use_max, sigma=0.0)
    assert not _check(emu, numpy.zeros(3, dtype=dtype), use_max, sigma=1e-160)


@pytest.mark.parametrize("dtype", [numpy.float32, numpy.float64])
@pytest.mark.parametrize("use_max", [0, 1])
def test_denormals_and_signed_zeros(emu, dtype, use_max):
    tiny = numpy.finfo(dtype).smallest_subnormal
    cells = numpy.array([tiny, -tiny, dtype(0), -dtype(0), tiny * dtype(7)], dtype=dtype)
    assert _check(emu, cells, use_max, sigma=1e-140 if dtype == numpy.float64 else 1e-30)
    assert _check(emu, cells, use_max, sigma=1.0)


def test_maximum_term_with_negative_values(emu):
    """maximum_exponential reads |I|: a block of large negative values is as far from 0 as its positive mirror."""
    for dtype in (numpy.float32, numpy.float64):
        cells = numpy.array([-300.0, -250.0, -280.0], dtype=dtype)
        assert not _check(emu, cells, 1, sigma=10.0)
        assert _check(emu, cells, 0, sigma=10.0)
        assert _check(emu, -cells, 0, sigma=10.0)
        assert not _check(emu, -cells, 1, sigma=10.0)
