"""Logic check of the sparse push-relabel without a GPU: the C ABI's host state (medpy_b200/csrc/gc_sparse_host.hpp)
and the per-node functions of medpy_b200/csrc/gc_sparse.cuh are compiled as host C++ (tests/emu/sparse_emu.cpp) and
compared with the label-term oracle and the real reference BK (oracle/_ref) on random sparse graphs and on the golden
region adjacency graphs.  gc_sparse_api.cu runs the same host code, and the CUDA kernels wrap exactly these functions."""
import ctypes
import os
import subprocess
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import energy_label_terms as elt  # noqa: E402
from oracle import solvers  # noqa: E402


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libsparse_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", so,
                           os.path.join(HERE, "emu", "sparse_emu.cpp")])
    lib = ctypes.CDLL(so)
    ip, dp, ll = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double), ctypes.c_longlong
    lib.emu_sparse_calls.restype = ll
    lib.emu_sparse_calls.argtypes = ([ctypes.c_int, ll, ip, ip, dp, dp, ll, ip, dp, dp, ctypes.c_int, ctypes.c_int, ip, ip]
                                     + [dp] * 4 + [ctypes.POINTER(ctypes.c_uint8), dp])
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.POINTER({numpy.int32: ctypes.c_int, numpy.uint8: ctypes.c_uint8}.get(a.dtype.type, ctypes.c_double)))


def run_emu(lib, n, i, j, cap, rev, tw_ops, steps=4, sweeps=16):
    """The raw calls through the C ABI's host state, whose merged pairs, tr and constant must equal the oracle's, and
    the solve of the CSR it lays out."""
    calls = [numpy.ascontiguousarray(a, dtype=t) for a, t in zip((i, j, cap, rev), (numpy.int32, numpy.int32, float, float))]
    tws = [numpy.ascontiguousarray(numpy.concatenate([numpy.asarray(op[k]) for op in tw_ops]), dtype=t)
           for k, t in enumerate((numpy.int32, float, float))]
    m = calls[0].size
    lo, hi, mask = numpy.zeros(m, numpy.int32), numpy.zeros(m, numpy.int32), numpy.zeros(n, numpy.uint8)
    c_lh, c_hl, tr, const, energy = (numpy.zeros(s) for s in (m, m, n, 1, 1))
    np_ = lib.emu_sparse_calls(n, m, *map(_p, calls), tws[0].size, *map(_p, tws), steps, sweeps,
                               *map(_p, (lo, hi, c_lh, c_hl, tr, const, mask, energy)))
    assert np_ >= 0
    order = numpy.lexsort((hi[:np_], lo[:np_]))                  # insertion order -> the oracle's (lo, hi) order
    for got, want in zip((lo, hi, c_lh, c_hl), elt.merge_edges(i, j, cap, rev)):
        assert numpy.array_equal(got[:np_][order], want)
    want_tr, want_const = elt.add_tweights_replay(n, tw_ops)
    assert numpy.array_equal(tr, want_tr) and const[0] == want_const
    return energy[0], mask


def random_graph(rng, n, m, integer):
    i = rng.integers(0, n, size=m)
    j = rng.integers(0, n, size=m)
    keep = i != j
    i, j = i[keep], j[keep]
    if integer:
        cap = rng.integers(1, 20, size=i.size).astype(float)
        rev = rng.integers(1, 20, size=i.size).astype(float)
        src = rng.integers(0, 30, size=n).astype(float)
        snk = rng.integers(0, 30, size=n).astype(float)
    else:
        cap = rng.uniform(1e-3, 2.0, size=i.size)
        rev = rng.uniform(1e-3, 2.0, size=i.size)
        src = rng.uniform(0, 3.0, size=n)
        snk = rng.uniform(0, 3.0, size=n)
    tw = [(numpy.arange(n), src, snk)]
    fg = rng.choice(n, size=max(1, n // 20), replace=False)
    bg = rng.choice(n, size=max(1, n // 20), replace=False)
    tw.append((fg, numpy.full(fg.size, 65535.0), numpy.zeros(fg.size)))
    tw.append((bg, numpy.zeros(bg.size), numpy.full(bg.size, 65535.0)))
    return i, j, cap, rev, tw


@pytest.mark.parametrize("seed", range(12))
def test_random_sparse_graphs_match_reference_bk(emu, seed):
    rng = numpy.random.default_rng(seed)
    n = int(rng.integers(2, 400))
    m = int(rng.integers(1, 6 * n))
    integer = seed % 2 == 0
    i, j, cap, rev, tw = random_graph(rng, n, m, integer)
    flow, mask, _ = solvers.solve_sparse(n, i, j, cap, rev, tw)
    e, got = run_emu(emu, n, i, j, cap, rev, tw, steps=1 + seed % 4, sweeps=1 + 5 * (seed % 3))
    assert numpy.array_equal(got, mask)
    if integer:
        assert e == flow
    else:
        assert e == pytest.approx(flow, rel=1e-9)


def test_isolated_and_terminal_only_nodes(emu):
    # node 0: source only, node 1: sink only, node 2: nothing, nodes 3-4 joined, 4 to the sink
    n = 5
    i, j = numpy.asarray([3]), numpy.asarray([4])
    cap, rev = numpy.asarray([2.0]), numpy.asarray([0.5])
    tw = [(numpy.asarray([0, 1, 3, 4]), numpy.asarray([5.0, 0.0, 7.0, 0.0]), numpy.asarray([0.0, 4.0, 0.0, 9.0]))]
    flow, mask, _ = solvers.solve_sparse(n, i, j, cap, rev, tw)
    e, got = run_emu(emu, n, i, j, cap, rev, tw)
    assert numpy.array_equal(got, mask) and e == flow == 2.0
    assert got.tolist() == [1, 0, 1, 1, 0]


def test_golden_region_graphs(emu):
    from test_oracle_labels import FULL, G, label_problem
    for nm in FULL:
        for tag in ("cut_stawiaski", "cut_means", "cut_directed_atlas"):
            n, i, j, cap, rev, tw = label_problem(nm, tag)
            e, got = run_emu(emu, n, i, j, cap, rev, tw)
            assert numpy.array_equal(got, G[nm + "/" + tag + "_mask"]), (nm, tag)
            assert e == pytest.approx(float(G[nm + "/" + tag + "_flow"]), rel=1e-9, abs=1e-300), (nm, tag)


def test_pairwise_sum_equals_numpy_sum(tmp_path):
    """csrc/gc_pairwise.cuh (what the regional_atlas reduction runs per region) against numpy.sum, bit for bit."""
    so = str(tmp_path / "libpairwise_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-o", so,
                           os.path.join(HERE, "emu", "pairwise_emu.cpp")])
    lib = ctypes.CDLL(so)
    lib.emu_pairwise_f32.restype = ctypes.c_float
    lib.emu_pairwise_f32.argtypes = [ctypes.c_void_p, ctypes.c_longlong]
    lib.emu_pairwise_f64.restype = ctypes.c_double
    lib.emu_pairwise_f64.argtypes = [ctypes.c_void_p, ctypes.c_longlong]
    rng = numpy.random.default_rng(7)
    for n in list(range(1, 300)) + [1000, 1001, 4097, 65536, 100003]:
        a32 = rng.uniform(0, 1, n).astype(numpy.float32)
        a64 = rng.normal(0, 100, n)
        assert numpy.float32(lib.emu_pairwise_f32(a32.ctypes.data, n)) == numpy.sum(a32), n
        assert lib.emu_pairwise_f64(a64.ctypes.data, n) == numpy.sum(a64), n


from hypothesis import given, settings, strategies as st  # noqa: E402

_graphs = st.integers(2, 14).flatmap(lambda n: st.tuples(
    st.just(n),
    st.lists(st.tuples(st.integers(0, n - 1), st.integers(0, n - 1), st.integers(0, 6), st.integers(0, 6)), min_size=0, max_size=50),
    st.lists(st.tuples(st.integers(0, n - 1), st.integers(-3, 8), st.integers(-3, 8)), min_size=1, max_size=24),
    st.integers(1, 4), st.integers(1, 9)))


@settings(max_examples=300, deadline=None)
@given(_graphs)
def test_small_integer_graphs_with_ties_match_bk_exactly(emu, g):
    """Small integer capacities make ties (several minimum cuts, saturated and zero arcs, negative t-weights, repeated
    add_tweights on one node) the rule: the product's algorithm must still return BK's flow and BK's sink set."""
    n, edges, tws, steps, sweeps = g
    edges = [e for e in edges if e[0] != e[1]]
    i = numpy.asarray([e[0] for e in edges], dtype=numpy.int64)
    j = numpy.asarray([e[1] for e in edges], dtype=numpy.int64)
    cap = numpy.asarray([e[2] for e in edges], dtype=float)
    rev = numpy.asarray([e[3] for e in edges], dtype=float)
    tw = [(numpy.asarray([t[0]]), numpy.asarray([float(t[1])]), numpy.asarray([float(t[2])])) for t in tws]
    flow, mask, _ = solvers.solve_sparse(n, i, j, cap, rev, tw)
    if i.size == 0:
        i, j, cap, rev = numpy.asarray([0]), numpy.asarray([1]), numpy.asarray([0.0]), numpy.asarray([0.0])
    e, got = run_emu(emu, n, i, j, cap, rev, tw, steps=steps, sweeps=sweeps)
    assert e == flow
    assert numpy.array_equal(got, mask)
