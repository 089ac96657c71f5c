"""Warm re-solves on the handles the lazy fused build does not make, opted in with GraphDouble.enable_warm() before the first
solve (MGC_OPT_WARM): 4-D lattices, 3-D graphs from the eager fused build (MEDPY_GC_LAZY_CAPS=0) and the four-pass build
(MEDPY_GC_FUSE=0), 3-D graphs built term by term or with a boundary from add_nweights_dense, and 1-D / 2-D graphs filled
element-wise.  After every step the mask must equal the oracle BK's on the from-scratch graph with all calls replayed, and
the energy must be within the bounds of test_gpu_warm_tweights.py: 1e-9 S of the oracle, 1e-12 S + 1e-10 of a cold GPU
rebuild that stages the same calls."""
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_erase_seeds import _vol_1d  # noqa: E402
from test_gpu_seeds import _ball, _env, _graph, _ids, _stroke, _volume  # noqa: E402
from test_gpu_warm_tweights import _apply, _box, _oracle, _regional_delta, _sequences  # noqa: E402

pytestmark = pytest.mark.gpu

_KIND = "difference_exponential"


def _terms(vol):
    """The oracle's problem of graph_from_voxels(regional + difference_exponential + markers) on `vol`."""
    from oracle import energy_terms as et
    return et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=(_KIND, vol["image"], vol["sigma"], False))


def _make(handle, vol):
    """A fresh, built, unsolved graph of the regional + boundary + marker energy of `vol` on the handle kind `handle`."""
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut.maxflow import GraphDouble
    shape = vol["fg"].shape
    n = int(numpy.prod(shape))
    if handle in ("4d", "eager", "fuse0"):
        return _graph(vol, _KIND, True, False)
    if handle == "per_term":
        g = GraphDouble(n, 0, shape=shape)
        g.add_regional_probability(vol["prob"], vol["alpha"], True)
        g.add_boundary(1, vol["image"], vol["sigma"], None, float("nan"))
        g.add_markers(vol["fg"], vol["bg"])
        return g
    prob = _terms(vol)
    src, snk = prob["src"], prob["snk"]
    if handle == "nweights":
        # graph_from_voxels with a boundary term of the user's own: the weights handed over as dense n-link arrays
        from oracle import energy_terms as et

        def boundary(graph, args):
            for d, w in enumerate(et.boundary_weights(_KIND, *args)):
                graph.set_nweights_dense(d, w, w)
        return gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                                    regional_term_args=(vol["prob"], vol["alpha"]), boundary_term=boundary,
                                    boundary_term_args=(vol["image"], vol["sigma"], False))
    # element-wise: the reference's call sequence node by node (regional pass, n-links, fg markers, bg markers)
    g = GraphDouble(n, 2 * n) if handle == "1d" else GraphDouble(n, 2 * n, shape=shape)
    for v in range(n):
        g.add_tweights(v, float(src[v]), float(snk[v]))
    strides = numpy.cumprod((1,) + shape[::-1])[:-1][::-1]
    for d in range(len(shape)):
        c = numpy.unravel_index(numpy.arange(n), shape)[d]
        for v in numpy.flatnonzero(c + 1 < shape[d]).tolist():
            w = float(prob["wf"][d][v])
            g.sum_edge(v, v + int(strides[d]), w, w)
    for v in numpy.flatnonzero(prob["fg"]).tolist():
        g.add_tweights(v, 65535.0, 0.0)
    for v in numpy.flatnonzero(prob["bg"]).tolist():
        g.add_tweights(v, 0.0, 65535.0)
    return g


_ENV = {"eager": dict(MEDPY_GC_LAZY_CAPS=0), "fuse0": dict(MEDPY_GC_FUSE=0)}


def _cold(handle, vol, steps):
    g = _make(handle, vol)
    for step in steps:
        _apply(g, step)
    return g.maxflow(), g.get_mask()


def _check(handle, vol, steps, env=None):
    env = dict(_ENV.get(handle, {}), **(env or {}))
    with _env(**env):
        g = _make(handle, vol)
        g.enable_warm()
        g.maxflow()
        done = []
        for step in steps:
            _apply(g, step)
            done.append(step)
            e = g.maxflow()
            m = g.get_mask()
            oe, om, scale = _oracle(vol, _KIND, True, False, done)
            bound = max(abs(oe), scale)
            assert numpy.array_equal(m, om), ("warm mask differs from the oracle", handle, len(done), int((m != om).sum()))
            assert abs(e - oe) <= 1e-9 * bound, (handle, len(done), e, oe, bound)
            ce, cm = _cold(handle, vol, done)
            assert numpy.array_equal(m, cm), ("warm mask differs from the cold rebuild", handle, len(done))
            assert abs(e - ce) <= 1e-12 * bound + 1e-10, (handle, len(done), e, ce, bound)
        st = g.stats()
        assert st["seed_folds"] == sum(len(s) for s in steps) and st["ms_seeds"] > 0
        return g


def _seq(shape, vol, which):
    """The warm t-link sequences plus a seed stroke and an erase of markers, as (ids or None, src, snk) calls."""
    if which == "add_stroke":
        return [[(_ids(_stroke(shape)), 65535.0, 0.0)]]
    if which == "erase_markers":
        fgm, bgm = _ids(vol["fg"]), _ids(vol["bg"])
        return [[(fgm[::2], -65535.0, 0.0), (bgm[1::3], 0.0, -65535.0)]]
    if which == "successive":
        carve = _ids(_ball(shape, 0.3, 0.05)) if len(shape) > 1 else _ids(vol["fg"])[:5]
        return (_seq(shape, vol, "add_stroke") + [[(carve, 0.0, 65535.0)]] + _seq(shape, vol, "erase_markers")
                + _sequences(shape, vol, "steps"))
    return _sequences(shape, vol, which)


_WHICH = ["add_stroke", "erase_markers", "soft_fg", "negative", "mixed", "regional_box", "successive"]

_HANDLES = [("4d", (6, 8, 8, 3)), ("4d", (9, 5, 17, 3)), ("4d", (12, 12, 16, 6)), ("eager", (24, 20, 32)),
            ("fuse0", (24, 20, 32)), ("per_term", (19, 27, 13)), ("nweights", (16, 16, 16)), ("2d", (20, 24)),
            ("1d", (300,))]


def _vol(shape, seed=3):
    return _vol_1d() if len(shape) == 1 else _volume(shape, seed=seed, dtype="float32")


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("handle,shape", _HANDLES, ids=["%s-%s" % (h, "x".join(map(str, s))) for h, s in _HANDLES])
def test_warm_matches_from_scratch(handle, shape, which):
    vol = _vol(shape)
    _check(handle, vol, _seq(shape, vol, which))


@pytest.mark.parametrize("handle,shape", _HANDLES, ids=["%s-%s" % (h, "x".join(map(str, s))) for h, s in _HANDLES])
def test_first_solve_is_unchanged(handle, shape):
    """The opt-in only records state: the first solve gives the same energy bit for bit and the same mask."""
    vol = _vol(shape, seed=5)
    out = []
    with _env(**_ENV.get(handle, {})):
        for warm in (False, True):
            g = _make(handle, vol)
            if warm:
                g.enable_warm()
            out.append((g.maxflow().hex(), g.get_mask().copy()))
    assert out[0][0] == out[1][0] and numpy.array_equal(out[0][1], out[1][1])


def test_lazily_built_graph_is_unchanged():
    """On a graph of the lazy fused build the option changes nothing: energies, masks and materialised tiles through a
    fold sequence."""
    shape = (33, 17, 40)
    vol = _volume(shape, seed=7, dtype="float32")
    steps = _seq(shape, vol, "successive")
    runs = []
    for warm in (False, True):
        g = _graph(vol, _KIND, True, False)
        if warm:
            g.enable_warm()
        trace = [(g.maxflow().hex(), g.get_mask().copy(), g.stats()["tiles_materialised"])]
        for step in steps:
            _apply(g, step)
            trace.append((g.maxflow().hex(), g.get_mask().copy(), g.stats()["tiles_materialised"]))
        runs.append(trace)
    for a, b in zip(*runs):
        assert a[0] == b[0] and numpy.array_equal(a[1], b[1]) and a[2] == b[2]


def test_native_fold_before_the_first_solve():
    """A C-ABI fold on an opted-in handle that was never solved initialises and records the state first."""
    for handle, shape in (("4d", (9, 5, 17, 3)), ("eager", (24, 20, 32)), ("per_term", (19, 27, 13))):
        vol = _vol(shape, seed=8)
        steps = _seq(shape, vol, "negative") + _seq(shape, vol, "add_stroke")
        with _env(**_ENV.get(handle, {})):
            g = _make(handle, vol)
            g.enable_warm()
            g._flush()
            for step in steps:
                for ids, src, snk in step:
                    m = int(numpy.prod(shape)) if ids is None else len(ids)
                    src = numpy.ascontiguousarray(numpy.broadcast_to(numpy.ravel(numpy.asarray(src, numpy.float64)), (m,)))
                    snk = numpy.ascontiguousarray(numpy.broadcast_to(numpy.ravel(numpy.asarray(snk, numpy.float64)), (m,)))
                    g._nat().add_tweights_warm(None if ids is None else numpy.asarray(ids, numpy.int64), src, snk)
            e, m = g.maxflow(), g.get_mask()
        oe, om, scale = _oracle(vol, _KIND, True, False, steps)
        assert numpy.array_equal(m, om), (handle, int((m != om).sum()))
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (handle, e, oe)


def test_enable_after_the_first_solve_raises():
    vol = _volume((6, 8, 8, 3), seed=1, dtype="float32")
    g = _graph(vol, _KIND, True, False)
    g.maxflow()
    with pytest.raises(RuntimeError, match=r"before the first maxflow\(\)"):
        g.enable_warm()
    with pytest.raises(RuntimeError, match="reset"):
        g.add_seeds(_ids(_stroke((6, 8, 8, 3))), None)


def test_option_survives_reset_and_rebuild():
    from medpy_b200.graphcut.maxflow import GraphDouble
    shape = (9, 5, 17, 3)
    vol = _volume(shape, seed=2, dtype="float32")
    g = GraphDouble(int(numpy.prod(shape)), 0, shape=shape)
    g.enable_warm()
    stroke = _ids(_stroke(shape))
    for _ in range(2):
        g.reset()
        g.add_regional_probability(vol["prob"], vol["alpha"], True)
        g.add_boundary(1, vol["image"], vol["sigma"], None, float("nan"))
        g.add_markers(vol["fg"], vol["bg"])
        g.maxflow()
        g.add_seeds(stroke, None)
        e, m = g.maxflow(), g.get_mask()
        oe, om, scale = _oracle(vol, _KIND, True, False, [[(stroke, 65535.0, 0.0)]])
        assert numpy.array_equal(m, om) and abs(e - oe) <= 1e-9 * max(abs(oe), scale)


def test_bad_ids_and_nan_leave_the_4d_result():
    shape = (9, 5, 17, 3)
    n = int(numpy.prod(shape))
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, _KIND, True, False)
    g.enable_warm()
    g.maxflow()
    ball = _ids(_ball(shape, 0.3, 0.1))
    g.add_tweights_warm(ball, 0.0, 30.0)
    e = g.maxflow()
    m = g.get_mask().copy()
    nat = g._nat()
    with pytest.raises(ValueError, match="out of range"):
        nat.add_tweights_warm(numpy.array([5, n], numpy.int64), numpy.ones(2), numpy.zeros(2))
    with pytest.raises(ValueError, match="NaN or infinite"):
        nat.add_tweights_warm(numpy.array([5, 6], numpy.int64), numpy.ones(2), numpy.array([0.0, numpy.nan]))
    dense = numpy.ones(n)
    dense[7] = numpy.inf
    with pytest.raises(ValueError, match="NaN or infinite"):
        nat.add_tweights_warm(None, dense, numpy.zeros(n))
    with pytest.raises(ValueError, match="out of range"):
        nat.add_seeds(numpy.array([0, -1], numpy.int64), None)
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 1
    # the solved result above is cached; a valid fold after the refused calls proves the state itself was left alone
    stroke = _ids(_stroke(shape))
    g.add_tweights_warm(stroke, 50.0, 0.0)
    e2, m2 = g.maxflow(), g.get_mask()
    oe, om, scale = _oracle(vol, _KIND, True, False, [[(ball, 0.0, 30.0)], [(stroke, 50.0, 0.0)]])
    assert numpy.array_equal(m2, om), int((m2 != om).sum())
    assert abs(e2 - oe) <= 1e-9 * max(abs(oe), scale), (e2, oe)


@pytest.mark.parametrize("env", [dict(MEDPY_GC_SWEEP=0), dict(MEDPY_GC_FIRST_CAP=0),
                                 dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_DEBUG=1)],
                         ids=["sweep0", "first_cap0", "partial_reset0", "debug"])
@pytest.mark.parametrize("handle,shape", [("4d", (12, 12, 16, 6)), ("eager", (32, 32, 32))])
def test_solver_options(handle, shape, env):
    """MEDPY_GC_DEBUG=1 checks the invariants and flow conservation around every solve after every fold."""
    vol = _volume(shape, seed=5, dtype="float32")
    _check(handle, vol, _seq(shape, vol, "successive"), env=env)


def test_config4_full_size_against_reference_bk():
    """BASELINE config 4 (256x256x128x4, maximum_exponential): three warm steps -- a fg line, a bg ball inside blob 1, every
    other fg marker erased -- each energy within 1e-9 S of the real reference BK's on the from-scratch graph, and each mask
    equal to BK's up to ties.  Config 4's maximum term has structural ties (test_gpu_fullsize.py), and inside the bright
    blobs its weights are tiny (inside the ball: median 1e-18, minimum 5e-35), far below the resolution of a t-link of
    65535 (ulp 7.3e-12).  Each add_tweights call rounds a voxel's residual t-link once at that scale, in BK and in the fold
    alike, and 7022 of the ball's 8084 voxels carry a fg marker, so their t-links become the rounding residue of 65535 -
    65535 + r.  Where the masks differ, the two cut capacities, summed exactly over the graph's float64 weights, must
    therefore agree to that resolution: half an ulp of 65535 per call replayed so far."""
    import medpy_b200.graphcut as gc
    from oracle import energy_terms as et, solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")
    from test_gpu_fullsize import _cut_difference_exact
    from test_gpu_warm_tweights import _replay
    shape = (256, 256, 128, 4)
    vol = _volume(shape, seed=0, dtype="float32")
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_maximum_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    g.enable_warm()
    g.maxflow()
    fgm = _ids(vol["fg"])
    steps = [[(_ids(_stroke(shape)), 65535.0, 0.0)], [(_ids(_ball(shape, 0.3, 0.05)), 0.0, 65535.0)],
             [(fgm[::2], -65535.0, 0.0)]]
    for k, step in enumerate(steps, 1):
        _apply(g, step)
        e = g.maxflow()
        m = g.get_mask()
        prob = et.build_problem(vol["fg"], vol["bg"], boundary=("maximum_exponential", vol["image"], vol["sigma"], False))
        scale = _replay(prob, steps[:k])
        ref = dict(prob, src=numpy.maximum(prob["tr"], 0.0), snk=numpy.maximum(-prob["tr"], 0.0),
                   fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool))
        oe, om, _ = solvers.solve_ref(ref)
        oe += prob["flow_const"]
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (k, e, oe, scale)
        if int((m != om).sum()):
            diff = _cut_difference_exact(prob, m, om)
            calls = sum(len(ids) for st in steps[:k] for ids, _, _ in st)
            assert abs(diff) <= 0.5 * numpy.spacing(65535.0) * calls, (k, int((m != om).sum()), diff, calls)
