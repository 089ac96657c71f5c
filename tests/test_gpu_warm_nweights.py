"""sum_edge calls folded into a solved lattice graph and solved warm (GraphDouble.add_nweights_warm /
add_nweights_dense_warm, mgc_add_nweights_warm / mgc_add_nweights_dense_warm): after each step the mask must equal the
oracle BK's on the from-scratch graph with every call so far replayed, and the energy must be within 1e-9 S of it and
within 1e-12 S + 1e-10 of a cold GPU rebuild that stages the same calls (S as in test_gpu_warm_tweights.py, plus the sum of
the n-link increments).

A step is a list of operations:
  ("n", i, j, cap, rev)   add_nweights_warm: sum_edge(i[k], j[k], cap[k], rev[k]) in order;
  ("d", axis, fwd, bwd)   add_nweights_dense_warm;
  ("t", ids, src, snk)    add_tweights_warm;
  ("s", fg, bg)           add_seeds;   ("r", fg, bg) remove_seeds."""
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_erase_seeds import _problem, _vol_1d  # noqa: E402
from test_gpu_seeds import _ball, _env, _graph, _ids, _stroke, _volume  # noqa: E402
from test_gpu_warm_eager import _ENV, _make  # noqa: E402
from test_gpu_warm_tweights import _box, _regional_delta, _replay  # noqa: E402

pytestmark = pytest.mark.gpu

_KIND = "difference_exponential"


def _strides(shape):
    return tuple(int(numpy.prod(shape[d + 1:])) for d in range(len(shape)))


def _pairs_in(mask):
    """Every lattice-neighbour pair (lo, hi) with both ends in `mask`, axis by axis."""
    shape = mask.shape
    st = _strides(shape)
    flat = numpy.ascontiguousarray(mask).ravel()
    c = numpy.unravel_index(numpy.arange(flat.size), shape)
    lo, hi = [], []
    for d in range(len(shape)):
        p = numpy.flatnonzero(flat & (c[d] + 1 < shape[d]))
        p = p[flat[p + st[d]]]
        lo.append(p)
        hi.append(p + st[d])
    return numpy.concatenate(lo), numpy.concatenate(hi)


def _brush(shape, centre=0.3, radius=0.12, w=5.0):
    """A boundary brush: +w on both arcs of every pair inside a ball, half of the pairs named from their upper end, the
    first few pairs twice."""
    lo, hi = _pairs_in(_ball(shape, centre, radius) if len(shape) > 1 else numpy.arange(shape[0]) % 7 < 4)
    flip = numpy.arange(lo.size) % 2 == 1
    i, j = numpy.where(flip, hi, lo), numpy.where(flip, lo, hi)
    k = min(5, i.size)
    i, j = numpy.concatenate([i, j[:k]]), numpy.concatenate([j, i[:k]])
    cap = numpy.full(i.size, w)
    rev = numpy.full(i.size, w)
    rev[::3] = 0.0                                          # one-sided increments, and some zero ones
    return ("n", i, j, cap, rev)


def _dense_box(shape, axis=0, w=3.0):
    f = numpy.zeros(shape)
    f[_box(shape)] = w
    return ("d", axis, f, 0.5 * f)


def _lambda_step(prob, shape, kappa=0.25):
    """Raise the boundary weight: dense kappa * w on every axis."""
    return [("d", d, kappa * prob["wf"][d].reshape(shape), kappa * prob["wb"][d].reshape(shape)) for d in range(len(shape))]


def _replay_all(prob, steps):
    """Every operation of every step applied to the oracle's problem in order; returns S."""
    shape = prob["shape"]
    st = _strides(shape)
    prob["wf"] = [w.copy() for w in prob["wf"]]
    prob["wb"] = [w.copy() for w in prob["wb"]]           # the boundary terms share one array for both directions
    scale = abs(prob["flow_const"])
    for step in steps:
        for op in step:
            if op[0] in "tsr":
                if op[0] == "t":
                    calls = [(op[1], op[2], op[3])]
                else:
                    cap = 65535.0 if op[0] == "s" else -65535.0
                    calls = [(x, c, t) for x, c, t in ((op[1], cap, 0.0), (op[2], 0.0, cap)) if x is not None]
                before = abs(prob["flow_const"])
                scale += _replay(prob, [calls]) - before
                continue
            if op[0] == "d":
                _, d, f, b = op
                c = numpy.unravel_index(numpy.arange(prob["tr"].size), shape)[d]
                keep = c + 1 < shape[d]
                f, b = numpy.where(keep, numpy.ravel(f), 0.0), numpy.where(keep, numpy.ravel(b), 0.0)
                prob["wf"][d] += f
                prob["wb"][d] += b
                scale += float(f.sum() + b.sum())
                continue
            _, i, j, cap, rev = op
            i, j = numpy.asarray(i, numpy.int64), numpy.asarray(j, numpy.int64)
            cap = numpy.broadcast_to(numpy.asarray(cap, numpy.float64), i.shape)
            rev = numpy.broadcast_to(numpy.asarray(rev, numpy.float64), i.shape)
            lo, dist = numpy.minimum(i, j), numpy.abs(i - j)
            up = i < j
            for d in range(len(shape)):
                cl = numpy.unravel_index(lo, shape)[d]
                sel = (dist == st[d]) & (cl + 1 < shape[d])
                numpy.add.at(prob["wf"][d], lo[sel], numpy.where(up, cap, rev)[sel])
                numpy.add.at(prob["wb"][d], lo[sel], numpy.where(up, rev, cap)[sel])
            scale += float(cap.sum() + rev.sum())
    return scale


def _apply(g, step, conv=None):
    cv = (lambda a: a) if conv is None else (lambda a: conv(numpy.asarray(a)) if numpy.ndim(a) else a)
    for op in step:
        if op[0] == "n":
            g.add_nweights_warm(*(cv(x) for x in op[1:]))
        elif op[0] == "d":
            g.add_nweights_dense_warm(op[1], cv(op[2]), cv(op[3]))
        elif op[0] == "t":
            g.add_tweights_warm(None if op[1] is None else cv(numpy.asarray(op[1], numpy.int64)), cv(op[2]), cv(op[3]))
        else:
            (g.add_seeds if op[0] == "s" else g.remove_seeds)(op[1], op[2])


def _oracle(prob, steps):
    from oracle import solvers
    scale = _replay_all(prob, steps)
    e, m = solvers.solve_port(prob)[:2]
    return e, m, scale


def _run(make, problem, steps, env=None, conv=None, warm=False):
    """Warm steps on make() against the oracle on problem() and a cold rebuild; returns the graph, energy and mask."""
    with _env(**(env or {})):
        g = make()
        if warm:
            g.enable_warm()
        g.maxflow()
        done = []
        for step in steps:
            _apply(g, step, conv)
            done.append(step)
            e = g.maxflow()
            m = g.get_mask()
            oe, om, scale = _oracle(problem(), done)
            bound = max(abs(oe), scale)
            assert numpy.array_equal(m, om), ("warm mask differs from the oracle", len(done), int((m != om).sum()))
            assert abs(e - oe) <= 1e-9 * bound, (len(done), e, oe, bound)
            cold = make()
            for s in done:
                _apply(cold, s)
            ce, cm = cold.maxflow(), cold.get_mask()
            assert numpy.array_equal(m, cm), ("warm mask differs from the cold rebuild", len(done))
            assert abs(e - ce) <= 1e-12 * bound + 1e-10, (len(done), e, ce, bound)
        st = g.stats()
        assert st["seed_folds"] == sum(len(s) for s in steps) and st["ms_seeds"] > 0
        return g, e, g.get_mask().copy()


def _seq(shape, vol, prob, which):
    stroke = _ids(_stroke(shape))
    fgm = _ids(vol["fg"])
    if which == "brush":                                   # list form, across tile borders
        return [[_brush(shape)]]
    if which == "box":
        return [[_dense_box(shape)]]
    if which == "lambda":
        return [_lambda_step(prob, shape)]
    if which == "successive":                              # interleaved with the t-link folds
        src, snk = _regional_delta(vol, _box(shape))
        return [[_brush(shape, 0.7, 0.1, 2.0)], [("s", stroke, None), _dense_box(shape, len(shape) - 1, 1.5)],
                [("r", fgm[::3], None), ("t", None, src, snk)], _lambda_step(prob, shape, 0.5),
                [_brush(shape, 0.3, 0.15, 50.0), ("t", stroke[::2], 0.0, 20.0)]]
    raise ValueError(which)


_WHICH = ["brush", "box", "lambda", "successive"]


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("shape,kind,regional,dtype,spacing", [
    ((24, 20, 32), "difference_exponential", True, "float32", False),
    ((33, 17, 40), "difference_exponential", True, "float64", False),
    ((24, 20, 32), "difference_linear", True, "float32", False),
    ((24, 20, 32), "maximum_exponential", True, "float32", False),
    ((24, 20, 32), "difference_exponential", False, "int16", False),
    ((24, 20, 32), "difference_power", True, "float64", (1.0, 2.0, 0.5)),
    ((48, 40), "difference_exponential", True, "float32", False),
    ((300,), "difference_exponential", True, "float32", False),
])
def test_lazy_warm_matches_from_scratch(shape, kind, regional, dtype, spacing, which):
    vol = _vol_1d() if len(shape) == 1 else _volume(shape, seed=3, dtype=dtype)
    prob0 = _problem(vol, kind, regional, spacing)
    _run(lambda: _graph(vol, kind, regional, spacing), lambda: _problem(vol, kind, regional, spacing),
         _seq(shape, vol, prob0, which))


_HANDLES = [("4d", (6, 8, 8, 3)), ("4d", (9, 5, 17, 3)), ("4d", (12, 12, 16, 6)), ("eager", (24, 20, 32)),
            ("per_term", (19, 27, 13)), ("nweights", (16, 16, 16)), ("2d", (20, 24)), ("1d", (300,))]


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("handle,shape", _HANDLES, ids=["%s-%s" % (h, "x".join(map(str, s))) for h, s in _HANDLES])
def test_opted_in_warm_matches_from_scratch(handle, shape, which):
    vol = _vol_1d() if len(shape) == 1 else _volume(shape, seed=3, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    _run(lambda: _make(handle, vol), lambda: _problem(vol, _KIND, True, False), _seq(shape, vol, prob0, which),
         env=_ENV.get(handle), warm=True)


@pytest.mark.parametrize("env", [dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_FIRST_TEST=1), dict(MEDPY_GC_DEBUG=1)])
def test_solver_options(env):
    """MEDPY_GC_DEBUG=1 checks the invariants (residual mask included) and flow conservation around every warm solve."""
    shape = (32, 32, 32)
    vol = _volume(shape, seed=5, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    _run(lambda: _graph(vol, _KIND, True, False), lambda: _problem(vol, _KIND, True, False),
         _seq(shape, vol, prob0, "successive"), env=env)
    _run(lambda: _make("4d", _volume((9, 5, 17, 3), seed=5, dtype="float32")),
         lambda: _problem(_volume((9, 5, 17, 3), seed=5, dtype="float32"), _KIND, True, False),
         [[_brush((9, 5, 17, 3))], _lambda_step(_problem(_volume((9, 5, 17, 3), seed=5, dtype="float32"), _KIND, True, False),
                                                (9, 5, 17, 3))], env=env, warm=True)


def test_integer_weights_are_bit_exact():
    """Integer t-links, integer n-links through add_nweights_dense and integer increments: every sum is exact, so the warm
    energy equals the oracle's bit for bit."""
    from medpy_b200.graphcut.maxflow import GraphDouble
    from oracle import solvers
    shape = (20, 18, 24)
    n = int(numpy.prod(shape))
    rng = numpy.random.default_rng(9)
    src, snk = rng.integers(0, 40, n).astype(float), rng.integers(0, 40, n).astype(float)
    w = [rng.integers(1, 12, n).astype(float) for _ in shape]
    for d, s in enumerate(shape):
        c = numpy.unravel_index(numpy.arange(n), shape)[d]
        w[d][c + 1 >= s] = 0.0

    def make():
        g = GraphDouble(n, 0, shape=shape)
        g.add_tweights_dense(src.reshape(shape), snk.reshape(shape))
        for d in range(len(shape)):
            g.add_nweights_dense(d, w[d].reshape(shape), w[d].reshape(shape))
        g.enable_warm()
        return g

    def problem():
        return dict(shape=shape, wf=[x.copy() for x in w], wb=[x.copy() for x in w], tr=src - snk,
                    flow_const=float(numpy.minimum(src, snk).sum()), fg=numpy.zeros(shape, numpy.uint8),
                    bg=numpy.zeros(shape, numpy.uint8), src=src, snk=snk)

    lo, hi = _pairs_in(_ball(shape, 0.5, 0.25))
    box = numpy.zeros(shape)
    box[_box(shape)] = 7.0
    steps = [[("n", lo, hi, rng.integers(0, 30, lo.size).astype(float), rng.integers(0, 30, lo.size).astype(float))],
             [("d", 1, box, 2.0 * box)], [("d", d, w[d].reshape(shape), 3.0 * w[d].reshape(shape)) for d in range(3)]]
    g = make()
    g.maxflow()
    for k in range(1, len(steps) + 1):
        _apply(g, steps[k - 1])
        e, m = g.maxflow(), g.get_mask()
        oe, om = _oracle(problem(), steps[:k])[:2]
        assert e == oe and numpy.array_equal(m, om), (k, e, oe)


def _reclamp_case(shape, handle):
    """An fg seed next to a weak boundary: strengthening the arcs that leave the seeded region toward the background must
    push the seeds' un-pushed source residual through them and move the cut."""
    vol = _volume(shape, seed=1, dtype="float32")
    fg = numpy.zeros(shape, bool)
    fg[tuple(slice(s // 2 - 1, s // 2 + 1) for s in shape)] = True
    vol["fg"] = fg
    lo, hi = _pairs_in(numpy.ones(shape, bool))
    leave = fg.ravel()[lo] != fg.ravel()[hi]
    i = numpy.where(fg.ravel()[lo[leave]], lo[leave], hi[leave])
    j = numpy.where(fg.ravel()[lo[leave]], hi[leave], lo[leave])
    return vol, [[("n", i, j, 1e4, 0.0)]]


@pytest.mark.parametrize("handle", ["lazy", "eager", "4d"])
def test_reclamp_moves_the_cut(handle):
    shape = (6, 8, 8, 3) if handle == "4d" else (16, 16, 16)
    vol, steps = _reclamp_case(shape, handle)
    make = (lambda: _graph(vol, _KIND, True, False)) if handle == "lazy" else (lambda: _make(handle, vol))
    g0 = make()
    e0 = g0.maxflow()
    m0 = g0.get_mask().copy()
    g, e, m = _run(make, lambda: _problem(vol, _KIND, True, False), steps, env=_ENV.get(handle),
                   warm=handle != "lazy")
    assert not numpy.array_equal(m, m0) and e > e0, "the stroke must move the cut"


def test_device_arrays_match_host_arrays_bit_for_bit():
    import torch
    shape = (20, 24, 32)
    vol = _volume(shape, seed=6, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    steps = _seq(shape, vol, prob0, "successive")
    make, problem = (lambda: _graph(vol, _KIND, True, False)), (lambda: _problem(vol, _KIND, True, False))
    _, e_host, m_host = _run(make, problem, steps)
    _, e_dev, m_dev = _run(make, problem, steps, conv=lambda a: torch.from_numpy(numpy.ascontiguousarray(a)).cuda())
    assert e_dev == e_host and numpy.array_equal(m_dev, m_host)


def test_empty_and_zero_calls_keep_the_result():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, _KIND, True, False)
    e = g.maxflow()
    m = g.get_mask().copy()
    g.add_nweights_warm(numpy.zeros(0, numpy.int64), numpy.zeros(0, numpy.int64), 1.0, 1.0)
    g.add_nweights_warm([5, 9], [6, 9 + 16], 0.0, 0.0)
    g.add_nweights_dense_warm(0, numpy.zeros(shape), numpy.zeros(shape))
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 0


def test_bad_calls_leave_the_result():
    """Ids out of range, non-neighbour pairs, NaN and negative weights are refused before anything changes the state; a
    valid fold afterwards still matches the oracle."""
    shape = (16, 16, 16)
    n = 16 ** 3
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, _KIND, True, False)
    g.maxflow()
    first = _brush(shape, 0.3, 0.1, 4.0)
    _apply(g, [first])
    e = g.maxflow()
    m = g.get_mask().copy()
    nat = g._nat()
    one, zero = numpy.ones(2), numpy.zeros(2)
    with pytest.raises(ValueError, match="out of range"):
        nat.add_nweights_warm(numpy.array([5, n - 1], numpy.int64), numpy.array([6, n], numpy.int64), one, one)
    with pytest.raises(ValueError, match="neighbours"):
        nat.add_nweights_warm(numpy.array([5, 16 * 16 - 1], numpy.int64), numpy.array([6, 16 * 16], numpy.int64), one, one)
    with pytest.raises(ValueError, match="neighbours"):
        nat.add_nweights_warm(numpy.array([5, 7], numpy.int64), numpy.array([6, 7], numpy.int64), one, one)
    with pytest.raises(ValueError, match="NaN or infinite"):
        nat.add_nweights_warm(numpy.array([5, 7], numpy.int64), numpy.array([6, 8], numpy.int64), one,
                              numpy.array([1.0, numpy.nan]))
    with pytest.raises(ValueError, match="[Nn]egative"):
        nat.add_nweights_warm(numpy.array([5, 7], numpy.int64), numpy.array([6, 8], numpy.int64), one,
                              numpy.array([1.0, -1.0]))
    bad = numpy.ones(shape)
    bad[3, 4, 5] = -2.0
    with pytest.raises(ValueError, match="[Nn]egative"):
        nat.add_nweights_dense_warm(2, bad, numpy.ones(shape))
    bad[3, 4, 5] = numpy.inf
    with pytest.raises(ValueError, match="NaN or infinite"):
        nat.add_nweights_dense_warm(2, numpy.ones(shape), bad)
    with pytest.raises(ValueError, match="neighbours"):
        g.add_nweights_warm([0], [2], 1.0, 1.0)
    with pytest.raises(ValueError, match="[Nn]egative"):
        g.add_nweights_warm([0], [1], -1.0, 1.0)
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 1
    second = _dense_box(shape, 1, 2.0)
    _apply(g, [second])
    e2, m2 = g.maxflow(), g.get_mask()
    oe, om, scale = _oracle(_problem(vol, _KIND, True, False), [[first], [second]])
    assert numpy.array_equal(m2, om) and abs(e2 - oe) <= 1e-9 * max(abs(oe), scale)


@pytest.mark.parametrize("case", ["eager", "4d", "per_term", "sparse"])
def test_handles_without_warm_path_refuse(case):
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut.maxflow import GraphDouble
    env = dict(eager=dict(MEDPY_GC_LAZY_CAPS=0)).get(case, {})
    shape = (12, 12, 16)
    with _env(**env):
        if case == "sparse":
            g = GraphDouble(4, 4, sparse=True)
            g.add_tweights(0, 5.0, 0.0)
            g.sum_edge(0, 1, 1.0, 1.0)
            g._solved = True
            with pytest.raises(RuntimeError, match="reset.*rebuild"):
                g.add_nweights_warm([0], [1], 1.0, 0.0)
            with pytest.raises(RuntimeError, match="reset.*rebuild"):
                g.add_nweights_dense_warm(0, numpy.ones(4), numpy.ones(4))
            return
        if case == "4d":
            vol = _volume((6, 8, 8, 3), seed=1, dtype="float32")
            g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                     boundary_term_args=(vol["image"], vol["sigma"], False))
        elif case == "per_term":
            vol = _volume(shape, seed=1, dtype="float32")
            g = _make("per_term", vol)
        else:
            vol = _volume(shape, seed=1, dtype="float32")
            g = _graph(vol, _KIND, True, False)
        g.maxflow()
        with pytest.raises(RuntimeError, match="reset"):
            g.add_nweights_warm([3], [4], 1.0, 0.0)
        with pytest.raises(RuntimeError, match="reset"):
            g.add_nweights_dense_warm(0, numpy.ones(g.shape), numpy.ones(g.shape))


@pytest.mark.parametrize("handle", ["lazy", "4d"])
def test_first_solve_is_unchanged(handle):
    """Staged before the first solve, the calls give bit for bit what the same sum_edge calls give."""
    shape = (6, 8, 8, 3) if handle == "4d" else (20, 24, 32)
    vol = _volume(shape, seed=4, dtype="float32")
    make = (lambda: _graph(vol, _KIND, True, False)) if handle == "lazy" else (lambda: _make("4d", vol))
    op = _brush(shape)
    g = make()
    g.add_nweights_warm(*op[1:])
    ref = make()
    for i, j, c, r in zip(op[1].tolist(), op[2].tolist(), op[3].tolist(), op[4].tolist()):
        ref.sum_edge(i, j, c, r)
    assert g.maxflow().hex() == ref.maxflow().hex() and numpy.array_equal(g.get_mask(), ref.get_mask())


def test_native_call_before_the_first_solve():
    """A C-ABI fold on a lazily built handle that was never solved materialises and folds like after a solve."""
    shape = (20, 24, 32)
    vol = _volume(shape, seed=8, dtype="float32")
    g = _graph(vol, _KIND, True, False)
    g._flush()
    op = _brush(shape)
    g._nat().add_nweights_warm(op[1].astype(numpy.int64), op[2].astype(numpy.int64), op[3], op[4])
    e, m = g.maxflow(), g.get_mask()
    oe, om, scale = _oracle(_problem(vol, _KIND, True, False), [[op]])
    assert numpy.array_equal(m, om) and abs(e - oe) <= 1e-9 * max(abs(oe), scale)


def test_stats_count_the_fold():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, _KIND, True, False)
    g.maxflow()
    before = g.stats()
    _apply(g, [_brush(shape)])
    after = g.stats()
    assert after["seed_folds"] == before["seed_folds"] + 1 and after["ms_seeds"] > before["ms_seeds"]
    assert after["kernel_launches"] - before["kernel_launches"] >= 3 + 2 + 4


def _full_size_steps(vol, prob, shape):
    return [[_brush(shape, 0.3, 0.05, 1.0)], _lambda_step(prob, shape)]


def test_config3_256_against_reference_bk():
    """Config 3 at 256^3: a boundary brush, then a lambda step -- masks equal to the real reference BK's on the
    from-scratch graph, energies within 1e-9 S."""
    from oracle import solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")
    shape = (256, 256, 256)
    vol = _volume(shape, seed=0, dtype="float32")
    steps = _full_size_steps(vol, _problem(vol, _KIND, True, False), shape)
    g = _graph(vol, _KIND, True, False)
    g.maxflow()
    for k, step in enumerate(steps, 1):
        _apply(g, step)
        e, m = g.maxflow(), g.get_mask()
        prob = _problem(vol, _KIND, True, False)
        scale = _replay_all(prob, steps[:k])
        ref = dict(prob, src=numpy.maximum(prob["tr"], 0.0), snk=numpy.maximum(-prob["tr"], 0.0),
                   fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool))
        oe, om, _ = solvers.solve_ref(ref)
        oe += prob["flow_const"]
        assert int((m != om).sum()) == 0, k
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (k, e, oe, scale)


def test_config4_full_size_against_reference_bk():
    """Config 4 (256x256x128x4, maximum_exponential): a brush and a lambda step.  The maximum term has structural ties
    (test_gpu_warm_eager.py), so where the masks differ the exact capacities of the two cuts must agree."""
    import medpy_b200.graphcut as gc
    from oracle import energy_terms as et, solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")
    from test_gpu_fullsize import _cut_difference_exact
    shape = (256, 256, 128, 4)
    vol = _volume(shape, seed=0, dtype="float32")

    def problem():
        return et.build_problem(vol["fg"], vol["bg"], boundary=("maximum_exponential", vol["image"], vol["sigma"], False))
    steps = _full_size_steps(vol, problem(), shape)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_maximum_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    g.enable_warm()
    g.maxflow()
    for k, step in enumerate(steps, 1):
        _apply(g, step)
        e, m = g.maxflow(), g.get_mask()
        prob = problem()
        scale = _replay_all(prob, steps[:k])
        ref = dict(prob, src=numpy.maximum(prob["tr"], 0.0), snk=numpy.maximum(-prob["tr"], 0.0),
                   fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool))
        oe, om, _ = solvers.solve_ref(ref)
        oe += prob["flow_const"]
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (k, e, oe, scale)
        if int((m != om).sum()):
            diff = _cut_difference_exact(prob, m, om)
            assert abs(diff) <= 1e-9 * max(abs(oe), scale), (k, int((m != om).sum()), diff)
