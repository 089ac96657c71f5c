"""n-link capacity taken off a lattice graph and solved warm (GraphDouble.remove_nweights_warm /
remove_nweights_dense_warm, mgc_remove_nweights_warm / mgc_remove_nweights_dense_warm): after each step the mask must
equal the oracle's on the from-scratch graph with every call so far replayed (decrements subtracted), and the energy must
be within 1e-9 S of it and within 1e-10 S of a cold GPU build of the final graph (S as in
test_gpu_warm_nweights.py, plus the sum of the decrements).

Steps are lists of the operations of test_gpu_warm_nweights.py plus
  ("rn", i, j, cap, rev)   remove_nweights_warm: sum_edge(i[k], j[k], -cap[k], -rev[k]) in order;
  ("rd", axis, fwd, bwd)   remove_nweights_dense_warm."""
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_erase_seeds import _problem, _vol_1d  # noqa: E402
from test_gpu_seeds import _env, _graph, _ids, _stroke, _volume  # noqa: E402
from test_gpu_warm_eager import _ENV, _make  # noqa: E402
from test_gpu_warm_nweights import _apply as _apply_add, _brush, _pairs_in, _replay_all  # noqa: E402
from test_gpu_warm_tweights import _box, _regional_delta  # noqa: E402

pytestmark = pytest.mark.gpu

_KIND = "difference_exponential"


def _apply(g, step, conv=None):
    cv = (lambda a: a) if conv is None else (lambda a: conv(numpy.asarray(a)) if numpy.ndim(a) else a)
    for op in step:
        if op[0] == "rn":
            g.remove_nweights_warm(*(cv(x) for x in op[1:]))
        elif op[0] == "rd":
            g.remove_nweights_dense_warm(op[1], cv(op[2]), cv(op[3]))
        else:
            _apply_add(g, [op], conv)


def _replay(prob, steps):
    """Every operation replayed on the oracle's problem in order (decrements as negative increments); returns S."""
    shape = prob["shape"]
    plain, extra = [], 0.0
    for step in steps:
        ops = []
        for op in step:
            if op[0] == "rn":
                i, j, c, r = numpy.broadcast_arrays(numpy.asarray(op[1]), numpy.asarray(op[2]),
                                                    numpy.asarray(op[3], float), numpy.asarray(op[4], float))
                ops.append(("n", i, j, -c, -r))
                extra += 2.0 * float(c.sum() + r.sum())
            elif op[0] == "rd":
                f, b = numpy.asarray(op[2], float), numpy.asarray(op[3], float)
                ops.append(("d", op[1], -f, -b))
                keep = numpy.unravel_index(numpy.arange(f.size), shape)[op[1]] + 1 < shape[op[1]]
                extra += 2.0 * float(f.ravel()[keep].sum() + b.ravel()[keep].sum())
            else:
                ops.append(op)
        plain.append(ops)
    return _replay_all(prob, plain) + extra


def _oracle(prob, steps):
    from oracle import solvers
    scale = _replay(prob, steps)
    e, m = solvers.solve_port(prob)[:2]
    return e, m, scale, prob


def _cold(prob):
    """A from-scratch GPU build of the replayed graph: its t-links and its final n-link capacities, staged term by term."""
    from medpy_b200.graphcut.maxflow import GraphDouble
    shape = prob["shape"]
    n = int(numpy.prod(shape))
    g = GraphDouble(n, 0, shape=shape)
    tr = prob["tr"]
    g.add_tweights_dense(numpy.maximum(tr, 0.0).reshape(shape), numpy.maximum(-tr, 0.0).reshape(shape))
    for d in range(len(shape)):
        g.add_nweights_dense(d, numpy.maximum(prob["wf"][d], 0.0).reshape(shape),
                             numpy.maximum(prob["wb"][d], 0.0).reshape(shape))
    return g.maxflow() + prob["flow_const"], g.get_mask()


def _same_cut(m, om, prob, bound, ties, what):
    """Equal masks; with `ties` (the maximum term, whose equal weights give cuts of equal capacity) masks that differ
    only between cuts of exactly equal capacity."""
    if numpy.array_equal(m, om):
        return
    assert ties, (what, int((m != om).sum()))
    from test_gpu_fullsize import _cut_difference_exact
    diff = _cut_difference_exact(prob, m, om)
    assert abs(diff) <= 1e-9 * bound, (what, int((m != om).sum()), diff)


def _run(make, problem, steps, env=None, conv=None, warm=False, ties=False):
    """Warm steps on make() against the oracle on problem() and a cold build; returns the graph, energy and mask."""
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
            oe, om, scale, prob = _oracle(problem(), done)
            bound = max(abs(oe), scale)
            _same_cut(m, om, prob, bound, ties, ("warm mask differs from the oracle", len(done)))
            assert abs(e - oe) <= 1e-9 * bound, (len(done), e, oe, bound)
            ce, cm = _cold(prob)
            _same_cut(m, cm, prob, bound, ties, ("warm mask differs from the cold build", len(done)))
            assert abs(e - ce) <= 1e-10 * bound, (len(done), e, ce, bound)
        st = g.stats()
        assert st["seed_folds"] == sum(len(s) for s in steps) and st["ms_seeds"] > 0
        return g, e, g.get_mask().copy()


def _unbrush(shape, w=5.0):
    add = _brush(shape, w=w)
    return [[add], [("rn",) + add[1:]]]


def _cut_pairs(shape, mask):
    lo, hi = _pairs_in(numpy.ones(shape, bool))
    flat = numpy.ascontiguousarray(mask).ravel()
    sel = flat[lo] != flat[hi]
    return lo[sel], hi[sel]


def _cut_relax(shape, prob, mask, frac=0.5):
    """-frac of the capacity on both arcs of every pair across the first solve's cut, list form (half named from the
    upper end)."""
    lo, hi = _cut_pairs(shape, mask)
    st = tuple(int(numpy.prod(shape[d + 1:])) for d in range(len(shape)))
    axis = numpy.zeros(lo.size, int)
    for d in range(len(shape)):
        axis[(hi - lo) == st[d]] = d
    wf = numpy.array([prob["wf"][a][p] for a, p in zip(axis, lo)])
    wb = numpy.array([prob["wb"][a][p] for a, p in zip(axis, lo)])
    flip = numpy.arange(lo.size) % 2 == 1
    i, j = numpy.where(flip, hi, lo), numpy.where(flip, lo, hi)
    return ("rn", i, j, numpy.where(flip, wb, wf) * frac, numpy.where(flip, wf, wb) * frac)


def _lambda_down(prob, shape, kappa=0.25):
    return [("rd", d, kappa * prob["wf"][d].reshape(shape), kappa * prob["wb"][d].reshape(shape)) for d in range(len(shape))]


def _box_down(prob, shape, axis=0, frac=1.0):
    f = numpy.zeros(shape)
    f[_box(shape)] = 1.0
    return ("rd", axis, frac * f * prob["wf"][axis].reshape(shape), frac * f * prob["wb"][axis].reshape(shape))


def _first_mask(make, warm=False, env=None):
    with _env(**(env or {})):
        g = make()
        if warm:
            g.enable_warm()
        g.maxflow()
        return g.get_mask().copy()


def _seq(shape, vol, prob, which, mask):
    stroke = _ids(_stroke(shape))
    if which == "unbrush":
        return _unbrush(shape)
    if which == "cut_relax":
        return [[_cut_relax(shape, prob, mask)]]
    if which == "lambda_down":
        return [_lambda_down(prob, shape)]
    if which == "box":
        return [[_box_down(prob, shape, len(shape) - 1, 0.75)]]
    if which == "successive":
        # interleaved with the other folds.  The brush comes last: adding +2 to an arc of weight 1e-15 and taking it off
        # again leaves roundings of 2 in place of that weight, so a later removal of part of the weight would exceed what
        # the pair holds (DESIGN.md §4.6, "N-link decrements")
        src, snk = _regional_delta(vol, _box(shape))
        add = _brush(shape, 0.7, 0.1, 2.0)
        return [[_box_down(prob, shape, 0, 0.5), ("s", stroke, None)],
                [("t", None, src, snk), _cut_relax(shape, prob, mask, 0.25)], _lambda_down(prob, shape, 0.25),
                [("r", stroke[::2], None), add], [("rn",) + add[1:], _brush(shape, 0.3, 0.15, 3.0)]]
    raise ValueError(which)


_WHICH = ["unbrush", "cut_relax", "lambda_down", "box", "successive"]


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("shape,kind,regional,dtype,spacing", [
    ((24, 20, 32), "difference_exponential", True, "float32", False),
    ((33, 17, 40), "difference_exponential", True, "float64", False),
    ((24, 20, 32), "maximum_exponential", False, "float32", False),
    ((24, 20, 32), "difference_power", True, "float64", (1.0, 2.0, 0.5)),
    ((48, 40), "difference_exponential", True, "float32", False),
    ((300,), "difference_exponential", True, "float32", False),
])
def test_lazy_warm_matches_from_scratch(shape, kind, regional, dtype, spacing, which):
    vol = _vol_1d() if len(shape) == 1 else _volume(shape, seed=3, dtype=dtype)
    prob0 = _problem(vol, kind, regional, spacing)
    make = lambda: _graph(vol, kind, regional, spacing)  # noqa: E731
    _run(make, lambda: _problem(vol, kind, regional, spacing), _seq(shape, vol, prob0, which, _first_mask(make)),
         ties=kind.startswith("maximum"))


_HANDLES = [("4d", (6, 8, 8, 3)), ("4d", (9, 5, 17, 3)), ("eager", (24, 20, 32)), ("per_term", (19, 27, 13)),
            ("1d", (300,))]


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("handle,shape", _HANDLES, ids=["%s-%s" % (h, "x".join(map(str, s))) for h, s in _HANDLES])
def test_opted_in_warm_matches_from_scratch(handle, shape, which):
    vol = _vol_1d() if len(shape) == 1 else _volume(shape, seed=3, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    make = lambda: _make(handle, vol)  # noqa: E731
    mask = _first_mask(make, True, _ENV.get(handle))
    _run(make, lambda: _problem(vol, _KIND, True, False), _seq(shape, vol, prob0, which, mask), env=_ENV.get(handle),
         warm=True)


@pytest.mark.parametrize("handle", ["lazy", "eager", "4d"])
def test_cut_relax_runs_the_shortfall_branch(handle):
    """The arcs across the solved cut are saturated: their residual is below the decrement, so the fold cancels flow and
    takes the shortfall from the terminal links.  get_edge reads the residual on a twin graph (it materialises every tile,
    which would change the lazy path under test)."""
    shape = (6, 8, 8, 3) if handle == "4d" else (24, 20, 32)
    vol = _volume(shape, seed=3, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    warm = handle != "lazy"
    make = (lambda: _graph(vol, _KIND, True, False)) if handle == "lazy" else (lambda: _make(handle, vol))
    with _env(**_ENV.get(handle, {})):
        twin = make()
        if warm:
            twin.enable_warm()
        twin.maxflow()
        mask = twin.get_mask().copy()
        op = _cut_relax(shape, prob0, mask)
        below = sum(twin.get_edge(int(i), int(j)) < c for i, j, c in zip(op[1][:64], op[2][:64], op[3][:64]))
        assert below > 0, "no saturated arc on the cut"
    _run(make, lambda: _problem(vol, _KIND, True, False), [[op]], env=_ENV.get(handle), warm=warm)


@pytest.mark.parametrize("handle", ["lazy", "eager", "4d"])
def test_undo_restores_the_first_cut(handle):
    """add_nweights_warm(brush), solve, remove_nweights_warm(brush), solve: the mask is the first solve's, and the energy
    is the first solve's to within the roundings of the brush's weight."""
    shape = (6, 8, 8, 3) if handle == "4d" else (24, 20, 32)
    vol = _volume(shape, seed=3, dtype="float32")
    make = (lambda: _graph(vol, _KIND, True, False)) if handle == "lazy" else (lambda: _make(handle, vol))
    with _env(**_ENV.get(handle, {})):
        g = make()
        if handle != "lazy":
            g.enable_warm()
        e0 = g.maxflow()
        m0 = g.get_mask().copy()
        lo, hi = _cut_pairs(shape, m0)
        add = ("n", lo, hi, numpy.full(lo.size, 50.0), numpy.full(lo.size, 50.0))    # "do not cut here" on the whole cut
        _apply(g, [add])
        e1 = g.maxflow()
        m1 = g.get_mask().copy()
        _apply(g, [("rn",) + add[1:]])
        e2 = g.maxflow()
        assert e1 > e0 and not numpy.array_equal(m1, m0), "the brush must move the cut"
        assert numpy.array_equal(g.get_mask(), m0)
        assert abs(e2 - e0) <= 1e-12 * (abs(e0) + float(add[3].sum() + add[4].sum())), (e2, e0)


def test_shortfall_over_many_blocks_is_reproducible():
    """A cut relax whose shortfall voxels span many blocks of the voxel pass: fresh graphs, host and device arguments,
    give the same energy bit for bit (the tails are sorted before the pass, so the per-block sums of the add_tweights
    constant do not depend on the order the atomics listed them in)."""
    import torch
    shape = (64, 64, 64)
    vol = _volume(shape, seed=7, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    make = lambda: _graph(vol, _KIND, True, False)  # noqa: E731
    op = _cut_relax(shape, prob0, _first_mask(make), 0.75)
    assert op[1].size > 8 * 256, op[1].size           # > 8 blocks of items, twice as many tails
    out = []
    for conv in (None, None, lambda a: torch.from_numpy(numpy.ascontiguousarray(a)).cuda(), None):
        g = make()
        g.maxflow()
        _apply(g, [op], conv)
        out.append((g.maxflow().hex(), g.get_mask().tobytes()))
    assert all(o == out[0] for o in out)
    oe, om, scale, _ = _oracle(_problem(vol, _KIND, True, False), [[op]])
    assert numpy.array_equal(numpy.frombuffer(out[0][1], numpy.uint8).reshape(shape), om)
    assert abs(float.fromhex(out[0][0]) - oe) <= 1e-9 * max(abs(oe), scale)


def _two_voxel():
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(2, 1, shape=(2,))
    g.add_tweights(0, 5.0, 0.0)
    g.add_tweights(1, 0.0, 5.0)
    g.sum_edge(0, 1, 5.0, 0.0)
    g.enable_warm()
    assert g.maxflow() == 5.0
    return g


def test_two_voxel_hand_check():
    g = _two_voxel()
    g.remove_nweights_warm([0], [1], 3.0, 0.0)
    assert g.maxflow() == 2.0
    g = _two_voxel()
    g.remove_nweights_warm([0], [1], 5.0, 0.0)
    assert g.maxflow() == 0.0
    g = _two_voxel()
    with pytest.raises(ValueError, match="exceeds"):
        g.remove_nweights_warm([0, 1], [1, 0], 3.0, 0.0)
    assert g.maxflow() == 5.0 and g.get_mask().tolist() == _two_voxel().get_mask().tolist()


@pytest.mark.parametrize("handle", ["lazy", "eager", "4d"])
def test_exact_removal_is_accepted_and_more_is_refused(handle):
    """Removing exactly the weight a box holds passes the pair check; 1e-6 relative more is refused with the handle
    unchanged, and the exact removal afterwards still matches the oracle."""
    shape = (6, 8, 8, 3) if handle == "4d" else (24, 20, 32)
    vol = _volume(shape, seed=4, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    warm = handle != "lazy"
    make = (lambda: _graph(vol, _KIND, True, False)) if handle == "lazy" else (lambda: _make(handle, vol))
    exact = _box_down(prob0, shape, 1, 1.0)
    with _env(**_ENV.get(handle, {})):
        g = make()
        if warm:
            g.enable_warm()
        e0 = g.maxflow()
        m0 = g.get_mask().copy()
        with pytest.raises(ValueError, match="exceeds"):
            g.remove_nweights_dense_warm(1, exact[2] * (1 + 1e-6), exact[3])
        assert g.maxflow() == e0 and numpy.array_equal(g.get_mask(), m0)
        assert g.stats()["seed_folds"] == 0
    _run(make, lambda: _problem(vol, _KIND, True, False), [[exact]], env=_ENV.get(handle), warm=warm)


def test_integer_weights_are_bit_exact():
    from medpy_b200.graphcut.maxflow import GraphDouble
    shape = (20, 18, 24)
    n = int(numpy.prod(shape))
    rng = numpy.random.default_rng(9)
    src, snk = rng.integers(0, 40, n).astype(float), rng.integers(0, 40, n).astype(float)
    w = [rng.integers(4, 12, n).astype(float) for _ in shape]
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

    g0 = make()
    g0.maxflow()
    mask = g0.get_mask()
    lo, hi = _cut_pairs(shape, mask)
    box = numpy.zeros(shape)
    box[_box(shape)] = 2.0
    steps = [[("rn", lo, hi, 3.0, 1.0)], [("rd", 1, box, box)],
             [("d", 0, w[0].reshape(shape), w[0].reshape(shape)), ("rd", 0, w[0].reshape(shape), 0 * box)],
             [("rd", d, numpy.maximum(w[d] - 6.0, 0.0).reshape(shape), 0 * box) for d in range(1, 3)]]
    g = make()
    g.maxflow()
    for k in range(1, len(steps) + 1):
        _apply(g, steps[k - 1])
        e, m = g.maxflow(), g.get_mask()
        oe, om = _oracle(problem(), steps[:k])[:2]
        assert e == oe and numpy.array_equal(m, om), (k, e, oe)


@pytest.mark.parametrize("env", [dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_FIRST_TEST=1), dict(MEDPY_GC_DEBUG=1)])
def test_solver_options(env):
    """MEDPY_GC_DEBUG=1 checks the invariants (residual mask included) and flow conservation around every warm solve."""
    shape = (32, 32, 32)
    vol = _volume(shape, seed=5, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    make = lambda: _graph(vol, _KIND, True, False)  # noqa: E731
    _run(make, lambda: _problem(vol, _KIND, True, False), _seq(shape, vol, prob0, "successive", _first_mask(make)), env=env)
    s4 = (9, 5, 17, 3)
    v4 = _volume(s4, seed=5, dtype="float32")
    p4 = _problem(v4, _KIND, True, False)
    make4 = lambda: _make("4d", v4)  # noqa: E731
    _run(make4, lambda: _problem(v4, _KIND, True, False),
         [[_cut_relax(s4, p4, _first_mask(make4, True))], _lambda_down(p4, s4), _unbrush(s4)[0], _unbrush(s4)[1]],
         env=env, warm=True)


def test_device_arrays_match_host_arrays_and_runs_repeat_bit_for_bit():
    import torch
    shape = (20, 24, 32)
    vol = _volume(shape, seed=6, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    make, problem = (lambda: _graph(vol, _KIND, True, False)), (lambda: _problem(vol, _KIND, True, False))
    steps = _seq(shape, vol, prob0, "successive", _first_mask(make))
    _, e_host, m_host = _run(make, problem, steps)
    _, e_again, m_again = _run(make, problem, steps)
    _, e_dev, m_dev = _run(make, problem, steps, conv=lambda a: torch.from_numpy(numpy.ascontiguousarray(a)).cuda())
    assert e_again == e_host and numpy.array_equal(m_again, m_host)
    assert e_dev == e_host and numpy.array_equal(m_dev, m_host)


def test_bad_calls_leave_the_result():
    """Negative or NaN decrements, ids out of range, non-neighbour pairs and pair-sum violations are refused before
    anything changes the state; a valid fold afterwards still matches the oracle."""
    shape = (16, 16, 16)
    n = 16 ** 3
    vol = _volume(shape, seed=2, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    g = _graph(vol, _KIND, True, False)
    g.maxflow()
    e = g.maxflow()
    m = g.get_mask().copy()
    nat = g._nat()
    one = numpy.ones(2)
    i2, j2 = numpy.array([5, 7], numpy.int64), numpy.array([6, 8], numpy.int64)
    with pytest.raises(ValueError, match="out of range"):
        nat.remove_nweights_warm(numpy.array([5, n - 1], numpy.int64), numpy.array([6, n], numpy.int64), one, one)
    with pytest.raises(ValueError, match="neighbours"):
        nat.remove_nweights_warm(numpy.array([5, 16 * 16 - 1], numpy.int64), numpy.array([6, 16 * 16], numpy.int64),
                                 one, one)
    with pytest.raises(ValueError, match="NaN or infinite"):
        nat.remove_nweights_warm(i2, j2, one, numpy.array([0.0, numpy.nan]))
    with pytest.raises(ValueError, match="[Nn]egative"):
        nat.remove_nweights_warm(i2, j2, one * 0, numpy.array([0.0, -1.0]))
    with pytest.raises(ValueError, match="exceeds"):
        nat.remove_nweights_warm(i2, j2, numpy.array([0.0, 1e6]), one * 0)
    bad = numpy.zeros(shape)
    bad[3, 4, 5] = -2.0
    with pytest.raises(ValueError, match="[Nn]egative"):
        nat.remove_nweights_dense_warm(2, bad, numpy.zeros(shape))
    bad[3, 4, 5] = 1e6
    with pytest.raises(ValueError, match="exceeds"):
        nat.remove_nweights_dense_warm(2, bad, numpy.zeros(shape))
    with pytest.raises(ValueError, match="neighbours"):
        g.remove_nweights_warm([0], [2], 1.0, 1.0)
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 0
    step = [_box_down(prob0, shape, 1, 0.5)]
    _apply(g, step)
    e2, m2 = g.maxflow(), g.get_mask()
    oe, om, scale, _ = _oracle(_problem(vol, _KIND, True, False), [step])
    assert numpy.array_equal(m2, om) and abs(e2 - oe) <= 1e-9 * max(abs(oe), scale)


@pytest.mark.parametrize("case", ["eager", "4d", "sparse"])
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
            g.maxflow()
            with pytest.raises(RuntimeError, match="reset.*rebuild"):
                g.remove_nweights_warm([0], [1], 1.0, 0.0)
            return
        if case == "4d":
            vol = _volume((6, 8, 8, 3), seed=1, dtype="float32")
            g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                     boundary_term_args=(vol["image"], vol["sigma"], False))
        else:
            vol = _volume(shape, seed=1, dtype="float32")
            g = _graph(vol, _KIND, True, False)
        g.maxflow()
        with pytest.raises(RuntimeError, match="reset"):
            g.remove_nweights_warm([3], [4], 0.0, 0.0)
        with pytest.raises(RuntimeError, match="reset"):
            g.remove_nweights_dense_warm(0, numpy.zeros(g.shape), numpy.zeros(g.shape))


def test_unsolved_graph_folds_after_the_flush():
    """Before the first solve the pending build is flushed and the decrement folds natively; the first solve then gives
    the decreased graph's cut."""
    shape = (20, 24, 32)
    vol = _volume(shape, seed=8, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    g = _graph(vol, _KIND, True, False)
    step = [_box_down(prob0, shape, 2, 0.5), _cut_relax(shape, prob0, _first_mask(lambda: _graph(vol, _KIND, True, False)))]
    _apply(g, step)
    e, m = g.maxflow(), g.get_mask()
    oe, om, scale, _ = _oracle(_problem(vol, _KIND, True, False), [step])
    assert numpy.array_equal(m, om) and abs(e - oe) <= 1e-9 * max(abs(oe), scale)


def test_stats_count_the_fold():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, _KIND, True, False)
    g.maxflow()
    before = g.stats()
    _apply(g, [_cut_relax(shape, _problem(vol, _KIND, True, False), g.get_mask())])
    after = g.stats()
    assert after["seed_folds"] == before["seed_folds"] + 1 and after["ms_seeds"] > before["ms_seeds"]
    # keys, sort, heads, scan, items (cub included), check, arcs, voxels, partial sum, push lists
    assert after["kernel_launches"] - before["kernel_launches"] >= 3 + 3 + 4


def test_config3_256_against_reference_bk():
    """Config 3 at 256^3: a brush added and removed, the cut relaxed, lambda lowered -- masks equal to the reference
    BK's on the from-scratch graph, energies within 1e-9 S."""
    from oracle import solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")
    shape = (256, 256, 256)
    vol = _volume(shape, seed=0, dtype="float32")
    prob0 = _problem(vol, _KIND, True, False)
    g = _graph(vol, _KIND, True, False)
    g.maxflow()
    add = _brush(shape, 0.3, 0.05, 1.0)
    steps = [[add], [("rn",) + add[1:]], [_cut_relax(shape, prob0, g.get_mask())], _lambda_down(prob0, shape)]
    for k, step in enumerate(steps, 1):
        _apply(g, step)
        e, m = g.maxflow(), g.get_mask()
        prob = _problem(vol, _KIND, True, False)
        scale = _replay(prob, steps[:k])
        ref = dict(prob, src=numpy.maximum(prob["tr"], 0.0), snk=numpy.maximum(-prob["tr"], 0.0),
                   fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool))
        oe, om, _ = solvers.solve_ref(ref)
        oe += prob["flow_const"]
        assert int((m != om).sum()) == 0, k
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (k, e, oe, scale)
