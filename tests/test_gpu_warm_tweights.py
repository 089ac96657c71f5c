"""Any add_tweights calls folded into a solved graph and solved warm (mgc_add_tweights_warm / GraphDouble.add_tweights_warm):
after each step the mask and energy must be those of the from-scratch graph with the same add_tweights sequence -- against
the oracle (the BK restatement, or the real reference BK at 256^3) and against a cold GPU rebuild that stages the same calls
before its solve.

Energy bound, as in test_gpu_erase_seeds.py: energies are compared relative to S = max(|E|, |build constant| + the sum over
the replayed calls of |s| + |t| + |t-link before the call|), which bounds the sum of the |add_tweights minima|:
1e-9 S against the oracle, 1e-12 S + 1e-10 against the cold rebuild."""
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_erase_seeds import _problem, _vol_1d  # noqa: E402
from test_gpu_seeds import _ball, _env, _graph, _ids, _stroke, _volume  # noqa: E402

pytestmark = pytest.mark.gpu


def _replay(prob, steps):
    """Every call of every step: a list call (ids, src, snk) applies add_tweights(ids[k], src[k], snk[k]), the k-th
    occurrence of an id in pass k (a voxel's t-link only depends on its own calls); a dense call (None, src, snk) is one
    pass over all nodes.  Returns S of the module docstring without |E|."""
    from oracle import energy_terms as et
    n = prob["tr"].size
    scale = abs(prob["flow_const"])
    for step in steps:
        for ids, src, snk in step:
            if ids is None:
                s, t = numpy.ravel(src).astype(numpy.float64), numpy.ravel(snk).astype(numpy.float64)
                scale += float((numpy.abs(prob["tr"]) + numpy.abs(s) + numpy.abs(t)).sum())
                prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], s, t)
                continue
            ids = numpy.asarray(ids, dtype=numpy.int64)
            if ids.size == 0:
                continue
            src = numpy.broadcast_to(numpy.asarray(src, dtype=numpy.float64), ids.shape)
            snk = numpy.broadcast_to(numpy.asarray(snk, dtype=numpy.float64), ids.shape)
            order = numpy.argsort(ids, kind="stable")
            sids = ids[order]
            starts = numpy.flatnonzero(numpy.r_[True, sids[1:] != sids[:-1]])
            rank = numpy.empty(ids.size, numpy.int64)
            rank[order] = numpy.arange(ids.size) - numpy.repeat(starts, numpy.diff(numpy.r_[starts, ids.size]))
            for r in range(int(rank.max()) + 1):
                sel = rank == r
                s, t = numpy.zeros(n), numpy.zeros(n)
                s[ids[sel]], t[ids[sel]] = src[sel], snk[sel]
                where = numpy.zeros(n, bool)
                where[ids[sel]] = True
                scale += float((numpy.abs(prob["tr"][where]) + numpy.abs(s[where]) + numpy.abs(t[where])).sum())
                prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], s, t, where=where)
    return scale


def _oracle(vol, kind, regional, spacing, steps):
    from oracle import solvers
    prob = _problem(vol, kind, regional, spacing)
    scale = _replay(prob, steps)
    e, m = solvers.solve_port(prob)[:2]
    return e, m, scale


def _apply(g, step, conv=None):
    for ids, src, snk in step:
        if ids is not None:
            ids = numpy.asarray(ids, dtype=numpy.int64)
        if conv is not None:
            ids = None if ids is None else conv(ids)
            src = conv(numpy.asarray(src)) if numpy.ndim(src) else src
            snk = conv(numpy.asarray(snk)) if numpy.ndim(snk) else snk
        g.add_tweights_warm(ids, src, snk)


def _cold(vol, kind, regional, spacing, steps):
    """The same sequence built from scratch on the GPU: every call staged before the first solve."""
    g = _graph(vol, kind, regional, spacing)
    for step in steps:
        _apply(g, step)
    return g.maxflow(), g.get_mask()


def _regional_delta(vol, box):
    """GrabCut-style re-estimation: the change of the regional term for p' = sigmoid((image - 55) / 15), as dense t-link
    deltas ((p' - p) alpha, ((1 - p') - (1 - p)) alpha), zero outside `box` (None: the whole lattice)."""
    img = vol["image"].astype(numpy.float64)
    p = vol["prob"].astype(numpy.float64)
    p2 = 1.0 / (1.0 + numpy.exp(-(img - 55.0) / 15.0))
    a = float(vol["alpha"])
    src, snk = (p2 - p) * a, ((1.0 - p2) - (1.0 - p)) * a
    if box is not None:
        keep = numpy.zeros(img.shape, bool)
        keep[box] = True
        src, snk = numpy.where(keep, src, 0.0), numpy.where(keep, snk, 0.0)
    return src, snk


def _box(shape):
    """A box around blob 1 (centre 0.3 of every axis)."""
    return tuple(slice(int(0.15 * s), max(int(0.45 * s), int(0.15 * s) + 1)) for s in shape)


def _sequences(shape, vol, which):
    """Steps of (ids or None, src, snk) calls; the graph is solved after every step."""
    stroke = _ids(_stroke(shape))                       # across the background
    fgm = _ids(vol["fg"])
    carve = _ids(_ball(shape, 0.3, 0.05)) if len(shape) > 1 else fgm[fgm.size // 4: fgm.size // 2]
    rng = numpy.random.default_rng(11)
    if which == "soft_fg":                              # a soft stroke toward the source
        return [[(stroke, 50.0, 0.0)]]
    if which == "soft_bg":                              # ... toward the sink, inside blob 1
        return [[(carve, 0.0, 40.0)]]
    if which == "negative":                             # negative weights: lower t-links, on markers too
        return [[(stroke, -30.0, 0.0), (fgm[::3], 0.0, -20.0), (carve, -5.0, -2.5)]]
    if which == "mixed":                                # mixed signs on one voxel within one call, repeated ids
        v, w = int(stroke[0]), int(carve[0])
        ids = numpy.concatenate([[v, w, v, v], stroke[1:], [w]])
        src = numpy.concatenate([[5.0, -8.0, -8.0, 1.5], rng.uniform(-20, 20, stroke.size - 1), [70.0]])
        snk = numpy.concatenate([[-3.0, 2.0, 2.0, 4.0], rng.uniform(-20, 20, stroke.size - 1), [-6.0]])
        return [[(ids, src, snk)]]
    if which == "regional_box":                         # dense, zero outside a box
        return [[(None,) + _regional_delta(vol, _box(shape))]]
    if which == "regional_all":
        return [[(None,) + _regional_delta(vol, None)]]
    if which == "steps":                                # three successive updates
        src, snk = _regional_delta(vol, _box(shape))
        return [[(stroke, 50.0, 0.0)], [(None, src, snk)],
                [(stroke[::2], -50.0, 0.0), (carve, rng.uniform(-10, 10, carve.size), rng.uniform(-10, 10, carve.size))]]
    raise ValueError(which)


_WHICH = ["soft_fg", "soft_bg", "negative", "mixed", "regional_box", "regional_all", "steps"]


def _check(vol, kind, regional, spacing, steps, env=None, conv=None):
    with _env(**(env or {})):
        g = _graph(vol, kind, regional, spacing)
        g.maxflow()
        done = []
        for step in steps:
            _apply(g, step, conv)
            done.append(step)
            e = g.maxflow()
            m = g.get_mask()
            oe, om, scale = _oracle(vol, kind, regional, spacing, done)
            bound = max(abs(oe), scale)
            assert numpy.array_equal(m, om), ("warm mask differs from the oracle", len(done), int((m != om).sum()))
            assert abs(e - oe) <= 1e-9 * bound, (len(done), e, oe, bound)
            ce, cm = _cold(vol, kind, regional, spacing, done)
            assert numpy.array_equal(m, cm), ("warm mask differs from the cold rebuild", len(done))
            assert abs(e - ce) <= 1e-12 * bound + 1e-10, (len(done), e, ce, bound)
        st = g.stats()
        assert st["seed_folds"] == sum(len(s) for s in steps) and st["ms_seeds"] > 0 and st["ms_seeds_host"] >= 0
        return g, e, g.get_mask().copy()


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("shape,kind,regional,dtype,spacing", [
    ((16, 16, 16), "difference_exponential", True, "float32", False),
    ((16, 16, 16), "difference_exponential", False, "float32", False),
    ((33, 17, 40), "difference_exponential", True, "float64", False),
    ((33, 17, 40), "difference_linear", True, "float32", False),
    ((64, 64, 64), "difference_exponential", True, "float32", False),
    ((64, 64, 64), "difference_exponential", False, "int16", False),
    ((24, 20, 32), "maximum_division", True, "float32", False),
    ((24, 20, 32), "difference_power", True, "float64", (1.0, 2.0, 0.5)),
    ((1, 48, 40), "difference_exponential", True, "float32", False),
])
def test_warm_tweights_match_from_scratch(shape, kind, regional, dtype, spacing, which):
    vol = _volume(shape, seed=3, dtype=dtype)
    _check(vol, kind, regional, spacing, _sequences(shape, vol, which))


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("shape", [(48, 40), (300,), (19, 27, 13)])
def test_warm_tweights_2d_1d_and_ragged(shape, which):
    vol = _vol_1d() if len(shape) == 1 else _volume(shape, seed=4, dtype="float32")
    _check(vol, "difference_exponential", True, False, _sequences(shape, vol, which))


@pytest.mark.parametrize("env", [dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_FIRST_TEST=1), dict(MEDPY_GC_DEBUG=1)])
def test_warm_tweights_solver_options(env):
    """MEDPY_GC_DEBUG=1 runs the conservation and invariant checks of every solve across the folds."""
    shape = (32, 32, 32)
    vol = _volume(shape, seed=5, dtype="float32")
    _check(vol, "difference_exponential", True, False, _sequences(shape, vol, "steps"), env=env)


def test_device_arrays_match_host_arrays_bit_for_bit():
    import torch
    shape = (20, 24, 32)
    vol = _volume(shape, seed=6, dtype="float32")
    steps = _sequences(shape, vol, "steps") + _sequences(shape, vol, "mixed")
    _, e_host, m_host = _check(vol, "difference_exponential", True, False, steps)
    _, e_dev, m_dev = _check(vol, "difference_exponential", True, False, steps, conv=lambda a: torch.from_numpy(a).cuda())
    assert e_dev == e_host and numpy.array_equal(m_dev, m_host)
    # float32 CUDA weights in the lattice shape, non-contiguous: widened and read in logical C order on the device
    src, snk = _regional_delta(vol, _box(shape))
    results = []
    for conv in (lambda a: a.astype(numpy.float32),
                 lambda a: torch.from_numpy(a.astype(numpy.float32)).cuda().transpose(0, 2).contiguous().transpose(0, 2)):
        g = _graph(vol, "difference_exponential", True, False)
        g.maxflow()
        g.add_tweights_warm(None, conv(src), conv(snk))
        results.append((g.maxflow(), g.get_mask().copy()))
    assert results[0][0] == results[1][0] and numpy.array_equal(results[0][1], results[1][1])


def test_hard_weights_equal_add_seeds_bit_for_bit():
    """add_tweights_warm(ids, 65535, 0) / (ids, 0, 65535) on a solved graph is add_seeds: the same energy bit for bit and
    the same mask."""
    shape = (33, 17, 40)
    vol = _volume(shape, seed=7, dtype="float32")
    stroke, carve = _ids(_stroke(shape)), _ids(_ball(shape, 0.3, 0.05))
    out = []
    for form in ("seeds", "tweights"):
        g = _graph(vol, "difference_exponential", True, False)
        g.maxflow()
        if form == "seeds":
            g.add_seeds(stroke, None)
            g.maxflow()
            g.add_seeds(None, carve)
        else:
            g.add_tweights_warm(stroke, 65535.0, 0.0)
            g.maxflow()
            g.add_tweights_warm(carve, 0.0, 65535.0)
        out.append((g.maxflow(), g.get_mask().copy()))
    assert out[0][0] == out[1][0] and numpy.array_equal(out[0][1], out[1][1])


def test_native_call_before_the_first_solve():
    """mgc_add_tweights_warm on a lazily built handle that was never solved: the build's source excess is still implicit
    in the tiles it listed; the result must still be the oracle's for the graph with the calls applied."""
    for shape, which in (((32, 32, 32), "negative"), ((33, 17, 40), "steps")):
        vol = _volume(shape, seed=8, dtype="float32")
        steps = _sequences(shape, vol, which)
        g = _graph(vol, "difference_exponential", True, False)
        for step in steps:
            for ids, src, snk in step:
                m = int(numpy.prod(shape)) if ids is None else len(ids)
                src = numpy.ascontiguousarray(numpy.broadcast_to(numpy.ravel(numpy.asarray(src, numpy.float64)), (m,)))
                snk = numpy.ascontiguousarray(numpy.broadcast_to(numpy.ravel(numpy.asarray(snk, numpy.float64)), (m,)))
                g._nat().add_tweights_warm(None if ids is None else numpy.asarray(ids, numpy.int64), src, snk)
        e, m = g.maxflow(), g.get_mask()
        oe, om, scale = _oracle(vol, "difference_exponential", True, False, steps)
        assert numpy.array_equal(m, om), int((m != om).sum())
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (e, oe)


def test_empty_and_zero_calls_keep_the_result():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    e = g.maxflow()
    m = g.get_mask().copy()
    g.add_tweights_warm(numpy.zeros(0, numpy.int64), 1.0, 2.0)
    g.add_tweights_warm([5, 9], 0.0, 0.0)
    g.add_tweights_warm(None, numpy.zeros(shape), 0.0)
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 0


def test_bad_ids_and_nan_leave_the_result():
    """An id out of range or a NaN / infinite weight is refused before anything changes the state: the previous result
    stays -- both through the Python checks and through the native ones."""
    shape = (16, 16, 16)
    n = 16 ** 3
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    g.add_tweights_warm(_ids(_ball(shape, 0.3, 0.1)), 0.0, 30.0)
    e = g.maxflow()
    m = g.get_mask().copy()
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_tweights_warm(numpy.array([0, n]), 1.0, 0.0)
    with pytest.raises(ValueError, match="NaN"):
        g.add_tweights_warm(numpy.array([0, 1]), numpy.array([1.0, numpy.nan]), 0.0)
    import torch
    with pytest.raises(ValueError, match="must all be host or all be device arrays"):
        g.add_tweights_warm(numpy.array([0, 1]), torch.ones(2, dtype=torch.float64, device="cuda"), 0.0)
    nat = g._nat()
    with pytest.raises(ValueError, match="out of range"):
        nat.add_tweights_warm(numpy.array([5, -1], numpy.int64), numpy.ones(2), numpy.zeros(2))
    with pytest.raises(ValueError, match="NaN or infinite"):
        nat.add_tweights_warm(numpy.array([5, 6], numpy.int64), numpy.ones(2), numpy.array([0.0, numpy.inf]))
    dense = numpy.ones(n)
    dense[n - 1] = numpy.nan
    with pytest.raises(ValueError, match="NaN or infinite"):
        nat.add_tweights_warm(None, dense, numpy.zeros(n))
    with pytest.raises(ValueError):
        nat.add_tweights_warm(None, numpy.ones(n - 1), numpy.zeros(n - 1))
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 1


@pytest.mark.parametrize("case", ["eager", "4d", "per_term", "sparse"])
def test_handles_without_warm_path_refuse(case):
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut.maxflow import GraphDouble
    env = {}
    shape = (12, 12, 16)
    if case == "eager":
        env = dict(MEDPY_GC_LAZY_CAPS=0)
    with _env(**env):
        if case == "sparse":
            g = GraphDouble(4, 4, sparse=True)
            g.add_tweights(0, 5.0, 0.0)
            g.add_tweights(3, 0.0, 5.0)
            g.sum_edge(0, 1, 1.0, 1.0)
            g.sum_edge(1, 3, 1.0, 1.0)
            g._solved = True
            g.maxflow()
            with pytest.raises(RuntimeError, match="reset.*rebuild"):
                g.add_tweights_warm([1], 1.0, 0.0)
            return
        if case == "4d":
            vol = _volume((6, 8, 8, 3), seed=1, dtype="float32")
            g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                     boundary_term_args=(vol["image"], vol["sigma"], False))
        elif case == "per_term":
            vol = _volume(shape, seed=1, dtype="float32")
            g = GraphDouble(int(numpy.prod(shape)), 0, shape=shape)
            g.add_regional_probability(vol["prob"], vol["alpha"], True)
            g.add_boundary(1, vol["image"], vol["sigma"], None, float("nan"))
            g.add_markers(vol["fg"], vol["bg"])
        else:
            vol = _volume(shape, seed=1, dtype="float32")
            g = _graph(vol, "difference_exponential", True, False)
        g.maxflow()
        with pytest.raises(RuntimeError, match="reset"):
            g.add_tweights_warm(numpy.array([3], numpy.int64), 1.0, 0.0)
        with pytest.raises(RuntimeError, match="reset"):
            g._nat().add_tweights_warm(None, numpy.ones(g.get_node_num()), numpy.zeros(g.get_node_num()))


def test_stats_count_the_grouping_kernels():
    """kernel_launches counts every kernel a call enqueues, cub's included.  List form: keys, heads and items kernels, the
    sort and the scan, the fold, the partial sum and the list rebuild; dense form: the flag and items kernels and the scan
    instead of the first five."""
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    before = g.stats()["kernel_launches"]
    g.add_tweights_warm(_ids(vol["fg"]), -3.0, 1.0)
    after = g.stats()["kernel_launches"]
    assert after - before >= 3 + 2 + 3
    g.maxflow()
    before = g.stats()["kernel_launches"]
    g.add_tweights_warm(None, *_regional_delta(vol, _box(shape)))
    assert g.stats()["kernel_launches"] - before >= 2 + 1 + 3


def test_config3_256_against_reference_bk():
    """BASELINE config 3 at 256^3: a soft stroke, then a regional update around blob 1, then one over the whole lattice --
    the mask after every step equal to the real reference BK's on the from-scratch graph with the calls so far (Hamming
    distance 0), the energy within 1e-9 of the bound in the module docstring."""
    from oracle import solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")
    shape = (256, 256, 256)
    vol = _volume(shape, seed=0, dtype="float32")
    stroke = _ids(_stroke(shape))
    steps = [[(stroke, 50.0, 0.0)], [(None,) + _regional_delta(vol, _box(shape))], [(None,) + _regional_delta(vol, None)]]
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    for k, step in enumerate(steps, 1):
        _apply(g, step)
        e = g.maxflow()
        m = g.get_mask()
        prob = _problem(vol, "difference_exponential", True, False)
        scale = _replay(prob, steps[:k])
        # solve_ref replays regional -> boundary -> fg -> bg itself: hand it the final t-links as one dense pass instead
        # (add_tweights(v, max(tr, 0), max(-tr, 0)) adds nothing to the constant), and add the constant here
        ref = dict(prob, src=numpy.maximum(prob["tr"], 0.0), snk=numpy.maximum(-prob["tr"], 0.0),
                   fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool))
        oe, om, _ = solvers.solve_ref(ref)
        oe += prob["flow_const"]
        assert int((m != om).sum()) == 0, k
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (k, e, oe, scale)
