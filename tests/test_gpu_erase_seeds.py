"""Seeds erased from a solved graph and solved warm (mgc_remove_seeds / GraphDouble.remove_seeds): after each step the mask
and energy must be those of the from-scratch graph with the same add_tweights sequence (erasing is add_tweights with
-65535) -- against the oracle (the BK restatement, or the real reference BK at 256^3) and against a cold GPU rebuild that
stages the same calls before its solve.

Energy bound: erasing cancels +-65535 constants, so the energy can be far smaller than the constants it was summed from,
and its rounding error scales with those.  Energies are compared relative to S = max(|E|, |build constant| + the sum over
the replayed add_tweights calls of 65535 + |t-link before the call|), which bounds the sum of the |add_tweights minima|
(|min(s, t)| <= 65535 + |tr|): 1e-9 S against the oracle, 1e-12 S + 1e-10 against the cold rebuild."""
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_seeds import _ball, _env, _graph, _ids, _stroke, _volume  # noqa: E402

pytestmark = pytest.mark.gpu

_CAP = {"add": 65535.0, "remove": -65535.0}


def _replay(prob, steps):
    """Every call of every step: add_tweights(v, cap, 0) per fg id in order, then add_tweights(v, 0, cap) per bg id,
    cap = +-65535; the k-th occurrence of an id within a call is applied in pass k (a voxel's t-link only depends on its
    own call sequence).  Returns S of the module docstring without |E|."""
    from oracle import energy_terms as et
    n = prob["tr"].size
    scale = abs(prob["flow_const"])
    for step in steps:
        for kind, fg, bg in step:
            cap = _CAP[kind]
            for ids, s, t in ((fg, cap, 0.0), (bg, 0.0, cap)):
                ids = numpy.asarray(ids, dtype=numpy.int64)
                if ids.size == 0:
                    continue
                counts = numpy.bincount(ids, minlength=n)
                for k in range(1, int(counts.max()) + 1):
                    where = counts >= k
                    scale += float(numpy.abs(prob["tr"][where]).sum()) + 65535.0 * int(where.sum())
                    prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], s, t, where=where)
    return scale


def _problem(vol, kind, regional, spacing):
    from oracle import energy_terms as et
    return et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]) if regional else None,
                            boundary=(kind, vol["image"], vol["sigma"], spacing))


def _oracle(vol, kind, regional, spacing, steps):
    from oracle import solvers
    prob = _problem(vol, kind, regional, spacing)
    scale = _replay(prob, steps)
    e, m = solvers.solve_port(prob)[:2]
    return e, m, scale


def _apply(g, step, conv=None):
    for kind, fg, bg in step:
        fg = numpy.asarray(fg, dtype=numpy.int64)
        bg = numpy.asarray(bg, dtype=numpy.int64)
        if conv is not None:
            fg, bg = conv(fg), conv(bg)
        getattr(g, kind + "_seeds")(fg, bg)


def _cold(vol, kind, regional, spacing, steps):
    """The same sequence built from scratch on the GPU: every call staged before the first solve."""
    g = _graph(vol, kind, regional, spacing)
    for step in steps:
        _apply(g, step)
    return g.maxflow(), g.get_mask()


def _sequences(shape, vol, which):
    """Steps of (kind, fg ids, bg ids) calls; the graph is solved after every step."""
    stroke = _ids(_stroke(shape))                       # across the background
    fgm, shell = _ids(vol["fg"]), _ids(vol["bg"])
    # inside blob 1, on its fg markers (a 1-D lattice: a run inside its fg markers)
    carve = _ids(_ball(shape, 0.3, 0.05)) if len(shape) > 1 else fgm[fgm.size // 4: fgm.size // 2]
    if which == "stroke":                               # add a stroke, then erase it
        return [[("add", stroke, carve)], [("remove", stroke, carve)]]
    if which == "markers":                              # part of the original fg markers and of the bg shell
        return [[("remove", fgm[::3], shell[::5])]]
    if which == "never":                                # seeds that were never added
        return [[("remove", stroke, carve)]]
    if which == "later":                                # erased a call after the one that added it; one id three times
        a, b = stroke[:2], carve[:2]
        return [[("add", a, b)], [("add", stroke[2:4], [])],
                [("remove", numpy.concatenate([a[:1], a[:1], a[:1], a[1:]]), b)]]
    if which == "both":                                 # one id in both lists of an erase call
        ids = numpy.concatenate([stroke[:3], fgm[:3], shell[:3]])
        return [[("remove", ids, ids)]]
    if which == "interleaved":                          # add and erase over three steps
        return [[("add", stroke, carve)],
                [("remove", stroke[::2], []), ("add", [], stroke[1::2])],
                [("remove", fgm[:4], carve[: max(1, carve.size // 2)]), ("add", stroke[::2][:3], [])]]
    raise ValueError(which)


_WHICH = ["stroke", "markers", "never", "later", "both", "interleaved"]


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
        return g


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
def test_warm_erase_matches_from_scratch(shape, kind, regional, dtype, spacing, which):
    vol = _volume(shape, seed=3, dtype=dtype)
    _check(vol, kind, regional, spacing, _sequences(shape, vol, which))


def _vol_1d():
    from medpy_b200 import synthetic
    rng = numpy.random.default_rng(4)
    x = numpy.arange(300)
    image = (100.0 * ((x >= 90) & (x < 210)) + rng.normal(0, 10, 300)).astype(numpy.float32)
    fg = numpy.zeros(300, bool)
    fg[140:160] = True
    bg = numpy.zeros(300, bool)
    bg[[0, 1, 298, 299]] = True
    prob = (1.0 / (1.0 + numpy.exp(-(image - 50.0) / 15.0))).astype(numpy.float32)
    return dict(image=image, fg=fg, bg=bg, prob=prob, alpha=0.1, sigma=synthetic.rms_neighbour_difference(image))


@pytest.mark.parametrize("which", _WHICH)
@pytest.mark.parametrize("shape", [(48, 40), (300,)])
def test_warm_erase_2d_and_1d(shape, which):
    vol = _vol_1d() if len(shape) == 1 else _volume(shape, seed=4, dtype="float32")
    _check(vol, "difference_exponential", True, False, _sequences(shape, vol, which))


@pytest.mark.parametrize("shape", [(32, 32, 32), (33, 17, 40), (48, 40)])
def test_round_trip_restores_the_pre_stroke_result(shape):
    """Add a stroke, solve, erase it, solve: the mask of the graph before the stroke, its energy to 1e-9 relative."""
    vol = _volume(shape, seed=7, dtype="float32")
    stroke, carve = _ids(_stroke(shape)), _ids(_ball(shape, 0.3, 0.05))
    g = _graph(vol, "difference_exponential", True, False)
    e0 = g.maxflow()
    m0 = g.get_mask().copy()
    g.add_seeds(stroke, carve)
    e1 = g.maxflow()
    assert e1 != e0
    g.remove_seeds(stroke, carve)
    e2 = g.maxflow()
    assert numpy.array_equal(g.get_mask(), m0)
    assert abs(e2 - e0) <= 1e-9 * abs(e0), (e2, e0)


@pytest.mark.parametrize("env", [dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_FIRST_TEST=1), dict(MEDPY_GC_DEBUG=1)])
def test_warm_erase_solver_options(env):
    """MEDPY_GC_DEBUG=1 runs the conservation and invariant checks of every solve across the erase folds."""
    shape = (32, 32, 32)
    vol = _volume(shape, seed=5, dtype="float32")
    _check(vol, "difference_exponential", True, False, _sequences(shape, vol, "interleaved"), env=env)


def test_device_ids_and_masks():
    import torch
    shape = (20, 24, 32)
    vol = _volume(shape, seed=6, dtype="float32")
    _check(vol, "difference_exponential", True, False, _sequences(shape, vol, "interleaved"),
           conv=lambda a: torch.from_numpy(a).cuda())
    # boolean masks (Fortran-strided on the host, a CUDA tensor on the device) give the ids in logical C order
    carve = _ball(shape, 0.3, 0.05)
    fgm = vol["fg"] & (numpy.arange(vol["fg"].size).reshape(shape) % 3 == 0)
    results = []
    for form in (numpy.asfortranarray, lambda a: torch.from_numpy(a).cuda(), _ids):
        g = _graph(vol, "difference_exponential", True, False)
        g.maxflow()
        g.add_seeds(bg=form(carve))
        g.maxflow()
        g.remove_seeds(fg=form(fgm), bg=form(carve))
        results.append((g.maxflow(), g.get_mask().copy()))
    for e, m in results[1:]:
        assert e == results[0][0] and numpy.array_equal(m, results[0][1])


def test_native_remove_seeds_before_the_first_solve():
    """mgc_remove_seeds on a lazily built handle that was never solved: the build's source excess is still implicit in
    the tiles it listed; the result must still be the oracle's for the graph with the calls applied."""
    for shape, which in (((32, 32, 32), "markers"), ((33, 17, 40), "interleaved")):
        vol = _volume(shape, seed=8, dtype="float32")
        steps = _sequences(shape, vol, which)
        g = _graph(vol, "difference_exponential", True, False)
        for step in steps:
            for kind, fg, bg in step:
                getattr(g._nat(), kind + "_seeds")(numpy.asarray(fg, numpy.int64), numpy.asarray(bg, numpy.int64))
        e, m = g.maxflow(), g.get_mask()
        oe, om, scale = _oracle(vol, "difference_exponential", True, False, steps)
        assert numpy.array_equal(m, om), int((m != om).sum())
        assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (e, oe)


def test_empty_call_keeps_the_result():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    e = g.maxflow()
    m = g.get_mask().copy()
    g.remove_seeds(numpy.zeros(0, numpy.int64), None)
    g.remove_seeds()
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 0


def test_out_of_range_ids_leave_the_result():
    """An id out of range is refused before anything changes the state: the previous result stays."""
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    g.add_seeds(bg=_ids(_ball(shape, 0.3, 0.1)))
    e = g.maxflow()
    m = g.get_mask().copy()
    with pytest.raises(ValueError, match="Invalid node id"):
        g.remove_seeds(numpy.array([0, 4096]))
    with pytest.raises(ValueError):
        g._nat().remove_seeds(numpy.array([5, -1], numpy.int64), None)
    with pytest.raises(ValueError):
        g._nat().remove_seeds(numpy.array([5], numpy.int64), numpy.array([7, 4096], numpy.int64))
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)
    assert g.stats()["seed_folds"] == 1


@pytest.mark.parametrize("case", ["eager", "4d", "per_term"])
def test_handles_without_warm_path_refuse(case):
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut.maxflow import GraphDouble
    env = {}
    shape = (12, 12, 16)
    if case == "eager":
        env = dict(MEDPY_GC_LAZY_CAPS=0)
    with _env(**env):
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
            g.remove_seeds(numpy.array([3], numpy.int64), None)
        with pytest.raises(RuntimeError, match="reset"):
            g._nat().remove_seeds(numpy.array([3], numpy.int64), None)


def test_config3_256_against_reference_bk():
    """BASELINE config 3 at 256^3: three warm steps -- a stroke and the carve ball added, the carve ball erased, part of
    the markers erased -- the mask after every step equal to the real reference BK's on the from-scratch graph with the
    calls so far (Hamming distance 0), the energy within 1e-9 of the bound in the module docstring."""
    from oracle import solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")
    shape = (256, 256, 256)
    vol = _volume(shape, seed=0, dtype="float32")
    stroke, carve = _ids(_stroke(shape)), _ids(_ball(shape, 0.3, 0.05))
    fgm, shell = _ids(vol["fg"]), _ids(vol["bg"])
    steps = [[("add", stroke, carve)], [("remove", [], carve)], [("remove", fgm[::4], shell[::7])]]
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


def test_stats_count_the_grouping_kernels():
    """kernel_launches counts every kernel a seed call enqueues, the ones cub's sort and scan launch included: at least
    the three grouping kernels, one each for the sort and the scan, the fold, the partial sum and the list rebuild."""
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    before = g.stats()["kernel_launches"]
    g.remove_seeds(fg=_ids(vol["fg"]))
    assert g.stats()["kernel_launches"] - before >= 3 + 2 + 3
