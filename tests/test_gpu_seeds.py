"""Seeds added to a solved graph and solved warm (mgc_add_seeds / GraphDouble.add_seeds): the mask and energy after each
refinement must be those of the from-scratch graph with the same add_tweights sequence -- against the oracle (the BK
restatement, or the real reference BK at 256^3) and against a cold GPU rebuild of that sequence."""
import os

import numpy
import pytest

pytestmark = pytest.mark.gpu


class _env:
    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kw}
        for k, v in self.kw.items():
            os.environ[k] = str(v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


_LINEAR = ("difference_linear", "maximum_linear")


def _volume(shape, seed, dtype):
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=seed, integer=dtype == "int16")
    if dtype == "float64":
        vol["image"] = vol["image"].astype(numpy.float64)
    elif dtype == "int16":
        vol["image"] = vol["image"].astype(numpy.int16)
    return vol


def _boundary_args(vol, kind, spacing):
    return (vol["image"], spacing) if kind in _LINEAR else (vol["image"], vol["sigma"], spacing)


def _graph(vol, kind, regional, spacing):
    import medpy_b200.graphcut as gc
    kw = dict(boundary_term=getattr(gc.energy_voxel, "boundary_" + kind), boundary_term_args=_boundary_args(vol, kind, spacing))
    if regional:
        kw.update(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=(vol["prob"], vol["alpha"]))
    return gc.graph_from_voxels(vol["fg"], vol["bg"], **kw)


def _oracle(vol, kind, regional, spacing, steps):
    from oracle import energy_terms as et, solvers
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]) if regional else None,
                            boundary=(kind, vol["image"], vol["sigma"], spacing))
    _replay(prob, steps)
    return solvers.solve_port(prob)[:2]


def _replay(prob, steps):
    """add_tweights(v, 65535, 0) per fg id in order, then add_tweights(v, 0, 65535) per bg id, for every step; the
    k-th occurrence of an id is applied in pass k (a voxel's t-link only depends on its own call sequence)."""
    from oracle import energy_terms as et
    n = prob["tr"].size
    for fg, bg in steps:
        for ids, s, t in ((fg, 65535.0, 0.0), (bg, 0.0, 65535.0)):
            ids = numpy.asarray(ids, dtype=numpy.int64)
            if ids.size == 0:
                continue
            counts = numpy.bincount(ids, minlength=n)
            for k in range(1, int(counts.max()) + 1):
                prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], s, t, where=counts >= k)


def _cold(vol, kind, regional, spacing, steps):
    """The same sequence built from scratch on the GPU: seeds staged before the first solve."""
    g = _graph(vol, kind, regional, spacing)
    for fg, bg in steps:
        g.add_seeds(numpy.asarray(fg, dtype=numpy.int64), numpy.asarray(bg, dtype=numpy.int64))
    return g.maxflow(), g.get_mask()


def _ids(mask):
    return numpy.flatnonzero(numpy.ascontiguousarray(mask))


def _ball(shape, centre, radius):
    from medpy_b200 import synthetic
    return synthetic._ball_mask(shape, (centre,), radius, min_radius=1.0)


def _stroke(shape):
    """fg line along the last axis through the background between the two blobs (centre of the lattice)."""
    m = numpy.zeros(shape, dtype=bool)
    idx = tuple(s // 2 for s in shape[:-1])
    x = shape[-1]
    m[idx + (slice(int(0.4 * x), max(int(0.6 * x), int(0.4 * x) + 1)),)] = True
    return m


def _refinements(shape, vol, which):
    """Refinement steps: lists of (fg ids, bg ids)."""
    carve = _ids(_ball(shape, 0.3, 0.05))              # bg ball inside blob 1
    stroke = _ids(_stroke(shape))                       # fg stroke across the background
    if which == "carve":
        return [([], carve)]
    if which == "stroke":
        return [(stroke, [])]
    if which == "both":
        return [(stroke, carve)]
    if which == "three":
        return [([], carve), (stroke, []), (carve[: max(1, carve.size // 2)], stroke[::2])]
    if which == "mixed":
        # fg on sink voxels that absorbed flow (the shell), fg and bg on one voxel, one id three times,
        # fg on a voxel whose -tr > 65535 after two bg seeds, seeds in tiles the first solve never reached
        shell = _ids(vol["bg"])
        far = _ids(_ball(shape, 0.9, 0.03))
        twice = stroke[:1]
        return [(numpy.concatenate([shell[:5], stroke[:3]]), numpy.concatenate([stroke[:3], carve[:1], carve[:1], carve[:1]])),
                ([], numpy.concatenate([twice, twice])),
                (numpy.concatenate([twice, far]), far[:2])]
    raise ValueError(which)


def _check(vol, kind, regional, spacing, steps, env=None, device_ids=False):
    with _env(**(env or {})):
        g = _graph(vol, kind, regional, spacing)
        g.maxflow()
        done = []
        for fg, bg in steps:
            fg = numpy.asarray(fg, dtype=numpy.int64)
            bg = numpy.asarray(bg, dtype=numpy.int64)
            if device_ids:
                import torch
                g.add_seeds(torch.from_numpy(fg).cuda(), torch.from_numpy(bg).cuda())
            else:
                g.add_seeds(fg, bg)
            done.append((fg, bg))
            e = g.maxflow()
            m = g.get_mask()
            oe, om = _oracle(vol, kind, regional, spacing, done)
            assert numpy.array_equal(m, om), ("warm mask differs from the oracle", int((m != om).sum()))
            assert abs(e - oe) <= 1e-9 * max(abs(oe), 1.0), (e, oe)
            ce, cm = _cold(vol, kind, regional, spacing, done)
            assert numpy.array_equal(m, cm), "warm mask differs from the cold rebuild"
            assert abs(e - ce) <= 1e-12 * max(abs(ce), 1.0) + 1e-10, (e, ce)
        st = g.stats()
        assert st["seed_folds"] == len(steps) and st["ms_seeds"] > 0 and st["ms_seeds_host"] >= 0
        return g


@pytest.mark.parametrize("shape,kind,regional,dtype,spacing,which", [
    ((16, 16, 16), "difference_exponential", True, "float32", False, "carve"),
    ((16, 16, 16), "difference_exponential", False, "float32", False, "stroke"),
    ((33, 17, 40), "difference_exponential", True, "float64", False, "both"),
    ((33, 17, 40), "difference_linear", True, "float32", False, "mixed"),
    ((64, 64, 64), "difference_exponential", True, "float32", False, "three"),
    ((64, 64, 64), "difference_exponential", False, "int16", False, "mixed"),
    ((24, 20, 32), "maximum_division", True, "float32", False, "both"),
    ((24, 20, 32), "difference_power", True, "float64", (1.0, 2.0, 0.5), "mixed"),
    ((1, 48, 40), "difference_exponential", True, "float32", False, "three"),
])
def test_warm_refinement_matches_from_scratch(shape, kind, regional, dtype, spacing, which):
    vol = _volume(shape, seed=3, dtype=dtype)
    _check(vol, kind, regional, spacing, _refinements(shape, vol, which))


def test_warm_refinement_2d_and_1d():
    from medpy_b200 import synthetic
    for shape in ((48, 40), (300,)):
        if len(shape) == 1:
            rng = numpy.random.default_rng(4)
            image = (100.0 * ((numpy.arange(300) >= 90) & (numpy.arange(300) < 210)) + rng.normal(0, 10, 300)).astype(numpy.float32)
            fg = numpy.zeros(300, bool)
            fg[140:160] = True
            bg = numpy.zeros(300, bool)
            bg[[0, 299]] = True
            prob = (1.0 / (1.0 + numpy.exp(-(image - 50.0) / 15.0))).astype(numpy.float32)
            vol = dict(image=image, fg=fg, bg=bg, prob=prob, alpha=0.1, sigma=synthetic.rms_neighbour_difference(image))
        else:
            vol = _volume(shape, seed=4, dtype="float32")
        n = int(numpy.prod(shape))
        rng = numpy.random.default_rng(1)
        steps = [(rng.integers(0, n, 6), rng.integers(0, n, 6)), ([], rng.integers(0, n, 3))]
        _check(vol, "difference_exponential", True, False, steps)


@pytest.mark.parametrize("env", [dict(MEDPY_GC_PARTIAL_RESET=0), dict(MEDPY_GC_FIRST_TEST=1), dict(MEDPY_GC_DEBUG=1)])
def test_warm_refinement_solver_options(env):
    shape = (32, 32, 32)
    vol = _volume(shape, seed=5, dtype="float32")
    _check(vol, "difference_exponential", True, False, _refinements(shape, vol, "three"), env=env)


def test_device_ids_and_masks():
    import torch
    shape = (20, 24, 32)
    vol = _volume(shape, seed=6, dtype="float32")
    _check(vol, "difference_exponential", True, False, _refinements(shape, vol, "both"), device_ids=True)
    # boolean masks (Fortran-strided on the host, a CUDA tensor on the device) give the ids in logical C order
    carve = _ball(shape, 0.3, 0.05)
    g1 = _graph(vol, "difference_exponential", True, False)
    g1.maxflow()
    g1.add_seeds(bg=numpy.asfortranarray(carve))
    g2 = _graph(vol, "difference_exponential", True, False)
    g2.maxflow()
    g2.add_seeds(bg=torch.from_numpy(carve).cuda())
    assert g1.maxflow() == g2.maxflow()
    assert numpy.array_equal(g1.get_mask(), g2.get_mask())


def test_empty_call_keeps_the_result():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    e = g.maxflow()
    m = g.get_mask().copy()
    g.add_seeds(numpy.zeros(0, numpy.int64), None)
    g.add_seeds()
    assert g.maxflow() == e
    assert numpy.array_equal(g.get_mask(), m)


def test_out_of_range_ids_raise_value_error():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    with pytest.raises(ValueError, match="Invalid node id"):
        g.add_seeds(numpy.array([0, 4096]))
    with pytest.raises(ValueError):
        g._nat().add_seeds(numpy.array([-1], numpy.int64), None)


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
            g.add_seeds(numpy.array([3], numpy.int64), None)
        with pytest.raises(RuntimeError, match="reset"):
            g._nat().add_seeds(numpy.array([3], numpy.int64), None)


def test_term_entry_points_still_refuse_after_a_fold():
    shape = (16, 16, 16)
    vol = _volume(shape, seed=2, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    g.add_seeds(bg=numpy.array([100], numpy.int64))
    g.maxflow()
    with pytest.raises(RuntimeError, match="reset"):
        g._nat().add_tweights_dense(numpy.zeros(shape), numpy.zeros(shape))


def test_config3_256_against_reference_bk():
    """BASELINE config 3 at 256^3: three warm refinements, each mask equal to the real reference BK's on the enlarged
    graph (Hamming distance 0)."""
    from oracle import energy_terms as et, solvers
    if not solvers.have_ref():
        pytest.skip("oracle/_ref (the reference BK) was not built")
    shape = (256, 256, 256)
    vol = _volume(shape, seed=0, dtype="float32")
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    steps = _refinements(shape, vol, "three")
    done = []
    for fg, bg in steps:
        g.add_seeds(numpy.asarray(fg, numpy.int64), numpy.asarray(bg, numpy.int64))
        done.append((fg, bg))
        e = g.maxflow()
        m = g.get_mask()
    # the reference BK on the from-scratch graph with all seeds as dense t-weights after the markers
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    _replay(prob, done)
    # solve_ref replays regional -> boundary -> fg -> bg itself: hand it the final t-links as one dense pass instead
    # (add_tweights(v, max(tr, 0), max(-tr, 0)) adds nothing to the constant), and add the constant here
    ref = dict(prob, src=numpy.maximum(prob["tr"], 0.0), snk=numpy.maximum(-prob["tr"], 0.0),
               fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool))
    oe, om, _ = solvers.solve_ref(ref)
    oe += prob["flow_const"]
    assert int((m != om).sum()) == 0
    assert abs(e - oe) <= 1e-9 * abs(oe), (e, oe)


def test_native_add_seeds_before_the_first_solve():
    """mgc_add_seeds on a lazily built handle that was never solved: the build's source excess is still implicit in the
    tiles it listed; the result must still be the oracle's for the enlarged graph."""
    for shape, which in (((32, 32, 32), "both"), ((33, 17, 40), "mixed")):
        vol = _volume(shape, seed=8, dtype="float32")
        steps = _refinements(shape, vol, which)
        g = _graph(vol, "difference_exponential", True, False)
        done = []
        for fg, bg in steps:
            g._nat().add_seeds(numpy.asarray(fg, numpy.int64), numpy.asarray(bg, numpy.int64))
            done.append((fg, bg))
        e, m = g.maxflow(), g.get_mask()
        oe, om = _oracle(vol, "difference_exponential", True, False, done)
        assert numpy.array_equal(m, om), int((m != om).sum())
        assert abs(e - oe) <= 1e-9 * abs(oe), (e, oe)


def test_same_voxel_folded_in_successive_calls():
    """A voxel seeded fg in two successive calls, then bg in two more: the source residual a fold leaves must read
    back for the next fold.  Inside the foreground (no net inflow) it reads back exactly; on a background voxel that
    absorbed flow to one rounding.  Warm and cold stay within 1e-13 relative at every step."""
    shape = (24, 24, 24)
    vol = _volume(shape, seed=9, dtype="float32")
    inside = int(numpy.flatnonzero(vol["fg"])[len(numpy.flatnonzero(vol["fg"])) // 2])
    outside = int(numpy.ravel_multi_index((12, 12, 12), shape))
    ids = numpy.array([inside, outside], numpy.int64)
    steps = [(ids, []), (ids, []), ([], ids), ([], ids)]
    g = _graph(vol, "difference_exponential", True, False)
    g.maxflow()
    done = []
    for fg, bg in steps:
        g.add_seeds(numpy.asarray(fg, numpy.int64), numpy.asarray(bg, numpy.int64))
        done.append((fg, bg))
        e, m = g.maxflow(), g.get_mask()
        ce, cm = _cold(vol, "difference_exponential", True, False, done)
        oe, om = _oracle(vol, "difference_exponential", True, False, done)
        assert numpy.array_equal(m, cm) and numpy.array_equal(m, om)
        assert abs(e - ce) <= 1e-13 * abs(ce), (len(done), e, ce)
        assert abs(e - oe) <= 1e-9 * abs(oe), (len(done), e, oe)
