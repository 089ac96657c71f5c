"""Warm edits on z-slab handles (run on an H100 with ``-m gpu``): seeds, t-link and n-link increments folded into N solved
slab handles of one lattice on one GPU, then re-solved warm under both exchange protocols of test_gpu_slabs.py.  After
every re-solve the mask and the energy must equal those of a single-lattice warm handle given the same edits in global
ids, and those of BK (``oracle.solvers.solve_port``) on the edited graph.  Tolerances are those of test_gpu_slabs.py:
masks identical, energies within 1e-9 relative, exactly equal for integer capacities.

Edits are the steps of test_gpu_warm_nweights.py in GLOBAL ids: ("s", fg, bg) / ("r", fg, bg) seeds added / erased,
("t", ids or None, src, snk) t-link calls, ("n", i, j, cap, rev) and ("d", axis, fwd, bwd) n-link increments.  Each
slab gets them in its own local ids (its planes plus its ghost planes, C order), ghost entries included: the handle
itself applies only what it owns, so an entry in a ghost plane must change nothing and an axis-0 pair across a border
is applied half on each side.

How SlabSolver maps global arguments to these local calls is tested on the CPU (test_host_slab_warm.py); the NCCL
transport by the >= 2-GPU test at the end."""
import copy
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_push_window import _env  # noqa: E402
from test_gpu_slabs import (PROTOCOLS, SLAB4_OPTIONS, Slabs, _bounds, check, reference, relay_case,  # noqa: E402
                            voxel_case, weak_boundary_case)
from test_gpu_warm_nweights_remove import _replay  # noqa: E402

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------------
# drivers: N warm slab handles, and one warm single-lattice handle of the same graph
# ------------------------------------------------------------------------------------------------------
def _opt_warm():
    from medpy_b200 import _lib
    return _lib._mgc.OPT_WARM


class Single(Slabs):
    """One ordinary (not z-slab) handle of the whole lattice, built by Slabs.build and solved with maxflow."""

    def __init__(self, shape):
        import torch
        from medpy_b200 import _lib
        self.torch = torch
        self.shape = tuple(int(s) for s in shape)
        self.bounds = [(0, self.shape[0])]
        self.hs = [_lib.Graph(list(self.shape), 0)]
        self.n = 1

    def solve(self, protocol=None):
        h = self.hs[0]
        return h.maxflow(), h.get_mask().copy()


def _make(kind, shape, bounds, c, form):
    s = Single(shape) if kind == "single" else Slabs(shape, bounds)
    for h in s.hs:
        h.set_option(_opt_warm(), 1)
    s.build(c, form)
    return s


def _span(s, r):
    """Local planes [a, b) of slab r in global plane numbers (its planes plus its ghost planes)."""
    z0, z1 = s.bounds[r]
    return z0 - (1 if z0 > 0 else 0), z1 + (1 if z1 < s.shape[0] else 0)


def _i64(x):
    return numpy.ascontiguousarray(numpy.asarray(x, numpy.int64).ravel())


def _f64(x, like):
    return numpy.ascontiguousarray(numpy.broadcast_to(numpy.asarray(x, numpy.float64), like.shape))


def apply_local(s, r, op):
    """One global edit on slab r (or on a Single) in its local ids, every entry of its local lattice included."""
    h = s.hs[r]
    a, b = _span(s, r)
    P = int(numpy.prod(s.shape[1:]))
    lo, hi = a * P, b * P
    inside = lambda x: (x >= lo) & (x < hi)  # noqa: E731
    k = op[0]
    if k in "sr":
        ids = [None if x is None else _i64(x) for x in op[1:3]]
        ids = [None if x is None else numpy.ascontiguousarray(x[inside(x)] - lo) for x in ids]
        (h.add_seeds if k == "s" else h.remove_seeds)(ids[0], ids[1])
    elif k == "t" and op[1] is None:
        flat = lambda w: numpy.ascontiguousarray(numpy.broadcast_to(numpy.asarray(w, numpy.float64), s.shape).ravel()[lo:hi])  # noqa: E731
        h.add_tweights_warm(None, flat(op[2]), flat(op[3]))
    elif k == "t":
        ids = _i64(op[1])
        src, snk = _f64(op[2], ids), _f64(op[3], ids)
        sel = inside(ids)
        h.add_tweights_warm(numpy.ascontiguousarray(ids[sel] - lo), numpy.ascontiguousarray(src[sel]),
                            numpy.ascontiguousarray(snk[sel]))
    elif k == "n":
        i, j = _i64(op[1]), _i64(op[2])
        cap, rev = _f64(op[3], i), _f64(op[4], i)
        sel = inside(i) & inside(j)
        h.add_nweights_warm(*(numpy.ascontiguousarray(x[sel] - (lo if x.dtype == numpy.int64 else 0)) for x in (i, j, cap, rev)))
    elif k in ("d", "rd"):
        fold = h.add_nweights_dense_warm if k == "d" else h.remove_nweights_dense_warm
        fold(op[1], numpy.ascontiguousarray(op[2][a:b]), numpy.ascontiguousarray(op[3][a:b]))
    elif k == "rn":
        i, j = _i64(op[1]), _i64(op[2])
        sel = inside(i) & inside(j)
        h.remove_nweights_warm(numpy.ascontiguousarray(i[sel] - lo), numpy.ascontiguousarray(j[sel] - lo),
                               _f64(op[3], i)[sel].copy(), _f64(op[4], i)[sel].copy())
    else:
        raise AssertionError(op)


def apply(s, step):
    for op in step:
        for r in range(s.n):
            apply_local(s, r, op)


def _same(a, b, exact):
    (ea, ma), (eb, mb) = a, b
    assert numpy.array_equal(ma, mb), ("masks differ", int((ma != mb).sum()))
    if exact:
        assert ea == eb, (ea, eb)
    else:
        assert abs(ea - eb) <= 1e-9 * max(1.0, abs(eb)), (ea, eb)


def edited(c, steps):
    """The case with its BK problem replayed through every step so far."""
    prob = copy.deepcopy(reference(c))
    _replay(prob, steps)
    return dict(c, prob_ref=prob)


def run_steps(c, bounds, protocol, form, steps, exact=False, env=None, before=()):
    """Build warm slabs and a warm single handle, fold `before` ahead of the first solve, then solve, and fold and
    re-solve every step; after each solve: slabs == single == BK on the edited graph."""
    shape = c["shape"]
    with _env(**(env or {})):
        s = _make("slabs", shape, bounds, c, form)
        one = _make("single", shape, bounds, c, form)
        done = list(before)
        for x in (s, one):
            apply(x, [op for step in before for op in step])
        res = None
        for k in range(len(steps) + 1):
            if k:
                apply(s, steps[k - 1])
                apply(one, steps[k - 1])
                done.append(steps[k - 1])
            res = s.solve(protocol)
            _same(res, one.solve(), exact)
            check(res[0], res[1], edited(c, done), exact=exact)
        st = [h.stats() for h in s.hs]
        assert sum(x["seed_folds"] for x in st) >= 1 and sum(x["ms_seeds"] for x in st) > 0
    return s, res


# ------------------------------------------------------------------------------------------------------
# edits in global ids
# ------------------------------------------------------------------------------------------------------
def _flat(shape, *coords):
    return int(numpy.ravel_multi_index(coords, shape))


def border_planes(bounds):
    """Every plane on either side of a slab border."""
    zs = set()
    for a, _ in bounds[1:]:
        zs.update((a - 1, a))
    return sorted(zs)


def stroke_ids(shape, planes, rng, frac=0.15):
    """A random stroke over the given axis-0 planes."""
    m = numpy.zeros(shape, bool)
    for z in planes:
        m[z] = rng.random(shape[1:]) < frac
    return numpy.flatnonzero(m)


def axis0_pairs(shape, planes):
    """Every axis-0 pair (p, p + plane) with p on one of `planes`: the pairs across each border when `planes` are the
    planes below the borders."""
    P = int(numpy.prod(shape[1:]))
    lo = numpy.concatenate([numpy.arange(z * P, (z + 1) * P) for z in planes if z + 1 < shape[0]])
    return lo, lo + P


def inner_pairs(shape, rng, count):
    """Random pairs along the last axis."""
    n = int(numpy.prod(shape))
    lo = rng.integers(0, n, size=count)
    lo = lo[(lo % shape[-1]) + 1 < shape[-1]]
    return lo, lo + 1


def steps_for(shape, bounds, seed):
    """The edit sequence of the layout tests: seeds on both border planes, t-link lists across borders, increments on
    every pair across every border (listed from either end), dense axis-0 and last-axis increments, dense t-links,
    and an erase."""
    rng = numpy.random.default_rng(seed)
    Z = shape[0]
    bp = border_planes(bounds) or [Z // 2 - 1, Z // 2]
    fg = stroke_ids(shape, bp, rng)
    bg = stroke_ids(shape, [Z - 2], rng, 0.3)
    bg = numpy.setdiff1d(bg, fg)
    tl = stroke_ids(shape, bp + [0, Z - 1], rng, 0.2)
    lo, hi = axis0_pairs(shape, [a - 1 for a, _ in bounds[1:]] or [Z // 2])
    flip = rng.random(lo.size) < 0.5
    i, j = numpy.where(flip, hi, lo), numpy.where(flip, lo, hi)
    li, lj = inner_pairs(shape, rng, 200)
    dense0 = [numpy.where(rng.random(shape) < 0.2, rng.random(shape) * 3.0, 0.0) for _ in range(2)]
    dense2 = [numpy.where(rng.random(shape) < 0.1, rng.random(shape) * 2.0, 0.0) for _ in range(2)]
    dsrc = numpy.where(rng.random(shape) < 0.05, rng.random(shape) * 4.0, 0.0)
    dsnk = numpy.where(rng.random(shape) < 0.05, rng.random(shape) * 4.0, 0.0)
    return [
        [("s", fg, bg)],
        [("t", tl, rng.random(tl.size) * 8.0 - 4.0, rng.random(tl.size) * 8.0 - 4.0)],
        [("n", numpy.concatenate([i, li]), numpy.concatenate([j, lj]), rng.random(i.size + li.size) * 5.0,
          rng.random(i.size + li.size) * 5.0)],
        [("d", 0, dense0[0], dense0[1]), ("t", None, dsrc, dsnk)],
        [("d", len(shape) - 1, dense2[0], dense2[1]), ("r", fg[::3], None)],
    ]


# ------------------------------------------------------------------------------------------------------
# layouts: N = 1, 2, 3, 5 and one plane per slab; ragged splits on and off the 8-plane tile boundary
# ------------------------------------------------------------------------------------------------------
LAYOUTS = {
    "n1": ((24, 20, 22), [(0, 24)]),
    "n2": ((24, 20, 22), _bounds(24, 2)),
    "n3_tile": ((24, 20, 22), [(0, 8), (8, 16), (16, 24)]),
    "n5": ((30, 16, 18), _bounds(30, 5)),
    "ragged_one_plane": ((24, 20, 21), [(0, 7), (7, 8), (8, 13), (13, 24)]),
    "every_plane": ((10, 16, 18), _bounds(10, 10)),
}


@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_warm_edits_on_layouts(layout, protocol):
    shape, bounds = LAYOUTS[layout]
    c = voxel_case(shape, seed=5)
    run_steps(c, bounds, protocol, "fused", steps_for(shape, bounds, 1))


@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("form", ["fused", "terms", "device"])
def test_warm_edits_under_build_forms(form, protocol):
    shape = (26, 20, 24)
    bounds = [(0, 9), (9, 10), (10, 17), (17, 26)]
    c = voxel_case(shape, seed=9)
    run_steps(c, bounds, protocol, form, steps_for(shape, bounds, 2))


@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("shape,bounds", [((20, 12, 16, 9), _bounds(20, 3)), ((17, 10, 8, 6), [(0, 4), (4, 5), (5, 8), (8, 17)])])
def test_warm_edits_on_4d_slabs(shape, bounds, protocol):
    c = voxel_case(shape, seed=29)
    run_steps(c, bounds, protocol, "terms", steps_for(shape, bounds, 3))


@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("opt", list(SLAB4_OPTIONS) + ["debug"])
@pytest.mark.parametrize("nd", [3, 4])
def test_warm_edits_under_solver_options(nd, opt, protocol):
    env = dict(MEDPY_GC_DEBUG=1) if opt == "debug" else SLAB4_OPTIONS[opt]
    if nd == 3:
        shape, bounds, form = (32, 24, 24), [(0, 12), (12, 13), (13, 24), (24, 32)], "fused"
    else:
        shape, bounds, form = (24, 16, 16, 12), _bounds(24, 5), "terms"
    c = voxel_case(shape, seed=31)
    run_steps(c, bounds, protocol, form, steps_for(shape, bounds, 4), env=env)


# ------------------------------------------------------------------------------------------------------
# integer capacities (exact energies): relay across slabs, a cut moved into another slab, edits before the first solve
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("n", [3, 5])
def test_seed_relayed_across_slabs(n, protocol):
    """A fg seed added in slab 0 outside the tube: its only way to the sink (the last plane) runs through every slab.
    Then the tube's weak end, in the last slab, gets increments that move the cut there."""
    shape = (32, 12, 12)
    bounds = _bounds(shape[0], n)
    c, tube = relay_case(shape, n)
    fg = numpy.zeros(shape, bool)
    fg[1, 0:2, 0:2] = True
    z = shape[0] * 3 // 4 - 1           # the tube's last plane: its axis-0 arcs to the next plane are weak
    lo, hi = axis0_pairs(shape, [z])
    tube_end = tube[z].ravel()
    steps = [[("s", numpy.flatnonzero(fg), None)],
             [("n", lo[tube_end], hi[tube_end], 2000.0, 2000.0)]]
    s, (e, m) = run_steps(c, bounds, protocol, "caps", steps, exact=True)
    assert m[1, 0, 0] == 1


@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("nd", [3, 4])
def test_edits_before_the_first_solve(nd, protocol):
    """Folds on built, unsolved warm slabs take the record first; the first solve then starts from the edited state."""
    shape = (24, 12, 12) if nd == 3 else (24, 12, 12, 4)
    bounds = [(0, 7), (7, 8), (8, 16), (16, 24)]
    inside = numpy.zeros(shape, bool)
    inside[:12] = True
    fg = numpy.zeros(shape, bool)
    fg[0] = True
    bg = numpy.zeros(shape, bool)
    bg[-1] = True
    c = weak_boundary_case(shape, inside, fg, bg, seed=nd)
    rng = numpy.random.default_rng(nd)
    before = steps_for(shape, bounds, 6)
    before = [[("s", stroke_ids(shape, [7, 8, 15, 16], rng), None)], [(op[0],) + tuple(
        numpy.round(x) if isinstance(x, numpy.ndarray) and x.dtype == numpy.float64 else x for x in op[1:])
        for op in before[2]]]
    run_steps(c, bounds, protocol, "caps", [[("s", None, stroke_ids(shape, [8], rng))]], exact=True, before=before)


@pytest.mark.parametrize("protocol", PROTOCOLS)
def test_edit_in_one_slab_moves_the_cut_in_another(protocol):
    """The cut lies on the lower border of slab 2.  A fg stroke deep in slab 0 leaves it there; raising the weak arcs
    across that border, listed from their upper ends, moves it into slab 2 or beyond."""
    shape = (24, 16, 18)
    bounds = _bounds(shape[0], 4)
    z0 = bounds[2][0]
    inside = numpy.zeros(shape, bool)
    inside[:z0] = True
    fg = numpy.zeros(shape, bool)
    fg[0] = True
    bg = numpy.zeros(shape, bool)
    bg[-1] = True
    c = weak_boundary_case(shape, inside, fg, bg, seed=z0)
    lo, hi = axis0_pairs(shape, [z0 - 1])
    steps = [[("s", _flat(shape, 2, 3, 3) + numpy.arange(4), None)], [("n", hi, lo, 3000.0, 3000.0)]]
    s, (e, m) = run_steps(c, bounds, protocol, "caps", steps, exact=True)
    assert m[z0].all() and not m[-1].any()


@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("bounds", [[(0, 48)], [(0, 24), (24, 48)]])
def test_sink_link_inside_a_settled_region(bounds, protocol):
    """An easy instance on slabs of >= 64 tiles (sink links everywhere but a small cube across the border), so later
    relabels reset only the tiles written since the last one.  After the solve the cube holds stranded excess at
    labels nothing rewrites; a bg seed inside it adds a sink link there, which only a full relabel reset after the fold
    lets the next solve see."""
    shape = (48, 40, 40)
    inside = numpy.zeros(shape, bool)
    inside[20:28, 16:24, 16:24] = True
    fg = numpy.zeros(shape, bool)
    fg[23:25, 19:21, 19:21] = True
    c = weak_boundary_case(shape, inside, fg, ~inside, seed=67)
    steps = [[("s", None, numpy.array([_flat(shape, 21, 17, 17), _flat(shape, 26, 22, 18)]))]]
    s, (e, m) = run_steps(c, bounds, protocol, "caps", steps, exact=True)
    assert not m[21, 17, 17] and not m[26, 22, 18] and m[fg].all()


# ------------------------------------------------------------------------------------------------------
# ghost entries change nothing
# ------------------------------------------------------------------------------------------------------
def _ghost_only(s, rng):
    """Per slab: edits in its local ids that lie in its ghost planes only (seeds, t-link lists and dense t-links, pairs
    inside a ghost plane, and the ghost-tail direction of the pairs across each border)."""
    P = int(numpy.prod(s.shape[1:]))
    out = []
    for r in range(s.n):
        a, b = _span(s, r)
        nloc = (b - a) * P
        z0, z1 = s.bounds[r]
        ghosts = ([0] if z0 > 0 else []) + ([b - a - 1] if z1 < s.shape[0] else [])
        ops = []
        for gz in ghosts:
            ids = gz * P + numpy.flatnonzero(rng.random(P) < 0.3)
            ops.append(("s", ids[::2], ids[1::2]))
            ops.append(("t", ids, rng.random(ids.size) * 50.0 - 25.0, rng.random(ids.size) * 50.0))
            lo = gz * P + numpy.arange(P)
            lo = lo[(lo % s.shape[-1]) + 1 < s.shape[-1]]
            ops.append(("n", lo, lo + 1, 40.0, 40.0))
            dsrc = numpy.zeros(nloc)
            dsrc[gz * P:(gz + 1) * P] = 30.0
            ops.append(("t", None, dsrc, 0.5 * dsrc))
            loc_shape = (b - a,) + s.shape[1:]
            f, bw = numpy.zeros(loc_shape), numpy.zeros(loc_shape)
            f[gz] = 40.0                           # last axis: pairs inside the ghost plane
            ops.append(("d", len(s.shape) - 1, f, bw))
            f0, b0 = numpy.zeros(loc_shape), numpy.zeros(loc_shape)
            if gz == 0:
                f0[0] = 60.0                       # ghost -> first owned plane: the neighbour's arc
            else:
                b0[gz - 1] = 60.0                  # ghost -> last owned plane
            ops.append(("d", 0, f0, b0))
        out.append(ops)
    return out


def _apply_raw(h, op):
    k = op[0]
    c = numpy.ascontiguousarray
    if k == "s":
        h.add_seeds(c(op[1], numpy.int64), c(op[2], numpy.int64))
    elif k == "t":
        ids = None if op[1] is None else c(op[1], numpy.int64)
        n = op[2].size if ids is None else ids.size
        h.add_tweights_warm(ids, c(numpy.broadcast_to(op[2], (n,)), numpy.float64), c(numpy.broadcast_to(op[3], (n,)), numpy.float64))
    elif k == "n":
        m = op[1].size
        h.add_nweights_warm(c(op[1], numpy.int64), c(op[2], numpy.int64), numpy.full(m, float(op[3])), numpy.full(m, float(op[4])))
    else:
        h.add_nweights_dense_warm(op[1], c(op[2]), c(op[3]))


@pytest.mark.parametrize("protocol", PROTOCOLS)
@pytest.mark.parametrize("nd,debug", [(3, False), (3, True), (4, False)])
def test_ghost_entries_change_nothing(nd, debug, protocol):
    shape = (26, 16, 18) if nd == 3 else (20, 12, 16, 5)
    bounds = [(0, 9), (9, 10), (10, 17), (17, shape[0])]
    c = voxel_case(shape, seed=37)
    with _env(**(dict(MEDPY_GC_DEBUG=1) if debug else {})):
        s = _make("slabs", shape, bounds, c, "fused" if nd == 3 else "terms")
        e0, m0 = s.solve(protocol)
        check(e0, m0, c)
        for r, ops in enumerate(_ghost_only(s, numpy.random.default_rng(nd))):
            for op in ops:
                _apply_raw(s.hs[r], op)
        e1, m1 = s.solve(protocol)
        assert e1.hex() == e0.hex() and numpy.array_equal(m1, m0)


# ------------------------------------------------------------------------------------------------------
# refusals leave the slabs as they were
# ------------------------------------------------------------------------------------------------------
def _solved(protocol, warm=True, shape=(24, 16, 18), bounds=None):
    bounds = bounds or _bounds(shape[0], 3)
    c = voxel_case(shape, seed=43)
    s = Slabs(shape, bounds)
    if warm:
        for h in s.hs:
            h.set_option(_opt_warm(), 1)
    s.build(c, "fused")
    return s, c, s.solve(protocol)


@pytest.mark.parametrize("protocol", PROTOCOLS)
def test_refusals_leave_the_slabs_unchanged(protocol):
    s, c, (e0, m0) = _solved(protocol)
    shape = s.shape
    n = int(numpy.prod(shape))
    P = int(numpy.prod(shape[1:]))
    lo, hi = axis0_pairs(shape, [s.bounds[1][0] - 1])
    for r in range(s.n):
        a, b = _span(s, r)
        nloc = (b - a) * P
        h = s.hs[r]
        # n-link decrements: refused on every slab handle, whatever the pairs (none at all included)
        for call in (lambda: h.remove_nweights_warm(lo[:4] - a * P, hi[:4] - a * P, numpy.ones(4), numpy.ones(4)),
                     lambda: h.remove_nweights_warm(numpy.zeros(0, numpy.int64), numpy.zeros(0, numpy.int64),
                                                    numpy.zeros(0), numpy.zeros(0)),
                     lambda: h.remove_nweights_dense_warm(0, numpy.zeros((b - a,) + shape[1:]),
                                                          numpy.zeros((b - a,) + shape[1:]))):
            with pytest.raises(RuntimeError, match="z-slab"):
                call()
        with pytest.raises(ValueError, match="range"):
            h.add_seeds(numpy.array([0, nloc], numpy.int64), None)
        with pytest.raises(ValueError, match="range"):
            h.add_tweights_warm(numpy.array([-1], numpy.int64), numpy.ones(1), numpy.ones(1))
        with pytest.raises(ValueError, match="neighbours"):
            h.add_nweights_warm(numpy.array([0], numpy.int64), numpy.array([2], numpy.int64), numpy.ones(1), numpy.ones(1))
        # NaN in a ghost plane (and in an owned one): refused as on one GPU
        bad = numpy.zeros(nloc)
        bad[0 if r > 0 else nloc - 1] = numpy.nan
        with pytest.raises(ValueError, match="NaN"):
            h.add_tweights_warm(None, bad, numpy.zeros(nloc))
        dn = numpy.zeros((b - a,) + shape[1:])
        dn[0, 0, 0] = numpy.nan
        with pytest.raises(ValueError, match="NaN"):
            h.add_nweights_dense_warm(1, dn, numpy.zeros_like(dn))
        with pytest.raises(ValueError, match="NaN"):
            h.add_nweights_warm(numpy.array([0], numpy.int64), numpy.array([1], numpy.int64),
                                numpy.array([numpy.nan]), numpy.ones(1))
        # the option after the first solve
        with pytest.raises(RuntimeError, match="MGC_OPT_WARM"):
            h.set_option(_opt_warm(), 0)
    e1, m1 = s.solve(protocol)
    assert e1.hex() == e0.hex() and numpy.array_equal(m1, m0)
    check(e1, m1, c)
    assert all(h.stats()["seed_folds"] == 0 for h in s.hs)
    assert n == m1.size


@pytest.mark.parametrize("protocol", PROTOCOLS)
def test_slabs_without_the_option_refuse(protocol):
    s, c, (e0, m0) = _solved(protocol, warm=False)
    with pytest.raises(RuntimeError, match="MGC_OPT_WARM"):
        apply_local(s, 1, ("s", numpy.arange(10), None))
    with pytest.raises(RuntimeError, match="MGC_OPT_WARM"):
        s.hs[1].set_option(_opt_warm(), 1)
    e1, m1 = s.solve(protocol)
    assert e1.hex() == e0.hex() and numpy.array_equal(m1, m0)


@pytest.mark.parametrize("protocol", PROTOCOLS)
def test_reset_and_rebuild_after_warm_edits_equals_fresh_handles(protocol):
    """The option survives reset(); a rebuild after warm edits solves and folds like fresh warm handles."""
    shape = (24, 16, 18)
    bounds = [(0, 7), (7, 8), (8, 24)]
    a = voxel_case(shape, seed=47)
    b = voxel_case(shape, seed=53, kind="difference_division", regional=False)
    steps = steps_for(shape, bounds, 8)
    s = _make("slabs", shape, bounds, a, "fused")
    s.solve(protocol)
    apply(s, steps[0] + steps[2])
    s.solve(protocol)
    s.reset()
    # after reset(): the decrements are still refused, and the option stays set
    with pytest.raises(RuntimeError, match="z-slab"):
        s.hs[0].remove_nweights_warm(numpy.zeros(0, numpy.int64), numpy.zeros(0, numpy.int64), numpy.zeros(0), numpy.zeros(0))
    s.build(b, "fused")
    got = [s.solve(protocol)]
    fresh = _make("slabs", shape, bounds, b, "fused")
    want = [fresh.solve(protocol)]
    for x in (s, fresh):
        apply(x, steps[1])
    got.append(s.solve(protocol))
    want.append(fresh.solve(protocol))
    for g, w in zip(got, want):
        assert g[0].hex() == w[0].hex() and numpy.array_equal(g[1], w[1])
    check(got[1][0], got[1][1], edited(b, [steps[1]]))


# ------------------------------------------------------------------------------------------------------
# SlabSolver on one rank, and over NCCL
# ------------------------------------------------------------------------------------------------------
def test_slab_solver_one_rank_warm(monkeypatch):
    """SlabSolver(warm=True) with one rank: global arguments, numpy and CUDA tensors, through the host loop."""
    import torch
    from medpy_b200.distributed import SlabSolver
    shape = (20, 16, 18)
    c = voxel_case(shape, seed=59)
    s = SlabSolver(shape, rank=0, world=1, warm=True)
    L = s.local_slice
    s.build(L(c["fg"]).view(numpy.uint8), L(c["bg"]).view(numpy.uint8), image_local=L(c["image"]), kind=c["kind"],
            sigma=c["sigma"], prob_local=L(c["prob"]), alpha=c["alpha"])
    s.solve()
    one = _make("single", shape, [(0, shape[0])], c, "fused")
    one.solve()
    steps = steps_for(shape, [(0, 10), (10, 20)], 10)
    cuda = lambda x: torch.from_numpy(numpy.ascontiguousarray(x)).cuda() if isinstance(x, numpy.ndarray) else x  # noqa: E731
    done = []
    for k, step in enumerate(steps):
        for op in step:
            args = [cuda(x) for x in op[1:]] if k % 2 else list(op[1:])
            {"s": s.add_seeds, "r": s.remove_seeds, "t": s.add_tweights_warm, "n": s.add_nweights_warm,
             "d": s.add_nweights_dense_warm}[op[0]](*args)
        apply(one, step)
        done.append(step)
        e = s.solve()
        m = s.mask()
        _same((e, m), one.solve(), False)
        check(e, m, edited(c, done))
    assert not hasattr(s, "remove_nweights_warm")


def test_multi_gpu_nccl_warm_seeds(tmp_path):
    """All visible GPUs (>= 2): build -> solve -> add_seeds -> solve through mgc_slab_solve, against one GPU."""
    import subprocess
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs at least 2 GPUs")
    shape = (48, 40, 40)
    out = str(tmp_path / "r0.npz")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(min(ngpu, 4)),
           "--master-addr", "127.0.0.1", "--master-port", "29619", os.path.join(root, "tests", "slab_warm_worker.py"),
           "x".join(map(str, shape)), out]
    subprocess.run(cmd, check=True, timeout=600)
    got = numpy.load(out)
    from slab_warm_worker import stroke, volume
    c = volume(shape)
    one = _make("single", shape, [(0, shape[0])], c, "fused")
    e0, m0 = one.solve()
    apply(one, [("s", stroke(shape), None)])
    e1, m1 = one.solve()
    assert numpy.array_equal(got["mask0"], m0) and abs(float(got["energy0"]) - e0) <= 1e-9 * abs(e0)
    assert numpy.array_equal(got["mask1"], m1) and abs(float(got["energy1"]) - e1) <= 1e-9 * abs(e1)
