"""Warm edits on a batch of independent images (graph_from_voxels_batch(..., warm=True)): seeds, t-link calls and
n-link increments and decrements folded into the batch's state and re-solved warm.  After every maxflow() each edited
image must equal a graph_from_voxels handle of that image alone given the same edits in its own ids (mask identical,
energy within 1e-9 relative) and BK on its edited graph; every image the edit left alone must keep its mask and the
bits of its energy.  The shapes put the seams inside 8-plane solver tiles and on their boundaries (Z = 5, 8, 13; 2-D
images share every tile eight at a time).

An edit is an operation in an image's own ids, in the format of test_gpu_warm_nweights_remove.py:
  ("s", fg, bg) add_seeds, ("r", fg, bg) remove_seeds, ("t", ids, src, snk) add_tweights_warm (ids None: dense),
  ("n", i, j, cap, rev) add_nweights_warm, ("d", axis, fwd, bwd) add_nweights_dense_warm (axis of the image),
  ("rn", ...) / ("rd", ...) their removals.
A step gives each edited image one operation of the same kind; the batch gets them as one call in batch ids."""
import contextlib
import math
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_warm_nweights_remove import _apply as _apply_single, _replay  # noqa: E402

pytestmark = pytest.mark.gpu

_KIND = "difference_exponential"


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _batch(batch, shape, seed=0):
    """B images with a bright blob, foreground seeds in the blob, background seeds on the border; one sigma per image."""
    rng = numpy.random.default_rng(seed)
    grids = numpy.meshgrid(*[numpy.linspace(-1.0, 1.0, s) for s in shape], indexing="ij")
    r = numpy.sqrt(sum(g * g for g in grids))
    image = numpy.empty((batch,) + shape, numpy.float32)
    fg = numpy.zeros((batch,) + shape, bool)
    bg = numpy.zeros((batch,) + shape, bool)
    border = numpy.zeros(shape, bool)
    for ax in range(len(shape)):
        idx = [slice(None)] * len(shape)
        idx[ax] = 0
        border[tuple(idx)] = True
        idx[ax] = -1
        border[tuple(idx)] = True
    for b in range(batch):
        rad = 0.3 + 0.4 * rng.random()
        image[b] = 100.0 * (r < rad) + rng.normal(0.0, 10.0, shape)
        fg[b] = r < rad * 0.3
        if not fg[b].any():
            fg[b].flat[r.argmin()] = True
        bg[b] = border & ~fg[b]
    prob = (1.0 / (1.0 + numpy.exp(-(image - 50.0) / 15.0))).astype(numpy.float32)
    sigmas = [8.0 + 4.0 * (b % 3) for b in range(batch)]
    return dict(image=image, fg=fg, bg=bg, prob=prob, sigmas=sigmas, alpha=0.1)


def _strides(shape):
    return tuple(int(numpy.prod(shape[d + 1:])) for d in range(len(shape)))


def _single(v, b):
    import medpy_b200.graphcut as gc
    return gc.graph_from_voxels(v["fg"][b], v["bg"][b], regional_term=gc.energy_voxel.regional_probability_map,
                                regional_term_args=(v["prob"][b], v["alpha"]),
                                boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                boundary_term_args=(v["image"][b], v["sigmas"][b], False))


def _bk(v, b, ops):
    """BK on image b's graph with `ops` replayed; returns its energy, mask and the energy scale S of the replay."""
    from oracle import energy_terms as et, solvers
    prob = et.build_problem(v["fg"][b], v["bg"][b], regional=(v["prob"][b], v["alpha"]),
                            boundary=(_KIND, v["image"][b], v["sigmas"][b], False))
    scale = _replay(prob, [ops])
    e, m = solvers.solve_port(prob)[:2]
    return e, numpy.asarray(m).reshape(v["image"].shape[1:]), scale


def _op(kind, v, b, rng, added=None):
    """One edit of image b in its own ids; `added` is the ("n", ...) / ("d", ...) edit a removal takes back."""
    shape = v["image"].shape[1:]
    n = math.prod(shape)
    if kind == "s":
        return ("s", numpy.unique(rng.choice(n, 4)), numpy.unique(rng.choice(n, 3)))
    if kind == "r":
        fg, bg = numpy.flatnonzero(v["fg"][b]), numpy.flatnonzero(v["bg"][b])
        return ("r", rng.choice(fg, min(2, fg.size), replace=False), rng.choice(bg, min(5, bg.size), replace=False))
    if kind == "t":
        k = 8
        return ("t", rng.choice(n, k), rng.uniform(-30.0, 30.0, k), rng.uniform(-30.0, 30.0, k))
    if kind == "T":
        src = numpy.where(rng.random(shape) < 0.2, rng.uniform(0.0, 20.0, shape), 0.0)
        snk = numpy.where(rng.random(shape) < 0.2, rng.uniform(-20.0, 20.0, shape), 0.0)
        return ("t", None, src, snk)
    if kind == "n":
        st = _strides(shape)
        axes = [d for d in range(len(shape)) if shape[d] > 1]
        lo, hi = [], []
        while len(lo) < 12:
            p, d = int(rng.integers(n)), int(rng.choice(axes))
            if numpy.unravel_index(p, shape)[d] + 1 < shape[d]:
                lo.append(p)
                hi.append(p + st[d])
        lo, hi = numpy.array(lo), numpy.array(hi)
        flip = numpy.arange(lo.size) % 2 == 1
        cap, rev = rng.uniform(0.5, 5.0, lo.size), rng.uniform(0.5, 5.0, lo.size)
        rev[::4] = 0.0
        return ("n", numpy.where(flip, hi, lo), numpy.where(flip, lo, hi), cap, rev)
    if kind == "d":
        axis = int(rng.integers(len(shape)))
        f = numpy.where(rng.random(shape) < 0.15, rng.uniform(0.5, 4.0, shape), 0.0)
        return ("d", axis, f, 0.5 * f)
    if kind in ("rn", "rd"):
        return (kind,) + tuple(added[1:])
    raise AssertionError(kind)


def _batch_call(g, v, ops, conv=None, masks=False):
    """The edits {b: op} of one kind as one call on the batch graph, in batch ids (image b's voxel p is b * N + p)."""
    shape = v["image"].shape
    n = math.prod(shape[1:])
    bs = sorted(ops)
    kind = ops[bs[0]][0]
    cv = (lambda a: a) if conv is None else conv

    def ids(k, dtype=numpy.int64):
        parts = [numpy.asarray(ops[b][k], numpy.int64) + b * n for b in bs if ops[b][k] is not None]
        return numpy.concatenate(parts).astype(dtype) if parts else None

    def cat(k, like):
        return numpy.concatenate([numpy.broadcast_to(numpy.asarray(ops[b][k], float), numpy.shape(ops[b][like]))
                                  for b in bs])

    def dense(k):
        a = numpy.zeros(shape)
        for b in bs:
            a[b] = ops[b][k]
        return a

    if kind in ("s", "r"):
        fg, bg = ids(1), ids(2)
        if masks:
            fg, bg = (None if x is None else numpy.isin(numpy.arange(math.prod(shape)), x).reshape(shape) for x in (fg, bg))
        (g.add_seeds if kind == "s" else g.remove_seeds)(*(None if x is None else cv(x) for x in (fg, bg)))
    elif kind == "t" and ops[bs[0]][1] is None:
        g.add_tweights_warm(None, cv(dense(2)), cv(dense(3)))
    elif kind == "t":
        g.add_tweights_warm(cv(ids(1)), cv(cat(2, 1)), cv(cat(3, 1)))
    elif kind in ("n", "rn"):
        call = g.add_nweights_warm if kind == "n" else g.remove_nweights_warm
        call(cv(ids(1)), cv(ids(2)), cv(cat(3, 1)), cv(cat(4, 1)))
    else:
        axes = {ops[b][1] for b in bs}
        for axis in sorted(axes):           # one call per image axis
            part = {b: op for b, op in ops.items() if op[1] == axis}
            a = {k: numpy.zeros(shape) for k in (2, 3)}
            for b, op in part.items():
                a[2][b], a[3][b] = op[2], op[3]
            call = g.add_nweights_dense_warm if kind == "d" else g.remove_nweights_dense_warm
            call(axis + 1, cv(a[2]), cv(a[3]))


def _close(a, b):
    return abs(a - b) <= 1e-9 * abs(b) + 1e-9


class _Run:
    """A warm batch graph, one single-image graph per image and the edits each image has had so far."""

    def __init__(self, v, env=None, solve=True, bk=True):
        import medpy_b200.graphcut as gc
        self.v, self.bk = v, bk
        self.B = v["image"].shape[0]
        with _env(**(env or {})):
            self.g = gc.graph_from_voxels_batch(v["fg"], v["bg"], v["image"], _KIND, sigma=v["sigmas"], prob=v["prob"],
                                                alpha=v["alpha"], warm=True)
        self.single = {}
        self.hist = {b: [] for b in range(self.B)}
        self.e = self.m = None
        if solve:
            self.solve(range(self.B))

    def _single(self, b):
        if b not in self.single:
            self.single[b] = _single(self.v, b)
            self.single[b].maxflow()
        return self.single[b]

    def edit(self, ops, conv=None, masks=False, single=True):
        """{b: op}: one batch call, and each image's op on its single graph."""
        _batch_call(self.g, self.v, ops, conv, masks)
        for b, op in ops.items():
            self.hist[b].append(op)
            if single:
                _apply_single(self._single(b), [op])

    def solve(self, edited):
        """maxflow(); the edited images against their single graphs (and BK), the others against the last solve."""
        e, m = self.g.maxflow(), self.g.get_mask()
        assert e.shape == (self.B,) and m.shape == self.v["image"].shape
        shape = self.v["image"].shape[1:]
        for b in range(self.B):
            if b in edited:
                s = self._single(b)
                e1, m1 = s.maxflow(), numpy.asarray(s.get_mask()).reshape(shape)
                assert (m[b] == m1).all(), ("mask differs from graph_from_voxels", b, int((m[b] != m1).sum()))
                assert _close(e[b], e1), ("energy differs from graph_from_voxels", b, e[b], e1)
                if self.bk:
                    e2, m2, scale = _bk(self.v, b, self.hist[b])
                    assert (m[b] == m2).all(), ("mask differs from BK", b, int((m[b] != m2).sum()))
                    assert abs(e[b] - e2) <= 1e-9 * scale, ("energy differs from BK", b, e[b], e2)
            else:
                assert (m[b] == self.m[b]).all(), ("an image the edit left alone changed its mask", b)
                assert e[b].tobytes() == self.e[b].tobytes(), ("an image the edit left alone changed its energy", b)
        self.e, self.m = e.copy(), m.copy()
        return e, m


_SEQUENCE = ["s", "r", "t", "T", "n", "d", "rn", "rd"]


def _edited(B, k):
    """The images step k edits: about two thirds of them, a different set each step (the only image of B = 1)."""
    return [b for b in range(B) if (b + k) % 3 != 0] or [0]


def _sequence(run, seed=0, conv=None, masks=False, kinds=_SEQUENCE):
    rng = numpy.random.default_rng(seed)
    added = {}
    steps = []
    for k, kind in enumerate(kinds):
        if kind in ("rn", "rd"):
            ops = {b: _op(kind, run.v, b, rng, op) for b, op in added[kind[1]].items()}
        else:
            ops = {b: _op(kind, run.v, b, rng) for b in _edited(run.B, k)}
            if kind in ("n", "d"):
                added[kind] = ops
        run.edit(ops, conv=conv, masks=masks)
        steps.append(run.solve(set(ops)))
    return steps


SHAPES = {
    "1d_b9": (9, (100,)),
    "2d_b16": (16, (19, 45)),
    "3d_z5": (4, (5, 12, 40)),
    "3d_z8": (3, (8, 10, 33)),
    "3d_z13": (3, (13, 20, 70)),
    "b1": (1, (9, 17, 35)),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_edit_sequence(name):
    B, shape = SHAPES[name]
    _sequence(_Run(_batch(B, shape, seed=B)), seed=B)


SOLVER_OPTIONS = {
    "eager": dict(MEDPY_GC_LAZY_CAPS=0),
    "no_tma": dict(MEDPY_GC_TMA=0),
    "hard": dict(MEDPY_GC_SWEEP_FRAC=1000000),
    "easy": dict(MEDPY_GC_SWEEP_FRAC=1),
    "first_cap0": dict(MEDPY_GC_FIRST_CAP=0),
    "debug": dict(MEDPY_GC_DEBUG=1),
}


@pytest.mark.parametrize("opt", list(SOLVER_OPTIONS))
@pytest.mark.parametrize("name", ["2d_b16", "3d_z13"])
def test_solver_options(opt, name):
    B, shape = SHAPES[name]
    _sequence(_Run(_batch(B, shape, seed=B), env=SOLVER_OPTIONS[opt], bk=False), seed=B + 1)


@pytest.mark.parametrize("env", [{}, dict(MEDPY_GC_LAZY_CAPS=0)], ids=["lazy", "eager"])
def test_edits_before_the_first_maxflow(env):
    v = _batch(5, (6, 11, 36), seed=21)
    run = _Run(v, env=env, solve=False)
    rng = numpy.random.default_rng(4)
    for kind in ("s", "t", "T", "n", "d"):
        run.edit({b: _op(kind, v, b, rng) for b in (0, 2, 3)})
    run.solve(range(run.B))


def test_cuda_tensors_and_masks_give_the_same_bits():
    import torch
    v = _batch(4, (5, 12, 40), seed=8)
    host = _sequence(_Run(v, bk=False), seed=3)
    dev = _sequence(_Run(v, bk=False), seed=3, conv=lambda a: torch.as_tensor(a, device="cuda"), masks=True)
    for (e0, m0), (e1, m1) in zip(host, dev):
        assert e0.tobytes() == e1.tobytes() and (m0 == m1).all()


@pytest.mark.parametrize("env", [{}, dict(MEDPY_GC_LAZY_CAPS=0)], ids=["lazy", "eager"])
@pytest.mark.parametrize("shape", [(5, 12, 40), (19, 45), (100,)])
def test_seam_pair_is_refused(shape, env):
    """A listed pair across the seam between two images is no pair: lattice neighbours along axis 0 (stride[0] apart,
    from the last plane of image 1 to the first of image 2, which only the seam rule refuses) are refused before anything
    is written, on lazily and eagerly built batches; a real pair of the same call does not get through either.  Then an
    edit still folds as on the image alone."""
    v = _batch(4, shape, seed=2)
    run = _Run(v, env=env, bk=False)
    n = math.prod(shape)
    stride0 = n // shape[0] if len(shape) == 3 else n       # the lattice's axis-0 stride: one plane, or one 1-D / 2-D image
    lo = 2 * n - stride0 + 3                    # on the last axis-0 plane of image 1
    hi = lo + stride0                           # its axis-0 lattice neighbour, on the first plane of image 2
    inner = numpy.array([5, 6]) + n             # a real pair of image 1
    for call in (run.g.add_nweights_warm, run.g.remove_nweights_warm):
        with pytest.raises(ValueError, match="not lattice neighbours"):
            call(numpy.array([inner[0], lo]), numpy.array([inner[1], hi]), 1.0, 1.0)
        with pytest.raises(ValueError, match="not lattice neighbours"):
            call(numpy.array([hi]), numpy.array([lo]), 1.0, 0.0)
    e, m = run.g.maxflow(), run.g.get_mask()
    assert e.tobytes() == run.e.tobytes() and (m == run.m).all()
    run.edit({1: ("n", inner[:1] - n, inner[1:] - n, 2.5, 1.5)})
    run.solve({1})


@pytest.mark.parametrize("B", [1, 3])
def test_long_runs_of_one_image(B):
    """Dense folds that touch every voxel of an image: each image's run of entries spans hundreds of the per-image sum's
    chunks (t-link items, and the endpoints of an n-link removal).  Every image must still equal its single handle, and
    a second batch given the same calls must give the same bits."""
    v = _batch(B, (40, 64, 64), seed=30)
    runs = [_Run(v, bk=B == 1), _Run(v, bk=False)]
    shape = v["image"].shape[1:]
    rng = numpy.random.default_rng(5)
    src, snk = rng.uniform(0.5, 20.0, shape), rng.uniform(-20.0, 20.0, shape)
    f = rng.uniform(0.5, 4.0, shape)
    edited = [b for b in range(B) if b != 1]
    out = []
    for run in runs:
        steps = []
        for op in (("t", None, src, snk), ("d", 0, f, 0.5 * f), ("rd", 0, f, 0.5 * f), ("d", 2, f, f), ("rd", 2, f, f)):
            run.edit({b: op for b in edited})
            steps.append(run.solve(set(edited)))
        out.append(steps)
    for (e0, m0), (e1, m1) in zip(*out):
        assert e0.tobytes() == e1.tobytes() and (m0 == m1).all()


@pytest.mark.parametrize("shape", [(5, 12, 40), (19, 45)])
def test_dense_weights_on_the_last_plane_of_every_image_are_ignored(shape):
    v = _batch(4, shape, seed=6)
    run = _Run(v, bk=False)
    big = numpy.zeros(v["image"].shape)
    big[:, -1] = 1e6
    run.g.add_nweights_dense_warm(1, big, big)
    run.solve(())
    run.g.remove_nweights_dense_warm(1, big, 2.0 * big)
    run.solve(())
    run.g.add_nweights_dense_warm(1, numpy.zeros_like(big), numpy.zeros_like(big))
    run.solve(())


@pytest.mark.parametrize("shape", [(7, 16, 32), (30, 50)])
def test_seam_adversary_after_seeds(shape):
    """Constant images: every would-be seam pair has the largest weight.  Image b has foreground seeds on its last
    plane, image b + 1 background seeds on its first; then more are added next to each seam."""
    B = 6
    v = _batch(B, shape)
    v["image"][:] = 7.0
    v["fg"][:] = False
    v["bg"][:] = False
    for b in range(B):
        v["fg"][b][-1] = True
        if b:
            v["bg"][b][0] = True
    run = _Run(v)
    plane = math.prod(shape[1:])
    n = math.prod(shape)
    ops = {b: ("s", numpy.arange(n - 2 * plane, n - plane), numpy.arange(plane, 2 * plane) if b else None)
           for b in range(B)}
    run.edit(ops)
    e, _ = run.solve(set(ops))
    assert (e[1:] > 0).all()


@pytest.mark.parametrize("refuse_all", [0, 1])
def test_sigma_span_under_folds(refuse_all):
    """sigma from 1e-3 to 1e3 across the images: the folds replay each image's capacities with its own constant, on
    blocks the lean build streamed and on blocks it refused (MEDPY_GC_BUILD_REFUSE_ALL=1: all of them)."""
    v = _batch(12, (5, 16, 64), seed=7)
    v["sigmas"] = list(numpy.logspace(-3, 3, 12))
    _sequence(_Run(v, env=dict(MEDPY_GC_BUILD_REFUSE_ALL=refuse_all)), seed=12)


def test_edits_above_image_65535():
    """70 000 1-D images of 16 voxels, seven patterns: edits in images on both sides of 65 535 (more images than a grid's
    y and z extents hold) against BK on each edited image, every other image unchanged bit for bit."""
    import medpy_b200.graphcut as gc
    B, P = 70_000, 7
    pat = _batch(P, (16,), seed=13)
    idx = numpy.arange(B) % P
    v = {k: pat[k][idx] for k in ("image", "fg", "bg", "prob")}
    v["sigmas"] = [pat["sigmas"][p] for p in idx]
    v["alpha"] = pat["alpha"]
    g = gc.graph_from_voxels_batch(v["fg"], v["bg"], v["image"], _KIND, sigma=v["sigmas"], prob=v["prob"],
                                   alpha=v["alpha"], warm=True)
    e0, m0 = g.maxflow(), g.get_mask()
    edited = [3, 65_534, 65_535, 65_536, 69_999]
    keep = numpy.ones(B, bool)
    keep[edited] = False
    rng = numpy.random.default_rng(1)
    added, hist = {}, {b: [] for b in edited}
    for kind in ("s", "r", "t", "n", "rn"):
        ops = {b: _op(kind, v, b, rng, added.get(b)) for b in edited}
        if kind == "n":
            added = ops
        _batch_call(g, v, ops)
        e, m = g.maxflow(), g.get_mask()
        assert e[keep].tobytes() == e0[keep].tobytes() and (m[keep] == m0[keep]).all()
        for b in edited:
            hist[b].append(ops[b])
            e2, m2, scale = _bk(v, b, hist[b])
            assert (m[b] == m2).all() and abs(e[b] - e2) <= 1e-9 * scale, (kind, b, e[b], e2)


def test_reset_restores_the_refusals():
    """After reset() a warm batch handle refuses the folds and has no energies, as any batch handle after a reset."""
    from medpy_b200 import _lib
    v = _batch(3, (4, 8, 32))
    nat = _lib.Graph.batch([4, 8, 32], 3, -1)
    nat.set_option(_lib._mgc.OPT_WARM, 1)
    nat.build_voxel_batch(None, 0.0, False, 1, v["image"], v["sigmas"], None, [float("nan")] * 3,
                          v["fg"].view(numpy.uint8), v["bg"].view(numpy.uint8))
    nat.maxflow()
    ids = numpy.array([5], numpy.int64)
    nat.add_seeds(ids, None)
    nat.maxflow()
    assert nat.get_batch_energies().shape == (3,)
    nat.reset()
    with pytest.raises(RuntimeError, match="batch handles"):
        nat.add_seeds(ids, None)
    nat.maxflow()
    with pytest.raises(RuntimeError, match="mgc_build_voxel_batch"):
        nat.get_batch_energies()
