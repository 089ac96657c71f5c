"""Batches of independent images (graph_from_voxels_batch) against graph_from_voxels on each image alone and against BK:
every image's mask must be the single-image mask and BK's, and its energy the single-image energy within 1e-9 relative.
The shapes put the seams between images inside 8-plane solver tiles and on their boundaries (Z = 5, 8, 13; 2-D images
share every tile eight at a time), and the seam adversary would change the energies if one arc leaked across a seam."""
import contextlib
import os

import numpy
import pytest

pytestmark = pytest.mark.gpu

TERMS = ["difference_linear", "difference_exponential", "difference_division", "difference_power",
         "maximum_linear", "maximum_exponential", "maximum_division", "maximum_power"]


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
    for b in range(batch):
        rad = 0.3 + 0.4 * rng.random()
        image[b] = 100.0 * (r < rad) + rng.normal(0.0, 10.0, shape)
        fg[b] = r < rad * 0.3
        if not fg[b].any():
            fg[b].flat[r.argmin()] = True
        border = numpy.zeros(shape, bool)
        for ax in range(len(shape)):
            idx = [slice(None)] * len(shape)
            idx[ax] = 0
            border[tuple(idx)] = True
            idx[ax] = -1
            border[tuple(idx)] = True
        bg[b] = border & ~fg[b]
    prob = (1.0 / (1.0 + numpy.exp(-(image - 50.0) / 15.0))).astype(numpy.float32)
    sigmas = [8.0 + 4.0 * (b % 3) for b in range(batch)]
    return dict(image=image, fg=fg, bg=bg, prob=prob, sigmas=sigmas, alpha=0.1)


def _term_args(term, image, sigma, spacing):
    return (image, spacing) if term.endswith("linear") else (image, sigma, spacing)


def _single(v, b, term, regional, spacing):
    import medpy_b200.graphcut as gc
    kw = {}
    if regional:
        kw = dict(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=(v["prob"][b], v["alpha"]))
    g = gc.graph_from_voxels(v["fg"][b], v["bg"][b], boundary_term=getattr(gc.energy_voxel, "boundary_" + term),
                             boundary_term_args=_term_args(term, v["image"][b], v["sigmas"][b], spacing), **kw)
    e = g.maxflow()
    return e, numpy.asarray(g.get_mask()).reshape(v["image"].shape[1:])


def _bk(v, b, term, regional, spacing):
    from oracle import energy_terms as et, solvers
    prob = et.build_problem(v["fg"][b], v["bg"][b], regional=(v["prob"][b], v["alpha"]) if regional else None,
                            boundary=(term, v["image"][b], v["sigmas"][b], spacing))
    e, m, _ = solvers.solve_port(prob)
    return e, m


def _run_batch(v, term, regional, spacing, image=None, fg=None, bg=None, prob=None):
    import medpy_b200.graphcut as gc
    g = gc.graph_from_voxels_batch(v["fg"] if fg is None else fg, v["bg"] if bg is None else bg,
                                   v["image"] if image is None else image, term, sigma=v["sigmas"], spacing=spacing,
                                   prob=((v["prob"] if prob is None else prob) if regional else None),
                                   alpha=v["alpha"] if regional else None)
    e = g.maxflow()
    return e, g.get_mask()


def _close(a, b):
    return abs(a - b) <= 1e-9 * abs(b)


def _check(v, term, regional=True, spacing=False, bk=True, **kw):
    e, m = _run_batch(v, term, regional, spacing, **kw)
    B = v["image"].shape[0]
    assert e.shape == (B,) and e.dtype == numpy.float64
    assert m.shape == v["image"].shape and m.dtype == numpy.uint8
    for b in range(B):
        e1, m1 = _single(v, b, term, regional, spacing)
        assert (m[b] == m1).all(), ("mask differs from graph_from_voxels", b, int((m[b] != m1).sum()))
        assert _close(e[b], e1), (b, e[b], e1)
        if bk:
            e2, m2 = _bk(v, b, term, regional, spacing)
            assert (m[b] == m2).all(), ("mask differs from BK", b)
            assert _close(e[b], e2), (b, e[b], e2)
    return e, m


SHAPES = {
    "1d_b9": (9, (100,)),
    "2d_b37": (37, (19, 45)),
    "2d_b8": (8, (64, 64)),
    "3d_z5": (4, (5, 12, 40)),
    "3d_z8": (3, (8, 10, 33)),
    "3d_z13": (3, (13, 20, 70)),
    "b1": (1, (9, 17, 35)),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_shapes_match_single_and_bk(name):
    B, shape = SHAPES[name]
    _check(_batch(B, shape, seed=B), "difference_exponential")


def test_one_image_is_graph_from_voxels():
    import medpy_b200.graphcut as gc
    v = _batch(1, (9, 17, 35), seed=3)
    e, m = _run_batch(v, "difference_exponential", True, False)
    g = gc.graph_from_voxels(v["fg"][0], v["bg"][0], regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(v["prob"][0], v["alpha"]),
                             boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(v["image"][0], v["sigmas"][0], False))
    e1 = g.maxflow()
    assert _close(e[0], e1)
    assert (m[0] == numpy.asarray(g.get_mask()).reshape(m.shape[1:])).all()


@pytest.mark.parametrize("term", TERMS)
@pytest.mark.parametrize("regional", [False, True])
@pytest.mark.parametrize("spacing", [False, True])
def test_terms(term, regional, spacing):
    v = _batch(5, (6, 11, 36), seed=11)
    sp = (1.5, 0.75, 1.25) if spacing else False
    _check(v, term, regional=regional, spacing=sp)


@pytest.mark.parametrize("term", ["difference_exponential", "maximum_linear", "difference_power"])
def test_integer_images(term):
    v = _batch(6, (3, 10, 40), seed=5)
    v["image"] = numpy.round(v["image"]).astype(numpy.int16)
    _check(v, term, regional=False, bk=False)


@pytest.mark.parametrize("shape", [(7, 16, 32), (30, 50)])
def test_seam_adversary(shape):
    """Constant images: every would-be seam pair has the largest weight.  Image b has foreground seeds on its last
    plane (row), image b + 1 background seeds on its first: a leaked arc carries flow between them."""
    B = 6
    v = _batch(B, shape)
    v["image"][:] = 7.0
    v["fg"][:] = False
    v["bg"][:] = False
    for b in range(B):
        v["fg"][b][-1] = True
        if b:
            v["bg"][b][0] = True
    e, _ = _check(v, "difference_exponential", regional=False)
    assert e[0] == 0.0 and (e[1:] > 0).all()


def test_sigma_span_and_refused_blocks():
    """sigma from 1e-3 to 1e3 across the images: blocks fail the range test.  Building every block through the refused
    path must give the same outputs."""
    v = _batch(12, (5, 16, 64), seed=7)
    v["sigmas"] = list(numpy.logspace(-3, 3, 12))
    e0, m0 = _check(v, "difference_exponential")
    with _env(MEDPY_GC_BUILD_REFUSE_ALL=1):
        e1, m1 = _run_batch(v, "difference_exponential", True, False)
    assert (e0 == e1).all() and (m0 == m1).all()


SOLVER_OPTIONS = {
    "eager": dict(MEDPY_GC_LAZY_CAPS=0),
    "no_tma": dict(MEDPY_GC_TMA=0),
    "hard": dict(MEDPY_GC_SWEEP_FRAC=1000000),
    "easy": dict(MEDPY_GC_SWEEP_FRAC=1),
    "first_cap0": dict(MEDPY_GC_FIRST_CAP=0),
    "debug": dict(MEDPY_GC_DEBUG=1),
}


@pytest.mark.parametrize("opt", list(SOLVER_OPTIONS))
@pytest.mark.parametrize("name", ["2d_b37", "3d_z13"])
def test_solver_options(opt, name):
    B, shape = SHAPES[name]
    v = _batch(B, shape, seed=B)
    with _env(**SOLVER_OPTIONS[opt]):
        _check(v, "difference_exponential", bk=False)


def test_cuda_inputs_and_strided_batch():
    import torch
    v = _batch(6, (7, 12, 40), seed=9)
    e0, m0 = _run_batch(v, "difference_exponential", True, False)
    dev = {k: torch.from_numpy(numpy.ascontiguousarray(v[k])).cuda() for k in ("image", "fg", "bg", "prob")}
    e1, m1 = _run_batch(v, "difference_exponential", True, False, image=dev["image"], fg=dev["fg"], bg=dev["bg"],
                        prob=dev["prob"])
    assert (e0 == e1).all() and (m0 == m1).all()
    # every other image of a batch twice as large
    big = {k: torch.stack([t, torch.zeros_like(t)], dim=1).flatten(0, 1) for k, t in dev.items()}
    e2, m2 = _run_batch(v, "difference_exponential", True, False, image=big["image"][::2], fg=big["fg"][::2],
                        bg=big["bg"][::2], prob=big["prob"][::2])
    assert (e0 == e2).all() and (m0 == m2).all()


def test_warm_calls_are_refused():
    v = _batch(3, (4, 8, 32))
    import medpy_b200.graphcut as gc
    g = gc.graph_from_voxels_batch(v["fg"], v["bg"], v["image"], "difference_exponential", sigma=10.0)
    g.maxflow()
    ids = numpy.array([1], numpy.int64)
    w = numpy.array([1.0])
    calls = [lambda: g.add_seeds(ids, None), lambda: g.remove_seeds(ids, None),
             lambda: g.add_tweights_warm(ids, w, w), lambda: g.add_nweights_warm(ids, ids + 1, w, w),
             lambda: g.remove_nweights_warm(ids, ids + 1, w, w),
             lambda: g.add_nweights_dense_warm(0, numpy.zeros(v["image"].shape), numpy.zeros(v["image"].shape)),
             lambda: g.remove_nweights_dense_warm(0, numpy.zeros(v["image"].shape), numpy.zeros(v["image"].shape))]
    for call in calls:
        with pytest.raises(RuntimeError, match="batch handles"):
            call()


def test_more_images_than_a_grid_axis_holds():
    """530 000 1-D images of 16 voxels: more images than gridDim.y holds (65 535) and more 8-plane build layers than
    gridDim.z holds (530 000 / 8 > 65 535).  The images repeat seven patterns, so every image is checked against the
    single-image cut of its pattern."""
    import medpy_b200.graphcut as gc
    B, P = 530_000, 7
    v = _batch(P, (16,), seed=13)
    e_ref, m_ref = [], []
    for p in range(P):
        e1, m1 = _single(v, p, "difference_exponential", True, False)
        e_ref.append(e1)
        m_ref.append(m1)
    idx = numpy.arange(B) % P
    g = gc.graph_from_voxels_batch(v["fg"][idx], v["bg"][idx], v["image"][idx], "difference_exponential",
                                   sigma=[v["sigmas"][p] for p in idx], prob=v["prob"][idx], alpha=v["alpha"])
    e = g.maxflow()
    m = g.get_mask()
    assert (m == numpy.stack(m_ref)[idx]).all()
    want = numpy.array(e_ref)[idx]
    assert (numpy.abs(e - want) <= 1e-9 * numpy.abs(want)).all()


def test_big_endian_probability_map():
    v = _batch(4, (6, 10, 32), seed=17)
    e0, m0 = _run_batch(v, "difference_exponential", True, False)
    e1, m1 = _run_batch(v, "difference_exponential", True, False, prob=v["prob"].astype(">f4"))
    assert (e0 == e1).all() and (m0 == m1).all()


def test_energies_need_a_batch_build():
    """A batch handle that was never built, or was reset after its build, has no per-image energies to read."""
    from medpy_b200 import _lib
    nat = _lib.Graph.batch([4, 8, 32], 3, -1)
    nat.maxflow()
    with pytest.raises(RuntimeError, match="mgc_build_voxel_batch"):
        nat.get_batch_energies()
    v = _batch(3, (4, 8, 32))
    nat = _lib.Graph.batch([4, 8, 32], 3, -1)
    nat.build_voxel_batch(None, 0.0, False, 1, v["image"], v["sigmas"], None, [float("nan")] * 3,
                          v["fg"].view(numpy.uint8), v["bg"].view(numpy.uint8))
    nat.maxflow()
    assert nat.get_batch_energies().shape == (3,)
    nat.reset()
    nat.maxflow()
    with pytest.raises(RuntimeError, match="mgc_build_voxel_batch"):
        nat.get_batch_energies()
