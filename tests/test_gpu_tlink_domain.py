"""The t-links of every build path against the reference, over the regional term's whole domain.

Every t-link of a voxel graph comes from ``regional_probability_map`` -- ``(p * alpha, (1 - p) * alpha)`` replayed
through ``Graph::add_tweights`` -- followed by the foreground and background markers.  The other tests drive this term
with p in about [0.15, 0.95] and alpha 0.1; here the map holds every special p (signed zeros, 1 and 0.5 with their
neighbours, subnormals, values far outside [0, 1], the dtype's extremes, infinities and NaNs), markers sit on top of
them in every combination, and alpha runs from 0 and -0 over subnormal to overflowing values, as Python floats and
ints and as numpy scalars.

  (a) every build path's t-links, read back with get_trcap before any solve, equal
      ``oracle.energy_terms.build_problem(...)["tr"]`` bit for bit (-0.0 apart from +0.0; any NaN where it has NaN);
  (b) the flow constant after maxflow() is within the order-free bound (K - 1) 2^-53 sum |m_i| of math.fsum of the K
      add_tweights minima, and is the right NaN or infinity when the minima are not all finite; so is each image's
      constant in a batch's per-image energies;
  (c) whole cuts with such t-links on the flow paths give the reference BK's mask (the real one where oracle/_ref is
      built, its restatement otherwise), and an energy within that bound plus the cut's n-links of ``cut_energy`` of
      the returned mask; the z-slab builds, whose handles are checked through their cut, give BK's mask and energy;
  (d) warm seed and t-link edits on voxels whose built t-link came from an out-of-range p are folded and match the
      from-scratch replay; after a build that held a non-finite t-link a warm seed edit is folded and matches it too.
"""
import contextlib
import math
import os
import sys

import numpy
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
MAX_T = 65535.0
PATHS_3D = {"lazy": {}, "refuse_all": {"MEDPY_GC_BUILD_REFUSE_ALL": "1"}, "eager": {"MEDPY_GC_LAZY_CAPS": "0"},
            "per_term": {"MEDPY_GC_FUSE": "0"}}
ALPHA_VALUES = (0.0, -0.0, 5e-324, 1e-30, 0.1, 1.0, -0.1, 3.4e38, 1e39, 1e300)
WORST = {"flow_const": 0.0}


def _alphas():
    import warnings
    out, seen = [], set()
    for v in ALPHA_VALUES:
        for make in (float, int, numpy.float32, numpy.float64):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                a = make(v)
            key = (type(a).__name__, numpy.asarray(a, dtype=numpy.float64).tobytes())
            if key not in seen:
                seen.add(key)
                out.append(a)
    return out


ALPHAS = _alphas()
# a spread over the kinds of alpha for the paths that are run once per alpha
FEW_ALPHAS = [0.1, -0.0, 5e-324, numpy.float32(1e39), 1e300, -0.1, numpy.float64(3.4e38), 1]


def _aid(a):
    return f"{type(a).__name__}({float(a)!r})"


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print(f"\nworst |flow_const - fsum| / bound: {WORST['flow_const']:.3g}")


# ------------------------------------------------------------------------------------------------------
# the domain
# ------------------------------------------------------------------------------------------------------
def _specials(dtype):
    dt = numpy.dtype(dtype)
    if dt.kind in "iu":
        ii = numpy.iinfo(dt)
        return numpy.array([0, 1, 2, ii.max, ii.min], dtype=dt)
    ft = dt.newbyteorder("=").type
    fi = numpy.finfo(ft)
    one, half = ft(1), ft(0.5)
    with numpy.errstate(all="ignore"):
        v = [ft(0), -ft(0), one, numpy.nextafter(one, ft(2)), numpy.nextafter(one, ft(0)), half,
             numpy.nextafter(half, ft(1)), numpy.nextafter(half, ft(0)), fi.smallest_subnormal, fi.tiny,
             ft(1e-30), ft(-1e-30), ft(1.5), ft(2), ft(-0.5), ft(1e30), fi.max, -fi.max,
             ft(numpy.inf), ft(-numpy.inf), ft(numpy.nan), numpy.array(-numpy.nan, ft)]
    return numpy.array(v, dtype=ft)


def _case(shape, dtype, seed=0):
    """(map, fg, bg, special cells): the specials four times at the head of the volume under no marker, fg, bg and both,
    sprinkled again over the rest with random markers, and p in [-1, 2] elsewhere."""
    rng = numpy.random.default_rng(seed)
    dt = numpy.dtype(dtype)
    sp = _specials(dt)
    n = int(numpy.prod(shape))
    k = sp.size
    if dt.kind in "iu":
        flat = rng.integers(0, 2, n).astype(dt.newbyteorder("="))
    else:
        flat = (rng.random(n) * 3.0 - 1.0).astype(dt.newbyteorder("="))
    fg = numpy.zeros(n, bool)
    bg = numpy.zeros(n, bool)
    head = min(4 * k, n)
    flat[:head] = numpy.tile(sp, 4)[:head]
    code = numpy.repeat(numpy.arange(4), k)[:head]
    fg[:head] = (code & 1) == 1
    bg[:head] = (code & 2) == 2
    spots = rng.choice(numpy.arange(head, n), size=min(3 * k, n - head), replace=False)
    flat[spots] = numpy.resize(sp, spots.size)
    fg[spots] = rng.random(spots.size) < 0.3
    bg[spots] = rng.random(spots.size) < 0.3
    cells = numpy.union1d(numpy.arange(min(160, n)), numpy.union1d(numpy.arange(head), spots))
    others = numpy.setdiff1d(numpy.arange(n), cells)
    cells = numpy.union1d(cells, rng.choice(others, size=min(200, others.size), replace=False))
    return flat.reshape(shape).astype(dt), fg.reshape(shape), bg.reshape(shape), cells


def _expected(prob, fg, bg, alpha):
    from oracle import energy_terms as et
    with numpy.errstate(all="ignore"):
        return et.build_problem(fg, bg, regional=(prob, alpha))


def _same_bits(got, want, what):
    got, want = numpy.asarray(got, numpy.float64), numpy.asarray(want, numpy.float64)
    nan = numpy.isnan(want)
    bad = numpy.flatnonzero((numpy.isnan(got) != nan) | (~nan & (got.view(numpy.int64) != want.view(numpy.int64))))
    assert bad.size == 0, (what, bad[:8], got[bad[:8]], want[bad[:8]])


def _read(get_trcap, cells, offset=0):
    return numpy.array([get_trcap(int(c) + offset) for c in cells])


def _single(prob, fg, bg, alpha, path="lazy"):
    import medpy_b200.graphcut as gc
    with _env(**PATHS_3D.get(path, {})):
        g = gc.graph_from_voxels(fg, bg, regional_term=gc.energy_voxel.regional_probability_map,
                                 regional_term_args=(prob, alpha))
        g.get_trcap(0)
    return g


# ------------------------------------------------------------------------------------------------------
# (a) built t-links
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("alpha", ALPHAS, ids=_aid)
def test_3d_paths(dtype, alpha):
    """The lazy, refuse-all, eager and per-term builds of a 3-D graph (n % 4 == 0: the f32x4 regional kernel on the
    per-term path)."""
    prob, fg, bg, cells = _case((12, 16, 20), dtype)
    want = _expected(prob, fg, bg, alpha)["tr"][cells]
    for path in PATHS_3D:
        with _env(**PATHS_3D[path]):
            g = _single(prob, fg, bg, alpha, path)
            _same_bits(_read(g.get_trcap, cells), want, (path, dtype, alpha))


@pytest.mark.parametrize("shape", [(997,), (31, 37), (5, 6, 7, 8), (11, 13, 7)], ids=str)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("alpha", FEW_ALPHAS, ids=_aid)
def test_other_shapes(shape, dtype, alpha):
    """1-D, 2-D, 4-D (per-term kernels) and a 3-D volume with n % 4 != 0 (the scalar regional kernel)."""
    prob, fg, bg, cells = _case(shape, dtype, seed=len(shape))
    want = _expected(prob, fg, bg, alpha)["tr"][cells]
    for path in (["lazy", "per_term"] if len(shape) == 3 else ["lazy"]):
        g = _single(prob, fg, bg, alpha, path)
        _same_bits(_read(g.get_trcap, cells), want, (shape, path, dtype, alpha))


def test_f32x4_against_scalar_kernel_on_a_misaligned_device_map():
    """The f32x4 regional kernel (n % 4 == 0 and a 16-byte aligned float32 map) against the scalar one on the same values:
    a CUDA view of the map at a 4-byte offset, which graph_from_device_arrays hands to the regional kernel in place (a
    host map is staged into an aligned buffer first, so only a device map reaches the kernel misaligned).  Without a
    boundary term the device build runs the per-term regional kernel.  n % 4 != 0 is test_other_shapes' (11, 13, 7)."""
    import torch
    from medpy_b200.graphcut.device import graph_from_device_arrays
    shape = (8, 12, 16)
    prob, fg, bg, cells = _case(shape, "float32", seed=5)
    n = prob.size
    views = {}
    for off in (0, 1):              # element offsets into a fresh (256-byte aligned) allocation
        v = torch.zeros(n + 4, dtype=torch.float32, device="cuda")[off:off + n].view(shape)
        v.copy_(torch.from_numpy(prob))
        views[off] = v
    assert views[0].data_ptr() % 16 == 0 and views[1].data_ptr() % 16 == 4
    dfg, dbg = torch.from_numpy(fg).cuda(), torch.from_numpy(bg).cuda()
    for alpha in (0.1, -0.1, numpy.float32(3.4e38), 1e-30, 1e300, -0.0):
        want = _expected(prob, fg, bg, alpha)["tr"][cells]
        for off, v in views.items():
            g = graph_from_device_arrays(dfg, dbg, prob=v, alpha=alpha)
            _same_bits(_read(g.get_trcap, cells), want, ("device map at offset", 4 * off, alpha))
        g = _single(prob, fg, bg, alpha, "per_term")          # the host map, staged aligned
        _same_bits(_read(g.get_trcap, cells), want, ("per_term host map", alpha))


@pytest.mark.parametrize("layout", ["fortran", "negative_stride", "broadcast", "big_endian"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_map_layouts(layout, dtype):
    shape = (10, 12, 14)
    prob, fg, bg, cells = _case(shape, dtype, seed=7)
    if layout == "fortran":
        m = numpy.asfortranarray(prob)
    elif layout == "negative_stride":
        m = numpy.ascontiguousarray(prob[::-1, :, ::-1])[::-1, :, ::-1]
    elif layout == "broadcast":
        m = numpy.broadcast_to(numpy.array(0.5, dtype), shape)
    else:
        m = prob.astype(prob.dtype.newbyteorder(">"))
    for alpha in (0.1, -0.1, 1e300, numpy.float32(1e-30)):
        want = _expected(m, fg, bg, alpha)["tr"][cells]
        for path in ("lazy", "per_term"):
            g = _single(m, fg, bg, alpha, path)
            _same_bits(_read(g.get_trcap, cells), want, (layout, path, dtype, alpha))


@pytest.mark.parametrize("dtype,alpha", [("float16", 0.1), ("float16", -1e300), ("uint8", 0.1), ("uint8", 1),
                                         ("int16", 0.1), ("int16", numpy.float32(0.1)), ("int32", 1e300),
                                         ("float32", numpy.float64(0.1)), ("float32", numpy.float64(1e39))])
def test_dense_fallback(dtype, alpha):
    """Maps and alphas whose products numpy forms in mixed or other dtypes go as dense arrays, formed by numpy."""
    shape = (9, 10, 12)
    prob, fg, bg, cells = _case(shape, dtype, seed=9)
    want = _expected(prob, fg, bg, alpha)["tr"][cells]
    for path in ("lazy", "per_term"):
        g = _single(prob, fg, bg, alpha, path)
        _same_bits(_read(g.get_trcap, cells), want, (dtype, path, alpha))


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_device_arrays(dtype):
    import torch
    from medpy_b200.graphcut.device import graph_from_device_arrays
    shape = (12, 10, 9)
    prob, fg, bg, cells = _case(shape, dtype, seed=11)
    for alpha in FEW_ALPHAS:
        if dtype == "float32" and isinstance(alpha, numpy.float64):
            with pytest.raises(ValueError, match="probability map"):
                graph_from_device_arrays(torch.from_numpy(fg).cuda(), torch.from_numpy(bg).cuda(),
                                         prob=torch.from_numpy(prob).cuda(), alpha=alpha)
            continue
        g = graph_from_device_arrays(torch.from_numpy(fg).cuda(), torch.from_numpy(bg).cuda(),
                                     prob=torch.from_numpy(prob).cuda(), alpha=alpha)
        want = _expected(prob, fg, bg, alpha)["tr"][cells]
        _same_bits(_read(g.get_trcap, cells), want, ("cuda", dtype, alpha))


@pytest.mark.parametrize("image_shape", [(6, 10, 12), (30, 40), (500,)], ids=str)
@pytest.mark.parametrize("dtype", ["float32", "float64", "int16"])
def test_batch_each_image_alone(image_shape, dtype):
    """Each image of a batch against the reference of that image alone, and bit for bit against graph_from_voxels on
    that image alone."""
    import medpy_b200.graphcut as gc
    B = 3
    cases = [_case(image_shape, dtype, seed=20 + b) for b in range(B)]
    if dtype == "int16":                 # maps whose 1 - p wraps are refused; keep the others
        cases = [(numpy.clip(p, -32766, None).astype(numpy.int16), f, b_, c) for p, f, b_, c in cases]
    prob = numpy.stack([c[0] for c in cases])
    fg = numpy.stack([c[1] for c in cases])
    bg = numpy.stack([c[2] for c in cases])
    img = numpy.zeros(prob.shape, numpy.float32)
    n = int(numpy.prod(image_shape))
    for alpha in FEW_ALPHAS:
        # refused: products numpy forms in float64 after rounding 1 - p in float32, or forms from an int16 map in
        # anything but float64 (a Python int or a numpy.float32 alpha)
        if dtype == "float32" and isinstance(alpha, numpy.float64) or dtype == "int16" and not isinstance(alpha, float):
            with pytest.raises(ValueError, match="probability map"):
                gc.graph_from_voxels_batch(fg, bg, img, "difference_exponential", sigma=1.0, prob=prob, alpha=alpha)
            continue
        g = gc.graph_from_voxels_batch(fg, bg, img, "difference_exponential", sigma=1.0, prob=prob, alpha=alpha)
        for b, (p, f, bb, cells) in enumerate(cases):
            want = _expected(p, f, bb, alpha)["tr"][cells]
            got = _read(g._native.get_trcap, cells, offset=b * n)
            _same_bits(got, want, ("batch", b, dtype, alpha))
            alone = _read(_single(p, f, bb, alpha).get_trcap, cells)
            _same_bits(got, alone, ("batch against the image alone", b, dtype, alpha))


# ------------------------------------------------------------------------------------------------------
# (b) the flow constant
# ------------------------------------------------------------------------------------------------------
def _minima(prob, fg, bg, alpha):
    """The minima of every add_tweights call of the build, in the reference's order, formed as graph.h forms them."""
    from oracle import energy_terms as et
    with numpy.errstate(all="ignore"):
        src, snk = et.regional_probability_tweights(prob, alpha)
        tr = numpy.zeros(src.size)
        out = []
        for s, t, where in ((src, snk, None), (MAX_T, 0.0, fg.ravel()), (0.0, MAX_T, bg.ravel())):
            idx = numpy.arange(tr.size) if where is None else numpy.flatnonzero(where)
            s = numpy.broadcast_to(numpy.asarray(s, float), tr.shape)[idx]
            t = numpy.broadcast_to(numpy.asarray(t, float), tr.shape)[idx]
            d = tr[idx]
            s2 = numpy.where(d > 0, s + d, s)
            t2 = numpy.where(d > 0, t, t - d)
            out.append(numpy.where(s2 < t2, s2, t2))
            tr[idx] = s2 - t2
    return numpy.concatenate(out)


def _check_flow_const(c, m, what):
    if numpy.isnan(m).any() or (numpy.isposinf(m).any() and numpy.isneginf(m).any()):
        assert math.isnan(c), (what, c)
        return
    if numpy.isinf(m).any():
        assert c == m[numpy.isinf(m)][0], (what, c)
        return
    try:
        a = math.fsum(numpy.abs(m))
        f = math.fsum(m)
    except OverflowError:
        a = math.inf
    if not a < sys.float_info.max:
        return       # partial sums may overflow in one order and not in another: no order-free value to hold it to
    bound = (m.size - 1) * U * a
    assert abs(c - f) <= bound, (what, c, f, bound)
    if bound > 0:
        WORST["flow_const"] = max(WORST["flow_const"], abs(c - f) / bound)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("alpha", ALPHAS, ids=_aid)
def test_flow_constant(dtype, alpha):
    """Minima of both signs and very different sizes (p > 1 next to small p), then the specials: with and without the
    non-finite cells."""
    shape = (12, 16, 20)
    prob, fg, bg, _ = _case(shape, dtype, seed=3)
    finite = prob.copy()             # the specials without the non-finite cells and the dtype's extremes, whose
    finite[~numpy.isfinite(finite)] = 2.5                    # products overflow the sum of float64 minima
    finite[numpy.abs(finite) > 1e200] = -3.0
    for p in (finite, prob):
        m = _minima(p, fg, bg, alpha)
        for path in ("lazy", "per_term"):
            g = _single(p, fg, bg, alpha, path)
            with _env(**PATHS_3D[path]):
                g.maxflow()
            _check_flow_const(g.stats()["flow_const"], m, (path, dtype, alpha, bool(numpy.isfinite(p).all())))


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("alpha", [0.1, -2.5, 1e20, numpy.float32(7.0), 1e-30], ids=_aid)
def test_batch_flow_constant_per_image(dtype, alpha):
    """A batch's per-image energies hold each image's own flow constant.  Every image's t-links have one sign (p above
    0.5 or below it, markers only on that side), so its min cut is empty and its energy is its constant alone: minima of
    both signs and very different sizes (p up to 1e30 next to p near 0.5), one image with a +inf cell and one with a NaN
    cell."""
    import medpy_b200.graphcut as gc
    shape = (6, 10, 12)
    n = int(numpy.prod(shape))
    rng = numpy.random.default_rng(17)
    a64 = float(alpha)
    # the largest p keeps every product finite in the map's dtype, so only the marked cells are non-finite
    hi = min(30.0 if dtype == "float32" else 200.0, math.log10(float(numpy.finfo(dtype).max) / abs(a64)) - 2)
    imgs, fgs, bgs = [], [], []
    for b in range(4):
        above = b % 2 == 0                    # p > 0.5: tr = (2p - 1) alpha has alpha's sign; p < 0.5: the other
        near = 0.5 + rng.uniform(0.01, 0.49, n) * (1 if above else -1)
        far = 10.0 ** rng.uniform(0.0, hi, n) * (1 if above else -1)
        p = numpy.where(rng.random(n) < 0.5, near, far).astype(dtype)
        if b == 2:
            p[5] = numpy.inf
        if b == 3:
            p[7] = numpy.nan
        src_side = above == (a64 > 0)
        mark = rng.random(n) < 0.1
        imgs.append(p.reshape(shape))
        fgs.append((mark & src_side).reshape(shape))
        bgs.append((mark & (not src_side)).reshape(shape))
    prob, fg, bg = numpy.stack(imgs), numpy.stack(fgs), numpy.stack(bgs)
    g = gc.graph_from_voxels_batch(fg, bg, numpy.zeros(prob.shape, numpy.float32), "difference_exponential", sigma=1.0,
                                   prob=prob, alpha=alpha)
    energies = g.maxflow()
    mask = g.get_mask()
    for b in range(4):
        tr = _expected(imgs[b], fgs[b], bgs[b], alpha)["tr"]
        side = tr[~numpy.isnan(tr)] > 0
        assert side.all() or not side.any(), "the case must put every t-link of an image on one side"
        if b != 3:
            assert (mask[b] == (1 if side[0] else 0)).all(), b
        _check_flow_const(float(energies[b]), _minima(imgs[b], fgs[b], bgs[b], alpha), ("batch image", b, dtype, alpha))


# ------------------------------------------------------------------------------------------------------
# (c) whole cuts
# ------------------------------------------------------------------------------------------------------
def _cut_case(shape, seed, non_finite):
    rng = numpy.random.default_rng(seed)
    n = int(numpy.prod(shape))
    image = rng.normal(0.0, 1.0, shape).astype(numpy.float32)
    prob = (rng.random(n) * 3.0 - 1.0).astype(numpy.float32)
    fg = rng.random(n) < 0.02
    bg = rng.random(n) < 0.02
    if non_finite:
        cells = rng.choice(n, 12, replace=False)
        prob[cells] = numpy.array([numpy.nan, numpy.inf, -numpy.inf] * 4, numpy.float32)
        fg[cells[:3]] = True          # some of them under markers
        bg[cells[3:6]] = True
    return image, prob.reshape(shape), fg.reshape(shape), bg.reshape(shape)


@pytest.mark.parametrize("shape", [(20, 24, 32), (40, 56), (5, 6, 7, 8)], ids=str)
@pytest.mark.parametrize("alpha", [0.5, -0.5, 3.0])
@pytest.mark.parametrize("non_finite", [False, True])
def test_whole_cut(shape, alpha, non_finite):
    import medpy_b200.graphcut as gc
    from oracle import energy_terms as et, solvers
    image, prob, fg, bg = _cut_case(shape, 31 + len(shape), non_finite)
    sigma = 1.0
    with numpy.errstate(all="ignore"):
        ref = et.build_problem(fg, bg, regional=(prob, alpha), boundary=("difference_exponential", image, sigma, False))
    _, want_m = (solvers.solve_ref(ref) if solvers.have_ref() else solvers.solve_port(ref))[:2]
    g = gc.graph_from_voxels(fg, bg, regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(prob, alpha),
                             boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(image, sigma, False))
    e = g.maxflow()
    mask = numpy.asarray(g.get_mask()).reshape(-1)
    assert numpy.array_equal(mask, numpy.asarray(want_m).reshape(-1)), (shape, alpha, non_finite)
    with numpy.errstate(all="ignore"):
        ce = et.cut_energy(ref["shape"], ref["wf"], ref["wb"], ref["tr"], ref["flow_const"], mask)
    if not math.isfinite(ce):
        assert (math.isnan(e) and math.isnan(ce)) or e == ce, (e, ce)
        return
    m = _minima(prob, fg, bg, alpha)
    tr = ref["tr"]
    scale = math.fsum(numpy.abs(m)) + math.fsum(numpy.abs(tr)) + sum(math.fsum(w) for w in ref["wf"])
    bound = (m.size + tr.size + len(shape) * tr.size) * U * scale
    assert abs(e - ce) <= bound, (e, ce, bound)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("alpha", [0.5, -0.5, 3.0])
@pytest.mark.parametrize("form", ["fused", "terms"])
@pytest.mark.parametrize("bounds", [[(0, 7), (7, 16)], [(0, 5), (5, 6), (6, 16)]], ids=["2slabs", "3slabs"])
def test_slab_builds(dtype, alpha, form, bounds):
    """The z-slab builds on one GPU, driven as test_gpu_slabs.py drives them: the fused slab build and the term-by-term
    one, with the finite specials and p in [-1, 2] on the flow paths and across the slab borders.  A slab handle's
    t-links are checked through its cut: BK's mask and energy on the whole volume."""
    from test_gpu_slabs import Slabs, check
    shape = (16, 20, 24)
    image, _, fg, bg = _cut_case(shape, 71, False)
    prob, _, _, _ = _case(shape, dtype, seed=71)
    flat = prob.reshape(-1)
    flat[~numpy.isfinite(flat) | (numpy.abs(flat) > 1e30)] = 1.75       # finite t-links: the slab solve needs them
    c = dict(shape=shape, fg=fg, bg=bg, image=image, kind="difference_exponential", sigma=1.0, spacing=False,
             norm=math.nan, prob=prob, alpha=alpha)
    s = Slabs(shape, bounds)
    s.build(c, form)
    energy, mask = s.solve("native")
    check(energy, mask, c)


# ------------------------------------------------------------------------------------------------------
# (d) warm edits
# ------------------------------------------------------------------------------------------------------
HANDLES = {"lazy": ((12, 16, 20), {}, False), "eager": ((12, 16, 20), {"MEDPY_GC_LAZY_CAPS": "0"}, True),
           "4d": ((4, 6, 7, 8), {}, True)}


def _warm_graph(shape, image, prob, fg, bg, alpha, env, enable):
    import medpy_b200.graphcut as gc
    with _env(**env):
        g = gc.graph_from_voxels(fg, bg, regional_term=gc.energy_voxel.regional_probability_map,
                                 regional_term_args=(prob, alpha),
                                 boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                 boundary_term_args=(image, 1.0, False))
        if enable:
            g.enable_warm()
    return g


@pytest.mark.parametrize("handle", list(HANDLES))
def test_warm_edits_on_out_of_range_tlinks(handle):
    """add_seeds, remove_seeds and add_tweights_warm on voxels whose built t-link came from p outside [0, 1]."""
    from oracle import energy_terms as et, solvers
    from test_gpu_warm_nweights import _apply, _replay_all
    shape, env, enable = HANDLES[handle]
    image, prob, fg, bg = _cut_case(shape, 51, False)
    prob = prob * numpy.float32(40.0)           # p in [-40, 80]: t-links far outside those of a probability
    alpha = 0.25
    p = prob.ravel()
    out = numpy.flatnonzero((p > 1) | (p < 0))
    rng = numpy.random.default_rng(3)
    pick = rng.choice(out, 60, replace=False)
    steps = [[("s", pick[:20], pick[20:30])], [("r", pick[:10], pick[20:25])],
             [("t", pick[30:60], rng.normal(0.0, 50.0, 30), rng.normal(0.0, 50.0, 30))]]
    with _env(**env):
        g = _warm_graph(shape, image, prob, fg, bg, alpha, env, enable)
        g.maxflow()
        for k in range(len(steps)):
            _apply(g, steps[k])
            e = g.maxflow()
            m = numpy.asarray(g.get_mask()).reshape(-1)
            ref = et.build_problem(fg, bg, regional=(prob, alpha), boundary=("difference_exponential", image, 1.0, False))
            scale = _replay_all(ref, steps[:k + 1])
            oe, om = solvers.solve_port(ref)[:2]
            assert numpy.array_equal(m, numpy.asarray(om).reshape(-1)), (handle, k)
            assert abs(e - oe) <= 1e-9 * max(abs(oe), scale), (handle, k, e, oe)
            st = g.stats()         # each edit was folded into the solved graph, not rebuilt
            assert st["seed_folds"] == k + 1 and st["ms_seeds"] > 0, (handle, k, st["seed_folds"])


@pytest.mark.parametrize("handle", list(HANDLES))
@pytest.mark.parametrize("cell", [math.inf, -math.inf, math.nan])
def test_warm_edits_after_a_non_finite_build(handle, cell):
    """A build that held a non-finite t-link: a warm seed edit after its solve must either raise or give the
    from-scratch replay.  Every lattice handle folds the edit (the seed fold counter moves) and matches the replay --
    mask equal, energy the replay's, or NaN / the same infinity where the replay's is -- for +inf, -inf and NaN cells
    alike; that outcome is pinned here."""
    from oracle import energy_terms as et, solvers
    from test_gpu_warm_nweights import _apply, _replay_all
    shape, env, enable = HANDLES[handle]
    image, prob, fg, bg = _cut_case(shape, 61, False)
    q = int(numpy.flatnonzero(~(fg | bg).ravel())[7])
    prob.reshape(-1)[q] = cell
    alpha = 0.5
    free = numpy.flatnonzero(~(fg | bg).ravel())
    step = [("s", free[20:25], free[30:35])]
    with _env(**env):
        g = _warm_graph(shape, image, prob, fg, bg, alpha, env, enable)
        g.maxflow()
        try:
            _apply(g, step)
            e = g.maxflow()
        except (RuntimeError, ValueError) as err:
            raise AssertionError(("the warm edit raised", handle, cell, str(err)))
        m = numpy.asarray(g.get_mask()).reshape(-1)
        assert g.stats()["seed_folds"] == 1, (handle, cell, "the edit was not folded")
    with numpy.errstate(all="ignore"):
        ref = et.build_problem(fg, bg, regional=(prob, alpha), boundary=("difference_exponential", image, 1.0, False))
        _replay_all(ref, [step])
    oe, om = solvers.solve_port(ref)[:2]
    assert numpy.array_equal(m, numpy.asarray(om).reshape(-1)), (handle, cell)
    assert (math.isnan(e) and math.isnan(oe)) or e == oe or abs(e - oe) <= 1e-9 * abs(oe), (e, oe)
