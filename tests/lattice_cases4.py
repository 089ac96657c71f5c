"""Seeded 4-D lattice instances for the 4-D tile solver (4 x 4 x 8 x 4 tiles, gc_tiles4.cuh): several tiles along the last
axis (neighbour tiles, halos, cross-face pushes and wake-ups across axis-3 faces), every extent class of the tile shape,
every kernel of the last axis' row sweep, instances on both sides of the 64-tile threshold below which the solver never
classifies an instance or sweeps, and both classifications.  No tests live here (test_lattice_cases4.py checks the
generators on the CPU, test_gpu_solver4_matrix.py solves them on the GPU).

Every instance is a dict in the layout of lattice_cases.py: ``name``, ``family``, ``kind`` (``"fused"``: ``vol`` holds
graph_from_voxels' inputs; ``"dense"``: ``src`` / ``snk`` / ``there`` / ``back`` for GCGraph.set_tweights_dense /
set_nweights_dense over four axes), ``prob`` (the BK solvers' input), ``exact``, ``easy`` and the geometry ``path``
(voxel ids of a tube's centre line, sink end last) and ``no_sink``.  Fused instances also carry ``boundary`` (the
boundary term's name).
"""
import math

import numpy

import lattice_cases as lc

TILE4 = (4, 4, 8, 4)
SWEEP_SHORT = 32        # the last axis' row sweep: one thread per row up to this extent (k_sweep_rows_short) ...
SWEEP_ROW_MAX = 1024    # ... one warp per row up to this one, segments with a carry beyond it (k_sweep_rows)


def tiles_per_axis(shape):
    return tuple(math.ceil(s / e) for s, e in zip(shape, TILE4))


def tiles4(shape):
    return int(numpy.prod(tiles_per_axis(shape)))


def row_kernel(shape):
    """The kernel that sweeps the rows of the last axis on a hard instance."""
    x = shape[-1]
    return "none" if x < 2 else "short" if x <= SWEEP_SHORT else "warp" if x <= SWEEP_ROW_MAX else "segmented"


def easy_by_default4(prob):
    """The solver's rule on 4 x 4 x 8 x 4 tiles: hard when more than 1/8 of the tiles hold a voxel without a sink link
    (the first relabel's worklist; every voxel here has residual out-arcs), easy otherwise."""
    shape = tuple(prob["shape"])
    unlabelled = numpy.asarray(prob["tr"]).reshape(shape) >= 0
    u = numpy.pad(unlabelled, [(0, -s % e) for s, e in zip(shape, TILE4)])
    nt = tiles_per_axis(shape)
    per_tile = u.reshape(nt[0], 4, nt[1], 4, nt[2], 8, nt[3], 4).any(axis=(1, 3, 5, 7))
    return int(per_tile.sum()) <= tiles4(shape) // 8


def _fused(name, family, vol, boundary="difference_exponential", **extra):
    from oracle import energy_terms as et
    assert vol["fg"].ndim == 4
    regional = (vol["prob"], vol["alpha"]) if vol.get("prob") is not None else None
    prob = et.build_problem(vol["fg"], vol["bg"], regional=regional, boundary=(boundary, vol["image"], vol["sigma"], False))
    return dict(dict(path=None, no_sink=False), name=name, family=family, kind="fused", vol=vol, boundary=boundary,
                prob=prob, exact=False, easy=easy_by_default4(prob), **extra)


def _dense(name, family, shape, t, there, back, exact, **extra):
    """t: net t-link per voxel (positive: source link); there / back: per-axis arc capacities p -> p+e_d / p+e_d -> p."""
    from oracle import energy_terms as et
    assert len(shape) == 4
    src = numpy.maximum(t, 0.0).ravel()
    snk = numpy.maximum(-t, 0.0).ravel()
    tr = numpy.zeros(src.size)
    flow = et.add_tweights_pass(tr, 0.0, src, snk)
    zeros = numpy.zeros(src.size, numpy.uint8)
    prob = dict(shape=tuple(shape), wf=et.dense_axis_arrays(shape, there), wb=et.dense_axis_arrays(shape, back),
                tr=tr, flow_const=flow, fg=zeros, bg=zeros, src=src, snk=snk)
    return dict(dict(path=None, no_sink=False), name=name, family=family, kind="dense", src=src, snk=snk, there=there,
                back=back, prob=prob, exact=exact, easy=easy_by_default4(prob), **extra)


# --------------------------------------------------------------------------------------------------- G / H: geometry
def _blobs(shape, seed, with_prob):
    """synthetic.two_blob_volume on `shape`; an axis of extent 1 is the middle plane of a 3-wide volume, so that a blob
    still crosses the lattice (the blobs of an extent-1 axis would be empty)."""
    from medpy_b200 import synthetic
    full = tuple(3 if s == 1 else s for s in shape)
    vol = synthetic.two_blob_volume(full, seed=seed, with_prob=with_prob)
    if full != shape:
        sl = tuple(slice(1, 2) if s == 1 else slice(None) for s in shape)
        vol = {k: (numpy.ascontiguousarray(v[sl]) if isinstance(v, numpy.ndarray) else v) for k, v in vol.items()}
        vol["sigma"] = lc._sigma(vol["image"])
    if not with_prob:
        vol["prob"] = None
    return vol


GEOMETRY = {
    # name: shape -- extents mod (4, 4, 8, 4), the row kernel of the last axis, the tile count
    "g-13x10x19x9": (13, 10, 19, 9),        # every axis ragged, nt (4, 3, 3, 3) = 108
    "g-10x15x21x14": (10, 15, 21, 14),      # 144 tiles
    "g-7x9x12x33": (7, 9, 12, 33),          # nt[3] = 9, warp rows
    "g-16x12x16x32": (16, 12, 16, 32),      # every axis a multiple of the tile, the short-row limit
    "g-6x5x9x1030": (6, 5, 9, 1030),        # 2064 tiles, rows of two segments
    "g-1x24x40x12": (1, 24, 40, 12),        # extent-1 axes
    "g-28x1x24x16": (28, 1, 24, 16),
    "g-20x16x1x20": (20, 16, 1, 20),
    "g-32x24x16x1": (32, 24, 16, 1),        # no row sweep
    "g-24x20x30x3": (24, 20, 30, 3),        # one partial tile along the last axis
    "g-9x7x11x6": (9, 7, 11, 6),            # 24 tiles: never classified, never swept
}
HARD = ["g-13x10x19x9", "g-7x9x12x33", "g-16x12x16x32", "g-6x5x9x1030"]


def geometry(name, regional=True):
    """G: regional + difference_exponential two-blob volumes: sink links everywhere but in the blobs, so the instance
    is easy by default where the blobs reach at most 1/8 of the tiles.  H (regional=False): the boundary-only version
    (sink links only on the marker shell), hard by default."""
    shape = GEOMETRY[name]
    vol = _blobs(shape, seed=800 + sorted(GEOMETRY).index(name), with_prob=regional)
    return _fused(name if regional else "h" + name[1:], "G" if regional else "H", vol)


MULTISPECTRAL = {"h-ms-16x12x16x9": (16, 12, 16, 9), "h-ms-8x8x16x33": (8, 8, 16, 33)}


def multispectral(name):
    """H: boundary_maximum_exponential on a multi-spectral volume (channel axis last, linked like the others) with 9 and
    33 channels: short and warp rows, many exact ties."""
    from medpy_b200 import synthetic
    vol = synthetic.multispectral_volume(MULTISPECTRAL[name], seed=850 + sorted(MULTISPECTRAL).index(name))
    vol["prob"] = None
    return _fused(name, "H", vol, boundary="maximum_exponential")


# ------------------------------------------------------------------------------------------------- L: deep labels
# a serpentine whose legs run along all four axes, both ways; centre lines at 3 mod 4 (7 mod 8 on axis 2), so a tube two
# voxels wide straddles tile faces in the three axes across a leg and tile edges / corners at the turns
SERPENTINE4 = [(3, 3, 7, 3), (3, 3, 7, 11), (3, 3, 23, 11), (11, 3, 23, 11), (11, 11, 23, 11), (11, 11, 23, 3),
               (11, 11, 7, 3), (19, 11, 7, 3), (19, 19, 7, 3), (19, 19, 7, 19), (11, 19, 7, 19), (11, 19, 23, 19),
               (11, 3, 23, 19), (19, 3, 23, 19)]


def serpentine4():
    """L: a tube two voxels wide along SERPENTINE4, 100 grey levels above the background; weak source links along it
    (p ~ 0.51), sink links around its last 4 centre-line voxels (p = 0.3) and everywhere outside it (p ~ 0.2).  Once
    the weak arcs across the wall are saturated the excess has to travel along the tube.  The lattice extends beyond
    the serpentine so that the instance is an easy one."""
    shape = (32, 32, 39, 32)
    rng = numpy.random.default_rng(900)
    line = lc._polyline(SERPENTINE4)
    tube = lc._tube_mask(shape, line, 2)
    end = lc._tube_mask(shape, line[-4:], 2)
    image = rng.normal(0.0, 10.0, size=shape).astype(numpy.float32)
    image[tube] += 100.0
    p = (0.2 + rng.uniform(-0.05, 0.05, size=shape)).astype(numpy.float32)
    p[tube] = (0.51 + rng.uniform(0.0, 0.02, size=int(tube.sum()))).astype(numpy.float32)
    p[end] = 0.3
    vol = dict(image=image, prob=p, alpha=0.1, fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool),
               sigma=lc._sigma(image))
    path = numpy.array([numpy.ravel_multi_index(q, shape) for q in line], numpy.int64)
    return _fused("l-serp4", "L", vol, path=path)


def long_tube():
    """L: a tube two voxels wide along axis 3 of an 8 x 8 x 10 x 400 lattice (centre line on the tile faces of axes 0, 1
    and 2), 100 grey levels above the background.  Source links (p = 1) on its first 8 voxels, sink links (p ~ 0.2) on
    the last 4 planes of the lattice along axis 3, no t-links anywhere else (p = 0.5).  The first relabel labels about
    400 arcs deep along axis 3, across 100 tiles, so the BFS runs as many passes across axis-3 faces, and the excess
    travels the length of the tube.  Hard by default."""
    shape = (8, 8, 10, 400)
    rng = numpy.random.default_rng(901)
    line = lc._polyline([(3, 3, 7, 0), (3, 3, 7, 399)])
    tube = lc._tube_mask(shape, line, 2)
    image = rng.normal(0.0, 10.0, size=shape).astype(numpy.float32)
    image[tube] += 100.0
    p = numpy.full(shape, 0.5, numpy.float32)
    p[lc._tube_mask(shape, line[:8], 2)] = 1.0
    p[..., -4:] = (0.2 + rng.uniform(-0.05, 0.05, size=shape[:3] + (4,))).astype(numpy.float32)
    vol = dict(image=image, prob=p, alpha=0.1, fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool),
               sigma=lc._sigma(image))
    path = numpy.array([numpy.ravel_multi_index(q, shape) for q in line], numpy.int64)
    return _fused("l-tube-axis3", "L", vol, path=path)


# ------------------------------------------------------------------------------------------- I / R: dense terms
def _random_arcs(rng, shape, draw):
    there, back = [], []
    for d in range(4):
        short = list(shape)
        short[d] -= 1
        there.append(draw(rng, short))
        back.append(draw(rng, short))
    return there, back


def integer_ties(far_sink):
    """I: n-weights drawn independently per direction from {1, 2, 3}, t-links from {-3 .. 3}: a graph with many minimum
    cuts, so the mask must be BK's bit for bit only because both take the voxels that cannot reach the sink.  Inside two
    balls the t-links are drawn from {1 .. 3}, outside from {-3 .. 1}.  far_sink=True keeps the sink links ({-3 .. 2})
    in the first tile layer along axis 3; beyond it 5 % of the voxels carry a source link of 1, up to 116 arcs from the
    nearest sink link.  Both are hard by default."""
    shape = (8, 8, 16, 120) if far_sink else (12, 12, 16, 20)
    rng = numpy.random.default_rng(950 + int(far_sink))
    if far_sink:
        t = (rng.random(shape) < 0.05).astype(numpy.float64)
        t[..., :TILE4[3]] = rng.integers(-3, 3, size=shape[:3] + (TILE4[3],))
    else:
        c = numpy.indices(shape)
        balls = (((c - numpy.reshape((4, 4, 5, 6), (4, 1, 1, 1, 1))) ** 2).sum(axis=0) <= 16) | \
                (((c - numpy.reshape((8, 8, 11, 14), (4, 1, 1, 1, 1))) ** 2).sum(axis=0) <= 25)
        t = numpy.where(balls, rng.integers(1, 4, size=shape), rng.integers(-3, 2, size=shape)).astype(numpy.float64)
    there, back = _random_arcs(rng, shape, lambda r, s: r.integers(1, 4, size=s).astype(numpy.float64))
    return _dense("i-ties-far" if far_sink else "i-ties", "I", shape, t, there, back, exact=True)


def dynamic_range():
    """R: capacities 10**U(-9, 6) on every arc and t-link (random sign), and every 81st voxel strongly source linked
    (1e6 .. 2e6) with all its arcs in 10**U(-9, -6): the source clamp and rounded subtractions over fifteen decades."""
    shape = (12, 12, 16, 24)
    rng = numpy.random.default_rng(990)
    t = 10.0 ** rng.uniform(-9, 6, size=shape) * rng.choice([-1.0, 1.0], size=shape)
    strong = numpy.zeros(shape, bool)
    strong[1::3, 1::3, 1::3, 1::3] = True
    t[strong] = rng.uniform(1e6, 2e6, size=int(strong.sum()))
    there, back = _random_arcs(rng, shape, lambda r, s: 10.0 ** r.uniform(-9, 6, size=s))
    for d in range(4):
        lo = [slice(None)] * 4
        hi = [slice(None)] * 4
        lo[d], hi[d] = slice(0, -1), slice(1, None)
        touch = strong[tuple(lo)] | strong[tuple(hi)]
        for w in (there[d], back[d]):
            w[touch] = 10.0 ** rng.uniform(-9, -6, size=int(touch.sum()))
    return _dense("r-range", "R", shape, t, there, back, exact=False)


# ------------------------------------------------------------------------------------------------------------ registry
CASES = {}
for _g in GEOMETRY:
    CASES[_g] = (lambda g=_g: geometry(g))
for _g in HARD:
    CASES["h" + _g[1:]] = (lambda g=_g: geometry(g, regional=False))
for _m in MULTISPECTRAL:
    CASES[_m] = (lambda m=_m: multispectral(m))
CASES["l-serp4"] = serpentine4
CASES["l-tube-axis3"] = long_tube
CASES["i-ties"] = lambda: integer_ties(False)
CASES["i-ties-far"] = lambda: integer_ties(True)
CASES["r-range"] = dynamic_range


def make(name):
    return CASES[name]()
